"""micro-sam's AIS decoder (DecoderAdapter over torch_em's UNETR, instance_segmentation.py:688-735) and the post-processing of
InstanceSegmentationWithDecoder.generate (:1081-1173) on the device, through csrc/ais.cu.

The decoder's layout is read from `decoder_state` (keys as micro-sam / torch_em write them, DESIGN.md section 2):
deconv1..4 (upsampler -> conv3x3 -> BatchNorm -> ReLU), base / decoder.blocks.i / decoder_head (InstanceNorm -> conv3x3 -> ReLU,
twice), decoder.samplers.i and deconv_out (upsamplers), out_conv (1x1).  The upsampler is bilinear x2 + conv1x1 (`.conv.`) or a
2x2 / stride 2 transposed convolution (`.block.`), chosen from the decoder.samplers keys as get_unetr does.  Channel counts come
from the weight shapes; the loader checks that they chain and names any missing, extra or unsupported key.  BatchNorm (eval) is
folded into the preceding convolution in fp64.  Torch only holds the weights and buffers: every layer runs in a csrc kernel."""
from __future__ import annotations

import ctypes
from typing import Dict, Tuple

import numpy as np
import torch

from . import _lib

BN_EPS = 1e-5
IN_EPS = 1e-5
IMG_SIZE = 1024


def uses_conv_transpose(decoder_state) -> bool:
    """get_unetr (instance_segmentation.py:772): transposed convolutions iff a decoder.samplers key contains '.block.'."""
    return any(".block." in k for k in decoder_state if k.startswith("decoder.samplers"))


def _shape(sd, key):
    return tuple(sd[key].shape)


def infer_plan(decoder_state) -> Dict:
    """The channel plan of a UNETR decoder state dict.  Raises ValueError naming the key on a missing or extra key, a norm
    layer with running statistics, or channel counts that do not chain."""
    sd = decoder_state
    tr = uses_conv_transpose(sd)
    expected, optional = set(), set()

    def need(*keys):
        for k in keys:
            if k not in sd:
                raise ValueError(f"decoder_state: missing key {k!r}")
        expected.update(keys)

    def sampler(p):   # -> (cin, cout)
        if tr:
            need(p + ".block.weight", p + ".block.bias")
            s = _shape(sd, p + ".block.weight")
            if len(s) != 4 or s[2:] != (2, 2):
                raise ValueError(f"decoder_state: {p}.block.weight has shape {s}, expected [Cin, Cout, 2, 2]")
            return s[0], s[1]
        need(p + ".conv.weight", p + ".conv.bias")
        s = _shape(sd, p + ".conv.weight")
        if len(s) != 4 or s[2:] != (1, 1):
            raise ValueError(f"decoder_state: {p}.conv.weight has shape {s}, expected [Cout, Cin, 1, 1]")
        return s[1], s[0]

    def conv3(key):   # -> (cin, cout)
        need(key + ".weight", key + ".bias")
        s = _shape(sd, key + ".weight")
        if len(s) != 4 or s[2:] != (3, 3):
            raise ValueError(f"decoder_state: {key}.weight has shape {s}, expected [Cout, Cin, 3, 3]")
        return s[1], s[0]

    def deconv(p):
        cin, c = sampler(p + ".block.0")
        ci2, co = conv3(p + ".block.1.block")
        if ci2 != c:
            raise ValueError(f"decoder_state: {p}.block.1.block.weight takes {ci2} channels, the upsampler gives {c}")
        need(*(f"{p}.block.2.{n}" for n in ("weight", "bias", "running_mean", "running_var")))
        optional.add(f"{p}.block.2.num_batches_tracked")
        return cin, co

    def conv_block(p):   # -> (cin, cout, affine)
        for j in (0, 3):
            for n in ("running_mean", "running_var", "num_batches_tracked"):
                if f"{p}.block.{j}.{n}" in sd:
                    raise ValueError(f"decoder_state: {p}.block.{j}.{n}: the InstanceNorm with running statistics is not supported")
        affine = f"{p}.block.0.weight" in sd
        if affine:
            need(f"{p}.block.0.weight", f"{p}.block.0.bias", f"{p}.block.3.weight", f"{p}.block.3.bias")
        cin, c = conv3(p + ".block.1")
        c2, cout = conv3(p + ".block.4")
        if c2 != c:
            raise ValueError(f"decoder_state: {p}.block.4.weight takes {c2} channels, {p}.block.1 gives {c}")
        return cin, cout, affine

    plan = {"transposed": tr, "deconv": [], "samplers": [], "blocks": []}
    prev = None
    for i in range(1, 5):
        cin, co = deconv(f"deconv{i}")
        if prev is not None and cin != prev:
            raise ValueError(f"decoder_state: deconv{i} takes {cin} channels, deconv{i - 1} gives {prev}")
        plan["deconv"].append((cin, co))
        prev = co
    emb = plan["deconv"][0][0]
    cin, x, aff = conv_block("base")
    if cin != emb:
        raise ValueError(f"decoder_state: base.block.1.weight takes {cin} channels, deconv1 takes {emb}")
    plan["base"] = (cin, x, aff)
    n_levels = 0
    while any(k.startswith(f"decoder.samplers.{n_levels}.") for k in sd):
        n_levels += 1
    if n_levels != 3:
        raise ValueError(f"decoder_state: {n_levels} decoder levels, the UNETR decoder has 3 (decoder.samplers.0..2)")
    for i in range(3):
        si, so = sampler(f"decoder.samplers.{i}")
        if si != x:
            raise ValueError(f"decoder_state: decoder.samplers.{i} takes {si} channels, the level before gives {x}")
        skip = plan["deconv"][i][1]
        bi, bo, aff = conv_block(f"decoder.blocks.{i}")
        if bi != so + skip:
            raise ValueError(f"decoder_state: decoder.blocks.{i}.block.1.weight takes {bi} channels, the concatenation gives "
                             f"{so} + {skip}")
        plan["samplers"].append((si, so))
        plan["blocks"].append((bi, bo, aff))
        x = bo
    oi, oo = sampler("deconv_out")
    if oi != x:
        raise ValueError(f"decoder_state: deconv_out takes {oi} channels, the decoder gives {x}")
    hi, ho, aff = conv_block("decoder_head")
    z0 = plan["deconv"][3][1]
    if hi != oo + z0:
        raise ValueError(f"decoder_state: decoder_head.block.1.weight takes {hi} channels, the concatenation gives {oo} + {z0}")
    plan["deconv_out"] = (oi, oo)
    plan["head"] = (hi, ho, aff)
    need("out_conv.weight", "out_conv.bias")
    s = _shape(sd, "out_conv.weight")
    if s != (3, ho, 1, 1):
        raise ValueError(f"decoder_state: out_conv.weight has shape {s}, expected [3, {ho}, 1, 1]")
    for k in sorted(sd):
        if k not in expected and k not in optional:
            raise ValueError(f"decoder_state: unexpected key {k!r}")
    return plan


def _check_kernel_channels(plan):
    chans = [c for pair in plan["deconv"] + plan["samplers"] + [plan["deconv_out"]] for c in pair]
    chans += [c for b in plan["blocks"] + [plan["base"], plan["head"]] for c in b[:2]]
    bad = [c for c in chans if c % 64]
    if bad:
        raise NotImplementedError(f"the AIS decoder kernels take channel counts that are multiples of 64, the plan has {bad[0]}")


class UNETRDecoder:
    """The AIS decoder on the device: `__call__(z12, input_size, original_size)` maps a [B, 256, 64, 64] image embedding to the
    foreground / center distance / boundary distance maps, fp32 [B, 3, *original_size] (DecoderAdapter.forward)."""

    def __init__(self, decoder_state, device=None):
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("the AIS decoder runs on a CUDA device only")
        sd = {k: v.detach().to("cpu", torch.float64) for k, v in decoder_state.items()}
        self.plan = infer_plan(sd)
        _check_kernel_channels(self.plan)
        self.transposed = self.plan["transposed"]
        dev = self.device

        def conv3(p, bn=None):
            w, b = sd[p + ".weight"], sd[p + ".bias"]
            if bn is not None:
                s = sd[bn + ".weight"] / torch.sqrt(sd[bn + ".running_var"] + BN_EPS)
                w = w * s[:, None, None, None]
                b = (b - sd[bn + ".running_mean"]) * s + sd[bn + ".bias"]
            cout, cin = w.shape[:2]
            return (w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).to(dev, torch.bfloat16).contiguous(),   # [N][K], K-major
                    b.to(dev, torch.float32).contiguous())

        def sampler(p):
            if self.transposed:
                w, b = sd[p + ".block.weight"], sd[p + ".block.bias"]
                cin, cout = w.shape[:2]
                return (w.permute(2, 3, 1, 0).reshape(4 * cout, cin).to(dev, torch.bfloat16).contiguous(),
                        b.to(dev, torch.float32).contiguous())
            w, b = sd[p + ".conv.weight"], sd[p + ".conv.bias"]
            return (w[:, :, 0, 0].to(dev, torch.bfloat16).contiguous(), b.to(dev, torch.float32).contiguous())

        def block(p, affine):
            norm = [(sd[f"{p}.block.{j}.weight"].to(dev, torch.float32).contiguous(),
                     sd[f"{p}.block.{j}.bias"].to(dev, torch.float32).contiguous()) if affine else None for j in (0, 3)]
            return {"norm": norm, "c1": conv3(p + ".block.1"), "c2": conv3(p + ".block.4")}

        self.deconv = [{"up": sampler(f"deconv{i}.block.0"), "conv": conv3(f"deconv{i}.block.1.block", f"deconv{i}.block.2")}
                       for i in range(1, 5)]
        self.base = block("base", self.plan["base"][2])
        self.samplers = [sampler(f"decoder.samplers.{i}") for i in range(3)]
        self.blocks = [block(f"decoder.blocks.{i}", self.plan["blocks"][i][2]) for i in range(3)]
        self.deconv_out = sampler("deconv_out")
        self.head = block("decoder_head", self.plan["head"][2])
        self.out_w = sd["out_conv.weight"][:, :, 0, 0].to(dev, torch.float32).contiguous()
        self.out_b = sd["out_conv.bias"].to(dev, torch.float32).contiguous()

    # ---------------------------------------------------------------- layers
    # An activation is (bf16 NHWC tensor [B, H, W, C], statistics): the InstanceNorm partial sums the convolution that wrote it
    # computed in its epilogue, as (fp64 tensor, chunks per image), or None when the norm computes them itself.
    def _conv(self, x0, x1, wb, ks, relu, transposed=False):
        L = _lib.lib()
        B, H, W, C0 = x0.shape
        C1 = 0 if x1 is None else x1.shape[3]
        w, b = wb
        cout = b.numel()
        shape = (B, 2 * H, 2 * W, cout) if transposed else (B, H, W, cout)
        out = torch.empty(shape, device=x0.device, dtype=torch.bfloat16)
        stats = torch.empty(int(L.msam_ais_conv_stats_size(B, H, W, cout, int(transposed))) // 8, device=x0.device,
                            dtype=torch.float64)
        _lib.check(L.msam_op_ais_conv(_lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(w), _lib.ptr(b), cout, int(relu),
                                      int(transposed), _lib.ptr(out), _lib.ptr(stats), _lib.cur_stream()))
        return out, (stats, stats.numel() // (2 * B * cout))

    def _norm(self, act, gb):
        L = _lib.lib()
        x, st = act
        B, H, W, C = x.shape
        ws = torch.empty(int(L.msam_ais_instnorm_workspace(B, H * W, C)), device=x.device, dtype=torch.uint8)
        out = torch.empty_like(x)
        g, b = gb if gb is not None else (None, None)
        sp, nch = (None, 0) if st is None else (_lib.ptr(st[0]), st[1])
        _lib.check(L.msam_op_ais_instnorm(_lib.ptr(x), B, H * W, C, sp, nch, _lib.ptr(g), _lib.ptr(b), IN_EPS, _lib.ptr(ws),
                                          ws.numel(), _lib.ptr(out), _lib.cur_stream()))
        return out

    def _up2(self, x):
        B, H, W, C = x.shape
        out = torch.empty(B, 2 * H, 2 * W, C, device=x.device, dtype=torch.bfloat16)
        _lib.check(_lib.lib().msam_op_ais_upsample2(_lib.ptr(x), B, H, W, C, _lib.ptr(out), _lib.cur_stream()))
        return out, None

    def _sampler(self, x, wb):
        if self.transposed:
            return self._conv(x, None, wb, 1, False, transposed=True)
        return self._up2(self._conv(x, None, wb, 1, False)[0])   # conv1x1 commutes with bilinear x2: run it at low resolution

    def _block(self, a0, a1, blk):
        n0, n1 = blk["norm"][0], blk["norm"][1]
        if a1 is None:
            x0, x1 = self._norm(a0, n0), None
        else:   # InstanceNorm is per channel: the concatenation's two parts are normalised apart
            c0 = a0[0].shape[3]
            x0 = self._norm(a0, None if n0 is None else (n0[0][:c0].contiguous(), n0[1][:c0].contiguous()))
            x1 = self._norm(a1, None if n0 is None else (n0[0][c0:].contiguous(), n0[1][c0:].contiguous()))
        y = self._conv(x0, x1, blk["c1"], 3, True)
        return self._conv(self._norm(y, n1), None, blk["c2"], 3, True)

    def forward_maps(self, z12: torch.Tensor) -> torch.Tensor:
        """_forward_impl + sigmoid: fp32 [B, 3, 16 h, 16 w] from the embedding [B, C, h, w]."""
        if z12.dim() != 4 or z12.shape[1] != self.plan["deconv"][0][0]:
            raise ValueError(f"the decoder takes embeddings [B, {self.plan['deconv'][0][0]}, h, w], got {tuple(z12.shape)}")
        x = z12.to(self.device).permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
        zs = []
        z = x
        for d in self.deconv:
            zs.append(self._conv(self._sampler(z, d["up"])[0], None, d["conv"], 3, True))
            z = zs[-1][0]
        h = self._block((x, None), None, self.base)
        for i in range(3):
            h = self._block(self._sampler(h[0], self.samplers[i]), zs[i], self.blocks[i])
        h = self._block(self._sampler(h[0], self.deconv_out), zs[3], self.head)[0]
        B, H, W, C = h.shape
        out = torch.empty(B, 3, H, W, device=self.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_op_ais_head(_lib.ptr(h), B, H * W, C, _lib.ptr(self.out_w), _lib.ptr(self.out_b), _lib.ptr(out),
                                               _lib.cur_stream()))
        return out

    def __call__(self, z12: torch.Tensor, input_size: Tuple[int, int], original_size: Tuple[int, int]) -> torch.Tensor:
        maps = self.forward_maps(z12)
        B, _, H, W = maps.shape
        if (H, W) != (IMG_SIZE, IMG_SIZE):
            raise NotImplementedError(f"the decoder output is {H}x{W}; postprocess_masks resizes from {IMG_SIZE}x{IMG_SIZE} only")
        return resize_maps(maps, input_size, original_size)


def resize_maps(maps: torch.Tensor, input_size, original_size) -> torch.Tensor:
    """postprocess_masks after the (identity) resize to 1024: crop to input_size, bilinear to original_size."""
    B, P, H, W = maps.shape
    ih, iw = int(input_size[0]), int(input_size[1])
    oh, ow = int(original_size[0]), int(original_size[1])
    out = torch.empty(B, P, oh, ow, device=maps.device, dtype=torch.float32)
    _lib.check(_lib.lib().msam_op_ais_resize(_lib.ptr(maps.contiguous()), B * P, H, W, ih, iw, oh, ow, _lib.ptr(out),
                                             _lib.cur_stream()))
    return out


# ------------------------------------------------------------------------------------------------ post-processing
def gaussian_taps(sigma: float) -> np.ndarray:
    """vigra.gaussianSmoothing's kernel as restated in DESIGN.md section 2: exp(-k^2 / 2 sigma^2) for |k| <= floor(3 sigma + 0.5),
    normalised to sum 1; empty for sigma == 0."""
    if sigma < 0:
        raise ValueError(f"smoothing sigma {sigma} < 0")
    if sigma == 0:
        return np.zeros(0, np.float64)
    r = int(3.0 * sigma + 0.5)
    k = np.arange(-r, r + 1, dtype=np.float64)
    w = np.exp(-(k * k) / (2.0 * sigma * sigma))
    return w / w.sum()


def postprocess(fg, cd, bd, center_distance_threshold=0.5, boundary_distance_threshold=0.5, foreground_threshold=0.5,
                foreground_smoothing=1.0, distance_smoothing=1.6, min_size=0):
    """generate()'s post-processing of fp32 device maps [H, W]: -> (int32 device label image, number of ids, watershed sweeps)."""
    L = _lib.lib()
    H, W = fg.shape
    maps = [m.to(torch.float32).contiguous() for m in (fg, cd, bd)]
    tf, td = np.ascontiguousarray(gaussian_taps(foreground_smoothing)), np.ascontiguousarray(gaussian_taps(distance_smoothing))
    nbytes = int(L.msam_ais_postprocess_workspace(H, W))
    if nbytes < 0:
        raise ValueError(f"image of {H}x{W} pixels is too large for the AIS post-processing")
    ws = torch.empty(nbytes, device=fg.device, dtype=torch.uint8)
    labels = torch.empty(H, W, device=fg.device, dtype=torch.int32)
    n_ids, sweeps = ctypes.c_int(0), ctypes.c_int(0)
    dp = ctypes.POINTER(ctypes.c_double)
    _lib.check(L.msam_ais_postprocess(_lib.ptr(maps[0]), _lib.ptr(maps[1]), _lib.ptr(maps[2]), H, W,
                                      tf.ctypes.data_as(dp), len(tf) // 2, td.ctypes.data_as(dp), len(td) // 2,
                                      float(foreground_threshold), float(center_distance_threshold),
                                      float(boundary_distance_threshold), int(min_size), _lib.ptr(ws), ws.numel(),
                                      _lib.ptr(labels), ctypes.byref(n_ids), ctypes.byref(sweeps), _lib.cur_stream()))
    return labels, n_ids.value, sweeps.value


def region_props(labels: torch.Tensor, n_ids: int) -> np.ndarray:
    """int32 [n_ids, 5]: area, x0, y0, x1, y1 (inclusive) of ids 1..n_ids."""
    props = torch.empty(max(n_ids, 1), 5, device=labels.device, dtype=torch.int32)
    H, W = labels.shape
    _lib.check(_lib.lib().msam_ais_props(_lib.ptr(labels), H, W, n_ids, _lib.ptr(props), _lib.cur_stream()))
    return props[:n_ids].cpu().numpy()
