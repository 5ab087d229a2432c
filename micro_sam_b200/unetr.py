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
BN_MOMENTUM = 0.1
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


# ------------------------------------------------------------------------------------------------ kernel operands and layers
def pack_conv3x3(w, device):
    """Conv2d [Cout, Cin, 3, 3] -> msam_op_ais_conv's bf16 operand [Cout][9 Cin] (K-major, K index (ky * 3 + kx) * Cin + ci),
    converted on `device`; so are the two sampler packings below"""
    return w.permute(0, 2, 3, 1).flatten(1).to(device, torch.bfloat16).contiguous()


def pack_conv_transpose2x2(w, device):
    """ConvTranspose2d [Cin, Cout, 2, 2] -> [4 Cout][Cin], row (i * 2 + j) * Cout + co"""
    return w.permute(2, 3, 1, 0).flatten(0, 2).to(device, torch.bfloat16).contiguous()


def pack_conv1x1(w, device):
    """Conv2d [Cout, Cin, 1, 1] -> [Cout][Cin]"""
    return w[:, :, 0, 0].to(device, torch.bfloat16).contiguous()


def conv(x0, x1, w, b, ks, relu, transposed=False, stats=False):
    """msam_op_ais_conv of bf16 NHWC x0 (channel-concatenated with x1 unless it is None) with a packed weight w and fp32 bias b:
    -> bf16 NHWC out, and with `stats` (out, (fp64 epilogue partial sums, chunks per image)) for the InstanceNorm after it."""
    L = _lib.lib()
    B, H, W, C0 = x0.shape
    C1 = 0 if x1 is None else x1.shape[3]
    cout = w.shape[0] // 4 if transposed else w.shape[0]
    out = torch.empty((B, 2 * H, 2 * W, cout) if transposed else (B, H, W, cout), device=x0.device, dtype=torch.bfloat16)
    st = torch.empty(int(L.msam_ais_conv_stats_size(B, H, W, cout, int(transposed))) // 8, device=x0.device,
                     dtype=torch.float64) if stats else None
    _lib.check(L.msam_op_ais_conv(_lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(w), _lib.ptr(b), cout, int(relu),
                                  int(transposed), _lib.ptr(out), _lib.ptr(st), _lib.cur_stream()))
    return (out, (st, st.numel() // (2 * B * cout))) if stats else out


def norm(x, per_image, gamma=None, beta=None, stats=None, relu=False, run=None, keep=False):
    """msam_op_ais_norm_forward of bf16 NHWC x: InstanceNorm (per_image) or BatchNorm on batch statistics, updating the running
    statistics run = (mean, var) when given; from a convolution's epilogue `stats` when given.  -> (out, mean, rstd); mean and
    rstd (for the backward pass) only with `keep`, else None."""
    L = _lib.lib()
    B, H, W, C = x.shape
    ws = torch.empty(int(L.msam_ais_norm_workspace(B, H * W, C)), device=x.device, dtype=torch.uint8)
    out = torch.empty_like(x)
    mean = torch.empty(B * C if per_image else C, device=x.device, dtype=torch.float32) if keep else None
    rstd = torch.empty_like(mean) if keep else None
    sp, nch = (None, 0) if stats is None else (_lib.ptr(stats[0]), stats[1])
    rm, rv = (None, None) if run is None else run
    _lib.check(L.msam_op_ais_norm_forward(_lib.ptr(x), B, H * W, C, int(per_image), sp, nch, _lib.ptr(gamma), _lib.ptr(beta),
                                          IN_EPS if per_image else BN_EPS, int(relu), BN_MOMENTUM, _lib.ptr(rm), _lib.ptr(rv),
                                          _lib.ptr(ws), ws.numel(), _lib.ptr(mean), _lib.ptr(rstd), _lib.ptr(out),
                                          _lib.cur_stream()))
    return out, mean, rstd


def upsample2(x):
    """msam_op_ais_upsample2: bilinear x2 of bf16 NHWC x"""
    B, H, W, C = x.shape
    out = torch.empty(B, 2 * H, 2 * W, C, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().msam_op_ais_upsample2(_lib.ptr(x), B, H, W, C, _lib.ptr(out), _lib.cur_stream()))
    return out


def head_maps(h, w, b):
    """msam_op_ais_head: out_conv (fp32 w [3][C], b [3]) + sigmoid of bf16 NHWC h -> fp32 maps [B, 3, H, W]"""
    B, H, W, C = h.shape
    out = torch.empty(B, 3, H, W, device=h.device, dtype=torch.float32)
    _lib.check(_lib.lib().msam_op_ais_head(_lib.ptr(h), B, H * W, C, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), _lib.cur_stream()))
    return out


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
            return pack_conv3x3(w, dev), b.to(dev, torch.float32).contiguous()

        def sampler(p):
            if self.transposed:
                w, b = sd[p + ".block.weight"], sd[p + ".block.bias"]
                return pack_conv_transpose2x2(w, dev), b.to(dev, torch.float32).contiguous()
            w, b = sd[p + ".conv.weight"], sd[p + ".conv.bias"]
            return pack_conv1x1(w, dev), b.to(dev, torch.float32).contiguous()

        def block(p, affine):
            gb = [(sd[f"{p}.block.{j}.weight"].to(dev, torch.float32).contiguous(),
                   sd[f"{p}.block.{j}.bias"].to(dev, torch.float32).contiguous()) if affine else None for j in (0, 3)]
            return {"norm": gb, "c1": conv3(p + ".block.1"), "c2": conv3(p + ".block.4")}

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
    @staticmethod
    def _norm(act, gb):
        return norm(act[0], True, *(gb or (None, None)), stats=act[1])[0]

    def _sampler(self, x, wb):
        if self.transposed:
            return conv(x, None, *wb, 1, False, True, stats=True)
        return upsample2(conv(x, None, *wb, 1, False, stats=True)[0]), None   # conv1x1 commutes with bilinear x2: at low resolution

    def _block(self, a0, a1, blk):
        n0, n1 = blk["norm"][0], blk["norm"][1]
        if a1 is None:
            x0, x1 = self._norm(a0, n0), None
        else:   # InstanceNorm is per channel: the concatenation's two parts are normalised apart
            c0 = a0[0].shape[3]
            x0 = self._norm(a0, None if n0 is None else (n0[0][:c0].contiguous(), n0[1][:c0].contiguous()))
            x1 = self._norm(a1, None if n0 is None else (n0[0][c0:].contiguous(), n0[1][c0:].contiguous()))
        y = conv(x0, x1, *blk["c1"], 3, True, stats=True)
        return conv(self._norm(y, n1), None, *blk["c2"], 3, True, stats=True)

    def forward_maps(self, z12: torch.Tensor) -> torch.Tensor:
        """_forward_impl + sigmoid: fp32 [B, 3, 16 h, 16 w] from the embedding [B, C, h, w]."""
        if z12.dim() != 4 or z12.shape[1] != self.plan["deconv"][0][0]:
            raise ValueError(f"the decoder takes embeddings [B, {self.plan['deconv'][0][0]}, h, w], got {tuple(z12.shape)}")
        x = z12.to(self.device).permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
        zs = []
        z = x
        for d in self.deconv:
            zs.append(conv(self._sampler(z, d["up"])[0], None, *d["conv"], 3, True, stats=True))
            z = zs[-1][0]
        h = self._block((x, None), None, self.base)
        for i in range(3):
            h = self._block(self._sampler(h[0], self.samplers[i]), zs[i], self.blocks[i])
        h = self._block(self._sampler(h[0], self.deconv_out), zs[3], self.head)[0]
        return head_maps(h, self.out_w, self.out_b)

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


# ------------------------------------------------------------------------------------------------ training
def default_decoder_state(emb=256, feats=(512, 256, 128, 64), deconv=(256, 128, 64, 64), head_in=64, transposed=False,
                          seed=0) -> Dict[str, torch.Tensor]:
    """A freshly initialised UNETR decoder (the production plan by default) with torch's default init, drawn from
    torch.Generator().manual_seed(seed) in key order: every convolution weight and bias uniform in +-1 / sqrt(fan_in)
    (kaiming_uniform with a = sqrt(5); fan_in = weight.shape[1] * k * k, so Cout * 4 for a transposed convolution), BatchNorm
    weight 1, bias 0, running mean 0, running variance 1.  The InstanceNorms are not affine, as in torch_em's UNETR."""
    g = torch.Generator().manual_seed(seed)

    def u(shape, fan_in):
        return ((torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / fan_in ** 0.5).to(torch.float32)

    sd = {}

    def sampler(p, cin, cout):
        if transposed:
            sd[p + ".block.weight"], sd[p + ".block.bias"] = u((cin, cout, 2, 2), cout * 4), u((cout,), cout * 4)
        else:
            sd[p + ".conv.weight"], sd[p + ".conv.bias"] = u((cout, cin, 1, 1), cin), u((cout,), cin)

    def conv(p, cin, cout, k=3):
        sd[p + ".weight"], sd[p + ".bias"] = u((cout, cin, k, k), cin * k * k), u((cout,), cin * k * k)

    cin = emb
    for i, c in enumerate(deconv, 1):
        sampler(f"deconv{i}.block.0", cin, c)
        conv(f"deconv{i}.block.1.block", c, c)
        sd[f"deconv{i}.block.2.weight"], sd[f"deconv{i}.block.2.bias"] = torch.ones(c), torch.zeros(c)
        sd[f"deconv{i}.block.2.running_mean"], sd[f"deconv{i}.block.2.running_var"] = torch.zeros(c), torch.ones(c)
        sd[f"deconv{i}.block.2.num_batches_tracked"] = torch.tensor(0)
        cin = c
    conv("base.block.1", emb, feats[0])
    conv("base.block.4", feats[0], feats[0])
    for i in range(3):
        sampler(f"decoder.samplers.{i}", feats[i], feats[i + 1])
        conv(f"decoder.blocks.{i}.block.1", feats[i + 1] + deconv[i], feats[i + 1])
        conv(f"decoder.blocks.{i}.block.4", feats[i + 1], feats[i + 1])
    sampler("deconv_out", feats[3], head_in)
    conv("decoder_head.block.1", head_in + deconv[3], head_in)
    conv("decoder_head.block.4", head_in, head_in)
    conv("out_conv", head_in, 3, k=1)
    return sd


def _off(t: torch.Tensor, elems: int):
    """pointer `elems` elements into a contiguous tensor (a channel offset into an NHWC tensor)"""
    return ctypes.c_void_p(t.data_ptr() + elems * t.element_size())


class TrainableUNETRDecoder:
    """The UNETR decoder in training mode on the device.  fp32 masters, gradients and AdamW moments live in `masters` / `grads`
    keyed as `decoder_state` is; the bf16 operands of the kernels (K-major forward weights, 180-degree rotated data-gradient
    weights) are refreshed from the masters after every optimizer step.  BatchNorm runs on batch statistics and updates its
    running statistics (momentum 0.1, unbiased variance); the InstanceNorms keep none.  `forward(z12)` keeps the activations
    the backward pass needs; `backward(d_maps)` writes every parameter gradient into `grads` and returns d z12.  Every reduction
    runs in a fixed order: two identical steps give bit-identical gradients."""

    def __init__(self, decoder_state, device=None):
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("the AIS decoder trains on a CUDA device only")
        sd = {k: v.detach().to("cpu") for k, v in decoder_state.items()}
        self.plan = infer_plan(sd)
        _check_kernel_channels(self.plan)
        self.transposed = self.plan["transposed"]
        dev = self.device
        self.masters, self.buffers = {}, {}
        for k, v in sd.items():
            if k.endswith("running_mean") or k.endswith("running_var"):
                self.buffers[k] = v.to(dev, torch.float32).contiguous()
            elif k.endswith("num_batches_tracked"):
                self.buffers[k] = int(v)
            else:
                self.masters[k] = v.to(dev, torch.float32).contiguous()
        for i in range(1, 5):
            self.buffers.setdefault(f"deconv{i}.block.2.num_batches_tracked", 0)
        self.grads = {k: torch.zeros_like(v) for k, v in self.masters.items()}
        self.moments = {}
        self.steps = {k: 0 for k in self.masters}
        cmax = max(v.shape[0] * (4 if self.transposed else 1) for v in self.masters.values() if v.dim() == 1) + 512
        self._zeros = torch.zeros(cmax, device=dev, dtype=torch.float32)
        self._saved = None
        self._written = False   # a gradient since the last step / zeroing
        self.refresh()

    # ---------------------------------------------------------------- operands
    def refresh(self):
        """bf16 kernel operands from the fp32 masters: (forward weight, data-gradient weight) per convolution."""
        m, self.ops, dev = self.masters, {}, self.device
        for k, w in m.items():
            if not k.endswith(".weight") or w.dim() != 4:
                continue
            if w.shape[2:] == (3, 3):
                self.ops[k] = (pack_conv3x3(w, dev), w.flip(2, 3).permute(1, 2, 3, 0).flatten(1).to(torch.bfloat16).contiguous())
            elif k.endswith(".block.weight") and w.shape[2:] == (2, 2):   # ConvTranspose2d [Cin, Cout, 2, 2]
                self.ops[k] = (pack_conv_transpose2x2(w, dev), w.permute(0, 2, 3, 1).flatten(1).to(torch.bfloat16).contiguous())
            elif k != "out_conv.weight":   # conv1x1 of the interpolation sampler
                self.ops[k] = (pack_conv1x1(w, dev), w[:, :, 0, 0].t().to(torch.bfloat16).contiguous())
        self.out_w = m["out_conv.weight"][:, :, 0, 0].contiguous()

    # ---------------------------------------------------------------- kernels
    def _conv(self, x0, x1, w, b, ks, relu, transposed=False):
        """b None: a zero bias (the data-gradient convolutions)"""
        return conv(x0, x1, w, b if b is not None else self._zeros, ks, relu, transposed)

    def _wgrad(self, dy, x0, x1, ks):
        L = _lib.lib()
        B, H, W, cout = dy.shape
        C0, C1 = x0.shape[3], (0 if x1 is None else x1.shape[3])
        ws = torch.empty(int(L.msam_ais_wgrad_workspace(cout, C0, C1, B, H, W, ks)), device=self.device, dtype=torch.uint8)
        dw = torch.empty(cout, ks * ks * (C0 + C1), device=self.device, dtype=torch.float32)
        _lib.check(L.msam_op_ais_wgrad(_lib.ptr(dy), cout, _lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(ws), ws.numel(),
                                       _lib.ptr(dw), _lib.cur_stream()))
        return dw

    def _norm_ws(self, B, HW, C):
        return torch.empty(int(_lib.lib().msam_ais_norm_workspace(B, HW, C)), device=self.device, dtype=torch.uint8)

    def _chan_sum(self, g):
        B, H, W, C = g.shape
        ws = self._norm_ws(B, H * W, C)
        out = torch.empty(C, device=self.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_op_ais_chan_sum(_lib.ptr(g), B, H * W, C, _lib.ptr(ws), ws.numel(), _lib.ptr(out), _lib.cur_stream()))
        return out

    @staticmethod
    def _norm_fwd(x, per_image, gamma=None, beta=None, relu=False, run=None):
        """-> (out, mean, rstd)"""
        return norm(x, per_image, gamma, beta, relu=relu, run=run, keep=True)

    def _norm_bwd(self, x, dy, dy_off, ldd, mean, rstd, per_image, gamma=None, relu_out=None, in_mask=False, dx=None, out_mode=0,
                  dgb=False):
        """dy: bf16 or fp32 NHWC with row stride ldd, read from channel dy_off on; returns (dx, dgamma, dbeta)"""
        B, H, W, C = x.shape
        ws = self._norm_ws(B, H * W, C)
        if dx is None:
            dx = torch.empty(B, H, W, C, device=self.device, dtype=torch.bfloat16 if out_mode == 0 else torch.float32)
        dg = torch.empty(C, device=self.device, dtype=torch.float32) if dgb else None
        db = torch.empty(C, device=self.device, dtype=torch.float32) if dgb else None
        _lib.check(_lib.lib().msam_op_ais_norm_backward(
            _lib.ptr(x), C, _off(dy, dy_off), int(dy.dtype == torch.float32), ldd, _lib.ptr(relu_out), B, H * W, C, int(per_image),
            _lib.ptr(gamma), _lib.ptr(mean), _lib.ptr(rstd), int(in_mask), _lib.ptr(ws), ws.numel(), _lib.ptr(dx), out_mode, C,
            _lib.ptr(dg), _lib.ptr(db), _lib.cur_stream()))
        return dx, dg, db

    def _relu_mask(self, g, out):
        _lib.check(_lib.lib().msam_op_ais_relu_mask(_lib.ptr(g), _lib.ptr(out), g.numel(), _lib.cur_stream()))

    def _add(self, acc, x):
        _lib.check(_lib.lib().msam_op_ais_add_bf16(_lib.ptr(acc), _lib.ptr(x), x.numel(), _lib.cur_stream()))

    # ---------------------------------------------------------------- layers: forward saves, backward consumes
    def _sampler_fwd(self, z, p):
        key = p + (".block" if self.transposed else ".conv")
        w = self.ops[key + ".weight"][0]
        b = self.masters[key + ".bias"]
        if self.transposed:
            return self._conv(z, None, w, b, 1, False, transposed=True), (p, z)
        return upsample2(self._conv(z, None, w, b, 1, False)), (p, z)

    def _sampler_bwd(self, g, saved):
        """g: bf16 d(sampler output) -> bf16 d(sampler input)"""
        p, z = saved
        B, H, W, cin = z.shape
        L = _lib.lib()
        if self.transposed:
            key = p + ".block"
            cout = g.shape[3]
            g4 = torch.empty(B, H, W, 4 * cout, device=self.device, dtype=torch.bfloat16)
            _lib.check(L.msam_op_ais_space_to_depth(_lib.ptr(g), B, H, W, cout, _lib.ptr(g4), _lib.cur_stream()))
            dwk = self._wgrad(g4, z, None, 1)   # [4 cout][cin], row (i * 2 + j) * cout + co
            self.grads[key + ".weight"].copy_(dwk.view(2, 2, cout, cin).permute(3, 2, 0, 1))
            self.grads[key + ".bias"].copy_(self._chan_sum(g))
            return self._conv(g4, None, self.ops[key + ".weight"][1], None, 1, False)
        key = p + ".conv"
        cout = g.shape[3]
        du = torch.empty(B, H, W, cout, device=self.device, dtype=torch.bfloat16)
        _lib.check(L.msam_op_ais_upsample2_backward(_lib.ptr(g), B, H, W, cout, _lib.ptr(du), _lib.cur_stream()))
        self.grads[key + ".weight"].copy_(self._wgrad(du, z, None, 1).view(cout, cin, 1, 1))
        self.grads[key + ".bias"].copy_(self._chan_sum(du))
        return self._conv(du, None, self.ops[key + ".weight"][1], None, 1, False)

    def _deconv_fwd(self, z, i):
        p = f"deconv{i}.block"
        s, ssave = self._sampler_fwd(z, p + ".0")
        c = self._conv(s, None, self.ops[p + ".1.block.weight"][0], self.masters[p + ".1.block.bias"], 3, False)
        run = (self.buffers[p + ".2.running_mean"], self.buffers[p + ".2.running_var"])
        out, mean, rstd = self._norm_fwd(c, False, self.masters[p + ".2.weight"], self.masters[p + ".2.bias"], relu=True, run=run)
        self.buffers[p + ".2.num_batches_tracked"] += 1
        return out, (p, ssave, s, c, out, mean, rstd)

    def _deconv_bwd(self, dz, saved):
        """dz: fp32 d(block output), before its ReLU -> bf16 d(block input)"""
        p, ssave, s, c, out, mean, rstd = saved
        C = c.shape[3]
        dc, dg, db = self._norm_bwd(c, dz, 0, C, mean, rstd, False, self.masters[p + ".2.weight"], relu_out=out, dgb=True)
        self.grads[p + ".2.weight"].copy_(dg)
        self.grads[p + ".2.bias"].copy_(db)
        k = p + ".1.block"
        cout, cin = self.masters[k + ".weight"].shape[:2]
        self.grads[k + ".weight"].copy_(self._wgrad(dc, s, None, 3).view(cout, 3, 3, cin).permute(0, 3, 1, 2))
        self.grads[k + ".bias"].copy_(self._chan_sum(dc))
        ds = self._conv(dc, None, self.ops[k + ".weight"][1], None, 3, False)
        return self._sampler_bwd(ds, ssave)

    def _gb(self, p, j, lo=None, hi=None):
        k = f"{p}.block.{j}"
        if k + ".weight" not in self.masters:
            return None, None
        g, b = self.masters[k + ".weight"], self.masters[k + ".bias"]
        return (g, b) if lo is None else (g[lo:hi].contiguous(), b[lo:hi].contiguous())

    def _block_fwd(self, a0, a1, p):
        c0 = a0.shape[3]
        ctot = c0 + (0 if a1 is None else a1.shape[3])
        g, b = self._gb(p, 0, 0, c0)
        x0, m0, r0 = self._norm_fwd(a0, True, g, b)
        x1 = m1 = r1 = None
        if a1 is not None:   # InstanceNorm is per channel: the concatenation's two parts are normalised apart
            g, b = self._gb(p, 0, c0, ctot)
            x1, m1, r1 = self._norm_fwd(a1, True, g, b)
        h1 = self._conv(x0, x1, self.ops[p + ".block.1.weight"][0], self.masters[p + ".block.1.bias"], 3, True)
        g, b = self._gb(p, 3)
        n1, m2, r2 = self._norm_fwd(h1, True, g, b)
        out = self._conv(n1, None, self.ops[p + ".block.4.weight"][0], self.masters[p + ".block.4.bias"], 3, True)
        return out, (p, a0, a1, m0, r0, m1, r1, x0, x1, h1, m2, r2, n1, out)

    def _conv_grads(self, k, dy, x0, x1):
        cout, cin = self.masters[k + ".weight"].shape[:2]
        self.grads[k + ".weight"].copy_(self._wgrad(dy, x0, x1, 3).view(cout, 3, 3, cin).permute(0, 3, 1, 2))
        self.grads[k + ".bias"].copy_(self._chan_sum(dy))

    def _block_bwd(self, g, saved, masked, d_a0=None, d_a1=None):
        """g: bf16 d(block output) (`masked`: already times the output ReLU's mask; it is masked in place otherwise).
        d(a0) is returned as bf16, or added into the fp32 `d_a0`; d(a1) is stored into the fp32 `d_a1`."""
        p, a0, a1, m0, r0, m1, r1, x0, x1, h1, m2, r2, n1, out = saved
        if not masked:
            self._relu_mask(g, out)
        self._conv_grads(p + ".block.4", g, n1, None)
        dn1 = self._conv(g, None, self.ops[p + ".block.4.weight"][1], None, 3, False)
        affine = p + ".block.0.weight" in self.masters
        C = h1.shape[3]
        dh1, dg, db = self._norm_bwd(h1, dn1, 0, C, m2, r2, True, self._gb(p, 3)[0], in_mask=True, dgb=affine)
        if affine:
            self.grads[p + ".block.3.weight"].copy_(dg)
            self.grads[p + ".block.3.bias"].copy_(db)
        self._conv_grads(p + ".block.1", dh1, x0, x1)
        dx01 = self._conv(dh1, None, self.ops[p + ".block.1.weight"][1], None, 3, False)
        c0, ctot = a0.shape[3], dx01.shape[3]
        gam = self._gb(p, 0)[0]
        if d_a0 is None:
            da0, dg0, db0 = self._norm_bwd(a0, dx01, 0, ctot, m0, r0, True, None if gam is None else gam[:c0].contiguous(), dgb=affine)
        else:
            da0, dg0, db0 = self._norm_bwd(a0, dx01, 0, ctot, m0, r0, True, None if gam is None else gam[:c0].contiguous(), dx=d_a0,
                                           out_mode=2, dgb=affine)
        if a1 is not None:
            _, dg1, db1 = self._norm_bwd(a1, dx01, c0, ctot, m1, r1, True, None if gam is None else gam[c0:].contiguous(), dx=d_a1,
                                         out_mode=1, dgb=affine)
            if affine:
                dg0, db0 = torch.cat([dg0, dg1]), torch.cat([db0, db1])
        if affine:
            self.grads[p + ".block.0.weight"].copy_(dg0)
            self.grads[p + ".block.0.bias"].copy_(db0)
        return da0

    # ---------------------------------------------------------------- whole decoder
    def forward(self, z12: torch.Tensor) -> torch.Tensor:
        """training forward: the embedding [B, C, h, w] -> sigmoid maps fp32 [B, 3, 16 h, 16 w]; keeps the activations"""
        if z12.dim() != 4 or z12.shape[1] != self.plan["deconv"][0][0]:
            raise ValueError(f"the decoder takes embeddings [B, {self.plan['deconv'][0][0]}, h, w], got {tuple(z12.shape)}")
        x = z12.to(self.device).permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
        zs, dsaved = [], []
        z = x
        for i in range(1, 5):
            z, sv = self._deconv_fwd(z, i)
            zs.append(z)
            dsaved.append(sv)
        h, bsaved = self._block_fwd(x, None, "base")
        blocks, samplers = [bsaved], []
        for i in range(3):
            s, ssv = self._sampler_fwd(h, f"decoder.samplers.{i}")
            h, bsv = self._block_fwd(s, zs[i], f"decoder.blocks.{i}")
            samplers.append(ssv)
            blocks.append(bsv)
        s, osv = self._sampler_fwd(h, "deconv_out")
        h, hsv = self._block_fwd(s, zs[3], "decoder_head")
        maps = head_maps(h, self.out_w, self.masters["out_conv.bias"])
        self._saved = dict(x=x, zs=zs, deconv=dsaved, blocks=blocks, samplers=samplers, out=osv, head=hsv, h=h, maps=maps)
        return maps

    def backward(self, d_maps: torch.Tensor) -> torch.Tensor:
        """d maps [B, 3, H, W] -> d embedding fp32 [B, C, h, w]; adds the parameter gradients into `grads` (torch's accumulation
        until the next optimizer step or zero_grads)"""
        sv, self._saved = self._saved, None
        if sv is None:
            raise RuntimeError("backward without a training forward (each forward allows one backward)")
        prev = {k: g.clone() for k, g in self.grads.items()} if self._written else None   # gradients accumulate until a step
        d_emb = self._backward(sv, d_maps)
        if prev is not None:
            for k, g in self.grads.items():
                g.add_(prev[k])
        self._written = True
        return d_emb

    def _backward(self, sv, d_maps):
        L = _lib.lib()
        h, maps = sv["h"], sv["maps"]
        B, H, W, C = h.shape
        dm = d_maps.to(self.device, torch.float32).contiguous()
        ws = torch.empty(int(L.msam_ais_head_backward_workspace(B, H * W, C)), device=self.device, dtype=torch.uint8)
        dh = torch.empty_like(h)
        dw = torch.empty(3, C, device=self.device, dtype=torch.float32)
        _lib.check(L.msam_op_ais_head_backward(_lib.ptr(h), B, H * W, C, _lib.ptr(self.out_w), _lib.ptr(maps), _lib.ptr(dm), _lib.ptr(ws),
                                               ws.numel(), _lib.ptr(dh), _lib.ptr(dw), _lib.ptr(self.grads["out_conv.bias"]),
                                               _lib.cur_stream()))
        self.grads["out_conv.weight"].copy_(dw.view(3, C, 1, 1))
        dzs = [torch.empty(z.shape, device=self.device, dtype=torch.float32) for z in sv["zs"]]
        g = self._block_bwd(dh, sv["head"], True, d_a1=dzs[3])
        g = self._sampler_bwd(g, sv["out"])
        for i in (2, 1, 0):
            g = self._block_bwd(g, sv["blocks"][i + 1], False, d_a1=dzs[i])
            g = self._sampler_bwd(g, sv["samplers"][i])
        x = sv["x"]
        d_emb = torch.zeros(x.shape, device=self.device, dtype=torch.float32)
        self._block_bwd(g, sv["blocks"][0], False, d_a0=d_emb)
        for i in (3, 2, 1, 0):
            g = self._deconv_bwd(dzs[i], sv["deconv"][i])
            self._add(dzs[i - 1] if i > 0 else d_emb, g)
        return d_emb.permute(0, 3, 1, 2).contiguous()

    # ---------------------------------------------------------------- optimizer and state
    def zero_grads(self) -> None:
        for g in self.grads.values():
            g.zero_()
        self._written = False

    def optimizer_step(self, lr: float = 1e-5, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01) -> None:
        """torch.optim.AdamW over the decoder tensors, then the operand refresh and zero_grads.  Every backward writes every
        tensor's gradient; without a backward since the last step or zero_grads there is none and the step does nothing (torch
        skips parameters whose grad is None).  Each tensor counts its own steps for the bias correction."""
        if not self._written:
            return
        L = _lib.lib()
        for k, w in self.masters.items():
            if k not in self.moments:
                self.moments[k] = (torch.zeros_like(w), torch.zeros_like(w))
            m, v = self.moments[k]
            self.steps[k] += 1
            _lib.check(L.msam_op_adamw(_lib.ptr(w), _lib.ptr(self.grads[k]), _lib.ptr(m), _lib.ptr(v), w.numel(), float(lr),
                                       float(betas[0]), float(betas[1]), float(eps), float(weight_decay), self.steps[k],
                                       _lib.cur_stream()))
        self.zero_grads()   # the trainer's optimizer.zero_grad() before the next backward
        self.refresh()

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """decoder_state with upstream keys: CPU fp32 weights, BatchNorm unfolded with its running statistics"""
        sd = {k: v.detach().cpu().clone() for k, v in self.masters.items()}
        for k, v in self.buffers.items():
            sd[k] = torch.tensor(v, dtype=torch.int64) if isinstance(v, int) else v.detach().cpu().clone()
        return sd
