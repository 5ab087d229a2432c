"""Float64 mirror of the ViT image encoder's training step (micro_sam_b200/csrc/encoder_train.cu: the forward pass that keeps its
activations, then the backward pass) that rounds to bf16 exactly where the device does.  Helper module for
tests/test_encoder_train_mirror_cpu.py and tests/test_gpu_encoder_train_mirror.py.

The structure restates the oracle (oracle/sam_ref.py: ImageEncoderViT, Block, window partition with zero padding from 64 to 70,
decomposed rel-pos, neck), not the CUDA code: with ROUND = False it reproduces the oracle under float64 autograd to ~1e-12, which
tests/test_encoder_train_mirror_cpu.py checks.  Only the placement of the rounding follows the implementation.

Weights go in as the engine stores them (`device_weights`): bf16 for the GEMM weights (qkv, proj, lin1, lin2, patch embedding,
the two neck convolutions) and the rel-pos tables; fp32 for biases, LayerNorm parameters and pos_embed.

Forward (Engine::vit_forward with activations kept): patches bf16; patch GEMM + bias + pos_embed fp32; LN1 -> bf16 (zero pad
rows in windowed blocks); qkv bf16; attention output bf16 (the probabilities are taken exactly, as tests/encoder_ops_ref.
attention_ref does: the fused kernels' rounding of the unnormalised probabilities is below the flip noise); proj fp32 + residual;
LN2 -> bf16; fc1 pre-activation bf16; gelu(pre) bf16; fc2 fp32 + residual.  Neck: bf16 cast, conv1x1 fp32, LN -> bf16, im2col,
conv3x3 fp32, LN2d.

Backward (Engine::encode_backward): every cast of the fp32 gradient to bf16 in front of a GEMM; dcol bf16; the fc2 dgrad bf16 and
again after GELU'; d(attention output) bf16; P = bf16(softmax) recomputed from the saved bf16 qkv; dP fp32; dS and dT bf16, with
dT summed from the unrounded dS; dq, dk, dv fp32, then packed to bf16; LayerNorm outputs recomputed in bf16 as wgrad operands; fp32
accumulation of dx across each LayerNorm backward.  GELU and GELU' are the oracle's exact ones.

Memory: the backward pass saves each block's float64 input and recomputes the block; weights stay in their stored precision and
are upcast one block at a time; each block's gradients go to the host as soon as they are done; attention runs over chunks of
(window | image, head) pairs so that the float64 logits of a chunk stay near CHUNK_BYTES.

FAULT (sensitivity tests only) plants one error in the backward pass:
  "rel_window" / "rel_global": factor   rel-pos gradients of every windowed / global block scaled
  "dk_no_pad": True                     dk of the windows' pad keys dropped before the pack to bf16
  "ln2_dgamma": factor                  every norm2.weight gradient scaled
  "pos_first_image": True               pos_embed gradient from image 0 only
  "col2im_drop_tap": k                  tap k (0..8) of the neck's 3x3 column gradient dropped
"""
import math

import torch
import torch.nn.functional as F

from oracle.sam_ref import get_rel_pos, window_partition, window_unpartition

ROUND = True       # False: every rounding is the identity (exact float64 math)
FAULT = {}
DT = torch.float64
EPS = 1e-6
WINDOW, PATCH, GRID = 14, 16, 64
CHUNK_BYTES = 1 << 28
E = "image_encoder."
GEMM_WEIGHTS = ("attn.qkv.weight", "attn.proj.weight", "mlp.lin1.weight", "mlp.lin2.weight")


def bf(x):
    return x.to(torch.bfloat16).to(x.dtype) if ROUND else x


def device_weights(sd, device=None):
    """the encoder's tensors of an upstream state dict as the engine stores them: bf16 GEMM weights and rel-pos tables, fp32 else"""
    out = {}
    for k, v in sd.items():
        if not k.startswith(E):
            continue
        low = k.endswith(GEMM_WEIGHTS) or "rel_pos" in k or k.endswith(("patch_embed.proj.weight", "neck.0.weight", "neck.2.weight"))
        out[k] = v.detach().to(device=device, dtype=torch.bfloat16 if low else torch.float32)
    return out


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def layer_norm(x, g, b):
    """over the last dim, biased variance (nn.LayerNorm / LayerNorm2d over channels)"""
    mu = x.mean(-1, keepdim=True)
    xh = (x - mu) * ((x - mu).pow(2).mean(-1, keepdim=True) + EPS).rsqrt()
    return xh * g + b


def layer_norm_bwd(x, g, dy):
    """(dx, dgamma, dbeta) of layer_norm over the last dim; rows = every other dim"""
    mu = x.mean(-1, keepdim=True)
    rstd = ((x - mu).pow(2).mean(-1, keepdim=True) + EPS).rsqrt()
    xh = (x - mu) * rstd
    gg = dy * g
    dx = rstd * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))
    return dx, (dy * xh).reshape(-1, x.shape[-1]).sum(0), dy.reshape(-1, x.shape[-1]).sum(0)


def _rows(x):
    return x.reshape(-1, x.shape[-1])


def _wgrad(dy, x):
    """dW = dy^T x over all rows"""
    return _rows(dy).t() @ _rows(x)


class _Weights:
    """one block's (or the stem's / neck's) tensors, upcast from their stored precision on first use"""

    def __init__(self, w, prefix):
        self.w, self.p, self.c = w, prefix, {}

    def __getitem__(self, k):
        if k not in self.c:
            self.c[k] = self.w[self.p + k].to(DT)
        return self.c[k]


def _chunks(n, per):
    step = max(1, CHUNK_BYTES // (per * 8))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def _heads(qkv, H):
    """[n, N, 3 D] -> q, k, v [n H, N, hd]"""
    n, N, D3 = qkv.shape
    t = qkv.view(n, N, 3, H, D3 // (3 * H)).permute(2, 0, 3, 1, 4)
    return [t[i].reshape(n * H, N, -1) for i in range(3)]


def _logits(q, k, Rh, Rw, side, scale):
    """Attention.forward's logits: (q scale) k^T + the decomposed rel-pos bias, from the unscaled q"""
    c, N, hd = q.shape
    attn = (q * scale) @ k.transpose(-2, -1)
    r_q = q.view(c, side, side, hd)
    rel_h = torch.einsum("bhwc,hkc->bhwk", r_q, Rh)
    rel_w = torch.einsum("bhwc,wkc->bhwk", r_q, Rw)
    return (attn.view(c, side, side, side, side) + rel_h[:, :, :, :, None] + rel_w[:, :, :, None, :]).view(c, N, N)


def attention_fwd(qkv, rel_h, rel_w, H, side):
    """qkv [n, N, 3 D] (n windows or images) -> [n, N, D] float64, exact softmax"""
    n, N, D3 = qkv.shape
    q, k, v = _heads(qkv, H)
    hd = q.shape[-1]
    Rh, Rw = get_rel_pos(side, side, rel_h), get_rel_pos(side, side, rel_w)
    out = torch.empty_like(q)
    for i0, i1 in _chunks(q.shape[0], N * N):
        p = _logits(q[i0:i1], k[i0:i1], Rh, Rw, side, hd ** -0.5).softmax(-1)
        out[i0:i1] = p @ v[i0:i1]
    return out.view(n, H, N, hd).transpose(1, 2).reshape(n, N, D3 // 3)


def attention_bwd(qkv, d_out, rel_h, rel_w, H, side):
    """(dqkv [n, N, 3 D] before the pack to bf16, d rel_pos_h, d rel_pos_w) for d_out [n, N, D] (bf16 values)"""
    n, N, D3 = qkv.shape
    q, k, v = _heads(qkv, H)
    hd = q.shape[-1]
    do = d_out.view(n, N, H, hd).transpose(1, 2).reshape(n * H, N, hd)
    scale = hd ** -0.5
    Rh, Rw = get_rel_pos(side, side, rel_h), get_rel_pos(side, side, rel_w)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    dRh, dRw = torch.zeros_like(Rh), torch.zeros_like(Rw)
    for i0, i1 in _chunks(q.shape[0], N * N):
        qc, kc, vc, doc = q[i0:i1], k[i0:i1], v[i0:i1], do[i0:i1]
        p = bf(_logits(qc, kc, Rh, Rw, side, scale).softmax(-1))
        dp = doc @ vc.transpose(-2, -1)
        ds_f = p * (dp - (p * dp).sum(-1, keepdim=True))
        del dp
        ds = bf(ds_f)
        d5 = ds_f.view(-1, side, side, side, side)       # [c, qh, qw, kh, kw]
        drel_h, drel_w = bf(d5.sum(4)), bf(d5.sum(3))     # [c, qh, qw, kh], [c, qh, qw, kw]
        del ds_f, d5
        dv[i0:i1] = p.transpose(-2, -1) @ doc
        dk[i0:i1] = scale * (ds.transpose(-2, -1) @ qc)
        r_q = qc.view(-1, side, side, hd)
        dq[i0:i1] = scale * (ds @ kc) + (torch.einsum("bhwk,hkc->bhwc", drel_h, Rh)
                                         + torch.einsum("bhwk,wkc->bhwc", drel_w, Rw)).reshape(-1, N, hd)
        dRh += torch.einsum("bhwk,bhwc->hkc", drel_h, r_q)
        dRw += torch.einsum("bhwk,bhwc->wkc", drel_w, r_q)
    # get_rel_pos's gather, adjoint: index [q, k] = q - k + side - 1
    idx = (torch.arange(side)[:, None] - torch.arange(side)[None, :] + side - 1).flatten().to(qkv.device)
    g_h = torch.zeros_like(rel_h).index_add_(0, idx, dRh.reshape(-1, hd))
    g_w = torch.zeros_like(rel_w).index_add_(0, idx, dRw.reshape(-1, hd))
    dqkv = torch.stack([t.view(n, H, N, hd).transpose(1, 2).reshape(n, N, D3 // 3) for t in (dq, dk, dv)], 2)
    return dqkv.reshape(n, N, D3), g_h, g_w


def _pad_rows(B, device):
    """bool [B * 25, 196]: the window-partitioned rows outside the 64 x 64 grid"""
    ones = torch.ones(B, GRID, GRID, 1, device=device, dtype=DT)
    return window_partition(ones, WINDOW)[0].view(-1, WINDOW * WINDOW) == 0


def block_forward(x, w, H, window):
    """Block.forward with the device's rounding; x [B, g, g, D].  Returns (output, activations for the backward pass)."""
    B, g, _, D = x.shape
    a = {}
    xn = bf(layer_norm(x, w["norm1.weight"], w["norm1.bias"]))
    pad_hw = None
    if window:
        xn, pad_hw = window_partition(xn, window)
    side = xn.shape[1]
    a["xw"] = xn = xn.reshape(xn.shape[0], side * side, D)
    a["qkv"] = qkv = bf(xn @ w["attn.qkv.weight"].t() + w["attn.qkv.bias"])
    o = attention_fwd(qkv, w["attn.rel_pos_h"], w["attn.rel_pos_w"], H, side).view(-1, side, side, D)
    if window:
        o = window_unpartition(o, window, pad_hw, (g, g))
    a["attn"] = o = bf(o)
    a["x_mid"] = xm = x + o @ w["attn.proj.weight"].t() + w["attn.proj.bias"]
    a["xn2"] = xn2 = bf(layer_norm(xm, w["norm2.weight"], w["norm2.bias"]))
    a["pre"] = pre = bf(xn2 @ w["mlp.lin1.weight"].t() + w["mlp.lin1.bias"])
    a["hid"] = h = bf(gelu(pre))
    a["side"], a["pad_hw"] = side, pad_hw
    return xm + h @ w["mlp.lin2.weight"].t() + w["mlp.lin2.bias"], a


def block_backward(x, dx, w, H, window):
    """(dx of the block input, gradients keyed as the block's parameters) for dx of its output; recomputes the block from x"""
    B, g, _, D = x.shape
    _, a = block_forward(x, w, H, window)
    gr = {}
    # MLP
    gb = bf(dx)
    gr["mlp.lin2.weight"], gr["mlp.lin2.bias"] = _wgrad(gb, a["hid"]), _rows(gb).sum(0)
    dh = bf(gb @ w["mlp.lin2.weight"])
    dpre = bf(dh * gelu_grad(a["pre"]))
    del dh
    gr["mlp.lin1.weight"], gr["mlp.lin1.bias"] = _wgrad(dpre, a["xn2"]), _rows(dpre).sum(0)
    dxn = dpre @ w["mlp.lin1.weight"]
    del dpre
    d, gr["norm2.weight"], gr["norm2.bias"] = layer_norm_bwd(a["x_mid"], w["norm2.weight"], dxn)
    if "ln2_dgamma" in FAULT:
        gr["norm2.weight"] = gr["norm2.weight"] * FAULT["ln2_dgamma"]
    dx = dx + d
    # attention
    gb = bf(dx)
    gr["attn.proj.weight"], gr["attn.proj.bias"] = _wgrad(gb, a["attn"]), _rows(gb).sum(0)
    da = bf(gb @ w["attn.proj.weight"])
    side = a["side"]
    if window:
        da = window_partition(da, window)[0]
    dqkv, gr["attn.rel_pos_h"], gr["attn.rel_pos_w"] = attention_bwd(a["qkv"], da.reshape(-1, side * side, D),
                                                                      w["attn.rel_pos_h"], w["attn.rel_pos_w"], H, side)
    f = FAULT.get("rel_window" if window else "rel_global")
    if f is not None:
        gr["attn.rel_pos_h"], gr["attn.rel_pos_w"] = gr["attn.rel_pos_h"] * f, gr["attn.rel_pos_w"] * f
    if window and FAULT.get("dk_no_pad"):
        dqkv[..., D:2 * D][_pad_rows(B, x.device)] = 0
    dqkv = bf(dqkv)
    gr["attn.qkv.weight"], gr["attn.qkv.bias"] = _wgrad(dqkv, a["xw"]), _rows(dqkv).sum(0)
    dxn = (dqkv @ w["attn.qkv.weight"]).view(-1, side, side, D)
    if window:
        dxn = window_unpartition(dxn, window, a["pad_hw"], (g, g))
    d, gr["norm1.weight"], gr["norm1.bias"] = layer_norm_bwd(x, w["norm1.weight"], dxn.view(B, g, g, D))
    return dx + d, gr


def _neck(x, w):
    """neck(x) with its activations; x [B, g, g, D] -> NCHW [B, C, g, g]"""
    B, g, _, D = x.shape
    a = {"xb": bf(x)}
    C = w["0.weight"].shape[0]
    a["n1"] = n1 = a["xb"] @ w["0.weight"].view(C, D).t()                               # conv1x1, token-major
    n1b = bf(layer_norm(n1, w["1.weight"], w["1.bias"]))
    a["col"] = col = F.unfold(n1b.permute(0, 3, 1, 2), 3, padding=1)                       # [B, 9 C, T], row c * 9 + k
    a["n2"] = n2 = (w["2.weight"].view(C, 9 * C) @ col).transpose(1, 2)                    # conv3x3, [B, T, C]
    out = layer_norm(n2, w["3.weight"], w["3.bias"])
    return out.transpose(1, 2).reshape(B, C, g, g), a


def _neck_backward(d_out, w, a, B, g):
    C = d_out.shape[1]
    gr = {}
    dtok = d_out.reshape(B, C, g * g).transpose(1, 2)
    d, gr["3.weight"], gr["3.bias"] = layer_norm_bwd(a["n2"], w["3.weight"], dtok)
    gb = bf(d)                                                                            # [B, T, C]
    gr["2.weight"] = torch.einsum("btc,bkt->ck", gb, a["col"]).reshape(C, C, 3, 3)
    dcol = bf(gb @ w["2.weight"].view(C, 9 * C)).transpose(1, 2)                          # [B, 9 C, T]
    if "col2im_drop_tap" in FAULT:
        dcol = dcol.reshape(B, C, 9, g * g).clone()
        dcol[:, :, FAULT["col2im_drop_tap"]] = 0
        dcol = dcol.reshape(B, 9 * C, g * g)
    dn1b = F.fold(dcol, (g, g), 3, padding=1).permute(0, 2, 3, 1)                         # col2im, [B, g, g, C]
    d, gr["1.weight"], gr["1.bias"] = layer_norm_bwd(a["n1"], w["1.weight"], dn1b)
    gb = bf(d)
    D = a["xb"].shape[-1]
    gr["0.weight"] = _wgrad(gb, a["xb"]).view(C, D, 1, 1)
    return gb @ w["0.weight"].view(C, D), gr


def _patchify(x):
    """[B, 3, 1024, 1024] -> [B, 64, 64, 768] in the conv weight's (c, ky, kx) order"""
    B = x.shape[0]
    return x.view(B, 3, GRID, PATCH, GRID, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(B, GRID, GRID, 3 * PATCH * PATCH)


def run(w, arch, x, d_out, device=None, keep_on_device=False):
    """One training step of the encoder: (embedding [B, 256, 64, 64], gradients keyed and shaped as the upstream state dict).
    w: the encoder's tensors as the engine stores them (`device_weights`; any precision); arch: ARCH entry; x: the preprocessed
    images [B, 3, 1024, 1024]; d_out: dL/d embedding.  Runs on `device` (default: where w lives); gradients come back on the host
    in float64 unless keep_on_device."""
    dev = device if device is not None else next(iter(w.values())).device
    H, depth, glob = arch["num_heads"], arch["depth"], set(arch["global_attn_indexes"])
    host = (lambda t: t) if keep_on_device else (lambda t: t.to("cpu"))
    stem = _Weights(w, E)
    x = x.to(device=dev, dtype=DT)
    B = x.shape[0]
    D = w[E + "patch_embed.proj.weight"].shape[0]
    patches = bf(_patchify(x))
    h = patches @ stem["patch_embed.proj.weight"].view(D, -1).t() + stem["patch_embed.proj.bias"] + stem["pos_embed"]
    saved = []
    with torch.no_grad():
        for i in range(depth):
            saved.append(h)
            h, _ = block_forward(h, _Weights(w, f"{E}blocks.{i}."), H, 0 if i in glob else WINDOW)
        neck = _Weights(w, E + "neck.")
        out, na = _neck(h, neck)
        del h
        grads = {}
        dx, gr = _neck_backward(d_out.to(device=dev, dtype=DT), neck, na, B, GRID)
        del na
        grads.update({E + "neck." + k: host(v) for k, v in gr.items()})
        for i in reversed(range(depth)):
            p = f"{E}blocks.{i}."
            dx, gr = block_backward(saved.pop(), dx.view(B, GRID, GRID, D), _Weights(w, p), H, 0 if i in glob else WINDOW)
            grads.update({p + k: host(v) for k, v in gr.items()})
        dpos = dx[:1] if FAULT.get("pos_first_image") else dx.sum(0, keepdim=True)
        grads[E + "pos_embed"] = host(dpos.reshape(1, GRID, GRID, D))
        gb = bf(dx)
        grads[E + "patch_embed.proj.weight"] = host(_wgrad(gb, patches).view(D, 3, PATCH, PATCH))
        grads[E + "patch_embed.proj.bias"] = host(_rows(gb).sum(0))
    return out, grads


# ------------------------------------------------------------------------------------------------ metrics
def family(k):
    """the bound family of a gradient key (a "[k]" / "[qv]" suffix marks the thirds of attn.qkv.bias)"""
    k = k[len(E):] if k.startswith(E) else k
    if k.startswith("blocks."):
        leaf = k.split(".", 2)[2]
        if leaf.startswith(GEMM_WEIGHTS):
            return "gemm_weight"
        if leaf.startswith("norm"):
            return "block_norm"
        if "rel_pos" in leaf:
            return "rel_pos"     # split into windowed / global by the caller, which knows the architecture
        return "bias"
    if k == "pos_embed":
        return "pos_embed"
    if k.startswith("patch_embed."):
        return "patch_embed"
    if k in ("neck.0.weight", "neck.2.weight"):
        return "neck_conv"
    return "neck_norm"


def split_qkv_bias(grads):
    """attn.qkv.bias -> "<key>[qv]" (q and v thirds) and "<key>[k]" (the k third, zero in exact arithmetic)"""
    out = {}
    for k, v in grads.items():
        if k.endswith("attn.qkv.bias"):
            D = v.numel() // 3
            out[k + "[qv]"] = torch.cat([v[:D], v[2 * D:]])
            out[k + "[k]"] = v[D:2 * D]
        else:
            out[k] = v
    return out


def slope(got, ref):
    """<got, ref> / <ref, ref>: the component of got along ref"""
    g, r = got.detach().double().flatten(), ref.detach().double().to(got.device).flatten()
    return float(g @ r / (r @ r))


def rel_l2(got, ref):
    g, r = got.detach().double().flatten(), ref.detach().double().to(got.device).flatten()
    return float((g - r).norm() / r.norm().clamp(min=1e-300))


# (rel-L2, |slope - 1|) bounds per family of gradient tensors against the float64 mirror, about twice the worst measured on an
# H100 over the cases of tests/test_gpu_encoder_train_mirror.py (its docstring lists the measurements)
GRAD_BOUNDS = {
    "gemm_weight": (1.8e-2, 1.7e-3),
    "bias": (1.8e-2, 1.7e-3),
    "block_norm": (1.8e-2, 2.6e-3),
    "rel_window": (5e-2, 1.2e-2),
    "rel_global": (4.7e-2, 1.2e-2),
    "pos_embed": (2.4e-2, 1.3e-4),
    "patch_embed": (1.7e-2, 1.4e-3),
    "neck_conv": (9.6e-3, 8.7e-4),
    "neck_norm": (9.8e-3, 1.3e-3),
}
TOL_EMBEDDING = 9.4e-3   # rel-L2 of the embedding
TOL_ZERO = 2.3e-5        # |k third of attn.qkv.bias gradient| / the largest gradient norm


def compare(got_out, got, want_out, want, arch):
    """(metrics, violations) of a device (or faulted mirror) step against the mirror under the bounds above"""
    glob = set(arch["global_attn_indexes"])
    g, w = split_qkv_bias(got), split_qkv_bias(want)
    big = max(float(v.double().norm()) for k, v in w.items() if not k.endswith("[k]"))
    res = {"embedding": rel_l2(got_out, want_out),
           "zero": max(float(v.double().norm()) / big for k, v in g.items() if k.endswith("[k]")), "families": {}}
    bad = []
    if not res["embedding"] <= TOL_EMBEDDING:
        bad.append(("embedding", res["embedding"], TOL_EMBEDDING))
    if not res["zero"] <= TOL_ZERO:
        bad.append(("zero", res["zero"], TOL_ZERO))
    for k in w:
        if k.endswith("[k]"):
            continue
        f = family(k)
        if f == "rel_pos":
            f = "rel_global" if int(k[len(E):].split(".")[1]) in glob else "rel_window"
        r, s = rel_l2(g[k], w[k]), abs(slope(g[k], w[k]) - 1)
        worst = res["families"].setdefault(f, [0.0, 0.0, None])
        if r > worst[0]:
            worst[0] = r
        if s > worst[1]:
            worst[1], worst[2] = s, k
        tol = GRAD_BOUNDS[f]
        if not (r <= tol[0] and s <= tol[1]):
            bad.append((k, r, s, tol))
    return res, bad
