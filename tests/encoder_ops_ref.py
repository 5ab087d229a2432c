"""Float64 references of the ViT encoder's kernels, one function per kernel, plus the comparison metrics and tolerances
that tests/test_gpu_encoder_ops.py applies to them.

Every reference takes exactly the bf16 / fp32 tensors the kernel receives and computes in float64 on the device those
tensors live on, so a difference measures the kernel's arithmetic and not the rounding of its inputs.  They are pinned
against the oracle's modules and against autograd in tests/test_encoder_ops_ref_cpu.py, which also shows, without a GPU,
that each (metric, tolerance) pair below flags the localised faults it is there for.
"""
import math

import torch
import torch.nn.functional as F

GRID, WINDOW = 64, 14
WPR = (GRID + WINDOW - 1) // WINDOW          # 5 windows per image side
WIN_ROWS = WPR * WPR * WINDOW * WINDOW       # 4900 window-partitioned rows per image


class Geom:
    """csrc/kernels.h:rel_table_geom -- the packed rel-pos table and the T = Q RelTable^T rows the attention kernels use."""

    def __init__(self, global_):
        self.global_ = bool(global_)
        self.side = GRID if global_ else WINDOW
        self.n_tok = self.side * self.side
        self.nt = 256 if global_ else 64
        self.woff = 128 if global_ else 32
        self.pitch = (self.n_tok + 7) & ~7    # row pitch of S / P / dS in the backward pass (200 / 4096)


def rel_table(rel_h, rel_w, geom):
    """bf16 [nt, 64 * ceil(hd / 64)]: rows [0, 2 side - 1) = rel_pos_h, rows [woff, woff + 2 side - 1) = rel_pos_w."""
    hd = rel_h.shape[1]
    tab = torch.zeros(geom.nt, ((hd + 63) // 64) * 64, device=rel_h.device, dtype=torch.bfloat16)
    tab[:2 * geom.side - 1, :hd] = rel_h
    tab[geom.woff:geom.woff + 2 * geom.side - 1, :hd] = rel_w
    return tab


def bias_index(geom, device):
    """(ih, iw) int64 [n_tok, n_tok]: columns of a T row that hold the rel_h / rel_w bias of (query, key)."""
    t = torch.arange(geom.n_tok, device=device)
    h, w = t // geom.side, t % geom.side
    ih = h[:, None] - h[None, :] + geom.side - 1
    iw = geom.woff + w[:, None] - w[None, :] + geom.side - 1
    return ih, iw


def gather_bias(T, geom):
    """T [n, n_tok, nt] -> bias [n, n_tok, n_tok] = T[q, qh - kh + side - 1] + T[q, woff + qw - kw + side - 1]."""
    ih, iw = bias_index(geom, T.device)
    n = T.shape[0]
    return torch.gather(T, 2, ih.expand(n, -1, -1)) + torch.gather(T, 2, iw.expand(n, -1, -1))


# ------------------------------------------------------------------------------------------------ forward attention
def unpartition(x, batch):
    """window-partitioned rows [batch * 4900, D] -> image order [batch * 4096, D] (the pad rows are cropped)."""
    D = x.shape[-1]
    x = x.view(batch, WPR, WPR, WINDOW, WINDOW, D).permute(0, 1, 3, 2, 4, 5).reshape(batch, WPR * WINDOW, WPR * WINDOW, D)
    return x[:, :GRID, :GRID].reshape(batch * GRID * GRID, D)


def attention_ref(qkv, rel_h, rel_w, batch, heads, head_dim, window, return_probs=False):
    """qkv [groups * G, 3 * heads * head_dim] as the kernel reads it (window: 25 windows of 196 rows per image, pad rows
    included as keys; global: 4096 rows per image) -> float64 [batch * 4096, heads * head_dim] in image order, and the
    probabilities [groups, heads, G, G] on request."""
    geom = Geom(window == 0)
    G, D = geom.n_tok, heads * head_dim
    groups = qkv.shape[0] // G
    x = qkv.double().view(groups, G, 3, heads, head_dim)
    rh, rw = rel_h.double(), rel_w.double()
    scale = head_dim ** -0.5
    tab = torch.zeros(geom.nt, head_dim, dtype=torch.float64, device=qkv.device)
    tab[:2 * geom.side - 1] = rh
    tab[geom.woff:geom.woff + 2 * geom.side - 1] = rw
    out = torch.empty(groups, G, heads, head_dim, dtype=torch.float64, device=qkv.device)
    probs = []
    step = max(1, (1 << 25) // (G * G))          # (group, head) pairs per chunk: bounds the float64 logits held at once
    for g0 in range(groups):
        for h0 in range(0, heads, step):
            q = x[g0, :, 0, h0:h0 + step].transpose(0, 1)       # [h, G, hd]
            k = x[g0, :, 1, h0:h0 + step].transpose(0, 1)
            v = x[g0, :, 2, h0:h0 + step].transpose(0, 1)
            logits = scale * (q @ k.transpose(1, 2)) + gather_bias(q @ tab.t(), geom)   # the bias uses the unscaled q
            p = logits.softmax(dim=-1)
            out[g0, :, h0:h0 + step] = (p @ v).transpose(0, 1)
            if return_probs:
                probs.append(p)
    out = out.reshape(groups * G, D)
    out = unpartition(out, batch) if window else out
    if return_probs:
        return out, torch.cat(probs).view(groups, heads, G, G)
    return out


# ------------------------------------------------------------------------------------------------ GEMM
def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gemm_ref(A, W, bias=None, residual=None, res_rows=0, act=0, act_after_res=0, ln=None):
    """act(A W^T + bias) + residual[row % res_rows], or act applied after the residual; ln = (gamma, beta, eps) normalises
    each row afterwards.  Returns (result, pre) with pre = the value the activation was applied to."""
    x = A.double() @ W.double().t()
    if bias is not None:
        x = x + bias.double()
    r = None
    if residual is not None:
        rr = res_rows if res_rows > 0 else A.shape[0]
        r = residual.double()[torch.arange(A.shape[0], device=A.device) % rr]
    fn = {0: lambda t: t, 1: gelu, 2: torch.relu}[act]
    if act_after_res:
        pre = x + r if r is not None else x
        x = fn(pre)
    else:
        pre = x
        x = fn(x)
        if r is not None:
            x = x + r
    if ln is not None:
        gamma, beta, eps = ln
        x = F.layer_norm(x, (x.shape[1],), gamma.double(), beta.double(), eps)
    return x, pre


def gemm_magnitude(A, W, bias=None, residual=None, res_rows=0):
    """sum_k |a| |w| + |bias| + |residual|: what the rounding error of an fp32 accumulation is proportional to."""
    m = A.double().abs() @ W.double().abs().t()
    if bias is not None:
        m = m + bias.double().abs()
    if residual is not None:
        rr = res_rows if res_rows > 0 else A.shape[0]
        m = m + residual.double().abs()[torch.arange(A.shape[0], device=A.device) % rr]
    return m


def bf16_ulp(x):
    """spacing of bf16 numbers at |x| (8 significant bits), at least the spacing at the smallest normal."""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


# ------------------------------------------------------------------------------------------------ attention backward stages
def attn_probs_ref(S, T, geom, scale):
    """S [n, n_tok, n_tok], T [n, n_tok, nt] -> softmax_k(scale S + bias(T))."""
    return (scale * S.double() + gather_bias(T.double(), geom)).softmax(dim=-1)


def attn_ds_ref(P, dP, geom):
    """P, dP [n, n_tok, n_tok] -> dS = P o (dP - sum_k P dP) [n, n_tok, n_tok] (the gradient of the logits) and dT
    [n, n_tok, nt], its pull-back through the bias gather, taken by autograd."""
    P, dP = P.double(), dP.double()
    dS = P * (dP - (P * dP).sum(-1, keepdim=True))
    T = torch.zeros(P.shape[0], geom.n_tok, geom.nt, dtype=torch.float64, device=P.device, requires_grad=True)
    (gather_bias(T, geom) * dS).sum().backward()
    return dS, T.grad


def gelu_grad_ref(x):
    """d/dx [x Phi(x)] = Phi(x) + x phi(x), exact erf form."""
    x = x.double()
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def gelu_grad_tanh(x):
    """derivative of the tanh approximation of GELU: the fault the gelu_bwd bound has to reject."""
    x = x.double()
    c = math.sqrt(2.0 / math.pi)
    u = c * (x + 0.044715 * x ** 3)
    t = torch.tanh(u)
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * c * (1.0 + 3 * 0.044715 * x * x)


def im2col3x3_ref(x, B, g, C):
    """x [B * g * g, C] -> [B * g * g, 9 * C] with column (ky * 3 + kx) * C + c: the layout im2col3x3_kernel writes."""
    col = F.unfold(x.view(B, g, g, C).permute(0, 3, 1, 2), 3, padding=1)        # [B, C * 9, g * g], row c * 9 + k
    return col.view(B, C, 9, g * g).permute(0, 3, 2, 1).reshape(B * g * g, 9 * C)


def col2im3x3_ref(dcol, B, g, C):
    """adjoint of im2col3x3_ref, by autograd."""
    x = torch.zeros(B * g * g, C, dtype=torch.float64, device=dcol.device, requires_grad=True)
    (im2col3x3_ref(x, B, g, C) * dcol.double()).sum().backward()
    return x.grad


def window_gather_ref(x, B):
    """image order [B * 4096, D] -> window-partitioned [B * 4900, D] with zero pad rows."""
    D = x.shape[1]
    pad = WPR * WINDOW - GRID
    x = F.pad(x.view(B, GRID, GRID, D), (0, 0, 0, pad, 0, pad))
    return x.view(B, WPR, WINDOW, WPR, WINDOW, D).permute(0, 1, 3, 2, 4, 5).reshape(B * WIN_ROWS, D)


def pad_rows_mask(B, device):
    """bool [B * 4900]: True at the window-partitioned rows that lie outside the 64 x 64 grid."""
    ones = torch.ones(B * GRID * GRID, 1, device=device)
    return window_gather_ref(ones, B)[:, 0] == 0


# ------------------------------------------------------------------------------------------------ metrics and tolerances
def errors(got, ref, rows):
    """rel-L2 over everything, worst per-row relative error, all finite.  A row's error is normalised by its own reference
    norm, floored at a quarter of the RMS row norm so that rows that are nearly zero do not dominate."""
    g = got.double().reshape(rows, -1)
    r = ref.double().reshape(rows, -1).to(g.device)
    d = (g - r).norm(dim=1)
    n = r.norm(dim=1)
    floor = 0.25 * float(n.pow(2).mean().sqrt())
    rel = float(d.norm() / n.norm())
    row = float((d / n.clamp_min(floor)).max())
    return rel, row, bool(torch.isfinite(g).all())


def within(got, ref, rows, tol):
    rel, row, finite = errors(got, ref, rows)
    return finite and rel <= tol[0] and row <= tol[1], (rel, row, finite)


# ------------------------------------------------------------------------------------------------ output sentinels
SENT_BF16, SENT_F32 = 1024.0, -7777.0


def guarded(n, dtype, margin=4096, device="cuda"):
    """A flat buffer of n elements with `margin` sentinel elements on each side; returns (whole, inner view)."""
    s = SENT_BF16 if dtype == torch.bfloat16 else SENT_F32
    buf = torch.full((n + 2 * margin,), s, device=device, dtype=dtype)
    return buf, buf[margin:margin + n]


def margins_intact(buf, n, margin=4096):
    s = SENT_BF16 if buf.dtype == torch.bfloat16 else SENT_F32
    return bool((buf[:margin] == s).all()) and bool((buf[margin + n:] == s).all())


def gelu_mismatch(got, ref, pre):
    """largest fraction, over windows of 256 neighbouring points with |pre| <= 3, of outputs that are not the bf16 rounding of
    the reference.  A derivative that is right to fp32 accuracy flips a rounding only at near-ties; one that is off by 1e-3
    (the tanh approximation) flips a sizeable share where bf16 spacing is 4e-3 .. 8e-3 of the value.  (Below -3 the
    derivative is under 1e-2 and fp32 cancellation in 1 + erf shows in the relative error of values that no longer matter.)"""
    differs = (got.double() != ref.to(torch.bfloat16).double()).view(-1, 256).double().mean(1)
    return float(differs[(pre.double().view(-1, 256).abs() <= 3).all(1)].max())


def head_rows(x, heads):
    """[tokens, heads * hd] -> [tokens * heads, hd]: a row of the attention metrics is one token of one head."""
    return x.reshape(x.shape[0], heads, -1).reshape(x.shape[0] * heads, -1)


# (rel-L2, worst row) bounds, about twice the worst value measured over the cases of a family on one H100 80GB HBM3 at a
# 700 W power limit (the measured values are listed in tests/test_gpu_encoder_ops.py).
TOL_ATTN_WINDOW = (3.6e-3, 7e-3)       # random qkv, production head counts
TOL_ATTN_GLOBAL = (3.7e-3, 7e-3)
TOL_ATTN_BIAS_ONLY = (4.5e-3, 7e-3)    # k = 0: the logits are the rel-pos bias alone
TOL_ATTN_PLANTED = (3.8e-3, 8.5e-3)     # dominant keys, monotone logits, offsets, uniform attention
TOL_GEMM_LN = (3.4e-3, 4e-3)         # fused LayerNorm(256) epilogue, bf16 out
GEMM_F32_C = 5e-7                    # |got - ref| <= C * (sum |a||w| + |bias| + |residual|) for fp32 output
GEMM_GELU_FAST = 3e-5                # absolute error of the bf16-output GELU (gemm.cu:gelu_fast documents 2.6e-5)
TOL_PROBS = (3.3e-3, 7e-3)           # attn_probs: bf16 probabilities
TOL_DS = (3.4e-3, 7.5e-3)            # attn_ds: dS
TOL_DT = (3.4e-3, 7e-3)              # attn_ds: dT
TOL_GELU_BWD = (2.1e-3, 5.3e-3)        # gelu_bwd, rows of 64 elements
TOL_GELU_MISMATCH = 0.02             # gelu_bwd: share of 256 neighbouring outputs that differ from the rounded reference
F32_SUM_C = 4e-7                     # colsum / col2im / sum_batch: |got - ref| <= C * sum |terms|
