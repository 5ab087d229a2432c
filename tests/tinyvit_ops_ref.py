"""Float64 references of the TinyViT (vit_t) encoder's CUDA-core kernels (csrc/tinyvit.cu), one function per kernel, the
inputs tests/test_gpu_tinyvit_ops.py feeds them and the tolerances it applies.

As in tests/encoder_ops_ref.py, whose metrics (errors, within, bf16_ulp) these share, every reference takes exactly the
bf16 / fp32 tensors the kernel receives and computes in float64 on the device they live on, so a difference measures the
kernel's arithmetic and not the rounding of its inputs.  tests/test_tinyvit_ops_ref_cpu.py pins each reference against the
oracle's module in float64 (oracle/tinyvit_ref.py) and shows, without a GPU, that each (metric, tolerance) pair flags the
faults it is there for.
"""
import torch
import torch.nn.functional as F

from tests.encoder_ops_ref import bf16_ulp, errors, gelu, head_rows, within  # noqa: F401  (the metrics the TinyViT tests apply)

HEAD_DIM = 32
SCALE = HEAD_DIM ** -0.5
# Sam.preprocess constants as the kernel holds them (fp32): the reference subtracts and divides by the same numbers
MEAN = torch.tensor((123.675, 116.28, 103.53), dtype=torch.float32).double()
STD = torch.tensor((58.395, 57.12, 57.375), dtype=torch.float32).double()


# ------------------------------------------------------------------------------------------------ weight layouts
def fold_conv_bn(m, eps=1e-5):
    """Conv2d_BN (eval) -> (weight, bias) of the equivalent plain conv, as csrc/tinyvit.cu:fold_conv_bn computes them."""
    s = m.bn.weight / torch.sqrt(m.bn.running_var + eps)
    return m.c.weight * s[:, None, None, None], m.bn.bias - m.bn.running_mean * s


def stem_weight(w):
    """conv weight [32, 3, 3, 3] -> the kernel's [27, 32], row (ky * 3 + kx) * 3 + c."""
    return w.permute(2, 3, 1, 0).reshape(27, w.shape[0])


def dw_weight(w):
    """depth-wise conv weight [C, 1, 3, 3] -> the kernel's [9, C], row ky * 3 + kx."""
    return w.reshape(w.shape[0], 9).t()


def gemm_conv_weight(w):
    """dense conv3x3 weight [out, C, 3, 3] -> the GEMM operand [out, 9 * C], column (ky * 3 + kx) * C + c (im2col's layout)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


# ------------------------------------------------------------------------------------------------ stem
def preprocess_u8(u8, img):
    """uint8 HWC [B, h, w, 3] -> float64 NCHW [B, 3, img, img]: Sam.preprocess, (x - mean) / std and a zero pad at the bottom
    and right (pad pixels are 0 after the normalisation, not -mean / std)."""
    x = u8.double().permute(0, 3, 1, 2)
    x = (x - MEAN.to(x.device).view(1, 3, 1, 1)) / STD.to(x.device).view(1, 3, 1, 1)
    return F.pad(x, (0, img - x.shape[3], 0, img - x.shape[2]))


def stem_ref(x, w27, b):
    """float64 NCHW [B, 3, img, img] -> (GELU(conv3x3/2 pad 1 + b), sum |x||w| + |b|), both NHWC [B, img/2, img/2, 32]."""
    W = w27.double().reshape(3, 3, 3, -1).permute(3, 2, 0, 1)
    pre = F.conv2d(x.double(), W, b.double(), stride=2, padding=1)
    mag = F.conv2d(x.double().abs(), W.abs(), b.double().abs(), stride=2, padding=1)
    return gelu(pre).permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)


def stem_pad_outputs(B, hh, ww, img, device):
    """bool [B, img/2, img/2]: outputs whose whole 3 x 3 field lies in the bottom / right zero pad of an hh x ww image."""
    o = torch.arange(img // 2, device=device)
    dead_y, dead_x = 2 * o - 1 >= hh, 2 * o - 1 >= ww
    return (dead_y[:, None] | dead_x[None, :]).expand(B, -1, -1)


# ------------------------------------------------------------------------------------------------ im2col / depth-wise conv
def nchw(x, B, H, C):
    return x.reshape(B, H, H, C).permute(0, 3, 1, 2)


def rows(x):
    """NCHW -> NHWC rows [B * H * W, C]."""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def im2col_ref(x, B, Hin, C, stride):
    """NHWC [B, Hin, Hin, C] -> [B * Ho * Ho, 9 * C] in x's dtype, column (ky * 3 + kx) * C + c, Ho = Hin / stride (Hin even
    with stride 2)."""
    Ho = Hin // stride
    col = F.unfold(nchw(x.double(), B, Hin, C), 3, padding=1, stride=stride)      # [B, C * 9, Ho * Ho], row c * 9 + k
    return col.view(B, C, 9, Ho * Ho).permute(0, 3, 2, 1).reshape(B * Ho * Ho, 9 * C).to(x.dtype)


def dwconv_ref(x, B, Hin, C, stride, w9, b, act=0):
    """Depth-wise conv3x3 pad 1 + b (+ GELU) of NHWC x -> (out, magnitude sum |x||w| + |b|), rows [B * Ho * Ho, C]."""
    X, W = nchw(x.double(), B, Hin, C), w9.double().t().reshape(C, 1, 3, 3)
    pre = F.conv2d(X, W, b.double(), stride, 1, groups=C)
    mag = F.conv2d(X.abs(), W.abs(), b.double().abs(), stride, 1, groups=C)
    return rows(gelu(pre) if act else pre), rows(mag)


def border_pixels(B, Ho, device):
    """bool [B * Ho * Ho]: output pixels in the first / last row or column (the ones with taps in the zero pad)."""
    o = torch.arange(Ho, device=device)
    e = (o == 0) | (o == Ho - 1)
    return (e[:, None] | e[None, :]).reshape(-1).repeat(B)


# ------------------------------------------------------------------------------------------------ windows
def n_windows(H, ws):
    return (H + ws - 1) // ws


def partition(x, B, H, ws):
    """token rows [B * H * H, D] -> window-partitioned rows [B * nw * nw * ws * ws, D], zero rows for the pad tokens
    (TinyViTBlock: F.pad of the bottom / right, then view / transpose into windows)."""
    D, nw = x.shape[-1], n_windows(H, ws)
    p = F.pad(x.reshape(B, H, H, D), (0, 0, 0, nw * ws - H, 0, nw * ws - H))
    return p.view(B, nw, ws, nw, ws, D).transpose(2, 3).reshape(-1, D)


def unpartition(x, B, H, ws):
    """window-partitioned rows -> token rows [B * H * H, D] (pad rows cropped)."""
    D, nw = x.shape[-1], n_windows(H, ws)
    x = x.reshape(B, nw, nw, ws, ws, D).transpose(2, 3).reshape(B, nw * ws, nw * ws, D)
    return x[:, :H, :H].reshape(B * H * H, D)


def pad_rows(B, H, ws, device):
    """bool [B * nw * nw * ws * ws]: window-partitioned rows of pad tokens."""
    return partition(torch.ones(B * H * H, 1, device=device), B, H, ws)[:, 0] == 0


def edge_tokens(B, H, ws, device):
    """bool [B * H * H]: tokens of the last window row or column (the windows that hold pad tokens when ws does not divide H)."""
    t = torch.arange(H, device=device) >= (n_windows(H, ws) - 1) * ws
    return (t[:, None] | t[None, :]).reshape(-1).repeat(B)


def ln_window_ref(x, B, H, D, ws, gamma, beta, eps=1e-5):
    """LayerNorm after the zero pad, in window order: float64 [B * nw * nw * ws * ws, D]; pad rows are exactly beta."""
    return F.layer_norm(partition(x.double(), B, H, ws), (D,), gamma.double(), beta.double(), eps)


def bias_index(ws, device, transposed=False):
    """int64 [N, N]: TinyViT's attention_bias_idxs, |dy| * ws + |dx| of (query, key) (transposed: |dx| * ws + |dy|)."""
    t = torch.arange(ws * ws, device=device)
    dy, dx = (t[:, None] // ws - t[None] // ws).abs(), (t[:, None] % ws - t[None] % ws).abs()
    return dx * ws + dy if transposed else dy * ws + dx


def attention_windows(qkv, bias, heads, key_bias=None):
    """Window attention in window order: qkv [windows * N, heads * 96] (per head [q | k | v]), bias [heads, N, N] added to the
    scaled logits, key_bias [windows, N] added to every query's logits (None: 0) -> float64 [windows * N, heads * 32]."""
    N = bias.shape[-1]
    x = qkv.double().view(-1, N, heads, 3, HEAD_DIM).permute(3, 0, 2, 1, 4)       # [3, windows, heads, N, 32]
    logits = SCALE * (x[0] @ x[1].transpose(-1, -2)) + bias.double()
    if key_bias is not None:
        logits = logits + key_bias.double()[:, None, None, :]
    return (logits.softmax(-1) @ x[2]).permute(0, 2, 1, 3).reshape(-1, heads * HEAD_DIM)


def attention_ref(qkv, bias_tab, B, H, ws, heads):
    """msam_op_tv_attention in float64: image-order [B * H * H, heads * 32]; every query attends to all ws * ws keys of its
    window, pad keys included (they are LN(0) = beta projected, not masked)."""
    bias = bias_tab.double()[:, bias_index(ws, qkv.device)]
    return unpartition(attention_windows(qkv, bias, heads), B, H, ws)


# ------------------------------------------------------------------------------------------------ per-element bound
def elementwise(got, ref, mag, c, bf16_out):
    """(all within, worst excess): |got - ref| <= c * mag (+ one bf16 ulp of ref for a bf16 output); the excess is
    max (|got - ref| - ulp) / mag, the figure c bounds."""
    err = (got.double() - ref.double()).abs()
    ulp = bf16_ulp(ref.double()) if bf16_out else torch.zeros_like(err)
    excess = float(((err - ulp).clamp_min(0) / mag.double().clamp_min(1e-30)).max())
    return bool(torch.isfinite(got).all()) and bool((err <= c * mag.double() + ulp).all()), excess


# ------------------------------------------------------------------------------------------------ inputs
def rand(shape, seed, scale=1.0, dtype=torch.bfloat16, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(device, dtype)


def make_qkv(B, H, ws, heads, seed, device="cpu"):
    """Random bf16 qkv in window order whose pad-token rows are one constant row, as in the model (qkv of LN(0) = beta)."""
    qkv = rand((B * n_windows(H, ws) ** 2 * ws * ws, heads * 3 * HEAD_DIM), seed, 1.0, device=device)
    qkv[pad_rows(B, H, ws, device)] = rand((heads * 3 * HEAD_DIM,), seed + 1, 0.5, device=device)
    return qkv


def make_bias_tab(heads, ws, seed, scale=1.0, device="cpu"):
    return rand((heads, ws * ws), seed, scale, torch.float32, device)


def make_dw(C, seed, device="cpu"):
    """Folded depth-wise weight [9, C] and bias [C], fp32, of the magnitude BN folding gives."""
    return rand((9, C), seed, 0.3, torch.float32, device), rand((C,), seed + 1, 0.2, torch.float32, device)


def make_ln(D, seed, device="cpu"):
    return 1.0 + rand((D,), seed, 0.2, torch.float32, device), rand((D,), seed + 1, 0.5, torch.float32, device)


def make_stem(seed, device="cpu"):
    return rand((27, 32), seed, 0.3, torch.float32, device), rand((32,), seed + 1, 0.5, torch.float32, device)


def make_u8(B, hh, ww, seed, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, hh, ww, 3), generator=g, dtype=torch.uint8).to(device)


# ------------------------------------------------------------------------------------------------ tolerances
# About twice the worst value measured over the cases of a family on one H100 80GB HBM3 at a 700 W power limit (the measured
# values are listed in tests/test_gpu_tinyvit_ops.py).  Per-element bounds: |got - ref| <= C * magnitude (+ one bf16 ulp of
# the reference for a bf16 output), magnitude = sum |x||w| + |b| for the convolutions, |gamma xhat| + |beta| for the LayerNorm.
STEM_C = 8e-8
DW_BF16_C = 1.1e-7
DW_F32_C = 5e-7
LN_C = 1e-5                          # the fp32 row mean is off by ~1e-7 of a row offset of 3: large next to |gamma xhat| + |beta| ~ 0.1
TOL_LN = (3.4e-3, 4.8e-3)            # window LayerNorm, rows of D
TOL_ATTN = (3.4e-3, 5.8e-3)          # random qkv, rows = one token of one head
TOL_ATTN_PLANTED = (3.4e-3, 6.2e-3)  # bias only (q = 0), uniform attention, one dominant key
F32_SUM_C = 1.2e-7                   # uniform attention: |got - mean V| <= ulp + C * sum |v| (fp32 sum of ws * ws terms)
# Encoder level (tests/test_gpu_real_arch.py): the worst token of a stage's token stream against the fp32 oracle, with
# errors()'s floor of a quarter of the RMS token norm.
TOL_STAGE_TOKEN = 3.2e-2
