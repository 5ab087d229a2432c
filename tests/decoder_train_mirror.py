"""Float64 mirror of the training-mode mask decoder (micro_sam_b200/csrc/decoder_train.cu) that rounds to bf16 exactly where the
CUDA tape does, and nowhere else.  Helper module for tests/test_decoder_mirror_cpu.py and tests/test_gpu_decoder_train.py.

The bf16 noise floor of this decoder against exact math is ~1e-1 per gradient tensor (tests/bf16_noise_floor.py), which hides a
gradient that is a few per cent wrong.  Almost all of that floor comes from *where* the tape rounds: GEMM operands, the attention
probabilities P, dS and the gradient casts.  This mirror computes everything in float64 and rounds to bf16 (round to nearest even)
at those points only, so the GPU differs from it by fp32-versus-fp64 accumulation and the rounding flips that causes.  Those
flips spread (comparison section below), so rel-L2 stays near the floor; the per-tensor projection slope is what tightens.

The structure below restates the oracle (oracle/sam_ref.py: PromptEncoder token assembly, MaskDecoder, TwoWayTransformer,
DecAttention), not the CUDA code: with ROUND = False it reproduces the oracle under torch autograd to ~1e-12, which
tests/test_decoder_mirror_cpu.py checks.  Only the placement of the rounding follows the implementation:

* weights: GEMM weights bf16; biases, LayerNorm parameters and embedding tables stay exact.
* a tensor consumed as a GEMM / attention operand is read rounded (B: round forward, identity backward); residuals, LayerNorm
  inputs and the query / key positional-encoding sums read the unrounded value.
* Linear: a bf16 output is rounded; backward rounds the incoming gradient (after the ReLU mask) before the weight, bias and input
  gradient products; the residual gradient passes unrounded.
* Attention: P = bf16(softmax(S)); backward dO = bf16(dO), dS = bf16(P o (dP - rowsum(P o dP))).
* GELU: y = bf16(gelu(x)); backward bf16(bf16(dy) o gelu'(x)).
* mask product: the gradient of the low-res logits is rounded before both products.

The prompt's sparse embeddings enter as a given tensor; the gradients of the learned tables behind them (point embeddings,
not-a-point embedding) are d(sparse) routed through `emb_index` (micro_sam_b200.sam.prompt_table_index), as the oracle's
autograd routes them.
"""
import math
import re

import torch
import torch.nn.functional as F

ROUND = True       # False: every rounding is the identity (exact float64 math)
FAULT = {}         # sensitivity test only: {"dk_scale": (attention key or "*" for every attention, factor)}
DT = torch.float64
TR = "mask_decoder.transformer."


def bf(x):
    return x.to(torch.bfloat16).to(x.dtype) if ROUND else x


class _B(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return bf(x)

    @staticmethod
    def backward(ctx, g):
        return g


def B(x):
    """The bf16 copy of a tensor that a GEMM or attention reads: rounded forward, gradient passed through."""
    return _B.apply(x) if ROUND else x


class Linear(torch.autograd.Function):
    """y = relu?(x bf16(W)^T + b) (+ res), rounded if bf16_out.  x must already be the operand's (rounded) value."""

    @staticmethod
    def forward(ctx, x, W, b, res, relu, bf16_out):
        Wb = bf(W)
        y = torch.matmul(x, Wb.t()) + b
        if relu:
            y = y.clamp_min(0)
        if res is not None:
            y = y + res
        if bf16_out:
            y = bf(y)
        ctx.save_for_backward(x, Wb, y if relu else None)
        ctx.relu, ctx.has_res = relu, res is not None
        return y

    @staticmethod
    def backward(ctx, g):
        x, Wb, y = ctx.saved_tensors
        s = bf(g * (y > 0) if ctx.relu else g)
        s2, x2 = s.reshape(-1, s.shape[-1]), x.reshape(-1, x.shape[-1])
        return s @ Wb, s2.t() @ x2, s2.sum(0), (g if ctx.has_res else None), None, None


def _heads(x, h):
    P, T, C = x.shape
    return x.reshape(P, T, h, C // h).transpose(1, 2)


class Attention(torch.autograd.Function):
    """softmax(q k^T / sqrt(head_dim)) v per (prompt, head); q [P, Tq, inner], k / v [P, Tk, inner] (rounded values)."""

    @staticmethod
    def forward(ctx, q, k, v, heads, dk_scale):
        qh, kh, vh = _heads(q, heads), _heads(k, heads), _heads(v, heads)
        scale = 1.0 / math.sqrt(qh.shape[-1])
        Pm = bf(torch.softmax((qh @ kh.transpose(-1, -2)) * scale, dim=-1))
        o = Pm @ vh
        ctx.save_for_backward(qh, kh, vh, Pm)
        ctx.scale, ctx.dk_scale = scale, dk_scale
        return o.transpose(1, 2).reshape(q.shape)

    @staticmethod
    def backward(ctx, g):
        qh, kh, vh, Pm = ctx.saved_tensors
        heads = qh.shape[1]
        dO = _heads(bf(g), heads)
        dV = Pm.transpose(-1, -2) @ dO
        dP = dO @ vh.transpose(-1, -2)
        dS = bf(Pm * (dP - (Pm * dP).sum(-1, keepdim=True)))
        dQ = ctx.scale * (dS @ kh)
        dK = (ctx.scale * ctx.dk_scale) * (dS.transpose(-1, -2) @ qh)

        def merge(t):
            return t.transpose(1, 2).reshape(t.shape[0], t.shape[2], -1)
        return merge(dQ), merge(dK), merge(dV), None, None


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    """d/dx [x Phi(x)] = Phi(x) + x phi(x)"""
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


class Gelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return bf(gelu(x))

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        return bf(bf(g) * gelu_grad(x))


class MaskProduct(torch.autograd.Function):
    """logits [P, N, 4] = up [P, N, 32] . hyper [P, 4, 32]^T; backward rounds d logits once for both products."""

    @staticmethod
    def forward(ctx, up, hyper):
        ctx.save_for_backward(up, hyper)
        return up @ hyper.transpose(1, 2)

    @staticmethod
    def backward(ctx, g):
        up, hyper = ctx.saved_tensors
        dm = bf(g)
        return dm @ hyper, dm.transpose(1, 2) @ up


# ------------------------------------------------------------------------------------------------ the decoder
def trainable_params(state_dict):
    """float64 leaves (requires_grad) for every prompt-encoder / mask-decoder tensor the training path differentiates."""
    return {k: v.detach().to(DT).clone().requires_grad_(True) for k, v in state_dict.items()
            if k.startswith(("mask_decoder.", "prompt_encoder.")) and "mask_downscaling" not in k
            and not k.endswith("positional_encoding_gaussian_matrix")}


def _lin(p, key, x, relu=False, bf16_out=True, res=None):
    return Linear.apply(x, p[key + ".weight"], p[key + ".bias"], res, relu, bf16_out)


def _ln(p, key, x, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), p[key + ".weight"], p[key + ".bias"], eps)


def _attn(p, key, q_in, k_in, v_in, res=None):
    q, k, v = _lin(p, key + ".q_proj", q_in), _lin(p, key + ".k_proj", k_in), _lin(p, key + ".v_proj", v_in)
    dk = FAULT["dk_scale"][1] if FAULT.get("dk_scale", (None,))[0] in (key, "*") else 1.0
    o = Attention.apply(q, k, v, 8, dk)
    return _lin(p, key + ".out_proj", B(o), bf16_out=False, res=res)


def _conv_t(p, key, x, bf16_out):
    """ConvTranspose2d(k = 2, s = 2) on token-major pixels: x [..., ci] -> [..., 4 (dy, dx), co]"""
    W = p[key + ".weight"]                                   # [ci, co, 2, 2]
    ci, co = W.shape[:2]
    Wg = W.permute(2, 3, 1, 0).reshape(4 * co, ci)
    y = Linear.apply(x, Wg, p[key + ".bias"].repeat(4), None, False, bf16_out)
    return y.reshape(*x.shape[:-1], 4, co)


def decoder(p, emb, sparse, dense_pe, multimask):
    """Prompt-encoder token assembly + MaskDecoder for ONE image and P prompts with the no-mask dense prompt.
    emb [256, 64, 64], sparse [P, Ts, 256], dense_pe [256, 64, 64] -> low_res [P, M, 256, 256], iou [P, M]."""
    P = sparse.shape[0]
    m = "mask_decoder."
    out_tok = torch.cat([p[m + "iou_token.weight"], p[m + "mask_tokens.weight"]], 0)
    tok = torch.cat([out_tok.expand(P, 5, 256), sparse], 1)                     # tokens = query positional encoding
    keys0 = (emb.reshape(256, 4096).t() + p["prompt_encoder.no_mask_embed.weight"]).expand(P, 4096, 256)
    pos = dense_pe.reshape(256, 4096).t()
    Q, K = tok, keys0
    for l in range(2):
        pre = f"{TR}layers.{l}."
        if l == 0:
            a = _attn(p, pre + "self_attn", B(Q), B(Q), B(Q))
        else:
            qin = B(Q + tok)
            a = _attn(p, pre + "self_attn", qin, qin, B(Q), res=Q)
        Q1 = _ln(p, pre + "norm1", a)
        qin, kin = B(Q1 + tok), B(K + pos)
        Q2 = _ln(p, pre + "norm2", _attn(p, pre + "cross_attn_token_to_image", qin, kin, B(K), res=Q1))
        h = _lin(p, pre + "mlp.lin1", B(Q2), relu=True)
        Q3 = _ln(p, pre + "norm3", _lin(p, pre + "mlp.lin2", h, bf16_out=False, res=Q2))
        qin = B(Q3 + tok)
        K = _ln(p, pre + "norm4", _attn(p, pre + "cross_attn_image_to_token", kin, qin, B(Q3), res=K))
        Q = Q3
    a = _attn(p, TR + "final_attn_token_to_image", B(Q + tok), B(K + pos), B(K), res=Q)
    hs = _ln(p, TR + "norm_final_attn", a)
    # upscaling: pixel (i, j) -> sub-pixel (dy1, dx1) -> (dy2, dx2); LayerNorm2d normalises each pixel's channels
    u1 = _conv_t(p, m + "output_upscaling.0", B(K), bf16_out=False)              # [P, 4096, 4, 64]
    a1 = Gelu.apply(B(_ln(p, m + "output_upscaling.1", u1, eps=1e-6)))
    up = Gelu.apply(_conv_t(p, m + "output_upscaling.3", a1, bf16_out=True))     # [P, 4096, 4, 4, 32]
    hyper = []
    for i in range(4):
        pre = f"{m}output_hypernetworks_mlps.{i}.layers."
        h = _lin(p, pre + "0", B(hs[:, 1 + i]), relu=True)
        h = _lin(p, pre + "1", h, relu=True)
        hyper.append(_lin(p, pre + "2", h, bf16_out=False))
    low4 = MaskProduct.apply(up.reshape(P, 65536, 32), B(torch.stack(hyper, 1)))
    low = low4.view(P, 64, 64, 2, 2, 2, 2, 4).permute(0, 7, 1, 3, 5, 2, 4, 6).reshape(P, 4, 256, 256)
    pre = m + "iou_prediction_head.layers."
    h = _lin(p, pre + "0", B(hs[:, 0]), relu=True)
    h = _lin(p, pre + "1", h, relu=True)
    iou = _lin(p, pre + "2", h, bf16_out=False)
    sl = slice(1, 4) if multimask else slice(0, 1)
    return low[:, sl], iou[:, sl]


def run(state_dict, emb, sparse, emb_index, dense_pe, multimask, d_low, d_iou):
    """Forward and backward for the upstream gradients d_low [P, M, 256, 256] and d_iou [P, M] (either may be None).
    Returns {"low_res", "iou", "d_emb", "grads"}; grads holds every prompt-encoder / mask-decoder gradient under upstream keys
    (exact zeros for tensors the prompts do not reach)."""
    p = trainable_params(state_dict)
    emb = emb.detach().to(DT).reshape(256, 64, 64).clone().requires_grad_(True)
    sparse = sparse.detach().to(DT).clone().requires_grad_(True)
    low, iou = decoder(p, emb, sparse, dense_pe.detach().to(DT).reshape(256, 64, 64), multimask)
    outs = [(low, d_low), (iou, d_iou)]
    torch.autograd.backward([o for o, g in outs if g is not None], [g.to(DT) for o, g in outs if g is not None])
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).detach() for k, v in p.items()}
    table = torch.zeros(5, 256, dtype=DT).index_add_(0, torch.as_tensor(emb_index).reshape(-1).cpu().long(),
                                                     sparse.grad.reshape(-1, 256))
    for i in range(4):
        grads[f"prompt_encoder.point_embeddings.{i}.weight"] = grads[f"prompt_encoder.point_embeddings.{i}.weight"] + table[i]
    grads["prompt_encoder.not_a_point_embed.weight"] = grads["prompt_encoder.not_a_point_embed.weight"] + table[4]
    return {"low_res": low.detach(), "iou": iou.detach(), "d_emb": emb.grad.detach(), "grads": grads}


# ------------------------------------------------------------------------------------------------ comparison with the GPU
# The GPU differs from this mirror by the flips that fp32 against fp64 accumulation causes, and those spread to about the whole
# bf16 noise floor (tests/test_gpu_decoder_train.py), so rel-L2 cannot be tight.  The projection slope <GPU, mirror> / <mirror,
# mirror> can: the flip noise is nearly orthogonal to the gradient and averages out of it, while a gradient that is scaled or
# partly lost moves it.  Its noise still differs by tensor (few elements, few prompts, ill-conditioned attention), so the
# bounds are per family of gradient tensors (layer / instance indices replaced by '*').
#
# Bounds are about twice the worst value measured over the case grid of tests/test_gpu_decoder_train.py on one H100 80GB HBM3
# at a 400 W power limit, rounded up to two digits; the measured worst values are listed in that file's docstring.
TOL_LOW = (1.7e-2, 4.2e-2)      # low_res: rel-L2, worst (prompt, mask, logit row)
TOL_IOU = (1.9e-2, 4.5e-2)      # iou: rel-L2, worst prompt
TOL_DEMB = (1.1e-1, 1.8e-1)     # dL/d embedding: rel-L2, worst channel
TOL_ZERO = 1e-4                 # analytically zero gradients: |GPU - mirror| / norm of the largest gradient
# gradient family: (rel-L2, |slope - 1|)
GRAD_BOUNDS = {
    "mask_decoder.iou_prediction_head.layers.*.bias": (0.42, 0.083),
    "mask_decoder.iou_prediction_head.layers.*.weight": (0.42, 0.083),
    "mask_decoder.iou_token.weight": (0.11, 0.024),
    "mask_decoder.mask_tokens.weight": (0.11, 0.024),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.bias": (0.24, 0.052),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.weight": (0.25, 0.053),
    "mask_decoder.output_upscaling.*.bias": (0.021, 0.0047),
    "mask_decoder.output_upscaling.*.weight": (0.022, 0.0063),
    "mask_decoder.transformer.final_attn_token_to_image.k_proj.weight": (0.16, 0.037),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.bias": (0.17, 0.029),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.weight": (0.18, 0.028),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.bias": (0.16, 0.046),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.weight": (0.16, 0.04),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.bias": (0.17, 0.03),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.weight": (0.17, 0.029),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.k_proj.weight": (0.13, 0.0078),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.bias": (0.11, 0.015),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.weight": (0.11, 0.015),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.bias": (0.16, 0.025),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.weight": (0.15, 0.022),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.bias": (0.11, 0.013),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.weight": (0.11, 0.012),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.k_proj.weight": (0.13, 0.016),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.bias": (0.11, 0.012),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.weight": (0.12, 0.013),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.bias": (0.14, 0.022),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.weight": (0.13, 0.018),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.bias": (0.12, 0.02),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.weight": (0.12, 0.02),
    "mask_decoder.transformer.layers.*.mlp.lin1.bias": (0.14, 0.012),
    "mask_decoder.transformer.layers.*.mlp.lin1.weight": (0.14, 0.012),
    "mask_decoder.transformer.layers.*.mlp.lin2.bias": (0.11, 0.017),
    "mask_decoder.transformer.layers.*.mlp.lin2.weight": (0.11, 0.016),
    "mask_decoder.transformer.layers.*.norm1.bias": (0.11, 0.011),
    "mask_decoder.transformer.layers.*.norm1.weight": (0.12, 0.015),
    "mask_decoder.transformer.layers.*.norm2.bias": (0.12, 0.011),
    "mask_decoder.transformer.layers.*.norm2.weight": (0.13, 0.015),
    "mask_decoder.transformer.layers.*.norm3.bias": (0.11, 0.017),
    "mask_decoder.transformer.layers.*.norm3.weight": (0.13, 0.015),
    "mask_decoder.transformer.layers.*.norm4.bias": (0.11, 0.014),
    "mask_decoder.transformer.layers.*.norm4.weight": (0.13, 0.018),
    "mask_decoder.transformer.layers.*.self_attn.k_proj.weight": (0.15, 0.021),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.bias": (0.11, 0.013),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.weight": (0.11, 0.012),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.bias": (0.15, 0.054),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.weight": (0.15, 0.022),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.bias": (0.11, 0.015),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.weight": (0.11, 0.015),
    "mask_decoder.transformer.norm_final_attn.bias": (0.18, 0.027),
    "mask_decoder.transformer.norm_final_attn.weight": (0.16, 0.03),
    "prompt_encoder.no_mask_embed.weight": (0.11, 0.018),
    "prompt_encoder.not_a_point_embed.weight": (0.14, 0.033),
    "prompt_encoder.point_embeddings.*.weight": (0.14, 0.015),
}


def family(key):
    return re.sub(r"\.\d+\.", ".*.", key)


def errors(got, ref, rows):
    """(rel-L2, worst per-row relative error).  A row's error is normalised by its own reference norm, floored at a quarter of
    the RMS row norm so that rows that are nearly zero do not dominate."""
    g = got.detach().double().cpu().reshape(rows, -1)
    r = ref.detach().double().cpu().reshape(rows, -1)
    d = (g - r).norm(dim=1)
    n = r.norm(dim=1)
    floor = 0.25 * float(n.pow(2).mean().sqrt())
    return float(d.norm() / n.norm().clamp_min(1e-300)), float((d / n.clamp_min(max(floor, 1e-300))).max())


def slope(got, ref):
    """<got, ref> / <ref, ref>: the component of got along ref."""
    g, r = got.detach().double().cpu().flatten(), ref.detach().double().cpu().flatten()
    return float(g @ r / (r @ r))


def compare(got, ref, P, M):
    """got / ref: {"low_res", "iou", "d_emb", "grads"} of P prompts with M masks each.  Returns ({name: (rel-L2, worst row)
    for an output, (rel-L2, |slope - 1|) for a gradient}, {name: abs error of an analytically zero gradient}, [violations]).
    Analytically zero: the k_proj biases (softmax ignores a constant added to every key's logit; the bf16 rounding of P and dS
    leaves noise) and tensors the prompts do not reach (exactly zero in the mirror)."""
    out, zero, bad = {}, {}, []
    for name, rows, tol in (("low_res", P * M * 256, TOL_LOW), ("iou", P, TOL_IOU), ("d_emb", 256, TOL_DEMB)):
        out[name] = errors(got[name], ref[name], rows)
        if not (out[name][0] <= tol[0] and out[name][1] <= tol[1]):
            bad.append((name, out[name], tol))
    scale = max(float(r.norm()) for r in ref["grads"].values())
    assert set(got["grads"]) == set(ref["grads"]), set(got["grads"]) ^ set(ref["grads"])
    for k, r in ref["grads"].items():
        g = got["grads"][k]
        assert tuple(g.shape) == tuple(r.shape), (k, g.shape, r.shape)
        if k.endswith("k_proj.bias") or float(r.norm()) == 0.0:
            zero[k] = float((g.detach().double().cpu() - r).norm()) / scale
            if not zero[k] <= TOL_ZERO:
                bad.append((k, zero[k], TOL_ZERO))
            continue
        tol = GRAD_BOUNDS[family(k)]
        out[k] = (errors(g, r, 1)[0], abs(slope(g, r) - 1.0))
        if not (out[k][0] <= tol[0] and out[k][1] <= tol[1]):
            bad.append((k, out[k], tol))
    return out, zero, bad
