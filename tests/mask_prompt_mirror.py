"""Mask prompts for the float64 training-decoder mirror (tests/decoder_train_mirror.py, imported and not changed): the dense prompt
is `mask_downscaling(mask)` of the oracle (oracle/sam_ref.py:PromptEncoder) instead of no_mask_embed.  Helper module for
tests/test_mask_prompt_mirror_cpu.py and tests/test_gpu_mask_prompt_train.py.

The CUDA mask-downscaling kernels (csrc/decoder_train.cu, md_*) compute in fp32 and round nowhere; the decoder reads the sum
embedding + dense prompt as a bf16 GEMM operand, where decoder_train_mirror.decoder already rounds it.  So this extension adds no
rounding of its own.  `decoder_train_mirror.decoder` takes the dense term through the no_mask_embed entry of its parameter dict,
which broadcasts against the [4096, 256] embedding; a [P, 4096, 256] tensor there is a per-prompt dense prompt.
"""
import torch
import torch.nn.functional as F

from tests import decoder_train_mirror as mirror

MD = "prompt_encoder.mask_downscaling."
MD_KEYS = [MD + k for k in ("0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias", "4.weight", "4.bias", "6.weight",
                            "6.bias")]
NO_MASK = "prompt_encoder.no_mask_embed.weight"


def perturbed_state_dict():
    """Seeded vit_test weights (oracle.sam_ref.seeded_state_dict, seed 1) with non-trivial LayerNorm2d affine parameters in
    mask_downscaling: the seeding sets gamma 1 and beta 0, which would leave the affine part of both stages untested."""
    from oracle import sam_ref
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    gen = torch.Generator().manual_seed(11)
    for k in ("1", "4"):
        n = sd[f"{MD}{k}.weight"].numel()
        sd[f"{MD}{k}.weight"] = 1.0 + 0.3 * torch.randn(n, generator=gen)
        sd[f"{MD}{k}.bias"] = 0.3 * torch.randn(n, generator=gen)
    return sd


def _ln2d(x, w, b, eps=1e-6):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    return w[:, None, None] * ((x - u) / torch.sqrt(s + eps)) + b[:, None, None]


def mask_downscaling(p, masks):
    """masks [P, 1, 256, 256] -> dense prompt [P, 256, 64, 64] (PromptEncoder.mask_downscaling)."""
    x = F.conv2d(masks, p[MD + "0.weight"], p[MD + "0.bias"], stride=2)
    x = mirror.gelu(_ln2d(x, p[MD + "1.weight"], p[MD + "1.bias"]))
    x = F.conv2d(x, p[MD + "3.weight"], p[MD + "3.bias"], stride=2)
    x = mirror.gelu(_ln2d(x, p[MD + "4.weight"], p[MD + "4.bias"]))
    return F.conv2d(x, p[MD + "6.weight"], p[MD + "6.bias"])


def run(state_dict, emb, sparse, emb_index, dense_pe, masks, multimask, d_low, d_iou):
    """decoder_train_mirror.run with mask prompts masks [P, 1, 256, 256]: the same outputs, plus the gradients of the ten
    mask_downscaling tensors; no_mask_embed gets an exact zero."""
    p = mirror.trainable_params(state_dict)
    for k in MD_KEYS:
        p[k] = state_dict[k].detach().to(mirror.DT).clone().requires_grad_(True)
    emb = emb.detach().to(mirror.DT).reshape(256, 64, 64).clone().requires_grad_(True)
    sparse = sparse.detach().to(mirror.DT).clone().requires_grad_(True)
    P = sparse.shape[0]
    dense = mask_downscaling(p, masks.detach().to(mirror.DT).reshape(P, 1, 256, 256))
    q = dict(p)
    q[NO_MASK] = dense.reshape(P, 256, 4096).transpose(1, 2)
    low, iou = mirror.decoder(q, emb, sparse, dense_pe.detach().to(mirror.DT).reshape(256, 64, 64), multimask)
    outs = [(low, d_low), (iou, d_iou)]
    torch.autograd.backward([o for o, g in outs if g is not None], [g.to(mirror.DT) for o, g in outs if g is not None])
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).detach() for k, v in p.items()}
    table = torch.zeros(5, 256, dtype=mirror.DT).index_add_(0, torch.as_tensor(emb_index).reshape(-1).cpu().long(),
                                                           sparse.grad.reshape(-1, 256))
    for i in range(4):
        grads[f"prompt_encoder.point_embeddings.{i}.weight"] = grads[f"prompt_encoder.point_embeddings.{i}.weight"] + table[i]
    grads["prompt_encoder.not_a_point_embed.weight"] = grads["prompt_encoder.not_a_point_embed.weight"] + table[4]
    return {"low_res": low.detach(), "iou": iou.detach(), "d_emb": emb.grad.detach(), "grads": grads}


# Bounds of the GPU comparison with mask prompts: the metrics of decoder_train_mirror.compare, at about twice the worst value measured
# over tests/test_gpu_mask_prompt_train.py's case grid on one H100 80GB HBM3 at a 700 W power limit, rounded up to two digits (the
# mask prompts change the image-side tensors, so the decoder's own families get bounds of their own; the measured worst values are
# listed in that file's docstring).
TOL_LOW = (0.017, 0.054)      # low_res: rel-L2, worst (prompt, mask, logit row)
TOL_IOU = (0.023, 0.11)       # iou: rel-L2, worst prompt
TOL_DEMB = (0.029, 0.054)      # dL/d embedding: rel-L2, worst channel
# gradient family: (rel-L2, |slope - 1|)
GRAD_BOUNDS = {
    "mask_decoder.iou_prediction_head.layers.*.bias": (0.41, 0.02),
    "mask_decoder.iou_prediction_head.layers.*.weight": (0.41, 0.019),
    "mask_decoder.iou_token.weight": (0.25, 0.025),
    "mask_decoder.mask_tokens.weight": (0.23, 0.023),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.bias": (0.27, 0.019),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.weight": (0.27, 0.017),
    "mask_decoder.output_upscaling.*.bias": (0.02, 0.0032),
    "mask_decoder.output_upscaling.*.weight": (0.019, 0.0025),
    "mask_decoder.transformer.final_attn_token_to_image.k_proj.weight": (0.17, 0.032),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.bias": (0.26, 0.012),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.weight": (0.26, 0.012),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.bias": (0.18, 0.055),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.weight": (0.17, 0.049),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.bias": (0.23, 0.018),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.weight": (0.23, 0.018),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.k_proj.weight": (0.11, 0.031),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.bias": (0.17, 0.012),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.weight": (0.17, 0.01),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.bias": (0.2, 0.032),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.weight": (0.11, 0.018),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.bias": (0.19, 0.031),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.weight": (0.19, 0.031),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.k_proj.weight": (0.26, 0.059),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.bias": (0.2, 0.018),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.weight": (0.2, 0.017),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.bias": (0.23, 0.048),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.weight": (0.23, 0.041),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.bias": (0.23, 0.033),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.weight": (0.23, 0.031),
    "mask_decoder.transformer.layers.*.mlp.lin1.bias": (0.22, 0.032),
    "mask_decoder.transformer.layers.*.mlp.lin1.weight": (0.22, 0.032),
    "mask_decoder.transformer.layers.*.mlp.lin2.bias": (0.21, 0.036),
    "mask_decoder.transformer.layers.*.mlp.lin2.weight": (0.21, 0.036),
    "mask_decoder.transformer.layers.*.norm1.bias": (0.2, 0.02),
    "mask_decoder.transformer.layers.*.norm1.weight": (0.22, 0.051),
    "mask_decoder.transformer.layers.*.norm2.bias": (0.2, 0.022),
    "mask_decoder.transformer.layers.*.norm2.weight": (0.21, 0.029),
    "mask_decoder.transformer.layers.*.norm3.bias": (0.21, 0.033),
    "mask_decoder.transformer.layers.*.norm3.weight": (0.22, 0.046),
    "mask_decoder.transformer.layers.*.norm4.bias": (0.17, 0.012),
    "mask_decoder.transformer.layers.*.norm4.weight": (0.14, 0.02),
    "mask_decoder.transformer.layers.*.self_attn.k_proj.weight": (0.23, 0.015),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.bias": (0.2, 0.021),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.weight": (0.2, 0.021),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.bias": (0.26, 0.033),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.weight": (0.24, 0.025),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.bias": (0.22, 0.031),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.weight": (0.22, 0.03),
    "mask_decoder.transformer.norm_final_attn.bias": (0.26, 0.015),
    "mask_decoder.transformer.norm_final_attn.weight": (0.29, 0.02),
    "prompt_encoder.mask_downscaling.*.bias": (0.26, 0.082),
    "prompt_encoder.mask_downscaling.*.weight": (0.38, 0.16),
    "prompt_encoder.not_a_point_embed.weight": (0.23, 0.013),
    "prompt_encoder.point_embeddings.*.weight": (0.21, 0.029),
}


def compare(got, ref, P, M):
    """decoder_train_mirror.compare under this module's bounds."""
    saved = mirror.GRAD_BOUNDS, mirror.TOL_LOW, mirror.TOL_IOU, mirror.TOL_DEMB
    mirror.GRAD_BOUNDS, mirror.TOL_LOW, mirror.TOL_IOU, mirror.TOL_DEMB = GRAD_BOUNDS, TOL_LOW, TOL_IOU, TOL_DEMB
    try:
        return mirror.compare(got, ref, P, M)
    finally:
        mirror.GRAD_BOUNDS, mirror.TOL_LOW, mirror.TOL_IOU, mirror.TOL_DEMB = saved
