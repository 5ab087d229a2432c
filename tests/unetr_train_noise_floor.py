"""bf16 noise floor of the UNETR decoder's training step (forward + backward), measured on the CPU.  The float64 training-mode
restatement (tests/unetr_train_ref.py) is compared with a float32 emulation of the device decoder that rounds to bf16 where the
kernels of csrc/ais.cu / csrc/ais_train.cu do: in the forward pass every stored activation (convolution, norm, conv1x1 and
bilinear outputs); in the backward pass every gradient stored as bf16 (the gradients of the convolution inputs and outputs, of
the upsamplers' inputs and outputs, and of the head block's output; the skip connections and d embedding stay fp32).  Both are
fed the same bf16-rounded weights and embedding, so the floor is what the device's own rounding adds.  Prints the floor per
parameter tensor and for d embedding, per plan, as JSON; the GPU bounds of tests/test_gpu_unetr_train.py are twice these."""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import unetr_ref  # noqa: E402
from tests import unetr_train_ref as ref  # noqa: E402

REDUCED = dict(emb=64, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), head_in=64)
# (state dict kwargs, embedding shape): the whole-decoder cases of the GPU test
CASES = {"interp": (dict(transposed=False, affine=False, **REDUCED), (2, 64, 16, 16)),
         "transposed": (dict(transposed=True, affine=False, **REDUCED), (2, 64, 16, 16)),
         "affine": (dict(transposed=False, affine=True, **REDUCED), (2, 64, 16, 16))}
STATE_SEED, DATA_SEED = 7, 8


def bf(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _Q(torch.autograd.Function):
    """rounds to bf16 in the forward pass (fwd) and / or the gradient in the backward pass (bwd)"""

    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd
        return bf(x) if fwd else x.clone()

    @staticmethod
    def backward(ctx, g):
        return (bf(g) if ctx.bwd else g), None, None


def q(x, fwd=True, bwd=True):
    return _Q.apply(x, fwd, bwd)


def case_inputs(name):
    """(state dict with bf16-rounded weights, bf16-rounded embedding, upstream gradient of the maps)"""
    kw, shape = CASES[name]
    sd = unetr_ref.seeded_state(seed=STATE_SEED, **kw)
    sd = {k: (bf(v) if v.is_floating_point() and v.dim() == 4 and not k.startswith("out_conv") else v) for k, v in sd.items()}
    g = torch.Generator().manual_seed(DATA_SEED)
    z = bf(torch.randn(shape, generator=g))
    dm = torch.randn(shape[0], 3, 16 * shape[2], 16 * shape[3], generator=g)
    return sd, z, dm


def _p(sd, k):
    return sd[k]


def emu_upsampler(sd, p, x):
    x = q(x, fwd=False)   # the sampler's data gradient (a GEMM output) is stored as bf16
    if p + ".block.weight" in sd:
        return q(F.conv_transpose2d(x, _p(sd, p + ".block.weight"), _p(sd, p + ".block.bias"), stride=2))
    u = q(F.conv2d(x, _p(sd, p + ".conv.weight"), _p(sd, p + ".conv.bias")))
    return q(F.interpolate(u, scale_factor=2, mode="bilinear", align_corners=False))


def emu_deconv(sd, p, x):
    x = emu_upsampler(sd, p + ".block.0", x)
    c = q(F.conv2d(x, _p(sd, p + ".block.1.block.weight"), _p(sd, p + ".block.1.block.bias"), padding=1))
    c = F.batch_norm(c, sd[p + ".block.2.running_mean"].clone(), sd[p + ".block.2.running_var"].clone(), _p(sd, p + ".block.2.weight"),
                     _p(sd, p + ".block.2.bias"), training=True, momentum=0.1, eps=ref.EPS)
    return q(F.relu(c), bwd=False)   # the skip's gradient is accumulated in fp32


def _in(sd, key, x):
    w = _p(sd, key + ".weight") if key + ".weight" in sd else None
    b = _p(sd, key + ".bias") if key + ".bias" in sd else None
    return F.instance_norm(x, weight=w, bias=b, eps=ref.EPS)


def emu_block(sd, p, a0, a1=None):
    c0 = a0.shape[1]
    if a1 is None:
        x = q(_in(sd, p + ".block.0", a0))
    else:
        w = sd.get(p + ".block.0.weight")
        b = sd.get(p + ".block.0.bias")
        x0 = F.instance_norm(a0, weight=None if w is None else w[:c0], bias=None if b is None else b[:c0], eps=ref.EPS)
        x1 = F.instance_norm(a1, weight=None if w is None else w[c0:], bias=None if b is None else b[c0:], eps=ref.EPS)
        x = q(torch.cat([x0, x1], 1))
    h1 = q(F.relu(F.conv2d(x, _p(sd, p + ".block.1.weight"), _p(sd, p + ".block.1.bias"), padding=1)))
    n1 = q(_in(sd, p + ".block.3", h1))
    return q(F.relu(F.conv2d(n1, _p(sd, p + ".block.4.weight"), _p(sd, p + ".block.4.bias"), padding=1)))


def emu_forward(sd, z12):
    """the device decoder's training forward in float32 with its bf16 rounding points"""
    x = q(z12, bwd=False)
    z9 = emu_deconv(sd, "deconv1", x)
    z6 = emu_deconv(sd, "deconv2", z9)
    z3 = emu_deconv(sd, "deconv3", z6)
    z0 = emu_deconv(sd, "deconv4", z3)
    h = emu_block(sd, "base", x)
    for i, skip in enumerate((z9, z6, z3)):
        h = emu_block(sd, f"decoder.blocks.{i}", q(emu_upsampler(sd, f"decoder.samplers.{i}", h)), skip)
    h = emu_block(sd, "decoder_head", q(emu_upsampler(sd, "deconv_out", h)), z0)
    return torch.sigmoid(F.conv2d(h, sd["out_conv.weight"], sd["out_conv.bias"]))


def grads(sd, z, dm, dtype, emulate):
    lv = {k: (v.detach().to(dtype).clone().requires_grad_(True) if v.is_floating_point() and not k.endswith(("running_mean", "running_var"))
              else (v.to(dtype) if v.is_floating_point() else v.clone())) for k, v in sd.items()}
    zz = z.to(dtype).requires_grad_(True)
    maps = emu_forward(lv, zz) if emulate else ref.forward_maps(lv, zz, train=True)
    (maps * dm.to(dtype)).sum().backward()
    out = {k: v.grad for k, v in lv.items() if isinstance(v, torch.Tensor) and v.grad is not None}
    out["d_embedding"] = zz.grad
    return out, maps.detach()


def zero_grad_keys(keys):
    """tensors whose true gradient is 0: a bias in front of a training-mode BatchNorm or an InstanceNorm (the norm removes it)"""
    return {k for k in keys if (k.startswith("deconv") and k.endswith(".block.1.block.bias"))
            or (k.startswith(("decoder.samplers.", "deconv_out.")) and k.endswith(".bias"))}


def floors(name):
    sd, z, dm = case_inputs(name)
    g64, _ = grads(sd, z, dm, torch.float64, False)
    g32, _ = grads(sd, z, dm, torch.float32, True)
    skip = zero_grad_keys(g64)
    return {k: ref.rel_l2(g32[k], g64[k]) for k in g64 if k not in skip}


def main():
    for name in CASES:
        f = floors(name)
        print(json.dumps({"plan": name, "max": max(f.values()), "d_embedding": f["d_embedding"], "per_tensor": f}))


if __name__ == "__main__":
    main()
