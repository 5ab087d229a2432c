"""A mirror of the UNETR decoder's training step on the device (unetr.TrainableUNETRDecoder over csrc/ais.cu / csrc/ais_train.cu),
in any float dtype, that rounds to bf16 exactly where the device stores bf16.  Autograd carries the backward pass; every norm is
an explicit autograd Function whose backward is the formula the kernels evaluate (ais_nt_bwd_*), so a fault can be planted in it.

Rounding points, read from TrainableUNETRDecoder:
  forward   the embedding; every `_conv` output (3x3, the conv1x1 of the interpolation sampler, the transposed convolution);
            every `_norm_fwd` output (InstanceNorm of a block input or of the middle activation, BatchNorm + ReLU of a deconv
            block); the bilinear x2 output.  The head (out_conv + sigmoid) stays fp32, with the fp32 out_conv weights.
  backward  dh from the head backward (times the ReLU mask); every `_conv` output of the backward pass (the data gradients of
            the 3x3 convolutions, i.e. of the norm outputs / concatenations they read, and `_sampler_bwd`'s output, the
            gradient of a sampler input); the bilinear x2 adjoint (the gradient of the conv1x1 output); the `_norm_bwd` outputs
            with out_mode 0 (the gradient of a block's first input a0, of its middle activation h1, and of a deconv block's
            convolution output).  Space-to-depth is a permutation and needs no rounding point of its own.
  fp32      the skip gradients dzs (out_mode 1), the base block's d a0 accumulated into d embedding (out_mode 2), and dz in front
            of each deconv block's BatchNorm: the skip's gradient plus the next deconv block's bf16 input gradient.
The weights go in as the bf16 operands `refresh()` builds (`device_weights`); biases, norm affines and out_conv stay fp32.

`run(sd, z, dm, dtype)` returns every parameter gradient keyed as decoder_state is, plus "d_embedding", the maps and the
updated BatchNorm running statistics.  With `rounding=False` it is the float64 training-mode restatement
(tests/unetr_train_ref.py) computed another way; tests/test_unetr_train_mirror_cpu.py ties the two together.

Faults (for the tests that show which metric sees what): "wgrad_scale:<key>[:<factor>]" scales that weight's gradient by the
factor (1.02 by default); "in_no_mean" drops mean(g) from every InstanceNorm backward, "in_no_mean:<norm key>" from that one;
"drop_skip:<block>" drops the gradient of that block's second concatenation input; "bn_biased_var" updates BatchNorm's
running variance with the biased batch variance."""
import torch
import torch.nn.functional as F

EPS = 1e-5
BN_MOMENTUM = 0.1

# (rel-L2, |slope - 1|) bounds per family of gradient tensors against the float64 mirror: about twice the worst measured on an
# H100 over the cases of tests/test_gpu_unetr_train_mirror.py (its docstring lists the measurements)
GRAD_BOUNDS = {
    "conv3x3.weight": (0.34, 0.028),
    "sampler.weight": (0.34, 0.036),
    "norm": (0.43, 0.072),
    "bias": (0.43, 0.096),
    "out_conv": (0.023, 0.0034),
}
TOL_RUNNING = 2e-6   # BatchNorm running statistics, largest absolute difference


def bf(t):
    return t.to(torch.bfloat16).to(t.dtype)


def family(k):
    if k.startswith("out_conv."):
        return "out_conv"
    if ".block.2." in k or any(f".block.{j}." in k and not k.startswith("deconv") for j in (0, 3)):
        return "norm"
    if k.endswith(".bias"):
        return "bias"
    if ".block.0." in k or k.startswith(("decoder.samplers.", "deconv_out.")):
        return "sampler.weight"
    return "conv3x3.weight"


def zero_grad_keys(keys):
    """tensors whose true gradient is 0: the bias of a convolution in front of a training-mode BatchNorm, and the biases of the
    samplers in front of a block's InstanceNorm (the norm removes a per-channel constant)"""
    return {k for k in keys if (k.startswith("deconv") and k.endswith(".block.1.block.bias"))
            or (k.startswith(("decoder.samplers.", "deconv_out.")) and k.endswith(".bias"))}


def device_weights(sd):
    """the state dict as the device computes with it: every convolution weight but out_conv rounded to bf16"""
    return {k: (bf(v) if v.is_floating_point() and v.dim() == 4 and not k.startswith("out_conv") else v) for k, v in sd.items()}


class _Q(torch.autograd.Function):
    """rounds to bf16 in the forward pass (fwd) and / or the gradient in the backward pass (bwd)"""

    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd
        return bf(x) if fwd else x.clone()

    @staticmethod
    def backward(ctx, g):
        return (bf(g) if ctx.bwd else g), None, None


class _Scale(torch.autograd.Function):
    """identity forward, gradient times s"""

    @staticmethod
    def forward(ctx, x, s):
        ctx.s = s
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g * ctx.s, None


class _Norm(torch.autograd.Function):
    """InstanceNorm (per_image: per image and channel) or BatchNorm (per channel over the batch), biased variance, optional
    affine.  backward: dx = gamma rstd (g - mean(g) - xhat mean(g xhat)) over the group, dgamma = sum g xhat, dbeta = sum g
    (ais_nt_bwd_finalize_kernel / ais_nt_bwd_apply_kernel)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, per_image, drop_mean):
        dims = (2, 3) if per_image else (0, 2, 3)
        mu = x.mean(dims, keepdim=True)
        rstd = (((x - mu) ** 2).mean(dims, keepdim=True) + EPS).rsqrt()
        xh = (x - mu) * rstd
        ctx.save_for_backward(xh, rstd, gamma)
        ctx.dims, ctx.drop_mean = dims, drop_mean
        if gamma is None:
            return xh
        return xh * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)

    @staticmethod
    def backward(ctx, g):
        xh, rstd, gamma = ctx.saved_tensors
        dims = ctx.dims
        gx = g * xh
        k = rstd if gamma is None else rstd * gamma.view(1, -1, 1, 1)
        dx = g - xh * gx.mean(dims, keepdim=True)
        if not ctx.drop_mean:
            dx = dx - g.mean(dims, keepdim=True)
        dx = k * dx
        if gamma is None:
            return dx, None, None, None, None
        return dx, gx.sum((0, 2, 3)), g.sum((0, 2, 3)), None, None


class Mirror:
    """the device decoder's training forward (`forward`) in the dtype of its inputs; rounding to bf16 where the device does when
    `rounding`, with the named faults planted"""

    def __init__(self, sd, rounding=True, faults=()):
        self.sd, self.rounding, self.faults = sd, rounding, set(faults)
        self.scaled = {f.split(":")[1]: float(f.split(":")[2]) if f.count(":") == 2 else 1.02
                       for f in self.faults if f.startswith("wgrad_scale:")}

    def q(self, x, fwd=True, bwd=True):
        if not self.rounding:
            return x
        return _Q.apply(x, fwd, bwd)

    def w(self, k):
        v = self.sd[k]
        return _Scale.apply(v, self.scaled[k]) if k in self.scaled else v

    def norm(self, x, key, per_image, lo=None, hi=None):
        g, b = self.sd.get(key + ".weight"), self.sd.get(key + ".bias")
        if g is not None and lo is not None:
            g, b = g[lo:hi], b[lo:hi]
        return _Norm.apply(x, g, b, per_image, per_image and ("in_no_mean" in self.faults or f"in_no_mean:{key}" in self.faults))

    def batch_norm(self, c, p):
        """training-mode BatchNorm; updates sd's running statistics as torch does (momentum 0.1, unbiased variance)"""
        with torch.no_grad():
            n = c.numel() // c.shape[1]
            var = c.var((0, 2, 3), unbiased=False)
            if "bn_biased_var" not in self.faults:
                var = var * (n / max(n - 1, 1))
            rm, rv = self.sd[p + ".running_mean"], self.sd[p + ".running_var"]
            rm.mul_(1 - BN_MOMENTUM).add_(BN_MOMENTUM * c.mean((0, 2, 3)))
            rv.mul_(1 - BN_MOMENTUM).add_(BN_MOMENTUM * var)
        return self.norm(c, p, False)

    def upsampler(self, p, x):
        x = self.q(x, fwd=False)   # _sampler_bwd's output: the gradient of the sampler input, stored as bf16
        if p + ".block.weight" in self.sd:   # transposed; its gradient is rounded where the block reading it rounds it
            return self.q(F.conv_transpose2d(x, self.w(p + ".block.weight"), self.sd[p + ".block.bias"], stride=2))
        u = self.q(F.conv2d(x, self.w(p + ".conv.weight"), self.sd[p + ".conv.bias"]))   # du: the bilinear adjoint's output
        return self.q(F.interpolate(u, scale_factor=2, mode="bilinear", align_corners=False))

    def deconv(self, p, x):
        s = self.upsampler(p + ".block.0", x)
        c = self.q(F.conv2d(s, self.w(p + ".block.1.block.weight"), self.sd[p + ".block.1.block.bias"], padding=1))
        return self.q(F.relu(self.batch_norm(c, p + ".block.2")), bwd=False)   # the skip's gradient accumulates in fp32

    def block(self, p, a0, a1=None):
        """a0: the sampler output (its gradient, _norm_bwd out_mode 0, is bf16 except for the base block's fp32 d a0); a1: the
        skip, whose gradient stays fp32"""
        if a1 is None:
            x = self.q(self.norm(a0, p + ".block.0", True))
        else:
            c0 = a0.shape[1]
            if f"drop_skip:{p}" in self.faults:
                a1 = a1.detach()
            x0 = self.norm(a0, p + ".block.0", True, 0, c0)
            x1 = self.norm(a1, p + ".block.0", True, c0, c0 + a1.shape[1])
            x = self.q(torch.cat([x0, x1], 1))
        h1 = self.q(F.relu(F.conv2d(x, self.w(p + ".block.1.weight"), self.sd[p + ".block.1.bias"], padding=1)))
        n1 = self.q(self.norm(h1, p + ".block.3", True))
        return self.q(F.relu(F.conv2d(n1, self.w(p + ".block.4.weight"), self.sd[p + ".block.4.bias"], padding=1)))

    def forward(self, z12):
        x = self.q(z12, bwd=False)
        z9 = self.deconv("deconv1", x)
        z6 = self.deconv("deconv2", z9)
        z3 = self.deconv("deconv3", z6)
        z0 = self.deconv("deconv4", z3)
        h = self.block("base", x)
        for i, skip in enumerate((z9, z6, z3)):
            h = self.block(f"decoder.blocks.{i}", self.q(self.upsampler(f"decoder.samplers.{i}", h)), skip)
        h = self.block("decoder_head", self.q(self.upsampler("deconv_out", h)), z0)   # h: dh is bf16
        return torch.sigmoid(F.conv2d(h, self.sd["out_conv.weight"], self.sd["out_conv.bias"]))


def leaves(sd, dtype, device=None):
    """the state dict in `dtype` on `device`: float tensors but the running statistics as leaves that require grad"""
    out = {}
    for k, v in sd.items():
        if v.is_floating_point():
            t = v.detach().to(device=device, dtype=dtype).clone()
            out[k] = t if k.endswith(("running_mean", "running_var")) else t.requires_grad_(True)
        else:
            out[k] = v.detach().clone()
    return out


def run(sd, z, dm, dtype, rounding=True, faults=(), device=None):
    """one training step of the mirror: (gradients with "d_embedding", maps, running statistics), all detached, in `dtype` on
    `device`.  sd: the state dict as the device computes with it (device_weights); z: the embedding [B, C, h, w]; dm: the
    gradient of the maps."""
    lv = leaves(sd, dtype, device)
    zz = z.detach().to(device=device, dtype=dtype).requires_grad_(True)
    maps = Mirror(lv, rounding, faults).forward(zz)
    maps.backward(dm.to(device=device, dtype=dtype))
    grads = {k: v.grad for k, v in lv.items() if isinstance(v, torch.Tensor) and v.requires_grad}
    grads["d_embedding"] = zz.grad
    running = {k: v for k, v in lv.items() if k.endswith(("running_mean", "running_var"))}
    return grads, maps.detach(), running


def slope(got, ref):
    """<got, ref> / <ref, ref>: the component of got along ref"""
    g, r = got.detach().double().flatten(), ref.detach().double().to(got.device).flatten()
    return float(g @ r / (r @ r))


def rel_l2(got, ref):
    g, r = got.detach().double().flatten(), ref.detach().double().to(got.device).flatten()
    return float((g - r).norm() / r.norm().clamp(min=1e-300))
