"""Noise floor of the bf16 AIS decoder (tool, not a test; run on CPU: PYTHONPATH=. python tests/ais_noise_floor.py).
The float64 oracle (oracle/unetr_ref.py) against an emulation of the device decoder in float32 that rounds to bf16 exactly where
the kernels do: the embedding, every weight (BatchNorm folded first), every convolution output (after bias and ReLU), every
InstanceNorm output and every bilinear x2 output; the interpolation upsampler's conv1x1 runs before the bilinear step, as on the
device.  Same seeded weights and embedding as tests/test_gpu_ais.py::test_decoder_against_oracle.  Prints the rel-L2 and the
worst pixel of the three sigmoid maps per plan; the test's tolerances are about twice the largest of them."""
import torch
import torch.nn.functional as F

from oracle import unetr_ref

PLANS = {"production-interp": dict(), "production-transposed": dict(transposed=True),
         "reduced-affine": dict(emb=256, feats=(128, 64, 64, 64), deconv=(128, 64, 64, 64), affine=True)}


def q(t):
    return t.to(torch.bfloat16).to(torch.float32)


def emulate(sd, z12):
    f = {k: v.to(torch.float64) for k, v in sd.items() if v.is_floating_point()}
    tr = any(".block." in k for k in sd if k.startswith("decoder.samplers"))

    def conv(x, w, b, pad, relu):
        y = F.conv2d(x, q(w.float()), b.float(), padding=pad)
        return q(F.relu(y) if relu else y)

    def sampler(p, x):
        if tr:
            return q(F.conv_transpose2d(x, q(f[p + ".block.weight"].float()), f[p + ".block.bias"].float(), stride=2))
        y = conv(x, f[p + ".conv.weight"], f[p + ".conv.bias"], 0, False)
        return q(F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=False))

    def norm(x, key):
        w, b = f.get(key + ".weight"), f.get(key + ".bias")
        return q(F.instance_norm(x, weight=None if w is None else w.float(), bias=None if b is None else b.float(), eps=1e-5))

    def deconv(p, x):
        s = f[p + ".block.2.weight"] / torch.sqrt(f[p + ".block.2.running_var"] + 1e-5)
        w = f[p + ".block.1.block.weight"] * s[:, None, None, None]
        b = (f[p + ".block.1.block.bias"] - f[p + ".block.2.running_mean"]) * s + f[p + ".block.2.bias"]
        return conv(sampler(p + ".block.0", x), w, b, 1, True)

    def block(p, x0, x1=None):
        x = torch.cat([x0, x1], 1) if x1 is not None else x0
        wk, bk = p + ".block.0.weight", p + ".block.0.bias"
        if wk in f:   # per channel: normalising the concatenation equals normalising its parts
            x = q(F.instance_norm(x, weight=f[wk].float(), bias=f[bk].float(), eps=1e-5))
        else:
            x = q(F.instance_norm(x, eps=1e-5))
        y = conv(x, f[p + ".block.1.weight"], f[p + ".block.1.bias"], 1, True)
        return conv(norm(y, p + ".block.3"), f[p + ".block.4.weight"], f[p + ".block.4.bias"], 1, True)

    x = q(z12.float())
    zs, z = [], x
    for i in range(1, 5):
        z = deconv(f"deconv{i}", z)
        zs.append(z)
    h = block("base", x)
    for i in range(3):
        h = block(f"decoder.blocks.{i}", sampler(f"decoder.samplers.{i}", h), zs[i])
    h = block("decoder_head", sampler("deconv_out", h), zs[3])
    return torch.sigmoid(F.conv2d(h, f["out_conv.weight"].float(), f["out_conv.bias"].float()))


def main():
    torch.set_num_threads(max(1, torch.get_num_threads()))
    z = torch.randn(1, 256, 64, 64, generator=torch.Generator().manual_seed(8)) * 0.5
    zb = z.to(torch.bfloat16)
    for name, kw in PLANS.items():
        sd = unetr_ref.seeded_state(seed=7, **kw)
        with torch.no_grad():
            ref = unetr_ref.forward_maps(sd, zb)
            emu = emulate(sd, zb).double()
        rel = float((emu - ref).norm() / ref.norm())
        worst = float((emu - ref).abs().max())
        print(f"{name}: rel-L2 {rel:.2e}, worst pixel {worst:.2e}")


if __name__ == "__main__":
    main()
