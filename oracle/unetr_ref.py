"""Float64 restatement of micro-sam's AIS decoder (DecoderAdapter over torch_em's UNETR, as DESIGN.md section 2 states it,
unpinned): every layer applied straight from the state dict keys with torch.nn.functional, channel counts from the weights."""
import torch
import torch.nn.functional as F

EPS = 1e-5


def _t(sd, k):
    return sd[k].to(torch.float64)


def upsampler(sd, p, x):
    """bilinear x2 then conv1x1 (`p.conv.*`), or ConvTranspose2d k2 s2 (`p.block.*`)."""
    if p + ".block.weight" in sd:
        return F.conv_transpose2d(x, _t(sd, p + ".block.weight"), _t(sd, p + ".block.bias"), stride=2)
    x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    return F.conv2d(x, _t(sd, p + ".conv.weight"), _t(sd, p + ".conv.bias"))


def deconv_block(sd, p, x):
    x = upsampler(sd, p + ".block.0", x)
    x = F.conv2d(x, _t(sd, p + ".block.1.block.weight"), _t(sd, p + ".block.1.block.bias"), padding=1)
    x = F.batch_norm(x, _t(sd, p + ".block.2.running_mean"), _t(sd, p + ".block.2.running_var"), _t(sd, p + ".block.2.weight"),
                     _t(sd, p + ".block.2.bias"), training=False, eps=EPS)
    return F.relu(x)


def _norm(sd, key, x):
    w = _t(sd, key + ".weight") if key + ".weight" in sd else None
    b = _t(sd, key + ".bias") if key + ".bias" in sd else None
    return F.instance_norm(x, weight=w, bias=b, eps=EPS)


def conv_block(sd, p, x):
    x = _norm(sd, p + ".block.0", x)
    x = F.relu(F.conv2d(x, _t(sd, p + ".block.1.weight"), _t(sd, p + ".block.1.bias"), padding=1))
    x = _norm(sd, p + ".block.3", x)
    return F.relu(F.conv2d(x, _t(sd, p + ".block.4.weight"), _t(sd, p + ".block.4.bias"), padding=1))


def forward_maps(sd, z12):
    """_forward_impl + sigmoid: [B, 3, 16 h, 16 w] float64."""
    z12 = z12.to(torch.float64)
    z9 = deconv_block(sd, "deconv1", z12)
    z6 = deconv_block(sd, "deconv2", z9)
    z3 = deconv_block(sd, "deconv3", z6)
    z0 = deconv_block(sd, "deconv4", z3)
    x = conv_block(sd, "base", z12)
    for i, skip in enumerate((z9, z6, z3)):
        x = upsampler(sd, f"decoder.samplers.{i}", x)
        x = conv_block(sd, f"decoder.blocks.{i}", torch.cat([x, skip], 1))
    x = upsampler(sd, "deconv_out", x)
    x = conv_block(sd, "decoder_head", torch.cat([x, z0], 1))
    return torch.sigmoid(F.conv2d(x, _t(sd, "out_conv.weight"), _t(sd, "out_conv.bias")))


def postprocess_masks(maps, input_size, original_size, img_size=1024):
    x = F.interpolate(maps, (img_size, img_size), mode="bilinear", align_corners=False)
    x = x[..., :input_size[0], :input_size[1]]
    return F.interpolate(x, tuple(original_size), mode="bilinear", align_corners=False)


def seeded_state(emb=256, feats=(512, 256, 128, 64), deconv=(256, 128, 64, 64), head_in=64, transposed=False, affine=False,
                 seed=0):
    """A UNETR decoder state dict with torch's default init scale (kaiming-uniform bound 1 / sqrt(fan_in)) and BatchNorm
    statistics away from identity.  The default is the production plan."""
    g = torch.Generator().manual_seed(seed)

    def u(shape, fan_in):
        return (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / fan_in ** 0.5

    sd = {}

    def sampler(p, cin, cout):
        if transposed:
            sd[p + ".block.weight"], sd[p + ".block.bias"] = u((cin, cout, 2, 2), cout * 4), u((cout,), cout * 4)
        else:
            sd[p + ".conv.weight"], sd[p + ".conv.bias"] = u((cout, cin, 1, 1), cin), u((cout,), cin)

    def conv(p, cin, cout, k=3):
        sd[p + ".weight"], sd[p + ".bias"] = u((cout, cin, k, k), cin * k * k), u((cout,), cin * k * k)

    def block(p, cin, cout):
        if affine:
            for j, c in ((0, cin), (3, cout)):
                sd[f"{p}.block.{j}.weight"] = 1 + 0.2 * u((c,), 1)
                sd[f"{p}.block.{j}.bias"] = 0.2 * u((c,), 1)
        conv(p + ".block.1", cin, cout)
        conv(p + ".block.4", cout, cout)

    cin = emb
    for i, c in enumerate(deconv, 1):
        sampler(f"deconv{i}.block.0", cin, c)
        conv(f"deconv{i}.block.1.block", c, c)
        sd[f"deconv{i}.block.2.weight"] = 1 + 0.2 * u((c,), 1)
        sd[f"deconv{i}.block.2.bias"] = 0.2 * u((c,), 1)
        sd[f"deconv{i}.block.2.running_mean"] = 0.1 * u((c,), 1)
        sd[f"deconv{i}.block.2.running_var"] = 1 + 0.5 * u((c,), 1).abs()
        sd[f"deconv{i}.block.2.num_batches_tracked"] = torch.tensor(0)
        cin = c
    block("base", emb, feats[0])
    for i in range(3):
        sampler(f"decoder.samplers.{i}", feats[i], feats[i + 1])
        block(f"decoder.blocks.{i}", feats[i + 1] + deconv[i], feats[i + 1])
    sampler("deconv_out", feats[3], head_in)
    block("decoder_head", head_in + deconv[3], head_in)
    conv("out_conv", head_in, 3, k=1)
    return {k: v.to(torch.float32) if v.is_floating_point() else v for k, v in sd.items()}
