"""Float64 restatement of the UNETR decoder in training mode (BatchNorm on batch statistics), with autograd: the reference
of the decoder's backward pass.  Layers as oracle/unetr_ref.py applies them; every float tensor of the state dict becomes a
float64 leaf that requires grad.  Also the distance-based Dice loss as DESIGN.md section 2 restates it."""
import torch
import torch.nn.functional as F

from oracle import unetr_ref

EPS = 1e-5


def leaves(sd):
    """float64 copies of the state dict's weights as leaves that require grad (running statistics and counters as they are)"""
    out = {}
    for k, v in sd.items():
        if v.is_floating_point() and not k.endswith(("running_mean", "running_var")):
            out[k] = v.detach().to(torch.float64).clone().requires_grad_(True)
        else:
            out[k] = v.detach().clone().to(torch.float64) if v.is_floating_point() else v.detach().clone()
    return out


def deconv_block(sd, p, x, train):
    x = unetr_ref.upsampler(sd, p + ".block.0", x)
    x = F.conv2d(x, sd[p + ".block.1.block.weight"], sd[p + ".block.1.block.bias"], padding=1)
    x = F.batch_norm(x, sd[p + ".block.2.running_mean"], sd[p + ".block.2.running_var"], sd[p + ".block.2.weight"],
                     sd[p + ".block.2.bias"], training=train, momentum=0.1, eps=EPS)
    return F.relu(x)


def forward_maps(sd, z12, train=True):
    """_forward_impl + sigmoid in float64; with `train` BatchNorm uses batch statistics and updates sd's running statistics"""
    z12 = z12.to(torch.float64)
    z9 = deconv_block(sd, "deconv1", z12, train)
    z6 = deconv_block(sd, "deconv2", z9, train)
    z3 = deconv_block(sd, "deconv3", z6, train)
    z0 = deconv_block(sd, "deconv4", z3, train)
    x = unetr_ref.conv_block(sd, "base", z12)
    for i, skip in enumerate((z9, z6, z3)):
        x = unetr_ref.upsampler(sd, f"decoder.samplers.{i}", x)
        x = unetr_ref.conv_block(sd, f"decoder.blocks.{i}", torch.cat([x, skip], 1))
    x = unetr_ref.upsampler(sd, "deconv_out", x)
    x = unetr_ref.conv_block(sd, "decoder_head", torch.cat([x, z0], 1))
    return torch.sigmoid(F.conv2d(x, sd["out_conv.weight"], sd["out_conv.bias"]))


def crop_resize(maps, input_size, original_size):
    """postprocess_masks after the identity resize to the decoder's output size"""
    x = maps[..., :input_size[0], :input_size[1]]
    return F.interpolate(x, tuple(original_size), mode="bilinear", align_corners=False)


def dice_based_distance_loss(x, y, mask_distances_in_bg=True, eps=1e-7):
    """sum over the 3 channels of 1 - 2 sum(x y) / max(sum x^2 + sum y^2, eps), each channel over the whole batch; with the
    mask, channels 1 and 2 of both x and y times y[:, 0]"""
    loss = 0.0
    for k in range(3):
        xk, yk = x[:, k], y[:, k]
        if mask_distances_in_bg and k > 0:
            xk, yk = xk * y[:, 0], yk * y[:, 0]
        d = ((xk * xk).sum() + (yk * yk).sum()).clamp(min=eps)
        loss = loss + 1.0 - 2.0 * (xk * yk).sum() / d
    return loss


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-300))
