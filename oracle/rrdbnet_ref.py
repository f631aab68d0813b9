"""Restatement of Real-ESRGAN's generator for the tests: RRDBNet(num_in_ch=3, num_out_ch=3, num_feat, num_block,
num_grow_ch, scale=4) as basicsr's rrdbnet_arch defines it, and SuperResolutionDrawer.synth (super_resolution.py:81-83),
which at tile 0 / pre_pad 0 / scale 4 is clamp_with_grad(RRDBNet(z), 0, 1) (real_esrganer.py:62-77, 159-169).

Written from the architecture's description, in the dtype of the input (float32 or float64):
  * every layer is a 3x3 convolution with padding 1 and a bias; LeakyReLU(0.2) after conv1..conv4 of each dense block
    and after conv_up1, conv_up2 and conv_hr;
  * dense block: conv_k reads cat([x, x1, ...]) and the block returns x5 * 0.2 + x;
  * RRDB: rdb3(rdb2(rdb1(x))) * 0.2 + x;  trunk: feat = conv_first(z), feat + conv_body(body(feat));
  * upsampling: nearest x2, conv_up1; nearest x2, conv_up2; then conv_last(lrelu(conv_hr(.))).

`matched=True` evaluates the network at the engine's rounding points (engine_superres.inc): fp16 weights with the dense
block's 0.2 folded into conv5's weights and bias, and straight-through fp16 rounding of every tensor the engine stores
in fp16 (the forward is rounded, the gradient passes unchanged).  Pure torch; no GPU and no reference checkout needed.
"""
import torch
from torch.nn import functional as F

from oracle.ref_path import clamp_with_grad


def _st16(t):
    """Straight-through fp16 rounding: the value of t.half(), the gradient of the identity."""
    return t + (t.to(torch.float16).to(t.dtype) - t).detach()


def num_blocks(sd):
    """The RRDB count of a state_dict (body.{i}.*)."""
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("body."))


def rrdbnet(z, sd, matched=False):
    """RRDBNet(z) [1, 3, 4h, 4w] of z [1, 3, h, w], weights from the checkpoint-keyed state_dict sd."""
    dt = z.dtype
    r = _st16 if matched else (lambda t: t)

    def conv(x, key, scale=1.0):
        w, b = sd[key + ".weight"], sd[key + ".bias"]
        if matched:  # the engine scales in fp32, then rounds the weights to fp16; the bias stays fp32
            w = (w.float() * scale).half().to(dt)
            b = (b.float() * scale).to(dt)
            return F.conv2d(x, w, b, padding=1)
        y = F.conv2d(x, w.to(dt), b.to(dt), padding=1)
        return y * scale if scale != 1.0 else y

    def lrelu(x):
        return F.leaky_relu(x, 0.2)

    def rdb(x, p):
        xs = [x]
        for k in range(1, 5):
            xs.append(r(lrelu(conv(torch.cat(xs, 1), f"{p}.conv{k}"))))
        return r(conv(torch.cat(xs, 1), f"{p}.conv5", 0.2) + x)

    feat = r(conv(r(z), "conv_first"))
    h = feat
    for i in range(num_blocks(sd)):
        out = rdb(rdb(rdb(h, f"body.{i}.rdb1"), f"body.{i}.rdb2"), f"body.{i}.rdb3")
        h = r(out * 0.2 + h)
    feat = r(feat + conv(h, "conv_body"))
    feat = r(lrelu(conv(F.interpolate(feat, scale_factor=2, mode="nearest"), "conv_up1")))
    feat = r(lrelu(conv(F.interpolate(feat, scale_factor=2, mode="nearest"), "conv_up2")))
    return conv(r(lrelu(conv(feat, "conv_hr"))), "conv_last")


def superres_synth(z, sd, matched=False):
    """SuperResolutionDrawer.synth: clamp_with_grad(RRDBNet(z), 0, 1)."""
    return clamp_with_grad(rrdbnet(z, sd, matched), 0, 1)


def latent_from_tensor(t):
    """SuperResolutionDrawer.get_z_from_tensor (super_resolution.py:75-76): bilinear (align_corners=False) resize of
    (t + 1) / 2 to a quarter of its size, rounded down."""
    return F.interpolate((t + 1) / 2, size=(torch.tensor(t.shape[-2:]) // 4).tolist(), mode="bilinear",
                         align_corners=False)
