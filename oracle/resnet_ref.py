"""float64 oracle of openai-CLIP's ModifiedResNet image tower (RN50 / RN101 / RN50x4 / RN50x16 / RN50x64), written from the
published architecture (Radford et al. 2021, openai/CLIP model.py's structure):

  stem        relu(bn1(conv1 3x3 s2)) -> relu(bn2(conv2 3x3)) -> relu(bn3(conv3 3x3)) -> AvgPool2d(2)
  bottleneck  relu(bn1(conv1 1x1)) -> relu(bn2(conv2 3x3)) -> AvgPool2d(stride) -> bn3(conv3 1x1); identity or
              AvgPool2d(stride) -> downsample.0 (1x1) -> downsample.1 (BN); relu(main + identity)
  attnpool    tokens = [mean, pixels (NHWC order)] + positional_embedding; multi-head attention with separate q / k / v
              projections, q scaled by 64^-1/2, token 0 the only query; c_proj

BatchNorm is evaluated unfolded (eval mode, eps 1e-5).  `fold()` gives what the engine uploads: each conv with its BN
folded in float64, the weight rounded through float32 to fp16 and the bias to float32; `ResnetRef(sd, folded=True)`
runs on those.  Everything is differentiable, so torch.autograd gives the VJP at any input for the backward tests.

`vjp_at(masks, x, de, tokens=...)` is the VJP at GIVEN forward values: every ReLU multiplies by a fixed 0 / 1 mask (taken
from the engine's stored fp16 activations) instead of testing its own float64 input, and the attention pool is
differentiated at the given tokens, so the comparison is free of the mask flips and softmax shifts that fp16 forward
values cause.  Mask keys: 'conv1' .. 'conv3' for the stem, 'layerS.i.a' / '.b' / '.y' for a
block's two inner ReLUs and its output.
"""
import torch
import torch.nn.functional as F

EPS = 1e-5


def _blocks(sd):
    return [len({k.split(".")[2] for k in sd if k.startswith(f"visual.layer{s}.")}) for s in (1, 2, 3, 4)]


def fold_conv(sd, conv, bn):
    """(weight, bias) of conv `conv` with BatchNorm `bn` folded in, float64, weight rounded as the engine stores it."""
    w = sd[conv + ".weight"].double()
    s = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + EPS)
    b = sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * s
    wf = (w * s.view(-1, 1, 1, 1)).float().half().double()
    return wf, b.float().double()


class ResnetRef:
    """The tower of one CLIP state_dict ('visual.*' keys).  folded=True runs on fold()'s weights (the engine's numbers in
    float64), folded=False on the raw convs and BatchNorms."""

    def __init__(self, sd, folded=False):
        self.sd = {k: v for k, v in sd.items() if k.startswith("visual.")}
        self.blocks = _blocks(self.sd)
        self.folded = folded
        self._fold = self.fold() if folded else None
        self.heads = self.sd["visual.attnpool.q_proj.weight"].shape[0] // 64
        self.masks = None

    def relu(self, t, key):
        return torch.relu(t) if self.masks is None else t * self.masks[key]

    def vjp_at(self, masks, x, de, drop=None, tokens=None):
        """d (e . de) / d x with every ReLU replaced by the given masks (float64 tensors shaped like its output); masks
        None keeps the float64 ReLUs.  tokens [B, T, C]: the attention pool's Jacobian is taken at these token values
        (the engine's), the only non-linear step left once the masks are fixed.  drop: as features()."""
        self.masks = masks
        try:
            x = x.detach().double().requires_grad_(True)
            t = self.tokens(self.features(x, drop)[1][-1])
            if tokens is not None:
                t = tokens.double() + (t - t.detach())
            (g,) = torch.autograd.grad(self.attnpool(t), x, de.double())
        finally:
            self.masks = None
        return g

    def fold(self):
        """{conv name: (weight, bias)} for every conv of the tower (stem conv1..3, blocks, downsample.0)."""
        out = {}
        for i in (1, 2, 3):
            out[f"conv{i}"] = fold_conv(self.sd, f"visual.conv{i}", f"visual.bn{i}")
        for s, n in enumerate(self.blocks):
            for i in range(n):
                p = f"layer{s + 1}.{i}"
                for j in (1, 2, 3):
                    out[f"{p}.conv{j}"] = fold_conv(self.sd, f"visual.{p}.conv{j}", f"visual.{p}.bn{j}")
                if f"visual.{p}.downsample.0.weight" in self.sd:
                    out[f"{p}.downsample"] = fold_conv(self.sd, f"visual.{p}.downsample.0", f"visual.{p}.downsample.1")
        return out

    def conv_bn(self, x, name, conv, bn, stride=1):
        """conv (same padding) followed by its eval-mode BatchNorm, or the folded conv with bias."""
        if self.folded:
            w, b = self._fold[name]
            return F.conv2d(x, w, b, stride=stride, padding=w.shape[-1] // 2)
        w = self.sd[conv + ".weight"].double()
        y = F.conv2d(x, w, None, stride=stride, padding=w.shape[-1] // 2)
        sd = self.sd
        s = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + EPS)
        return (y - sd[bn + ".running_mean"].double().view(1, -1, 1, 1)) * s.view(1, -1, 1, 1) + \
            sd[bn + ".bias"].double().view(1, -1, 1, 1)

    def stem(self, x):
        x = self.relu(self.conv_bn(x, "conv1", "visual.conv1", "visual.bn1", stride=2), "conv1")
        x = self.relu(self.conv_bn(x, "conv2", "visual.conv2", "visual.bn2"), "conv2")
        x = self.relu(self.conv_bn(x, "conv3", "visual.conv3", "visual.bn3"), "conv3")
        return F.avg_pool2d(x, 2)

    def block(self, x, s, i, drop=None):
        """drop: 'main' or 'identity' leaves that branch out of the backward (a planted bug for the tests' bounds)"""
        p = f"layer{s + 1}.{i}"
        v = "visual." + p
        stride = 2 if (s > 0 and i == 0) else 1
        out = self.relu(self.conv_bn(x, p + ".conv1", v + ".conv1", v + ".bn1"), p + ".a")
        out = self.relu(self.conv_bn(out, p + ".conv2", v + ".conv2", v + ".bn2"), p + ".b")
        if stride > 1:
            out = F.avg_pool2d(out, stride)
        out = self.conv_bn(out, p + ".conv3", v + ".conv3", v + ".bn3")
        if drop == "main":
            out = out.detach()
        idn = x
        if v + ".downsample.0.weight" in self.sd:
            if stride > 1:
                idn = F.avg_pool2d(idn, stride)
            idn = self.conv_bn(idn, p + ".downsample", v + ".downsample.0", v + ".downsample.1")
        if drop == "identity":
            idn = idn.detach()
        return self.relu(out + idn, p + ".y")

    def tokens(self, x):
        """[B, C, h, w] -> [B, hw + 1, C]: the mean token, then the pixels in row-major order, plus positions."""
        t = x.flatten(2).transpose(1, 2)
        t = torch.cat([t.mean(dim=1, keepdim=True), t], dim=1)
        return t + self.sd["visual.attnpool.positional_embedding"].double()

    def attnpool(self, t):
        """Single-query attention of token 0 over all tokens, then c_proj: [B, T, C] -> [B, D]."""
        p = "visual.attnpool."
        lin = lambda x, nm: x @ self.sd[p + nm + ".weight"].double().T + self.sd[p + nm + ".bias"].double()  # noqa: E731
        B, T, Cc = t.shape
        H = self.heads
        q = lin(t[:, :1], "q_proj").view(B, 1, H, 64).transpose(1, 2) * 64 ** -0.5
        k = lin(t, "k_proj").view(B, T, H, 64).transpose(1, 2)
        v = lin(t, "v_proj").view(B, T, H, 64).transpose(1, 2)
        a = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
        o = (a @ v).transpose(1, 2).reshape(B, Cc)
        return lin(o, "c_proj")

    def features(self, x, drop=None):
        """(stem output, [every block's output]) for an input that is already normalised; drop = (stage, block, branch)
        plants a missing branch gradient in that block"""
        x = self.stem(x)
        stem, outs = x, []
        for s, n in enumerate(self.blocks):
            for i in range(n):
                x = self.block(x, s, i, drop[2] if drop and drop[:2] == (s, i) else None)
                outs.append(x)
        return stem, outs

    def encode_image(self, x, drop=None):
        """[B, 3, R, R] normalised images -> un-normalised embeddings [B, D] (float64)."""
        return self.attnpool(self.tokens(self.features(x.double(), drop)[1][-1]))
