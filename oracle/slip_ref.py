"""CPU oracle for the SLIP perceptors: a float restatement of the image tower of SLIP_Base (slip.py:84-157).

TEST INFRASTRUCTURE ONLY, like oracle/ref_path.py.  SLIP's `encode_image(x) = visual(x) @ image_projection`
(SLIP/models.py:130-134) with `visual` = timm's VisionTransformer(num_classes=0) (SLIP/models.py:288-331; SLIP was
tested against timm 0.5.0).  timm is not vendored, so the leaf is restated here [UPSTREAM, un-vendored] and cross-checked
against transformers.ViTModel with copied weights (tests/test_slip_perceptor.py); everything in-tree around it
(SLIP_Base.preprocess / encode_image, the checkpoint's `module.` prefix) is pinned by tests/golden/slip_perceptor.npz,
which oracle/make_golden_slip.py writes by running the unmodified slip.py on top of this restatement.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import ref_path as R

IMAGENET_MEAN = (0.485, 0.456, 0.406)  # slip.py:117-121
IMAGENET_STD = (0.229, 0.224, 0.225)


class PatchEmbed(nn.Module):
    """timm PatchEmbed: Conv2d(3, W, P, stride P) with bias, flattened to tokens."""

    def __init__(self, img_size, patch_size, embed_dim):
        super().__init__()
        self.num_patches = (img_size // patch_size) ** 2
        self.proj = nn.Conv2d(3, embed_dim, patch_size, patch_size)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class Attention(nn.Module):
    """timm Attention: qkv Linear with bias (q | k | v, heads contiguous), softmax(q k^T / sqrt(d)) v, proj."""

    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x):
        B, N, C = x.shape
        qkv = self.qkv(x).reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        a = ((q @ k.transpose(-2, -1)) * self.scale).softmax(dim=-1)
        return self.proj((a @ v).transpose(1, 2).reshape(B, N, C))


class Mlp(nn.Module):
    """timm Mlp: fc1, nn.GELU() (exact erf form), fc2."""

    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class Block(nn.Module):
    """timm Block: pre-norm attention and MLP, LayerNorm eps 1e-6."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = Attention(dim, num_heads)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class VisionTransformer(nn.Module):
    """timm 0.5 VisionTransformer(num_classes=0): tokens [cls_token; patches] + pos_embed (no LayerNorm before the
    blocks), the blocks, the final norm, then the class token (pre_logits and head are identities)."""

    def __init__(self, img_size=224, patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0):
        super().__init__()
        self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size, patch_size, embed_dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + 1, embed_dim))
        self.blocks = nn.Sequential(*[Block(embed_dim, num_heads, mlp_ratio) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=1e-6)

    def forward(self, x):
        x = self.patch_embed(x)
        x = torch.cat([self.cls_token.expand(x.shape[0], -1, -1), x], dim=1) + self.pos_embed
        x = self.norm(self.blocks(x))
        return x[:, 0]


class SlipVisual(nn.Module):
    """Holder giving the checkpoint's key names ('visual.*', 'image_projection') and SLIP's encode_image
    (SLIP/models.py:130-134) on ImageNet-normalised input."""

    def __init__(self, input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512):
        super().__init__()
        self.visual = VisionTransformer(input_resolution, patch_size, width, layers, heads)
        self.image_projection = nn.Parameter(torch.zeros(width, output_dim))

    def encode_image(self, x):
        return self.visual(x) @ self.image_projection


def slip_preprocess(imgs):
    """SLIP_Base.preprocess without input_range (slip.py:147-149): global min/max range normalise, then ImageNet
    mean / std (Resize / CenterCrop at 224 are identities for 224x224 cutouts)."""
    minv = imgs.min()
    imgs = imgs - minv
    maxv = imgs.max()
    if maxv != 0:
        imgs = imgs / maxv
    mean = torch.tensor(IMAGENET_MEAN, dtype=imgs.dtype).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=imgs.dtype).view(1, 3, 1, 1)
    return (imgs - mean) / std


def encode_image(model, imgs):
    """SLIP_Base.encode_image (slip.py:151-157): unit embeddings of the preprocessed cutouts."""
    e = model.encode_image(slip_preprocess(imgs))
    return e / e.norm(dim=-1, keepdim=True)


class SlipPerceptor(nn.Module):
    """A SlipVisual behind the interface ref_path.iterate drives: its encode_image receives the CLIP-normalised input
    ref_path.encode_image makes, y = (x01 - clip_mean) / clip_std with x01 the range-normalised cutouts, and maps it
    affinely to SLIP's (x01 - imagenet_mean) / imagenet_std before the tower."""

    def __init__(self, slip_visual):
        super().__init__()
        self.slip = slip_visual

    def encode_image(self, x):
        cm = torch.tensor(R.CLIP_MEAN, dtype=x.dtype).view(1, 3, 1, 1)
        cs = torch.tensor(R.CLIP_STD, dtype=x.dtype).view(1, 3, 1, 1)
        im = torch.tensor(IMAGENET_MEAN, dtype=x.dtype).view(1, 3, 1, 1)
        ist = torch.tensor(IMAGENET_STD, dtype=x.dtype).view(1, 3, 1, 1)
        return self.slip.encode_image((x * cs + cm - im) / ist)


def make_model(arch, state_dict):
    """SlipVisual of an engine.SLIP_ARCH-style dict with `state_dict` loaded strictly, frozen (slip.py:139-140)."""
    m = SlipVisual(arch["image_res"], arch["patch"], arch["width"], arch["layers"], arch["heads"], arch["out_dim"])
    m.load_state_dict(state_dict, strict=True)
    return m.eval().requires_grad_(False)


def gelu(u):
    """nn.GELU() in float64 for the epilogue tests: 0.5 u (1 + erf(u / sqrt 2)) and its derivative Phi(u) + u phi(u)."""
    u = u.double()
    return F.gelu(u), 0.5 * (1 + torch.erf(u / 2 ** 0.5)) + u * torch.exp(-0.5 * u * u) / (2 * torch.pi) ** 0.5
