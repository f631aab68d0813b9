"""CPU oracle: torch-fp32 restatement of pixray's per-iteration hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is imported by the product (pixray_b200/); only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, and only as the checker or
the CPU baseline.

Parity status: the reference's own tests pin nothing on this path (SURVEY.md 4, 8c) -> "parity unpinned" for the
un-vendored third-party leaves restated here (kornia 0.6.2 warps, openai-CLIP VisionTransformer, taming Decoder).
The in-tree parts (Prompt, spherical_dist_loss, vector_quantize, ClampWithGrad, MakeCutouts pooling / group split /
noise, CLIP_Base.preprocess, FastPixelDrawer.synth, Adam + clip_z) ARE pinned: oracle/make_golden.py imports the
real reference (under oracle/shim.py) in the authoring container and writes tests/golden/*.npz, which
tests/test_oracle_golden.py checks this file against.  The ViT restatement is additionally cross-checked against
transformers' CLIPVisionModelWithProjection (hidden_act="quick_gelu") with copied weights.

Every function cites the reference file:line it follows (paths relative to the pixray checkout).
"""
import math
from collections import OrderedDict

import torch
import torch.nn as nn
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)  # slip.py:55
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

# ------------------------------------------------------------------------------------------------ small autograd ops


class _ReplaceGrad(torch.autograd.Function):
    """pixray.py:249-259 / vqgan.py:48-58: forward value of the first arg, gradient routed to the second."""

    @staticmethod
    def forward(ctx, x_forward, x_backward):
        ctx.shape = x_backward.shape
        return x_forward

    @staticmethod
    def backward(ctx, g):
        return None, g.sum_to_size(ctx.shape)


replace_grad = _ReplaceGrad.apply


class _ClampWithGrad(torch.autograd.Function):
    """vqgan.py:66-79: clamp forward; backward keeps the gradient only where it points back into range."""

    @staticmethod
    def forward(ctx, x, lo, hi):
        ctx.lo, ctx.hi = lo, hi
        ctx.save_for_backward(x)
        return x.clamp(lo, hi)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * (g * (x - x.clamp(ctx.lo, ctx.hi)) >= 0), None, None


clamp_with_grad = _ClampWithGrad.apply


def spherical_dist_loss(x, y):
    """pixray.py:262-265."""
    x = F.normalize(x, dim=-1)
    y = F.normalize(y, dim=-1)
    return (x - y).norm(dim=-1).div(2).arcsin().pow(2).mul(2)


def prompt_loss(embeds, embed, weight, stop):
    """Prompt.forward, pixray.py:275-280.  embeds [cutn, D]; embed [n, D]; scalar weight / stop."""
    weight = torch.as_tensor(weight, dtype=embeds.dtype)
    stop = torch.as_tensor(stop, dtype=embeds.dtype)
    input_normed = F.normalize(embeds.unsqueeze(1), dim=2)
    embed_normed = F.normalize(embed.unsqueeze(0), dim=2)
    dists = input_normed.sub(embed_normed).norm(dim=2).div(2).arcsin().pow(2).mul(2)
    dists = dists * weight.sign()
    return weight.abs() * replace_grad(dists, torch.maximum(dists, stop)).mean()


# ------------------------------------------------------------------------------------------------ MakeCutouts


def adaptive_pool_bounds(in_size, out_size):
    """Integer window bounds of Adaptive{Avg,Max}Pool2d (pixray.py:442-443 -> ATen start_index / end_index):
    start = floor(i * in / out), end = ceil((i + 1) * in / out).  Bit-exact bookkeeping, returned as int lists."""
    starts = [(i * in_size) // out_size for i in range(out_size)]
    ends = [-((-(i + 1) * in_size) // out_size) for i in range(out_size)]
    return starts, ends


def pool_avg_max(img, cut_size):
    """pixray.py:463: (av_pool(input) + max_pool(input)) / 2 on the whole image -> [1, C, cs, cs]."""
    return (F.adaptive_avg_pool2d(img, (cut_size, cut_size)) + F.adaptive_max_pool2d(img, (cut_size, cut_size))) / 2


def _normal_transform_pixel(h, w):
    """kornia 0.6.2 normal_transform_pixel: pixel -> [-1, 1] with the (size-1)/2 convention."""
    eps = 1e-14
    tr = torch.tensor([[1.0, 0.0, -1.0], [0.0, 1.0, -1.0], [0.0, 0.0, 1.0]])
    tr[0, 0] = tr[0, 0] * 2.0 / (w - 1.0 if w != 1 else eps)
    tr[1, 1] = tr[1, 1] * 2.0 / (h - 1.0 if h != 1 else eps)
    return tr[None]


def normalize_homography(dst_pix_trans_src_pix, dsize_src, dsize_dst):
    """kornia 0.6.2 normalize_homography (used by warp_perspective, pixray.py:482-485)."""
    src_h, src_w = dsize_src
    dst_h, dst_w = dsize_dst
    src_norm_trans_src_pix = _normal_transform_pixel(src_h, src_w).to(dst_pix_trans_src_pix)
    src_pix_trans_src_norm = torch.inverse(src_norm_trans_src_pix)
    dst_norm_trans_dst_pix = _normal_transform_pixel(dst_h, dst_w).to(dst_pix_trans_src_pix)
    return dst_norm_trans_dst_pix @ (dst_pix_trans_src_pix @ src_pix_trans_src_norm)


def _transform_points(trans, pts):
    """kornia transform_points on a [B, H, W, 2] grid with [B, 3, 3] transforms (homogeneous divide, eps 1e-8)."""
    ones = torch.ones_like(pts[..., :1])
    ph = torch.cat([pts, ones], dim=-1)  # B,H,W,3
    out = torch.einsum("bij,bhwj->bhwi", trans, ph)
    z = out[..., 2:3]
    scale = torch.where(z.abs() > 1e-8, 1.0 / z, torch.ones_like(z))
    return out[..., :2] * scale


def warp_grid(M, src_hw, dst_hw):
    """Sampling grid of kornia warp_perspective(src, M, dsize) in normalised coords, [B, h_out, w_out, 2]."""
    B = M.shape[0]
    h_out, w_out = dst_hw
    dst_norm_trans_src_norm = normalize_homography(M, src_hw, dst_hw)
    src_norm_trans_dst_norm = torch.inverse(dst_norm_trans_src_norm)
    xs = torch.linspace(-1, 1, w_out)
    ys = torch.linspace(-1, 1, h_out)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    grid = torch.stack([gx, gy], dim=-1)[None].repeat(B, 1, 1, 1).to(M.dtype)
    return _transform_points(src_norm_trans_dst_norm, grid)


def warp_perspective(src, M, dsize, padding_mode="zeros", fill_value=None, align_corners=True):
    """kornia 0.6.2 warp_perspective as called on MakeCutouts' cached path (pixray.py:480-486; default
    align_corners=True, bilinear).  padding_mode 'fill' = grid_sample(zeros) + (1 - grid_sample(ones)) * fill
    (kornia _fill_and_warp; pixray.py:351-352, 364-365, 484-485)."""
    grid = warp_grid(M, src.shape[-2:], dsize)
    if padding_mode == "fill":
        ones = torch.ones_like(src)
        inv = 1 - F.grid_sample(ones, grid, align_corners=align_corners, mode="bilinear", padding_mode="zeros")
        fv = torch.as_tensor(fill_value, dtype=src.dtype).reshape(1, -1, 1, 1)
        return F.grid_sample(src, grid, align_corners=align_corners, mode="bilinear", padding_mode="zeros") + inv * fv
    return F.grid_sample(src, grid, align_corners=align_corners, mode="bilinear", padding_mode=padding_mode)


def rescale_for_aspect(pooled, aspect):
    """pixray.py:468-472: kornia.geometry.transform.rescale(cutout, (1, aspect)) / ((1 / aspect, 1)) -- kornia 0.6.2 rescale
    is resize(input, (int(h * fv), int(w * fh)), 'bilinear', align_corners=None), i.e. F.interpolate(..., align_corners=False)
    [UPSTREAM, un-vendored]."""
    if aspect == 1.0:
        return pooled
    h, w = pooled.shape[-2:]
    size = (int(h * 1), int(w * aspect)) if aspect > 1.0 else (int(h * (1.0 / aspect)), int(w * 1))
    return F.interpolate(pooled, size=size, mode="bilinear", align_corners=False)


def make_cutouts(img, transforms, cut_size, zoom_padding, fill, noise_facs=None, noise=None, cutn_zoom=None,
                 jitter=None, aspect=1.0, spot=None, spot_mask=None):
    """MakeCutouts.forward on explicit (cached) transforms, pixray.py:445-511.

    img [1, 3, H, W]; transforms [cutn, 3, 3]; zoom group = first int(0.6 * cutn) (pixray.py:407) warped with
    `zoom_padding` ('reflection' | 'border'); wide group with constant grey `fill`; then ColorJitter on the rows of
    `jitter` (the live stacks' last stage, pixray.py:416, 436), then batch + facs * noise (pixray.py:508-510)
    when both are given."""
    cutn = transforms.shape[0]
    if cutn_zoom is None:
        cutn_zoom = int(0.6 * cutn)
    pooled = pool_avg_max(img, cut_size)  # identical for every cutout (pixray.py:461-478)
    if spot is not None:
        # pixray.py:453-466: spot == 0 zeroes mask_indexes_off (mask < 0.5), anything else zeroes mask_indexes (mask >= 0.5);
        # spot_mask: bool [3, cs, cs] = mask_image_tensor.ge(0.5) of fetch_spot_indexes (pixray.py:370-394)
        sel = ~spot_mask if spot == 0 else spot_mask
        pooled = pooled.masked_fill(sel[None], 0.0)
    pooled = rescale_for_aspect(pooled, aspect)  # global_aspect_width != 1 (pixray.py:468-472)
    src = pooled.expand(cutn, -1, -1, -1)
    parts = []
    if cutn_zoom > 0:
        parts.append(warp_perspective(src[:cutn_zoom], transforms[:cutn_zoom], (cut_size, cut_size),
                                      padding_mode=zoom_padding))
    if cutn_zoom < cutn:
        parts.append(warp_perspective(src[cutn_zoom:], transforms[cutn_zoom:], (cut_size, cut_size),
                                      padding_mode="fill", fill_value=[fill, fill, fill]))
    batch = torch.cat(parts)
    if jitter is not None:
        batch = color_jitter(batch, jitter)
    if noise_facs is not None and noise is not None:
        batch = batch + noise_facs.reshape(cutn, 1, 1, 1) * noise
    return batch


# K.ColorJitter(hue=0.1, saturation=0.1, p=0.8, return_transform=True): last stage of augs_zoom and augs_wide
# (pixray.py:416, 436).  kornia==0.6.2 (requirements.txt) is not vendored under /root/reference and not installed here:
# the functions below restate its published algorithm (kornia/color/hsv.py rgb_to_hsv / hsv_to_rgb,
# kornia/enhance/adjust.py adjust_{brightness,contrast,saturation,hue}, kornia/augmentation ColorJitter.apply_transform
# with random_color_jitter_generator's parameters).  Parity for this stage is therefore UNPINNED against kornia itself;
# it is anchored on the reference's call site (which factors, which probability) and on the kernel matching this
# restatement forward and backward; the rgb<->hsv maps themselves are cross-checked against OpenCV's float conversions and
# the standard library's colorsys (tests/test_color_jitter.py::test_oracle_hsv_maps_agree_with_opencv_and_colorsys).


def rgb_to_hsv(image, eps=1e-8):
    """kornia.color.rgb_to_hsv: [*, 3, H, W] in [0, 1] -> h in [0, 2pi), s, v."""
    max_rgb, argmax_rgb = image.max(-3)
    min_rgb, _ = image.min(-3)
    deltac = max_rgb - min_rgb
    v = max_rgb
    s = deltac / (max_rgb + eps)
    deltac = torch.where(deltac == 0, torch.ones_like(deltac), deltac)
    rc, gc, bc = torch.unbind(max_rgb.unsqueeze(-3) - image, dim=-3)
    h = torch.stack(((bc - gc), (rc - bc) + 2.0 * deltac, (gc - rc) + 4.0 * deltac), dim=-3) / deltac.unsqueeze(-3)
    h = torch.gather(h, dim=-3, index=argmax_rgb.unsqueeze(-3)).squeeze(-3)
    h = (h / 6.0) % 1.0
    h = 2.0 * math.pi * h
    return torch.stack((h, s, v), dim=-3)


def hsv_to_rgb(image):
    """kornia.color.hsv_to_rgb: h in radians."""
    h = image[..., 0, :, :] / (2 * math.pi)
    s = image[..., 1, :, :]
    v = image[..., 2, :, :]
    hi = torch.floor(h * 6) % 6
    f = ((h * 6) % 6) - hi
    p = v * (1.0 - s)
    q = v * (1.0 - f * s)
    t = v * (1.0 - (1.0 - f) * s)
    hi = hi.long()
    indices = torch.stack([hi, hi + 6, hi + 12], dim=-3)
    out = torch.stack((v, q, p, p, t, v, t, v, v, q, p, p, p, p, t, v, v, q), dim=-3)
    return torch.gather(out, -3, indices)


def _adjust_saturation(x, factor):
    hsv = rgb_to_hsv(x)
    h, s, v = torch.chunk(hsv, 3, dim=-3)
    return hsv_to_rgb(torch.cat([h, torch.clamp(s * factor, 0, 1), v], dim=-3))


def _adjust_hue(x, factor_rad):
    hsv = rgb_to_hsv(x)
    h, s, v = torch.chunk(hsv, 3, dim=-3)
    return hsv_to_rgb(torch.cat([torch.fmod(h + factor_rad, 2 * math.pi), s, v], dim=-3))


def jitter_code(order):
    """Pack an application order (a permutation of 0 brightness, 1 contrast, 2 saturation, 3 hue) as the engine does."""
    return 256 + order[0] + 4 * order[1] + 16 * order[2] + 64 * order[3]


def color_jitter(batch, jitter):
    """ColorJitter.apply_transform on the cutouts its Bernoulli(p) selected.  jitter [n, 3] float32 rows
    {code, saturation_factor, hue_factor}: code 0 = not selected, else jitter_code(order); brightness=contrast=0 at
    the call site, so those two stages are adjust_brightness(x, 0) / adjust_contrast(x, 1) = clamp(x, 0, 1)."""
    out = []
    for n in range(batch.shape[0]):
        x = batch[n:n + 1]
        code = int(jitter[n, 0])
        if code:
            sat = jitter[n, 1].to(x.dtype)
            hue = jitter[n, 2].to(x.dtype) * 2 * math.pi
            for k in range(4):
                op = (code >> (2 * k)) & 3
                if op == 0:
                    x = torch.clamp(x + 0.0, 0.0, 1.0)
                elif op == 1:
                    x = torch.clamp(x * 1.0, 0.0, 1.0)
                elif op == 2:
                    x = _adjust_saturation(x, sat)
                else:
                    x = _adjust_hue(x, hue)
        out.append(x)
    return torch.cat(out)


# ------------------------------------------------------------------------------------------------ filters (filters/*.py)
# FilterInterface.forward(img) -> (img, loss), applied to the drawer's output before MakeCutouts (do_synth_and_filter,
# pixray.py:1203-1222).  The reference draws rand_w = randint(0, W) and rand_h = randint(0, H) inside forward; here they are
# arguments so that both sides of a parity test use the same draws.


def filter_tiler(img, rand_h, rand_w):
    """filters/tiler.py:16-23."""
    return torch.roll(img, shifts=(rand_h, rand_w), dims=(2, 3)), torch.zeros(())


def filter_wallpaper(img, wallpaper_type, edge_match, rand_h, rand_w):
    """filters/wallpaper.py:27-93."""
    loss = torch.zeros(())
    B, C, H, W = img.shape
    em, em2 = edge_match, int(edge_match / 2)
    if wallpaper_type == "shift":
        row2 = torch.roll(img, shifts=(int(W / 2),), dims=(3,))
        return torch.roll(torch.cat([img, row2], dim=2), shifts=(rand_h, rand_w), dims=(2, 3)), loss
    if wallpaper_type == "horizontal":
        if em != 0:
            loss = F.mse_loss(img[:, :, :, :em], img[:, :, :, -em:]) / em
            img = img[:, :, :, em2:-em2]
        return torch.roll(img, shifts=(rand_w,), dims=(3,)), loss
    if wallpaper_type == "vertical":
        if em != 0:
            loss = F.mse_loss(img[:, :, :em, :], img[:, :, -em:, :]) / em
            img = img[:, :, em2:-em2, :]
        return torch.roll(img, shifts=(rand_h,), dims=(2,)), loss
    if em != 0:
        loss1 = F.mse_loss(img[:, :, :, :em], img[:, :, :, -em:]) / em
        img = img[:, :, :, em2:-em2]
        loss2 = F.mse_loss(img[:, :, :em, :], img[:, :, -em:, :]) / em
        img = img[:, :, em2:-em2, :]
        loss = loss1 + loss2
    return torch.roll(img, shifts=(rand_h, rand_w), dims=(2, 3)), loss


COLORLOOKUP_DEFAULT_TABLE = [[0, 0, 0], [255, 255, 255], [63, 40, 50], [38, 43, 68], [90, 105, 136], [139, 155, 180],
                             [25, 60, 62], [38, 92, 66], [62, 137, 72], [99, 199, 77], [254, 231, 97], [254, 174, 52],
                             [254, 174, 52], [247, 118, 34], [184, 111, 80], [116, 63, 57]]  # colorlookup.py:10-26


def filter_colorlookup(img, color_table=None, beta=10.0):
    """filters/colorlookup.py:51-86 (3-channel path): nearest table colour, straight-through value, VQ-style loss.  The
    table takes the image's dtype (float32 in the reference)."""
    if color_table is None:
        color_table = [[c / 255.0 for c in rgb] for rgb in COLORLOOKUP_DEFAULT_TABLE]
    table = torch.as_tensor(color_table, dtype=img.dtype)
    z3 = img.permute(0, 2, 3, 1).contiguous()
    ind = torch.cdist(z3, table).argmin(dim=-1)
    z_q = torch.index_select(table, 0, ind.flatten()).view(z3.shape)
    loss = beta * torch.mean((z_q.detach() - z3) ** 2) + torch.mean((z_q - z3.detach()) ** 2)
    z_q = z3 + (z_q - z3).detach()
    return z_q.permute(0, 3, 1, 2).contiguous(), loss


# ------------------------------------------------------------------------------------------------ perceptor


def clip_preprocess(imgs):
    """CLIP_Base.preprocess, slip.py:21-42, 52-60: global min/max range normalise, then per-channel mean/std.
    (Resize / CenterCrop at 224 are identities for 224x224 cutouts.)"""
    minv = imgs.min()
    imgs = imgs - minv
    maxv = imgs.max()
    if maxv != 0:
        imgs = imgs / maxv
    mean = torch.tensor(CLIP_MEAN, dtype=imgs.dtype).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, dtype=imgs.dtype).view(1, 3, 1, 1)
    return (imgs - mean) / std


class QuickGELU(nn.Module):
    """SLIP/models.py:27-29."""

    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class ResidualAttentionBlock(nn.Module):
    """SLIP/models.py:32-53 (vendored copy of openai-CLIP's block): pre-LN MHA + pre-LN MLP with QuickGELU."""

    def __init__(self, d_model, n_head):
        super().__init__()
        self.attn = nn.MultiheadAttention(d_model, n_head)
        self.ln_1 = nn.LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(d_model, d_model * 4)), ("gelu", QuickGELU()),
                                              ("c_proj", nn.Linear(d_model * 4, d_model))]))
        self.ln_2 = nn.LayerNorm(d_model)

    def forward(self, x):
        h = self.ln_1(x)
        x = x + self.attn(h, h, h, need_weights=False)[0]
        return x + self.mlp(self.ln_2(x))


class Transformer(nn.Module):
    """SLIP/models.py:56-64."""

    def __init__(self, width, layers, heads):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(*[ResidualAttentionBlock(width, heads) for _ in range(layers)])

    def forward(self, x):
        return self.resblocks(x)


class VisionTransformer(nn.Module):
    """openai-CLIP clip/model.py VisionTransformer [UPSTREAM, un-vendored; call sites slip.py:49-50, 65]."""

    def __init__(self, input_resolution, patch_size, width, layers, heads, output_dim):
        super().__init__()
        self.input_resolution, self.output_dim = input_resolution, output_dim
        self.conv1 = nn.Conv2d(3, width, patch_size, patch_size, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = Transformer(width, layers, heads)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))

    def forward(self, x):
        x = self.conv1(x)
        x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
        cls = self.class_embedding.to(x.dtype) + torch.zeros(x.shape[0], 1, x.shape[-1], dtype=x.dtype)
        x = torch.cat([cls, x], dim=1) + self.positional_embedding.to(x.dtype)
        x = self.ln_pre(x)
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        x = self.ln_post(x[:, 0, :])
        return x @ self.proj


class ClipVisual(nn.Module):
    """Holder giving the state_dict the reference's key names ('visual.*') and `encode_image` (slip.py:65)."""

    def __init__(self, input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512):
        super().__init__()
        self.visual = VisionTransformer(input_resolution, patch_size, width, layers, heads, output_dim)

    def encode_image(self, x):
        return self.visual(x)


def init_clip_weights(model, seed=0):
    """Seeded synthetic CLIP-style init (pattern of SLIP/models.py:106-120; no pretrained weights offline)."""
    g = torch.Generator().manual_seed(seed)
    v = model.visual
    W, L = v.transformer.width, v.transformer.layers
    proj_std, attn_std, fc_std = (W ** -0.5) * ((2 * L) ** -0.5), W ** -0.5, (2 * W) ** -0.5
    with torch.no_grad():
        v.conv1.weight.copy_(torch.randn(v.conv1.weight.shape, generator=g) * (3 * v.conv1.kernel_size[0] ** 2) ** -0.5)
        v.class_embedding.copy_(torch.randn(W, generator=g) * W ** -0.5)
        v.positional_embedding.copy_(torch.randn(v.positional_embedding.shape, generator=g) * 0.01)
        v.proj.copy_(torch.randn(v.proj.shape, generator=g) * W ** -0.5)
        for blk in v.transformer.resblocks:
            blk.attn.in_proj_weight.copy_(torch.randn(blk.attn.in_proj_weight.shape, generator=g) * attn_std)
            blk.attn.in_proj_bias.copy_(torch.randn(3 * W, generator=g) * 0.02)
            blk.attn.out_proj.weight.copy_(torch.randn(W, W, generator=g) * proj_std)
            blk.attn.out_proj.bias.copy_(torch.randn(W, generator=g) * 0.02)
            blk.mlp.c_fc.weight.copy_(torch.randn(4 * W, W, generator=g) * fc_std)
            blk.mlp.c_fc.bias.copy_(torch.randn(4 * W, generator=g) * 0.02)
            blk.mlp.c_proj.weight.copy_(torch.randn(W, 4 * W, generator=g) * proj_std)
            blk.mlp.c_proj.bias.copy_(torch.randn(W, generator=g) * 0.02)
            for ln in (blk.ln_1, blk.ln_2):
                ln.weight.copy_(1 + 0.1 * torch.randn(W, generator=g))
                ln.bias.copy_(0.05 * torch.randn(W, generator=g))
        for ln in (v.ln_pre, v.ln_post):
            ln.weight.copy_(1 + 0.1 * torch.randn(W, generator=g))
            ln.bias.copy_(0.05 * torch.randn(W, generator=g))
    return model.eval().requires_grad_(False)  # slip.py:176


def encode_image(model, imgs):
    """CLIP_Base.encode_image, slip.py:62-66."""
    e = model.encode_image(clip_preprocess(imgs))
    return e / e.norm(dim=-1, keepdim=True)


# ------------------------------------------------------------------------------------------------ VQGAN drawer


def vector_quantize(x, codebook):
    """vqgan.py:60-64.  Returns (straight-through quantised x, argmin indices)."""
    d = x.pow(2).sum(dim=-1, keepdim=True) + codebook.pow(2).sum(dim=1) - 2 * x @ codebook.T
    indices = d.argmin(-1)
    x_q = F.one_hot(indices, codebook.shape[0]).to(d.dtype) @ codebook
    return replace_grad(x_q, x), indices


def _swish(x):
    return x * torch.sigmoid(x)


def _gn(c):
    return nn.GroupNorm(32, c, eps=1e-6, affine=True)


class ResnetBlock(nn.Module):
    """taming.modules.diffusionmodules.model.ResnetBlock with temb_channels=0 [UPSTREAM, un-vendored]."""

    def __init__(self, cin, cout):
        super().__init__()
        self.norm1, self.conv1 = _gn(cin), nn.Conv2d(cin, cout, 3, 1, 1)
        self.norm2, self.conv2 = _gn(cout), nn.Conv2d(cout, cout, 3, 1, 1)
        if cin != cout:
            self.nin_shortcut = nn.Conv2d(cin, cout, 1, 1, 0)

    def forward(self, x):
        h = self.conv1(_swish(self.norm1(x)))
        h = self.conv2(_swish(self.norm2(h)))
        if hasattr(self, "nin_shortcut"):
            x = self.nin_shortcut(x)
        return x + h


class AttnBlock(nn.Module):
    """taming AttnBlock: GN -> q,k,v 1x1 -> softmax(q^T k * C^-1/2) -> proj 1x1, residual [UPSTREAM]."""

    def __init__(self, c):
        super().__init__()
        self.norm = _gn(c)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(c, c, 1) for _ in range(4))

    def forward(self, x):
        h = self.norm(x)
        q, k, v = self.q(h), self.k(h), self.v(h)
        b, c, hh, ww = q.shape
        q = q.reshape(b, c, hh * ww).permute(0, 2, 1)
        k = k.reshape(b, c, hh * ww)
        w_ = torch.softmax(torch.bmm(q, k) * (int(c) ** -0.5), dim=2)
        v = v.reshape(b, c, hh * ww)
        h = torch.bmm(v, w_.permute(0, 2, 1)).reshape(b, c, hh, ww)
        return x + self.proj_out(h)


class _Up(nn.Module):
    pass


class _Upsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, 1, 1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class Decoder(nn.Module):
    """taming Decoder (vqgan.py:195 via model.decode) [UPSTREAM].  Module names mirror the checkpoint keys."""

    def __init__(self, ch=128, out_ch=3, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2, attn_resolutions=(16,),
                 resolution=256, z_channels=256):
        super().__init__()
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        block_in = ch * ch_mult[-1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        ups = []
        for i_level in reversed(range(self.num_resolutions)):
            up = _Up()
            up.block, up.attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(num_res_blocks + 1):
                up.block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    up.attn.append(AttnBlock(block_in))
            if i_level != 0:
                up.upsample = _Upsample(block_in)
                curr_res *= 2
            ups.insert(0, up)
        self.up = nn.ModuleList(ups)
        self.norm_out = _gn(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)

    def forward(self, z):
        h = self.conv_in(z)
        h = self.mid.block_2(self.mid.attn_1(self.mid.block_1(h)))
        for i_level in reversed(range(self.num_resolutions)):
            up = self.up[i_level]
            for i_block in range(self.num_res_blocks + 1):
                h = up.block[i_block](h)
                if len(up.attn) > 0:
                    h = up.attn[i_block](h)
            if i_level != 0:
                h = up.upsample(h)
        return self.conv_out(_swish(self.norm_out(h)))


class _Downsample(nn.Module):
    """taming Downsample(with_conv=True): F.pad(x, (0, 1, 0, 1)) then Conv2d(k=3, stride=2, padding=0) [UPSTREAM]."""

    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class Encoder(nn.Module):
    """taming Encoder (VQModel.encode, used by VqganDrawer.init_from_tensor / reapply_from_tensor / get_z_from_tensor,
    vqgan.py:174-185) [UPSTREAM taming/modules/diffusionmodules/model.py, un-vendored: parity unpinned for the leaf; module
    names mirror the checkpoint keys].  double_z = False (the VQ models)."""

    def __init__(self, ch=128, in_channels=3, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2, attn_resolutions=(16,),
                 resolution=256, z_channels=256, **ignore):
        super().__init__()
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.conv_in = nn.Conv2d(in_channels, ch, 3, 1, 1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        block_in = ch
        for i_level in range(self.num_resolutions):
            down = _Up()
            down.block, down.attn = nn.ModuleList(), nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(num_res_blocks):
                down.block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    down.attn.append(AttnBlock(block_in))
            if i_level != self.num_resolutions - 1:
                down.downsample = _Downsample(block_in)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        self.norm_out = _gn(block_in)
        self.conv_out = nn.Conv2d(block_in, z_channels, 3, 1, 1)

    def forward(self, x):
        h = self.conv_in(x)
        for i_level in range(self.num_resolutions):
            down = self.down[i_level]
            for i_block in range(self.num_res_blocks):
                h = down.block[i_block](h)
                if len(down.attn) > 0:
                    h = down.attn[i_block](h)
            if i_level != self.num_resolutions - 1:
                h = down.downsample(h)
        h = self.mid.block_2(self.mid.attn_1(self.mid.block_1(h)))
        return self.conv_out(_swish(self.norm_out(h)))


class VQModel(nn.Module):
    """The slice of taming VQModel pixray uses (vqgan.py:122-142, 174-195): codebook, post_quant_conv, decoder and -- with
    with_encoder -- the encoder + quant_conv behind model.encode."""

    def __init__(self, n_embed=16384, embed_dim=256, with_encoder=False, **dd):
        super().__init__()
        self.quantize = nn.Module()
        self.quantize.embedding = nn.Embedding(n_embed, embed_dim)
        self.post_quant_conv = nn.Conv2d(embed_dim, dd.get("z_channels", 256), 1)
        self.decoder = Decoder(**dd)
        if with_encoder:
            self.encoder = Encoder(**dd)
            self.quant_conv = nn.Conv2d(dd.get("z_channels", 256), embed_dim, 1)

    def decode(self, zq):
        return self.decoder(self.post_quant_conv(zq))

    def encode(self, x):
        """taming VQModel.encode: quantize(quant_conv(encoder(x))) -> (quant [B, C, h, w], indices, pre-quantisation h);
        VectorQuantizer: nearest code by squared L2, value = the codebook row."""
        h = self.quant_conv(self.encoder(x))
        b, c, hh, ww = h.shape
        flat = h.permute(0, 2, 3, 1).reshape(-1, c)
        cb = self.quantize.embedding.weight
        d = flat.pow(2).sum(dim=1, keepdim=True) + cb.pow(2).sum(dim=1) - 2 * flat @ cb.T
        idx = d.argmin(dim=1)
        quant = cb[idx].reshape(b, hh, ww, c).permute(0, 3, 1, 2).contiguous()
        return quant, idx, h


def init_vqgan_weights(model, seed=0):
    """Seeded synthetic weights: default conv init under a fixed seed, GN affine perturbed, codebook spread so the
    argmin is well separated (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name == "quantize.embedding.weight":
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            elif p.dim() == 4:
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 / fan_in) ** 0.5)
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
    return model.eval().requires_grad_(False)  # vqgan.py:125


def vqgan_synth(model, z):
    """VqganDrawer.synth, vqgan.py:190-195.  z [1, C, h, w] -> image [1, 3, H, W] in [0, 1]."""
    zq, _ = vector_quantize(z.movedim(1, 3), model.quantize.embedding.weight)
    return clamp_with_grad(model.decode(zq.movedim(3, 1)).add(1).div(2), 0, 1)


def vqgan_z_bounds(model):
    """vqgan.py:141-142: per-channel codebook min / max, used by clip_z (vqgan.py:202-204)."""
    w = model.quantize.embedding.weight
    return w.min(dim=0).values[None, :, None, None], w.max(dim=0).values[None, :, None, None]


def pixel_synth(z, out_hw):
    """FastPixelDrawer.synth, fast_pixeldrawer.py:89-91: nearest upsample + clamp_with_grad."""
    return clamp_with_grad(F.interpolate(z, size=out_hw, mode="nearest"), 0, 1)


# ------------------------------------------------------------------------------------------------ FFT drawer

# aphantasia.image.to_valid_rgb's colour-correlation matrix [UPSTREAM pixray/aphantasia@7e6b3bb, un-vendored]
_COLOR_SVD_SQRT = ((0.26, 0.09, 0.02), (0.27, 0.00, -0.05), (0.27, -0.09, 0.03))


def fft_freq_scale(h, w, decay_power=1.5, dtype=torch.float32):
    """aphantasia fft_image's per-frequency scale [UPSTREAM]: 1 / max(|f|, 4/max(h,w))**decay * sqrt(w*h) on the
    rfft2 grid (SURVEY.md 8c).  Returns [h, w//2+1] (computed in float64, returned in `dtype`)."""
    import numpy as np
    fy = np.fft.fftfreq(h)[:, None]
    fx = np.fft.fftfreq(w)[: w // 2 + 1]
    freqs = np.sqrt(fx * fx + fy * fy)
    scale = 1.0 / np.maximum(freqs, 4.0 / max(h, w)) ** decay_power
    scale *= np.sqrt(w * h)
    return torch.tensor(scale, dtype=dtype)


def color_matrix(colors=1.5, dtype=torch.float32):
    """to_valid_rgb's colour matrix, first column / colors, over the largest column norm, evaluated in `dtype`."""
    import numpy as np
    nt = np.float64 if dtype == torch.float64 else np.float32
    m = np.asarray(_COLOR_SVD_SQRT, dtype=nt)
    m = m / np.asarray([colors, 1.0, 1.0], dtype=nt)
    m = m / np.max(np.linalg.norm(m, axis=0))
    return torch.tensor(m, dtype=dtype)


def fft_synth(spectrum, decay_power=1.5, colors=1.5, contrast=0.9):
    """FftDrawer.synth, fftdrawer.py:78-84: to_valid_rgb(fft_image(...))(contrast=0.9).
    spectrum [1, 3, H, W//2+1, 2] (real, imag); returns [1, 3, H, W] in (0, 1), in the spectrum's dtype (float32 or
    float64) and on its device: the scale grid and the colour matrix follow it."""
    _, _, h, w2, _ = spectrum.shape
    w = (w2 - 1) * 2
    scale = fft_freq_scale(h, w, decay_power, spectrum.dtype).to(spectrum.device)
    scaled = scale[None, None, :, :, None] * spectrum
    image = torch.fft.irfftn(torch.view_as_complex(scaled.contiguous()), s=(h, w), norm="ortho")
    image = image * contrast / image.std()
    m = color_matrix(colors, spectrum.dtype).to(spectrum.device)
    image = torch.matmul(image.permute(0, 2, 3, 1), m.T).permute(0, 3, 1, 2)
    return torch.sigmoid(image)


# ------------------------------------------------------------------------------------------------ optimiser / loop



# ------------------------------------------------------------------------------------------------ auxiliary losses
# Losses/*.py (LossInterface.get_loss(cur_cutouts, out, args, globals, lossGlobals)); `out` is the synthesised image
# [1,3,H,W], `cutouts` the (noised) MakeCutouts batch [cutn,3,cs,cs], `embeds` the last perceptor's unit embeddings.


def symmetry_loss(out, symmetry_weight=1.0):
    """Losses/SymmetryLoss.py:14-17: MSE between the image and its horizontal mirror."""
    return F.mse_loss(out, torch.flip(out, [3])) * symmetry_weight


def saturation_loss(cutouts, saturation_weight=1.0):
    """Losses/SaturationLoss.py:15-30: Hasler-Suesstrunk colourfulness over all cutout pixels, negated."""
    px = cutouts.permute(0, 2, 3, 1).reshape(-1, 3)
    rg = px[:, 0] - px[:, 1]
    yb = 0.5 * (px[:, 0] + px[:, 1]) - px[:, 2]
    rg_std, rg_mean = torch.std_mean(rg)
    yb_std, yb_mean = torch.std_mean(yb)
    std_rggb = torch.sqrt(rg_std ** 2 + yb_std ** 2)
    mean_rggb = torch.sqrt(rg_mean ** 2 + yb_mean ** 2)
    return -(std_rggb + 0.3 * mean_rggb) * saturation_weight / 10.0


def palette_loss(cutouts, palette, palette_weight=1.0):
    """Losses/PaletteLoss.py:25-35: L2 distance of every cutout pixel to its nearest palette colour.
    Returns (loss, best_guesses) -- the argmin indices are the path's integer bookkeeping."""
    target = torch.as_tensor(palette, dtype=torch.float32)
    px = cutouts.permute(0, 2, 3, 1).reshape(-1, 3)
    best = torch.cdist(target, px, p=2).argmin(axis=0)
    diffs = px - target[best]
    loss = torch.mean(torch.norm(diffs, 2, dim=1)) * cutouts.shape[0]
    return loss * palette_weight / 10.0, best


def smoothness_loss(cutouts, smoothness_weight=1.0, smoothness_type="default", spacing=1, edge_order=1):
    """Losses/SmoothnessLoss.py:89-108 (smoothness_gaussian_kernel = 0).  NB the reference stacks the cutouts' rows:
    `_pixels` is [cutn*H, W, 3], so the finite difference along dim 0 runs ACROSS cutout boundaries."""
    px = cutouts.permute(0, 2, 3, 1).reshape(-1, cutouts.shape[2], 3)
    sq = 0
    for c in range(3):
        gy, gx = torch.gradient(px[:, :, c], spacing=spacing, edge_order=edge_order)
        sq = sq + gy ** 2 + gx ** 2
    sharp = torch.sqrt(sq)
    if smoothness_type == "clipped":
        sharp = torch.clamp(sharp, max=0.5)
    elif smoothness_type == "log":
        sharp = torch.log(torch.ones_like(sharp) + sharp)
    return torch.mean(sharp) * smoothness_weight


def edge_margins_px(edge_margins, H, W):
    """Losses/EdgeLoss.py:82-88: percent margins (left, right, up, down) -> pixels, util.map_number + int()."""
    left, right, upper, lower = edge_margins
    return (int(left / 100.0 * W), int(right / 100.0 * W), int(upper / 100.0 * H), int(lower / 100.0 * H))


def edge_loss(out, edge_color, margins_px, edge_color_weight=0.1, global_color_weight=0.05):
    """Losses/EdgeLoss.py:60-108, colour target, no input image / mask."""
    lmax, rmax = out.shape[2], out.shape[3]
    left, right, upper, lower = margins_px
    zers = torch.zeros_like(out)
    for c in range(3):
        zers[:, c] = edge_color[c]
    cur = torch.zeros(())
    if left != 0:
        cur = cur + F.mse_loss(out[:, :, :, :left], zers[:, :, :, :left])
    if right != 0:
        cur = cur + F.mse_loss(out[:, :, :, rmax - right:], zers[:, :, :, rmax - right:])
    if upper != 0:
        cur = cur + F.mse_loss(out[:, :, :upper, left:rmax - right], zers[:, :, :upper, left:rmax - right])
    if lower != 0:
        cur = cur + F.mse_loss(out[:, :, lmax - lower:, left:rmax - right], zers[:, :, lmax - lower:, left:rmax - right])
    if global_color_weight:
        cur = cur + F.mse_loss(out, zers) * global_color_weight
    return cur * edge_color_weight


def gaussian_window(ylen, xlen, stdy, stdx):
    """Losses/GaussianLoss.py:6-17 (gaussian_fn / gkern)."""
    def fn(M, std):
        n = torch.arange(0, M) - (M - 1.0) / 2.0
        return torch.exp(-n ** 2 / (2 * std * std))
    return torch.outer(fn(ylen, stdy), fn(xlen, stdx))


def gaussian_loss(out, gaussian_std=(40, 40), gaussian_color=(255, 255, 255), gaussian_weight=1.0):
    """Losses/GaussianLoss.py:31-44."""
    gaus = gaussian_window(out.shape[2], out.shape[3], *gaussian_std)
    color = torch.zeros_like(out)
    for c in range(3):
        color[:, c] = gaussian_color[c] / 255
    return torch.mean(torch.abs(out - color) * torch.abs(1 - gaus)) * gaussian_weight


def aesthetic_loss(embeds, weight, bias, aesthetic_target=10.0):
    """Losses/AestheticLoss.py:30-33: linear AVA head on the (re-)normalised embeddings, MSE to the target * 0.02."""
    rating = F.linear(F.normalize(embeds, dim=-1), weight, bias)
    target = torch.ones(embeds.shape[0], 1) * aesthetic_target
    return (rating - target).square().mean() * 0.02


# ------------------------------------------------------------------------------------------------ vdiff drawer (config 4)
# v-diffusion-pytorch/diffusion/models/cc12m_1.py (CC12M1Model) restated table-driven.  Modules are created in the same
# order, with the same torch constructors, as the reference's __init__ (skip projections before the main path:
# cc12m_1.py:21, 43; net arguments left to right: 135-236), so `torch.manual_seed(s); VDiffCC12M1()` reproduces the
# reference's own seeded initialisation bit for bit -- that is how tests/golden pins this restatement without a
# 2.4 GB weight fixture.  `ref_state_dict()` returns the weights under the reference checkpoint's keys.

VDIFF_C = 128


def vdiff_spec(c=VDIFF_C):
    """The `net` of cc12m_1.py:135-236 as nested tuples: ("b", c_in, c_mid, c_out, is_last), ("a", c, heads),
    ("s", [children]) with AvgPool2d first and bilinear Upsample last inside every SkipBlock."""
    cs = [c, c * 2, c * 2, c * 4, c * 4, c * 8, c * 8]

    def stage(lv):
        # the SkipBlock entered below resolution level lv - 1 (levels 1..6)
        cin, cc = cs[lv - 1], cs[lv]
        attn = lv >= 4
        items = ["down"]
        if lv < 6:
            chain = [(cin, cc, cc), (cc, cc, cc), (cc, cc, cc), (cc, cc, cc)]
            for (a, m, o) in chain:
                items.append(("b", a, m, o, False))
                if attn:
                    items.append(("a", o, o // 64))
            items.append(stage(lv + 1))
            up = [(cc * 2, cc, cc), (cc, cc, cc), (cc, cc, cc), (cc, cc, cin)]
            for (a, m, o) in up:
                items.append(("b", a, m, o, False))
                if attn:
                    items.append(("a", o, o // 64))
        else:  # 4x4 level: eight blocks, the last one narrows back (cc12m_1.py:183-199)
            chain = [(cin, cc, cc)] + [(cc, cc, cc)] * 6 + [(cc, cc, cin)]
            for (a, m, o) in chain:
                items.append(("b", a, m, o, False))
                items.append(("a", o, o // 64))
        items.append("up")
        return ("s", items)

    top = [("b", 3 + 16, cs[0], cs[0], False)] + [("b", cs[0], cs[0], cs[0], False)] * 3
    top.append(stage(1))
    top += [("b", cs[0] * 2, cs[0], cs[0], False), ("b", cs[0], cs[0], cs[0], False), ("b", cs[0], cs[0], cs[0], False),
            ("b", cs[0], cs[0], 3, True)]
    return top


class VDiffCC12M1(nn.Module):
    def __init__(self, c=VDIFF_C):
        super().__init__()
        self.mods = nn.ModuleList()
        self.keys = []  # (reference key prefix, module) in creation order

        def reg(key, m):
            self.mods.append(m)
            self.keys.append((key, m))
            return m

        # cc12m_1.py:117-123: FourierFeatures(1, 128) (weight = randn [64, 1]), mapping = 2 ResLinearBlocks, *= sqrt(1/2)
        self.map_ff = nn.Parameter(torch.randn(64, 1), requires_grad=False)
        self.map_skip0 = reg("mapping.0.skip", nn.Linear(512 + 128, 1024, bias=False))  # cc12m_1.py:21 (before main)
        self.map_00 = reg("mapping.0.main.0", nn.Linear(512 + 128, 1024))
        self.map_02 = reg("mapping.0.main.2", nn.Linear(1024, 1024))
        self.map_10 = reg("mapping.1.main.0", nn.Linear(1024, 1024))
        self.map_12 = reg("mapping.1.main.2", nn.Linear(1024, 1024))
        with torch.no_grad():
            for m in (self.map_skip0, self.map_00, self.map_02, self.map_10, self.map_12):
                for prm in m.parameters():
                    prm *= 0.5 ** 0.5
        self.t_ff = nn.Parameter(torch.randn(8, 1), requires_grad=False)  # timestep_embed = FourierFeatures(1, 16)
        self.spec = vdiff_spec(c)
        first_net = len(self.mods)

        def build(items, prefix):
            out = []
            for i, it in enumerate(items):
                key = f"{prefix}.{i}"
                if it in ("down", "up"):
                    out.append(it)
                elif it[0] == "b":
                    _, cin, cmid, cout, last = it
                    skip = reg(key + ".skip", nn.Conv2d(cin, cout, 1, bias=False)) if cin != cout else None  # :43
                    blk = dict(kind="b", key=key, last=last, skip=skip, conv1=reg(key + ".main.0", nn.Conv2d(cin, cmid, 3, padding=1)),
                               mod1=reg(key + ".main.2.layer", nn.Linear(1024, cmid * 2, bias=False)),
                               conv2=reg(key + ".main.4", nn.Conv2d(cmid, cout, 3, padding=1)),
                               mod2=None if last else reg(key + ".main.6.layer", nn.Linear(1024, cout * 2, bias=False)))
                    out.append(blk)
                elif it[0] == "a":
                    _, ch, heads = it
                    out.append(dict(kind="a", key=key, heads=heads, norm=reg(key + ".norm", nn.GroupNorm(1, ch)),
                                    qkv=reg(key + ".qkv_proj", nn.Conv2d(ch, ch * 3, 1)),
                                    out=reg(key + ".out_proj", nn.Conv2d(ch, ch, 1))))
                else:
                    out.append(dict(kind="s", key=key, main=build(it[1], key + ".main")))
            return out

        self.net = build(self.spec, "net")
        self.taps = None  # tests: set to a list to collect (key, output tensor) of every block / attention / skip
        # tests: quant = True rounds the stored activations to fp16 (straight-through) at the points where the engine
        # stores fp16 tensors, so that ReLU branches are decided on (nearly) the same values as in the engine
        self.quant = False
        with torch.no_grad():  # cc12m_1.py:239-241
            for m in list(self.mods)[first_net:]:
                for prm in m.parameters():
                    prm *= 0.5 ** 0.5

    def _q(self, t):
        return t + (t.half().float() - t).detach() if self.quant else t

    def round_weights_to_fp16_(self):
        """Round every conv / linear weight to fp16 in place (biases and norm affines stay fp32, like in the engine)."""
        with torch.no_grad():
            for _, m in self.keys:
                if isinstance(m, (nn.Conv2d, nn.Linear)):
                    m.weight.copy_(m.weight.half().float())
        return self

    def ref_state_dict(self):
        sd = OrderedDict()
        sd["mapping_timestep_embed.weight"] = self.map_ff.detach()
        sd["timestep_embed.weight"] = self.t_ff.detach()
        for key, m in self.keys:
            for n, prm in m.named_parameters():
                sd[f"{key}.{n}"] = prm.detach()
        return sd

    @staticmethod
    def fourier(t, w):  # cc12m_1.py:73-75
        f = 2 * math.pi * t[:, None] @ w.T
        return torch.cat([f.cos(), f.sin()], dim=-1)

    def cond(self, t, clip_embed):  # cc12m_1.py:244-246
        ce = F.normalize(clip_embed, dim=-1) * clip_embed.shape[-1] ** 0.5
        h = torch.cat([ce, self.fourier(t, self.map_ff)], dim=1)
        h = F.relu(self.map_02(F.relu(self.map_00(h)))) + self.map_skip0(h)
        return self.map_12(F.relu(self.map_10(h))) + h  # is_last: no final ReLU, identity skip

    def _run(self, items, x, cond):
        for it in items:
            if it == "down":
                x = self._q(F.avg_pool2d(x, 2))
            elif it == "up":
                x = self._q(F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False))
            elif it["kind"] == "b":
                def mod(lin, h):  # Modulation2d, cc12m_1.py:36-38
                    sc, sh = lin(cond).chunk(2, dim=-1)
                    return torch.addcmul(sh[..., None, None], h, sc[..., None, None] + 1)
                q = self._q
                h = q(it["conv1"](x))
                h = q(F.relu(mod(it["mod1"], F.group_norm(h, 1))))
                h = it["conv2"](h)
                sk = q(it["skip"](x)) if it["skip"] is not None else x
                if not it["last"]:
                    h = F.relu(mod(it["mod2"], F.group_norm(q(h), 1)))
                    x = q(h + sk)
                else:
                    x = h + sk
            elif it["kind"] == "a":  # SelfAttention2d, cc12m_1.py:88-97
                n, c, hh, ww = x.shape
                qkv = self._q(it["qkv"](self._q(it["norm"](x)))).view(n, it["heads"] * 3, c // it["heads"], hh * ww).transpose(2, 3)
                q, k, v = qkv.chunk(3, dim=1)
                scale = k.shape[3] ** -0.25
                att = ((q * scale) @ (k.transpose(2, 3) * scale)).softmax(3)
                y = self._q((att @ v).transpose(2, 3).contiguous().view(n, c, hh, ww))
                x = self._q(x + it["out"](y))
            else:  # SkipBlock, cc12m_1.py:57-58
                x = torch.cat([self._run(it["main"], x, cond), x], dim=1)
            if self.taps is not None and isinstance(it, dict) and x.requires_grad:
                x.retain_grad()
                self.taps.append((it["key"], x))
        return x

    def forward(self, x, t, clip_embed):
        cond = self.cond(t, clip_embed)
        te = self.fourier(t, self.t_ff)[..., None, None].repeat(1, 1, x.shape[2], x.shape[3])
        return self._run(self.net, self._q(torch.cat([x, te], dim=1)), cond)


def vdiff_t_to_alpha_sigma(t):
    """diffusion/utils.py:52-55."""
    return torch.cos(t * math.pi / 2), torch.sin(t * math.pi / 2)


def vdiff_schedule(iterations, vdiff_skip=0.0):
    """VdiffDrawer.init_from_tensor (vdiff.py:113-126) with the default spliced DDPM/cosine schedule
    (diffusion/utils.py:63-78): returns (steps, alphas, sigmas), each [iterations + 1]."""
    top = 1.0 - vdiff_skip / 100.0
    t = torch.linspace(top, 0, iterations + 2)[:-1]
    ddpm_crossover, cosine_crossover = 0.48536712, 0.80074257
    big_t = t * (1 + cosine_crossover - ddpm_crossover)
    ddpm_t = big_t + ddpm_crossover - cosine_crossover
    log_snr = -torch.special.expm1(1e-4 + 10 * ddpm_t ** 2).log()
    alpha, sigma = log_snr.sigmoid().sqrt(), log_snr.neg().sigmoid().sqrt()
    ddpm_part = torch.atan2(sigma, alpha) / math.pi * 2
    steps = torch.where(big_t < cosine_crossover, big_t, ddpm_part)
    a, s = vdiff_t_to_alpha_sigma(steps)
    return steps, a, s


def vdiff_synth(model, x, t, clip_embed, alpha, sigma):
    """VdiffDrawer.synth (vdiff.py:159-172) through sampling.sample_step_pred (sampling.py:7-15): returns
    (pixels in [0,1] with ClampWithGrad, pred, v)."""
    v = model(x, t, clip_embed).float()
    pred = x * alpha - v * sigma
    return clamp_with_grad(pred.add(1).div(2), 0, 1), pred, v


def vdiff_renoise(x, pred, v, alphas, sigmas, i, noise, eta=1.0):
    """sampling.sample_step_noise (sampling.py:18-39) with the fresh noise passed in."""
    eps = x * sigmas[i] + v * alphas[i]
    if i < len(alphas) - 1:
        ddim_sigma = eta * (sigmas[i + 1] ** 2 / sigmas[i] ** 2).sqrt() * (1 - alphas[i] ** 2 / alphas[i + 1] ** 2).sqrt()
        adjusted_sigma = (sigmas[i + 1] ** 2 - ddim_sigma ** 2).sqrt()
        x = pred * alphas[i + 1] + eps * adjusted_sigma
        if eta:
            x = x + noise * ddim_sigma
    return x


class AdamState:
    """optim.Adam([z], lr) as rebuilt by rebuild_optimisers (pixray.py:520-555): betas 0.9/0.999, eps 1e-8."""

    def __init__(self, z, beta1=0.9, beta2=0.999, eps=1e-8):
        self.m = torch.zeros_like(z)
        self.v = torch.zeros_like(z)
        self.t = 0
        self.b1, self.b2, self.eps = beta1, beta2, eps

    def step(self, z, grad, lr):
        self.t += 1
        self.m.mul_(self.b1).add_(grad, alpha=1 - self.b1)
        self.v.mul_(self.b2).addcmul_(grad, grad, value=1 - self.b2)
        bc1, bc2 = 1 - self.b1 ** self.t, 1 - self.b2 ** self.t
        denom = (self.v.sqrt() / math.sqrt(bc2)).add_(self.eps)
        return z - (lr / bc1) * self.m / denom


def anchor_loss(kind, weight, z, out, ref):
    """The init_weight family / image_labels of ascend_txt (pixray.py:1344-1375): z = drawer.get_z(), ref = z_orig (or an
    encoded label image); "pix": out vs init_image_tensor."""
    if kind == "spherical":   # pixray.py:1346-1349, 1352-1356
        return spherical_dist_loss(z.reshape(1, -1), ref.reshape(1, -1))[0] * weight
    if kind == "mse":         # pixray.py:1359-1361
        return F.mse_loss(z, ref) * weight / 2
    if kind == "cos":         # pixray.py:1370-1375 (the reference passes y = ones_like(f[0]); every element says "similar")
        f, f2 = z.reshape(1, -1), ref.reshape(1, -1)
        return F.cosine_embedding_loss(f, f2, torch.ones(1)) * weight
    if kind == "pix":         # pixray.py:1363-1368
        return F.l1_loss(out, ref) * weight / 2
    raise ValueError(kind)


def iterate(synth_fn, z, clip_models, prompts, transforms, cut_size, zoom_padding, fill, noise_facs, noise, aux=(),
            jitter=None, image_prompts=(), aspect=1.0, spot_mask=None, spot_prompts=None, spot_prompts_off=None,
            filters=(), anchors=()):
    """One ascend_txt + backward (pixray.py:1243-1406, 1481-1482) on explicit cutout parameters.

    synth_fn: z -> image [1,3,H,W]; clip_models: list of ClipVisual; prompts: per model list of
    (embed [n,D], weight, stop); aux: custom losses (pixray.py:1384-1393) as (weight, fn(out, batch, embeds) ->
    scalar), appended to the loss list in order; image_prompts: (target image [1,3,H,W], weight), scored per model
    after its text prompts (the explicit noise is replayed for their cutouts); anchors: (kind, weight, ref) with kind in
    "spherical" (init_weight / image_labels), "mse" (init_weight_dist), "cos" (init_weight_cos), "pix" (init_weight_pix),
    between the prompts and the custom losses (pixray.py:1344-1375).  Returns dict(image, batch, embeds[], losses[], z_grad)."""
    z = z.detach().clone().requires_grad_(True)
    out = synth_fn(z)
    filter_losses = []
    for (weight, fn) in filters:  # do_synth_and_filter (pixray.py:1212-1222): fn(img) -> (img, loss); losses lead the list
        out, fl = fn(out)
        filter_losses.append(weight * fl)
    out.retain_grad()
    batch = make_cutouts(out, transforms, cut_size, zoom_padding, fill, noise_facs, noise, jitter=jitter, aspect=aspect)
    batch.retain_grad()
    losses, embeds = list(filter_losses), []
    # spot prompts (pixray.py:1262-1293): per kind ONE more make_cutouts on the cached transforms (no ColorJitter; the
    # explicit noise is replayed), encoded by every perceptor that has such prompts, scored before the regular prompts
    spot_batches = {}
    for which, table in ((1, spot_prompts), (0, spot_prompts_off)):
        if table is not None and any(len(t) for t in table):
            spot_batches[which] = make_cutouts(out, transforms, cut_size, zoom_padding, fill, noise_facs, noise, aspect=aspect,
                                               spot=which, spot_mask=spot_mask)
    for mi, (model, pms) in enumerate(zip(clip_models, prompts)):
        for which, table in ((1, spot_prompts), (0, spot_prompts_off)):
            if which in spot_batches and len(table[mi]):
                iii_s = encode_image(model, spot_batches[which]).float()
                for (embed, weight, stop) in table[mi]:
                    losses.append(prompt_loss(iii_s, embed, weight, stop))
        iii = encode_image(model, batch).float()
        embeds.append(iii)
        for (embed, weight, stop) in pms:
            losses.append(prompt_loss(iii, embed, weight, stop))
        # image prompts (pixray.py:1308-1336): make_cutouts(timg) replays the cached transforms -- the warp-only path,
        # no ColorJitter (pixray.py:480-486) -- and the [cutn, D] embedding becomes a throwaway Prompt(embed, weight)
        for (timg, weight) in image_prompts:
            with torch.no_grad():
                tb = make_cutouts(timg, transforms, cut_size, zoom_padding, fill, noise_facs, noise, aspect=aspect)
                te = encode_image(model, tb).float()
            losses.append(prompt_loss(iii, te, weight, float("-inf")))
    for (kind, weight, ref) in anchors:
        losses.append(anchor_loss(kind, weight, z, out, ref))
    for (lossweight, fn) in aux:
        losses.append(lossweight * fn(out, batch, embeds[-1]))
    total = sum(losses)
    total.backward()
    return dict(image=out.detach(), batch=batch.detach(), embeds=[e.detach() for e in embeds],
                losses=[l.detach() for l in losses], z_grad=z.grad.detach(), image_grad=out.grad.detach(),
                batch_grad=batch.grad.detach())
