"""Seeded synthetic weights / prompts / latents with the reference's state_dict names and shapes.

No pretrained checkpoints are reachable (the reference downloads them at run time, vqgan.py:19-46, slip.py:175), so
bench.py, smoke() and the tests run on random weights of the named architectures (imagenet_f16_16384 VQGAN,
openai-CLIP ViT-B/16 / ViT-B/32).  Plain torch on the CPU; nothing here touches the oracle or the GPU.
"""
import math

import torch


def _randn(g, *shape, std=1.0):
    return torch.randn(*shape, generator=g) * std


def clip_state_dict(arch, seed=0):
    """openai-CLIP 'visual.*' tensors (init pattern of SLIP/models.py:106-120)."""
    g = torch.Generator().manual_seed(seed)
    W, L, P, D = arch["width"], arch["layers"], arch["patch"], arch["out_dim"]
    T = (arch["image_res"] // P) ** 2 + 1
    sd = {}
    sd["visual.conv1.weight"] = _randn(g, W, 3, P, P, std=(3 * P * P) ** -0.5)
    sd["visual.class_embedding"] = _randn(g, W, std=W ** -0.5)
    sd["visual.positional_embedding"] = _randn(g, T, W, std=0.01)
    sd["visual.proj"] = _randn(g, W, D, std=W ** -0.5)
    proj_std, attn_std, fc_std = (W ** -0.5) * ((2 * L) ** -0.5), W ** -0.5, (2 * W) ** -0.5
    for nm in ("ln_pre", "ln_post"):
        sd[f"visual.{nm}.weight"] = 1 + 0.1 * _randn(g, W)
        sd[f"visual.{nm}.bias"] = 0.05 * _randn(g, W)
    for i in range(L):
        p = f"visual.transformer.resblocks.{i}."
        sd[p + "attn.in_proj_weight"] = _randn(g, 3 * W, W, std=attn_std)
        sd[p + "attn.in_proj_bias"] = _randn(g, 3 * W, std=0.02)
        sd[p + "attn.out_proj.weight"] = _randn(g, W, W, std=proj_std)
        sd[p + "attn.out_proj.bias"] = _randn(g, W, std=0.02)
        sd[p + "mlp.c_fc.weight"] = _randn(g, 4 * W, W, std=fc_std)
        sd[p + "mlp.c_fc.bias"] = _randn(g, 4 * W, std=0.02)
        sd[p + "mlp.c_proj.weight"] = _randn(g, W, 4 * W, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = _randn(g, W, std=0.02)
        for nm in ("ln_1", "ln_2"):
            sd[p + nm + ".weight"] = 1 + 0.1 * _randn(g, W)
            sd[p + nm + ".bias"] = 0.05 * _randn(g, W)
    return sd


def clip_text_state_dict(width, layers, out_dim, seed=0, vocab=49408, context=77):
    """The text-tower tensors of a CLIP / SLIP checkpoint (token_embedding, positional_embedding, transformer.resblocks.*,
    ln_final, text_projection; init pattern of SLIP/models.py:106-120), to merge with a visual state_dict."""
    g = torch.Generator().manual_seed(seed)
    W, L = width, layers
    sd = {"token_embedding.weight": _randn(g, vocab, W, std=0.02), "positional_embedding": _randn(g, context, W, std=0.01)}
    proj_std, attn_std, fc_std = (W ** -0.5) * ((2 * L) ** -0.5), W ** -0.5, (2 * W) ** -0.5
    for i in range(L):
        p = f"transformer.resblocks.{i}."
        sd[p + "attn.in_proj_weight"] = _randn(g, 3 * W, W, std=attn_std)
        sd[p + "attn.in_proj_bias"] = _randn(g, 3 * W, std=0.02)
        sd[p + "attn.out_proj.weight"] = _randn(g, W, W, std=proj_std)
        sd[p + "attn.out_proj.bias"] = _randn(g, W, std=0.02)
        sd[p + "mlp.c_fc.weight"] = _randn(g, 4 * W, W, std=fc_std)
        sd[p + "mlp.c_fc.bias"] = _randn(g, 4 * W, std=0.02)
        sd[p + "mlp.c_proj.weight"] = _randn(g, W, 4 * W, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = _randn(g, W, std=0.02)
        for nm in ("ln_1", "ln_2"):
            sd[p + nm + ".weight"] = 1 + 0.1 * _randn(g, W)
            sd[p + nm + ".bias"] = 0.05 * _randn(g, W)
    sd["ln_final.weight"] = 1 + 0.1 * _randn(g, W)
    sd["ln_final.bias"] = 0.05 * _randn(g, W)
    sd["text_projection"] = _randn(g, W, out_dim, std=W ** -0.5)
    return sd


def slip_state_dict(arch, seed=0):
    """The image-tower tensors of a SLIP_Base checkpoint (after `module.` is stripped, slip.py:126-128): timm's
    VisionTransformer under 'visual.*' and 'image_projection' (SLIP/models.py:130-134), at the scales of clip_state_dict."""
    g = torch.Generator().manual_seed(seed)
    W, L, P, D = arch["width"], arch["layers"], arch["patch"], arch["out_dim"]
    T = (arch["image_res"] // P) ** 2 + 1
    sd = {}
    sd["visual.cls_token"] = _randn(g, 1, 1, W, std=W ** -0.5)
    sd["visual.pos_embed"] = _randn(g, 1, T, W, std=0.01)
    sd["visual.patch_embed.proj.weight"] = _randn(g, W, 3, P, P, std=(3 * P * P) ** -0.5)
    sd["visual.patch_embed.proj.bias"] = _randn(g, W, std=0.02)
    proj_std, attn_std, fc_std = (W ** -0.5) * ((2 * L) ** -0.5), W ** -0.5, (2 * W) ** -0.5
    for i in range(L):
        p = f"visual.blocks.{i}."
        for nm in ("norm1", "norm2"):
            sd[p + nm + ".weight"] = 1 + 0.1 * _randn(g, W)
            sd[p + nm + ".bias"] = 0.05 * _randn(g, W)
        sd[p + "attn.qkv.weight"] = _randn(g, 3 * W, W, std=attn_std)
        sd[p + "attn.qkv.bias"] = _randn(g, 3 * W, std=0.02)
        sd[p + "attn.proj.weight"] = _randn(g, W, W, std=proj_std)
        sd[p + "attn.proj.bias"] = _randn(g, W, std=0.02)
        sd[p + "mlp.fc1.weight"] = _randn(g, 4 * W, W, std=fc_std)
        sd[p + "mlp.fc1.bias"] = _randn(g, 4 * W, std=0.02)
        sd[p + "mlp.fc2.weight"] = _randn(g, W, 4 * W, std=proj_std)
        sd[p + "mlp.fc2.bias"] = _randn(g, W, std=0.02)
    sd["visual.norm.weight"] = 1 + 0.1 * _randn(g, W)
    sd["visual.norm.bias"] = 0.05 * _randn(g, W)
    sd["image_projection"] = _randn(g, W, D, std=W ** -0.5)
    return sd


def vqgan_state_dict(v, seed=0, with_encoder=False):
    """taming VQModel tensors pixray uses: quantize.embedding, post_quant_conv, decoder.* (vqgan.py:122-142) and, with
    with_encoder, encoder.* + quant_conv (model.encode: VqganDrawer.init_from_tensor, vqgan.py:174-185)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(name, cin, cout, k):
        sd[name + ".weight"] = _randn(g, cout, cin, k, k, std=(1.0 / (cin * k * k)) ** 0.5)
        sd[name + ".bias"] = 0.05 * _randn(g, cout)

    def norm(name, c):
        sd[name + ".weight"] = 1 + 0.1 * _randn(g, c)
        sd[name + ".bias"] = 0.05 * _randn(g, c)

    def res(name, cin, cout):
        norm(name + ".norm1", cin)
        conv(name + ".conv1", cin, cout, 3)
        norm(name + ".norm2", cout)
        conv(name + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(name + ".nin_shortcut", cin, cout, 1)

    def attn(name, c):
        norm(name + ".norm", c)
        for q in ("q", "k", "v", "proj_out"):
            conv(f"{name}.{q}", c, c, 1)

    zc, ch, mult, nrb = v["z_channels"], v["ch"], v["ch_mult"], v["num_res_blocks"]
    L = len(mult)
    sd["quantize.embedding.weight"] = _randn(g, v["n_embed"], zc, std=0.5)
    conv("post_quant_conv", zc, zc, 1)
    block_in = ch * mult[-1]
    curr = v["resolution"] // 2 ** (L - 1)
    conv("decoder.conv_in", zc, block_in, 3)
    res("decoder.mid.block_1", block_in, block_in)
    attn("decoder.mid.attn_1", block_in)
    res("decoder.mid.block_2", block_in, block_in)
    for lv in reversed(range(L)):
        block_out = ch * mult[lv]
        for ib in range(nrb + 1):
            res(f"decoder.up.{lv}.block.{ib}", block_in, block_out)
            block_in = block_out
            if curr == v["attn_resolution"]:
                attn(f"decoder.up.{lv}.attn.{ib}", block_in)
        if lv != 0:
            conv(f"decoder.up.{lv}.upsample.conv", block_in, block_in, 3)
            curr *= 2
    norm("decoder.norm_out", block_in)
    conv("decoder.conv_out", block_in, 3, 3)
    if with_encoder:  # a separate generator: the decoder tensors above do not depend on this flag
        g = torch.Generator().manual_seed(seed + 7919)
        conv("encoder.conv_in", 3, ch, 3)
        curr, block_in = v["resolution"], ch
        in_mult = (1,) + tuple(mult)
        for lv in range(L):
            block_in, block_out = ch * in_mult[lv], ch * mult[lv]
            for ib in range(nrb):
                res(f"encoder.down.{lv}.block.{ib}", block_in, block_out)
                block_in = block_out
                if curr == v["attn_resolution"]:
                    attn(f"encoder.down.{lv}.attn.{ib}", block_in)
            if lv != L - 1:
                conv(f"encoder.down.{lv}.downsample.conv", block_in, block_in, 3)
                curr //= 2
        res("encoder.mid.block_1", block_in, block_in)
        attn("encoder.mid.attn_1", block_in)
        res("encoder.mid.block_2", block_in, block_in)
        norm("encoder.norm_out", block_in)
        conv("encoder.conv_out", block_in, zc, 3)
        conv("quant_conv", zc, zc, 1)
    return sd


def prompts(out_dim, weights=(1.0, 0.1), seed=0):
    """Seeded unit-norm Gaussian prompt embeddings: the reference's own noise-prompt recipe (pixray.py:955-958)."""
    out = []
    for k, w in enumerate(weights):
        e = torch.empty(1, out_dim).normal_(generator=torch.Generator().manual_seed(seed + k))
        out.append((e / e.norm(dim=-1, keepdim=True), float(w), float("-inf")))
    return out


def z0_vqgan(codebook, hw, seed=0):
    """z0 = seeded random codebook rows + small noise (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(codebook.shape[0], (hw[0] * hw[1],), generator=g)
    z = codebook[idx].T.reshape(1, codebook.shape[1], hw[0], hw[1]).contiguous()  # dense NCHW (not a permuted view)
    return (z + 0.05 * torch.randn(z.shape, generator=g)).contiguous()


def vit_fwd_flops(arch):
    """Algorithmic forward FLOPs of one image through the ViT (SURVEY.md 8d formula)."""
    W, L, P = arch["width"], arch["layers"], arch["patch"]
    T = (arch["image_res"] // P) ** 2 + 1
    per_layer = 2 * T * (4 * W * W + 2 * W * 4 * W) + 4 * T * T * W
    return L * per_layer + 2 * (T - 1) * W * 3 * P * P + 2 * W * arch["out_dim"]


def vqgan_decoder_fwd_flops(v, image_hw):
    """Algorithmic forward FLOPs of post_quant_conv + Decoder at image_hw (conv: 2*H*W*Cin*Cout*k^2)."""
    zc, ch, mult, nrb = v["z_channels"], v["ch"], v["ch_mult"], v["num_res_blocks"]
    L = len(mult)
    f = 2 ** (L - 1)
    h, w = image_hw[0] // f, image_hw[1] // f
    fl = 0.0

    def conv(cin, cout, k, px):
        return 2.0 * px * cin * cout * k * k

    def res(cin, cout, px):
        r = conv(cin, cout, 3, px) + conv(cout, cout, 3, px)
        return r + (conv(cin, cout, 1, px) if cin != cout else 0)

    def attn(c, px):
        return 4 * conv(c, c, 1, px) + 4.0 * px * px * c

    px = h * w
    fl += conv(zc, zc, 1, px)
    block_in = ch * mult[-1]
    curr = v["resolution"] // f
    fl += conv(zc, block_in, 3, px) + 2 * res(block_in, block_in, px) + attn(block_in, px)
    for lv in reversed(range(L)):
        block_out = ch * mult[lv]
        for _ in range(nrb + 1):
            fl += res(block_in, block_out, px)
            block_in = block_out
            if curr == v["attn_resolution"]:
                fl += attn(block_in, px)
        if lv != 0:
            px *= 4
            fl += conv(block_in, block_in, 3, px)
            curr *= 2
    fl += conv(block_in, 3, 3, px)
    return fl


def vdiff_state_dict(seed=0, c=128):
    """cc12m_1's tensors under the checkpoint's own keys (diffusion/models/cc12m_1.py:115-241), seeded random with the
    module defaults' scale (uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)), then * sqrt(1/2) as cc12m_1.py:239-241 does)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def uni(*shape, fan_in):
        b = (1.0 / fan_in) ** 0.5 * 0.5 ** 0.5
        return (torch.rand(*shape, generator=g) * 2 - 1) * b

    def linear(key, cin, cout, bias=True):
        sd[key + ".weight"] = uni(cout, cin, fan_in=cin)
        if bias:
            sd[key + ".bias"] = uni(cout, fan_in=cin)

    def conv(key, cin, cout, k, bias=True):
        sd[key + ".weight"] = uni(cout, cin, k, k, fan_in=cin * k * k)
        if bias:
            sd[key + ".bias"] = uni(cout, fan_in=cin * k * k)

    sd["mapping_timestep_embed.weight"] = torch.randn(64, 1, generator=g)
    sd["timestep_embed.weight"] = torch.randn(8, 1, generator=g)
    linear("mapping.0.skip", 640, 1024, bias=False)
    linear("mapping.0.main.0", 640, 1024)
    linear("mapping.0.main.2", 1024, 1024)
    linear("mapping.1.main.0", 1024, 1024)
    linear("mapping.1.main.2", 1024, 1024)
    cs = [c, c * 2, c * 2, c * 4, c * 4, c * 8, c * 8]

    def block(key, cin, cmid, cout, last=False):
        if cin != cout:
            conv(key + ".skip", cin, cout, 1, bias=False)
        conv(key + ".main.0", cin, cmid, 3)
        linear(key + ".main.2.layer", 1024, cmid * 2, bias=False)
        conv(key + ".main.4", cmid, cout, 3)
        if not last:
            linear(key + ".main.6.layer", 1024, cout * 2, bias=False)

    def attn(key, ch):
        sd[key + ".norm.weight"] = torch.ones(ch)
        sd[key + ".norm.bias"] = torch.zeros(ch)
        conv(key + ".qkv_proj", ch, ch * 3, 1)
        conv(key + ".out_proj", ch, ch, 1)

    def stage(prefix, lv):
        # SkipBlock: main = [AvgPool2d, blocks (+ attention from level 4 on), nested SkipBlock, blocks, Upsample]
        cin, cc = cs[lv - 1], cs[lv]
        i = 1  # index 0 is the AvgPool2d
        if lv < 6:
            for (a, m, o) in [(cin, cc, cc), (cc, cc, cc), (cc, cc, cc), (cc, cc, cc)]:
                block(f"{prefix}.{i}", a, m, o)
                i += 1
                if lv >= 4:
                    attn(f"{prefix}.{i}", o)
                    i += 1
            stage(f"{prefix}.{i}.main", lv + 1)
            i += 1
            for (a, m, o) in [(cc * 2, cc, cc), (cc, cc, cc), (cc, cc, cc), (cc, cc, cin)]:
                block(f"{prefix}.{i}", a, m, o)
                i += 1
                if lv >= 4:
                    attn(f"{prefix}.{i}", o)
                    i += 1
        else:
            for (a, m, o) in [(cin, cc, cc)] + [(cc, cc, cc)] * 6 + [(cc, cc, cin)]:
                block(f"{prefix}.{i}", a, m, o)
                i += 1
                attn(f"{prefix}.{i}", o)
                i += 1

    block("net.0", 3 + 16, cs[0], cs[0])
    for k in (1, 2, 3):
        block(f"net.{k}", cs[0], cs[0], cs[0])
    stage("net.4.main", 1)
    block("net.5", cs[0] * 2, cs[0], cs[0])
    block("net.6", cs[0], cs[0], cs[0])
    block("net.7", cs[0], cs[0], cs[0])
    block("net.8", cs[0], cs[0], 3, last=True)
    return sd


def rrdbnet_state_dict(seed=0, num_feat=64, num_block=23, num_grow_ch=32, last_bias=0.5):
    """Real-ESRGAN's RRDBNet tensors under the checkpoint's own keys (basicsr rrdbnet_arch), seeded random with basicsr's
    initialisation: the dense-block convolutions kaiming-normal (fan_in, gain sqrt(2)) times 0.1 with zero bias
    (default_init_weights(..., 0.1)), every other convolution PyTorch's default (uniform(+-1/sqrt(fan_in)) for weight and
    bias).  conv_last's bias is centred on `last_bias`, so that most pixels of the image land inside (0, 1) rather than
    on ClampWithGrad's edges."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def default(key, cin, cout):
        b = (1.0 / (cin * 9)) ** 0.5
        sd[key + ".weight"] = (torch.rand(cout, cin, 3, 3, generator=g) * 2 - 1) * b
        sd[key + ".bias"] = (torch.rand(cout, generator=g) * 2 - 1) * b

    def dense(key, cin, cout):
        sd[key + ".weight"] = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5 * 0.1
        sd[key + ".bias"] = torch.zeros(cout)

    nf, gc = num_feat, num_grow_ch
    default("conv_first", 3, nf)
    for i in range(num_block):
        for j in (1, 2, 3):
            for k in range(1, 6):
                dense(f"body.{i}.rdb{j}.conv{k}", nf + gc * (k - 1), gc if k < 5 else nf)
    for key in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
        default(key, nf, nf)
    default("conv_last", nf, 3)
    sd["conv_last.bias"] = sd["conv_last.bias"] + last_bias
    return sd


def superres_fwd_flops(h, w, num_feat=64, num_block=23, num_grow_ch=32):
    """Multiply-add FLOPs (2 per MAC) of one RRDBNet forward on an h x w latent (image 4h x 4w); the dgrad costs the same."""
    nf, gc, px = num_feat, num_grow_ch, h * w
    per_px = lambda cin, cout: 2.0 * 9 * cin * cout  # noqa: E731
    dense = sum(per_px(nf + gc * k, gc) for k in range(4)) + per_px(nf + 4 * gc, nf)
    low = per_px(3, nf) + 3 * num_block * dense + per_px(nf, nf)
    return px * low + 4 * px * per_px(nf, nf) + 16 * px * (2 * per_px(nf, nf) + per_px(nf, 3))
