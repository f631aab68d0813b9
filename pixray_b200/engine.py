"""Python face of the C-ABI engine (include/pixray_b200.h).

torch is used only for device memory: tensors are handed to the library as raw device pointers.  Every method
maps 1:1 onto a C entry point, which in turn replaces one method of the reference's loop (see the header).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

DRAWER_VQGAN, DRAWER_PIXEL, DRAWER_FFT, DRAWER_VDIFF, DRAWER_POLYGON, DRAWER_SUPERRES, DRAWER_STROKES = 0, 1, 2, 3, 4, 5, 6
LOSS_SYMMETRY, LOSS_SATURATION, LOSS_PALETTE, LOSS_SMOOTHNESS, LOSS_EDGE, LOSS_GAUSSIAN, LOSS_AESTHETIC = range(7)
ANCHOR_SPHERICAL, ANCHOR_MSE, ANCHOR_COS, ANCHOR_PIX = 0, 1, 2, 3
FILTER_TILER, FILTER_WALLPAPER, FILTER_LOOKUP = range(3)
PAD_REFLECTION, PAD_BORDER = 0, 1
MOD_VQGAN, MOD_CLIP0, MOD_CLIP1, MOD_CLIP2, MOD_CLIP3 = 0, 1, 2, 3, 4
# optimiser update rules (pxr_set_optimizer), by the reference's args.optimiser names (pixray.py:536-551)
OPT_ADAM, OPT_ADAMW, OPT_ADAGRAD, OPT_ADAMAX, OPT_DIFFGRAD = range(5)
OPTIMISERS = {"Adam": OPT_ADAM, "AdamW": OPT_ADAMW, "Adagrad": OPT_ADAGRAD, "Adamax": OPT_ADAMAX, "DiffGrad": OPT_DIFFGRAD}

# RRDBNet of RealESRGAN_x4plus (super_resolution.py:53): RRDBNet(3, 3, num_feat=64, num_block=23, num_grow_ch=32, scale=4)
RRDBNET_X4PLUS = dict(num_feat=64, num_block=23, num_grow_ch=32)
VQGAN_F16_16384 = dict(z_channels=256, n_embed=16384, ch=128, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2,
                       attn_resolution=16, resolution=256)
# the shapes the tensor-core nearest-code search covers (kernels_vq_tc.cu, vq_tc_supported); vqgan_config refuses the rest
VQ_TC_CHANNEL_MULTIPLE, VQ_TC_CODE_MULTIPLE, VQ_TC_MAX_CODES = 64, 8, 16384
CLIP_ARCH = {
    "ViT-B/32": dict(width=768, layers=12, heads=12, patch=32, image_res=224, out_dim=512),
    "ViT-B/16": dict(width=768, layers=12, heads=12, patch=16, image_res=224, out_dim=512),
    "ViT-L/14": dict(width=1024, layers=24, heads=16, patch=14, image_res=224, out_dim=768),
    # 24^2 + 1 = 577 tokens: its attention runs on the streaming kernels (attn_long.cu)
    "ViT-L/14@336px": dict(width=1024, layers=24, heads=16, patch=14, image_res=336, out_dim=768),
}
# Image towers (pxr_set_clip_tower): openai-CLIP's VisionTransformer, the timm VisionTransformer of SLIP_Base, or
# openai-CLIP's ModifiedResNet
TOWER_OPENAI_CLIP, TOWER_TIMM_VIT, TOWER_CLIP_RESNET = 0, 1, 2
# openai-CLIP ModifiedResNet towers.  In the ClipCfg, width = the stem width w, layers = the bottleneck blocks of all four
# stages, heads = the attention pool's (32 w / 64).  `blocks` (per stage) is what a checkpoint's visual.layerN.i. keys are
# checked against (resnet_arch_of); like `tower` it is not a ClipCfg field.
RESNET_ARCH = {
    name: dict(width=w, layers=sum(b), heads=w // 2, patch=0, image_res=res, out_dim=d, tower=TOWER_CLIP_RESNET, blocks=b)
    for name, w, b, res, d in (("RN50", 64, (3, 4, 6, 3), 224, 1024), ("RN101", 64, (3, 4, 23, 3), 224, 512),
                               ("RN50x4", 80, (4, 6, 10, 6), 288, 640), ("RN50x16", 96, (6, 8, 18, 8), 384, 768),
                               ("RN50x64", 128, (3, 15, 36, 10), 448, 1024))
}
_NOT_CLIPCFG = ("tower", "blocks")


def resnet_arch_of(state_dict):
    """The ModifiedResNet shape a CLIP state_dict describes, as openai-CLIP's build_model derives it: the block count of
    each stage from the visual.layerN.i. keys, the stem width from layer1.0.conv1, the input side from the attention
    pool's positional_embedding (32 * sqrt(rows - 1)), out_dim from c_proj."""
    blocks = tuple(len({k.split(".")[2] for k in state_dict if k.startswith(f"visual.layer{s}.")}) for s in (1, 2, 3, 4))
    w = int(state_dict["visual.layer1.0.conv1.weight"].shape[0])
    side = round((state_dict["visual.attnpool.positional_embedding"].shape[0] - 1) ** 0.5)
    return dict(width=w, layers=sum(blocks), heads=w // 2, patch=0, image_res=32 * side,
                out_dim=int(state_dict["visual.attnpool.c_proj.weight"].shape[0]), tower=TOWER_CLIP_RESNET, blocks=blocks)


def check_resnet_state_dict(name, state_dict):
    """Refuse a checkpoint whose ModifiedResNet shape is not the one RESNET_ARCH gives `name`."""
    got, want = resnet_arch_of(state_dict), RESNET_ARCH[name]
    if got != want:
        raise EngineError(f"perceptor '{name}': the weights describe a ResNet with {got['blocks']} blocks per stage, stem "
                          f"width {got['width']}, input {got['image_res']} and out_dim {got['out_dim']}; {name} has "
                          f"{want['blocks']}, {want['width']}, {want['image_res']} and {want['out_dim']}")


# SLIP_Base models (slip.py:84-157, SLIP/models.py:288-331) whose image tower the engine builds: timm ViTs with 64-wide
# heads.  SLIP_CC3M / SLIP_CC12M are the B/16 architecture on other data (slip.py:134-135).  `tower` is not a ClipCfg
# field: B200Engine hands it to pxr_set_clip_tower.
_VIT_B16 = dict(width=768, layers=12, heads=12, patch=16, image_res=224, out_dim=512, tower=TOWER_TIMM_VIT)
_VIT_L16 = dict(width=1024, layers=24, heads=16, patch=16, image_res=224, out_dim=512, tower=TOWER_TIMM_VIT)
SLIP_ARCH = {"SLIP_VITB16": _VIT_B16, "SLIP_CC3M": _VIT_B16, "SLIP_CC12M": _VIT_B16, "CLIP_VITB16": _VIT_B16,
             "SLIP_VITL16": _VIT_L16, "CLIP_VITL16": _VIT_L16}
# SLIP models the engine refuses, with the reason
SLIP_UNSUPPORTED = {
    "SLIP_VITS16": "its vit_small_mocov3 tower has 12 heads over width 384 (32-wide heads); the fused attention and the "
                   "ViT builder cover 64-wide heads only",
    "CLIP_VITS16": "its vit_small_mocov3 tower has 12 heads over width 384 (32-wide heads); the fused attention and the "
                   "ViT builder cover 64-wide heads only",
    "SIMCLR_VITS16": "SIMCLR has no image_projection and no text tower, so it cannot score text prompts",
}


class EngineError(RuntimeError):
    pass


def vqgan_config(state_dict):
    """The architecture a taming VQGAN state_dict (VQModel or GumbelVQ keys, loss.* and any wrapper prefix removed)
    describes, as the dict B200Engine(vqgan=...) takes plus `gumbel` (the codebook is GumbelQuantize's quantize.embed):
    n_embed / embed_dim from the codebook, z_channels from post_quant_conv and decoder.conv_in, ch from decoder.conv_out,
    ch_mult and num_res_blocks from the decoder.up.* keys, attn_resolution from the level that carries attn.* keys.
    `resolution` is taming's 256: with the attention level it only places the attention blocks.  Refuses, naming the
    tensor, weights whose shapes disagree, and architectures the engine does not build."""
    def shape(name):
        if name not in state_dict:
            raise EngineError(f"VQGAN checkpoint: tensor '{name}' is missing")
        return tuple(int(d) for d in state_dict[name].shape)

    def refuse(name, why):
        raise EngineError(f"VQGAN checkpoint: '{name}' {why}")

    gumbel = "quantize.embed.weight" in state_dict
    if gumbel == ("quantize.embedding.weight" in state_dict):
        raise EngineError("VQGAN checkpoint: expected one codebook, 'quantize.embedding.weight' (VQModel) or "
                          f"'quantize.embed.weight' (GumbelVQ); found {'both' if gumbel else 'neither'}")
    cb_key = "quantize.embed.weight" if gumbel else "quantize.embedding.weight"
    cb = shape(cb_key)
    if len(cb) != 2:
        refuse(cb_key, f"has shape {list(cb)}; a codebook is [n_embed, embed_dim]")
    n_embed, embed_dim = cb
    pq = shape("post_quant_conv.weight")
    if len(pq) != 4 or pq[1:] != (embed_dim, 1, 1):
        refuse("post_quant_conv.weight", f"has shape {list(pq)}; the codebook {cb_key} has embed_dim {embed_dim}, so "
                                         f"it must be [z_channels, {embed_dim}, 1, 1]")
    zc = pq[0]
    if embed_dim != zc:
        refuse(cb_key, f"has embed_dim {embed_dim} but post_quant_conv.weight has z_channels {zc}; the engine builds "
                       "VQGANs with embed_dim == z_channels only")
    levels = sorted({int(k.split(".")[2]) for k in state_dict if k.startswith("decoder.up.")})
    if not levels or levels != list(range(len(levels))) or len(levels) > 8:
        raise EngineError(f"VQGAN checkpoint: the decoder.up.* keys name levels {levels}; expected 0 .. L-1 with 1 <= L <= 8")
    co = shape("decoder.conv_out.weight")
    ch = co[1]
    blocks, ch_mult = [], []
    for lv in levels:
        blocks.append(len({k.split(".")[4] for k in state_dict if k.startswith(f"decoder.up.{lv}.block.")}))
        name = f"decoder.up.{lv}.block.0.conv1.weight"
        out = shape(name)[0]
        if out % ch:
            refuse(name, f"has {out} output channels, not a multiple of ch = {ch} (decoder.conv_out.weight's input)")
        ch_mult.append(out // ch)
    if len(set(blocks)) != 1 or blocks[0] < 1:
        raise EngineError(f"VQGAN checkpoint: the decoder.up.<level>.block.* keys give {blocks} blocks per level; "
                          "expected the same num_res_blocks + 1 at every level")
    if ch_mult[0] != 1:
        refuse("decoder.up.0.block.0.conv1.weight", f"has {ch * ch_mult[0]} output channels but decoder.conv_out.weight "
                                                   f"reads {ch}; they must agree")
    cin = shape("decoder.conv_in.weight")
    if cin[:2] != (ch * ch_mult[-1], zc):
        refuse("decoder.conv_in.weight", f"has shape {list(cin)}; z_channels {zc} (post_quant_conv.weight) and the last "
                                         f"level's {ch * ch_mult[-1]} channels make it [{ch * ch_mult[-1]}, {zc}, 3, 3]")
    attn = [lv for lv in levels if any(k.startswith(f"decoder.up.{lv}.attn.") for k in state_dict)]
    if len(attn) > 1:
        raise EngineError(f"VQGAN checkpoint: decoder.up.<level>.attn.* keys at levels {attn}; the engine places attention "
                          "at one resolution")
    resolution = 256
    attn_resolution = resolution >> attn[0] if attn else 0
    if "encoder.conv_in.weight" in state_dict:
        if shape("encoder.conv_in.weight")[0] != ch:
            refuse("encoder.conv_in.weight", f"has {shape('encoder.conv_in.weight')[0]} output channels; the decoder's "
                                             f"ch is {ch}")
        enc_attn = [lv for lv in levels if any(k.startswith(f"encoder.down.{lv}.attn.") for k in state_dict)]
        if enc_attn != attn:
            raise EngineError(f"VQGAN checkpoint: encoder.down.<level>.attn.* keys at levels {enc_attn}, "
                              f"decoder.up.<level>.attn.* at {attn}; they must match")
        if gumbel and shape("quantize.proj.weight") != (n_embed, zc, 1, 1):
            refuse("quantize.proj.weight", f"has shape {list(shape('quantize.proj.weight'))}; GumbelQuantize's projection "
                                           f"is [{n_embed}, {zc}, 1, 1]")
    if zc % VQ_TC_CHANNEL_MULTIPLE:
        refuse("post_quant_conv.weight", f"gives z_channels {zc}; the engine needs a multiple of {VQ_TC_CHANNEL_MULTIPLE}")
    if n_embed % VQ_TC_CODE_MULTIPLE or n_embed > VQ_TC_MAX_CODES:
        refuse(cb_key, f"has {n_embed} codes; the engine's nearest-code search takes a multiple of {VQ_TC_CODE_MULTIPLE} "
                       f"up to {VQ_TC_MAX_CODES}")
    return dict(z_channels=zc, n_embed=n_embed, ch=ch, ch_mult=tuple(ch_mult), num_res_blocks=blocks[0] - 1,
                attn_resolution=attn_resolution, resolution=resolution, gumbel=gumbel)


def aux_loss_width(kind, n_sets):
    """Loss-vector entries of one auxiliary loss: a cutout-space loss (saturation, palette, smoothness) has one per
    cutout set, in set order (its get_loss returns a list, spliced in by pixray.py:1392-1398); the others one."""
    return n_sets if kind in (LOSS_SATURATION, LOSS_PALETTE, LOSS_SMOOTHNESS) else 1


def cutout_sets(cut_size, image_res):
    """(cut sizes, set of each perceptor): set 0 at cut_size (the first perceptor's resolution), then every other
    resolution in order of first appearance, as the reference fills cutoutsTable (pixray.py:642-649)."""
    sizes, set_of = [int(cut_size)], []
    for i, r in enumerate(image_res):
        r = int(cut_size) if i == 0 else int(r)
        if r not in sizes:
            sizes.append(r)
        set_of.append(sizes.index(r))
    return sizes, set_of


def stroke_z_layout(n_paths, n_segments):
    """Sizes of the line drawer's z ranges: (points, widths, paper RGBA)."""
    return n_paths * (3 * n_segments + 1) * 2, n_paths, 4


class B200Engine:
    # the image-tower kinds this library builds (pxr_set_clip_tower)
    TOWERS = (TOWER_OPENAI_CLIP, TOWER_TIMM_VIT, TOWER_CLIP_RESNET)
    # perceptors per session, and whether they may have different input resolutions (one cutout set each)
    MAX_PERCEPTORS = 4
    MIXED_RESOLUTIONS = True

    def __init__(self, *, drawer=DRAWER_VQGAN, image_hw=(256, 256), vqgan=None, grid=None, cutn=64, cut_size=224,
                 clip=(), noise_fac=0.1, seed=0, device=0, rank=0, world=1, grad_scale=0.0, lr_betas=(0.9, 0.999),
                 adam_eps=1e-8, fft_decay=0.0, fft_colors=0.0, fft_contrast=0.0, cut_aspect=1.0, polygons=None,
                 superres=None, strokes=None, vdiff_gen_hw=None):
        if not torch.cuda.is_available():
            raise EngineError("pixray_b200 needs a CUDA device (H100); there is no CPU fallback")
        self.lib = _lib.load()
        cfg = _lib.Config()
        cfg.device, cfg.rank, cfg.world = device, rank, world
        cfg.drawer = drawer
        cfg.image_h, cfg.image_w = image_hw
        if drawer == DRAWER_VQGAN:
            v = dict(VQGAN_F16_16384) if vqgan is None else dict(vqgan)
            cfg.z_channels, cfg.n_embed, cfg.ch = v["z_channels"], v["n_embed"], v["ch"]
            cfg.num_res_blocks, cfg.attn_resolution, cfg.resolution = v["num_res_blocks"], v["attn_resolution"], v["resolution"]
            cfg.n_levels = len(v["ch_mult"])
            for i, m in enumerate(v["ch_mult"]):
                cfg.ch_mult[i] = m
            f = 2 ** (cfg.n_levels - 1)
            self.z_shape = (1, cfg.z_channels, image_hw[0] // f, image_hw[1] // f)
            # a GumbelVQ (vqgan_config's `gumbel`): the engine reads its codebook from quantize.embed.weight and encodes
            # with vqgan_encode_gumbel
            self.gumbel = bool(v.get("gumbel", False))
        elif drawer == DRAWER_VDIFF:
            # VdiffDrawer's x (vdiff.py:118): [1, 3, gen_height, gen_width]; vdiff_gen_hw = (gen_h, gen_w), each side a
            # multiple of 64 and at least the canvas's (None: the canvas); the image is the canvas-size window centred in it
            gen_hw = tuple(image_hw) if vdiff_gen_hw is None else (int(vdiff_gen_hw[0]), int(vdiff_gen_hw[1]))
            self.z_shape = (1, 3, gen_hw[0], gen_hw[1])
        elif drawer == DRAWER_SUPERRES:
            # SuperResolutionDrawer's z (super_resolution.py:75-76): [1, 3, H/4, W/4]; the canvas is 4x the latent
            if image_hw[0] % 4 or image_hw[1] % 4:
                raise EngineError("drawer=DRAWER_SUPERRES needs canvas sides that are multiples of 4")
            r = dict(RRDBNET_X4PLUS) if superres is None else dict(superres)
            cfg.ch, cfg.num_block, cfg.num_grow_ch = r["num_feat"], r["num_block"], r["num_grow_ch"]
            self.z_shape = (1, 3, image_hw[0] // 4, image_hw[1] // 4)
        elif drawer == DRAWER_FFT:
            # FftDrawer params (fftdrawer.py:57-61): rfft2 spectrum [1, 3, H, W/2+1, 2]
            self.z_shape = (1, 3, image_hw[0], image_hw[1] // 2 + 1, 2)
        elif drawer == DRAWER_POLYGON:
            # PixelDrawer's shaped cells (pixeldrawer.py:200-304): polygons = (xy [total_vertices, 2], offsets [n + 1]) from
            # pixel_shapes.polygons; z = the [n, 4] RGBA fill colours, get_z's layout (pixeldrawer.py:384-390)
            if polygons is None:
                raise EngineError("drawer=DRAWER_POLYGON needs polygons=(xy, offsets)")
            xy = np.ascontiguousarray(np.asarray(polygons[0], dtype=np.float32).reshape(-1, 2))
            off = np.ascontiguousarray(np.asarray(polygons[1], dtype=np.int32).reshape(-1))
            self.z_shape = (int(off.size) - 1, 4)
        elif drawer == DRAWER_STROKES:
            # LineDrawer (linedrawer.py:44-126): strokes = (n_paths, n_segments, max_width, paper_trainable); z = the packed
            # [points n_paths * (3 n_segments + 1) * 2 | widths n_paths | paper RGBA 4] (stroke_z_layout)
            if strokes is None:
                raise EngineError("drawer=DRAWER_STROKES needs strokes=(n_paths, n_segments, max_width, paper_trainable)")
            n_paths, n_segments = int(strokes[0]), int(strokes[1])
            self.z_shape = (sum(stroke_z_layout(n_paths, n_segments)),)
        else:
            cfg.grid_rows, cfg.grid_cols = grid
            self.z_shape = (1, 3, grid[0], grid[1])
        cfg.cutn, cfg.cut_size = cutn, cut_size
        cfg.n_clip = len(clip)
        for i, c in enumerate(clip):
            for k, val in c.items():
                if k not in _NOT_CLIPCFG:
                    setattr(cfg.clip[i], k, val)
        cfg.noise_fac, cfg.seed = noise_fac, seed
        cfg.op_dtype, cfg.grad_scale = 0, grad_scale
        cfg.beta1, cfg.beta2, cfg.adam_eps = lr_betas[0], lr_betas[1], adam_eps
        cfg.fft_decay, cfg.fft_colors, cfg.fft_contrast = fft_decay, fft_colors, fft_contrast  # 0 -> 1.5 / 1.5 / 0.9
        cfg.cut_aspect = float(cut_aspect)  # global_aspect_width (pixray.py:1931); 1 = square canvas
        self.cut_aspect = float(cut_aspect)
        if self.cut_aspect != 1.0:  # the stretched source size in Python double arithmetic, like the reference computes it
            from .cutouts import source_size
            cfg.cut_src_h, cfg.cut_src_w = source_size(cut_size, self.cut_aspect)
        self.cfg = cfg
        self.device = torch.device("cuda", device)
        self.cutn, self.cut_size, self.world, self.rank = cutn, cut_size, world, rank
        self.n_local = cutn // world
        self.image_hw = tuple(image_hw)
        self.clip_dims = [c["out_dim"] for c in clip]
        # the cutout sets (the reference's cutoutsTable, pixray.py:642-649): set 0 at cut_size, then every other input
        # resolution in order of first appearance; set_of[i] is perceptor i's set
        self.cut_sets, self.set_of = cutout_sets(cut_size, [c["image_res"] for c in clip])
        self.n_prompts = [0 for _ in clip]  # loss slots per perceptor: text prompts + image prompts
        self._n_text = [0 for _ in clip]
        self._n_spot = [[0, 0] for _ in clip]  # [spot off, spot] prompts per perceptor (scored in the fused path only)
        self._n_img = 0
        h = C.c_void_p()
        rc = self.lib.pxr_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise EngineError(f"pxr_create failed ({rc}): {self.lib.pxr_last_error(None).decode()}")
        self.h = h
        self._keep = []
        for i, c in enumerate(clip):
            if c.get("tower", TOWER_OPENAI_CLIP) != TOWER_OPENAI_CLIP:
                self._check(self.lib.pxr_set_clip_tower(self.h, i, int(c["tower"])), "pxr_set_clip_tower")
        if drawer == DRAWER_POLYGON:
            rc = self.lib.pxr_set_polygons(self.h, xy.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p),
                                           int(off.size) - 1)
            self._check(rc, "pxr_set_polygons")
        if drawer == DRAWER_STROKES:
            rc = self.lib.pxr_set_strokes(self.h, n_paths, n_segments, C.c_float(float(strokes[2])), int(bool(strokes[3])))
            self._check(rc, "pxr_set_strokes")
        if drawer == DRAWER_VDIFF and vdiff_gen_hw is not None:
            self._check(self.lib.pxr_vdiff_set_gen_size(self.h, gen_hw[0], gen_hw[1]), "pxr_vdiff_set_gen_size")
        self._ext = None  # torch view of the engine's stream (ordering against torch-side producers of z / noise)

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc, what):
        if rc != 0:
            raise EngineError(f"{what} failed ({rc}): {self.lib.pxr_last_error(self.h).decode()}")

    def close(self):
        if getattr(self, "h", None):
            self.lib.pxr_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        self._check(self.lib.pxr_sync(self.h), "pxr_sync")

    @staticmethod
    def _p(t):
        return None if t is None else C.c_void_p(t.data_ptr())

    def _p_inplace(self, t, what):
        """Raw pointer of a tensor the library reads AND writes in place: it must be a dense, contiguous fp32 CUDA
        tensor (the C ABI sees plain NCHW memory; a permuted-stride tensor would be silently misread)."""
        if t is None:
            return None
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise EngineError(f"{what} must be a contiguous float32 CUDA tensor (got dtype={t.dtype}, "
                              f"device={t.device}, strides={tuple(t.stride())})")
        return C.c_void_p(t.data_ptr())

    def _new(self, *shape):
        return torch.empty(*shape, device=self.device, dtype=torch.float32)

    # ------------------------------------------------------------------ setup
    def load_module(self, module_id, state_dict):
        """Feed a reference-style state_dict (taming VQModel or openai-CLIP 'visual.*' keys)."""
        for name, t in state_dict.items():
            if not torch.is_floating_point(t):
                continue
            a = t.detach().to(torch.float32).contiguous().cpu()
            dims = (C.c_int64 * max(a.dim(), 1))(*(a.shape if a.dim() else (1,)))
            rc = self.lib.pxr_load_weight(self.h, module_id, name.encode(), C.c_void_p(a.data_ptr()), dims,
                                          max(a.dim(), 1))
            self._check(rc, f"pxr_load_weight({name})")

    def finalize(self):
        self._check(self.lib.pxr_finalize(self.h), "pxr_finalize")

    def set_prompts(self, clip_idx, embeds, weights, stops):
        e = np.ascontiguousarray(np.asarray(embeds, dtype=np.float32))
        w = np.ascontiguousarray(np.asarray(weights, dtype=np.float32))
        s = np.ascontiguousarray(np.asarray(stops, dtype=np.float32))
        s = np.maximum(s, np.float32(-3.0e38))  # -inf -> lowest finite (maximum(d, -inf) == d either way)
        n, D = e.shape
        rc = self.lib.pxr_set_prompts(self.h, clip_idx, e.ctypes.data_as(C.c_void_p), n, D,
                                      w.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p))
        self._check(rc, "pxr_set_prompts")
        self._n_text[clip_idx] = n
        self.n_prompts[clip_idx] = n + self._n_img

    def set_image_prompts(self, imgs, weights=None):
        """Image prompts (pixray.py:1308-1336): target images in [0, 1], each [1|-, 3, h, w] at ITS OWN size (a list), or one
        [n, 3, H, W] tensor.  Every iteration each is cut with that iteration's cached transforms, encoded by every
        perceptor and scored as a throwaway Prompt(embed [cutn, D], weight) appended after the perceptor's text prompts.
        n = 0 clears them."""
        if imgs is None or len(imgs) == 0:
            items = []
        elif torch.is_tensor(imgs):
            items = [t for t in torch.as_tensor(imgs, dtype=torch.float32).reshape(-1, 3, *imgs.shape[-2:])]
        else:
            items = [torch.as_tensor(t, dtype=torch.float32).reshape(3, *t.shape[-2:]) for t in imgs]
        items = [t.contiguous().cpu() for t in items]
        n = len(items)
        ptrs = (C.c_void_p * max(n, 1))(*[t.data_ptr() for t in items])
        hs = (C.c_int * max(n, 1))(*[t.shape[1] for t in items])
        ws = (C.c_int * max(n, 1))(*[t.shape[2] for t in items])
        wp = None
        if n and weights is not None:
            w = np.ascontiguousarray(np.asarray(weights, dtype=np.float32).reshape(n))
            wp = w.ctypes.data_as(C.c_void_p)
        self._check(self.lib.pxr_set_image_prompts_sized(self.h, ptrs, hs, ws, n, wp), "pxr_set_image_prompts_sized")
        self._n_img = n
        self.n_prompts = [t_ + n for t_ in self._n_text]

    def set_spot_mask(self, mask):
        """fetch_spot_indexes (pixray.py:370-394): bool / 0-1 array [3, cut_size, cut_size] (or [cut_size, cut_size]), True
        where the resized mask image is >= 0.5."""
        m = np.asarray(mask.cpu() if torch.is_tensor(mask) else mask)
        if m.ndim == 2:
            m = np.broadcast_to(m[None], (3,) + m.shape)
        m = np.ascontiguousarray((m != 0).astype(np.uint8).reshape(3, self.cut_size, self.cut_size))
        self._check(self.lib.pxr_set_spot_mask(self.h, m.ctypes.data_as(C.c_void_p)), "pxr_set_spot_mask")

    def set_spot_prompts(self, clip_idx, which, embeds, weights, stops):
        """args.spot_prompts (which = 1) / args.spot_prompts_off (which = 0) of one perceptor (pixray.py:917-931): scored on
        the cutouts of the masked image, ahead of the regular prompts in the loss vector.  Empty list clears."""
        w = np.ascontiguousarray(np.asarray(weights, dtype=np.float32).reshape(-1))
        n = int(w.size)
        s = np.maximum(np.ascontiguousarray(np.asarray(stops, dtype=np.float32).reshape(-1)), np.float32(-3.0e38))
        D = self.clip_dims[clip_idx]
        e = np.ascontiguousarray(np.asarray(embeds, dtype=np.float32).reshape(n, D)) if n else np.zeros((1, D), np.float32)
        rc = self.lib.pxr_set_spot_prompts(self.h, clip_idx, int(which), e.ctypes.data_as(C.c_void_p), n, D,
                                           w.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p))
        self._check(rc, "pxr_set_spot_prompts")
        self._n_spot[clip_idx][int(which)] = n

    def add_aux_loss(self, kind, weight, params):
        """One more entry of the loss vector / term of the gradient (pxr_add_aux_loss; Losses/*.py).  Returns the
        index of its value in the loss vector."""
        a = np.ascontiguousarray(np.asarray(params, dtype=np.float32).reshape(-1))
        rc = self.lib.pxr_add_aux_loss(self.h, int(kind), C.c_float(float(weight)), a.ctypes.data_as(C.c_void_p), int(a.size))
        self._check(rc, "pxr_add_aux_loss")
        return self.num_losses() - aux_loss_width(kind, len(self.cut_sets))

    def add_filter(self, kind, weight, params):
        """One more filter between synth and the cutouts (pxr_add_filter; filters/*.py).  Its loss takes the next entry at the
        FRONT of the loss vector.  Returns the filter's index."""
        a = np.ascontiguousarray(np.asarray(params, dtype=np.float32).reshape(-1))
        rc = self.lib.pxr_add_filter(self.h, int(kind), C.c_float(float(weight)), a.ctypes.data_as(C.c_void_p), int(a.size))
        self._check(rc, "pxr_add_filter")
        self._n_filters = getattr(self, "_n_filters", 0) + 1
        return self._n_filters - 1

    def clear_filters(self):
        self._check(self.lib.pxr_clear_filters(self.h), "pxr_clear_filters")
        self._n_filters = 0

    def set_filter_shifts(self, filter_idx, rand_h, rand_w):
        """Fix one filter's (rand_h, rand_w) draws (replays / parity tests); negative values hand them back to the engine."""
        self._check(self.lib.pxr_set_filter_shifts(self.h, int(filter_idx), int(rand_h), int(rand_w)), "pxr_set_filter_shifts")

    def add_anchor(self, kind, weight, ref):
        """One anchor term between the latent (or the image, ANCHOR_PIX) and a stored copy (pxr_add_anchor; the init_weight
        family and image_labels, pixray.py:1344-1375).  `ref`: torch tensor (any device) or array; copied."""
        if torch.is_tensor(ref):
            r = ref.detach().to(torch.float32).contiguous()
            ptr, n, keep = C.c_void_p(r.data_ptr()), r.numel(), r
        else:
            keep = np.ascontiguousarray(np.asarray(ref, dtype=np.float32).reshape(-1))
            ptr, n = keep.ctypes.data_as(C.c_void_p), keep.size
        rc = self.lib.pxr_add_anchor(self.h, int(kind), C.c_float(float(weight)), ptr, C.c_longlong(int(n)))
        self._check(rc, "pxr_add_anchor")
        del keep

    def clear_anchors(self):
        self._check(self.lib.pxr_clear_anchors(self.h), "pxr_clear_anchors")

    def clear_aux_losses(self):
        self._check(self.lib.pxr_clear_aux_losses(self.h), "pxr_clear_aux_losses")

    def num_losses(self):
        n = C.c_int()
        self.lib.pxr_num_losses(self.h, C.byref(n))
        return n.value

    def read_losses(self):
        """The loss vector of the last forward/backward: prompts of every perceptor, then the auxiliary losses."""
        out = np.zeros(max(self.num_losses(), 1), dtype=np.float32)
        self._check(self.lib.pxr_read_losses(self.h, out.ctypes.data_as(C.c_void_p)), "pxr_read_losses")
        return out[:self.num_losses()]

    # ------------------------------------------------------------------ vdiff drawer
    def vdiff_set_schedule(self, steps, alphas, sigmas):
        """sample_state's steps / alphas / sigmas (vdiff.py:113-126, sampling.py:41-51)."""
        a = [np.ascontiguousarray(np.asarray(v, dtype=np.float32).reshape(-1)) for v in (steps, alphas, sigmas)]
        rc = self.lib.pxr_vdiff_set_schedule(self.h, *(v.ctypes.data_as(C.c_void_p) for v in a), int(a[0].size))
        self._check(rc, "pxr_vdiff_set_schedule")

    def vdiff_set_clip_embed(self, embed):
        e = np.ascontiguousarray(np.asarray(embed, dtype=np.float32).reshape(-1))
        self._check(self.lib.pxr_vdiff_set_clip_embed(self.h, e.ctypes.data_as(C.c_void_p), int(e.size)), "pxr_vdiff_set_clip_embed")

    def vdiff_set_iteration(self, i):
        self.lib.pxr_vdiff_set_iteration(self.h, int(i))

    def vdiff_renoise(self, z, i, noise=None):
        """drawer.makenoise(cur_it) (vdiff.py:156-157): in place on z; noise [1,3,H,W] ~ N(0,1) or None (eta = 0)."""
        if noise is not None:
            noise = noise.to(self.device, torch.float32).contiguous()
            torch.cuda.current_stream().synchronize()
        rc = self.lib.pxr_vdiff_renoise(self.h, self._p_inplace(z, "z"), int(i), self._p(noise))
        self._check(rc, "pxr_vdiff_renoise")
        self.sync()
        return z

    def init_comm(self):
        """Cutout-sharded multi-GPU mode: rank 0 draws an ncclUniqueId, torch.distributed (already initialised by the
        launcher) broadcasts it, and the engine builds its own communicator (pxr_set_comm)."""
        import os

        import torch.distributed as dist
        if self.world == 1:
            return
        if "PXR_NCCL_LIB" not in os.environ:
            try:
                import nvidia.nccl
                cand = os.path.join(os.path.dirname(nvidia.nccl.__file__), "lib", "libnccl.so.2")
                if os.path.exists(cand):
                    os.environ["PXR_NCCL_LIB"] = cand
            except Exception:
                pass
        buf = (C.c_ubyte * 128)()
        if self.rank == 0:
            rc = self.lib.pxr_get_unique_id(buf)
            if rc != 0:
                raise EngineError(f"pxr_get_unique_id failed ({rc}): {self.lib.pxr_last_error(None).decode()}")
        dev = self.device if dist.get_backend() == "nccl" else torch.device("cpu")
        t = torch.tensor(list(buf), dtype=torch.uint8, device=dev)
        dist.broadcast(t, src=0)
        raw = bytes(t.cpu().tolist())
        self._check(self.lib.pxr_set_comm(self.h, raw, self.rank, self.world), "pxr_set_comm")

    def z_bounds(self):
        zc = self.z_shape[1]
        lo, hi = self._new(zc), self._new(zc)
        self._check(self.lib.pxr_z_bounds(self.h, self._p(lo), self._p(hi)), "pxr_z_bounds")
        self.sync()
        return lo, hi

    def set_color_jitter(self, p=0.8, saturation=0.1, hue=0.1):
        """Distribution of the engine-drawn K.ColorJitter stage (pixray.py:416, 436); p=0 turns it off."""
        self._check(self.lib.pxr_set_color_jitter(self.h, C.c_float(p), C.c_float(saturation), C.c_float(hue)),
                    "pxr_set_color_jitter")

    def _cut_params(self, transforms, zoom_padding, fill, noise_facs, noise, color_jitter=None, cs=None, keep=None):
        """pxr_cut_params for a set of cut size cs; the arrays it points to are kept alive in `keep` (default: until
        the next call)."""
        p = _lib.CutParams()
        if keep is None:
            keep = []
            self._keep = keep
        if color_jitter is not None:
            cj = np.ascontiguousarray(np.asarray(color_jitter, dtype=np.float32).reshape(self.cutn, 3))
            keep.append(cj)
            p.color_jitter = cj.ctypes.data_as(C.c_void_p)
        if transforms is not None:
            t = np.ascontiguousarray(np.asarray(transforms, dtype=np.float32).reshape(self.cutn, 9))
            keep.append(t)
            p.transforms = t.ctypes.data_as(C.c_void_p)
        p.zoom_padding, p.fill = int(zoom_padding), float(fill)
        if noise_facs is not None:
            f = np.ascontiguousarray(np.asarray(noise_facs, dtype=np.float32).reshape(self.cutn))
            keep.append(f)
            p.noise_facs = f.ctypes.data_as(C.c_void_p)
        if noise is not None:
            nz = noise.to(self.device, torch.float32).contiguous()
            if cs is not None and nz.numel() != self.cutn * 3 * cs * cs:
                raise EngineError(f"noise must be [cutn, 3, {cs}, {cs}] for a cutout set of size {cs}")
            keep.append(nz)
            p.noise = C.c_void_p(nz.data_ptr())
        return p

    # ------------------------------------------------------------------ per-op entry points (parity tests)
    def synth(self, z):
        z = z.to(self.device, torch.float32).contiguous()
        out = self._new(1, 3, *self.image_hw)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.pxr_synth(self.h, self._p(z), self._p(out)), "pxr_synth")
        self.sync()
        return out

    def set_synth_iteration(self, it):
        """The iteration the next synth() renders (drawer.synth(cur_iteration)): keys the polygon drawer's samples."""
        self._check(self.lib.pxr_set_synth_iteration(self.h, int(it)), "pxr_set_synth_iteration")

    def vqgan_encode(self, img):
        """z = model.encode(img)[0] (vqgan.py:174-185): img [1, 3, H, W] in [-1, 1] -> z [1, C, h, w] (codebook rows)."""
        img = img.to(self.device, torch.float32).reshape(1, 3, *self.image_hw).contiguous()
        out = self._new(*self.z_shape)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.pxr_vqgan_encode(self.h, self._p(img), self._p(out)), "pxr_vqgan_encode")
        self.sync()
        return out

    def vqgan_encode_gumbel(self, img, noise):
        """z = model.encode(img)[0] of a GumbelVQ (GumbelQuantize in eval mode, vqgan.py:174-185): img [1, 3, H, W] in
        [-1, 1], noise the Gumbel draws F.gumbel_softmax adds to quantize.proj's logits, [1|-, n_embed, h, w] ->
        z [1, C, h, w] (codebook rows)."""
        img = img.to(self.device, torch.float32).reshape(1, 3, *self.image_hw).contiguous()
        noise = noise.to(self.device, torch.float32).reshape(self.cfg.n_embed, *self.z_shape[2:]).contiguous()
        out = self._new(*self.z_shape)
        torch.cuda.current_stream().synchronize()
        self._check(self.lib.pxr_vqgan_encode_gumbel(self.h, self._p(img), self._p(noise), self._p(out)),
                    "pxr_vqgan_encode_gumbel")
        self.sync()
        return out

    def make_cutouts(self, img=None, *, transforms=None, zoom_padding=PAD_REFLECTION, fill=0.0, noise_facs=None,
                     noise=None, it=0, use_engine_rng=False, color_jitter=None, cut_set=0):
        """The cutouts of cutout set `cut_set` (pxr_make_cutouts_set): [cutn_local, 3, cs, cs] at that set's size."""
        if img is not None:
            img = img.to(self.device, torch.float32).contiguous()
        cs = self.cut_sets[cut_set]
        out = self._new(self.n_local, 3, cs, cs)
        p = None if use_engine_rng else self._cut_params(transforms, zoom_padding, fill, noise_facs, noise,
                                                                color_jitter, cs)
        torch.cuda.current_stream().synchronize()
        rc = self.lib.pxr_make_cutouts_set(self.h, int(cut_set), self._p(img), None if p is None else C.byref(p), it,
                                           self._p(out))
        self._check(rc, "pxr_make_cutouts_set")
        self.sync()
        return out

    def cutout_sets(self):
        """The engine's cutout sets as it built them (pxr_cutout_sets): their cut sizes, in set order."""
        sizes = (C.c_int * 4)()
        rc = self.lib.pxr_cutout_sets(self.h, sizes)
        if rc < 0:
            self._check(rc, "pxr_cutout_sets")
        return list(sizes[:rc])

    def encode_image(self, clip_idx=0, batch=None):
        """Unit-norm embeddings of the current cutouts of the perceptor's set, or of `batch` [cutn_local,3,cs,cs] at
        that set's size when given."""
        out = self._new(self.n_local, self.clip_dims[clip_idx])
        if batch is not None:
            cs = self.cut_sets[self.set_of[clip_idx]]
            if tuple(batch.shape) != (self.n_local, 3, cs, cs):
                raise EngineError(f"encode_image: perceptor {clip_idx} reads {cs} x {cs} cutouts, got a batch of shape "
                                  f"{tuple(batch.shape)} (expected {(self.n_local, 3, cs, cs)})")
            batch = batch.to(self.device, torch.float32).contiguous()
            torch.cuda.current_stream().synchronize()
        self._check(self.lib.pxr_encode_image(self.h, clip_idx, self._p(batch), self._p(out)), "pxr_encode_image")
        self.sync()
        return out

    def text_tower(self, clip_idx=0):
        """dict(width, layers, ctx, out_dim) of perceptor clip_idx's text tower, or None when its weights had no text keys
        (pxr_text_tower)."""
        v = [C.c_int() for _ in range(4)]
        rc = self.lib.pxr_text_tower(self.h, int(clip_idx), *(C.byref(x) for x in v))
        if rc < 0:
            self._check(rc, "pxr_text_tower")
        return dict(zip(("width", "layers", "ctx", "out_dim"), (x.value for x in v))) if rc == 1 else None

    def encode_text(self, clip_idx, tokens):
        """encode_text(tokens).float() of perceptor clip_idx: token ids [n, ctx] (pixray_b200.tokenizer) -> un-normalised
        embeddings [n, D] on the device (pxr_encode_text)."""
        t = np.ascontiguousarray(np.asarray(tokens.cpu() if torch.is_tensor(tokens) else tokens, dtype=np.int64))
        t = t.reshape(-1, t.shape[-1])
        if t.size and (t.min() < 0 or t.max() > np.iinfo(np.int32).max):
            raise EngineError(f"token ids must lie in [0, 2^31): got [{t.min()}, {t.max()}]")
        t = t.astype(np.int32)
        out = self._new(t.shape[0], self.clip_dims[clip_idx])
        torch.cuda.current_stream().synchronize()
        rc = self.lib.pxr_encode_text(self.h, int(clip_idx), t.ctypes.data_as(C.c_void_p), int(t.shape[0]),
                                      int(t.shape[1]), self._p(out))
        self._check(rc, "pxr_encode_text")
        return out

    def prompt_loss(self, clip_idx=0, embeds=None):
        if embeds is not None:
            embeds = embeds.to(self.device, torch.float32).contiguous()
            torch.cuda.current_stream().synchronize()
        out = self._new(self.n_prompts[clip_idx])
        self._check(self.lib.pxr_prompt_loss(self.h, clip_idx, self._p(embeds), self._p(out)), "pxr_prompt_loss")
        self.sync()
        return out

    def backward(self):
        g = self._new(*self.z_shape)
        self._check(self.lib.pxr_backward(self.h, self._p(g)), "pxr_backward")
        self.sync()
        return g

    def step(self, z, lr, it=0):
        self._check(self.lib.pxr_step(self.h, self._p_inplace(z, "z"), C.c_float(lr), it), "pxr_step")
        self.sync()
        return z

    def reset_optimizer(self):
        self._check(self.lib.pxr_reset_optimizer(self.h), "pxr_reset_optimizer")

    def set_optimizer(self, kind):
        """Switch the update rule to `kind` (OPT_*) with fresh state, as reset_optimizer leaves it (pxr_set_optimizer)."""
        self._check(self.lib.pxr_set_optimizer(self.h, int(kind)), "pxr_set_optimizer")

    def save_state(self):
        """bytes: z, the optimiser's state and step count, and the drop bookkeeping (pxr_save_state)."""
        n = C.c_int64()
        self.lib.pxr_state_size(self.h, C.byref(n))
        buf = (C.c_ubyte * n.value)()
        self._check(self.lib.pxr_save_state(self.h, buf), "pxr_save_state")
        return bytes(buf)

    def load_state(self, blob):
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(self.lib.pxr_load_state(self.h, buf), "pxr_load_state")

    def read_z(self):
        """The engine's current latent (a copy)."""
        return self.debug_read("z", self.z_shape)

    def set_z_grad(self, g):
        """The gradient the next step() applies (the plugin loop accumulates z.grad over several passes itself)."""
        self._check(self.lib.pxr_set_z_grad(self.h, self._p_inplace(g, "z.grad")), "pxr_set_z_grad")

    def set_batches(self, batches):
        """args.batches (pixray.py:1464-1482): passes per iterate(), gradients accumulated, one optimiser step."""
        self._check(self.lib.pxr_set_batches(self.h, int(batches)), "pxr_set_batches")

    def set_schedule(self, base_lr, iter_drop_delay=12, max_loss_drops=0, auto_stop=False, drops=()):
        """checkdrop / learning-rate drops / auto-stop on the device (pxr_set_schedule): iterate() then ignores `lr`."""
        d = np.ascontiguousarray(np.asarray(list(drops), dtype=np.int32).reshape(-1))
        self._check(self.lib.pxr_set_schedule(self.h, C.c_float(float(base_lr)), int(iter_drop_delay), int(max_loss_drops),
                                              int(bool(auto_stop)), d.ctypes.data_as(C.c_void_p), int(d.size)),
                    "pxr_set_schedule")

    def poll_status(self):
        """The last completed managed iteration's record, read from pinned memory WITHOUT synchronising; None when no
        consistent record is available yet."""
        st = _lib.Status()
        rc = self.lib.pxr_poll_status(self.h, C.byref(st))
        if rc != 0:
            return None
        return dict(iter=st.iter, loss_sum=st.loss_sum, best_loss=st.best_loss, best_iter=st.best_iter,
                    num_loss_drop=st.num_loss_drop, stopped=bool(st.stopped), rebuilt=bool(st.rebuilt), lr=st.lr,
                    losses=np.array(st.losses[:st.n_losses], dtype=np.float32))

    # ------------------------------------------------------------------ the fast path (what bench.py times)
    def iterate(self, z, lr, it, *, params=None, losses_out=None):
        """One train() iteration entirely inside the library.  params: dict(transforms, zoom_padding, fill,
        noise_facs, noise, color_jitter), a list of such dicts (one per cutout set, pxr_iterate_sets), or None for the
        engine's own Philox draws.  losses_out: float32 numpy array (host) to receive the per-prompt losses (forces a
        stream sync), or None."""
        p = None
        per_set = isinstance(params, (list, tuple))
        if per_set and len(params) != len(self.cut_sets):
            raise EngineError(f"iterate: {len(params)} cutout parameter sets for {len(self.cut_sets)} cutout sets")
        if params is not None:
            keep = []
            self._keep = keep
            plist = [self._cut_params(q.get("transforms"), q.get("zoom_padding", it % 2), q.get("fill", 0.0),
                                      q.get("noise_facs"), q.get("noise"), q.get("color_jitter"), cs, keep)
                     for q, cs in zip(params if per_set else [params], self.cut_sets)]
            p = (_lib.CutParams * len(plist))(*plist)
        # z / noise may have been produced on torch's stream (e.g. an H2D copy still in flight): order the engine's
        # non-blocking stream after it without a host sync
        if self._ext is None:
            self._ext = torch.cuda.ExternalStream(self.stream_ptr())
        self._ext.wait_stream(torch.cuda.current_stream())
        lp = None if losses_out is None else losses_out.ctypes.data_as(C.c_void_p)
        fn, name = (self.lib.pxr_iterate_sets, "pxr_iterate_sets") if per_set else (self.lib.pxr_iterate, "pxr_iterate")
        rc = fn(self.h, self._p_inplace(z, "z"), C.c_float(lr), it, p, lp)
        self._check(rc, name)

    def debug_read(self, name, shape, dtype=torch.float32):
        out = torch.empty(*shape, device=self.device, dtype=dtype)
        rc = self.lib.pxr_debug_read(self.h, name.encode(), self._p(out), C.c_int64(out.numel() * out.element_size()))
        self._check(rc, f"pxr_debug_read({name})")
        return out

    def profile_iteration(self, z, lr, it):
        out = (C.c_double * 6)()
        tb = C.c_double(0.0)
        self._check(self.lib.pxr_profile_iteration2(self.h, self._p_inplace(z, "z"), C.c_float(lr), it, out, C.byref(tb)),
                    "pxr_profile_iteration2")
        return dict(gemm_ms=out[0], gemm_launches=int(out[1]), gemm_flops=out[2], other_ms=out[3],
                    other_launches=int(out[4]), total_ms=out[5], gemm_bytes=tb.value)

    def stream_ptr(self):
        p = C.c_void_p()
        self.lib.pxr_get_stream(self.h, C.byref(p))
        return p.value

    def num_launches(self):
        n = C.c_int64()
        self.lib.pxr_num_kernel_launches(self.h, C.byref(n))
        return n.value
