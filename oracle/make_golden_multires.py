"""Generate tests/golden/multires_ascend.npz by running the REAL reference ascend_txt with perceptors of two input
resolutions (container-only).

    python -m oracle.make_golden_multires

The unmodified pixray.ascend_txt (pixray.py:1243-1406) runs through oracle/shim.py with
  * two MakeCutouts in cutoutsTable (cut sizes 16 and 24, in that order), each with cached `transforms` and
    noise_fac = 0 (the cached path, pixray.py:480-486, is the one the stubbed kornia supports);
  * three small seeded perceptors with the CLIP_Base surface (slip.py:44-66) over the restated ViT: "A" and "C" at 16
    pixels share a cutout batch, "B" reads the 24-pixel one;
  * text prompts, one image prompt, and the reference's SaturationLoss, PaletteLoss and SmoothnessLoss classes as
    custom losses (each returns one entry per cutout size, pixray.py:1392-1398);
  * a canvas with global_aspect_width = 1.5.  kornia is not vendored: its `rescale` (the stretch of the pooled image,
    pixray.py:468-472) is stood in by the same bilinear F.interpolate as oracle/ref_path.rescale_for_aspect.
The ordered loss vector and d loss / d out are frozen with every input; tests/test_multires.py requires
oracle/multires_ref.iterate_sets to reproduce them.
"""
import os
import random
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref_path as R
from oracle import shim
from pixray_b200 import cutouts

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "multires_ascend.npz")
CUTN, SIZES, ASPECT = 5, (16, 24), 1.5
# name: (input resolution, patch, width, layers, heads, out_dim, seed of oracle/ref_path.init_clip_weights)
MODELS = {"A": (16, 8, 32, 1, 1, 16, 11), "B": (24, 8, 32, 2, 1, 16, 12), "C": (16, 4, 32, 1, 2, 16, 13)}


def _rescale(x, factor, *a, **k):  # kornia.geometry.transform.rescale: resize to int(size * factor), bilinear
    return F.interpolate(x, size=(int(x.shape[2] * factor[0]), int(x.shape[3] * factor[1])), mode="bilinear",
                         align_corners=False)


def main():
    px = shim.install()
    sys.modules["kornia.geometry.transform"].rescale = _rescale
    import slip
    from Losses.PaletteLoss import PaletteLoss
    from Losses.SaturationLoss import SaturationLoss
    from Losses.SmoothnessLoss import SmoothnessLoss

    G = {}
    g = torch.Generator().manual_seed(2468)
    out = torch.rand(1, 3, 20, 30, generator=g).requires_grad_(True)
    G["out"] = out.detach().numpy()
    px.global_aspect_width = ASPECT
    px.device = "cpu"
    px.cur_iteration, px.cur_anim_index = 1, None
    px.filters = None
    px.drawer = types.SimpleNamespace(synth=lambda it: out)
    px.cutoutsTable, px.cutoutSizeTable, px.perceptors = {}, {}, {}
    for cs in SIZES:
        mc = px.MakeCutouts(cs, CUTN)
        mc.noise_fac = 0
        px.cutoutsTable[cs] = mc
    T = {}
    for cs in SIZES:
        T[cs] = torch.from_numpy(cutouts.sample_transforms(CUTN, cs, 100 + cs, aspect=ASPECT))
        G[f"T{cs}"] = T[cs].numpy()
    pms, pims = {}, {}
    timg = torch.rand(1, 3, 14, 18, generator=g)
    G["timg"] = timg.numpy()
    for name, (res, patch, width, layers, heads, dim, seed) in MODELS.items():
        vit = R.init_clip_weights(R.ClipVisual(res, patch, width, layers, heads, dim), seed)
        px.perceptors[name] = slip.CLIP_Base(vit, None, "cpu")
        px.cutoutSizeTable[name] = res
        emb = torch.randn(2, dim, generator=g)
        G[f"pe_{name}"] = emb.numpy()
        pms[name] = [px.Prompt(emb[0:1], 1.0, float("-inf")), px.Prompt(emb[1:2], -0.4, float("-inf"))]
        pims[name] = [timg]
    px.pmsTable, px.pmsImageTable = pms, pims
    px.spotPmsTable, px.spotOffPmsTable, px.pmsTargetTable = {}, {}, {n: [] for n in MODELS}
    px.lossGlobals = {}
    palette = [[0.9, 0.1, 0.1], [0.1, 0.8, 0.2], [0.2, 0.2, 0.9]]
    G["palette"] = np.array(palette, dtype=np.float32)
    args = types.SimpleNamespace(
        clip_models=list(MODELS), spot_prompts=[], spot_prompts_off=[], image_prompt_shuffle=False,
        image_prompt_weight=0.7, image_labels=None, init_weight=0, init_weight_dist=0, init_weight_pix=0,
        init_weight_cos=0, transparent_weight=0, make_video=False, transparent=False,
        saturation_weight=1.3, palette=palette, palette_weight=0.8, smoothness_weight=0.9, smoothness_type="default",
        smoothness_gaussian_kernel=0, smoothness_gaussian_std=1, smoothness_spacing=1, smoothness_edge_order=1,
        custom_loss=[{"loss": SaturationLoss(device="cpu"), "weight": 1.0}, {"loss": PaletteLoss(device="cpu"), "weight": 0.5},
                     {"loss": SmoothnessLoss(device="cpu"), "weight": 2.0}])
    G["loss_weights"] = np.array([1.0, 0.5, 2.0], dtype=np.float32)
    for cs in SIZES:
        px.cutoutsTable[cs].transforms = T[cs].clone()
    random.seed(13)
    cwd = os.getcwd()
    os.chdir("/tmp")
    try:
        result = px.ascend_txt(args)
    finally:
        os.chdir(cwd)
    G["fill"] = np.float32(px.global_fill_color[0])
    G["zoom_padding"] = np.array(px.global_padding_mode)
    total = sum(result)
    total.backward()
    G["losses"] = np.array([float(r.detach()) for r in result], dtype=np.float32)
    G["d_out"] = out.grad.numpy()
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **G)
    print("wrote", OUT, "with", len(G), "arrays,", os.path.getsize(OUT), "bytes; losses", G["losses"])


if __name__ == "__main__":
    main()
