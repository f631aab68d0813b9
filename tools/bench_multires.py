"""Perceptors of different input resolutions (one cutout set each) on the engine, in one call on one GPU, with seeded
synthetic weights, VQGAN 256^2:

  * iterations per second of pxr_iterate (CUDA events around `steps` iterations after a warm-up) for
      best        RN50x4 (288) + ViT-B/32 + ViT-B/16 (224), cutn 12 (quality="best"'s perceptors and cut count)
      supreme     RN50x4 (288) + RN101 + ViT-B/32 + ViT-B/16 (224), cutn 8 (quality="supreme")
      l336_b16    ViT-L/14@336px (336) + ViT-B/16 (224), cutn 32
    one pass per iteration (the presets' `batches` repeat it);
  * the cutout stage of each set in one profiled iteration (pxr_profile_iteration's "cutouts_fwd set k" / "cutouts_bwd set k"
    records: pooling, stretch, warps, range; the range terms, warp adjoint and pool adjoint), against the whole
    iteration's kernel time -- what a grouped launch across sets could save at most;
  * the GPU's name, power limit and maximum SM clock.
Prints one JSON line; writes nothing outside a temporary directory.

    python tools/bench_multires.py [steps]
"""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from bench_resnet import gpu_info, profile_rows, time_steps  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

SIDE = 256
CONFIGS = {
    "best": (["RN50x4", "ViT-B/32", "ViT-B/16"], 12),
    "supreme": (["RN50x4", "RN101", "ViT-B/32", "ViT-B/16"], 8),
    "l336_b16": (["ViT-L/14@336px", "ViT-B/16"], 32),
}


def build(models, cutn, vq_sd):
    archs = [E.RESNET_ARCH.get(m) or E.CLIP_ARCH[m] for m in models]
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE), cutn=cutn, cut_size=archs[0]["image_res"], clip=archs,
                       seed=0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    for i, (m, a) in enumerate(zip(models, archs)):
        sd = S.clip_resnet_state_dict(a, 1 + i) if m in E.RESNET_ARCH else S.clip_state_dict(a, 1 + i)
        eng.load_module(E.MOD_CLIP0 + i, sd)
    eng.finalize()
    for i, a in enumerate(archs):
        pr = S.prompts(a["out_dim"], (1.0, 0.1), 2 + i)
        eng.set_prompts(i, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3)
    return eng, z.cuda().contiguous()


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    res = dict(workload=f"VQGAN {SIDE}^2 drawer, synthetic weights, one pass per iteration", **gpu_info())
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    for name, (models, cutn) in CONFIGS.items():
        eng, z = build(models, cutn, vq_sd)
        try:
            time_steps(eng, z, 0, 3)
            s = time_steps(eng, z, 3, steps) / steps
            rows = profile_rows(eng, z, 3 + steps)
            sets = eng.cut_sets
        finally:
            eng.close()
        cut = {r["op"]: round(float(r["ms"]), 3) for r in rows if r["op"].startswith("cutouts_")}
        total = sum(float(r["ms"]) for r in rows)
        res[name] = dict(perceptors=models, cutn=cutn, cut_sets=sets, it_per_s=round(1.0 / s, 2),
                         cutout_stage_ms=cut, cutout_share=round(sum(cut.values()) / max(total, 1e-9), 4),
                         profiled_kernel_ms=round(total, 3))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
