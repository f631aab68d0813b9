"""The super-resolution drawer (Real-ESRGAN RRDBNet x4, 23 RRDBs, seeded synthetic weights) in the whole iteration:
ViT-B/16, cutn 64, at 512 x 512 and 1024 x 1024 canvases (128^2 and 256^2 latents).  Prints the GPU and its power limit,
iterations per second of pxr_iterate (CUDA events on the engine's stream, host wall time beside them), and the drawer's
share of one profiled iteration (pxr_profile_iteration2's per-op CUDA events, median of several iterations): the
drawer's convolutions (GEMM) and its other kernels, with the TFLOP/s its convolutions reach against the FLOPs the net
needs (synthetic.superres_fwd_flops, forward and dgrad).  Writes nothing but a temporary file.

    python tools/bench_super_resolution.py [steps]
"""
import csv
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

MODEL, CUTN, SIZES = "ViT-B/16", 64, (512, 1024)
# the drawer's ops in the profile: its convolutions and split-K reduces, and its pointwise passes
DRAWER_GEMM = ("conv3x3",)
DRAWER_OTHER = ("splitk_reduce", "sr_axpy", "sr_zgrad", "upsample2x", "downsum2x", "image_finish", "image_to_nhwc64")


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # the name alone still identifies the card
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def build(side, sd):
    eng = E.B200Engine(drawer=E.DRAWER_SUPERRES, image_hw=(side, side), cutn=CUTN, clip=[E.CLIP_ARCH[MODEL]], seed=0)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(E.CLIP_ARCH[MODEL], 1))
    eng.finalize()
    pr = S.prompts(512, (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z = torch.rand(eng.z_shape, generator=torch.Generator().manual_seed(1)).cuda().contiguous()
    return eng, z


def measure(side, sd, steps, warm=3, profiles=5):
    eng, z = build(side, sd)
    lr = 0.05
    for i in range(warm):
        eng.iterate(z, lr, i)
    eng.sync()
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.time()
    e0.record(ext)
    for i in range(warm, warm + steps):
        eng.iterate(z, lr, i)
    e1.record(ext)
    eng.sync()
    torch.cuda.synchronize()
    wall_ms = (time.time() - w0) * 1e3 / steps
    ms = e0.elapsed_time(e1) / steps
    if not ms > 0.5 * wall_ms:  # the events on the engine's stream did not bracket the work: no trustworthy GPU time
        raise RuntimeError(f"{side}: CUDA events read {ms:.3f} ms/step against {wall_ms:.3f} ms/step of host wall time")
    gemm, other, total = [], [], []
    with tempfile.TemporaryDirectory() as d:
        os.environ["PXR_PROFILE_DUMP"] = os.path.join(d, "ops.csv")
        for j in range(profiles):
            prof = eng.profile_iteration(z, lr, warm + steps + j)
            g = o = 0.0
            for row in csv.DictReader(open(os.environ["PXR_PROFILE_DUMP"])):
                if row["op"].startswith(DRAWER_GEMM):
                    g += float(row["ms"])
                elif row["op"].startswith(DRAWER_OTHER):
                    o += float(row["ms"])
            gemm.append(g)
            other.append(o)
            total.append(prof["total_ms"])
        del os.environ["PXR_PROFILE_DUMP"]
    h = side // 4
    flops = 2 * S.superres_fwd_flops(h, h)
    g_ms, o_ms, t_ms = (float(np.median(v)) for v in (gemm, other, total))
    out = {"canvas": f"{side}x{side}", "latent": f"{h}x{h}", "iters_per_sec": 1e3 / ms, "ms_per_step": ms,
           "ms_per_step_clock": "CUDA events on the engine's stream", "wall_ms_per_step": wall_ms,
           "profiled_ms_per_step": t_ms, "drawer_gemm_ms": g_ms, "drawer_other_ms": o_ms,
           "drawer_share_of_profiled_step": (g_ms + o_ms) / t_ms, "drawer_tflop_fwd_plus_dgrad": flops / 1e12,
           "drawer_gemm_tflops_per_s": flops / (g_ms * 1e-3) / 1e12, "finite_z": bool(torch.isfinite(z).all())}
    eng.close()
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    sd = S.rrdbnet_state_dict(0)
    res = dict(gpu_info(), workload=f"RRDBNet x4 (23 RRDBs), {MODEL}, cutn {CUTN}", steps=steps,
               runs=[measure(s, sd, steps) for s in SIZES])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
