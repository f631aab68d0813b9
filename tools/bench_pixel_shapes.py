"""The pixel drawer's shaped cells against its square-grid fast path, at the reference's quality `normal`: 384x216 canvas,
ViT-B/32 + ViT-B/16, cutn 30, seeded synthetic weights.  Prints the GPU and its power limit, iterations per second of
pixel_type hex (5071 polygons on the polygon rasteriser) and of rect (the 80x45 nearest-upsample grid), and the CUDA-event
times of the drawer's own kernels (median of several profiled iterations).  Step times come from CUDA events on the
engine's stream; the host wall time is printed beside them, and the run stops with an error when the events read less
than half of it (they did not bracket the work).  Writes nothing but a temporary file.

    python tools/bench_pixel_shapes.py [steps]
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
from pixray_b200 import pixel_shapes as PS  # noqa: E402
from pixray_b200 import plugins as P  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

W, H, CUTN, MODELS = 384, 216, 30, ("ViT-B/32", "ViT-B/16")


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # the name alone still identifies the card
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def build(pixel_type):
    clip = [E.CLIP_ARCH[m] for m in MODELS]
    if pixel_type == "rect":
        rows, cols = P.FastPixelDrawer.grid_for((W, H), verbose=False)
        eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(H, W), grid=(rows, cols), cutn=CUTN, clip=clip, seed=0,
                           cut_aspect=W / H)
        z = torch.rand(eng.z_shape, device="cuda")
        kernels, n = ("pixel_synth", "pixel_synth_backward"), rows * cols
    else:
        rows, cols = PS.grid_for((W, H), pixel_type, verbose=False)
        xy, off = PS.polygons((W, H), rows, cols, pixel_type)
        eng = E.B200Engine(drawer=E.DRAWER_POLYGON, image_hw=(H, W), polygons=(xy, off), cutn=CUTN, clip=clip, seed=0,
                           cut_aspect=W / H)
        z = torch.from_numpy(PS.init_colours(torch.rand(1, 3, H, W) * 2 - 1, rows, cols, pixel_type)).cuda()
        kernels, n = ("raster_forward", "raster_backward"), len(off) - 1
    for i, m in enumerate(MODELS):
        eng.load_module(E.MOD_CLIP0 + i, S.clip_state_dict(E.CLIP_ARCH[m], 1 + i))
    eng.finalize()
    for i in range(len(MODELS)):
        pr = S.prompts(512, (1.0, 0.1), 2 + i)
        eng.set_prompts(i, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    return eng, z.contiguous(), kernels, n


def measure(pixel_type, steps, warm=5, profiles=7):
    eng, z, kernels, n = build(pixel_type)
    lr = 0.03 if pixel_type != "rect" else 0.2
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
        raise RuntimeError(f"{pixel_type}: CUDA events read {ms:.3f} ms/step against {wall_ms:.3f} ms/step of host wall time")
    times = {k: [] for k in kernels}
    with tempfile.TemporaryDirectory() as d:
        os.environ["PXR_PROFILE_DUMP"] = os.path.join(d, "ops.csv")
        for j in range(profiles):
            eng.profile_iteration(z, lr, warm + steps + j)
            for row in csv.DictReader(open(os.environ["PXR_PROFILE_DUMP"])):
                if row["op"] in times:
                    times[row["op"]].append(float(row["ms"]))
        del os.environ["PXR_PROFILE_DUMP"]
    out = {"pixel_type": pixel_type, "shapes_or_cells": n, "iters_per_sec": 1e3 / ms, "ms_per_step": ms,
           "ms_per_step_clock": "CUDA events on the engine's stream", "wall_ms_per_step": wall_ms,
           "finite_z": bool(torch.isfinite(z).all())}
    for k, v in times.items():
        out[k + "_us"] = float(np.median(v)) * 1e3
    eng.close()
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    res = dict(gpu_info(), workload=f"{W}x{H}, {' + '.join(MODELS)}, cutn {CUTN}", steps=steps,
               runs=[measure("hex", steps), measure("rect", steps)])
    res["hex_over_rect_time"] = res["runs"][0]["ms_per_step"] / res["runs"][1]["ms_per_step"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
