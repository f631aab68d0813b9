"""The line-sketch drawer's kernels and whole iteration.  Prints the GPU and its power limit, then for each workload the
CUDA-event times of the drawer's ops (median over profiled iterations: stroke_flatten, stroke_bin = count + scan + fill,
stroke_raster_fwd, stroke_raster_bwd = pixel weights + boundary quadrature + fold) and iterations per second of the
whole iteration at ViT-B/16, cutn 64, next to the vqgan drawer on the same canvas in the same call.  Workloads: the
reference's default 384 x 216 canvas with 24 paths x 8 segments, and a 1024 x 1024 canvas with 256 x 8.  Step times
come from CUDA events on the engine's stream; the run stops with an error when they read less than half the host wall
time.  Writes nothing but a temporary file.

    python tools/bench_line_sketch.py [steps]
"""
import csv
import json
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import plugins as P  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402
from bench_pixel_shapes import gpu_info  # noqa: E402

CUTN, MODEL = 64, "ViT-B/16"
OPS = ("stroke_flatten", "stroke_bin", "stroke_raster_fwd", "stroke_raster_bwd")


def build(kind, W, H, N=0, L=0):
    clip = [E.CLIP_ARCH[MODEL]]
    if kind == "line_sketch":
        mw = 2 * H / 100
        eng = E.B200Engine(drawer=E.DRAWER_STROKES, image_hw=(H, W), strokes=(N, L, mw, False), cutn=CUTN, clip=clip,
                           seed=0, cut_aspect=W / H)
        pts = P.line_start_points(W, H, N, L, rng=random.Random(0))
        z = torch.cat([pts.reshape(-1), torch.full((N,), max(1.0, mw / 2)), torch.tensor(P.PAPER_RGBA)])
    else:
        H, W = H // 16 * 16, W // 16 * 16
        eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(H, W), cutn=CUTN, clip=clip, seed=0, cut_aspect=W / H)
        vq = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
        eng.load_module(E.MOD_VQGAN, vq)
        code = torch.as_tensor(vq["quantize.embedding.weight"], dtype=torch.float32)
        idx = torch.randint(code.shape[0], (eng.z_shape[2] * eng.z_shape[3],), generator=torch.Generator().manual_seed(0))
        z = code[idx].T.reshape(eng.z_shape)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(E.CLIP_ARCH[MODEL], 1))
    eng.finalize()
    pr = S.prompts(512, (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    return eng, z.contiguous().cuda()


def measure(kind, W, H, N, L, steps, warm=5, profiles=9):
    eng, z = build(kind, W, H, N, L)
    lr = 1.0 if kind == "line_sketch" else 0.2
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
    if not ms > 0.5 * wall_ms:
        raise RuntimeError(f"{kind}: CUDA events read {ms:.3f} ms/step against {wall_ms:.3f} ms/step of host wall time")
    times = {k: [] for k in OPS}
    with tempfile.TemporaryDirectory() as d:
        os.environ["PXR_PROFILE_DUMP"] = os.path.join(d, "ops.csv")
        for j in range(profiles):
            eng.profile_iteration(z, lr, warm + steps + j)
            for row in csv.DictReader(open(os.environ["PXR_PROFILE_DUMP"])):
                if row["op"] in times:
                    times[row["op"]].append(float(row["ms"]))
        del os.environ["PXR_PROFILE_DUMP"]
    out = {"drawer": kind, "canvas": f"{W}x{H}", "iters_per_sec": 1e3 / ms, "ms_per_step": ms, "wall_ms_per_step": wall_ms,
           "finite_z": bool(torch.isfinite(z).all())}
    if kind == "line_sketch":
        out["paths"] = f"{N}x{L}"
        for k, v in times.items():
            out[k + "_us"] = float(np.median(v)) * 1e3
    eng.close()
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    res = dict(gpu_info(), workload=f"{MODEL}, cutn {CUTN}", steps=steps,
               runs=[measure("line_sketch", 384, 216, 24, 8, steps), measure("vqgan", 384, 216, 0, 0, steps),
                     measure("line_sketch", 1024, 1024, 256, 8, steps)])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
