"""BASELINE config 4 (vdiff cc12m_1 256x256, ViT-B/16, cutn=64) on one GPU: iterations/sec of the full body
(U-Net synth -> cutouts -> CLIP -> loss -> backward -> Adam -> makenoise), seeded random weights.  Informational
(bench.py measures config 2, the configuration BASELINE.json's metric is quoted on).

    python tools/bench_vdiff.py [steps] [--canvas WxH]

--canvas runs the drawer at any canvas the way the API does: the U-Net at the canvas rounded up to 128 per side, the
image its centre crop.  The JSON line adds the card's name and power limit, the engine's device allocation and the
three-kernel GroupNorm's achieved bytes/s (compulsory bytes from its shapes over its profiled time)."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_path as R  # noqa: E402  (only to build the seeded reference-initialised weights)
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402
from pixray_b200 import util as U  # noqa: E402

argv = [a for a in sys.argv[1:]]
canvas_w, canvas_h = 256, 256
if "--canvas" in argv:
    i = argv.index("--canvas")
    canvas_w, canvas_h = (int(v) for v in argv[i + 1].lower().split("x"))
    del argv[i:i + 2]
steps_n, warm = int(argv[0]) if argv else 10, 3
gen_w, gen_h, _, _ = U.vdiff_gen_size(canvas_w, canvas_h)
img_w, img_h = U.vdiff_image_size(canvas_w, canvas_h)
gen_kw = {} if (canvas_w, canvas_h) == (256, 256) else dict(vdiff_gen_hw=(gen_h, gen_w))
torch.manual_seed(0)
t0 = time.time()
sd = R.VDiffCC12M1().ref_state_dict()
clip_sd = S.clip_state_dict(E.CLIP_ARCH["ViT-B/16"], 1)
prompts = S.prompts(512, (1.0, 0.1), 2)
eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(img_h, img_w), cutn=64, clip=[E.CLIP_ARCH["ViT-B/16"]], seed=0,
                   cut_aspect=canvas_w / canvas_h, **gen_kw)
eng.load_module(E.MOD_VQGAN, sd)
eng.load_module(E.MOD_CLIP0, clip_sd)
eng.finalize()
print(f"setup {time.time() - t0:.1f} s", flush=True)
eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
iters = steps_n + warm
st, al, sg = U.vdiff_schedule(iters)
eng.vdiff_set_schedule(st, al, sg)
eng.vdiff_set_clip_embed(prompts[0][0].numpy())
z = (torch.randn(1, 3, gen_h, gen_w) * float(sg[0])).cuda().contiguous()
noise = torch.randn(1, 3, gen_h, gen_w, device="cuda")
ext = torch.cuda.ExternalStream(eng.stream_ptr())


def one(i):
    lr = min(float(sg[i] / al[i]) * 0.001, 0.01)  # pixray.py:1490-1494
    eng.reset_optimizer()
    eng.iterate(z, lr, i)
    eng.lib.pxr_vdiff_renoise(eng.h, eng._p_inplace(z, "z"), i, eng._p(noise))


for i in range(warm):
    one(i)
eng.sync()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize()
w0 = time.time()
e0.record(ext)
for i in range(warm, iters):
    one(i)
e1.record(ext)
eng.sync()
torch.cuda.synchronize()
wall_ms = (time.time() - w0) * 1e3 / steps_n
ms = e0.elapsed_time(e1) / steps_n
print(f"events {ms:.3f} ms/step, wall {wall_ms:.3f} ms/step", flush=True)
ms = max(ms, 0.0) if ms > 0.5 * wall_ms else wall_ms  # an ExternalStream event pair that does not bracket the work reads ~0
os.makedirs("gpurun_out", exist_ok=True)
os.environ["PXR_PROFILE_DUMP"] = "gpurun_out/vdiff_ops.tmp"
prof = eng.profile_iteration(z, 0.001, iters - 1)
import collections  # noqa: E402
import csv  # noqa: E402
import re  # noqa: E402
agg = collections.OrderedDict()
gn3_bytes, gn3_ms = 0.0, 0.0
for row in csv.DictReader(open("gpurun_out/vdiff_ops.tmp")):
    a = agg.setdefault(row["op"], [0, 0.0, 0.0])
    a[0] += 1
    a[1] += float(row["ms"])
    a[2] += float(row["gflop"])
    m = re.match(r"vd_gn3_(fwd|bwd) px=(\d+) C=(\d+)( \+d?res)?", row["op"])
    if m:  # compulsory traffic: forward x (+ res) in, y out; backward dy, x (+ dres) in, dx out (fp16)
        tensors = (2 if m.group(1) == "fwd" else 3) + (1 if m.group(4) else 0)
        gn3_bytes += tensors * int(m.group(2)) * int(m.group(3)) * 2
        gn3_ms += float(row["ms"])
with open("gpurun_out/vdiff_ops.csv", "w") as f:
    f.write("op,count_per_iter,us_per_iter,us_each,tflops\n")
    for k, (n, t_ms, gf) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        f.write(f"{k},{n},{t_ms * 1e3:.1f},{t_ms / n * 1e3:.1f},{gf / t_ms if gf else 0:.0f}\n")
lib, n = eng.lib, ctypes.c_int()
eng._check(lib.pxr_test_allocations(eng.h, None, None, 0, ctypes.byref(n)), "pxr_test_allocations")
sizes = (ctypes.c_longlong * n.value)()
eng._check(lib.pxr_test_allocations(eng.h, None, sizes, n.value, ctypes.byref(n)), "pxr_test_allocations")
try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as exc:  # the measurement stands without it, but says so
    smi = f"unavailable ({exc})"
print(json.dumps({"workload": f"vdiff cc12m_1 canvas {canvas_w}x{canvas_h} (U-Net {gen_w}x{gen_h}), ViT-B/16, cutn=64",
                  "gpu": smi, "n_gpus": 1,
                  "iters_per_sec": 1e3 / ms, "ms_per_step": ms, "steps": steps_n, "finite_z": bool(torch.isfinite(z).all()),
                  "gemm_family_ms": prof["gemm_ms"], "other_ms": prof["other_ms"],
                  "gemm_family_tflops": prof["gemm_flops"] / (prof["gemm_ms"] * 1e-3) / 1e12,
                  "device_alloc_mib": sum(sizes) / 2 ** 20,
                  "gn3_ms_per_iter": gn3_ms, "gn3_gbytes_per_s": gn3_bytes / (gn3_ms * 1e-3) / 1e9 if gn3_ms else None}))
