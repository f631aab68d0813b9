"""The VQGAN drawer at BASELINE config 2's shape (256 x 256, ViT-B/16, cutn 64) with 16384, 8192 and 1024 codes, and the
time of one GumbelVQ encode (openimages_f16_8192's shape) -- informational; bench.py measures the 16384-code default.

    python tools/bench_vqgan_models.py [steps] [rounds]

Seeded random weights, engine-drawn cutout parameters.  Each model is timed with CUDA events on the engine stream over
`steps` fused iterations, `rounds` times, the models alternating within each round; the median round is reported.  The
encode is timed by the host clock around pxr_vqgan_encode_gumbel, which ends in a device synchronise.  The card's name
and power limit are read in the same run and printed with the numbers."""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

steps_n = int(sys.argv[1]) if len(sys.argv) > 1 else 20
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
warm = 5
CLIP = E.CLIP_ARCH["ViT-B/16"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q)


def build(n_embed, gumbel=False, with_encoder=False):
    cfg = dict(E.VQGAN_F16_16384, n_embed=n_embed)
    sd = S.vqgan_state_dict(cfg, 0, with_encoder=with_encoder, gumbel=gumbel)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(256, 256), vqgan=E.vqgan_config(sd), cutn=64, clip=[CLIP], seed=0)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(CLIP, 1))
    eng.finalize()
    pr = S.prompts(CLIP["out_dim"], (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z = S.z0_vqgan(sd["quantize.embed.weight" if gumbel else "quantize.embedding.weight"], (16, 16), 3).cuda().contiguous()
    return eng, z


def time_steps(eng, z, it0):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for it in range(it0, it0 + steps_n):
        eng.iterate(z, 0.1, it)
    e1.record(ext)
    eng.sync()
    return e0.elapsed_time(e1) / steps_n


models = {n: build(n) for n in (16384, 8192, 1024)}
for eng, z in models.values():
    for it in range(warm):
        eng.iterate(z, 0.1, it)
    eng.sync()
ms = {n: [] for n in models}
for r in range(rounds):
    for n, (eng, z) in models.items():
        ms[n].append(time_steps(eng, z, warm + r * steps_n))
for eng, _ in models.values():
    eng.close()

eng, _ = build(8192, gumbel=True, with_encoder=True)
img = (torch.rand(1, 3, 256, 256, device="cuda") * 2 - 1).contiguous()
enc_ms = []
for i in range(3 + 20):
    noise = -torch.empty(8192, 16, 16, device="cuda").exponential_().log()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.vqgan_encode_gumbel(img, noise)
    if i >= 3:
        enc_ms.append((time.perf_counter() - t0) * 1e3)
eng.close()

out = dict(workload="vqgan 256x256, ViT-B/16, cutn=64 (BASELINE config 2's shape), seeded weights", card=card(),
           steps_per_round=steps_n, rounds=rounds,
           it_per_sec={str(n): 1e3 / statistics.median(v) for n, v in ms.items()},
           ms_per_step_rounds={str(n): v for n, v in ms.items()},
           gumbel_encode_8192_ms_median=statistics.median(enc_ms), gumbel_encode_8192_ms_min=min(enc_ms))
print(json.dumps(out))
