"""Cost of the optimiser update rules (pxr_set_optimizer), in one call on one GPU:

  * microseconds per pxr_step launch (the fused update + clip_z kernel alone, CUDA events over `launches` launches on
    the engine's stream) for every rule, at the 1 x 256 x 16 x 16 latent of a 256 x 256 VQGAN canvas and at a
    3 x 256 x 256 vdiff x, with the bytes each launch moves and the rate that makes;
  * iterations per second of pxr_iterate at a 256 x 256 VQGAN canvas, cutn 64, ViT-B/16, seeded synthetic weights, every
    rule timed in alternating rounds with Adam on the same engine;
  * the GPU's name and power limit.
Prints one JSON line; writes nothing.

    python tools/bench_optimisers.py [launches] [steps] [rounds]
"""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_slip import gpu_info  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

CUTN, SIDE = 64, 256
ARCH = E.CLIP_ARCH["ViT-B/16"]


def state_arrays(kind):
    return 3 if kind == E.OPT_DIFFGRAD else 2


def step_bytes(kind, n):
    """Bytes one launch reads and writes: z and g read, z written, each state array read and written (Adagrad reads and
    writes only its sum)."""
    arrays = 1 if kind == E.OPT_ADAGRAD else state_arrays(kind)
    return 4 * n * (3 + 2 * arrays)


def time_launches(eng, launches, it0):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(launches):
        rc = eng.lib.pxr_step(eng.h, None, C.c_float(0.01), it0 + i)
        assert rc == 0
    e1.record(ext)
    eng.sync()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches * 1e3


def step_times(eng, n, launches, rounds):
    g = torch.Generator().manual_seed(3)
    eng.set_z_grad(torch.randn(*eng.z_shape, generator=g).cuda().contiguous())
    us = {name: [] for name in E.OPTIMISERS}
    for name, kind in E.OPTIMISERS.items():  # warm every instance
        eng.set_optimizer(kind)
        time_launches(eng, 20, 0)
    for r in range(rounds):
        for name, kind in E.OPTIMISERS.items():
            eng.set_optimizer(kind)
            us[name].append(time_launches(eng, launches, 0))
    out = {}
    for name, kind in E.OPTIMISERS.items():
        med = float(np.median(us[name]))
        out[name] = {"us_per_launch_median": med, "us_min": float(np.min(us[name])), "us_max": float(np.max(us[name])),
                     "bytes": step_bytes(kind, n), "gb_per_s": step_bytes(kind, n) / (med * 1e-6) / 1e9}
    return out


def time_iterations(eng, z, it0, steps):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(it0, it0 + steps):
        eng.iterate(z, 0.1, i)
    e1.record(ext)
    eng.sync()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    launches = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    res = dict(gpu_info(), launches=launches, steps=steps, rounds=rounds)

    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE), cutn=CUTN, clip=[ARCH], seed=0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(ARCH, 1))
    eng.finalize()
    pr = S.prompts(ARCH["out_dim"], (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z0 = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3).cuda().contiguous()
    eng.synth(z0)
    n = z0.numel()
    res["step_vqgan_latent"] = dict(shape=list(z0.shape), rules=step_times(eng, n, launches, rounds))

    # pxr_iterate with every rule, alternating rounds with Adam, each from the same start
    ms = {name: [] for name in E.OPTIMISERS}
    for name, kind in E.OPTIMISERS.items():
        eng.set_optimizer(kind)
        time_iterations(eng, z0.clone(), 0, 3)
    for r in range(rounds):
        for name, kind in E.OPTIMISERS.items():
            eng.set_optimizer(kind)
            z = z0.clone()
            ms[name].append(time_iterations(eng, z, 3 + r * steps, steps))
            assert torch.isfinite(z).all()
    res["iterate"] = dict(workload=f"VQGAN {SIDE}x{SIDE}, cutn {CUTN}, ViT-B/16", rules={
        name: {"iters_per_sec": 1e3 / float(np.median(v)), "ms_per_iter_median": float(np.median(v)),
               "ms_min": float(np.min(v)), "ms_max": float(np.max(v))} for name, v in ms.items()})
    eng.close()

    vd = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(SIDE, SIDE), cutn=8, clip=[ARCH], seed=0)
    vd.load_module(E.MOD_VQGAN, S.vdiff_state_dict(0))
    vd.load_module(E.MOD_CLIP0, S.clip_state_dict(ARCH, 1))
    vd.finalize()
    x = torch.randn(1, 3, SIDE, SIDE, generator=torch.Generator().manual_seed(4)).cuda()
    blob = bytearray(vd.save_state())  # z in through the state blob (version 1: 64-byte header, z, m, v)
    blob[64:64 + 4 * x.numel()] = x.cpu().numpy().tobytes()
    vd.load_state(bytes(blob))
    res["step_vdiff_x"] = dict(shape=list(x.shape), rules=step_times(vd, x.numel(), launches, rounds))
    vd.close()
    res["power_limit_read_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
