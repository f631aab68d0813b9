"""Cost of the auxiliary-loss options (SmoothnessLoss pre-blur and edge_order, EdgeLoss target / mask images) at
config 2 (VQGAN 256 x 256, cutn 64, ViT-B/16, seeded synthetic weights), in one call on one GPU:

  * per kernel of each case, the median over `steps` iterations of its device time per iteration (torch.profiler with
    CUDA activities around pxr_iterate), with the bytes it moves per iteration (from the shapes) and the rate that makes;
  * milliseconds per pxr_iterate with the case and without any auxiliary loss, alternating (CUDA events);
  * the GPU's name, power limit and SM clocks.
Prints one JSON line; writes nothing.

    python tools/bench_aux_loss_options.py [steps] [rounds]
"""
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_slip import gpu_info  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import losses as L  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

CUTN, SIDE, CS = 64, 256, 224
ARCH = E.CLIP_ARCH["ViT-B/16"]
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
KERNELS = ("blur_axis_kernel", "blur_axis_adjoint_kernel", "smooth_sharp_kernel", "smooth_grad_kernel", "edge_kernel",
           "aux_final_kernel")


def smooth_args(k, order):
    return types.SimpleNamespace(smoothness_weight=1.0, smoothness_type="default", smoothness_gaussian_kernel=k,
                                 smoothness_gaussian_std=2.0, smoothness_spacing=1, smoothness_edge_order=order)


def smooth_bytes(n):
    """Bytes per iteration and kernel, fp32, each element read or written once (the stencils' neighbour reads are
    cache hits)."""
    P, c2 = 3 * CUTN, CS - (n - 1 if n else 0)
    big, mid, small = 4 * P * CS * CS, 4 * P * CS * c2, 4 * P * c2 * c2
    A = 4 * (CUTN * c2 + 2) * c2
    b = {"smooth_sharp_kernel": small + A, "smooth_grad_kernel": small + A + (small if n else 2 * small)}
    if n:
        b["blur_axis_kernel"] = (big + mid) + (mid + small)
        b["blur_axis_adjoint_kernel"] = (small + mid) + (mid + 2 * big)  # the last pass adds into g_batch
    return b


def edge_bytes(mode):
    hw = 4 * SIDE * SIDE
    return {"edge_kernel": 3 * hw * 3 + (3 * hw if mode & 1 else 0) + (hw if mode & 2 else 0)}


def kernel_times(eng, z, steps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            eng.iterate(z, 0.1, 1000 + i)
        eng.sync()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in KERNELS:
            if k + "(" in ev.name or ev.name.endswith(k) or ("::" + k + "<") in ev.name:
                per.setdefault(k, []).append((ev.time_range.start, ev.device_time))
    out = {}
    for k, v in per.items():
        v.sort()
        d = np.array([t for _, t in v], dtype=np.float64)
        if d.size % steps:
            continue
        out[k] = float(np.median(d.reshape(steps, -1).sum(1)))  # microseconds per iteration
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


def clocks():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        sm, smax, mem = (float(v) for v in q.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": sm, "sm_clock_max_mhz": smax, "mem_clock_mhz": mem}
    except Exception as e:
        return {"clocks": f"unavailable ({type(e).__name__})"}


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    res = dict(gpu_info(), steps=steps, rounds=rounds, workload=f"VQGAN {SIDE}x{SIDE}, cutn {CUTN}, ViT-B/16")
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE), cutn=CUTN, clip=[ARCH], seed=0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(ARCH, 1))
    eng.finalize()
    pr = S.prompts(ARCH["out_dim"], (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z0 = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3).cuda().contiguous()
    session = types.SimpleNamespace(engine=eng)

    def edge(img, mask):
        el = L.EdgeLoss(device="cuda")
        a = types.SimpleNamespace(edge_thickness=5, edge_margins=None, edge_color="white", edge_color_weight=0.1,
                                  global_color_weight=0.05, edge_input_image=os.path.join(GOLDEN, "edge_target.png") if img else "",
                                  edge_mask_image=os.path.join(GOLDEN, "edge_mask.png") if mask else "")
        return el, el.parse_settings(a)

    cases = {}
    for k in (0, 5, 15, 31):
        for order in ((1, 2) if k == 0 else (1,)):
            cases[f"smooth_k{k}_order{order}"] = (L.SmoothnessLoss(device="cuda"), smooth_args(k, order),
                                                  smooth_bytes(len(range(k)) if k else 0))
    cases["edge_colour"] = edge(False, False) + (edge_bytes(0),)
    cases["edge_image_mask"] = edge(True, True) + (edge_bytes(3),)

    out = {}
    for name, (loss, args, nbytes) in cases.items():
        eng.clear_aux_losses()
        loss.attach(session, args, 1.0)
        z = z0.clone()
        time_iterations(eng, z, 0, 3)
        kt = kernel_times(eng, z0.clone(), steps)
        ms_with, ms_without = [], []
        for r in range(rounds):
            eng.clear_aux_losses()
            ms_without.append(time_iterations(eng, z0.clone(), 0, steps))
            loss.attach(session, args, 1.0)
            ms_with.append(time_iterations(eng, z0.clone(), 0, steps))
        eng.clear_aux_losses()
        out[name] = {"kernels_us_per_iter": kt,
                     "bytes_per_iter": nbytes,
                     "gb_per_s": {k: nbytes[k] / (kt[k] * 1e-6) / 1e9 for k in nbytes if kt.get(k)},
                     "ms_per_iter_with": float(np.median(ms_with)), "ms_per_iter_without": float(np.median(ms_without))}
    res["cases"] = out
    res.update(clocks())
    res["power_limit_read_after"] = gpu_info()["power_limit_w"]
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
