"""SLIP perceptor cost on the engine, in one call on one GPU:

  * iterations per second of pxr_iterate at a 256 x 256 VQGAN canvas, cutn 64, with SLIP_VITB16 (timm ViT-B/16: exact
    GELU, patch-embed bias, no ln_pre) against openai-CLIP ViT-B/16, seeded synthetic weights, the two sessions timed in
    alternating rounds (CUDA events on each engine's stream);
  * microseconds per launch of the ViT-B/16 MLP GEMMs of 64 cutouts (M = 64 x 197) with their activation epilogues:
    fc1 forward (bias + activation + pre-activation to aux) and the fc2 dgrad (times the activation's derivative), exact
    GELU against QuickGELU, on the tensor-map epilogue the engine picks, alternating;
  * the GPU's name and power limit.
Prints one JSON line; writes nothing.

    python tools/bench_slip.py [steps] [rounds]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from gemm_util import run_gemm  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

CUTN, SIDE = 64, 256
MODELS = {"SLIP_VITB16": E.SLIP_ARCH["SLIP_VITB16"], "ViT-B/16": E.CLIP_ARCH["ViT-B/16"]}


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # the name alone still identifies the card
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def build(arch, vq_sd):
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE), cutn=CUTN, clip=[arch], seed=0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    slip = arch.get("tower") == E.TOWER_TIMM_VIT
    eng.load_module(E.MOD_CLIP0, S.slip_state_dict(arch, 1) if slip else S.clip_state_dict(arch, 1))
    eng.finalize()
    pr = S.prompts(arch["out_dim"], (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3).cuda().contiguous()
    return eng, z


def time_steps(eng, z, it0, steps):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(it0, it0 + steps):
        eng.iterate(z, 0.1, i)
    e1.record(ext)
    eng.sync()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def iterate_rates(steps, rounds):
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    sessions = {name: build(arch, vq_sd) for name, arch in MODELS.items()}
    for eng, z in sessions.values():  # warm every shape
        time_steps(eng, z, 0, 3)
    ms = {name: [] for name in sessions}
    for r in range(rounds):
        for name, (eng, z) in sessions.items():
            ms[name].append(time_steps(eng, z, 3 + r * steps, steps))
    out = {name: {"iters_per_sec": 1e3 / float(np.median(v)), "ms_per_step_median": float(np.median(v)),
                  "ms_per_step_min": float(np.min(v)), "ms_per_step_max": float(np.max(v))} for name, v in ms.items()}
    for eng, z in sessions.values():
        assert torch.isfinite(z).all()
        eng.close()
    return out


def epilogue_times(reps, rounds):
    g = torch.Generator().manual_seed(9)
    M, W = 64 * 197, 768
    h = torch.randn(M, W, generator=g).mul(0.1).half().cuda()
    gx = torch.randn(M, W, generator=g).mul(0.1).half().cuda()
    w1 = torch.randn(4 * W, W, generator=g).mul(0.05).half().cuda()
    w2 = torch.randn(W, 4 * W, generator=g).mul(0.05).half().cuda()
    b1 = torch.randn(4 * W, generator=g).cuda()
    u = torch.zeros(M, 4 * W, device="cuda", dtype=torch.half)
    o = torch.zeros(M, 4 * W, device="cuda", dtype=torch.half)

    def fc1(act):
        return lambda r: run_gemm(h, w1, M, 4 * W, W, lda=W, ldb=W, block_n=128, bias=b1, act=act, aux_out=u, out_f16=o,
                                  ldc=4 * W, repeat=r)

    def fc2_dgrad(act):
        return lambda r: run_gemm(gx, w2, M, 4 * W, W, lda=W, b_mode=1, ldb=4 * W, block_n=128, act=act, aux_in=u,
                                  out_f16=o, ldc=4 * W, repeat=r)

    cases = {"fc1 fwd GELU": fc1(6), "fc1 fwd QuickGELU": fc1(1), "fc2 dgrad GELU bwd": fc2_dgrad(7),
             "fc2 dgrad QuickGELU bwd": fc2_dgrad(2)}
    us = {k: [] for k in cases}
    for fn in cases.values():
        fn(3)
    for _ in range(rounds):
        for k, fn in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            fn(reps)
            e1.record()
            torch.cuda.synchronize()
            us[k].append(e0.elapsed_time(e1) / reps * 1e3)
    flops = 2.0 * M * 4 * W * W
    return {k: {"us_median": float(np.median(v)), "us_min": float(np.min(v)),
                "tflops_per_s": flops / (float(np.median(v)) * 1e-6) / 1e12} for k, v in us.items()}


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    res = dict(gpu_info(), workload=f"VQGAN {SIDE}x{SIDE}, cutn {CUTN}, one perceptor", steps=steps, rounds=rounds,
               iterate=iterate_rates(steps, rounds), mlp_gemm_M=64 * 197, mlp_gemm_epilogues=epilogue_times(50, rounds))
    res["power_limit_read_after"] = gpu_info()["power_limit_w"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
