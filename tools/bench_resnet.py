"""CLIP ResNet perceptor cost on the engine, in one call on one GPU, with seeded synthetic weights:

  * iterations per second of pxr_iterate (CUDA events around `steps` iterations after a warm-up) for
      rn50       VQGAN 256^2, cutn 64, RN50 (in place of ViT-B/16)
      better     VQGAN 256^2, cutn 64, RN50 + ViT-B/32 + ViT-B/16 (quality="better"'s perceptors)
      rn50x4     VQGAN 256^2, cutn 64, RN50x4 alone at cut 288;
  * the per-op kernel-time split of one profiled iteration (pxr_profile_iteration's CUDA events per op), summed by op kind;
  * the towers' conv / GEMM throughput: a session with the pixel drawer (no GEMM of its own) profiles one iteration, and
    the algorithmic FLOPs of the forward and the data backward (2 x synthetic.resnet_fwd_flops per cutout) over the
    kernel time of its GEMM / conv ops give TFLOP/s;
  * device memory in use by each session (cudaMemGetInfo before the engine is built and after it has iterated);
  * the GPU's name and power limit.
Prints one JSON line; writes nothing outside a temporary directory.

    python tools/bench_resnet.py [steps]
"""
import csv
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

SIDE, CUTN = 256, 64
CONFIGS = {
    "rn50": (["RN50"], 224),
    "better": (["RN50", "ViT-B/32", "ViT-B/16"], 224),
    "rn50x4": (["RN50x4"], 288),
}


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        pl, clk = q.stdout.strip().splitlines()[0].split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception as e:  # the name alone still identifies the card
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def used_bytes():
    free, total = torch.cuda.mem_get_info()
    return total - free


def arch_of(name):
    return E.RESNET_ARCH.get(name) or E.CLIP_ARCH[name]


def build(models, cs, drawer, vq_sd):
    archs = [arch_of(m) for m in models]
    kw = dict(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE)) if drawer == "vqgan" else \
        dict(drawer=E.DRAWER_PIXEL, image_hw=(SIDE, SIDE), grid=(32, 32))
    eng = E.B200Engine(cutn=CUTN, cut_size=cs, clip=archs, seed=0, **kw)
    if drawer == "vqgan":
        eng.load_module(E.MOD_VQGAN, vq_sd)
    for i, (m, a) in enumerate(zip(models, archs)):
        sd = S.clip_resnet_state_dict(a, 1 + i) if m in E.RESNET_ARCH else S.clip_state_dict(a, 1 + i)
        eng.load_module(E.MOD_CLIP0 + i, sd)
    eng.finalize()
    for i, a in enumerate(archs):
        pr = S.prompts(a["out_dim"], (1.0, 0.1), 2 + i)
        eng.set_prompts(i, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    if drawer == "vqgan":
        z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3)
    else:
        z = torch.rand(eng.z_shape, generator=torch.Generator().manual_seed(3))
    return eng, z.cuda().contiguous()


def time_steps(eng, z, it0, steps):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(it0, it0 + steps):
        eng.iterate(z, 0.2, i)
    e1.record(ext)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def profile_rows(eng, z, it):
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ops.csv")
        os.environ["PXR_PROFILE_DUMP"] = path
        try:
            eng.profile_iteration(z, 0.2, it)
        finally:
            del os.environ["PXR_PROFILE_DUMP"]
        return list(csv.DictReader(open(path)))


def kind(op):
    return op.split(" ")[0].split("+")[0]


def split(rows):
    ms = defaultdict(float)
    for r in rows:
        ms[kind(r["op"])] += float(r["ms"])
    return {k: round(v, 3) for k, v in sorted(ms.items(), key=lambda kv: -kv[1])}


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    res = dict(workload=f"VQGAN {SIDE}^2 drawer, cutn {CUTN}, synthetic weights", **gpu_info())
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    for name, (models, cs) in CONFIGS.items():
        torch.cuda.synchronize()
        base = used_bytes()
        eng, z = build(models, cs, "vqgan", vq_sd)
        try:
            time_steps(eng, z, 0, 3)
            s = time_steps(eng, z, 3, steps) / steps
            mem = used_bytes() - base
            rows = profile_rows(eng, z, 3 + steps)
        finally:
            eng.close()
        res[name] = dict(perceptors=models, cut=cs, it_per_s=round(1.0 / s, 2), engine_memory_gib=round(mem / 2 ** 30, 2),
                         kernel_ms_by_op=split(rows), kernel_ms_total=round(sum(float(r["ms"]) for r in rows), 2))
    # the towers alone (pixel drawer: its ops are row kernels, every GEMM / conv of the iteration is the tower's)
    for name in ("RN50", "RN50x4"):
        a = E.RESNET_ARCH[name]
        torch.cuda.synchronize()
        base = used_bytes()
        eng, z = build([name], a["image_res"], "pixel", None)
        try:
            time_steps(eng, z, 0, 3)
            rows = profile_rows(eng, z, 3)
            mem = used_bytes() - base
        finally:
            eng.close()
        gemm = [r for r in rows if kind(r["op"]) in ("gemm", "conv3x3", "conv1x1")]
        g_ms = sum(float(r["ms"]) for r in gemm)
        fl = 2.0 * S.resnet_fwd_flops(a) * CUTN
        conv3 = [r for r in gemm if kind(r["op"]) == "conv3x3"]
        c3_ms = sum(float(r["ms"]) for r in conv3)
        c3_fl = sum(float(r["gflop"]) for r in conv3) * 1e9  # padded-channel FLOPs the launches execute
        res[f"{name}_tower_alone"] = dict(
            gemm_conv_ms=round(g_ms, 3), algorithmic_gflop=round(fl / 1e9, 1),
            tflops_algorithmic=round(fl / g_ms / 1e9, 1), conv3x3_ms=round(c3_ms, 3),
            conv3x3_tflops_executed=round(c3_fl / c3_ms / 1e9, 1) if c3_ms else None,
            row_kernel_ms=round(sum(float(r["ms"]) for r in rows) - g_ms, 3), engine_memory_gib=round(mem / 2 ** 30, 2),
            slowest_ops=[(r["op"], float(r["ms"])) for r in sorted(gemm, key=lambda r: -float(r["ms"]))[:6]])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
