"""ViT-L/14@336px perceptor cost on the engine, in one call on one GPU:

  * per-layer attention forward + backward at the tower's shape (64 cutouts x 16 heads x 577 tokens): the streaming
    kernels (attn_long.cu) against the batched-GEMM chain (S GEMM, row softmax, PV GEMM and their backward: what
    PXR_FUSED_ATTN=0 builds), from the engine's per-op CUDA-event profile of whole iterations, sessions in alternating
    rounds; TFLOP/s over the algorithmic FLOPs (2 T^2 d per pair forward, 4 T^2 d backward, 2 for multiply-add);
  * the streaming kernels alone through pxr_test_attention_long, CUDA events over repeated calls;
  * iterations per second of pxr_iterate at a 256 x 256 VQGAN canvas, cutn 64, on both paths (alternating rounds);
  * device memory in use by each session (cudaMemGetInfo before the engine is built and after it has iterated: the
    engine allocates every buffer when it is built);
  * whether cutn 128 builds and iterates on the streaming path, and its memory;
  * the GPU's name and power limit.
Seeded synthetic weights.  Prints one JSON line; writes nothing.

    python tools/bench_vit_l336.py [steps] [rounds]
"""
import csv
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from pixray_b200 import _lib  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

ARCH = E.CLIP_ARCH["ViT-L/14@336px"]
SIDE, CUTN = 256, 64
T = (ARCH["image_res"] // ARCH["patch"]) ** 2 + 1
H, L = ARCH["heads"], ARCH["layers"]
PAIR_FLOP = 2.0 * T * T * 64          # one T x T x 64 product, multiply-add = 2
FWD_FLOP, BWD_FLOP = 2 * PAIR_FLOP, 4 * PAIR_FLOP


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


def build(fused, cutn, vq_sd, clip_sd):
    os.environ["PXR_FUSED_ATTN"] = "1" if fused else "0"
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(SIDE, SIDE), cutn=cutn, cut_size=ARCH["image_res"], clip=[ARCH],
                       seed=0)
    eng.load_module(E.MOD_VQGAN, vq_sd)
    eng.load_module(E.MOD_CLIP0, clip_sd)
    eng.finalize()
    pr = S.prompts(ARCH["out_dim"], (1.0, 0.1), 2)
    eng.set_prompts(0, torch.cat([p[0] for p in pr]).numpy(), [p[1] for p in pr], [p[2] for p in pr])
    z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (SIDE // 16, SIDE // 16), 3).cuda().contiguous()
    return eng, z


def time_steps(eng, z, it0, steps):
    ext = torch.cuda.ExternalStream(eng.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(it0, it0 + steps):
        eng.iterate(z, 0.2, i)
    e1.record(ext)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def attention_ms(eng, z, it, fused):
    """Attention milliseconds of one profiled iteration (all layers, forward + backward): the attn_long ops, or the
    chain's head-batched GEMMs (batch = cutn x heads) and the row softmax."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ops.csv")
        os.environ["PXR_PROFILE_DUMP"] = path
        try:
            eng.profile_iteration(z, 0.2, it)
        finally:
            del os.environ["PXR_PROFILE_DUMP"]
        rows = list(csv.DictReader(open(path)))
    fwd = bwd = 0.0
    batch = f"batch={CUTN * H} "
    n_batched = 0
    # the VQGAN decoder's attention blocks use the same row softmax: the tower's are the last L forward ones (the drawer
    # runs first) and the first L backward ones (the tower's backward runs first)
    sm_f = [float(r["ms"]) for r in rows if r["op"].startswith("softmax_forward")]
    sm_b = [float(r["ms"]) for r in rows if r["op"].startswith("softmax_backward")]
    if not fused:
        fwd, bwd = sum(sm_f[-L:]), sum(sm_b[:L])
    for r in rows:
        op, ms = r["op"], float(r["ms"])
        if fused:
            fwd += ms if op.startswith("attn_long_fwd") else 0.0
            bwd += ms if op.startswith("attn_long_bwd") else 0.0
        elif op.startswith("gemm") and batch in op:
            # the forward runs first: its S and PV GEMMs are the first 2 L head-batched GEMMs of the iteration
            if n_batched < 2 * L:
                fwd += ms
            else:
                bwd += ms
            n_batched += 1
    return fwd, bwd


def kernel_alone(reps=20):
    lib = _lib.load()
    B, W = CUTN, 64 * H
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = (torch.randn(B * T, 3 * W, generator=g, device="cuda") * 1.5).half()
    d_o = torch.randn(B * T, W, generator=g, device="cuda").half()
    o = torch.empty(B * T, W, dtype=torch.half, device="cuda")
    lse = torch.empty(B * H * T, device="cuda")
    gq = torch.empty(B * T, 3 * W, dtype=torch.half, device="cuda")
    err = C.create_string_buffer(256)
    out = {}
    for name, dd in (("fwd", None), ("fwd_bwd", d_o)):
        args = [C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), C.c_void_p(lse.data_ptr()),
                C.c_void_p(dd.data_ptr()) if dd is not None else None, C.c_void_p(gq.data_ptr()), B, T, H, W,
                C.c_float(0.125)]
        assert lib.pxr_test_attention_long(*args, 2, err, 256) == 0, err.value
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        assert lib.pxr_test_attention_long(*args, reps, err, 256) == 0, err.value
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        fl = B * H * (FWD_FLOP + (BWD_FLOP if dd is not None else 0))
        out[name] = dict(ms=round(ms, 3), tflops=round(fl / ms / 1e9, 1))
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    res = dict(config=f"VQGAN {SIDE}^2, ViT-L/14@336px (T={T}, {H} heads, {L} layers), cutn {CUTN}, synthetic weights",
               **gpu_info())
    res["kernels_alone_B64_T577_H16"] = kernel_alone()
    vq_sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0)
    clip_sd = S.clip_state_dict(ARCH, 1)
    paths = {"streaming": True, "chain": False}
    secs = {k: [] for k in paths}
    att = {k: [] for k in paths}
    mem = {}
    it = 0
    for r in range(rounds):
        for name, fused in (paths.items() if r % 2 == 0 else reversed(list(paths.items()))):
            torch.cuda.synchronize()
            base = used_bytes()
            eng, z = build(fused, CUTN, vq_sd, clip_sd)
            try:
                time_steps(eng, z, it, 3)  # warm-up
                it += 3
                secs[name].append(time_steps(eng, z, it, steps) / steps)
                it += steps
                att[name].append(attention_ms(eng, z, it, fused))
                it += 1
                mem[name] = round((used_bytes() - base) / 2 ** 30, 2)
            finally:
                eng.close()
    per_layer = {}
    for name in paths:
        f = min(a[0] for a in att[name]) / L
        b = min(a[1] for a in att[name]) / L
        fl_f, fl_b = CUTN * H * FWD_FLOP, CUTN * H * BWD_FLOP
        per_layer[name] = dict(fwd_ms=round(f, 3), bwd_ms=round(b, 3), fwd_bwd_ms=round(f + b, 3),
                               fwd_tflops=round(fl_f / f / 1e9, 1), bwd_tflops=round(fl_b / b / 1e9, 1),
                               fwd_bwd_tflops=round((fl_f + fl_b) / (f + b) / 1e9, 1))
    res["attention_per_layer_B64_T577_H16"] = per_layer
    res["per_layer_speedup"] = round(per_layer["chain"]["fwd_bwd_ms"] / per_layer["streaming"]["fwd_bwd_ms"], 2)
    res["it_per_s"] = {k: round(1.0 / min(v), 2) for k, v in secs.items()}
    res["it_per_s_all_rounds"] = {k: [round(1.0 / s, 2) for s in v] for k, v in secs.items()}
    res["engine_memory_gib"] = mem
    # cutn 128 on the streaming path
    torch.cuda.synchronize()
    base = used_bytes()
    try:
        eng, z = build(True, 2 * CUTN, vq_sd, clip_sd)
        try:
            time_steps(eng, z, 0, 2)
            s = time_steps(eng, z, 2, max(2, steps // 2)) / max(2, steps // 2)
            res["cutn128_streaming"] = dict(runs=True, it_per_s=round(1.0 / s, 2),
                                            engine_memory_gib=round((used_bytes() - base) / 2 ** 30, 2))
        finally:
            eng.close()
    except E.EngineError as e:
        res["cutn128_streaming"] = dict(runs=False, error=str(e)[:200])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
