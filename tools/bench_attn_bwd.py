"""Time the fused attention backward alone on both kernels (attn_bwd_kernel = mma, attn_bwd_wg = wg) through
pxr_test_attention_bwd_select, at the ViT shapes that dominate: CUDA events around the forward followed by `reps`
backward launches, less the forward alone, in alternating rounds; the median per shape and kernel.

    python tools/bench_attn_bwd.py [rounds] [reps]

Prints us per call, algorithmic TFLOP/s (dP, dQ, dK, dV: 4 T^2 64 2 per pair) and executed TFLOP/s (what each kernel
multiplies: mma recomputes S and dP in both phases over 16-row tiles, wg forms each product once over 64-row tiles), and
the card's name, power limit and SM clock read in the same process.
"""
import ctypes as C
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixray_b200 import _lib  # noqa: E402

SHAPES = [(64, 197, 12), (128, 50, 12), (64, 197, 16)]
KERNELS = (("mma", 1), ("wg", 2))


def executed_flops(kernel, B, T, H):
    r16, r64 = (T + 15) // 16 * 16, (T + 63) // 64 * 64
    mm = 2.0 * 64 * B * H
    if kernel == "mma":  # 7 products over 16-row tiles: S, dP, dV, dK in phase 1; S, dP, dQ in phase 2
        return 7 * mm * r16 * r16
    return mm * (4 * r64 * r16 + r64 * r64)  # S, dP, dV, dK per 64-key tile; dQ per 64-query tile


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    lib = _lib.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    for B, T, H in SHAPES:
        W = 64 * H
        g = torch.Generator(device="cuda").manual_seed(T)
        qkv = (torch.randn(B * T, 3 * W, generator=g, device="cuda") * 1.5).half()
        d_o = torch.randn(B * T, W, generator=g, device="cuda").half()
        o = torch.empty(B * T, W, dtype=torch.half, device="cuda")
        lse = torch.empty(B * H * T, device="cuda")
        gqkv = torch.empty(B * T, 3 * W, dtype=torch.half, device="cuda")
        err = C.create_string_buffer(512)

        def call(sel, n):
            used = C.c_int(0)
            rc = lib.pxr_test_attention_bwd_select(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()),
                                                   C.c_void_p(lse.data_ptr()), C.c_void_p(d_o.data_ptr()),
                                                   C.c_void_p(gqkv.data_ptr()), B, T, H, W, C.c_float(0.125), sel, n,
                                                   C.byref(used), err, 512)
            assert rc == 0 and used.value == sel, err.value.decode()

        def timed(sel, n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            call(sel, n)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3

        for _, sel in KERNELS:  # warm-up: module load, plan, tensor maps
            call(sel, 3)
        times = {name: [] for name, _ in KERNELS}
        for _ in range(rounds):
            for name, sel in KERNELS:
                times[name].append((timed(sel, reps) - timed(sel, 0)) / reps)
        alg = 4 * 2.0 * 64 * T * T * B * H
        for name, _ in KERNELS:
            us = statistics.median(times[name])
            print(f"attn_bwd {name:3s} B={B} T={T} H={H}: {us:7.1f} us per call (spread {min(times[name]):.1f}-"
                  f"{max(times[name]):.1f}), {alg / us / 1e6:6.1f} TFLOP/s algorithmic, "
                  f"{executed_flops(name, B, T, H) / us / 1e6:6.1f} TFLOP/s executed")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")


if __name__ == "__main__":
    main()
