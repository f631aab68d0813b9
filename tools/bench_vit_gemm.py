"""Per-launch time and TFLOP/s of the eight ViT linear-layer GEMMs per layer (qkv, out_proj, fc1, fc2 forward with their
pipeline epilogues, and their dgrads with an MN-major weight), at the ViT-B/16 cutn-64 and ViT-L/14 cutn-256 shapes:

  * bn=128      the 288-thread kernel with 128-column tiles,
  * bn=192/256  the 384-thread kernel (gemm_wide_kernel),
  * cuBLAS      torch.nn.functional.linear in fp16 on the plain shape (no epilogue): what this card does at its power
                limit with the vendor library, as a yardstick.

Rounds alternate the variants, each round timing `--reps` back-to-back launches with CUDA events; the median round is
reported.  The GPU name, power limit and SM clock are read in the same run.

    python tools/bench_vit_gemm.py [--rounds 5] [--reps 20] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gemm_util import run_gemm  # noqa: E402

TOWERS = [("ViT-B/16 cutn 64", 768, 197, 64), ("ViT-L/14 cutn 256", 1024, 257, 256)]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def layer_gemms(W, M):
    """(name, N, K, B MN-major, epilogue kwargs builder)"""
    def fwd_bias(N):
        return lambda t: dict(bias=t["bias"][:N], out_f16=t["out"])

    def res(N):
        return lambda t: dict(bias=t["bias"][:N], res_f16=t["res"], out_f16=t["res"])

    return [
        ("qkv", 3 * W, W, False, fwd_bias(3 * W)),
        ("out_proj +res", W, W, False, res(W)),
        ("fc1 +gelu", 4 * W, W, False, lambda t: dict(bias=t["bias"][:4 * W], act=1, aux_out=t["aux"], out_f16=t["out"])),
        ("fc2 +res", W, 4 * W, False, res(W)),
        ("fc2 dgrad gelu-bwd", 4 * W, W, True, lambda t: dict(act=2, aux_in=t["aux"], out_f16=t["out"])),
        ("fc1 dgrad +res", W, 4 * W, True, lambda t: dict(res_f16=t["res"], out_f16=t["res"])),
        ("out_proj dgrad", W, W, True, lambda t: dict(out_f16=t["out"])),
        ("qkv dgrad +res", W, 3 * W, True, lambda t: dict(res_f16=t["res"], out_f16=t["res"])),
    ]


def time_reps(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn(reps)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_vit_gemm: no CUDA device")
    info = gpu_info()
    print(f"# GPU: {info}")
    torch.manual_seed(0)
    results = []
    for tower, W, T, cutn in TOWERS:
        M = T * cutn
        buf = {
            "A": (torch.randn(M, 4 * W, device="cuda") * 0.1).half(),
            "B": (torch.randn(4 * W, 4 * W, device="cuda") * 0.02).half(),
            "bias": torch.randn(4 * W, device="cuda"),
            "out": torch.empty(M, 4 * W, device="cuda", dtype=torch.half),
            "aux": (torch.randn(M, 4 * W, device="cuda")).half(),
            "res": torch.randn(M, 4 * W, device="cuda").half(),
        }
        for name, N, K, b_mn, epi in layer_gemms(W, M):
            A = buf["A"][:, :K].contiguous()
            Bw = buf["B"][:N, :K].contiguous()  # [N, K]; the dgrads read it as MN-major [K, N]
            Bop, b_mode, ldb = (Bw.t().contiguous(), 1, N) if b_mn else (Bw, 0, K)
            kw = epi(buf)

            def ours(bn):
                return lambda r: run_gemm(A, Bop, M, N, K, lda=K, b_mode=b_mode, ldb=ldb, block_n=bn, ldc=N, repeat=r, **kw)

            def cublas(r):
                for _ in range(r):
                    F.linear(A, Bw)

            variants = {"bn=128": ours(128), "bn=192": ours(192), "bn=256": ours(256), "cuBLAS": cublas}
            for fn in variants.values():
                fn(3)
            times = {k: [] for k in variants}
            for _ in range(args.rounds):
                for k, fn in variants.items():
                    times[k].append(time_reps(fn, args.reps))
            flop = 2.0 * M * N * K
            row = {"tower": tower, "gemm": name, "M": M, "N": N, "K": K}
            parts = []
            for k, ts in times.items():
                us = statistics.median(ts)
                row[k] = {"us": us, "tflops": flop / us / 1e6}
                parts.append(f"{k} {us:8.1f} us {flop / us / 1e6:6.1f} TF/s")
            results.append(row)
            print(f"{tower:18s} {name:20s} M={M} N={N} K={K}: " + " | ".join(parts), flush=True)
    print(f"# GPU (after): {gpu_info()}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "rounds": args.rounds, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
