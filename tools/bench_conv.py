"""Per-launch time and TFLOP/s of the VQGAN decoder's implicit-GEMM convolutions at the 256^2 and 128^2 levels, forward
(with the decoder's epilogues) and dgrad (the transposed conv: input and output channels swapped, no bias):

  * 288-thread  the plan on the 288-thread kernel (128-column tiles, two-stage ring, staged fp32 epilogue),
  * wide bn=N   the same plan on the 384-thread kernel (gemm_wide_kernel) with N-column tiles,
  * F.conv2d    torch on channels-last fp16 (cuDNN, plain conv with bias, no residual): what this card does at its power
                limit with the vendor library, as a yardstick.

Rounds alternate the variants, each round timing `--reps` back-to-back launches with CUDA events; the median round is
reported.  The GPU name, power limit and SM clock are read in the same run.

    python tools/bench_conv.py [--rounds 5] [--reps 30] [--json out.json]
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
from conv_kernel_util import run_conv_on  # noqa: E402

# (name, H = W, Cin, Cout, ksize, bias, residual)
CONVS = [
    ("256^2 ResBlock conv +bias", 256, 128, 128, 3, True, False),
    ("256^2 ResBlock conv2 +bias+res", 256, 128, 128, 3, True, True),
    ("256^2 conv dgrad", 256, 128, 128, 3, False, False),
    ("128^2 conv 256->128 +bias", 128, 256, 128, 3, True, False),
    ("128^2 conv 128->256 dgrad", 128, 128, 256, 3, False, False),
    ("128^2 upsample conv 256->256 +bias", 128, 256, 256, 3, True, False),
    ("128^2 upsample conv dgrad", 128, 256, 256, 3, False, False),
    ("128^2 nin_shortcut 256->128 +bias", 128, 256, 128, 1, True, False),
    ("128^2 nin_shortcut dgrad 128->256", 128, 128, 256, 1, False, False),
]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


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
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_conv: no CUDA device")
    info = gpu_info()
    print(f"# GPU: {info}")
    torch.manual_seed(0)
    results = []
    for name, S, Cin, Cout, ks, has_bias, has_res in CONVS:
        x = (torch.randn(1, S, S, Cin, device="cuda") * 0.5).half()
        w = (torch.randn(Cout, Cin, ks, ks, device="cuda") * 0.02).half()
        wt = w.permute(2, 3, 0, 1).reshape(ks * ks, Cout, Cin).contiguous()
        bias = torch.randn(Cout, device="cuda") if has_bias else None
        out = torch.empty(1, S, S, Cout, device="cuda", dtype=torch.half)
        res = torch.randn(1, S, S, Cout, device="cuda").half() if has_res else None
        x_cl = x.permute(0, 3, 1, 2)  # NCHW view of NHWC memory: channels-last
        w_cl = w.contiguous(memory_format=torch.channels_last)

        def ours(bn, narrow):
            return lambda r: run_conv_on(x, wt, Cout, Cout, ks, block_n=bn, bias=bias, res_f16=res, out_f16=out,
                                         ldc=Cout, repeat=r, narrow_kernel=narrow)

        def cudnn(r):
            for _ in range(r):
                F.conv2d(x_cl, w_cl, bias.half() if bias is not None else None, padding=ks // 2)

        variants = {"288-thread": ours(128, 1), "wide bn=128": ours(128, 0)}
        if Cout >= 256:
            variants["wide bn=256"] = ours(256, 0)
        variants["F.conv2d"] = cudnn
        for fn in variants.values():
            fn(3)
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                times[k].append(time_reps(fn, args.reps))
        flop = 2.0 * S * S * Cout * Cin * ks * ks
        row = {"conv": name, "H": S, "W": S, "Cin": Cin, "Cout": Cout, "ksize": ks}
        parts = []
        for k, ts in times.items():
            us = statistics.median(ts)
            row[k] = {"us": us, "tflops": flop / us / 1e6}
            parts.append(f"{k} {us:8.1f} us {flop / us / 1e6:6.1f} TF/s")
        results.append(row)
        print(f"{name:36s}: " + " | ".join(parts), flush=True)
    print(f"# GPU (after): {gpu_info()}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "rounds": args.rounds, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
