"""The CLIP ViT-B/16 cutn=64 GEMM shapes with their pipeline epilogues, one launch each through the pxr_test_gemm hook
-- the target for `ncu --set full -k regex:gemm_tc`.  Prints the launch order."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gemm_util import run_gemm  # noqa: E402

torch.manual_seed(0)
dev = "cuda"
M = 64 * 197


def r16(*s):
    return (torch.randn(*s, device=dev) * 0.1).half()


which = sys.argv[1].split(",") if len(sys.argv) > 1 else None
cases = []


def case(name, fn):
    if which is None or name in which:
        cases.append((name, fn))


A768, A3072 = r16(M, 768), r16(M, 3072)
W_fc1, W_fc2, W_proj = r16(3072, 768), r16(768, 3072), r16(768, 768)
o3072, aux3072 = torch.zeros(M, 3072, device=dev, dtype=torch.half), torch.zeros(M, 3072, device=dev, dtype=torch.half)
o768_32, res32 = torch.zeros(M, 768, device=dev), torch.randn(M, 768, device=dev)
bias3072, bias768 = torch.randn(3072, device=dev), torch.randn(768, device=dev)
qkv = r16(M, 2304)
S = torch.zeros(64 * 12 * 197, 200, device=dev, dtype=torch.half)

case("plain_cg1", lambda: run_gemm(A768, W_fc1, M, 3072, 768, lda=768, ldb=768, block_n=256, out_f16=o3072, ldc=3072, cta_group=1))
case("plain_cg2", lambda: run_gemm(A768, W_fc1, M, 3072, 768, lda=768, ldb=768, block_n=256, out_f16=o3072, ldc=3072, cta_group=2))
case("fc1_gelu", lambda: run_gemm(A768, W_fc1, M, 3072, 768, lda=768, ldb=768, block_n=192, bias=bias3072, act=1,
                                  aux_out=aux3072, out_f16=o3072, ldc=3072, cta_group=1))
case("fc2_dgrad_gelubwd", lambda: run_gemm(A768, W_fc2, M, 3072, 768, lda=768, b_mode=1, ldb=3072, block_n=192, act=2,
                                           aux_in=aux3072, out_f16=o3072, ldc=3072, cta_group=1))
case("fc2_res32", lambda: run_gemm(A3072, W_fc2, M, 768, 3072, lda=3072, ldb=3072, block_n=192, bias=bias768, res_f32=res32,
                                   out_f32=o768_32, ldc=768, cta_group=1))
case("proj_res32", lambda: run_gemm(A768, W_proj, M, 768, 768, lda=768, ldb=768, block_n=192, bias=bias768, res_f32=res32,
                                    out_f32=o768_32, ldc=768, cta_group=1))
case("scores", lambda: run_gemm(qkv, qkv[:, 768:], 197, 197, 64, lda=2304, ldb=2304, nb0=12, nb1=64, a_bs=(64, 197 * 2304),
                                b_bs=(64, 197 * 2304), b_batched=1, block_n=208, alpha=0.125, out_f16=S, ldc=200,
                                c_bs=(197 * 200, 12 * 197 * 200), cta_group=1))
for name, fn in cases:
    fn()
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    print(f"{name}: {e0.elapsed_time(e1) * 1e3:.1f} us (3 launches each)")
