"""The 192- / 256-column GEMM kernel (gemm_wide_kernel) against the 128-column one on the same inputs.

A requested block_n of 192 or 256 runs in the 384-thread kernel when the plan allows it (fp16, A K-major and
unbatched, one of the fp16 tensor-map epilogues); 128 runs in the 288-thread kernel.  Both accumulate every output in
the same k order and share the per-element epilogue arithmetic, so their outputs (and the saved pre-activation) must
agree bit for bit.  Rows and columns outside [M, N] inside a wider row pitch must stay untouched, two runs must give the
same bits, and both are also held against torch fp32 at the tolerances of test_gemm_gpu.py, so that a mistake the two
kernels share is caught too."""
import pytest
import torch

from gemm_util import run_gemm

pytestmark = pytest.mark.gpu

CANARY = 3.0
PAD_COLS, PAD_ROWS = 64, 3

# (M, N, K): the ViT-B/16 cutn-64 linear layers (M = 64 * 197) forward and dgrad, ViT-L/14's fc1, ragged M
# (591 = 3 * 197, 129, 1), N not a multiple of 192, K = 64 (fewer k-blocks than stages), fewer tiles than SMs.
SHAPES = [(12608, 2304, 768), (12608, 768, 768), (12608, 3072, 768), (12608, 768, 3072), (12608, 768, 2304),
          (3 * 257, 4096, 1024), (591, 768, 768), (129, 1024, 192), (1, 768, 64), (1000, 1024, 64)]

# name -> (act, bias, residual, aux_in, aux_out)
MODES = {
    "f16 bias": (0, True, False, False, False),
    "f16": (0, False, False, False, False),
    "res16 bias": (0, True, True, False, False),
    "res16": (0, False, True, False, False),
    "quickgelu": (1, True, False, False, True),
    "quickgelu bwd": (2, False, False, True, False),
    "gelu": (6, True, False, False, True),
    "gelu bwd": (7, False, False, True, False),
}


def _inputs(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.2).half()
    B = (torch.randn(N, K, device="cuda", generator=g) * (0.05 * (768 / K) ** 0.5)).half()
    bias = torch.randn(N, device="cuda", generator=g)
    ld = N + PAD_COLS
    res = torch.randn(M + PAD_ROWS, ld, device="cuda", generator=g).half()
    u = torch.randn(M + PAD_ROWS, ld, device="cuda", generator=g).half()
    return A, B, bias, res, u


def _run(A, B, M, N, K, bn, b_mn, mode, bias, res, u):
    act, has_bias, has_res, has_in, has_aux = MODES[mode]
    ld = N + PAD_COLS
    out = torch.full((M + PAD_ROWS, ld), CANARY, device="cuda", dtype=torch.half)
    aux = torch.full((M + PAD_ROWS, ld), CANARY, device="cuda", dtype=torch.half) if has_aux else None
    Bop, b_mode, ldb = (B.t().contiguous(), 1, N) if b_mn else (B, 0, K)
    run_gemm(A, Bop, M, N, K, lda=K, b_mode=b_mode, ldb=ldb, block_n=bn, alpha=0.75 if act == 0 else 1.0,
             bias=bias if has_bias else None, act=act, aux_in=u if has_in else None, aux_out=aux,
             res_f16=res if has_res else None, out_f16=out, ldc=ld)
    return out, aux


def _reference(A, B, M, N, mode, bias, res, u):
    act, has_bias, has_res, has_in, _ = MODES[mode]
    x = (A.float() @ B.float().T) * (0.75 if act == 0 else 1.0)
    if has_bias:
        x = x + bias
    if has_res:
        x = x + res[:M, :N].float()
    if act == 1:
        return x * torch.sigmoid(1.702 * x), x
    if act == 6:
        return torch.nn.functional.gelu(x), x
    uf = u[:M, :N].float()
    if act == 2:  # the QuickGELU backward multiplies packed fp16 pairs: the sum is rounded to fp16 first
        s = torch.sigmoid(1.702 * uf)
        return x.half().float() * (s * (1 + 1.702 * uf * (1 - s))), None
    if act == 7:
        phi = 0.5 * torch.erfc(-uf / 2 ** 0.5)
        return x * (phi + uf * torch.exp(-0.5 * uf * uf) / (2 * torch.pi) ** 0.5), None
    return x, None


def _check_ref(out, ref, name):
    err = (out.float() - ref).abs().max().item()
    mag = ref.abs().max().item()
    assert err <= 3e-3 * max(mag, 1.0), f"{name}: err {err} vs ref max {mag}"


def _check_canaries(t, M, N, name):
    assert (t[:M, N:] == CANARY).all(), f"{name}: columns past N written"
    assert (t[M:] == CANARY).all(), f"{name}: rows past M written"


@pytest.mark.parametrize("bn", [192, 256])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_wide_matches_128(M, N, K, bn):
    A, B, bias, res, u = _inputs(M, N, K, seed=M + 7 * N + 13 * K + bn)
    for b_mn in (False, True):
        for mode in MODES:
            name = f"{mode} B{'mn' if b_mn else 'k'} bn={bn} M={M} N={N} K={K}"
            o_w, a_w = _run(A, B, M, N, K, bn, b_mn, mode, bias, res, u)
            o_w2, a_w2 = _run(A, B, M, N, K, bn, b_mn, mode, bias, res, u)
            o_n, a_n = _run(A, B, M, N, K, 128, b_mn, mode, bias, res, u)
            assert torch.equal(o_w, o_w2), f"{name}: two runs differ"
            assert torch.equal(o_w, o_n), f"{name}: {bn}-wide output differs from 128-wide " \
                f"(max {(o_w.float() - o_n.float()).abs().max().item():.3e})"
            _check_canaries(o_w, M, N, name)
            if a_w is not None:
                assert torch.equal(a_w, a_w2) and torch.equal(a_w, a_n), f"{name}: saved pre-activation differs"
                _check_canaries(a_w, M, N, name + " aux")
            ref, pre = _reference(A, B, M, N, mode, bias, res, u)
            _check_ref(o_w[:M, :N], ref, name)
            if pre is not None:
                _check_ref(a_w[:M, :N], pre, name + " aux")


def test_wide_residual_in_place():
    """out_f16 == res_f16, as the fp16 residual stream runs the out_proj / fc2 GEMMs."""
    M, N, K = 12608, 768, 3072
    A, B, bias, res, _ = _inputs(M, N, K, seed=3)
    outs = []
    for bn in (256, 128):
        r = res.clone()
        run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, bias=bias, res_f16=r, out_f16=r, ldc=N + PAD_COLS)
        outs.append(r)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0][:, N:], res[:, N:]) and torch.equal(outs[0][M:], res[M:])
    _check_ref(outs[0][:M, :N], A.float() @ B.float().T + bias + res[:M, :N].float(), "res16 in place")
