"""Helpers to drive the pxr_test_gemm / pxr_test_conv hooks from torch tensors (test infrastructure)."""
import ctypes as C

import torch

from pixray_b200 import _lib


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def run_gemm(A, B, M, N, K, *, a_mode=0, b_mode=0, lda=None, ldb=None, a_mn=None, a_k=None, b_mn=None, b_k=None,
             nb0=1, nb1=1, a_bs=(0, 0), b_bs=(0, 0), b_batched=0, block_n=128, fmt=0, alpha=1.0, bias=None,
             bias_per_row=0, act=0, aux_in=None, aux_out=None, res_f32=None, res_f16=None, out_f32=None, out_f16=None,
             ldc=None, c_bs=(0, 0), repeat=1, cta_group=0, tma_epi=0, k_splits=0):
    lib = _lib.load()
    d = _lib.TestGemmDesc()
    d.k_splits = k_splits
    d.cta_group = cta_group
    d.tma_epi = tma_epi
    d.a, d.a_mode = _ptr(A), a_mode
    d.lda = lda
    d.a_mn_extent = a_mn if a_mn is not None else M
    d.a_k_extent = a_k if a_k is not None else K
    d.a_bs0, d.a_bs1 = a_bs
    d.b, d.b_mode, d.b_batched = _ptr(B), b_mode, b_batched
    d.ldb = ldb
    d.b_mn_extent = b_mn if b_mn is not None else N
    d.b_k_extent = b_k if b_k is not None else K
    d.b_bs0, d.b_bs1 = b_bs
    d.nb0, d.nb1 = nb0, nb1
    d.M, d.N, d.K, d.block_n, d.fmt = M, N, K, block_n, fmt
    d.alpha = alpha
    d.bias, d.bias_per_row, d.act = _ptr(bias), bias_per_row, act
    d.aux_in, d.aux_out = _ptr(aux_in), _ptr(aux_out)
    d.res_f32, d.res_f16 = _ptr(res_f32), _ptr(res_f16)
    d.out_f32, d.out_f16 = _ptr(out_f32), _ptr(out_f16)
    d.ldc = ldc
    d.c_bs0, d.c_bs1 = c_bs
    d.stream = None
    d.repeat = repeat
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_gemm(C.byref(d), err, 512)
    if rc != 0:
        raise RuntimeError(f"pxr_test_gemm rc={rc}: {err.value.decode()}")
    torch.cuda.synchronize()


def run_conv(x_nhwc, wt, n_out, cout_pad, ksize, *, block_n=128, fmt=0, bias=None, out_f32=None, out_f16=None,
             res_f16=None, res_f32=None, ldc=None, alpha=1.0, repeat=1, cta_group=0, tma_epi=0, k_splits=0):
    lib = _lib.load()
    Bn, H, W, Cin = x_nhwc.shape
    d = _lib.TestGemmDesc()
    d.k_splits = k_splits
    d.a, d.lda = _ptr(x_nhwc), x_nhwc.stride(2)
    d.b = _ptr(wt)
    d.N, d.block_n, d.fmt = n_out, block_n, fmt
    d.alpha = alpha
    d.bias = _ptr(bias)
    d.res_f32, d.res_f16 = _ptr(res_f32), _ptr(res_f16)
    d.out_f32, d.out_f16 = _ptr(out_f32), _ptr(out_f16)
    d.ldc = ldc
    d.repeat = repeat
    d.cta_group = cta_group
    d.tma_epi = tma_epi
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_conv(C.byref(d), Bn, H, W, Cin, cout_pad, ksize, err, 512)
    if rc != 0:
        raise RuntimeError(f"pxr_test_conv rc={rc}: {err.value.decode()}")
    torch.cuda.synchronize()
