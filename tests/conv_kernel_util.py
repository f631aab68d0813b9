"""Drive the pxr_test_conv hook on a chosen kernel from torch tensors (test infrastructure).

narrow_kernel = 1 runs the plan on the 288-thread kernel even where the 384-thread one would take it, so that tests and
tools/bench_conv.py can compare the two kernels on one plan.  Epilogue: fp16 output with optional bias and fp16 residual
(the epilogues the 384-thread kernel takes for convolutions)."""
import ctypes as C

import torch

from pixray_b200 import _lib


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def run_conv_on(x_nhwc, wt, n_out, cout_pad, ksize, *, block_n, out_f16, ldc, bias=None, res_f16=None, repeat=1,
                narrow_kernel=0):
    lib = _lib.load()
    Bn, H, W, Cin = x_nhwc.shape
    d = _lib.TestGemmDesc()
    d.a, d.lda = _ptr(x_nhwc), x_nhwc.stride(2)
    d.b = _ptr(wt)
    d.N, d.block_n, d.fmt = n_out, block_n, 0
    d.alpha = 1.0
    d.bias = _ptr(bias)
    d.res_f16 = _ptr(res_f16)
    d.out_f16 = _ptr(out_f16)
    d.ldc = ldc
    d.repeat = repeat
    d.narrow_kernel = narrow_kernel
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_conv(C.byref(d), Bn, H, W, Cin, cout_pad, ksize, err, 512)
    if rc != 0:
        raise RuntimeError(f"pxr_test_conv rc={rc}: {err.value.decode()}")
    torch.cuda.synchronize()
