"""The wgmma attention backward (attn_bwd_wg, pixray_b200/csrc/attn_wg.cu) against the float64 restatement and the
per-element budgets of test_attn_gpu.py (c = 4, u = 2^-11, the TINY floor), through pxr_test_attention_bwd_select:
every tile edge the kernel meets up to T = 208, the hard-input cases, determinism, agreement with attn_bwd_kernel and the
rule that picks the kernel (not causal, at least one (image, head) pair per SM, T <= 208)."""
import ctypes as C
import math

import pytest
import torch

from pixray_b200 import _lib
from test_attn_gpu import C_BUDGET, FLOOR, GUARD, SENTINEL, U, _check, _guarded, _inputs, _reference, _split

pytestmark = pytest.mark.gpu

AUTO, MMA, WG = 0, 1, 2


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(qkv, d_o, B, T, H, scale, sel):
    """Forward, then the backward on kernel `sel`; returns o, lse, gqkv and the kernel the plan took."""
    lib = _lib.load()
    W = 64 * H
    o_buf, lse_buf, g_buf = _guarded(B * T, W, torch.half), _guarded(B * H * T, 1, torch.float32), _guarded(B * T, 3 * W, torch.half)
    o, lse, gqkv = o_buf[GUARD:-GUARD], lse_buf[GUARD:-GUARD, 0], g_buf[GUARD:-GUARD]
    err, used = C.create_string_buffer(512), C.c_int(-1)
    rc = lib.pxr_test_attention_bwd_select(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), C.c_void_p(lse.data_ptr()),
                                           C.c_void_p(d_o.data_ptr()), C.c_void_p(gqkv.data_ptr()), B, T, H, W,
                                           C.c_float(scale), sel, 1, C.byref(used), err, 512)
    assert rc == 0, err.value.decode()
    torch.cuda.synchronize()
    for name, buf in (("o", o_buf), ("lse", lse_buf), ("gqkv", g_buf)):
        assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all(), f"{name}: write outside the tensor"
        assert not torch.isnan(buf[GUARD:-GUARD]).any(), f"{name}: element left unwritten (or NaN)"
    return o, lse, gqkv, used.value


def _case(label, qkv, d_o, B, T, H, scale, sel=WG):
    o, lse, gqkv, used = _run(qkv, d_o, B, T, H, scale, sel)
    assert used == WG, f"{label}: the plan took backward kernel {used}"
    ref, mag = _reference(qkv, d_o, B, T, H, scale)
    _check(label, o, lse, gqkv, ref, mag, B, T, H)
    return gqkv


@pytest.mark.parametrize("T", [1, 15, 16, 17, 50, 63, 64, 65, 127, 128, 129, 191, 192, 193, 197, 207, 208])
def test_wg_tile_edges(T):
    """64-key tiles, 64-query chunks and their 16-row tails; enough pairs that the engine's own choice is attn_bwd_wg."""
    H = 12
    B = math.ceil(_sms() / H)
    qkv, d_o = _inputs(B, T, H, 17 * T + 3)
    _case(f"wg edges B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125, sel=AUTO)


@pytest.mark.parametrize("g_scale", [4096.0, 2.0 ** -8])
def test_wg_gradient_dynamic_range(g_scale):
    B, T, H = 2, 197, 12
    qkv, d_o = _inputs(B, T, H, 11)
    d_o = (d_o.float() * g_scale).half()
    _case(f"wg dO x {g_scale} B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("T", [50, 197])
def test_wg_near_one_hot_rows(T):
    B, H = 2, 4
    qkv, d_o = _inputs(B, T, H, 5 + T, qkv_std=5.0)
    _case(f"wg near one-hot B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("T", [1, 65, 197])
def test_wg_tied_scores(T):
    B, H = 2, 2
    W = 64 * H
    qkv, d_o = _inputs(B, T, H, 77 + T)
    qkv.view(B, T, 3, W)[:, :, 1] = qkv.view(B, T, 3, W)[:, :1, 1]
    _case(f"wg tied scores B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("B,T,H", [(3, 50, 12), (2, 197, 12), (4, 65, 2)])
def test_wg_class_row_gradient(B, T, H):
    """dO zero except on the class row: dq of every other row is exactly 0."""
    qkv, d_o = _inputs(B, T, H, 3 * T + B)
    d_o.view(B, T, -1)[:, 1:] = 0
    gqkv = _case(f"wg class-row dO B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)
    W = 64 * H
    dq_rest = gqkv.view(B, T, 3 * W)[:, 1:, :W]
    assert torch.equal(dq_rest, torch.zeros_like(dq_rest))


def test_wg_is_deterministic():
    H, T = 12, 197
    B = math.ceil(_sms() / H)
    qkv, d_o = _inputs(B, T, H, 123 + T)
    g1 = _run(qkv, d_o, B, T, H, 0.125, WG)[2]
    g2 = _run(qkv, d_o, B, T, H, 0.125, WG)[2]
    assert torch.equal(g1, g2)


@pytest.mark.parametrize("B,T,H", [(2, 197, 12), (3, 65, 4), (2, 208, 2)])
def test_wg_agrees_with_mma_kernel(B, T, H):
    """Both backward kernels on the same inputs: their difference is within one element budget."""
    qkv, d_o = _inputs(B, T, H, 41 * T + B)
    g_mma = _run(qkv, d_o, B, T, H, 0.125, MMA)[2]
    g_wg = _run(qkv, d_o, B, T, H, 0.125, WG)[2]
    _, mag = _reference(qkv, d_o, B, T, H, 0.125)
    a, b = _split(g_mma.cpu().double(), B, T, H), _split(g_wg.cpu().double(), B, T, H)
    for i, name in enumerate(("dq", "dk", "dv")):
        over = (a[i] - b[i]).abs() > C_BUDGET * U * mag[name] + FLOOR
        assert not over.any(), f"{name}: {int(over.sum())} elements differ by more than the budget"


def test_wg_dispatch():
    """The engine's choice: attn_bwd_wg with at least one pair per SM and T <= 208, attn_bwd_kernel otherwise."""
    H = 12
    few, many = max(1, _sms() // H - 1), math.ceil(_sms() / H)
    for B, T, want in ((many, 197, WG), (many, 208, WG), (many, 209, MMA), (many, 240, MMA), (few, 197, MMA),
                       (few, 50, MMA), (many, 1, WG)):
        qkv, d_o = _inputs(B, T, H, T + B)
        assert _run(qkv, d_o, B, T, H, 0.125, AUTO)[3] == want, f"B={B} T={T} H={H}"
    # forced: the old kernel anywhere, the new one not past its shared-memory budget
    qkv, d_o = _inputs(2, 197, H, 9)
    assert _run(qkv, d_o, 2, 197, H, 0.125, MMA)[3] == MMA
    lib = _lib.load()
    T, W = 209, 64 * H
    qkv, d_o = _inputs(2, T, H, 10)
    o = torch.empty(2 * T, W, dtype=torch.half, device="cuda")
    lse = torch.empty(2 * H * T, device="cuda")
    g = torch.empty(2 * T, 3 * W, dtype=torch.half, device="cuda")
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_attention_bwd_select(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), C.c_void_p(lse.data_ptr()),
                                           C.c_void_p(d_o.data_ptr()), C.c_void_p(g.data_ptr()), 2, T, H, W, C.c_float(0.125),
                                           WG, 1, None, err, 512)
    assert rc != 0 and b"T <= 208" in err.value
