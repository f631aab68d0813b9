"""Streaming fused attention (pixray_b200/csrc/attn_long.cu, pxr_test_attention_long) against the float64 restatement
and the per-element error budget of tests/test_attn_gpu.py (imported, not restated): O, lse, dq, dk and dv.

The kernels stream K / V (backward: Q / dO) through shared memory in 64-row tiles, with 128-row query / key blocks per
CTA; the sequence lengths below cross those edges on both sides (241 = past the tile-staging kernel, 256 / 257 = the
vdiff 16^2 level and ViT-L/14, 577 = ViT-L/14@336px = 9 * 64 + 1, 1024 = 16 tiles), and one case runs the full
ViT-L/14@336px layer shape (64 images x 16 heads x 577 tokens), checked on a sample of images."""
import ctypes as C

import pytest
import torch

from pixray_b200 import _lib
from test_attn_gpu import GUARD, SENTINEL, _check, _guarded, _inputs, _peaked, _reference

pytestmark = pytest.mark.gpu


def _run(qkv, d_o, B, T, H, scale, W=None, repeat=1):
    """pxr_test_attention_long on guarded buffers; returns (o, lse, gqkv) views, or raises with the hook's message."""
    lib = _lib.load()
    W = 64 * H if W is None else W
    o_buf = _guarded(B * T, W, torch.half)
    lse_buf = _guarded(B * H * T, 1, torch.float32)
    g_buf = _guarded(B * T, 3 * W, torch.half) if d_o is not None else None
    o, lse = o_buf[GUARD:-GUARD], lse_buf[GUARD:-GUARD, 0]
    gqkv = g_buf[GUARD:-GUARD] if g_buf is not None else None
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_attention_long(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), C.c_void_p(lse.data_ptr()),
                                     C.c_void_p(d_o.data_ptr()) if d_o is not None else None,
                                     C.c_void_p(gqkv.data_ptr()) if gqkv is not None else None, B, T, H, W,
                                     C.c_float(scale), repeat, err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    torch.cuda.synchronize()
    for name, buf in (("o", o_buf), ("lse", lse_buf), ("gqkv", g_buf)):
        if buf is None:
            continue
        assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all(), f"{name}: write outside the tensor"
        assert not torch.isnan(buf[GUARD:-GUARD]).any(), f"{name}: element left unwritten (or NaN)"
    return o, lse, gqkv


def _case(label, qkv, d_o, B, T, H, scale):
    o, lse, gqkv = _run(qkv, d_o, B, T, H, scale)
    ref, mag = _reference(qkv, d_o, B, T, H, scale)
    _check(label, o, lse, gqkv, ref, mag, B, T, H)
    return o, lse, gqkv


@pytest.mark.parametrize("T", [1, 241, 256, 257, 258, 320, 511, 577, 1024])
@pytest.mark.parametrize("B,H", [(1, 1), (2, 3)])
def test_attention_long_matches_float64(T, B, H):
    qkv, d_o = _inputs(B, T, H, 17 * T + 5 * B + H)
    _case(f"long B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("T", [16, 64, 65, 127, 128, 129, 191, 192, 193])
def test_attention_long_block_edges(T):
    """The kernels are not dispatched below 258 tokens, but they cover any T >= 1: the 64-row tile and 128-row block
    edges."""
    qkv, d_o = _inputs(2, T, 2, 3 * T)
    _case(f"long edges B=2 T={T} H=2", qkv, d_o, 2, T, 2, 0.125)


@pytest.mark.parametrize("scale", [1.0, 0.03])
def test_attention_long_any_scale(scale):
    qkv, d_o = _inputs(2, 577, 2, 41)
    _case(f"long B=2 T=577 H=2 scale={scale}", qkv, d_o, 2, 577, 2, scale)


@pytest.mark.parametrize("where", ["first", "last"])
def test_attention_long_row_max_in_first_or_last_key_tile(where):
    """The online softmax meets the row maximum in its first key tile (never rescales) or in the one-key last tile of
    T = 577 (rescales the whole running sum and output at the end)."""
    B, T, H = 2, 577, 2
    qkv, d_o = _peaked(B, T, H, 0 if where == "first" else T - 1, 9)
    _case(f"long row max in the {where} key tile B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


def test_attention_long_class_row_gradient():
    """dO zero except on each image's class row (the class-rows-only last layer): dq of every other row is exactly 0."""
    B, T, H = 3, 577, 2
    qkv, d_o = _inputs(B, T, H, 23)
    d_o.view(B, T, -1)[:, 1:] = 0
    _, _, gqkv = _case(f"long class-row dO B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)
    dq_rest = gqkv.view(B, T, 3 * 64 * H)[:, 1:, :64 * H]
    assert torch.equal(dq_rest, torch.zeros_like(dq_rest))


def test_attention_long_full_vit_l336_layer():
    """The ViT-L/14@336px layer shape at cutn 64 (1024 (image, head) pairs, 10 CTAs each way per pair): every element
    written, and images 0, 37 and 63 (all heads) within the float64 budget."""
    B, T, H = 64, 577, 16
    W = 64 * H
    qkv, d_o = _inputs(B, T, H, 2024)
    o, lse, gqkv = _run(qkv, d_o, B, T, H, 0.125)
    for b in (0, 37, 63):
        rows = slice(b * T, (b + 1) * T)
        q1, g1 = qkv[rows], d_o[rows]
        ref, mag = _reference(q1, g1, 1, T, H, 0.125)
        _check(f"long full layer image {b} of B={B} T={T} H={H}", o[rows], lse.view(B, H * T)[b], gqkv[rows], ref, mag,
               1, T, H)
    assert o.shape == (B * T, W)


@pytest.mark.parametrize("B,T,H", [(3, 577, 4), (64, 577, 16), (2, 1024, 2)])
def test_attention_long_is_deterministic(B, T, H):
    """One writer per output element, no atomics: two calls give the same bits, and the forward alone gives the same
    o / lse as the forward of a forward + backward call."""
    qkv, d_o = _inputs(B, T, H, 321 + T)
    o1, l1, g1 = _run(qkv, d_o, B, T, H, 0.125)
    o2, l2, g2 = _run(qkv, d_o, B, T, H, 0.125)
    o3, l3, _ = _run(qkv, None, B, T, H, 0.125)
    assert torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(g1, g2)
    assert torch.equal(o1, o3) and torch.equal(l1, l3)


@pytest.mark.parametrize("H,W", [(2, 64), (4, 512), (3, 190)])
def test_attention_long_refuses_other_head_widths(H, W):
    """Heads of width 32 or 128 (or a width the heads do not divide) are refused with a message, not computed."""
    T = 300
    qkv = torch.zeros(T, 3 * W, dtype=torch.half, device="cuda")
    with pytest.raises(RuntimeError, match="64-wide heads"):
        _run(qkv, torch.zeros(T, W, dtype=torch.half, device="cuda"), 1, T, H, 0.125, W=W)
