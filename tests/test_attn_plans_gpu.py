"""Every attention the engine plans, replayed against float64 with the engine's own routing, buffers and kernels.

`add_attention` records each call (pxr_test_attention_records): its call site, the path it took -- the fused kernels of
attn_tc.cu (T <= 240), the streaming ones of attn_long.cu (T > 257) or the batched-GEMM chain -- its shape, scale and
tensors, the fused plan's splits and backward kernel, and for the chain the indices of the GEMM records its six GEMMs
made.  These tests build engines from synthetic weights (finalize() plans; nothing runs) and check

- routing: every record follows the rule restated below, the fused backward is attn_bwd_wg exactly when the call has a
  backward, is not causal, has at least one (image, head) pair per SM and T <= 208, and each engine still reaches the
  paths it is here for; a chain record's GEMMs are the chain (operands, batch strides, extents, alpha, output pitch);
- footprint: every tensor a record addresses lies inside one allocation (a shared dP too), and what a backward reads
  from its forward (qkv, lse and O of the fused and streaming paths, qkv and P of the chain) overlaps no tensor of
  another record with a backward, nor what its own backward writes.  go, gqkv and dP shared across layers are intended;
- replay: each distinct record rebuilt on caller tensors at the engine's pointer alignment (the fused and streaming
  plans by pxr_test_attention_plan, which must report the record's splits and backward kernel; the chain from its GEMM
  records through pxr_test_gemm and the row softmax hook), outputs inside SENTINEL guards and NaN-filled, two runs bit
  for bit equal, on the random case and the hard ones of test_attn_gpu.py: near-one-hot rows, the row maximum at the
  last key, and a large dO (x 4096; on the chain the largest power of two up to 4096 that keeps max |dO v^T| below
  2^15, because the chain stores dP in fp16 and 4096 times a unit dO overflows it).

Budgets, per output element, against float64 from the same fp16 inputs (u = 2^-11, c = 4, TINY = 2^-14, |.| products
in float64, P, dP = dO v^T, D = sum_j P_ij dP_ij, dS = P o (dP - D) the float64 values):
  fused and streaming: those of test_attn_gpu.py.
  chain: c E + 2^-24, E the first-order propagation of every fp16 rounding the chain stores and of the GEMMs'
  2^-16 sum |a||b| fp32 accumulation term:
    E_S  = u |S| + 2^-16 scale |q| |k|^T                                      S = scale q k^T, stored fp16
    E_P  = P o (E_S + rowsum(P o E_S)) + u (P + TINY)                         through the softmax, dP = P o (dS - P.dS),
                                                                              and P's own fp16 store
    o    = E_P |v| + 2^-16 P |v| + u |o|
    E_dP = u |dP| + 2^-16 |dO| |v|^T
    E_D  = rowsum(E_P o |dP| + P o E_dP)                                      D is formed from the stored P and dP
    E_dS = E_P o |dP - D| + P o (E_dP + E_D) + u (|dS| + TINY)
    dq   = scale (E_dS |k| + 2^-16 |dS| |k|) + u |dq|        dk = scale (E_dS^T |q| + 2^-16 |dS|^T |q|) + u |dk|
    dv   = E_P^T |dO| + 2^-16 P^T |dO| + u |dv|
  TINY is the absolute 2^-25 = u TINY an fp16 store makes below the smallest normal, where P or dS is an MMA operand.
  Masked keys of the causal softmax are exact zeros and take no part.  The chain has no lse.
Each engine prints its worst err / bound per output; CPU tests show the chain budget accepts a float64 emulation of
the chain with fp16 stores at S, P, dP, dS and the outputs, and rejects a zero pad column in the softmax, a dropped
last key, dk without the scale, dS without its D term and dq from the neighbouring head's K.
"""
import ctypes as C
import math
import os
import re

import pytest
import torch

from pixray_b200 import _lib
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_attn_gpu import C_BUDGET, FLOOR, GUARD, SENTINEL, TINY, U, _inputs, _log, _peaked, _reference, _split
from test_gemm_plans_gpu import (ROOT, SMALL_CLIP, _desc, _p, _signature, _vit, _vqgan, _with_env, aligned, aligned_copy,
                                 allocations, gemm_records)

FUSED, STREAMING, CHAIN = _lib.ATTN_FUSED, _lib.ATTN_STREAMING, _lib.ATTN_CHAIN
MMA, WG = 1, 2  # AttnPlan::bwd: attn_bwd_kernel, attn_bwd_wg
ABS = 2.0 ** -16
OP_K, OP_MN = 0, 1


# ------------------------------------------------------------------------------------------------------- the hooks
def attention_records(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_attention_records(eng.h, None, 0, C.byref(n)), "pxr_test_attention_records")
    recs = (_lib.TestAttnRec * n.value)()
    eng._check(lib.pxr_test_attention_records(eng.h, recs, n.value, C.byref(n)), "pxr_test_attention_records")
    return list(recs)


# ------------------------------------------------------------------------------------------------------- engines
def _vitb16(cutn):
    def make():
        arch = dict(E.CLIP_ARCH["ViT-B/16"], layers=2)
        return _vit(arch, cutn, S.clip_state_dict(arch, 0))
    return make


def _vitb32_text():
    arch = dict(E.CLIP_ARCH["ViT-B/32"], layers=2)
    return _vit(arch, 8, S.clip_state_dict(arch, 0), S.clip_text_state_dict(512, 2, 512, 1))


def _vitl14():
    arch = dict(E.CLIP_ARCH["ViT-L/14"], layers=2)
    return _vit(arch, 8, S.clip_state_dict(arch, 0))


def _vitl14_336():
    arch = dict(E.CLIP_ARCH["ViT-L/14@336px"], layers=2)
    return _vit(arch, 4, S.clip_state_dict(arch, 0))


def _vdiff(hw):
    def make():
        eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=hw, cutn=8, clip=[SMALL_CLIP], seed=0)
        eng.load_module(E.MOD_VQGAN, S.vdiff_state_dict(0, c=128))
        eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
        return eng
    return make


# name: (constructor, environment, the kinds of attention the engine must reach)
ENGINES = {
    "vitb16_cutn64": (_vitb16(64), {}, {"fused197", "bwd_wg"}),
    "vitb32_text": (_vitb32_text, {}, {"fused50", "split", "bwd_mma", "causal_fused77"}),
    "vitb32_text_chain": (_vitb32_text, {"PXR_FUSED_ATTN": "0"}, {"chain50", "causal_chain77"}),
    "vitb16_cutn64_mma": (_vitb16(64), {"PXR_ATTN_BWD": "mma"}, {"fused197", "bwd_mma", "pairs768"}),
    "vitl14": (_vitl14, {}, {"chain257", "heads16"}),
    "vitl14_336": (_vitl14_336, {}, {"stream577"}),
    "vdiff64": (_vdiff((64, 64)), {}, {"fused16", "fused4", "fused1", "one_image"}),
    "vdiff256": (_vdiff((256, 256)), {}, {"chain256", "fused64", "fused16"}),
    # No U-Net reaches the streaming kernels: its sides are powers of two, and at 512^2 (T = 1024 at the 32^2 attention
    # level) its GroupNorm single-kernel path does not cover 512^2 x 128 channels, so the engine refuses to build it.
    "vqgan256": (_vqgan((256, 256)), {}, {"single_chain256_d512"}),
    "vqgan288x432": (_vqgan((288, 432)), {}, {"single_chain486_d512"}),
}
SLOW = {"vqgan288x432"}


def _build(env, make):
    """The engine with every switch cleared but those in env (PXR_ATTN_BWD included, which _with_env does not hold)."""
    old = os.environ.pop("PXR_ATTN_BWD", None)
    try:
        return _with_env(env, make)
    finally:
        if old is not None:
            os.environ["PXR_ATTN_BWD"] = old


class Built:
    def __init__(self, name):
        self.name = name
        make, self.env, self.expect = ENGINES[name]
        self.eng = _build(self.env, make)
        self.recs = attention_records(self.eng)
        self.grecs = gemm_records(self.eng)
        self.allocs = allocations(self.eng)
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.fused_on = self.env.get("PXR_FUSED_ATTN") != "0"
        self.force_mma = self.env.get("PXR_ATTN_BWD") == "mma"

    def alloc_of(self, lo, hi):
        for a, n in self.allocs:
            if a <= lo and hi <= a + n:
                return a, n
        return None

    def close(self):
        self.eng.close()


def _params():
    return [pytest.param(n, marks=[pytest.mark.gpu] + ([pytest.mark.slow] if n in SLOW else [])) for n in ENGINES]


@pytest.fixture(scope="module", params=_params())
def built(request):
    b = Built(request.param)
    yield b
    b.close()


def _name(b, r):
    return f"{b.name}: {r.site.decode()} T={r.T} heads={r.heads} images={r.images}"


# ------------------------------------------------------------------------------------------------------- routing
def expected_path(r, fused_on):
    """add_attention's rule: attn_supported (64-wide heads, T <= 240) -> fused, attn_long_supported past T = 257 ->
    streaming, the chain otherwise (T = 241 .. 257, other head widths, single-head calls, PXR_FUSED_ATTN=0)."""
    heads64 = r.d == 64 and r.W % 64 == 0
    if r.multihead and fused_on and heads64 and 1 <= r.T <= 240:
        return FUSED
    if r.multihead and fused_on and heads64 and r.T > 257:
        return STREAMING
    return CHAIN


def expected_splits(T, pairs, sms):
    """attn_plan_make: a pair's 16-row tiles over up to ceil(SMs / pairs) CTAs, none without a tile."""
    nt = -(-T // 16)
    want = min(nt, max(1, -(-sms // pairs)))
    per = -(-nt // want)
    return -(-nt // per)


def expected_bwd(backward, causal, pairs, T, sms, force_mma):
    return WG if backward and not causal and pairs >= sms and T <= 208 and not force_mma else MMA


def kinds(r):
    k = set()
    if r.path == FUSED:
        k.add(f"{'causal_' if r.causal else ''}fused{r.T}")
        if r.splits > 1:
            k.add("split")
        if r.backward:
            k.add("bwd_wg" if r.bwd == WG else "bwd_mma")
            k.add(f"pairs{r.images * r.heads}")
    elif r.path == STREAMING:
        k.add(f"stream{r.T}")
    else:
        k.add(f"{'causal_' if r.causal else ''}chain{r.T}" if r.multihead else f"single_chain{r.T}_d{r.d}")
    k.add(f"heads{r.heads}")
    if r.images == 1:
        k.add("one_image")
    return k


def chain_gemms(r):
    """The chain as add_attention builds it: (name, A, B, M, N, K, alpha, out, ldc, out batch strides) with operands
    (ptr, mode, ld, mn extent, k extent, batch strides); batches (heads, images) on both operands and the output."""
    W, T, d, ldT, h = r.W, r.T, r.d, r.ldT, r.heads
    qs, os_, ps = (d, T * 3 * W), (d, T * W), (T * ldT, h * T * ldT)
    q, k, v = r.qkv, r.qkv + 2 * W, r.qkv + 4 * W  # byte addresses of the q / k / v thirds
    gq, gk, gv = r.gqkv, (r.gqkv or 0) + 2 * W, (r.gqkv or 0) + 4 * W
    return [
        ("S", (q, OP_K, 3 * W, T, d, qs), (k, OP_K, 3 * W, T, d, qs), T, T, d, r.scale, r.P, ldT, ps),
        ("O", (r.P, OP_K, ldT, T, ldT, ps), (v, OP_MN, 3 * W, d, T, qs), T, d, T, 1.0, r.o, W, os_),
        ("dP", (r.d_o, OP_K, W, T, d, os_), (v, OP_K, 3 * W, T, d, qs), T, T, d, 1.0, r.dP, ldT, ps),
        ("dq", (r.dP, OP_K, ldT, T, ldT, ps), (k, OP_MN, 3 * W, d, T, qs), T, d, T, r.scale, gq, 3 * W, qs),
        ("dk", (r.dP, OP_MN, ldT, T, T, ps), (q, OP_MN, 3 * W, d, T, qs), T, d, T, r.scale, gk, 3 * W, qs),
        ("dv", (r.P, OP_MN, ldT, T, T, ps), (r.d_o, OP_MN, W, d, T, os_), T, d, T, 1.0, gv, 3 * W, qs),
    ]


def check_chain_gemms(b, r):
    name = _name(b, r)
    n = 6 if r.backward else 2
    assert all(i >= 0 for i in r.gemm[:n]) and all(i < 0 for i in r.gemm[n:]), f"{name}: GEMM links {list(r.gemm)}"
    assert len(set(r.gemm[:n])) == n
    for (g, A, Bop, M, N, K, alpha, out, ldc, cbs), i in zip(chain_gemms(r)[:n], r.gemm[:n]):
        gr = b.grecs[i]
        got = dict(A=(gr.a, gr.a_mode, gr.lda, gr.a_mn_extent, gr.a_k_extent, (gr.a_bs0, gr.a_bs1)),
                   B=(gr.b, gr.b_mode, gr.ldb, gr.b_mn_extent, gr.b_k_extent, (gr.b_bs0, gr.b_bs1)),
                   batch=((gr.a_nb0, gr.a_nb1), (gr.b_nb0, gr.b_nb1)), MNK=(gr.M, gr.N, gr.K), alpha=gr.alpha,
                   out=(gr.out_f16, gr.ldc, (gr.c_bs0, gr.c_bs1)),
                   rest=(gr.bias, gr.act, gr.aux_in, gr.aux_out, gr.res_f16, gr.res_f32, gr.out_f32, gr.k_splits > 1))
        want = dict(A=A, B=Bop, batch=((r.heads, r.images),) * 2, MNK=(M, N, K), alpha=alpha, out=(out, ldc, cbs),
                    rest=(None, 0, None, None, None, None, None, False))
        for f in want:
            assert got[f] == want[f], f"{name}: the chain's {g} GEMM (record {i}) has {f} {got[f]}, expected {want[f]}"


def test_routing(built):
    b = built
    assert b.recs, "no attention recorded"
    seen = set()
    for r in b.recs:
        name = _name(b, r)
        assert r.W == r.heads * r.d, name
        want = expected_path(r, b.fused_on)
        assert r.path == want, f"{name}: path {r.path}, the rule gives {want}"
        if r.causal:
            assert r.multihead and not r.backward and r.T <= 240, f"{name}: a causal attention with a backward"
        pairs = r.images * r.heads
        if r.path == FUSED:
            assert r.lse and not r.delta and not r.P and not r.dP and r.gemm[0] < 0, name
            assert r.splits == expected_splits(r.T, pairs, b.sms), f"{name}: {r.splits} splits for {pairs} pairs"
            want_bwd = expected_bwd(bool(r.d_o and r.gqkv), r.causal, pairs, r.T, b.sms, b.force_mma)
            assert r.bwd == want_bwd, f"{name}: backward kernel {r.bwd}, the rule gives {want_bwd} ({pairs} pairs)"
        elif r.path == STREAMING:
            assert r.lse and bool(r.delta) == bool(r.backward) and not r.P and r.gemm[0] < 0, name
            assert (r.splits, r.bwd) == (1, 0), name
        else:
            assert r.P and not r.lse and not r.delta and r.ldT == -(-r.T // 8) * 8, name
            assert bool(r.dP) == bool(r.backward) and (r.dP_shared == 0 or r.backward), name
            check_chain_gemms(b, r)
        seen |= kinds(r)
    print(f"[attn plans] {b.name}: {len(b.recs)} attentions, kinds {sorted(seen)}")
    missing = b.expect - seen
    assert not missing, f"{b.name}: no attention of the kinds {sorted(missing)} any more"


@pytest.mark.gpu
def test_backward_kernel_rule_edges():
    """The plan's own choice at the edges of the attn_bwd_wg rule, on the hook (the engines reach only some of them)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lib = _lib.load()
    for T, pairs, causal, backward in ((208, sms, 0, 1), (209, sms, 0, 1), (208, sms - 1, 0, 1), (16, sms, 0, 1),
                                       (240, 2 * sms, 0, 1), (208, sms, 1, 0), (208, sms, 0, 0)):
        r = _lib.TestAttnRec(path=FUSED, multihead=1, causal=causal, backward=backward, images=pairs, heads=1, T=T, d=64,
                             W=64, scale=0.125)
        qkv = torch.zeros(pairs * T, 192, dtype=torch.half, device="cuda")
        o = torch.empty(pairs * T, 64, dtype=torch.half, device="cuda")
        lse = torch.empty(pairs * T, device="cuda")
        d_o = torch.zeros_like(o) if backward else None
        gqkv = torch.empty_like(qkv) if backward else None
        out2, err = (C.c_int * 2)(), C.create_string_buffer(512)
        rc = lib.pxr_test_attention_plan(C.byref(r), _p(qkv), _p(o), _p(d_o), _p(gqkv), _p(lse), None, 0, out2, err, 512)
        assert rc == 0, err.value.decode()
        want = (expected_splits(T, pairs, sms), expected_bwd(backward, causal, pairs, T, sms, False))
        assert tuple(out2) == want, f"T={T} pairs={pairs} causal={causal}: the plan takes {tuple(out2)}, the rule {want}"


# ------------------------------------------------------------------------------------------------------- footprint
def tensors(r):
    """(name, ptr, bytes) of every tensor the record addresses."""
    B, T, H, W = r.images, r.T, r.heads, r.W
    t = [("qkv", r.qkv, 2 * B * T * 3 * W), ("o", r.o, 2 * B * T * W), ("d_o", r.d_o, 2 * B * T * W),
         ("gqkv", r.gqkv, 2 * B * T * 3 * W), ("lse", r.lse, 4 * B * H * T), ("delta", r.delta, 4 * B * H * T),
         ("P", r.P, 2 * B * H * T * r.ldT), ("dP", r.dP, 2 * B * H * T * r.ldT)]
    return [x for x in t if x[1]]


def saved(r):
    """What the backward reads from its forward."""
    keep = ("qkv", "P") if r.path == CHAIN else ("qkv", "lse", "o")
    return [x for x in tensors(r) if x[0] in keep]


def _overlap(a, b):
    return a[1] < b[1] + b[2] and b[1] < a[1] + a[2]


def test_footprint(built):
    b = built
    for r in b.recs:
        for t, ptr, n in tensors(r):
            assert b.alloc_of(ptr, ptr + n), f"{_name(b, r)}: {t} [{ptr:#x}, +{n}) lies in no allocation"
        if r.dP_shared:  # the caller's scratch holds every call that uses it
            a = b.alloc_of(r.dP, r.dP + 2 * r.images * r.heads * r.T * r.ldT)
            assert a, f"{_name(b, r)}: the shared dP is smaller than {r.images * r.heads} x {r.T} x {r.ldT}"
    bwd = [r for r in b.recs if r.backward]
    for i, r in enumerate(bwd):
        own_writes = [x for x in tensors(r) if x[0] in ("gqkv", "dP", "delta")]
        for s in saved(r):
            for w in own_writes:
                assert not _overlap(s, w), f"{_name(b, r)}: its backward writes {w[0]} over the saved {s[0]}"
            for j, q in enumerate(bwd):
                if j == i:
                    continue
                for t in tensors(q):
                    assert not _overlap(s, t), \
                        f"{_name(b, r)}: the saved {s[0]} overlaps {t[0]} of {_name(b, q)}"
    print(f"[attn plans] {b.name}: {len(b.recs)} attentions inside {len(b.allocs)} allocations, {len(bwd)} with a "
          f"backward, {sum(r.dP_shared for r in b.recs)} on a shared dP")


# ------------------------------------------------------------------------------------------------------- budgets
def fused_check(ref, mag, got):
    """Worst err / bound per output under test_attn_gpu.py's budgets (lse: 2^-16 mag)."""
    out = {}
    for n, g in got.items():
        err = (g - ref[n]).abs()
        bound = ABS * mag[n] if n == "lse" else C_BUDGET * U * mag[n] + FLOOR
        out[n] = (err / bound).max().item()
    return out


def chain_reference(q, k, v, g, scale, causal=False):
    """float64 outputs of the chain and their budgets c E + 2^-24 (module docstring), [..., T, d] each."""
    T = q.shape[-2]
    s = scale * (q @ k.transpose(-1, -2))
    sa = scale * (q.abs() @ k.abs().transpose(-1, -2))
    es = U * s.abs() + ABS * sa
    tiny = TINY
    if causal:
        keep = torch.ones(T, T, dtype=torch.bool, device=q.device).tril()
        s = s.masked_fill(~keep, float("-inf"))
        es = es.masked_fill(~keep, 0)
        tiny = TINY * keep
    p = torch.softmax(s, -1)
    o = p @ v
    ep = p * (es + (p * es).sum(-1, keepdim=True)) + U * (p + tiny)
    ref = dict(o=o)
    e = dict(o=ep @ v.abs() + ABS * (p @ v.abs()) + U * o.abs())
    if g is not None:
        dp = g @ v.transpose(-1, -2)
        dd = (p * dp).sum(-1, keepdim=True)
        ds = p * (dp - dd)
        edp = U * dp.abs() + ABS * (g.abs() @ v.abs().transpose(-1, -2))
        ed = (ep * dp.abs() + p * edp).sum(-1, keepdim=True)
        eds = ep * (dp - dd).abs() + p * (edp + ed) + U * (ds.abs() + TINY)
        ref.update(dq=scale * ds @ k, dk=scale * ds.transpose(-1, -2) @ q, dv=p.transpose(-1, -2) @ g)
        e.update(dq=scale * (eds @ k.abs() + ABS * ds.abs() @ k.abs()) + U * ref["dq"].abs(),
                 dk=scale * (eds.transpose(-1, -2) @ q.abs() + ABS * ds.abs().transpose(-1, -2) @ q.abs())
                 + U * ref["dk"].abs(),
                 dv=ep.transpose(-1, -2) @ g.abs() + ABS * p.transpose(-1, -2) @ g.abs() + U * ref["dv"].abs())
    return ref, {n: C_BUDGET * x + FLOOR for n, x in e.items()}


def chain_ratios(ref, bound, got):
    return {n: ((got[n] - ref[n]).abs() / bound[n]).max().item() for n in got}


# ------------------------------------------------------------------------------------------------------- replay
def guarded(rows, cols, dtype, like):
    """[GUARD + rows + GUARD, cols]: SENTINEL guards, NaN inside, the inside at the engine pointer `like` modulo 256."""
    eb = torch.tensor([], dtype=dtype).element_size()
    n = (rows + 2 * GUARD) * cols
    off = ((like % 256) - GUARD * cols * eb) % 256 // eb
    raw = torch.full((n + 256 // eb,), SENTINEL, dtype=dtype, device="cuda")
    assert raw.data_ptr() % 256 == 0
    buf = raw[off:off + n].view(rows + 2 * GUARD, cols)
    buf[GUARD:GUARD + rows] = float("nan")
    assert buf[GUARD:].data_ptr() % 256 == like % 256
    return buf


def _inner(buf):
    return buf[GUARD:-GUARD]


def _guards_ok(name, what, buf):
    assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all(), f"{name}: {what} written outside"
    assert not torch.isnan(_inner(buf)).any(), f"{name}: {what} has elements left unwritten (or NaN)"


def case_inputs(r, case, seed):
    B, T, H, d = r.images, r.T, r.heads, r.d
    if case == "one_hot":
        qkv, d_o = _inputs(B, T, H, seed, qkv_std=5.0, d=d)
    elif case == "last_key":
        qkv, d_o = _peaked(B, T, H, T - 1, seed, d=d, scale=r.scale)
    else:
        qkv, d_o = _inputs(B, T, H, seed, d=d)
    if case == "big_dO":
        f = 4096.0
        if r.path == CHAIN:  # dP is stored fp16: the largest power of two <= 4096 with max |dO v^T| < 2^15
            x = _split(qkv.double(), B, T, H, d)
            dp = (_split(d_o.double(), B, T, H, d)[0] @ x[2].transpose(-1, -2)).abs().max().item()
            f = min(f, 2.0 ** math.floor(math.log2(2.0 ** 15 / dp)))
        d_o = (d_o.float() * f).half()
    return qkv, (d_o if r.backward else None)


def run_fused(b, r, qkv, d_o):
    lib = _lib.load()
    B, T, H, W = r.images, r.T, r.heads, r.W
    o = guarded(B * T, W, torch.half, r.o)
    lse = guarded(B * H * T, 1, torch.float32, r.lse)
    g = guarded(B * T, 3 * W, torch.half, r.gqkv) if d_o is not None else None
    delta = aligned(B * H * T, torch.float32, r.delta, float("nan")) if r.delta and d_o is not None else None
    out2, err = (C.c_int * 2)(), C.create_string_buffer(512)
    rc = lib.pxr_test_attention_plan(C.byref(r), _p(qkv), _p(_inner(o)), _p(d_o), _p(_inner(g)) if g is not None else None,
                                     _p(_inner(lse)), _p(delta), MMA if b.force_mma else 0, out2, err, 512)
    assert rc == 0, f"{_name(b, r)}: pxr_test_attention_plan rc={rc}: {err.value.decode()}"
    got = (out2[0], out2[1]) if r.backward else (out2[0], r.bwd)
    assert got == (r.splits, r.bwd), f"{_name(b, r)}: the hook plans {tuple(out2)}, the engine planned ({r.splits}, {r.bwd})"
    bufs = dict(o=o, lse=lse, gqkv=g)
    for k, v in bufs.items():
        if v is not None:
            _guards_ok(_name(b, r), k, v)
    return bufs


def run_chain(b, r, qkv, d_o):
    lib = _lib.load()
    B, T, H, W, ldT = r.images, r.T, r.heads, r.W, r.ldT
    rows = B * H * T
    o = guarded(B * T, W, torch.half, r.o)
    g = guarded(B * T, 3 * W, torch.half, r.gqkv) if d_o is not None else None
    P = aligned(rows * ldT, torch.half, r.P, float("nan"))  # the chain must write all it reads, pad columns included
    dP = aligned(rows * ldT, torch.half, r.dP, float("nan")) if d_o is not None else None
    mine = dict(qkv=qkv, o=_inner(o), P=P)
    if d_o is not None:
        mine.update(d_o=d_o, gqkv=_inner(g), dP=dP)
    spans = [(base, nb, mine[n]) for n, base, nb in tensors(r) if n in mine]

    def view(ptr):
        for base, nb, t in spans:
            if base <= ptr < base + nb:
                assert (ptr - base) % 2 == 0
                return t.reshape(-1)[(ptr - base) // 2:]
        raise AssertionError(f"{_name(b, r)}: a chain GEMM addresses {ptr:#x}, outside the record's tensors")

    def gemm(i):
        gr = b.grecs[i]
        d = _desc(gr, view(gr.a), view(gr.b), {"out_f16": view(gr.out_f16)})
        info = (C.c_int * 6)()
        assert lib.pxr_test_gemm_plan_info(C.byref(d), info) == 0
        got = dict(zip(("wide", "block_n", "stages", "tma_epi", "grid", "k_splits"), list(info)))
        want = {k: getattr(gr, k) for k in got}
        assert got == want, f"{_name(b, r)}: the hook plans {got} for {gr.label.decode()}, the engine planned {want}"
        err = C.create_string_buffer(512)
        assert lib.pxr_test_gemm(C.byref(d), err, 512) == 0, err.value.decode()

    gemm(r.gemm[0])
    assert lib.pxr_test_softmax(2 if r.causal else 0, _p(P), None, rows, T, ldT) == 0
    gemm(r.gemm[1])
    if d_o is not None:
        gemm(r.gemm[2])
        assert lib.pxr_test_softmax(1, _p(P), _p(dP), rows, T, ldT) == 0
        for i in r.gemm[3:6]:
            gemm(i)
    torch.cuda.synchronize()
    bufs = dict(o=o, gqkv=g)
    for k, v in bufs.items():
        if v is not None:
            _guards_ok(_name(b, r), k, v)
    return bufs


CASES = ("random", "one_hot", "last_key", "big_dO")


def replay(b, r, case, seed):
    """Worst err / bound per output of record r on one input case; asserts the budgets, guards and determinism."""
    name = _name(b, r)
    B, T, H, d = r.images, r.T, r.heads, r.d
    qkv, d_o = case_inputs(r, case, seed)
    qkv_a = aligned_copy(qkv.reshape(-1), r.qkv)
    d_o_a = aligned_copy(d_o.reshape(-1), r.d_o) if d_o is not None else None
    run = run_chain if r.path == CHAIN else run_fused
    first, again = run(b, r, qkv_a, d_o_a), run(b, r, qkv_a, d_o_a)
    for k, v in first.items():
        if v is not None:
            assert torch.equal(v.view(torch.uint8), again[k].view(torch.uint8)), f"{name}: two runs differ in {k}"
    got = dict(o=_split(_inner(first["o"]).double(), B, T, H, d)[0])
    if d_o is not None:
        gq = _split(_inner(first["gqkv"]).double(), B, T, H, d)
        got.update(dq=gq[0], dk=gq[1], dv=gq[2])
    if r.path == CHAIN:
        x = _split(qkv.double(), B, T, H, d)
        gd = _split(d_o.double(), B, T, H, d)[0] if d_o is not None else None
        ref, bound = chain_reference(x[0], x[1], x[2], gd, r.scale, bool(r.causal))
        q = chain_ratios(ref, bound, got)
    else:
        got["lse"] = _inner(first["lse"]).double().reshape(B, H, T)
        ref, mag = _reference(qkv, d_o, B, T, H, r.scale, d=d, causal=bool(r.causal), device="cuda")
        q = fused_check(ref, mag, got)
    bad = {n: v for n, v in q.items() if not v <= 1.0}
    assert not bad, f"{name}, {case}: err / bound {bad}"
    return q


def _attn_signature(b, r):
    ptrs = (r.qkv, r.o, r.d_o, r.gqkv, r.lse, r.delta, r.P, r.dP)
    g = tuple(_signature(b.grecs[i]) for i in r.gemm if i >= 0)
    return (r.path, r.images, r.heads, r.T, r.d, r.W, r.scale, r.causal, r.multihead, r.backward, r.splits, r.bwd, r.ldT,
            r.dP_shared) + tuple((bool(p), (p or 0) % 256) for p in ptrs) + g


def test_replay_every_attention(built):
    b = built
    first = {}
    for r in b.recs:
        first.setdefault(_attn_signature(b, r), r)
    worst = {}  # path -> output -> (err / bound, where)
    for k, r in enumerate(first.values()):
        for c, case in enumerate(CASES):
            if case == "big_dO" and not r.backward:
                continue
            w = worst.setdefault(r.path, {})
            for n, v in replay(b, r, case, seed=100 * k + c).items():
                if v > w.get(n, (-1.0,))[0]:
                    w[n] = (v, f"{r.site.decode()} T={r.T} {case}")
        torch.cuda.empty_cache()
    lines = [f"[attn plans] {b.name}: {len(b.recs)} attentions, {len(first)} replayed; worst err/bound"]
    for path, w in sorted(worst.items()):
        lines.append(f"  {('fused', 'streaming', 'chain')[path]}: " + ", ".join(
            f"{n} {w[n][0]:.3f} ({w[n][1]})" if n in w else f"{n} -" for n in ("o", "lse", "dq", "dk", "dv")))
    _log(lines)


# ------------------------------------------------------------------------------------------------------- the chain budget
def _h(x):
    return x.half().double()


def emulate_chain(q, k, v, g, scale, mutation=None):
    """float64 chain with an fp16 store at S, P, O, dP, dS and the gradients; a mutation plants one defect."""
    s = _h(scale * (q @ k.transpose(-1, -2)))
    if mutation == "pad_column":  # a zero pad column counted in the denominator
        sp = torch.cat([s, torch.zeros_like(s[..., :1])], -1)
        p = _h(torch.softmax(sp, -1)[..., :-1])
    elif mutation == "drop_last_key":
        p = torch.cat([torch.softmax(s[..., :-1], -1), torch.zeros_like(s[..., -1:])], -1)
        p = _h(p)
    else:
        p = _h(torch.softmax(s, -1))
    out = dict(o=_h(p @ v))
    dp = _h(g @ v.transpose(-1, -2))
    dd = 0 if mutation == "no_D" else (p * dp).sum(-1, keepdim=True)
    ds = _h(p * (dp - dd))
    kk = torch.roll(k, 1, dims=-3) if mutation == "neighbour_K" else k  # dims: [..., heads, T, d]
    out["dq"] = _h(scale * ds @ kk)
    out["dk"] = _h((1.0 if mutation == "dk_unscaled" else scale) * ds.transpose(-1, -2) @ q)
    out["dv"] = _h(p.transpose(-1, -2) @ g)
    return out


def _cpu_case(kind, T, H=2, d=64, seed=0):
    """fp16-exact float64 q, k, v, dO [H, T, d] on the CPU.  "random": as test_attn_gpu's (std 1.5, dO std 1);
    "negative": every score near -4 with v around 1, where a zero pad column takes a sixth of the weight;
    "last_key": every row's maximum at the last key; "mean_v": v around 1, so that D = dO . O is not small."""
    gen = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(3, H, T, d, generator=gen) * 1.5).unbind(0)
    g = torch.randn(H, T, d, generator=gen)
    if kind == "negative":
        q, k = q * 0.1, k * 0.1
        q[..., 0], k[..., 0] = 4.0, -8.0
        v = 1 + 0.5 * v
    elif kind == "last_key":
        q, k = q / 3, k / 3
        q[..., 0], k[..., 0] = 4.0, 0.5 * torch.randn(H, T, generator=gen)
        k[..., -1, 0] = 16.0
    elif kind == "mean_v":
        v = 1 + 0.5 * v
    return _h(q), _h(k), _h(v), _h(g)


@pytest.mark.parametrize("kind,T", [("random", 257), ("random", 256), ("negative", 257), ("last_key", 256),
                                    ("mean_v", 197), ("random", 77)])
def test_chain_budget_accepts_the_fp16_chain(kind, T):
    """The chain's budget admits a float64 emulation of the chain with every fp16 store it makes."""
    q, k, v, g = _cpu_case(kind, T)
    ref, bound = chain_reference(q, k, v, g, 0.125)
    q_ = chain_ratios(ref, bound, emulate_chain(q, k, v, g, 0.125))
    assert max(q_.values()) <= 1.0, q_


@pytest.mark.parametrize("mutation,kind,T", [("pad_column", "negative", 257), ("drop_last_key", "last_key", 256),
                                             ("dk_unscaled", "random", 257), ("no_D", "mean_v", 197),
                                             ("neighbour_K", "random", 257)])
def test_chain_budget_rejects_planted_defects(mutation, kind, T):
    """Each planted defect pushes some output past its budget."""
    q, k, v, g = _cpu_case(kind, T)
    ref, bound = chain_reference(q, k, v, g, 0.125)
    q_ = chain_ratios(ref, bound, emulate_chain(q, k, v, g, 0.125, mutation))
    assert max(q_.values()) > 1.0, f"{mutation} passes the chain budget: {q_}"


def test_chain_budget_single_head_d512():
    """The VQGAN decoder's shape (one head, d = 512, scale 512^-1/2): the emulation passes, a dropped last key fails."""
    gen = torch.Generator().manual_seed(5)
    T, d, scale = 256, 512, 512 ** -0.5
    q, k, v = (torch.randn(1, T, d, generator=gen) * 0.5 for _ in range(3))
    g = _h(torch.randn(1, T, d, generator=gen))
    q[..., 0], k[..., 0] = 4.0, 0.5 * torch.randn(1, T, generator=gen)
    k[..., -1, 0] = 2.0 / scale  # the last key scores about 8 above the rest against every query
    q, k, v = _h(q), _h(k), _h(v)
    ref, bound = chain_reference(q, k, v, g, scale)
    assert max(chain_ratios(ref, bound, emulate_chain(q, k, v, g, scale)).values()) <= 1.0
    assert max(chain_ratios(ref, bound, emulate_chain(q, k, v, g, scale, "drop_last_key")).values()) > 1.0


def test_record_struct_follows_the_header():
    """ctypes lays the record out by its field list: it must name the header's fields in its order."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pixray_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} pxr_test_attn_rec;", src).group(1)
    names = []
    for decl in filter(None, (x.strip() for x in body.split(";"))):
        first, *rest = decl.split(",")
        names += [re.sub(r"\[.*\]$", "", re.sub(r"^.*[\s*]", "", first.strip()))] + [x.strip() for x in rest]
    assert [f[0] for f in _lib.TestAttnRec._fields_] == names
    assert (_lib.ATTN_FUSED, _lib.ATTN_STREAMING, _lib.ATTN_CHAIN) == tuple(
        int(re.search(rf"PXR_ATTN_{n} = (\d+)", src).group(1)) for n in ("FUSED", "STREAMING", "CHAIN"))
