"""Every convolution plan the engine builds, replayed against float64 with the engine's own packed weights.

The VQGAN decoder / encoder, the vdiff U-Net, a CLIP ResNet tower and the RRDBNet all run their convolutions through one
operator: `pack_conv` lays a checkpoint weight out as the implicit-GEMM operand (tap-flipped and transposed for a dgrad,
restricted to an input-channel window for the RRDB dgrad slices), and `add_conv` picks the tile width, split-K and
kernel.  The engine records both (pxr_test_packed_weights / pxr_test_conv_records).  These tests build each engine at
real shapes (finalize() makes the plans; nothing runs) and check

- packing: every forward operand is fp16 of its checkpoint weight in the [tap][cout_pad][cin] layout the plan reads,
  zeros elsewhere, bit for bit (ResNet: the float64 BatchNorm fold within 1 ulp; RRDB conv5: times the block's 0.2), and
  every dgrad operand is the tap-flipped transpose of its verified forward partner over its input-channel window;
- routing: what the wide kernel, split-K and the epilogues may combine, and that the decoder and the U-Net do reach the
  wide kernel in both directions;
- replay: each distinct plan, rebuilt by the test hook from the record (the hook must report the engine's own choices),
  run on random inputs whose pitch padding is NaN, against a float64 reference of the same operand, bias, residual and
  activation, with element bound |err| <= 2^-11 |ref| + 2^-16 S (S = sum |a||w| + |bias| + |res|); canaries outside the
  output untouched, two runs bit-identical;
- that this bound rejects references with a dropped tap block, two swapped taps or a halo shifted at the border.
"""
import ctypes as C
import os
import re
import sys

import pytest
import torch
import torch.nn.functional as F

from pixray_b200 import _lib
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.resnet_ref import fold_conv  # noqa: E402

TE_F16, TE_RES16 = 1, 5
ACT_NONE, ACT_LRELU, ACT_LRELU_BWD, ACT_RELU, ACT_RELU_BWD = 0, 4, 5, 8, 9
SMALL_CLIP = dict(width=128, layers=2, heads=2, patch=32, image_res=224, out_dim=64)
PAD_PIX = 37
CANARY = -7.0
REL, ABS = 2.0 ** -11, 2.0 ** -16


# ------------------------------------------------------------------------------------------------------- the bound
def bound_ratio(out, ref, s):
    """max over elements of |out - ref| / (2^-11 |ref| + 2^-16 S); <= 1 passes.  All float64."""
    err = (out - ref).abs()
    bound = REL * ref.abs() + ABS * s
    return (err / bound.clamp_min(1e-300)).max().item()


def conv_ref(x, wt, ks, cout_pad, n_out):
    """out[b, h, w, n] = sum_{tap, c} x[b, h + dy, w + dx, c] Wt[tap cout_pad + n, c] (tap = ks (dy + r) + dx + r) and
    S = the same sum of |x| |Wt|, float64 NHWC.  x [B, H, W, c_in], wt [taps cout_pad, c_in]."""
    w4 = wt.double().view(ks, ks, cout_pad, -1)[:, :, :n_out].permute(2, 3, 0, 1)
    xd = x.double().permute(0, 3, 1, 2)
    acc = F.conv2d(xd, w4, padding=ks // 2).permute(0, 2, 3, 1)
    s = F.conv2d(xd.abs(), w4.abs(), padding=ks // 2).permute(0, 2, 3, 1)
    return acc, s


def epilogue_ref(acc, s, bias, res, aux, act, act_col0):
    """The epilogue of gemm_tc.cu in float64: bias, then LeakyReLU before the residual, the backward masks and ReLU
    after it."""
    y = acc.clone()
    if bias is not None:
        y = y + bias.double()
        s = s + bias.double().abs()
    if act == ACT_LRELU:
        y = torch.where(y > 0, y, 0.2 * y)
    if res is not None:
        y = y + res.double()
        s = s + res.double().abs()
    if act == ACT_LRELU_BWD:
        cols = torch.arange(y.shape[-1], device=y.device)
        y = torch.where((cols >= act_col0) & ~(aux > 0), 0.2 * y, y)
    elif act == ACT_RELU_BWD:
        y = torch.where(aux > 0, y, torch.zeros_like(y))
    elif act == ACT_RELU:
        y = y.clamp_min(0)
    return y, s


# ------------------------------------------------------------------------------------------------------- the hooks
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def conv_records(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_conv_records(eng.h, None, 0, C.byref(n)), "pxr_test_conv_records")
    recs = (_lib.TestConvRec * n.value)()
    eng._check(lib.pxr_test_conv_records(eng.h, recs, n.value, C.byref(n)), "pxr_test_conv_records")
    return list(recs)


def pack_records(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_packed_weights(eng.h, None, 0, C.byref(n), -1, None, None, None, 0), "pxr_test_packed_weights")
    recs = (_lib.TestPackRec * n.value)()
    eng._check(lib.pxr_test_packed_weights(eng.h, recs, n.value, C.byref(n), -1, None, None, None, 0),
               "pxr_test_packed_weights")
    return list(recs)


def packed_operand(eng, index, n, bias=None, n_bias=0):
    """Copy of packed operand `index` (fp16 [n]) and, optionally, n_bias floats of the engine bias pointer `bias`."""
    w = torch.empty(n, device="cuda", dtype=torch.half)
    b = torch.empty(max(n_bias, 1), device="cuda") if bias else None
    rc = _lib.load().pxr_test_packed_weights(eng.h, None, 0, None, index, _p(w), C.c_void_p(bias) if bias else None,
                                             _p(b), n_bias)
    eng._check(rc, "pxr_test_packed_weights")
    return w, (b[:n_bias] if bias else None)


# ------------------------------------------------------------------------------------------------------- engines
def _vqgan(hw, seed=0):
    sd = S.vqgan_state_dict(E.VQGAN_F16_16384, seed, with_encoder=True)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=hw, vqgan=E.VQGAN_F16_16384, cutn=8, clip=[SMALL_CLIP], seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    return eng, sd


def _vdiff(hw, seed=0):
    sd = S.vdiff_state_dict(seed, c=128)
    eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=hw, cutn=8, clip=[SMALL_CLIP], seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    return eng, sd


def _resnet(seed=0):
    arch = E.RESNET_ARCH["RN50x4"]
    sd = S.clip_resnet_state_dict(arch, seed)
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=4, cut_size=arch["image_res"],
                       clip=[arch], seed=seed)
    eng.load_module(E.MOD_CLIP0, sd)
    return eng, sd


RRDB = dict(num_feat=64, num_block=2, num_grow_ch=32)


def _rrdb(seed=0):
    sd = S.rrdbnet_state_dict(seed, **RRDB)
    eng = E.B200Engine(drawer=E.DRAWER_SUPERRES, image_hw=(192, 256), superres=RRDB, cutn=8, clip=[SMALL_CLIP], seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    return eng, sd


ENGINES = {
    "vqgan256": lambda: _vqgan((256, 256)),
    "vqgan288x432": lambda: _vqgan((288, 432)),  # latent 18 x 27: ragged at tile width 16 and at 8
    "vdiff256": lambda: _vdiff((256, 256)),
    "vdiff64": lambda: _vdiff((64, 64)),
    "rn50x4": _resnet,
    "rrdb": _rrdb,
    "vqgan512": lambda: _vqgan((512, 512)),
}
SLOW = {"vqgan512"}
WIDE_AT_SCALE = {"vqgan256", "vqgan288x432", "vqgan512", "vdiff256"}


class Built:
    def __init__(self, name):
        self.name = name
        self.eng, self.sd = ENGINES[name]()
        self.eng.finalize()
        self.convs = conv_records(self.eng)
        self.packs = pack_records(self.eng)
        # the first operand packed from a (tag, host weights) pair is the forward, later ones its dgrad operands
        self.partner, seen = {}, {}
        for i, p in enumerate(self.packs):
            key = (p.tag, p.src)
            if key in seen:
                self.partner[i] = seen[key]
            else:
                seen[key] = i
        self.by_ptr = {p.ptr: i for i, p in enumerate(self.packs)}
        self.plans_of = {}
        for r in self.convs:
            self.plans_of.setdefault(r.wt, []).append(r)

    def is_dgrad(self, i):
        return i in self.partner

    def part(self, r):
        """'encoder' / 'decoder' (VQGAN), 'unet', 'resnet', 'rrdb' for a plan record."""
        tag = self.packs[self.by_ptr[r.wt]].tag.decode()
        if self.name.startswith("vqgan"):
            return "encoder" if tag.startswith(("encoder.", "quant_conv")) else "decoder"
        return "unet" if self.name.startswith("vdiff") else "resnet" if self.name == "rn50x4" else "rrdb"

    def close(self):
        self.eng.close()


def _params():
    return [pytest.param(n, marks=[pytest.mark.gpu] + ([pytest.mark.slow] if n in SLOW else [])) for n in ENGINES]


@pytest.fixture(scope="module", params=_params())
def built(request):
    b = Built(request.param)
    yield b
    b.close()


# ------------------------------------------------------------------------------------------------------- packing
def _checkpoint_fp16(b, rec):
    """The checkpoint weight of a pack record as the engine should store it: fp16 [cout, cin, taps] (cuda), and the
    allowed ulp distance."""
    tag = rec.tag.decode()
    if b.name == "rn50x4":
        bn = re.sub(r"conv(\d)$", r"bn\1", tag) if not tag.endswith("downsample.0") else tag[:-1] + "1"
        w, _ = fold_conv(b.sd, tag, bn)
        return w.half().reshape(rec.cout, rec.cin, rec.taps).cuda(), 1
    w = b.sd[tag + ".weight"].float()
    if b.name == "rrdb" and re.fullmatch(r"body\.\d+\.rdb\d\.conv5", tag):
        w = w * 0.2  # the dense block's residual scale, folded into conv5 (fp32 product, then fp16)
    return w.half().reshape(rec.cout, rec.cin, rec.taps).cuda(), 0


def _canonical(b, i, got):
    """Operand i as [taps, rows, K]: the [tap][rows][K] layout the conv plan reads (rows = the plan's cout_pad, K its
    c_in) when a plan uses it, else the GEMM layouts of the operands only GEMMs read: [rows][K] (ResNet 1x1 / stem),
    [rows][taps][cin] (vdiff tiny forward), [cin][taps][cout_k] (vdiff tiny dgrad)."""
    p = b.packs[i]
    dgrad = b.is_dgrad(i)
    plans = b.plans_of.get(p.ptr, [])
    if plans:
        r = plans[0]
        assert all((q.cout_pad, q.c_in, q.ks) == (r.cout_pad, r.c_in, r.ks) for q in plans)
        assert r.ks * r.ks == p.taps, f"{p.tag}: a {r.ks}x{r.ks} plan on a {p.taps}-tap operand"
        assert p.n == p.taps * r.cout_pad * r.c_in, f"{p.tag}: operand of {p.n} elements, plan reads " \
            f"{p.taps} x {r.cout_pad} x {r.c_in}"
        return got.view(p.taps, r.cout_pad, r.c_in)
    if p.s_tap * p.taps == p.n:  # tap-major (one tap: a plain [rows][K] GEMM operand)
        K = p.s_ci if dgrad else p.s_co
        assert (p.s_co if dgrad else p.s_ci) == 1 and p.n % (p.taps * K) == 0
        return got.view(p.taps, p.n // (p.taps * K), K)
    K = p.s_tap
    assert (p.s_co, p.s_ci) == ((1, p.taps * K) if dgrad else (p.taps * K, 1)), f"{p.tag}: unknown layout"
    return got.view(p.n // (p.taps * K), p.taps, K).permute(1, 0, 2)


def _expected_windows(b, tag, cin):
    """The input-channel windows the dgrad operands of a conv must cover: all of its inputs, except an RRDB conv5's,
    split at num_feat (the block input x, then the concatenated x1..x4)."""
    if b.name == "rrdb" and re.fullmatch(r"body\.\d+\.rdb\d\.conv5", tag):
        nf = RRDB["num_feat"]
        return {(0, nf), (nf, cin)}
    return {(0, cin)}


def test_packed_operands(built):
    b = built
    forward = {}
    windows = {}
    n_fwd = n_dg = 0
    for i, p in enumerate(b.packs):
        got, _ = packed_operand(b.eng, i, p.n)
        canon = _canonical(b, i, got)
        tag = p.tag.decode()
        if not b.is_dgrad(i):
            w16, ulp = _checkpoint_fp16(b, p)
            taps, rows, K = canon.shape
            assert rows >= p.cout and K >= p.cin, f"{tag}: {rows} x {K} cannot hold {p.cout} x {p.cin}"
            exp = torch.zeros(taps, rows, K, device="cuda", dtype=torch.half)
            exp[:, :p.cout, :p.cin] = w16.permute(2, 0, 1)
            d = (canon.view(torch.int16).int() - exp.view(torch.int16).int()).abs().max().item()
            assert d <= ulp, f"{tag}: forward operand differs from the checkpoint by {d} ulp (allowed {ulp})"
            assert not p.flip
            forward[i] = canon
            n_fwd += 1
        else:
            fw = forward[b.partner[i]]
            assert p.flip, f"{tag}: dgrad operand packed without the tap flip"
            assert 0 <= p.ci0 < p.ci1 <= p.cin, f"{tag}: dgrad window [{p.ci0}, {p.ci1}) of {p.cin} input channels"
            windows.setdefault(tag, (p.cin, set()))[1].add((p.ci0, p.ci1))
            taps, rows, K = canon.shape
            m = p.ci1 - p.ci0
            assert rows >= m and K >= p.cout, f"{tag}: dgrad {rows} x {K} cannot hold window {m} x {p.cout}"
            exp = torch.zeros(taps, rows, K, device="cuda", dtype=torch.half)
            exp[:, :m, :p.cout] = fw.flip(0)[:, :p.cout, p.ci0:p.ci1].transpose(1, 2)
            assert torch.equal(canon.view(torch.int16), exp.view(torch.int16)), \
                f"{tag}: dgrad operand [{p.ci0}, {p.ci1}) is not the flipped transpose of its forward operand"
            n_dg += 1
    for tag, (cin, got) in windows.items():
        assert got == _expected_windows(b, tag, cin), f"{tag}: dgrad windows {sorted(got)}"
    print(f"[conv plans] {b.name}: {n_fwd} forward and {n_dg} dgrad operands bit-exact")


# ------------------------------------------------------------------------------------------------------- routing
def test_routing_invariants(built):
    b = built
    assert b.convs, "no conv plans recorded"
    for r in b.convs:
        name = r.label.decode()
        if r.wide:
            assert r.k_splits == 1 and r.block_n in (128, 192, 256) and r.tma_epi in (TE_F16, TE_RES16), name
            assert r.act == ACT_NONE and not r.out_f32, name
        if r.k_splits > 1:
            assert r.batch == 1 and not r.out_f32 and r.act == ACT_NONE and not r.has_aux, name
    wide = {}
    for r in b.convs:
        key = (b.part(r), "dgrad" if b.is_dgrad(b.by_ptr[r.wt]) else "forward")
        wide[key] = wide.get(key, 0) + r.wide
    if b.name in WIDE_AT_SCALE:  # at 64^2 every U-Net level is small enough for split-K or the tiny GEMMs
        for part in ("decoder", "unet"):
            for d in ("forward", "dgrad"):
                if any(k[0] == part for k in wide):
                    assert wide.get((part, d), 0) >= 1, f"{b.name}: no {part} {d} convolution on the wide kernel"
    sigs = {_signature(r) for r in b.convs}
    print(f"[conv plans] {b.name}: {len(b.convs)} records, {len(sigs)} distinct signatures, "
          f"{sum(r.wide for r in b.convs)} wide, {sum(r.k_splits > 1 for r in b.convs)} split-K; wide by part {wide}")


# ------------------------------------------------------------------------------------------------------- replay
SIG_FIELDS = [f for f, _ in _lib.TestConvRec._fields_ if f not in ("label", "wt", "bias")]


def _signature(r):
    return tuple(getattr(r, f) for f in SIG_FIELDS)


def _desc(r, x, wt, bias, aux, res, out):
    d = _lib.TestGemmDesc()
    d.a, d.lda, d.b = _p(x), r.in_ld, _p(wt)
    d.N, d.block_n, d.fmt, d.alpha = r.n_out, r.block_n, 0, 1.0
    if r.k_splits > 1:
        d.out_f32, d.ldc, d.k_splits = _p(out), r.n_out, r.k_splits
        return d
    d.bias, d.act, d.act_col0, d.aux_in, d.res_f16 = _p(bias), r.act, r.act_col0, _p(aux), _p(res)
    if r.out_f32:
        d.out_f32 = _p(out)
    else:
        d.out_f16 = _p(out)
    d.ldc = r.ldc
    return d


def _run(r, x, wt, bias, aux, res):
    """One run of the recorded plan through the conv hook (+ the split-K reduce): the [px + PAD_PIX, ldc] output."""
    lib = _lib.load()
    px = r.batch * r.H * r.W
    dtype = torch.float32 if r.out_f32 else torch.half
    out = res.clone() if r.in_place else torch.full((px + PAD_PIX, r.ldc), CANARY, device="cuda", dtype=dtype)
    res_arg = out if r.in_place else res
    ws = torch.zeros(r.k_splits, px, r.n_out, device="cuda") if r.k_splits > 1 else None
    d = _desc(r, x, wt, bias, aux, res_arg, ws if ws is not None else out)
    info = (C.c_int * 6)()
    assert lib.pxr_test_conv_plan_info(C.byref(d), r.batch, r.H, r.W, r.c_in, r.cout_pad, r.ks, info) == 0
    got = dict(zip(("wide", "block_n", "stages", "tma_epi", "grid", "k_splits"), list(info)))
    want = {k: getattr(r, k) for k in got}
    assert got == want, f"{r.label.decode()}: the hook plans {got}, the engine planned {want}"
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_conv(C.byref(d), r.batch, r.H, r.W, r.c_in, r.cout_pad, r.ks, err, 512)
    assert rc == 0, f"pxr_test_conv rc={rc}: {err.value.decode()}"
    if ws is not None:
        rc = lib.pxr_test_splitk_reduce(_p(ws), r.k_splits, C.c_longlong(px), r.n_out, r.n_out, _p(bias), _p(res_arg),
                                        _p(out), int(r.ldc))
        assert rc == 0
    torch.cuda.synchronize()
    return out


def replay(b, r, seed):
    """Worst err / bound of plan record r over its output; asserts plan identity, canaries and determinism."""
    name = f"{b.name}: {r.label.decode()}"
    g = torch.Generator(device="cuda").manual_seed(seed)
    px = r.batch * r.H * r.W
    x = torch.full((r.batch, r.H, r.W, r.in_ld), float("nan"), device="cuda", dtype=torch.half)
    x[..., :r.c_in] = (torch.randn(r.batch, r.H, r.W, r.c_in, device="cuda", generator=g) * 0.5).half()
    i = b.by_ptr[r.wt]
    wt, bias = packed_operand(b.eng, i, b.packs[i].n, r.bias if r.has_bias else None, r.n_out if r.has_bias else 0)
    assert b.packs[i].n == r.ks * r.ks * r.cout_pad * r.c_in
    aux = torch.randn(px + PAD_PIX, r.ldc, device="cuda", generator=g).half() if r.has_aux else None
    res = (torch.randn(px + PAD_PIX, r.ldc, device="cuda", generator=g) * 0.5).half() if r.has_res else None
    out = _run(r, x, wt, bias, aux, res)
    again = _run(r, x, wt, bias, aux, res)
    assert torch.equal(out, again), f"{name}: two runs differ"
    # untouched: pixels past the output, and channels past the 16-byte block that holds the last output column
    untouched = res if r.in_place else torch.full_like(out, CANARY)
    gran = 4 if r.out_f32 else 8
    c8 = -(-r.n_out // gran) * gran
    assert torch.equal(out[px:], untouched[px:]), f"{name}: pixels past the output written"
    assert torch.equal(out[:px, c8:], untouched[:px, c8:]), f"{name}: channels past {c8} written"
    acc, s = conv_ref(x[..., :r.c_in], wt.view(-1, r.c_in), r.ks, r.cout_pad, r.n_out)
    n = r.n_out
    ref, s = epilogue_ref(acc.reshape(px, n), s.reshape(px, n), bias, res[:px, :n] if r.has_res else None,
                          aux[:px, :n] if r.has_aux else None, r.act, r.act_col0)
    got = out[:px, :n].double()
    assert torch.isfinite(got).all(), f"{name}: non-finite outputs (the NaN pitch padding was read?)"
    q = bound_ratio(got, ref, s)
    assert q <= 1.0, f"{name}: err / bound {q:.3f}"
    return q


def test_replay_every_plan(built):
    b = built
    first = {}
    for r in b.convs:
        first.setdefault(_signature(r), r)
    worst, worst_name = 0.0, ""
    for k, r in enumerate(first.values()):
        q = replay(b, r, seed=k)
        if q > worst:
            worst, worst_name = q, r.label.decode()
    print(f"[conv plans] {b.name}: {len(b.convs)} records, {len(first)} signatures replayed, "
          f"{sum(r.wide for r in b.convs)} wide, {sum(r.k_splits > 1 for r in b.convs)} split-K; worst err/bound "
          f"{worst:.3f} ({worst_name})")


# ------------------------------------------------------------------------------------------------------- the bound
# one representative shape per engine: (batch, H, W, c_in, n_out, ks)
SENS_SHAPES = {
    "vqgan": (1, 16, 16, 512, 512, 3),
    "vdiff": (1, 16, 16, 256, 256, 3),
    "resnet": (2, 18, 18, 192, 192, 3),
    "rrdb": (1, 24, 32, 192, 64, 3),
}


@pytest.mark.parametrize("engine", list(SENS_SHAPES))
def test_bound_rejects_planted_defects(engine):
    """Pure float64 on the CPU: a perfectly rounded fp16 output passes the bound, and references with a dropped 64-channel
    tap block in one 128-pixel tile, two swapped taps or a halo shifted by one pixel at the border all fail it."""
    B, H, W, cin, n, ks = SENS_SHAPES[engine]
    g = torch.Generator().manual_seed(len(engine))
    x = (torch.randn(B, H, W, cin, generator=g) * 0.5).half()
    wt = (torch.randn(ks * ks * n, cin, generator=g) / (ks * ks * cin) ** 0.5).half()
    acc, s = conv_ref(x, wt, ks, n, n)
    out = acc.half().double()  # the best any fp16 kernel can do
    assert bound_ratio(out, acc, s) <= 1.0

    w4 = wt.double().view(ks, ks, n, cin)
    # one tap's 64-channel block dropped for the first 128-pixel tile (8 rows x 16 columns) of image 0
    w_drop = w4.clone()
    w_drop[1, 1, :, 64:128] = 0
    acc_drop, _ = conv_ref(x, w_drop.view(-1, cin), ks, n, n)
    bad = acc.clone()
    bad[0, :8, :16] = acc_drop[0, :8, :16]
    assert bound_ratio(out, bad, s) > 1.0, "a dropped tap block passes the bound"
    # taps (0, 0) and (2, 2) swapped
    w_swap = w4.clone()
    w_swap[0, 0], w_swap[2, 2] = w4[2, 2], w4[0, 0]
    acc_swap, _ = conv_ref(x, w_swap.view(-1, cin), ks, n, n)
    assert bound_ratio(out, acc_swap, s) > 1.0, "swapped taps pass the bound"
    # the halo shifted by one pixel at the right border: the last column reads its own column again instead of zeros
    xs = x.clone()
    xs = torch.cat([xs, xs[:, :, -1:]], dim=2)
    acc_shift, _ = conv_ref(xs, wt, ks, n, n)
    bad = acc.clone()
    bad[:, :, -1] = acc_shift[:, :, -2]
    assert bound_ratio(out, bad, s) > 1.0, "a shifted border halo passes the bound"


def test_record_structs_follow_the_header():
    """ctypes lays the record structs out by their field lists: they must name the header's fields in its order."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pixray_b200.h")).read(), flags=re.S)
    for struct, cls in (("pxr_test_pack_rec", _lib.TestPackRec), ("pxr_test_conv_rec", _lib.TestConvRec)):
        body = re.search(r"typedef struct \{([^}]*)\} " + struct + ";", src).group(1)
        names = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            first, *rest = decl.split(",")
            names += [re.sub(r"\[.*\]$", "", re.sub(r"^.*[\s*]", "", first.strip()))] + [r.strip() for r in rest]
        assert [f[0] for f in cls._fields_] == names, struct
