"""The row kernels of kernels_clip.cu against float64 references computed on the CPU from the same fp16 / fp32 inputs.

Row softmax (softmax_forward / softmax_backward: the unfused attention of the VQGAN decoder and encoder, the vdiff U-Net
and the ViT beyond 240 tokens), with u = 2^-11:
  forward   |p - P| <= 2u P + 2^-24
  backward  |ds - dS| <= 2u |dS| + P sum_j |P_j| |dP_j| 2^-20 + 2^-24
Pad columns [cols, ld) come back 0, and rows outside the call are left alone.

LayerNorm (eps 1e-5) -- the fp32-stream kernel, the fp16-stream kernel with 8-byte vectors and the one with 16-byte
vectors, each chosen explicitly.  Per element, c = 4, x^ = (x - mean) rstd, g = dy gamma:
  forward   c u (|gamma| |x^| + |beta|) + 2^-24
  backward  c u rstd (|g| + mean|g| + |x^| mean|g x^|) + u |prev| + 2^-24   (accumulate: prev is what gx held)
with u = 2^-11 for fp16 outputs and 2^-18 for the fp32 outputs of the fp32-stream kernel."""
import ctypes as C

import pytest
import torch

from pixray_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -11
U32 = 2.0 ** -18
FLOOR = 2.0 ** -24
SENTINEL = -1234.0  # exact in fp16 and fp32


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _round_up(n, m):
    return (n + m - 1) // m * m


# ------------------------------------------------------------------------------------------------------------- softmax
SOFTMAX_COLS = [1, 7, 8, 50, 197, 256, 257, 1024, 1025, 1200, 2304, 4096]
ROWS = 13  # not a multiple of the 8 rows a thread block covers


def _softmax(backward, a, b, rows, cols, ld):
    lib = _lib.load()
    rc = lib.pxr_test_softmax(backward, _p(a), _p(b), rows, cols, ld)
    assert rc == 0, rc


def _guarded_rows(vals, ld, pad_fill):
    """[1 + rows + 1, ld] fp16: SENTINEL guard rows around the rows `vals` [rows, cols]; pad columns hold pad_fill."""
    rows, cols = vals.shape
    buf = torch.full((rows + 2, ld), SENTINEL, dtype=torch.half, device="cuda")
    buf[1:-1] = pad_fill
    buf[1:-1, :cols] = vals
    return buf


def _check_frame(buf, cols, what):
    assert (buf[0] == SENTINEL).all() and (buf[-1] == SENTINEL).all(), f"{what}: a guard row changed"
    pad = buf[1:-1, cols:]
    assert torch.equal(pad.float().abs(), torch.zeros_like(pad.float())), f"{what}: pad columns are not 0"


@pytest.mark.parametrize("cols", SOFTMAX_COLS)
@pytest.mark.parametrize("wide", [False, True])
def test_softmax_forward_and_backward_match_float64(cols, wide):
    ld = _round_up(cols, 8) + (72 if wide else 0)
    g = torch.Generator(device="cuda").manual_seed(cols * 2 + wide)
    s = (torch.randn(ROWS, cols, generator=g, device="cuda") * 3).half()
    s[0, -1] = 20.0  # the row maximum on the last column (past the first 1024 on long rows)
    buf = _guarded_rows(s, ld, 7.0)
    _softmax(0, buf[1:], None, ROWS, cols, ld)
    _check_frame(buf, cols, "forward")
    p = buf[1:-1, :cols].double().cpu()
    ref = torch.softmax(s.double().cpu(), -1)
    err = (p - ref).abs()
    bound = 2 * U * ref + FLOOR
    print(f"[softmax fwd] cols={cols} ld={ld}: max err/(u P) {((err - FLOOR).clamp_min(0) / (U * ref)).max().item():.3f}")
    assert (err <= bound).all(), f"forward: {int((err > bound).sum())} elements over budget, max err {err.max().item():.3e}"

    # backward from the kernel's own fp16 P
    P16 = buf[1:-1, :cols].clone()
    dp = (torch.randn(ROWS, cols, generator=g, device="cuda") * 2).half()
    pbuf = _guarded_rows(P16, ld, 0.0)
    dbuf = _guarded_rows(dp, ld, -3.0)
    _softmax(1, pbuf[1:], dbuf[1:], ROWS, cols, ld)
    _check_frame(dbuf, cols, "backward")
    assert torch.equal(pbuf[1:-1, :cols], P16), "backward changed P"
    Pd, dPd = P16.double().cpu(), dp.double().cpu()
    dS = Pd * (dPd - (Pd * dPd).sum(-1, keepdim=True))
    ds = dbuf[1:-1, :cols].double().cpu()
    err = (ds - dS).abs()
    bound = 2 * U * dS.abs() + Pd * (Pd.abs() * dPd.abs()).sum(-1, keepdim=True) * 2.0 ** -20 + FLOOR
    print(f"[softmax bwd] cols={cols} ld={ld}: max err/bound {(err / bound).max().item():.3f}")
    assert (err <= bound).all(), f"backward: {int((err > bound).sum())} elements over budget, max err {err.max().item():.3e}"


def test_softmax_rejects_bad_arguments():
    lib = _lib.load()
    t = torch.zeros(4, 64, dtype=torch.half, device="cuda")
    assert lib.pxr_test_softmax(0, _p(t), None, 4, 60, 60) != 0   # ld % 8
    assert lib.pxr_test_softmax(0, _p(t), None, 4, 65, 64) != 0   # cols > ld
    assert lib.pxr_test_softmax(1, _p(t), None, 4, 64, 64) != 0   # backward without dP


# ----------------------------------------------------------------------------------------------------------- LayerNorm
F32, F16, F16_WIDE = 0, 1, 2
WIDTHS = [128 * k for k in range(1, 9)]


def _ln(variant, backward, x, x_stride, pos, T, gamma, beta, rows, W, y16=None, y32=None, stats=None, dy=None,
        accumulate=0, gx=None, gx16=None):
    lib = _lib.load()
    return lib.pxr_test_layernorm(C.c_int(variant), C.c_int(backward), _p(x), C.c_longlong(x_stride), _p(pos),
                                  C.c_int(T), _p(gamma), _p(beta), C.c_int(rows), C.c_int(W), C.c_float(1e-5), _p(y16),
                                  _p(y32), _p(stats), _p(dy), C.c_int(accumulate), _p(gx), _p(gx16))


def _ln_case(W, class_rows, with_pos, seed):
    """x [B*T, W] (the rows used: all, or the class row of each image), pos [T, W], gamma, beta, dy [rows, W]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, T = 3, 50
    x = torch.randn(B * T, W, generator=g, device="cuda") * 1.5 + 0.5 * torch.randn(B * T, 1, generator=g, device="cuda")
    pos = 0.3 * torch.randn(T, W, generator=g, device="cuda") if with_pos else None
    gamma = 1 + 0.3 * torch.randn(W, generator=g, device="cuda")
    beta = 0.3 * torch.randn(W, generator=g, device="cuda")
    rows, stride = (B, T * W) if class_rows else (B * T, W)
    dy = (torch.randn(rows, W, generator=g, device="cuda") * 4).half()
    return dict(x=x, pos=pos, gamma=gamma, beta=beta, rows=rows, stride=stride, T=T, dy=dy, g=g)


def _ln_reference(xs, pos_rows, gamma, beta, dy):
    """float64 forward / backward on the used rows xs [rows, W] (the stream's own precision), pos_rows [rows, W] or None."""
    x = xs.double().cpu()
    if pos_rows is not None:
        x = x + pos_rows.double().cpu()
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-5)
    xh = (x - mean) * rstd
    ga, be = gamma.double().cpu(), beta.double().cpu()
    y = xh * ga + be
    gg = dy.double().cpu() * ga
    m1, m2 = gg.mean(-1, keepdim=True), (gg * xh).mean(-1, keepdim=True)
    gx = rstd * (gg - m1 - xh * m2)
    fmag = ga.abs() * xh.abs() + be.abs()
    bmag = rstd * (gg.abs() + gg.abs().mean(-1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(-1, keepdim=True))
    return dict(y=y, gx=gx, mean=mean[:, 0], rstd=rstd[:, 0], fmag=fmag, bmag=bmag)


def _assert_within(name, got, ref, bound):
    err = (got.double().cpu() - ref).abs()
    ok = err <= bound
    print(f"[layernorm] {name}: max err/bound {(err / bound).max().item():.3f}")
    assert ok.all(), f"{name}: {int((~ok).sum())} elements over budget, max err {err.max().item():.3e}"


def _used_rows(t, case):
    return t.view(-1, case["T"], t.shape[-1])[:, 0] if case["stride"] != t.shape[-1] else t


def _variants(W, with_pos):
    v = [F32, F16]
    if W % 256 == 0 and not with_pos:
        v.append(F16_WIDE)
    return v


@pytest.mark.parametrize("W", WIDTHS)
@pytest.mark.parametrize("layout", ["rows", "class_rows", "pos"])
def test_layernorm_matches_float64(W, layout):
    class_rows, with_pos = layout == "class_rows", layout == "pos"
    case = _ln_case(W, class_rows, with_pos, W + len(layout))
    rows, stride, T = case["rows"], case["stride"], case["T"]
    outs = {}
    for variant in _variants(W, with_pos):
        x = case["x"] if variant == F32 else case["x"].half()
        xs = _used_rows(x, case)
        pos_rows = case["pos"].repeat(rows // T, 1) if with_pos else None
        ref = _ln_reference(xs, pos_rows, case["gamma"], case["beta"], case["dy"])
        y16 = torch.full((rows, W), float("nan"), dtype=torch.half, device="cuda")
        y32 = torch.full((rows, W), float("nan"), device="cuda") if variant == F32 else None
        stats = torch.full((rows, 2), float("nan"), device="cuda")
        rc = _ln(variant, 0, x, stride, case["pos"], T, case["gamma"], case["beta"], rows, W, y16=y16, y32=y32, stats=stats)
        assert rc == 0, rc
        tag = f"W={W} {layout} variant {variant}"
        _assert_within(f"{tag} y16", y16, ref["y"], 4 * U * ref["fmag"] + FLOOR)
        if y32 is not None:
            _assert_within(f"{tag} y32", y32, ref["y"], 4 * U32 * ref["fmag"] + FLOOR)
        _assert_within(f"{tag} mean", stats[:, 0], ref["mean"], U32 * (xs.double().cpu().abs().amax(-1) + 1))
        _assert_within(f"{tag} rstd", stats[:, 1], ref["rstd"], U32 * ref["rstd"])
        outs[variant] = y16

        # backward, overwrite then accumulate; gx / gx16 rows are x_stride apart, the rows in between must stay as they were
        for accumulate in (0, 1):
            fill = torch.randn(x.shape, generator=case["g"], device="cuda")
            gx16 = fill.half()
            gx = fill.clone() if variant == F32 else None
            prev = (gx if gx is not None else gx16).double().cpu()
            before16 = gx16.clone()
            rc = _ln(variant, 1, x, stride, case["pos"], T, case["gamma"], None, rows, W, stats=stats, dy=case["dy"],
                     accumulate=accumulate, gx=gx, gx16=gx16)
            assert rc == 0, rc
            want = ref["gx"] + (_used_rows(prev, case) if accumulate else 0)
            acc = U * _used_rows(prev, case).abs() if accumulate else 0
            _assert_within(f"{tag} gx16 accumulate={accumulate}", _used_rows(gx16, case), want,
                           4 * U * ref["bmag"] + acc + FLOOR)
            if gx is not None:
                acc32 = U32 * _used_rows(prev, case).abs() if accumulate else 0
                _assert_within(f"{tag} gx accumulate={accumulate}", _used_rows(gx, case), want,
                               4 * U32 * ref["bmag"] + acc32 + FLOOR)
            if class_rows:
                other = torch.ones(x.shape[0], dtype=torch.bool)
                other[::T] = False
                assert torch.equal(gx16[other], before16[other]), "backward wrote a row it was not given"
                if gx is not None:
                    assert torch.equal(gx[other], fill[other])
    if F16_WIDE in outs:  # the two fp16-stream kernels agree within the budget on the same input
        ref = _ln_reference(_used_rows(case["x"].half(), case), None, case["gamma"], case["beta"], case["dy"])
        _assert_within(f"W={W} {layout} 8-byte vs 16-byte", outs[F16], outs[F16_WIDE].double().cpu(),
                       8 * U * ref["fmag"] + 2 * FLOOR)


@pytest.mark.parametrize("W", [64, 192, 320, 576, 960, 1152])
def test_layernorm_width_without_a_kernel_is_an_error(W):
    x = torch.zeros(8, W, device="cuda")
    gamma, beta = torch.ones(W, device="cuda"), torch.zeros(W, device="cuda")
    y16 = torch.full((8, W), SENTINEL, dtype=torch.half, device="cuda")
    stats = torch.zeros(8, 2, device="cuda")
    for variant in (F32, F16, F16_WIDE):
        xv = x if variant == F32 else x.half()
        assert _ln(variant, 0, xv, W, None, 1, gamma, beta, 8, W, y16=y16, stats=stats) != 0
        assert _ln(variant, 1, xv, W, None, 1, gamma, None, 8, W, stats=stats, dy=y16, gx16=y16) != 0
    assert (y16 == SENTINEL).all(), "a refused call wrote its output"


def test_layernorm_wide_kernel_refuses_what_it_cannot_do():
    W = 384  # not a multiple of 256
    x = torch.zeros(8, W, dtype=torch.half, device="cuda")
    gamma, beta = torch.ones(W, device="cuda"), torch.zeros(W, device="cuda")
    y16 = torch.zeros(8, W, dtype=torch.half, device="cuda")
    stats = torch.zeros(8, 2, device="cuda")
    assert _ln(F16_WIDE, 0, x, W, None, 1, gamma, beta, 8, W, y16=y16, stats=stats) != 0
    assert _ln(F16, 0, x, W, None, 1, gamma, beta, 8, W, y16=y16, stats=stats) == 0
    W = 256  # pos and fp32 outputs only exist in the 8-byte kernels
    x, gamma, beta = x[:, :W].contiguous(), gamma[:W].contiguous(), beta[:W].contiguous()
    y16, y32, pos = y16[:, :W].contiguous(), torch.zeros(8, W, device="cuda"), torch.zeros(8, W, device="cuda")
    assert _ln(F16_WIDE, 0, x, W, pos, 8, gamma, beta, 8, W, y16=y16, stats=stats) != 0
    assert _ln(F16_WIDE, 0, x, W, None, 1, gamma, beta, 8, W, y16=y16, y32=y32, stats=stats) != 0
    assert _ln(3, 0, x, W, None, 1, gamma, beta, 8, W, y16=y16, stats=stats) != 0
