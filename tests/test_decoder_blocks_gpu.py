"""The decoders' building blocks at the kernel level, each against a float64 reference computed from the same fp16
inputs: split-K convolutions and GEMMs slab by slab, the split-K reduce bit for bit, the three-kernel GroupNorm, the
U-Net's GroupNorm(1, C) + modulation, the statistics at a large mean / spread ratio, the resampling and copy kernels with
their adjoints, and the fp16-weight GEMV.

Split-K: split s of a plan with `kbps` k-blocks per split writes the partial sum over k-blocks [s kbps, (s + 1) kbps) to
slab s of the fp32 workspace.  Block kb of a convolution is filter tap kb // (c_in / 64), channels 64 (kb % (c_in / 64))
... + 64, so a split that starts on the wrong tap or drops a block changes its slab even where the total would hide it.
Slab bound: 1e-5 * sum |a b| over the slab's terms, per element."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from gemm_util import run_conv, run_gemm
from pixray_b200 import _lib

pytestmark = pytest.mark.gpu

NUM_SMS = 132  # the engine's split-K rule is restated for an H100 SXM
SPLITK_WS_ELEMS = 8 << 20
SENTINEL = -12345.5


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def splitk_count(rows, N, nkb, tiles, num_sms=NUM_SMS):
    """Engine::splitk_count for an fp16-output epilogue: enough splits to fill the idle SMs with >= 4 k-blocks each."""
    if tiles * 2 > num_sms or nkb < 8 or N % 8:
        return 1
    splits = 1
    want = min(num_sms // tiles, nkb // 4)
    if want >= 2:
        kbps = -(-nkb // want)
        splits = -(-nkb // kbps)
    return 1 if splits * rows * N > SPLITK_WS_ELEMS else splits


def effective_splits(nkb, requested):
    """The plan's rounding: ceil(nkb / requested) k-blocks per split, as many splits as that takes."""
    kbps = -(-nkb // requested)
    return -(-nkb // kbps), kbps


def _prefix(contrib):
    """[nkb, ...] float64 per-block terms -> [nkb + 1, ...] prefix sums (slab = P[end] - P[begin])."""
    z = torch.zeros_like(contrib[:1])
    return torch.cat([z, contrib.cumsum(0)])


def _check_slabs(ws, ld, N, nkb, requested, pre, pre_abs, tag):
    """Slab s == float64 sum over its k-blocks; slabs past the effective count and pitch columns past N untouched."""
    eff, kbps = effective_splits(nkb, requested)
    worst = 0.0
    for s in range(eff):
        b, e = s * kbps, min(nkb, (s + 1) * kbps)
        ref = pre[e] - pre[b]
        bound = 1e-5 * (pre_abs[e] - pre_abs[b])
        err = (ws[s, :, :N].double() - ref).abs()
        assert bool((err <= bound).all()), f"{tag}: slab {s} (k-blocks {b}..{e - 1}) max err {err.max().item():.3e}"
        worst = max(worst, (err / bound.clamp_min(1e-300)).max().item())
    assert bool((ws[eff:] == SENTINEL).all()), f"{tag}: a slab past the {eff} splits was written"
    if ld > N:
        assert bool((ws[:eff, :, N:] == SENTINEL).all()), f"{tag}: pitch columns past N were written"
    return eff, kbps, worst


# ------------------------------------------------------------------------------------------------- split-K convolution
def _conv_setup(H, W, cin, N, ks, seed):
    g = _gen(seed)
    x = (torch.randn(1, H, W, cin, generator=g, device="cuda") * 0.5).half()
    taps = ks * ks
    wt = (torch.randn(taps, N, cin, generator=g, device="cuda") * 0.05).half()
    # per-block float64 terms [nkb, px, N]: block kb = tap kb // kpt, channels 64 (kb % kpt) ... + 64
    xp = F.pad(x[0].double(), (0, 0, 1, 1, 1, 1)) if ks == 3 else x[0].double()
    kpt = cin // 64
    contrib, contrib_abs = [], []
    for t in range(taps):
        dy, dx = (t // 3, t % 3) if ks == 3 else (0, 0)
        xs = xp[dy:dy + H, dx:dx + W].reshape(H * W, cin)
        wd = wt[t].double()
        for j in range(kpt):
            a, b = xs[:, 64 * j:64 * j + 64], wd[:, 64 * j:64 * j + 64]
            contrib.append(a @ b.T)
            contrib_abs.append(a.abs() @ b.abs().T)
    return x, wt, _prefix(torch.stack(contrib)), _prefix(torch.stack(contrib_abs))


CONV_SHAPES = [(H, W, cin, ks) for ks in (3, 1) for cin in (64, 128, 512) for (H, W) in ((16, 16), (32, 32), (9, 9), (5, 36))]


@pytest.mark.parametrize("H,W,cin,ks", CONV_SHAPES)
def test_split_k_conv_slab_by_slab(H, W, cin, ks):
    N = 512 if cin == 512 else 128
    ld = N + 8
    nkb = ks * ks * cin // 64
    x, wt, pre, pre_abs = _conv_setup(H, W, cin, N, ks, seed=H * 1000 + W * 10 + cin + ks)
    m_tiles = -(-H * W // 128)
    for bn in (64, 128):
        engine = splitk_count(H * W, N, nkb, m_tiles * -(-N // bn))
        for req in sorted({2, 3, 5, 7, nkb, nkb + 3, engine}):
            eff, kbps = effective_splits(nkb, req)
            ws = torch.full((eff + 1, H * W, ld), SENTINEL, device="cuda")
            run_conv(x, wt, N, N, ks, block_n=bn, out_f32=ws, ldc=ld, k_splits=req)
            tag = f"conv{ks}x{ks} {H}x{W} {cin}->{N} bn={bn} k_splits={req}"
            eff, kbps, worst = _check_slabs(ws, ld, N, nkb, req, pre, pre_abs, tag)
            again = torch.full_like(ws, SENTINEL)
            run_conv(x, wt, N, N, ks, block_n=bn, out_f32=again, ldc=ld, k_splits=req)
            assert torch.equal(ws, again), f"{tag}: two runs differ"
            print(f"[split-K conv] {tag}{' (engine)' if req == engine else ''}: {eff} splits of {kbps} k-blocks, "
                  f"max err / bound {worst:.2e}")


# ------------------------------------------------------------------------------------------------- split-K plain GEMM
GEMM_SHAPES = [(M, N, K) for M in (1, 4, 16) for N in (64, 256, 1024) for K in (576, 18432)] + [(4, 256, 200), (16, 64, 200)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_split_k_gemm_slab_by_slab(M, N, K):
    g = _gen(M * 7 + N + K)
    A = torch.randn(M, K, generator=g, device="cuda").half()
    B = (torch.randn(N, K, generator=g, device="cuda") * 0.1).half()
    nkb = -(-K // 64)
    Ad, Bd = F.pad(A.double(), (0, nkb * 64 - K)).view(M, nkb, 64), F.pad(B.double(), (0, nkb * 64 - K)).view(N, nkb, 64)
    pre = _prefix(torch.einsum("mkc,nkc->kmn", Ad, Bd))
    pre_abs = _prefix(torch.einsum("mkc,nkc->kmn", Ad.abs(), Bd.abs()))
    ld = N + 8
    for bn in (64, 128):
        engine = splitk_count(M, N, nkb, -(-N // bn))
        for req in sorted({2, 3, 5, 7, nkb, nkb + 3, engine}):
            eff, kbps = effective_splits(nkb, req)
            ws = torch.full((eff + 1, M, ld), SENTINEL, device="cuda")
            run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, out_f32=ws, ldc=ld, tma_epi=-1, k_splits=req)
            tag = f"gemm {M}x{N}x{K} bn={bn} k_splits={req}"
            eff, kbps, worst = _check_slabs(ws, ld, N, nkb, req, pre, pre_abs, tag)
            again = torch.full_like(ws, SENTINEL)
            run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, out_f32=again, ldc=ld, tma_epi=-1, k_splits=req)
            assert torch.equal(ws, again), f"{tag}: two runs differ"
            print(f"[split-K gemm] {tag}{' (engine)' if req == engine else ''}: {eff} splits of {kbps} k-blocks, "
                  f"max err / bound {worst:.2e}")


def test_split_k_refuses_what_the_reduce_cannot_finish():
    g = _gen(5)
    M, N, K = 16, 64, 576
    A = torch.randn(2, M, K, generator=g, device="cuda").half()
    B = torch.randn(N, K, generator=g, device="cuda").half()
    ws = torch.zeros(4, M, N, device="cuda")
    bias = torch.zeros(N, device="cuda")
    aux = torch.zeros(M, N, device="cuda", dtype=torch.half)
    out16 = torch.zeros(M, N, device="cuda", dtype=torch.half)
    common = dict(lda=K, ldb=K, block_n=64, out_f32=ws, ldc=N, k_splits=3)
    for extra in (dict(nb0=2, a_bs=(M * K, 0)), dict(bias=bias), dict(out_f16=out16), dict(act=1, aux_out=aux)):
        with pytest.raises(RuntimeError, match=r"rc=-22\b"):
            run_gemm(A, B, M, N, K, **common, **extra)
    x = torch.randn(2, 16, 16, 64, generator=g, device="cuda").half()
    wt = torch.randn(9, 64, 64, generator=g, device="cuda").half()
    with pytest.raises(RuntimeError, match=r"rc=-32\b"):
        run_conv(x, wt, 64, 64, 3, block_n=64, out_f32=torch.zeros(4, 2 * 256, 64, device="cuda"), ldc=64, k_splits=3)


# ------------------------------------------------------------------------------------------------- split-K reduce
def _reduce(ws, splits, px, N, ld_ws, bias, res, out, ld_out):
    rc = _lib.load().pxr_test_splitk_reduce(_ptr(ws), splits, C.c_longlong(px), N, ld_ws, _ptr(bias), _ptr(res), _ptr(out),
                                            ld_out)
    assert rc == 0, rc


@pytest.mark.parametrize("splits", [1, 2, 3, 4, 5, 8, 9, 18])
@pytest.mark.parametrize("with_bias,with_res", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_splitk_reduce_is_bit_exact(splits, with_bias, with_res):
    """bias first, partials in split order, residual last, one fp16 rounding: plain fp32 adds, so the order fixes the bits."""
    g = _gen(100 * splits + 10 * with_bias + with_res)
    px, N, ld_ws, ld_out = 997, 136, 144, 152  # 997 * 17 vectors: the last block is partly empty
    ws = torch.randn(splits, px, ld_ws, generator=g, device="cuda") * 3
    ws[:, :, N:] = float("nan")  # a read of the pitch columns would poison the output
    bias = torch.randn(N, generator=g, device="cuda") if with_bias else None
    res = (torch.randn(px, ld_out, generator=g, device="cuda") * 2).half() if with_res else None
    out = torch.full((px, ld_out), 777.0, device="cuda", dtype=torch.half)
    _reduce(ws, splits, px, N, ld_ws, bias, res, out, ld_out)
    acc = bias.expand(px, N).clone() if bias is not None else torch.zeros(px, N, device="cuda")
    for s in range(splits):
        acc = acc + ws[s, :, :N]
    if res is not None:
        acc = acc + res[:, :N].float()
    ref = acc.half()
    n_diff = (out[:, :N].view(torch.int16) != ref.view(torch.int16)).sum().item()
    print(f"[splitk_reduce] splits={splits} bias={with_bias} res={with_res}: {n_diff} differing fp16 outputs")
    assert n_diff == 0
    assert bool((out[:, N:] == 777.0).all()), "pad columns of the output were written"


@pytest.mark.parametrize("H,W,cin,N", [(16, 16, 512, 512), (9, 9, 128, 128), (5, 36, 256, 64)])
def test_split_k_conv_and_reduce_match_the_one_split_conv(H, W, cin, N):
    g = _gen(H * W + cin)
    x = (torch.randn(1, H, W, cin, generator=g, device="cuda") * 0.5).half()
    wt = (torch.randn(9, N, cin, generator=g, device="cuda") * 0.05).half()
    bias = torch.randn(N, generator=g, device="cuda")
    res = torch.randn(1, H, W, N, generator=g, device="cuda").half()
    bn = min(128, N)
    one = torch.zeros(1, H, W, N, device="cuda", dtype=torch.half)
    run_conv(x, wt, N, N, 3, block_n=bn, bias=bias, res_f16=res, out_f16=one, ldc=N)
    nkb = 9 * cin // 64
    req = max(2, splitk_count(H * W, N, nkb, -(-H * W // 128) * -(-N // bn)))
    eff, _ = effective_splits(nkb, req)
    ws = torch.zeros(eff, H * W, N, device="cuda")
    run_conv(x, wt, N, N, 3, block_n=bn, out_f32=ws, ldc=N, k_splits=req)
    split = torch.zeros(H * W, N, device="cuda", dtype=torch.half)
    _reduce(ws, eff, H * W, N, N, bias, res.view(H * W, N), split, N)
    w64 = wt.double().view(3, 3, N, cin).permute(2, 3, 0, 1)
    conv = F.conv2d(x.double().permute(0, 3, 1, 2), w64, padding=1).permute(0, 2, 3, 1).reshape(H * W, N)
    s_abs = F.conv2d(x.double().abs().permute(0, 3, 1, 2), w64.abs(), padding=1).permute(0, 2, 3, 1).reshape(H * W, N)
    ref = conv + bias.double() + res.view(H * W, N).double()
    half_ulp = 2.0 ** -11 * ref.abs() + 2.0 ** -25
    tol = 1e-5 * (s_abs + bias.double().abs() + res.view(H * W, N).double().abs())
    e_split = (split.double() - ref).abs()
    e_one = (one.view(H * W, N).double() - ref).abs()
    e_pair = (split.double() - one.view(H * W, N).double()).abs()
    print(f"[split-K conv + reduce] {H}x{W} {cin}->{N}, {eff} splits: vs float64 {e_split.max().item():.2e} "
          f"(one split {e_one.max().item():.2e}); differing fp16 outputs {(e_pair > 0).sum().item()}")
    assert bool((e_split <= tol + half_ulp).all()) and bool((e_one <= tol + half_ulp).all())
    assert bool((e_pair <= 2 * (tol + half_ulp)).all()), "split and one-split results differ by more than reassociation"


# ------------------------------------------------------------------------------------------------- GroupNorm
def gn_scratch(variant, px, c):
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    if variant == 2:  # gn_num_partials: blocks of ceil(px / 592) rows rounded up to a multiple of 32
        rpb = max(32, -(-(-(-px // 592)) // 32) * 32)
        return torch.zeros(128 * -(-px // rpb) + 64, device="cuda")
    return torch.zeros(64 * (nsm + 2) + 2, device="cuda")


def run_gn(variant, x, gamma, beta, swish, dy=None, dres=None):
    px, c = x.shape
    y = torch.empty_like(x)
    stats = torch.zeros(64, device="cuda")
    dx = torch.empty_like(x) if dy is not None else None
    rc = _lib.load().pxr_test_groupnorm(variant, _ptr(x), None, 0, None, None, None, _ptr(gamma), _ptr(beta), px, c, swish,
                                        _ptr(y), _ptr(stats), _ptr(dy), None, 0, _ptr(dres), _ptr(dx),
                                        _ptr(gn_scratch(variant, px, c)), 1)
    assert rc == 0, rc
    return y, stats, dx


def run_gn_unet(x, gamma, beta, gamma_add, act, res, eps, dy=None, dres=None):
    px, c = x.shape
    y = torch.empty_like(x)
    stats = torch.zeros(64, device="cuda")
    dx = torch.empty_like(x) if dy is not None else None
    rc = _lib.load().pxr_test_groupnorm_unet(_ptr(x), _ptr(gamma), _ptr(beta), C.c_float(gamma_add), act, _ptr(res),
                                             C.c_float(eps), px, c, _ptr(y), _ptr(stats), _ptr(dy), _ptr(dres), _ptr(dx),
                                             _ptr(gn_scratch(0, px, c)))
    assert rc == 0, rc
    return y, stats, dx


def gn_reference(x16, groups, gamma, beta, act, eps, res16=None, dy16=None, dres16=None):
    """float64 group_norm (+ act, + residual) and its autograd; also each group's (mean, rstd)."""
    x = x16.double().requires_grad_(True)
    px, c = x.shape
    h = F.group_norm(x.t().reshape(1, c, px), groups, None, None, eps=eps).reshape(c, px).t()
    a = h * gamma.double() + beta.double()
    y = a * torch.sigmoid(a) if act == 1 else (torch.relu(a) if act == 2 else a)
    if res16 is not None:
        y = y + res16.double()
    xg = x16.double().t().reshape(groups, -1)
    mean = xg.mean(1)
    rstd = 1.0 / torch.sqrt(xg.var(1, unbiased=False) + eps)
    dx = None
    if dy16 is not None:
        (dx,) = torch.autograd.grad(y, x, dy16.double())
        if dres16 is not None:
            dx = dx + dres16.double()
    return y.detach(), dx, a.detach(), mean, rstd


def check_gn(tag, y, stats, dx, ref, groups):
    y_ref, dx_ref, _, mean, rstd = ref
    st = stats.view(32, 2).double()
    rep = 32 // groups
    m_ref, r_ref = mean.repeat_interleave(rep), rstd.repeat_interleave(rep)
    e_y = (y.double() - y_ref).abs().max().item()
    e_dx = (dx.double() - dx_ref).abs().max().item() if dx is not None else 0.0
    e_m = ((st[:, 0] - m_ref).abs() / torch.maximum(m_ref.abs(), 1 / r_ref)).max().item()
    e_r = ((st[:, 1] - r_ref).abs() / r_ref).max().item()
    print(f"[gn] {tag}: y {e_y:.2e} dx {e_dx:.2e} | mean {e_m:.2e} rstd {e_r:.2e} (relative)")
    assert e_y <= 6e-3 and e_dx <= 8e-3 and e_m <= 2e-5 and e_r <= 2e-5, tag


def _gn_inputs(px, c, seed, m=0.0, s=1.0):
    g = _gen(seed)
    x = (m + s * (torch.randn(px, c, generator=g, device="cuda") + 0.3 * torch.randn(1, c, generator=g, device="cuda"))).half()
    gamma = 1 + 0.2 * torch.randn(c, generator=g, device="cuda")
    beta = 0.2 * torch.randn(c, generator=g, device="cuda")
    dy = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    dres = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    return x, gamma, beta, dy, dres


@pytest.mark.parametrize("px,c", [(4096, 128), (1024, 256), (4096, 512), (262144, 128)])
@pytest.mark.parametrize("swish", [0, 1])
def test_three_kernel_groupnorm(px, c, swish):
    """gn_stats + gn_apply and gn_backward: what add_gn / add_gn_bwd run when neither single-kernel path fits
    (262144 x 128 is the 512 x 512 canvas's top decoder level)."""
    x, gamma, beta, dy, dres = _gn_inputs(px, c, px + c + swish)
    y, stats, dx = run_gn(2, x, gamma, beta, swish, dy, dres)
    check_gn(f"3-kernel px={px} C={c} swish={swish}", y, stats, dx,
             gn_reference(x, 32, gamma, beta, swish, 1e-6, dy16=dy, dres16=dres), 32)


def _relu_safe(x, gamma_eff, beta, eps, tau=2e-3):
    """Move every element whose float64 pre-activation lies within tau of 0 away from it (a few fp16 steps), so the
    kernel's ReLU takes the same branch as the reference everywhere."""
    for _ in range(8):
        xd = x.double()
        mean, var = xd.mean(), xd.var(unbiased=False)
        a = (xd - mean) / torch.sqrt(var + eps) * gamma_eff.double() + beta.double()
        near = a.abs() < tau
        if not bool(near.any()):
            return x
        step = 3 * tau * torch.sqrt(var + eps) / gamma_eff.double().abs()
        push = torch.where(a >= 0, 1.0, -1.0) * torch.sign(gamma_eff.double()) * step
        x = torch.where(near, xd + push, xd).half()
    raise AssertionError("could not move the pre-activations away from 0")


# the U-Net's norms (vd_block's two, vd_attn's one) at a 64 x 64 and a 256 x 256 canvas: (pixels, C) per level
UNET_SHAPES = sorted({(px, c) for side in (64, 256) for lv, c in enumerate((128, 256, 256, 512, 512, 1024, 1024))
                      for px in [(side >> lv) ** 2]})


@pytest.mark.parametrize("px,c", UNET_SHAPES)
@pytest.mark.parametrize("act", [0, 1, 2])
def test_unet_groupnorm(px, c, act):
    g = _gen(px + c + act)
    x = (torch.randn(px, c, generator=g, device="cuda") + 0.3 * torch.randn(1, c, generator=g, device="cuda")).half()
    gamma = 0.2 * torch.randn(c, generator=g, device="cuda")  # the modulation's scale; the kernel adds gamma_add = 1
    beta = 0.2 * torch.randn(c, generator=g, device="cuda")
    res = torch.randn(px, c, generator=g, device="cuda").half()
    dy = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    dres = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    if act == 2:
        x = _relu_safe(x, gamma + 1, beta, 1e-5)
    y, stats, dx = run_gn_unet(x, gamma, beta, 1.0, act, res, 1e-5, dy, dres)
    check_gn(f"U-Net px={px} C={c} act={act}", y, stats, dx,
             gn_reference(x, 1, gamma + 1, beta, act, 1e-5, res, dy, dres), 1)


@pytest.mark.parametrize("ratio", [8.0, 64.0])
@pytest.mark.parametrize("path,px,c", [(0, 1024, 256), (0, 4096, 512), (1, 1024, 256), (1, 4096, 512), (2, 4096, 128),
                                       (2, 262144, 128), ("unet", 4096, 128), ("unet", 65536, 128), ("unet", 1, 1024)])
def test_groupnorm_statistics_at_a_large_mean(path, px, c, ratio):
    """x = m + s randn with m / s up to 64: the variance must not lose its precision to the mean."""
    x, gamma, beta, dy, dres = _gn_inputs(px, c, px + c + int(ratio), m=ratio, s=1.0)
    if path == "unet":
        y, stats, dx = run_gn_unet(x, gamma - 1, beta, 1.0, 1, None, 1e-5, dy, dres)
        ref = gn_reference(x, 1, gamma, beta, 1, 1e-5, dy16=dy, dres16=dres)
        groups = 1
    else:
        y, stats, dx = run_gn(path, x, gamma, beta, 1, dy, dres)
        ref = gn_reference(x, 32, gamma, beta, 1, 1e-6, dy16=dy, dres16=dres)
        groups = 32
    check_gn(f"m/s={ratio:g} path={path} px={px} C={c}", y, stats, dx, ref, groups)


# ------------------------------------------------------------------------------------------------- resampling and copies
UPSAMPLE, DOWNSUM, AVGPOOL, AVGPOOL_BWD, BILINEAR, BILINEAR_BWD, IM2COL, COPY = range(8)
IN_PAD, OUT_PAD = -777.0, 1234.0  # fp16-exact fillers of the pad channels: reads of IN_PAD would show, OUT_PAD must stay


def resample(op, x, ld_in, out, ld_out, H, W, Cc, accumulate=0):
    rc = _lib.load().pxr_test_resample(op, _ptr(x), ld_in, _ptr(out), ld_out, H, W, Cc, accumulate)
    assert rc == 0, (op, rc)


def _strided(t, ld, fill):
    """[..., C] -> a buffer of pixel stride ld whose channels C..ld hold `fill`, and the view of its first C channels."""
    buf = torch.full((*t.shape[:-1], ld), fill, dtype=torch.half, device="cuda")
    buf[..., :t.shape[-1]] = t
    return buf


def _shapes(op, H, W):
    """(input [h, w], output [h, w]) of `op` for the hook's H, W."""
    return {UPSAMPLE: ((H, W), (2 * H, 2 * W)), DOWNSUM: ((2 * H, 2 * W), (H, W)), AVGPOOL: ((H, W), (H // 2, W // 2)),
            AVGPOOL_BWD: ((H // 2, W // 2), (H, W)), BILINEAR: ((H, W), (2 * H, 2 * W)),
            BILINEAR_BWD: ((2 * H, 2 * W), (H, W)), IM2COL: ((H, W), (H * W, 9)), COPY: ((H, W), (H, W))}[op]


def _forward64(op, x):
    """float64 torch restatement of a forward op on an [h, w, C] tensor."""
    h, w, c = x.shape
    if op == IM2COL:
        return F.unfold(x.permute(2, 0, 1)[None], 3, padding=1).view(c, 9, h * w).permute(2, 1, 0)
    if op == COPY:
        return x
    if op == AVGPOOL and (h < 2 or w < 2):  # avg_pool2d refuses an empty output
        return x.new_zeros(h // 2, w // 2, c)
    xc = x.permute(2, 0, 1)[None]
    if op == UPSAMPLE:
        y = F.interpolate(xc, scale_factor=2, mode="nearest")
    elif op == AVGPOOL:
        y = F.avg_pool2d(xc, 2)
    else:
        y = F.interpolate(xc, scale_factor=2, mode="bilinear", align_corners=False)
    return y[0].permute(1, 2, 0)


ADJOINT_OF = {DOWNSUM: UPSAMPLE, AVGPOOL_BWD: AVGPOOL, BILINEAR_BWD: BILINEAR}


def _reference(op, x, out_hw):
    """float64 result of op on x [h, w, C]: forwards directly, adjoints through autograd of their forward."""
    if op not in ADJOINT_OF:
        return _forward64(op, x)
    z = torch.zeros(*out_hw, x.shape[2], dtype=torch.float64, device="cuda", requires_grad=True)
    y = _forward64(ADJOINT_OF[op], z)
    if y.numel() == 0:
        return torch.zeros_like(z).detach()
    (g,) = torch.autograd.grad(y, z, x)
    return g


def _dev(t):
    """an empty tensor has no device address: hand the kernel a dummy it must not read"""
    return t if t.numel() else torch.zeros(16, dtype=t.dtype, device="cuda")


RESAMPLE_HW = [(1, 1), (2, 2), (3, 3), (5, 7), (64, 64)]


@pytest.mark.parametrize("op", range(8))
@pytest.mark.parametrize("H,W", RESAMPLE_HW)
def test_resample_kernel_against_float64(op, H, W):
    (hi, wi), (ho, wo) = _shapes(op, H, W)
    worst = 0.0
    for Cc in (8, 64, 200):
        for pad in (0, 8):
            for acc in ((0, 1) if op in (AVGPOOL_BWD, COPY) else (0,)):
                g = _gen(op * 1000 + H * 10 + W + Cc + pad + acc)
                ld_in = Cc + pad if op in (UPSAMPLE, AVGPOOL, BILINEAR_BWD, COPY) else Cc
                ld_out = Cc + pad if op in (BILINEAR, COPY) else Cc
                x = torch.randn(hi, wi, Cc, generator=g, device="cuda").half()
                xb = _strided(x, ld_in, IN_PAD)
                if op == IM2COL:
                    prior = torch.randn(H * W, 9 * Cc, generator=g, device="cuda").half()
                    ob = prior.clone()
                else:
                    prior = torch.randn(ho, wo, Cc, generator=g, device="cuda").half()
                    ob = _strided(prior, ld_out, OUT_PAD)
                resample(op, _dev(xb), ld_in, _dev(ob), ld_out, H, W, Cc, acc)
                ref = _reference(op, x.double(), (ho, wo))
                slack = 1e-6 * _reference(op, x.double().abs(), (ho, wo))  # fp32 arithmetic before the fp16 rounding
                if acc:
                    ref, slack = ref + prior.double(), slack + 1e-6 * prior.double().abs()
                out = (ob if op == IM2COL else ob[..., :Cc]).reshape(ref.shape)
                tag = f"op={op} H={H} W={W} C={Cc} ld_in={ld_in} ld_out={ld_out} acc={acc}"
                err = (out.double() - ref).abs()
                if op in (UPSAMPLE, IM2COL) or (op == COPY and not acc):
                    assert torch.equal(out.double(), ref), f"{tag}: a copy must be exact"
                else:
                    assert bool((err <= 2.0 ** -11 * ref.abs() + slack + 2.0 ** -25).all()), \
                        f"{tag}: max err {err.max().item():.3e}"
                if err.numel():
                    worst = max(worst, err.max().item())
                if op != IM2COL and ld_out > Cc:
                    assert bool((ob[..., Cc:] == OUT_PAD).all()), f"{tag}: pad channels of the output were written"
    print(f"[resample] op={op} {H}x{W}: max err {worst:.2e} over C in (8, 64, 200), dense and strided"
          + (", accumulate" if op in (AVGPOOL_BWD, COPY) else ""))


@pytest.mark.parametrize("pair", [(UPSAMPLE, DOWNSUM), (AVGPOOL, AVGPOOL_BWD), (BILINEAR, BILINEAR_BWD)])
@pytest.mark.parametrize("H,W", RESAMPLE_HW)
def test_resample_adjoint_identity(pair, H, W):
    """<A x, y> == <x, A^T y> exactly in float64: small-integer inputs make every kernel output exact in fp16."""
    fwd, adj = pair
    (hi, wi), (ho, wo) = _shapes(fwd, H, W)
    Cc = 64
    g = _gen(H * 100 + W + fwd)
    x = torch.randint(-8, 9, (hi, wi, Cc), generator=g, device="cuda").half()
    y = torch.randint(-8, 9, (ho, wo, Cc), generator=g, device="cuda").half()
    ax = torch.empty(ho, wo, Cc, dtype=torch.half, device="cuda")
    aty = torch.empty(hi, wi, Cc, dtype=torch.half, device="cuda")
    resample(fwd, _dev(x), 0, _dev(ax), 0, H, W, Cc)
    resample(adj, _dev(y), 0, _dev(aty), 0, H, W, Cc)
    lhs = (ax.double() * y.double()).sum().item()
    rhs = (x.double() * aty.double()).sum().item()
    print(f"[adjoint] ops {fwd}/{adj} {H}x{W}: <Ax, y> = {lhs:g}, <x, A^T y> = {rhs:g}")
    assert lhs == rhs


def test_resample_refuses_unsupported_arguments():
    lib = _lib.load()
    buf = torch.zeros(4096, dtype=torch.half, device="cuda")
    p = _ptr(buf)
    assert lib.pxr_test_resample(COPY, p, 0, p, 0, 2, 2, 12, 0) == -1  # C % 8
    assert lib.pxr_test_resample(COPY, p, 8, p, 0, 2, 2, 16, 0) == -1  # ld < C
    assert lib.pxr_test_resample(COPY, p, 20, p, 0, 2, 2, 16, 0) == -1  # ld % 8
    assert lib.pxr_test_resample(8, p, 0, p, 0, 2, 2, 16, 0) == -2
    assert lib.pxr_test_resample(DOWNSUM, p, 24, p, 0, 2, 2, 16, 0) == -3  # no input stride
    assert lib.pxr_test_resample(UPSAMPLE, p, 0, p, 0, 2, 2, 16, 1) == -3  # no accumulate


# ------------------------------------------------------------------------------------------------- gemv_f16
@pytest.mark.parametrize("K", [8, 264, 1024])
@pytest.mark.parametrize("R", [1, 7, 1000])
def test_gemv_f16(K, R):
    lib = _lib.load()
    for with_bias, relu, with_res in [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 1), (1, 1, 1)]:
        g = _gen(K * 10 + R + 4 * with_bias + 2 * relu + with_res)
        w = (torch.randn(R, K, generator=g, device="cuda") / math.sqrt(K)).half()
        x = torch.randn(K, generator=g, device="cuda")
        bias = torch.randn(R, generator=g, device="cuda") if with_bias else None
        res = torch.randn(R, generator=g, device="cuda") if with_res else None
        y = torch.full((R,), SENTINEL, device="cuda")
        rc = lib.pxr_test_gemv(_ptr(w), K, R, _ptr(x), _ptr(bias), relu, _ptr(res), _ptr(y))
        assert rc == 0, rc
        ref = w.double() @ x.double() + (bias.double() if bias is not None else 0)
        if relu:
            ref = ref.clamp_min(0)
        if res is not None:
            ref = ref + res.double()
        bound = 1e-5 * ((w.double().abs() @ x.double().abs()) + (bias.double().abs() if bias is not None else 0)
                        + (res.double().abs() if res is not None else 0))
        err = (y.double() - ref).abs()
        print(f"[gemv] K={K} R={R} bias={with_bias} relu={relu} res={with_res}: max err / bound "
              f"{(err / bound).max().item():.2e}")
        assert bool((err <= bound).all())
