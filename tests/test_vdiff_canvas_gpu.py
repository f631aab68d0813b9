"""The vdiff drawer at canvases that are not powers of two: the U-Net at the gen size (the canvas rounded up to 128 per
side), the image its centre crop, and GroupNorm(1, C) on the three-kernel path where the single-kernel one does not hold
a level.

1. The three-kernel GroupNorm(1, C) (gn_stats + gn_apply, gn_backward with GnOpts) against float64 at the U-Net norm
   shapes the single kernel does not cover, with the bounds of tests/test_decoder_blocks_gpu.py: y 6e-3, dx 8e-3, mean
   and rstd 2e-5 relative.  Both paths agree where both run; a rerun gives the same bits.
2. Engine parity against oracle.ref_path.VDiffCC12M1 with the bounds of tests/test_vdiff_gpu.py.  At 200 x 100 the whole
   iteration (synth, cutouts, CLIP, loss, backward) runs against R.iterate on the CPU.  At 288 x 288 and 576 x 324 the
   oracle's U-Net runs in fp32 on the GPU (TF32 off) and is driven by the engine's own d loss / d image, which the
   200 x 100 case and the cutout tests pin: v, pred, the image and z.grad are compared.  Every case also checks the crop
   (the image is the window of clamp((pred + 1) / 2) read back at gen size, to the bit), a zero g_pred outside the
   window, the re-noising at gen size, and which attention kernels the U-Net reached.
3. An engine built with vdiff_gen_hw equal to the canvas is the engine built without it.
4. api.do_init + three api.train steps at pixray's default settings with drawer="vdiff".
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import _lib
from pixray_b200 import engine as E
from pixray_b200 import util as U
from test_decoder_blocks_gpu import _relu_safe, check_gn, gn_reference
from test_pipeline_gpu import SMALL_CLIP, plant_extremes, random_transforms, report

pytestmark = pytest.mark.gpu


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ 1. GroupNorm(1, C)
CS = (128, 256, 256, 512, 512, 1024, 1024)


def unet_norm_shapes(gh, gw):
    """(pixels, C) of every U-Net norm: level lv has cs[lv] channels and the stage's last block cs[lv - 1]."""
    out = set()
    for lv in range(7):
        px = (gh >> lv) * (gw >> lv)
        out.add((px, CS[lv]))
        if lv:
            out.add((px, CS[lv - 1]))
    return out


def coop_covers(px, c, nsm=132):
    """gn_coop_supported (kernels_decoder.cu) at the H100 SXM's 132 SMs: a block's slab of x fits 216 KB."""
    rpb = max(16, -(-px // nsm))
    return 4 * 1024 * 4 + rpb * c * 2 <= 216 * 1024


def three_kernel_shapes():
    shapes = set()
    for gh, gw in ((384, 384), (384, 640), (512, 768)):
        shapes |= {s for s in unet_norm_shapes(gh, gw) if not coop_covers(*s)}
    return sorted(shapes)


def run_path(path, x, gamma, beta, gamma_add, act, res, eps, dy=None, dres=None):
    px, c = x.shape
    lib = _lib.load()
    y = torch.empty_like(x)
    stats = torch.zeros(64, device="cuda")
    dx = torch.empty_like(x) if dy is not None else None
    if path == 1:
        scratch = torch.zeros(128 * lib.pxr_test_groupnorm_partials(px, c) + 64, device="cuda")
    else:
        scratch = torch.zeros(64 * (torch.cuda.get_device_properties(0).multi_processor_count + 2) + 2, device="cuda")
    rc = lib.pxr_test_groupnorm_unet_path(path, _ptr(x), _ptr(gamma), _ptr(beta), C.c_float(gamma_add), act, _ptr(res),
                                          C.c_float(eps), px, c, _ptr(y), _ptr(stats), _ptr(dy), _ptr(dres), _ptr(dx),
                                          _ptr(scratch))
    assert rc == 0, rc
    return y, stats, dx


def _inputs(px, c, seed, m=0.0, s=1.0):
    g = _gen(seed)
    x = (m + s * (torch.randn(px, c, generator=g, device="cuda") + 0.3 * torch.randn(1, c, generator=g, device="cuda"))).half()
    gamma = 0.2 * torch.randn(c, generator=g, device="cuda")  # the modulation's scale; the kernels add gamma_add = 1
    beta = 0.2 * torch.randn(c, generator=g, device="cuda")
    res = torch.randn(px, c, generator=g, device="cuda").half()
    dy = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    dres = (0.7 * torch.randn(px, c, generator=g, device="cuda")).half()
    return x, gamma, beta, res, dy, dres


def test_three_kernel_shapes_are_the_uncovered_ones():
    shapes = three_kernel_shapes()
    print(f"[gn3] U-Net norm shapes beyond the single kernel: {shapes}")
    for s in ((147456, 128), (245760, 128), (61440, 256), (393216, 128), (98304, 256)):
        assert s in shapes


@pytest.mark.parametrize("px,c", three_kernel_shapes())
@pytest.mark.parametrize("act", [0, 1, 2])
def test_three_kernel_unet_groupnorm(px, c, act):
    x, gamma, beta, res, dy, dres = _inputs(px, c, px + c + act)
    if act == 2:
        x = _relu_safe(x, gamma + 1, beta, 1e-5)
    y, stats, dx = run_path(1, x, gamma, beta, 1.0, act, res, 1e-5, dy, dres)
    check_gn(f"3-kernel U-Net px={px} C={c} act={act}", y, stats, dx,
             gn_reference(x, 1, gamma + 1, beta, act, 1e-5, res, dy, dres), 1)


@pytest.mark.parametrize("ratio", [8.0, 64.0])
@pytest.mark.parametrize("px,c", [(147456, 128), (61440, 256)])
def test_three_kernel_unet_groupnorm_at_a_large_mean(px, c, ratio):
    x, gamma, beta, _, dy, dres = _inputs(px, c, px + c + int(ratio), m=ratio)
    y, stats, dx = run_path(1, x, gamma, beta, 1.0, 1, None, 1e-5, dy, dres)
    check_gn(f"3-kernel m/s={ratio:g} px={px} C={c}", y, stats, dx,
             gn_reference(x, 1, gamma + 1, beta, 1, 1e-5, dy16=dy, dres16=dres), 1)


def test_three_kernel_without_modulation():
    """The attention's norm: gamma / beta given, gamma_add 0, no activation; and null gamma / beta with gamma_add 1."""
    px, c = 147456, 128
    x, gamma, beta, _, dy, dres = _inputs(px, c, 5)
    y, stats, dx = run_path(1, x, gamma + 1, beta, 0.0, 0, None, 1e-5, dy, dres)
    check_gn("3-kernel gamma_add 0", y, stats, dx, gn_reference(x, 1, gamma + 1, beta, 0, 1e-5, dy16=dy, dres16=dres), 1)
    y, stats, dx = run_path(1, x, None, None, 1.0, 0, None, 1e-5, dy, None)
    one, zero = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    check_gn("3-kernel null gamma / beta", y, stats, dx, gn_reference(x, 1, one, zero, 0, 1e-5, dy16=dy), 1)


@pytest.mark.parametrize("act", [1, 2])
def test_paths_agree_where_both_run(act):
    px, c = 65536, 128
    assert coop_covers(px, c)
    x, gamma, beta, res, dy, dres = _inputs(px, c, 11 + act)
    if act == 2:
        x = _relu_safe(x, gamma + 1, beta, 1e-5)
    y0, s0, dx0 = run_path(0, x, gamma, beta, 1.0, act, res, 1e-5, dy, dres)
    y1, s1, dx1 = run_path(1, x, gamma, beta, 1.0, act, res, 1e-5, dy, dres)
    ref = gn_reference(x, 1, gamma + 1, beta, act, 1e-5, res, dy, dres)
    check_gn(f"single kernel act={act}", y0, s0, dx0, ref, 1)
    check_gn(f"three kernels act={act}", y1, s1, dx1, ref, 1)
    e_y = (y0.double() - y1.double()).abs().max().item()
    e_dx = (dx0.double() - dx1.double()).abs().max().item()
    a, b = s0.view(32, 2).double(), s1.view(32, 2).double()
    e_m = ((a[:, 0] - b[:, 0]).abs() / torch.maximum(a[:, 0].abs(), 1 / a[:, 1])).max().item()
    e_r = ((a[:, 1] - b[:, 1]).abs() / a[:, 1]).max().item()
    print(f"[gn3] paths differ by y {e_y:.2e} dx {e_dx:.2e} mean {e_m:.2e} rstd {e_r:.2e} (relative)")
    assert e_y <= 6e-3 and e_dx <= 8e-3 and e_m <= 2e-5 and e_r <= 2e-5


def test_three_kernel_rerun_is_bit_identical():
    px, c = 245760, 128
    x, gamma, beta, res, dy, dres = _inputs(px, c, 21)
    a = run_path(1, x, gamma, beta, 1.0, 2, res, 1e-5, dy, dres)
    b = run_path(1, x, gamma, beta, 1.0, 2, res, 1e-5, dy, dres)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int16) if u.dtype == torch.half else u.view(torch.int32),
                           v.view(torch.int16) if v.dtype == torch.half else v.view(torch.int32))


# ------------------------------------------------------------------------------------------------ 2. engine parity
@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    return R.VDiffCC12M1().eval().requires_grad_(False)


def attention_records(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_attention_records(eng.h, None, 0, C.byref(n)), "pxr_test_attention_records")
    recs = (_lib.TestAttnRec * n.value)()
    eng._check(lib.pxr_test_attention_records(eng.h, recs, n.value, C.byref(n)), "pxr_test_attention_records")
    return list(recs)


def allocations(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_allocations(eng.h, None, None, 0, C.byref(n)), "pxr_test_allocations")
    ptrs, sizes = (C.c_void_p * n.value)(), (C.c_longlong * n.value)()
    eng._check(lib.pxr_test_allocations(eng.h, ptrs, sizes, n.value, C.byref(n)), "pxr_test_allocations")
    return list(sizes)


def build_engine(model, canvas_wh, gen=True, cutn=8, seed=3):
    w, h = canvas_wh
    gw, gh, _, _ = U.vdiff_gen_size(w, h)
    iw, ih = U.vdiff_image_size(w, h)
    clip = R.init_clip_weights(R.ClipVisual(224, SMALL_CLIP["patch"], SMALL_CLIP["width"], SMALL_CLIP["layers"],
                                            SMALL_CLIP["heads"], SMALL_CLIP["out_dim"]), seed + 1)
    kw = dict(vdiff_gen_hw=(gh, gw)) if gen else {}
    eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(ih, iw), cutn=cutn, clip=[SMALL_CLIP], noise_fac=0.1, seed=seed,
                       **kw)
    eng.load_module(E.MOD_VQGAN, model.ref_state_dict())
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, SMALL_CLIP["out_dim"], generator=g), wt, float("-inf")) for wt in (1.0, -0.3)]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
    steps, alphas, sigmas = U.vdiff_schedule(20)
    eng.vdiff_set_schedule(steps, alphas, sigmas)
    ce = torch.randn(1, 512, generator=g)
    eng.vdiff_set_clip_embed(ce.numpy())
    return eng, clip, prompts, ce, torch.from_numpy(steps), torch.from_numpy(alphas), torch.from_numpy(sigmas), g


def _crop(t, h, w, my, mx):
    return t[:, :, my:my + h, mx:mx + w]


def _check_canvas(model, canvas_wh, it, full_iteration):
    w, h = canvas_wh
    gw, gh, mx, my = U.vdiff_gen_size(w, h)
    eng, clip, prompts, ce, steps, alphas, sigmas, g = build_engine(model, canvas_wh)
    assert eng.z_shape == (1, 3, gh, gw) and eng.image_hw == (h, w)
    x = torch.randn(1, 3, gh, gw, generator=g) * float(sigmas[it]) + 0.3 * torch.rand(1, 3, gh, gw, generator=g)
    t = steps[it:it + 1]
    cutn, cs = 8, 224
    T = random_transforms(cutn, cs, 5)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    eng.vdiff_set_iteration(it)
    img = eng.synth(x)
    assert tuple(img.shape) == (1, 3, h, w)
    v = eng.debug_read("vd_v", (1, 3, gh, gw))
    pred = eng.debug_read("vd_pred", (1, 3, gh, gw))
    # the crop, to the bit
    assert torch.equal(img, _crop(((pred + 1) * 0.5).clamp(0, 1), h, w, my, mx))
    eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    zg = eng.backward().cpu()
    g_img = eng.debug_read("g_img", (1, 3, h, w)).cpu() / 4096.0
    gpred = eng.debug_read("vd_gpred", (1, 3, gh, gw))
    inside = torch.zeros(1, 3, gh, gw, dtype=torch.bool, device="cuda")
    inside[:, :, my:my + h, mx:mx + w] = True
    assert bool((gpred[~inside] == 0).all()), "g_pred outside the canvas window"
    tag = f"vdiff canvas {w}x{h} (U-Net {gw}x{gh})"
    if full_iteration:
        synth = lambda zz: _crop(R.vdiff_synth(model, zz, t, ce, alphas[it], sigmas[it])[0], h, w, my, mx)  # noqa: E731
        ref = R.iterate(synth, x, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
        _, ref_pred, ref_v = R.vdiff_synth(model, x, t, ce, alphas[it], sigmas[it])
        ref_img, ref_zg = ref["image"], ref["z_grad"]
        e_gi, m_gi = report(f"{tag}: d/d image", g_img, ref["image_grad"])
        assert e_gi <= 3e-2 * m_gi
    else:  # the oracle's U-Net on the GPU in fp32, driven by the engine's d loss / d image
        tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            mg = model.cuda()
            xg = x.cuda().requires_grad_(True)
            out, ref_pred, ref_v = R.vdiff_synth(mg, xg, t.cuda(), ce.cuda(), alphas[it].cuda(), sigmas[it].cuda())
            ref_img = _crop(out, h, w, my, mx)
            ref_img.backward(g_img.cuda())
            ref_zg = xg.grad.detach().cpu()
            ref_img, ref_pred, ref_v = ref_img.detach().cpu(), ref_pred.detach().cpu(), ref_v.detach().cpu()
        finally:
            model.cpu()
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    e_v, m_v = report(f"{tag}: v", v, ref_v)
    e_p, _ = report("pred", pred, ref_pred)
    e_i, _ = report("image", img, ref_img)
    e_g, m_g = report("z.grad", zg, ref_zg)
    d = zg - ref_zg
    l2 = d.norm().item() / ref_zg.norm().item()
    cos = torch.nn.functional.cosine_similarity(zg.reshape(1, -1), ref_zg.reshape(1, -1)).item()
    print(f"[parity] {tag}: z.grad rel-L2 {l2:.3e}, cosine {cos:.5f}")
    assert torch.isfinite(zg).all()
    assert e_v <= 2e-2 * m_v and e_p <= 2e-2 * max(m_v, 1.0) and e_i <= 1e-2
    assert e_g <= 8e-2 * m_g and l2 <= 0.12 and cos >= 0.99
    # makenoise at gen size on the pred / v of the synth above
    rn = torch.randn(1, 3, gh, gw, generator=torch.Generator().manual_seed(9))
    xr = R.vdiff_renoise(x, pred.cpu(), v.cpu(), alphas, sigmas, it, rn)
    xe = eng.vdiff_renoise(x.clone().cuda(), it, rn.cuda())
    assert tuple(xe.shape) == (1, 3, gh, gw)
    e, m = report("renoise", xe, xr)
    assert e <= 1e-5 * max(m, 1.0)
    recs = attention_records(eng)
    kinds = sorted({(r.T, r.path) for r in recs})
    print(f"[parity] {tag}: attention (T, path) {kinds}")
    for r in recs:
        if r.T > 257:
            assert r.path == _lib.ATTN_STREAMING, (r.T, r.path)
    return eng, kinds


def test_canvas_200x100(model):
    """U-Net 256 x 128: non-square, margins (28, 14), a 4 x 2 bottom level on the im2col path."""
    _check_canvas(model, (200, 100), it=12, full_iteration=True)


@pytest.mark.slow
def test_canvas_288x288(model):
    """U-Net 384 x 384: the three-kernel norm at level 0, streaming attention at T = 576, a 6 x 6 tiny level."""
    eng, kinds = _check_canvas(model, (288, 288), it=12, full_iteration=False)
    assert (576, _lib.ATTN_STREAMING) in kinds


@pytest.mark.slow
def test_canvas_576x324(model):
    """U-Net 640 x 384: the three-kernel norm at levels 0 and 1, T = 960, the 10 x 6 bottom level on the implicit-GEMM
    convolutions."""
    eng, kinds = _check_canvas(model, (576, 324), it=12, full_iteration=False)
    assert (960, _lib.ATTN_STREAMING) in kinds


# ------------------------------------------------------------------------------------------------ 3. nothing changes
def test_gen_equal_to_canvas_is_the_plain_build(model):
    a = build_engine(model, (256, 256), gen=True)
    b = build_engine(model, (256, 256), gen=False)
    ea, eb = a[0], b[0]
    assert ea.z_shape == eb.z_shape == (1, 3, 256, 256)
    assert allocations(ea) == allocations(eb)
    ra, rb = attention_records(ea), attention_records(eb)
    assert [(r.T, r.path, r.backward) for r in ra] == [(r.T, r.path, r.backward) for r in rb]
    g = torch.Generator().manual_seed(17)
    x = torch.randn(1, 3, 256, 256, generator=g) * 0.8
    T = random_transforms(8, 224, 5)
    facs, noise = torch.rand(8, generator=g) * 0.1, torch.randn(8, 3, 224, 224, generator=g)
    out = []
    for eng in (ea, eb):
        eng.vdiff_set_iteration(10)
        img = eng.synth(x)
        eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
        eng.encode_image(0)
        out.append((img, eng.backward()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


# ------------------------------------------------------------------------------------------------ 4. the API
def test_api_default_settings(tmp_path, monkeypatch):
    from pixray_b200 import api
    monkeypatch.chdir(tmp_path)
    api.reset_settings()
    try:
        api.add_settings(prompts="a lighthouse at dawn", drawer="vdiff", clip_models="ViT-B/16", iterations=3, outdir="",
                         seed="7", b200_allow_synthetic=True, vector_prompts="none")
        args = api.apply_settings()
        api.do_init(args)
        st = api._state
        assert st.engine.image_hw == (216, 384) and st.engine.z_shape == (1, 3, 256, 384)
        for it in range(3):
            api.train(args, it)
            st.cur_iteration = it + 1
            assert np.isfinite(np.asarray(st.losses)).all(), st.losses
        st.engine.sync()
        z = st.drawer.get_z()
        assert tuple(z.shape) == (1, 3, 256, 384) and bool(torch.isfinite(z).all())
        img = st.drawer.synth(2)
        assert tuple(img.shape) == (1, 3, 216, 384) and bool(torch.isfinite(img).all())
    finally:
        api.reset_settings()
