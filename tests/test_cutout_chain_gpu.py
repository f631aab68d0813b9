"""The image <-> patch-matrix chain of the engine against float64: pool_forward -> rescale_bilinear (non-square canvases)
-> cutout_forward -> min / max partials + minmax_reduce -> patchify_forward, and back: patchify_backward +
range_sums_finish -> cutout_backward (fixed-point scatter with the d/dmin, d/dmax terms) -> rescale_bilinear_backward ->
pool_backward (kernels_cutouts.cu).

The ViT is taken out of the comparison: the reference reads the engine's own upstream gradient clip{i}.g_patches (fp16,
the first 3 P^2 columns) and differentiates L = sum_i <patches_i, g_patches_i> in float64, where patches_i is the conv1
im2col (k = (c P + iy) P + ix) of CLIP_Base.preprocess (slip.py:21-60, with the tower's mean / std) of R.make_cutouts on
img.double().  What is compared, and how tightly:

  clip{i}.patches   within 1 fp16 ulp (+ 2^-20 for the fp32 cancellation in a - mean near 0) of the float64 preprocess
                    of the engine's own batch; pad columns k >= 3 P^2 exactly 0
  range, irange     exactly: float64 min / max / arg-min / arg-max of the engine's batch, R = fp32(max - min); the
                    indices also equal those of the float64 reference batch
  g_batch           (the direct term; the range terms are added inside cutout_backward) <= 2e-6 max|ref|
  sums              sum g and sum g (a - min) / R in float64 on the engine's batch, <= SUMS_REL = 1e-7 of the sum of
                    |terms| (fp32 block partials, then 64-bit fixed point; measured <= 2.3e-9)
  g_pooled, g_img   elementwise <= TAU * M + A + 1e-6 max|ref|.  M = the same float64 adjoint (warp, un-stretch, pooling:
                    all non-negative weights) applied to |d L / d batch| (range terms included): the magnitude that can
                    round.  A = that adjoint applied to the sums' allowance (SUMS_REL of their sums of |terms|) at the two
                    extreme elements: the range terms are differences of those sums, and where they cancel, the sums'
                    rounding is the larger error there.

TAU is about 3x the largest value measured over the cases (each case prints its own).  Measured on an H100 (80 GB HBM3,
700 W), g_pooled: zoom_out_border 2.3e-4, zoom_out_reflection 1.4e-4, cutn1 7.0e-5, canvas_512x448_p14 6.8e-5,
wide_18x32 6.3e-5, tall_48x32 6.0e-5, the others <= 3e-5; g_img: canvas_512x448_p14 6.3e-5, the others <= 1.3e-5.  The
remaining error comes from the fp32 sample coordinates through the bilinear weights: the engine inverts the homography in
double, rounds it to fp32 and evaluates it per pixel in fp32 (about 1e-4 px where a zoom-out to 0.3 puts the source
coordinates hundreds of pixels outside the image), and the reference samples on a grid from a float32 linspace (about
6e-6 px off in the cutout, magnified 1 / 0.3 times in the source by a zoom-out).

Out of scope: exact ties of the batch extremes (torch's full-reduction min() / max() backward spreads the gradient over
tied elements, the engine gives it to the first index; pixray always adds noise, pixray.py:508-510, so such ties do not
occur in the reference -- each case plants two unmistakable extremes); spot-prompt passes (only the last pass's
g_patches can be read back; tests/test_spot_prompts_gpu.py covers them); colour jitter (tests/test_color_jitter.py, at a
bound derived from its HSV discontinuities); the FFT drawer's backward.
"""
import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import cutouts
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu

TAU = 7e-4
SUMS_REL = 1e-7
CLIP_NORM = (R.CLIP_MEAN, R.CLIP_STD)
IMAGENET_NORM = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))  # SLIP_Base towers, slip.py:117-121
PAD_NAMES = {E.PAD_REFLECTION: "reflection", E.PAD_BORDER: "border"}


def _tower(patch, cs=224, timm=False):
    c = dict(width=128, layers=1, heads=2, patch=patch, image_res=cs, out_dim=64)
    if timm:
        c["tower"] = E.TOWER_TIMM_VIT
    return c


CASES = {
    # pooling upsamples (overlapping windows); P = 32: the vector patchify kernels
    "canvas_32x32_p32": dict(hw=(32, 32), clips=[_tower(32)], pad=E.PAD_REFLECTION),
    # pooling downsamples over ragged windows; P = 14: the generic patchify, Kp = 640 > K = 588
    "canvas_512x448_p14": dict(hw=(512, 448), clips=[_tower(14)], pad=E.PAD_BORDER),
    # non-square canvases: rescale_bilinear forward and backward
    "wide_32x48": dict(hw=(32, 48), clips=[_tower(32)], pad=E.PAD_REFLECTION, aspect=True),
    "wide_18x32": dict(hw=(18, 32), clips=[_tower(14)], pad=E.PAD_BORDER, aspect=True),
    "tall_48x32": dict(hw=(48, 32), clips=[_tower(32)], pad=E.PAD_REFLECTION, aspect=True),
    # two perceptors share the batch, in both orders: each patchify_backward variant with accumulate 0 and 1; the timm
    # tower normalises with the ImageNet mean / std
    "two_p14_then_timm_p32": dict(hw=(40, 40), clips=[_tower(14), _tower(32, timm=True)], pad=E.PAD_BORDER),
    "two_timm_p32_then_p14": dict(hw=(40, 40), clips=[_tower(32, timm=True), _tower(14)], pad=E.PAD_REFLECTION),
    # 336^2 / 4 is not a multiple of 256: partial last blocks in cutout_fwd / cutout_bwd, idle lanes in the min / max
    # partials; cutn 5 -> cutn_zoom 3
    "cut336_p48_cutn5": dict(hw=(40, 40), cs=336, cutn=5, clips=[_tower(48, cs=336)], pad=E.PAD_BORDER),
    # cutn_zoom = 0: every cutout takes the fill path
    "cutn1": dict(hw=(32, 32), cutn=1, clips=[_tower(32)], pad=E.PAD_REFLECTION),
    # zoom-out to ~0.3 with perspective terms: reflection flips several times, the wide group's (1 - cover) fill matters
    "zoom_out_reflection": dict(hw=(32, 32), clips=[_tower(32)], pad=E.PAD_REFLECTION, transforms="zoom_out"),
    "zoom_out_border": dict(hw=(32, 32), clips=[_tower(14)], pad=E.PAD_BORDER, transforms="zoom_out"),
    # a clamped drawer output with exact 0 and 1 plateaus: max-pool ties route to the first maximum, as in ATen
    "plateaus_48x40": dict(hw=(48, 40), clips=[_tower(16)], pad=E.PAD_BORDER, image="plateaus"),
}


def _zoom_out_transforms(cutn, cs, seed):
    """dst <- src homographies that shrink the source to ~0.3 about the centre, with shear and perspective terms."""
    g = np.random.default_rng(seed)
    T = np.zeros((cutn, 3, 3), dtype=np.float32)
    c = (cs - 1) / 2.0
    for n in range(cutn):
        s = g.uniform(0.28, 0.35)
        b, d = g.uniform(-0.05, 0.05, 2)
        p, q = g.uniform(-3e-4, 3e-4, 2)
        tx, ty = (1 - s) * c + g.uniform(-0.1, 0.1, 2) * cs
        T[n] = [[s, b, tx], [d, s, ty], [p, q, 1.0]]
    return T


def _plant_extremes(facs, noise):
    """plant_extremes of test_pipeline_gpu.py, for any cutn: one unmistakable maximum in cutout 0 and one minimum in
    cutout min(1, cutn - 1), so the range terms of both sides land on the same two elements."""
    facs, noise = facs.clone(), noise.clone()
    lo = min(1, facs.shape[0] - 1)
    facs[0] = facs[lo] = 0.1
    noise[0, 0, 5, 7] = 30.0
    noise[lo, 2, 100, 50] = -30.0
    return facs, noise


def _im2col(x, P):
    n, _, cs, _ = x.shape
    gp = cs // P
    return x.reshape(n, 3, gp, P, gp, P).permute(0, 2, 4, 1, 3, 5).reshape(n * gp * gp, 3 * P * P)


def _col2im(cols, n, cs, P):
    gp = cs // P
    return cols.reshape(n, gp, gp, 3, P, P).permute(0, 3, 1, 4, 2, 5).reshape(n, 3, cs, cs)


def _preprocess(x, norm):
    """CLIP_Base.preprocess (slip.py:21-60) with the tower's mean / std (R.clip_preprocess for the CLIP mean / std)."""
    if norm == CLIP_NORM:
        return R.clip_preprocess(x)
    x = x - x.min()
    mx = x.max()
    if mx != 0:
        x = x / mx
    mean = torch.tensor(norm[0], dtype=x.dtype).view(1, 3, 1, 1)
    std = torch.tensor(norm[1], dtype=x.dtype).view(1, 3, 1, 1)
    return (x - mean) / std


def _norm(c):
    return IMAGENET_NORM if c.get("tower") == E.TOWER_TIMM_VIT else CLIP_NORM


def _ulp16(x):
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -14)))
    return torch.exp2(e - 10)


def _patch_tol(x):
    """1 fp16 ulp of the float64 value, plus 2^-20 for the fp32 evaluation of ((v - min) / R - mean_c) / std_c, which
    cancels near 0 (about 1e-7 absolute in a - mean_c, over std_c >= 0.22), where the fp16 spacing is finer."""
    return _ulp16(x) + 2.0 ** -20


def _engine(hw, cs, cutn, clips, seed, aspect):
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=hw, grid=(8, 8), cutn=cutn, cut_size=cs, clip=clips, noise_fac=0.1,
                       seed=seed, cut_aspect=aspect)
    for i, c in enumerate(clips):
        sd = (S.slip_state_dict if c.get("tower") == E.TOWER_TIMM_VIT else S.clip_state_dict)(c, seed + 1 + i)
        eng.load_module(E.MOD_CLIP0 + i, sd)
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 10)
    for i in range(len(clips)):
        eng.set_prompts(i, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    return eng


def _tau(name, got, ref, M, A):
    """Smallest tau with |got - ref| <= tau M + A + 1e-6 max|ref| everywhere (inf where M = 0 and that is exceeded)."""
    floor = 1e-6 * ref.abs().max().item() + A
    excess = ((got.double() - ref).abs() - floor).clamp(min=0)
    tau = torch.where(excess > 0, excess / M, torch.zeros_like(excess)).max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"[chain] {name}: max err {err:.3e}  max|ref| {ref.abs().max().item():.3e}  measured tau {tau:.3e} (<= {TAU:g})")
    return tau


@pytest.mark.parametrize("case", sorted(CASES))
def test_cutout_chain_against_float64(case, monkeypatch):
    spec = CASES[case]
    H, W = spec["hw"]
    cs, cutn, clips = spec.get("cs", 224), spec.get("cutn", 8), spec["clips"]
    aspect = W / H if spec.get("aspect") else 1.0
    pad, fill = spec["pad"], 0.37
    seed = sorted(CASES).index(case) + 3
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(1, 3, H, W, generator=g)
    if spec.get("image") == "plateaus":
        img = (img * 1.6 - 0.3).clamp(0, 1)
        assert bool((img == 0).any()) and bool((img == 1).any())
    if spec.get("transforms") == "zoom_out":
        T = _zoom_out_transforms(cutn, cs, seed)
    else:
        T = cutouts.sample_transforms(cutn, cs, seed, aspect=aspect)
    facs, noise = _plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))

    eng = _engine((H, W), cs, cutn, clips, seed, aspect)
    eng.synth(torch.rand(1, 3, 8, 8, generator=g))
    eng.make_cutouts(img, transforms=T, zoom_padding=pad, fill=fill, noise_facs=facs.numpy(), noise=noise)
    for i in range(len(clips)):
        eng.encode_image(i)
        eng.prompt_loss(i)
    eng.backward()
    rd = lambda name, shape, dt=torch.float32: eng.debug_read(name, shape, dt).cpu()
    b_e = rd("batch", (cutn, 3, cs, cs))
    rng, ir, sums = rd("range", (4,)), rd("irange", (4,), torch.int32), rd("sums", (4,))
    gb_e, gpool_e, gimg_e = rd("g_batch", (cutn, 3, cs, cs)), rd("g_pooled", (1, 3, cs, cs)), rd("g_img", (1, 3, H, W))
    towers = []
    for i, c in enumerate(clips):
        P = c["patch"]
        K, rows = 3 * P * P, cutn * (cs // P) ** 2
        Kp = (K + 63) // 64 * 64
        towers.append((P, K, _norm(c), rd(f"clip{i}.patches", (rows, Kp), torch.float16),
                       rd(f"clip{i}.g_patches", (rows, Kp), torch.float16)))
    eng.close()

    # range / irange: exact on the engine's batch
    bd = b_e.double()
    mn, mx = bd.min().item(), bd.max().item()
    Rf = float(np.float32(mx - mn))
    assert rng.tolist() == [np.float32(mn), Rf, np.float32(mx), 1.0]
    assert ir[:2].tolist() == [int(bd.reshape(-1).argmin()), int(bd.reshape(-1).argmax())]

    # the float64 reference chain; R.make_cutouts pools internally: keep that tensor to differentiate to it
    kept = {}
    pool = R.pool_avg_max
    monkeypatch.setattr(R, "pool_avg_max", lambda x, s: kept.setdefault("pooled", pool(x, s)))
    img64 = img.double().requires_grad_(True)
    batch_r = R.make_cutouts(img64, torch.from_numpy(T).double(), cs, PAD_NAMES[pad], fill, facs.double(), noise.double(),
                             aspect=aspect)
    pooled = kept["pooled"]
    flat_r = batch_r.detach().reshape(-1)
    assert ir[:2].tolist() == [int(flat_r.argmin()), int(flat_r.argmax())], "irange against the float64 batch"
    print(f"[chain] {case}: batch max err {(bd - batch_r.detach()).abs().max().item():.3e}")

    L = 0.0
    ref_gb = torch.zeros_like(bd)
    for P, K, norm, pt, gp in towers:
        # patches: 1 fp16 ulp of the float64 preprocess of the engine's batch; pad columns exactly 0
        std = torch.tensor(norm[1], dtype=torch.float64).view(1, 3, 1, 1)
        pre = _im2col(((bd - mn) / Rf - torch.tensor(norm[0], dtype=torch.float64).view(1, 3, 1, 1)) / std, P)
        err_p = (pt[:, :K].double() - pre).abs() / _patch_tol(pre)
        print(f"[chain] {case}: P={P} patches err / (fp16 ulp + 2^-20) {err_p.max().item():.3f} (<= 1)")
        assert bool((err_p <= 1).all())
        assert bool((pt[:, K:] == 0).all())
        up = gp[:, :K].double()
        L = L + (_im2col(_preprocess(batch_r, norm), P) * up).sum()
        ref_gb += _col2im(up, cutn, cs, P) / (std * Rf)

    # g_batch, the direct term of every tower
    e_gb = (gb_e.double() - ref_gb).abs().max().item()
    print(f"[chain] {case}: g_batch err {e_gb / ref_gb.abs().max().item():.3e} of max (<= 2e-6)")
    assert e_gb <= 2e-6 * ref_gb.abs().max().item()

    # the two range sums
    a = (bd - mn) / Rf
    t1, t2 = ref_gb, ref_gb * a
    for k, t in enumerate((t1, t2)):
        e_s = abs(sums[k].item() - t.sum().item())
        print(f"[chain] {case}: sums[{k}] err {e_s / t.abs().sum().item():.3e} of sum|terms| (<= {SUMS_REL:g})")
        assert e_s <= SUMS_REL * t.abs().sum().item()

    # g_pooled and g_img
    g_img_r, g_pool_r, g_batch_r = torch.autograd.grad(L, (img64, pooled, batch_r), retain_graph=True)
    M_img, M_pool = torch.autograd.grad((batch_r * g_batch_r.abs()).sum(), (img64, pooled), retain_graph=True)
    # the rounding of the two sums reaches the image only through the range terms at the two extreme elements
    sums_err = torch.zeros_like(g_batch_r).reshape(-1)
    sums_err[int(ir[0])] = SUMS_REL * (t1.abs().sum() + t2.abs().sum())      # d/dmin = -(sum g + d/dR)
    sums_err[int(ir[1])] = SUMS_REL * t2.abs().sum()                          # d/dR = -sum g (a - min) / R
    A_img, A_pool = torch.autograd.grad((batch_r * sums_err.reshape(batch_r.shape)).sum(), (img64, pooled))
    tau_pool = _tau(f"{case} g_pooled", gpool_e, g_pool_r, M_pool, A_pool)
    tau_img = _tau(f"{case} g_img", gimg_e, g_img_r, M_img, A_img)
    assert tau_pool <= TAU and tau_img <= TAU


def test_caller_batch_range_takes_the_lowest_tied_index():
    """encode_image(0, batch=...) recomputes the range of a caller's batch with minmax_partials + minmax_reduce.  Exact
    ties of the minimum and of the maximum, spread over different partial blocks (block (i // 256) % nparts of the
    grid-stride loop, nparts = 392 here) with the lowest index in a higher block than the others: the range is exact and
    irange holds the lowest tied index of each, the order minmax_reduce_kernel promises."""
    cutn, cs = 8, 224
    clips = [_tower(32)]
    eng = _engine((32, 32), cs, cutn, clips, 21, 1.0)
    g = torch.Generator().manual_seed(22)
    batch = torch.rand(cutn, 3, cs, cs, generator=g) * 0.8 + 0.1
    ties_min = [90_000, 100_500, 1_100_000, 90_000 + 392 * 256]
    ties_max = [99_000, 102_400, 1_003_520, 99_001]
    nparts = cutn * ((cs * cs // 4 + 255) // 256)
    print("[chain] min ties in blocks", [(i // 256) % nparts for i in ties_min], "max ties in blocks",
          [(i // 256) % nparts for i in ties_max])
    flat = batch.reshape(-1)
    flat[ties_min] = -0.25
    flat[ties_max] = 1.5
    eng.encode_image(0, batch=batch)
    rng = eng.debug_read("range", (4,)).cpu()
    ir = eng.debug_read("irange", (4,), torch.int32).cpu()
    pt = eng.debug_read("clip0.patches", (cutn * 49, 3072), torch.float16).cpu()
    eng.close()
    assert rng.tolist() == [-0.25, float(np.float32(1.5) - np.float32(-0.25)), 1.5, 1.0]
    assert ir[:2].tolist() == [min(ties_min), min(ties_max)]
    pre = _im2col(((batch.double() + 0.25) / 1.75 - torch.tensor(R.CLIP_MEAN, dtype=torch.float64).view(1, 3, 1, 1))
                  / torch.tensor(R.CLIP_STD, dtype=torch.float64).view(1, 3, 1, 1), 32)
    assert bool(((pt.double() - pre).abs() <= _patch_tol(pre)).all())
