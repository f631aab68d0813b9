"""The FFT drawer (kernels_fft.cu, Engine::build_fft; FftDrawer.synth, fftdrawer.py:78-84) against float64, forward and
backward, on its own: image = sigmoid(M (irfft2(scale * z, ortho) * contrast / std)).

Each case runs one engine iteration (synth -> make_cutouts -> encode_image -> prompt_loss -> backward, a tiny ViT) and
reads img_pre (the unnormalised cuFFT C2R output x), img, g_img and z_grad.  What is compared, and how tightly:

  x / sqrt(HW)  against float64 irfftn(scale * z, norm="ortho"): cuFFT and the scale grid alone,
                <= X_TOL of max|ref|
  img           against float64 R.fft_synth (scale grid, std, colour matrix, sigmoid), <= IMG_TOL absolute
  z_grad        against the float64 gradient of <fft_synth(z), g_img / S> at the engine's own g_img (S = 4096, the
                engine's gradient scale), which takes the ViT out of the comparison.  The sigmoid's derivative is
                s (1 - s) of the engine's fp32 img, as torch's sigmoid backward forms it from its stored fp32 output: where
                the image saturates, fp32 1 - s keeps few digits, and that rounding belongs to the image, not to the
                kernels.  Both gradients are divided by the per-frequency factor scale * c_kx (c = 1 on the DC and Nyquist
                columns, 2 inside) and compared to G_TOL of their maximum separately over the DC column, the Nyquist
                column and the interior columns, so a wrong factor on an edge column is a 100 % error.

Spectra: the seeded N(0, 0.01^2) initialisation (fft_image(sd=0.01), fftdrawer.py:57); the same with a DC term 100x the
rest, so mean >> std and the unbiased variance and the mean-subtracted std term of the backward carry the result; one
that is non-zero only in the kx = 0 and Nyquist columns, with ky and H - ky not conjugate.  A random spectrum is not
Hermitian in those two columns, so every spectrum here depends on how the C2R transform projects them: the reference is
also evaluated with float64 torch.fft.irfftn on CUDA (what pixray runs, on cuFFT), and the CUDA result is the one
compared when the two differ; each case prints the CPU / CUDA difference.

Every bound is about 3x the largest value measured over the cases (each case prints its own).  Measured on an H100
(80 GB HBM3, 700 W): x 3.7e-7 of max (576x1024, DC-heavy); img 5.5e-7 (576x1024, DC-heavy), <= 2.5e-7 at the other
shapes; spectrum gradient 2.8e-6 of max (64x2, DC-heavy: mean / std = 32 there, and the fp32 x - mean of the std term
cancels that much), <= 1.1e-6 in every other case.  The float64 irfftn on the CPU and on CUDA agreed to 1.1e-15 of max
on every spectrum here.
"""
import math

import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu

GS = 4096.0  # the engine's gradient scale: g_img holds GS * dL/dimg
CUTN, CS = 4, 224
TOWER = dict(width=128, layers=1, heads=2, patch=32, image_res=CS, out_dim=64)

X_TOL = 1.1e-6
IMG_TOL = 1.6e-6
G_TOL = 8e-6

CASES = {
    "64x64": dict(hw=(64, 64)),
    # fy comes from H and fx from W
    "48x80": dict(hw=(48, 80)),
    "80x48": dict(hw=(80, 48)),
    # odd H: fftfreq splits the positive and negative frequencies at (H + 1) / 2
    "45x64": dict(hw=(45, 64)),
    # W2 = 2: every column is a DC or a Nyquist column
    "64x2": dict(hw=(64, 2)),
    # past the 1184-block cap of the grid-stride loops; the 296-block moment and A reductions
    "512x512": dict(hw=(512, 512)),
    "576x1024": dict(hw=(576, 1024)),
    "64x64_decay0.5": dict(hw=(64, 64), decay=0.5),
    "48x80_decay1.5": dict(hw=(48, 80), decay=1.5),
    "64x64_decay3": dict(hw=(64, 64), decay=3.0),
}
SPECTRA = ("init", "dc_heavy", "edge_columns")


def _spectrum(kind, H, W, g):
    W2 = W // 2 + 1
    z = torch.randn(1, 3, H, W2, 2, generator=g) * 0.01
    if kind == "dc_heavy":
        z[0, :, 0, 0, 0] = 1.0
    elif kind == "edge_columns":
        keep = torch.zeros(W2, dtype=torch.bool)
        keep[0] = keep[W2 - 1] = True
        z = z * keep.view(1, 1, 1, W2, 1)
    return z.contiguous()


def _engine(hw, decay, seed):
    eng = E.B200Engine(drawer=E.DRAWER_FFT, image_hw=hw, cutn=CUTN, cut_size=CS, clip=[TOWER], noise_fac=0.1, seed=seed,
                       fft_decay=decay)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(TOWER, seed + 1))
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    return eng


def _run(eng, z, H, W):
    """One engine iteration; returns (img_pre, img, g_img, z_grad) on the CPU."""
    eng.synth(z)
    eng.make_cutouts(use_engine_rng=True)
    eng.encode_image(0)
    eng.prompt_loss(0)
    eng.backward()
    rd = lambda name, shape: eng.debug_read(name, shape).cpu()
    return (rd("img_pre", (1, 3, H, W)), rd("img", (1, 3, H, W)), rd("g_img", (1, 3, H, W)),
            rd("z_grad", tuple(z.shape)))


def _irfft(z64, decay):
    _, _, H, W2, _ = z64.shape
    W = (W2 - 1) * 2
    scale = R.fft_freq_scale(H, W, decay, torch.float64).to(z64.device)
    return torch.fft.irfftn(torch.view_as_complex((scale[None, None, :, :, None] * z64).contiguous()), s=(H, W),
                            norm="ortho")


def _pre_sigmoid(z64, decay):
    """R.fft_synth before its sigmoid, on the spectrum's device."""
    x = _irfft(z64, decay)
    y = x * 0.9 / x.std()
    m = R.color_matrix(1.5, torch.float64).to(z64.device)
    return torch.matmul(y.permute(0, 2, 3, 1), m.T).permute(0, 3, 1, 2)


def _column_errors(got, ref, H, W, decay):
    """max |got - ref| / max |ref| over the DC column, the Nyquist column and the interior columns, after dividing both
    by scale * c_kx."""
    W2 = W // 2 + 1
    c = torch.full((W2,), 2.0, dtype=torch.float64)
    c[0] = c[W2 - 1] = 1.0
    f = (R.fft_freq_scale(H, W, decay, torch.float64) * c).view(1, 1, H, W2, 1)
    a, b = got.double() / f, ref / f
    groups = {"dc": [0], "nyquist": [W2 - 1], "interior": list(range(1, W2 - 1))}
    out = {}
    for name, cols in groups.items():
        if not cols:
            continue
        ga, gb = a[:, :, :, cols], b[:, :, :, cols]
        out[name] = ((ga - gb).abs().max() / gb.abs().max()).item()
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_fft_drawer_against_float64(case):
    spec = CASES[case]
    H, W = spec["hw"]
    decay = spec.get("decay", 0.0)
    d = decay if decay > 0 else 1.5
    seed = list(CASES).index(case) + 60
    eng = _engine((H, W), decay, seed)
    g = torch.Generator().manual_seed(seed + 3)
    worst = dict(x=0.0, img=0.0, grad=0.0)
    try:
        for kind in SPECTRA:
            z = _spectrum(kind, H, W, g)
            x_e, img_e, gimg_e, zg_e = _run(eng, z, H, W)

            # forward: cuFFT + the scale grid, then the whole synth, against float64 on the CPU and on CUDA
            z64 = z.double()
            x_cpu, x_gpu = _irfft(z64, d), _irfft(z64.cuda(), d).cpu()
            dev = (x_cpu - x_gpu).abs().max().item() / x_gpu.abs().max().item()
            x_ref = x_gpu
            e_x = (x_e.double() / math.sqrt(H * W) - x_ref).abs().max().item() / x_ref.abs().max().item()
            img_ref = R.fft_synth(z64.cuda(), d).cpu()
            e_img = (img_e.double() - img_ref).abs().max().item()

            # backward at the engine's g_img, with the engine's sigmoid output in the derivative
            z64g = z64.cuda().requires_grad_(True)
            t = _pre_sigmoid(z64g, d)
            s = img_e.double().cuda()
            (zg_ref,) = torch.autograd.grad(t, z64g, grad_outputs=gimg_e.double().cuda() * s * (1 - s) / GS)
            errs = _column_errors(zg_e, zg_ref.cpu(), H, W, d)
            e_g = max(errs.values())
            print(f"[fft] {case} {kind}: x err {e_x:.3e} of max (<= {X_TOL:g}); img err {e_img:.3e} (<= {IMG_TOL:g}); "
                  f"grad err of max " + ", ".join(f"{k} {v:.3e}" for k, v in errs.items()) + f" (<= {G_TOL:g}); "
                  f"irfftn CPU vs CUDA {dev:.3e} of max")
            worst = dict(x=max(worst["x"], e_x), img=max(worst["img"], e_img), grad=max(worst["grad"], e_g))
    finally:
        eng.close()
    assert worst["x"] <= X_TOL and worst["img"] <= IMG_TOL and worst["grad"] <= G_TOL, worst


def test_fft_drawer_runs_are_bit_identical():
    """Two identical iterations: the moment and A reductions run in a fixed order and nothing else accumulates, so img and
    z_grad are bit-identical (on the 296-block reductions' largest case here)."""
    H, W = 576, 1024
    eng = _engine((H, W), 0.0, 90)
    try:
        z = _spectrum("init", H, W, torch.Generator().manual_seed(91))
        a = _run(eng, z, H, W)
        b = _run(eng, z, H, W)
    finally:
        eng.close()
    assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])


def test_fft_drawer_refuses_an_odd_width():
    """pixray accepts an odd width; the engine's C2R / R2C pair assumes a Nyquist column and refuses it."""
    eng = E.B200Engine(drawer=E.DRAWER_FFT, image_hw=(64, 63), cutn=CUTN, cut_size=CS, clip=[TOWER], seed=1)
    try:
        with pytest.raises(E.EngineError, match="fft drawer needs an even canvas width"):
            eng.finalize()
    finally:
        eng.close()
