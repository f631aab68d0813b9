"""K.ColorJitter stage of MakeCutouts (pixray.py:416, 436).

CPU part: the per-pixel body the cutout kernels run (csrc/color_jitter.cuh, host+device code, evaluated on the host through
the pxr_test_color_jitter_host hook) against the oracle's restatement of kornia 0.6.2 -- forward and the
vector-Jacobian product -- plus the host samplers.  GPU part: the kernels themselves, through pxr_make_cutouts /
pxr_iterate, against oracle.make_cutouts / oracle.iterate."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import _lib, cutouts

E_PAD_BORDER = 1


def _host_jitter(rgb, code, sat, hue, g_out=None):
    lib = _lib.load()
    rgb = np.ascontiguousarray(rgb, dtype=np.float32)
    out = np.zeros_like(rgb)
    g_in = np.zeros_like(rgb)
    g = None if g_out is None else np.ascontiguousarray(g_out, dtype=np.float32)
    f = lib.pxr_test_color_jitter_host
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = f(rgb.ctypes.data, rgb.shape[0], int(code), float(sat), float(hue), None if g is None else g.ctypes.data,
           out.ctypes.data, g_in.ctypes.data)
    assert rc == 0
    return out, g_in


def _oracle_jitter(rgb, code, sat, hue, g_out=None):
    x = torch.from_numpy(rgb).t().reshape(1, 3, 1, -1).clone().requires_grad_(True)  # [1,3,1,n]
    j = torch.tensor([[float(code), sat, hue]], dtype=torch.float32)
    y = R.color_jitter(x, j)
    g_in = None
    if g_out is not None:
        y.backward(torch.from_numpy(g_out).t().reshape(1, 3, 1, -1))
        g_in = x.grad.reshape(3, -1).t().numpy()
    return y.detach().reshape(3, -1).t().numpy(), g_in


def _colours(n, seed):
    g = np.random.default_rng(seed)
    rgb = g.uniform(0, 1, (n, 3)).astype(np.float32)
    rgb[:8] = [[0, 0, 0], [1, 1, 1], [0.5, 0.5, 0.5], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0.25, 0.25, 0.75], [0.9, 0.2, 0.9]]
    return rgb


def test_pixel_body_matches_the_oracle_for_every_order():
    rgb = _colours(4096, 0)
    g = np.random.default_rng(1).standard_normal(rgb.shape).astype(np.float32)
    worst_f = worst_g = 0.0
    for k, order in enumerate(itertools.permutations(range(4))):
        code = cutouts.jitter_code(list(order))
        assert code == R.jitter_code(list(order))
        sat = 0.9 + 0.2 * ((k * 7) % 24) / 23.0
        hue = -0.1 + 0.2 * ((k * 5) % 24) / 23.0
        out, g_in = _host_jitter(rgb, code, sat, hue, g)
        ref, ref_g = _oracle_jitter(rgb, code, sat, hue, g)
        worst_f = max(worst_f, float(np.abs(out - ref).max()))
        # the Jacobian is piecewise: compare where neither side sits on a sector / clamp boundary (rounding may pick the
        # other piece there); those are a vanishing fraction of random colours
        err = np.abs(g_in - ref_g).max(axis=1)
        tol = 2e-3 * (1.0 + np.abs(ref_g).max(axis=1))
        assert (err > tol).mean() < 2e-3, (order, float((err > tol).mean()))
        worst_g = max(worst_g, float(np.median(err)))
    assert worst_f <= 2e-6, worst_f
    assert worst_g <= 1e-5, worst_g


def test_pixel_body_at_exact_channel_ties():
    """Clamped images are full of exact ties (white, black, grey, two saturated channels): there the Jacobian is one-sided
    and must follow torch's choice (first arg-max / arg-min channel, zero hue gradient at delta == 0, closed clamp)."""
    g = np.random.default_rng(0)
    n = 1000
    a, b = g.uniform(0, 1, n).astype(np.float32), g.uniform(0, 1, n).astype(np.float32)
    hi, lo, one, zero = np.maximum(a, b), np.minimum(a, b), np.ones(n, np.float32), np.zeros(n, np.float32)
    cases = {"grey": [a, a, a], "white": [one, one, one], "black": [zero, zero, zero], "max tie rg": [hi, hi, lo],
             "max tie gb": [lo, hi, hi], "max tie rb": [hi, lo, hi], "min tie rg": [lo, lo, hi], "min tie gb": [hi, lo, lo],
             "r=1": [one, a, b], "b=0": [a, b, zero], "r=g=1": [one, one, b], "g=b=0": [a, zero, zero]}
    go = g.standard_normal((n, 3)).astype(np.float32)
    for name, cols in cases.items():
        rgb = np.stack(cols, 1)
        for order in ([2, 3, 0, 1], [3, 2, 1, 0], [0, 2, 1, 3]):
            code = cutouts.jitter_code(order)
            out, g_in = _host_jitter(rgb, code, 1.07, -0.083, go)
            ref, ref_g = _oracle_jitter(rgb, code, 1.07, -0.083, go)
            assert np.abs(out - ref).max() <= 2e-6, (name, order)
            assert np.abs(g_in - ref_g).max() <= 2e-5, (name, order, float(np.abs(g_in - ref_g).max()))


def test_backward_algorithm_of_the_cutout_kernel_equals_autograd():
    """What cutout_bwd does with the stage on -- recompute the warped colour, push the incoming gradient through the pixel
    body's VJP, then through the warp's adjoint -- against autograd through the oracle's whole jittered make_cutouts."""
    torch.manual_seed(0)
    cutn, cs = 5, 40
    img = torch.rand(1, 3, 16, 16)
    img[:, :, :4] = 1.0                      # a saturated band: exact ties inside, kinks at its border
    img[:, 1:, 12:] = 0.0
    img.requires_grad_(True)
    T = torch.eye(3).repeat(cutn, 1, 1)
    T[:, 0, 0] = torch.tensor([1.3, 1.1, 1.5, 0.9, 0.8])
    T[:, 1, 1] = torch.tensor([1.2, 1.4, 1.1, 0.9, 0.85])
    T[:, 0, 2] = torch.tensor([-3.0, 1.5, -6.0, 1.0, 2.0])
    J = torch.from_numpy(cutouts.sample_color_jitter(cutn, 3, p=1.0))
    J[2, 0] = 0
    facs, noise = torch.rand(cutn) * 0.1, torch.randn(cutn, 3, cs, cs)
    full = R.make_cutouts(img, T, cs, "reflection", 0.4, facs, noise, jitter=J)
    g_out = torch.randn_like(full)
    want, = torch.autograd.grad(full, img, g_out, retain_graph=True)
    pre = R.make_cutouts(img, T, cs, "reflection", 0.4)                      # the warp alone
    g_pre = torch.zeros_like(pre)
    for n in range(cutn):
        rgb = pre[n].detach().reshape(3, -1).t().contiguous().numpy()
        go = g_out[n].reshape(3, -1).t().contiguous().numpy()
        out, gi = _host_jitter(rgb, int(J[n, 0]), float(J[n, 1]), float(J[n, 2]), go)
        g_pre[n] = torch.from_numpy(gi).t().reshape(3, cs, cs)
        got_fwd = torch.from_numpy(out).t().reshape(3, cs, cs) + facs[n] * noise[n]
        assert (got_fwd - full[n].detach()).abs().max() <= 2e-6
    got, = torch.autograd.grad(pre, img, g_pre)
    assert (got - want).abs().max() <= 2e-5 * want.abs().max()


def test_oracle_hsv_maps_agree_with_opencv_and_colorsys():
    """kornia itself is not installable here, so the oracle's rgb<->hsv restatement cannot be pinned to it; it is
    cross-checked against two independent implementations of the same published transform instead (OpenCV's float
    RGB2HSV / HSV2RGB, H in degrees; the standard library's colorsys, h in turns)."""
    import colorsys
    import math
    cv2 = pytest.importorskip("cv2")
    rgb = _colours(4096, 5)
    hsv = R.rgb_to_hsv(torch.from_numpy(rgb).t().reshape(1, 3, 1, -1)).reshape(3, -1).t().numpy()
    ref = cv2.cvtColor(rgb.reshape(1, -1, 3), cv2.COLOR_RGB2HSV).reshape(-1, 3)
    dh = np.abs(hsv[:, 0] - np.deg2rad(ref[:, 0]))
    dh = np.minimum(dh, 2 * math.pi - dh)
    sat = ref[:, 1] > 1e-3                                            # hue is arbitrary at zero saturation
    assert dh[sat].max() < 2e-4 and np.abs(hsv[:, 1] - ref[:, 1]).max() < 1e-5 and np.abs(hsv[:, 2] - ref[:, 2]).max() < 1e-7
    for i in range(0, 4096, 97):
        h, s_, v = colorsys.rgb_to_hsv(*[float(c) for c in rgb[i]])
        d = abs(hsv[i, 0] / (2 * math.pi) - h)
        assert (min(d, 1 - d) < 1e-5 or s_ < 1e-3) and abs(hsv[i, 1] - s_) < 1e-5 and abs(hsv[i, 2] - v) < 1e-6
    # and back: hue shifted by a fixed angle, saturation scaled, through the oracle vs through OpenCV
    shifted = ref.copy()
    shifted[:, 0] = np.mod(shifted[:, 0] + 25.0, 360.0)
    shifted[:, 1] = np.clip(shifted[:, 1] * 1.07, 0, 1)
    want = cv2.cvtColor(shifted.reshape(1, -1, 3), cv2.COLOR_HSV2RGB).reshape(-1, 3)
    t = torch.from_numpy(hsv.copy())
    t[:, 0] = torch.fmod(t[:, 0] + math.radians(25.0), 2 * math.pi)
    t[:, 1] = torch.clamp(t[:, 1] * 1.07, 0, 1)
    got = R.hsv_to_rgb(t.t().reshape(1, 3, 1, -1)).reshape(3, -1).t().numpy()
    assert np.abs(got - want).max() < 2e-5


def test_not_selected_cutouts_pass_through():
    rgb = _colours(256, 2)
    g = np.ones_like(rgb)
    out, g_in = _host_jitter(rgb, 0, 1.1, 0.1, g)
    assert np.array_equal(out, rgb) and np.array_equal(g_in, g)
    # identity parameters reproduce the colour up to the hsv round trip
    out, _ = _host_jitter(rgb, cutouts.jitter_code([0, 1, 2, 3]), 1.0, 0.0)
    assert np.abs(out - rgb).max() <= 1e-6


def test_host_sampler_distribution():
    js = np.concatenate([cutouts.sample_color_jitter(64, s) for s in range(200)])
    applied = js[:, 0] != 0
    assert abs(applied.mean() - 0.8) < 0.02                              # Bernoulli(0.8)
    assert js[:, 1].min() >= 0.9 and js[:, 1].max() <= 1.1 and abs(js[:, 1].mean() - 1.0) < 5e-3
    assert js[:, 2].min() >= -0.1 and js[:, 2].max() <= 0.1 and abs(js[:, 2].mean()) < 5e-3
    one = cutouts.sample_color_jitter(64, 7)
    zoom = int(0.6 * 64)
    for grp in (one[:zoom], one[zoom:]):                                  # one order per stack
        codes = set(grp[grp[:, 0] != 0, 0].astype(int).tolist())
        assert len(codes) == 1
        c = codes.pop() - 256
        assert sorted((c >> (2 * k)) & 3 for k in range(4)) == [0, 1, 2, 3]


# ------------------------------------------------------------------------------------------------ GPU: the kernels
@pytest.mark.gpu
def test_cutout_kernels_apply_color_jitter_like_the_oracle():
    import test_pipeline_gpu as P
    cutn, cs = 8, 224
    vq, clip, eng, prompts, z = P.build(cutn=cutn)
    torch.manual_seed(5)
    img = torch.rand(1, 3, 32, 32)
    T = torch.from_numpy(P.random_transforms(cutn, cs, 11))
    J = cutouts.sample_color_jitter(cutn, 12, p=1.0)
    J[0, 0] = 0                                   # one cutout the Bernoulli missed
    J[1, 0] = cutouts.jitter_code([3, 0, 2, 1])   # and a different order in the same batch
    facs = torch.rand(cutn) * 0.1
    noise = torch.randn(cutn, 3, cs, cs)
    for pad_name, pad in (("reflection", 0), ("border", 1)):
        got = eng.make_cutouts(img, transforms=T.numpy(), zoom_padding=pad, fill=0.4, noise_facs=facs.numpy(),
                               noise=noise, color_jitter=J).cpu()
        want = R.make_cutouts(img, T, cs, pad_name, 0.4, facs, noise, jitter=torch.from_numpy(J))
        plain = R.make_cutouts(img, T, cs, pad_name, 0.4, facs, noise)
        assert (want - plain).abs().max() > 1e-2                           # the stage does something
        err = (got - want).abs()
        frac = float((err > 1e-4).float().mean())
        print(f"[parity] jittered cutouts ({pad_name}): max_abs_err={float(err.max()):.3e}  frac>1e-4={frac:.2e}")
        # hue sectors are decided on fp32 values that differ in the last bits between the two bilinear samplers; the
        # map is continuous across sectors, so the error stays small
        assert err.max() <= 1e-3 and frac < 1e-4
        assert (got[0] - plain[0]).abs().max() <= 1e-4                     # code 0 passes through


@pytest.mark.gpu
def test_iteration_gradient_with_color_jitter():
    """The backward through the stage.  rgb->hsv->rgb is continuous but its Jacobian is piecewise (arg-max / arg-min
    channel, hue sector, the saturation clamp).  The device body uses exactly-rounded fp32 operations, so it lands on the
    same piece as the oracle whenever it sees the same colour (test_zz_host_paths: device vs host body, 0 pixels off-piece;
    round 1's 2.5e-2 gap was __fdividef / FMA contraction flipping the sector at saturated-channel ties, see
    tests/diag_color_jitter.py).
      (a) decisive: the ORACLE's image goes into the engine's cutouts -> the jittered batch matches to 2e-4 and d loss / d
          image to 5e-3 of max (measured 1.6e-3, the level of the un-jittered path);
      (b) whole chain from z: the engine's fp16 decoder image differs from the oracle's by ~1e-3 before the clamp, which
          moves a few pixels across a piece boundary on either side.  The CPU oracle's own z.grad moves by 2.7e-2..3.3e-2 of
          its maximum under a perturbation of that size (0.1e-2..1.2e-2 without the stage), so the bound is 4e-2 of
          max|z.grad| (measured 2.96e-2) with cosine >= 0.995."""
    import test_pipeline_gpu as P
    cutn, cs = 8, 224
    vq, clip, eng, prompts, z = P.build(cutn=cutn, seed=3)
    T = P.random_transforms(cutn, cs, 13)
    J = cutouts.sample_color_jitter(cutn, 22, p=1.0)
    g = torch.Generator().manual_seed(19)
    facs, noise = P.plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    ref = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z, [clip], [prompts], torch.from_numpy(T), cs, "border", 0.3,
                    facs, noise, jitter=torch.from_numpy(J))
    ref_plain = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z, [clip], [prompts], torch.from_numpy(T), cs, "border",
                          0.3, facs, noise)
    # the stage must matter for the gradient, or the comparison proves nothing
    assert (ref["z_grad"] - ref_plain["z_grad"]).abs().max() > 0.05 * ref["z_grad"].abs().max()

    # (a) oracle image in
    img_r = ref["image"].clone().requires_grad_(True)
    batch_r = R.make_cutouts(img_r, torch.from_numpy(T), cs, "border", 0.3, facs, noise, jitter=torch.from_numpy(J))
    batch_r.retain_grad()
    emb = R.encode_image(clip, batch_r).float()
    sum(R.prompt_loss(emb, *p) for p in prompts).backward()
    eng.synth(z)
    batch = eng.make_cutouts(ref["image"], transforms=T, zoom_padding=E_PAD_BORDER, fill=0.3, noise_facs=facs.numpy(),
                             noise=noise, color_jitter=J)
    e_b, _ = P.report("jittered batch (oracle image in)", batch, batch_r.detach())
    eng.encode_image(0)
    eng.prompt_loss(0)
    eng.backward()
    S = 4096.0
    g_img = eng.debug_read("g_img", (1, 3, 32, 32)) / S
    e_gi, m_gi = P.report("d/d image through ColorJitter (oracle image in)", g_img, img_r.grad)
    assert e_b <= 2e-4
    assert e_gi <= 5e-3 * m_gi  # measured 1.6e-3

    # (b) the engine's own chain
    eng.synth(z)
    batch = eng.make_cutouts(None, transforms=T, zoom_padding=E_PAD_BORDER, fill=0.3, noise_facs=facs.numpy(),
                             noise=noise, color_jitter=J)
    P.report("jittered batch (engine image in)", batch, ref["batch"])
    eng.encode_image(0)
    losses = eng.prompt_loss(0)
    e_l, _ = P.report("prompt losses", losses, torch.stack([l.reshape(()) for l in ref["losses"]]))
    zg = eng.backward()
    e_g, m_g = P.report("z.grad with ColorJitter", zg, ref["z_grad"])
    cos = torch.nn.functional.cosine_similarity(zg.cpu().reshape(-1), ref["z_grad"].reshape(-1), dim=0).item()
    print(f"[parity] z.grad cosine {cos:.5f}")
    assert e_l < 2e-3
    assert e_g <= 4e-2 * m_g and cos >= 0.995
