"""The Prompt loss kernel (prompt_loss_kernel, kernels_clip.cu; Prompt.forward, pixray.py:275-280) against float64 autograd of
the oracle's R.prompt_loss, through the pxr_test_prompt_loss hook and once through the engine.

The kernel normalises each embedding (slip.py:66), measures the spherical distance to every prompt row, sums
|w| dist / (cutn rows of the Prompt) into the row's loss slot, and takes the gradient back through the
normalisation, keeping it only where dist > stop (replace_grad(dists, maximum(dists, stop)), pixray.py:280).  The loss
terms are summed over the rows in a fixed order (the last block adds them up), so repeated calls give the same bits.  The
reference is sum over the loss slots of R.prompt_loss(e, rows of the slot, w, stop) * B / cutn_global (a shard of B of the
cutn_global cutouts: the Prompt's mean runs over all cutouts), and the gradient is grad_scale times its autograd.

Bounds (fp32 kernel against float64):
  e_unit  <= 1e-6 absolute
  losses  <= 1e-5 of the slot's sum of |w dist| / rows; bit-identical between two calls
  de      <= 1e-5 of the row's largest |de| + 1e-7 of the largest |de| of the call, elementwise.  Rows with r / 2 = 1 - 1e-4
             (nearly antipodal to the prompt) have their own bound, 3e-4 of the row's largest |de|: the derivative
             2 asin(r/2) / sqrt(1 - r^2 / 4) there amplifies the fp32 rounding of r through the cancellation in
             1 - r^2 / 4 = 2e-4 (up to about 1e-3 of the gradient in the worst case; 8.5e-5 measured on an H100).
  de16    bit-equal to de.half()
  the pass / stop mask of every row exactly (a stopped row of a one-prompt call has de == 0 exactly).
Measured on an H100 (80 GB HBM3, 700 W) over these cases: e_unit 4e-8, losses 1.5e-6, de 7.6e-7 of the row maximum.

Out of scope: dist == stop exactly (torch.maximum splits the gradient in halves there; the kernel does not), so every stop
here keeps at least 1e-4 from every distance.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ref_path as R
from pixray_b200 import _lib

pytestmark = pytest.mark.gpu

NEG_INF = float("-inf")
ANTIPODAL_BOUND = 3e-4


def _kernel(e, prompts, weights, stops, slots, inv_rows, cutn_global, grad_scale, n_slots):
    """Runs pxr_test_prompt_loss; returns (e_unit, losses, de, de16) on the CPU."""
    lib = _lib.load()
    f = lib.pxr_test_prompt_loss
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                  C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    B, D = e.shape
    n = prompts.shape[0]
    dev = lambda t, dt=torch.float32: t.to("cuda", dt).contiguous()
    e_d, p_d, w_d, s_d = dev(e), dev(prompts), dev(weights), dev(stops)
    slot_d, inv_d = dev(slots, torch.int32), dev(inv_rows)
    e_unit = torch.full((B, D), float("nan"), device="cuda")
    losses = torch.zeros(max(n_slots, 1), device="cuda")
    de = torch.full((B, D), float("nan"), device="cuda")
    de16 = torch.full((B, D), float("nan"), device="cuda", dtype=torch.float16)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    torch.cuda.synchronize()
    rc = f(ptr(e_d), B, D, ptr(p_d), ptr(w_d), ptr(s_d), ptr(slot_d), ptr(inv_d), n, cutn_global, grad_scale, ptr(e_unit),
           ptr(losses), ptr(de), ptr(de16))
    assert rc == 0
    return e_unit.cpu(), losses.cpu()[:n_slots], de.cpu(), de16.cpu()


def _reference(e, prompts, weights, stops, slots, cutn_global, grad_scale, n_slots):
    """float64: (e_unit, losses, de, loss scale per slot = sum |w dist| / rows / cutn_global, signed dists [B, n])."""
    B = e.shape[0]
    e64 = e.double().requires_grad_(True)
    p64 = prompts.double()
    losses, scale = [], []
    for s in range(n_slots):
        rows = [j for j in range(prompts.shape[0]) if int(slots[j]) == s]
        w, stop = float(weights[rows[0]]), float(stops[rows[0]])
        assert all(float(weights[j]) == w and float(stops[j]) == stop for j in rows), "one weight and stop per Prompt"
        losses.append(R.prompt_loss(e64, p64[rows], w, stop) * B / cutn_global)
        d = R.spherical_dist_loss(e64.detach().unsqueeze(1), p64[rows].unsqueeze(0))
        scale.append(abs(w) * d.sum().item() / len(rows) / cutn_global)
    total = torch.stack([l.reshape(()) for l in losses]).sum()
    (de,) = torch.autograd.grad(total * grad_scale, e64)
    en = F.normalize(e64.detach(), dim=1)
    pn = F.normalize(p64, dim=1)
    r = (en.unsqueeze(1) - pn.unsqueeze(0)).norm(dim=2)
    dists = 2 * torch.asin(r / 2) ** 2 * torch.sign(weights.double()).unsqueeze(0)
    return en, torch.stack([l.detach().reshape(()) for l in losses]), de, torch.tensor(scale), dists


def _compare(name, got, ref, antipodal_rows=(), zero_rows=()):
    """The bounds of the module docstring; returns the measured (e_unit, losses, de) errors.  zero_rows: rows along a
    prompt's direction (r ~ 0), whose true gradient is 0 and whose computed one is rounding noise: they are held to
    1e-5 of the call's largest |de| instead of their own."""
    e_unit, losses, de, de16 = got
    en, l_ref, de_ref, l_scale, _ = ref
    err_u = (e_unit.double() - en).abs().max().item()
    err_l = ((losses.double() - l_ref).abs() / l_scale.clamp(min=1e-30)).max().item() if len(l_ref) else 0.0
    assert torch.equal(de16, de.half()), f"{name}: de16 is not de rounded to fp16"
    gmax = de_ref.abs().max().item()
    rowmax = de_ref.abs().amax(dim=1, keepdim=True)
    err = (de.double() - de_ref).abs()
    assert bool(torch.isfinite(de).all()), name
    if len(zero_rows):
        z = list(zero_rows)
        print(f"[prompt_loss] {name}: rows along the prompt: err {err[z].max().item() / gmax:.2e} of max|de| (<= 1e-5)")
        assert err[z].max().item() <= 1e-5 * gmax, name
    regular = torch.ones(de.shape[0], dtype=torch.bool)
    regular[list(antipodal_rows) + list(zero_rows)] = False
    meas = (err / (rowmax + 1e-300))[regular].max().item() if regular.any() else 0.0
    ok = bool((err[regular] <= 1e-5 * rowmax[regular] + 1e-7 * gmax).all())
    meas_a = 0.0
    if len(antipodal_rows):
        a = list(antipodal_rows)
        meas_a = (err[a] / rowmax[a]).max().item()
    print(f"[prompt_loss] {name}: e_unit err {err_u:.2e} (<= 1e-6)  losses rel err {err_l:.2e} (<= 1e-5)  "
          f"de err / row max {meas:.2e} (<= 1e-5)" + (f"  antipodal rows {meas_a:.2e} (<= {ANTIPODAL_BOUND:g})" if antipodal_rows else ""))
    assert err_u <= 1e-6, name
    assert err_l <= 1e-5, name
    assert ok, f"{name}: de error {meas:.3e} of the row maximum"
    assert meas_a <= ANTIPODAL_BOUND, name
    return err_u, err_l, meas


def _unit(t):
    return F.normalize(t.double(), dim=-1).float()


def _rows_at_cosines(p, cosines, norms, g):
    """Embeddings whose direction has the given cosine to the unit row p, at the given norms (float64 construction)."""
    p = p.double()
    out = []
    for c, nrm in zip(cosines, norms):
        u = torch.randn(p.shape[0], generator=g, dtype=torch.float64)
        u = u - (u @ p) * p
        u = u / u.norm()
        out.append((c * p + math.sqrt(max(1 - c * c, 0.0)) * u) * nrm)
    return torch.stack(out).float()


@pytest.mark.parametrize("shard", [False, True])
@pytest.mark.parametrize("B", [1, 64, 256])
@pytest.mark.parametrize("D", [64, 512, 768, 1024])
def test_prompt_loss_shapes(D, B, shard):
    """Text prompts with positive, negative and zero weights (stops -inf and the engine's -3e38) and one image prompt
    (16 rows sharing a loss slot, 1 / rows each), over every embedding width and batch, whole and as a shard."""
    g = torch.Generator().manual_seed(D * 7 + B + shard)
    cutn_global = 4 * B if shard else B
    text_w = [1.0, -0.7, 0.0, 2.5, -0.05]
    e = torch.randn(B, D, generator=g) * (0.5 + torch.rand(B, 1, generator=g) * 3)
    text = _unit(torch.randn(len(text_w), D, generator=g))
    img_rows = _unit(torch.randn(16, D, generator=g))
    prompts = torch.cat([text, img_rows])
    weights = torch.tensor(text_w + [0.8] * 16)
    stops = torch.tensor([NEG_INF, -3.0e38, NEG_INF, -3.0e38, NEG_INF] + [NEG_INF] * 16)
    slots = torch.tensor(list(range(5)) + [5] * 16)
    inv_rows = torch.tensor([1.0] * 5 + [1 / 16] * 16)
    args = (e, prompts, weights, stops, slots)
    got = _kernel(*args, inv_rows, cutn_global, 4096.0, 6)
    _compare(f"D={D} B={B} cutn={cutn_global}", got, _reference(*args, cutn_global, 4096.0, 6))
    again = _kernel(*args, inv_rows, cutn_global, 4096.0, 6)
    assert all(torch.equal(a, b) for a, b in zip(got, again)), "two calls on the same inputs differ"
    assert got[1][2].item() == 0.0 and bool((got[2][:, :] != 0).any())


@pytest.mark.parametrize("n", [1, 2, 7, 33, 64])
def test_prompt_loss_prompt_counts(n):
    """1 to 64 text prompts with random weights of both signs (every fourth one 0)."""
    g = torch.Generator().manual_seed(100 + n)
    B, D = 64, 512
    e = torch.randn(B, D, generator=g)
    prompts = _unit(torch.randn(n, D, generator=g))
    weights = torch.randn(n, generator=g)
    weights[::4] = 0.0
    stops = torch.full((n,), NEG_INF)
    slots = torch.arange(n)
    args = (e, prompts, weights, stops, slots)
    got = _kernel(*args, torch.ones(n), 128, 1.0, n)
    _compare(f"n={n}", got, _reference(*args, 128, 1.0, n))


def _stop_between(d, g, min_gap=2e-4):
    """A stop between two neighbouring row distances near the middle, at least min_gap / 2 from both."""
    s = torch.sort(d).values
    mid = len(s) // 2
    for k in sorted(range(len(s) - 1), key=lambda k: abs(k - mid)):
        if s[k + 1] - s[k] >= min_gap:
            return float((s[k] + s[k + 1]) / 2)
    raise AssertionError("no gap between the row distances")


@pytest.mark.parametrize("weight", [0.9, -0.6])
def test_stop_mask_per_row(weight):
    """One prompt, rows spread from cosine -0.8 to 0.9 and a stop between two of them: the rows above the stop get their
    gradient, the others none -- the same mask for a negative weight, whose signed distances are negative."""
    g = torch.Generator().manual_seed(7 if weight > 0 else 8)
    B, D = 64, 512
    p = _unit(torch.randn(1, D, generator=g))
    cos = torch.linspace(-0.8, 0.9, B)[torch.randperm(B, generator=g)]
    e = _rows_at_cosines(p[0], cos.tolist(), (0.5 + torch.rand(B, generator=g) * 2).tolist(), g)
    w = torch.tensor([weight])
    d = _reference(e, p, w, torch.tensor([NEG_INF]), torch.tensor([0]), B, 1.0, 1)[4][:, 0]
    stop = _stop_between(d, g)
    assert (d - stop).abs().min().item() >= 1e-4
    args = (e, p, w, torch.tensor([stop]), torch.tensor([0]))
    got = _kernel(*args, torch.ones(1), B, 4096.0, 1)
    ref = _reference(*args, B, 4096.0, 1)
    passed = (got[2] != 0).any(dim=1)
    expect = d > stop
    print(f"[prompt_loss] w={weight}: stop {stop:.4f}, {int(expect.sum())}/{B} rows pass")
    assert 0 < int(expect.sum()) < B
    assert torch.equal(passed, expect), "pass / stop mask"
    _compare(f"stop mask w={weight}", got, ref)


def test_stops_with_several_prompts():
    """Four prompts of both signs, each with a stop between its own row distances, summed into one gradient."""
    g = torch.Generator().manual_seed(12)
    B, D = 128, 768
    p = _unit(torch.randn(4, D, generator=g))
    # rows spread in cosine towards prompt 0 and 2, so their distances spread; the others see nearly orthogonal rows
    half = B // 2
    e = torch.cat([_rows_at_cosines(p[0], torch.linspace(-0.7, 0.9, half).tolist(), [1.3] * half, g),
                   _rows_at_cosines(p[2], torch.linspace(-0.9, 0.7, B - half).tolist(), [0.7] * (B - half), g)])
    e = e[torch.randperm(B, generator=g)]
    w = torch.tensor([1.2, -0.4, -2.0, 0.3])
    d = _reference(e, p, w, torch.full((4,), NEG_INF), torch.arange(4), B, 1.0, 4)[4]
    stops = torch.tensor([_stop_between(d[:, j], g) for j in range(4)])
    assert (d - stops).abs().min().item() >= 1e-4
    for j in range(4):
        assert 0 < int((d[:, j] > stops[j]).sum()) < B
    args = (e, p, w, stops, torch.arange(4))
    _compare("four prompts with stops", _kernel(*args, torch.ones(4), 2 * B, 4096.0, 4), _reference(*args, 2 * B, 4096.0, 4))


def test_all_rows_stopped():
    """Every stop above every distance: de is exactly 0, and e_unit and the loss values are still written."""
    g = torch.Generator().manual_seed(13)
    B, D = 64, 512
    e = torch.randn(B, D, generator=g)
    p = _unit(torch.randn(3, D, generator=g))
    w = torch.tensor([1.0, -0.5, 0.25])
    stops = torch.tensor([5.0, 0.5, 5.0])  # dist <= 2 (pi/2)^2 < 5; the negative weight's dists are <= 0 < 0.5
    args = (e, p, w, stops, torch.arange(3))
    got = _kernel(*args, torch.ones(3), B, 4096.0, 3)
    assert bool((got[2] == 0).all()) and bool((got[3] == 0).all())
    _compare("all rows stopped", got, _reference(*args, B, 4096.0, 3))


def test_degenerate_geometry():
    """Rows equal to the prompt direction (r ~ 0), nearly antipodal to it (r / 2 = 1 - 1e-4), and of norms 1e-3 and
    1e3."""
    g = torch.Generator().manual_seed(14)
    D = 512
    p = _unit(torch.randn(1, D, generator=g))
    phi = 2 * math.acos(1 - 1e-4)                      # the angle to -p at which r / 2 = cos(phi / 2) = 1 - 1e-4
    cos = [1.0, 1.0, -math.cos(phi), -math.cos(phi), 0.3, -0.2, 0.5, 0.0]
    norms = [3.7, 1e-3, 1.0, 1e3, 1e-3, 1e3, 1.0, 2.0]
    e = _rows_at_cosines(p[0], cos, norms, g)
    e[0] = p[0] * 3.7                                   # exactly the prompt's direction
    for w in (1.0, -1.0):
        args = (e, p, torch.tensor([w]), torch.tensor([NEG_INF]), torch.tensor([0]))
        ref = _reference(*args, 8, 4096.0, 1)
        r_half = 1 - ref[4][:, 0].abs().div(2).sqrt().sin()
        assert abs(r_half[2].item() - 1e-4) < 2e-5 and abs(r_half[3].item() - 1e-4) < 2e-5
        _compare(f"degenerate rows w={w}", _kernel(*args, torch.ones(1), 8, 4096.0, 1), ref, antipodal_rows=(2, 3),
                 zero_rows=(0, 1))


def test_engine_prompts_with_finite_stops():
    """Through the engine: set_prompts with finite stops between the rows' distances (and one -inf, which the host clamps
    to -3e38), encode_image + prompt_loss on the device prompt rows; clip0.de against float64 on the engine's clip0.e."""
    from pixray_b200 import engine as E
    from pixray_b200 import synthetic as S
    cfg = dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=64)
    cutn, cs = 8, 224
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(8, 8), cutn=cutn, clip=[cfg], noise_fac=0.1, seed=5)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(cfg, 6))
    eng.finalize()
    g = torch.Generator().manual_seed(15)
    raw = torch.randn(3, 64, generator=g)
    w = torch.tensor([1.0, -0.6, 0.4])
    eng.set_prompts(0, raw.numpy(), w.tolist(), [NEG_INF] * 3)
    eng.synth(torch.rand(1, 3, 8, 8, generator=g))
    T = np.tile(np.eye(3, dtype=np.float32), (cutn, 1, 1))
    T[:, 0, 0] = T[:, 1, 1] = np.linspace(0.6, 1.4, cutn)
    eng.make_cutouts(torch.rand(1, 3, 32, 32, generator=g), transforms=T, zoom_padding=E.PAD_BORDER, fill=0.3,
                     noise_facs=torch.full((cutn,), 0.05).numpy(), noise=torch.randn(cutn, 3, cs, cs, generator=g))
    e_unit = eng.encode_image(0).cpu()
    e = eng.debug_read("clip0.e", (cutn, 64)).cpu()
    p = F.normalize(raw.double(), dim=1).float()        # the rows pxr_set_prompts uploads
    d = _reference(e, p, w, torch.full((3,), NEG_INF), torch.arange(3), cutn, 1.0, 3)[4]
    stops = [_stop_between(d[:, 0], g), _stop_between(d[:, 1], g), NEG_INF]
    assert min((d[:, j] - stops[j]).abs().min().item() for j in range(2)) >= 1e-4
    eng.set_prompts(0, raw.numpy(), w.tolist(), stops)
    losses = eng.prompt_loss(0).cpu()
    de = eng.debug_read("clip0.de", (cutn, 64)).cpu()
    ref = _reference(e, p, w, torch.tensor(stops), torch.arange(3), cutn, 4096.0, 3)
    _compare("engine, finite stops", (e_unit, losses, de, de.half()), ref)   # clip0.de16 has no debug name
    for j in range(2):
        print(f"[prompt_loss] engine prompt {j}: {int((d[:, j] > stops[j]).sum())}/{cutn} rows pass")
