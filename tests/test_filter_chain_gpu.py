"""The filter chain between the drawer and the cutouts (kernels_filters.cu, Engine::rebuild_filters / filters_forward /
filters_backward; filters/{tiler,wallpaper,colorlookup}.py through do_synth_and_filter, pixray.py:1203-1222) against the
float64 oracle filters (oracle/ref_path.py, pinned to the reference classes by tests/golden/filter_vectors.npz), applied
to the engine's own drawer image with the engine's shifts.

The drawer is the fast pixel drawer with one grid cell per pixel, so the image is the latent itself and every pixel is
distinct (an off-by-one crop or roll cannot hide in a block of equal pixels).  One fused iteration (a tiny ViT behind the
cutouts) gives the chain's output `filtered`, the gradient arriving at it `g_filtered`, the drawer image's gradient
`g_img` and the loss vector, whose first entries are the filters' losses.  What is compared, and how tightly:

  filtered   equal to the float64 chain: rolls, the "shift" wallpaper and the edge crops are copies, and the colour
             lookup returns a table entry.  The latent is drawn so that every pixel's two nearest distinct table colours
             are more than 1e-5 apart in distance, so the fp32 and float64 nearest-colour decisions agree everywhere.
  losses     each filter's slot within 1e-6 of the float64 loss (0 exactly for the loss-free filters)
  g_img      the float64 VJP of the chain at the engine's g_filtered, plus S * weight * dloss/dx of every filter (S = 4096,
             the engine's gradient scale), elementwise within
               2^-24 m C + TAU T
             C: the chain's adjoint applied to |g_filtered| (all adjoints here are copies and sums with weight 1).  The
             copies are exact; m counts the fp32 additions an element's value can go through (_roundings), each of
             which rounds once, so a chain of copies and two-term sums is held to 1 fp32 ulp per addition.  T: the same
             adjoint applied to the magnitudes of the edge-match and lookup loss
             gradients, which the engine forms in fp32 (a few roundings each), summed term by term: where the strips
             overlap (2 em > size) or the two axes' strips meet, an element takes two terms that can cancel while each
             keeps its own rounding.

TAU is about 3x the largest value measured over the cases (each case prints its own).  Measured on an H100 (80 GB HBM3,
700 W): 1.9e-7 (lookup_then_tiler), 1.5e-7 (lookup_beta10), <= 1.4e-7 in the other cases.
"""
import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu

GS = 4096.0
CUTN, CS = 4, 224
TOWER = dict(width=128, layers=1, heads=2, patch=32, image_res=CS, out_dim=64)
TAU = 6e-7
MARGIN = 1e-5

TILER, WALL, LOOKUP = E.FILTER_TILER, E.FILTER_WALLPAPER, E.FILTER_LOOKUP
WP = {"shift": 1, "horizontal": 2, "vertical": 3, "both": 0}
# the default table in fp32, as the engine receives it; entries 11 and 12 are the same colour (colorlookup.py:10-26)
DEFAULT_TABLE = [[float(np.float32(c / 255.0)) for c in rgb] for rgb in R.COLORLOOKUP_DEFAULT_TABLE]
PAL = [[float(np.float32(v)) for v in c] for c in
       [[0.9, 0.1, 0.1], [0.1, 0.8, 0.2], [0.2, 0.2, 0.9], [0.95, 0.95, 0.9], [0.05, 0.05, 0.05], [0.5, 0.45, 0.55]]]


def tiler(w=1.0):
    return dict(kind=TILER, weight=w, params=[], ref=lambda im, rh, rw: R.filter_tiler(im, rh, rw))


def wallpaper(t, em, w=2.0):
    return dict(kind=WALL, weight=w, params=[WP[t], em], shift=t == "shift",
                ref=lambda im, rh, rw: R.filter_wallpaper(im, None if t == "both" else t, em, rh, rw))


def lookup(table=None, beta=10.0, w=0.7):
    tbl = DEFAULT_TABLE if table is None else table
    return dict(kind=LOOKUP, weight=w, params=[beta] + [v for c in tbl for v in c], table=tbl,
                ref=lambda im, rh, rw: R.filter_colorlookup(im, tbl, beta))


# name: (canvas (H, W), [filter], [(rand_h, rand_w) per filter]); shifts are drawn in [0, input size), like the reference
CASES = {
    "tiler_0_0": ((32, 40), [tiler()], [(0, 0)]),
    "tiler_last": ((33, 45), [tiler()], [(32, 44)]),
    # the second row of tiles is offset by W / 2 (rounded down: odd W); sh = H - 1 wraps across the 2H canvas
    "shift_even_w": ((32, 40), [wallpaper("shift", 0)], [(31, 7)]),
    "shift_odd_w": ((33, 45), [wallpaper("shift", 0)], [(32, 44)]),
    # em = 2: em2 = 1; odd em = 7: the crop takes em2 = 3 from each side while the strips are 7 wide
    "horizontal_em2": ((32, 40), [wallpaper("horizontal", 2)], [(5, 9)]),
    "horizontal_em7_odd": ((33, 45), [wallpaper("horizontal", 7)], [(5, 30)]),
    # the largest accepted em: W on an odd canvas (one column left), W - 1 on an even one
    "horizontal_em_w_odd": ((33, 45), [wallpaper("horizontal", 45)], [(3, 44)]),
    "horizontal_em_w-1_even": ((32, 40), [wallpaper("horizontal", 39)], [(3, 39)]),
    # 2 em > W: the two strips overlap and the elements of the overlap take both gradient terms
    "horizontal_overlap": ((32, 40), [wallpaper("horizontal", 30)], [(0, 13)]),
    "vertical_em2": ((32, 40), [wallpaper("vertical", 2)], [(17, 3)]),
    "vertical_em7_odd": ((33, 45), [wallpaper("vertical", 7)], [(20, 2)]),
    "vertical_em_h_odd": ((33, 45), [wallpaper("vertical", 33)], [(32, 1)]),
    "vertical_overlap_odd": ((33, 45), [wallpaper("vertical", 25)], [(11, 0)]),
    "both_em2": ((32, 40), [wallpaper("both", 2)], [(31, 39)]),
    "both_em7_odd": ((33, 45), [wallpaper("both", 7)], [(8, 21)]),
    "both_overlap_odd": ((33, 45), [wallpaper("both", 25, w=0.5)], [(4, 40)]),
    "lookup_default": ((32, 40), [lookup()], [(0, 0)]),
    "lookup_beta10": ((33, 45), [lookup(PAL, 10.0)], [(0, 0)]),
    "lookup_beta0": ((33, 45), [lookup(PAL, 0.0)], [(0, 0)]),
    "lookup_then_tiler": ((32, 40), [lookup(PAL, 3.0), tiler()], [(0, 0), (13, 27)]),
    "both_then_lookup": ((33, 45), [wallpaper("both", 6), lookup(PAL, 3.0)], [(11, 21), (0, 0)]),
    # every "shift" wallpaper doubles the height: the lookup sees 8 H x W pixels
    "shift3_then_lookup": ((24, 36), [wallpaper("shift", 0), wallpaper("shift", 0), wallpaper("shift", 0),
                                      lookup(None, 10.0)], [(23, 5), (47, 35), (60, 17), (0, 0)]),
}


def _clear_of_ties(px, table):
    """px [N, 3] float64: True where the two nearest DISTINCT table colours are more than MARGIN apart in distance."""
    uniq = torch.unique(torch.tensor(table, dtype=torch.float64), dim=0)
    top2 = torch.cdist(px, uniq).topk(2, dim=1, largest=False).values
    return (top2[:, 1] - top2[:, 0]) > MARGIN


def _latent(H, W, filters, g):
    """The pixel drawer's latent (= its image, one cell per pixel), redrawn where a lookup would face a near-tie.  The
    default table's doubled colour (entries 11 / 12) is planted near a few pixels so that the first-minimum rule is used."""
    z = torch.rand(1, 3, H, W, generator=g)
    tables = [f["table"] for f in filters if f["kind"] == LOOKUP]
    if any(t is DEFAULT_TABLE for t in tables):
        z[0, :, 0, :6] = torch.tensor(DEFAULT_TABLE[11]).view(3, 1) + (torch.rand(3, 6, generator=g) - 0.5) * 0.04
        z = z.clamp(0, 1)
    for _ in range(100):
        px = z.permute(0, 2, 3, 1).reshape(-1, 3).double()
        bad = torch.zeros(px.shape[0], dtype=torch.bool)
        for t in tables:
            bad |= ~_clear_of_ties(px, t)
        if not bad.any():
            return z.contiguous()
        flat = z.permute(0, 2, 3, 1).reshape(-1, 3)
        flat[bad] = torch.rand(int(bad.sum()), 3, generator=g)
        z = flat.reshape(1, H, W, 3).permute(0, 3, 1, 2)
    raise AssertionError("could not draw a latent clear of near-ties")


def _engine(hw, seed):
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=hw, grid=hw, cutn=CUTN, cut_size=CS, clip=[TOWER], noise_fac=0.1,
                       seed=seed)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(TOWER, seed + 1))
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    return eng


def _iterate(eng, z, n_loss, hw, out_hw):
    losses = np.zeros(n_loss, dtype=np.float32)
    eng.iterate(z.clone().cuda(), 0.0, 0, losses_out=losses)
    rd = lambda name, shape: eng.debug_read(name, shape).cpu()
    return dict(losses=losses, img=rd("img", (1, 3) + hw), g_img=rd("g_img", (1, 3) + hw),
                filtered=rd("filtered", (1, 3) + out_hw), g_filtered=rd("g_filtered", (1, 3) + out_hw))


def _reference(img, filters, shifts):
    """The float64 chain on `img`: output, per-filter losses, and each filter's input (for the loss-gradient magnitudes)."""
    x = img.double().requires_grad_(True)
    cur, losses, inputs = x, [], []
    for f, (rh, rw) in zip(filters, shifts):
        inputs.append(cur)
        cur, loss = f["ref"](cur, rh, rw)
        losses.append(f["weight"] * loss)
    return x, cur, losses, inputs


def _edge_magnitude(t, dim, em):
    """sum over the pairs of |d (mse(first em, last em) / em) / d t|, term by term: where the strips overlap an element
    takes two terms, which can cancel in the gradient but each carry their own rounding."""
    t = t.detach()
    n = t.shape[dim]
    d = (t.narrow(dim, 0, em) - t.narrow(dim, n - em, em)).abs() * (2.0 / (t.narrow(dim, 0, em).numel() * em))
    mag = torch.zeros_like(t)
    mag.narrow(dim, 0, em).add_(d)
    mag.narrow(dim, n - em, em).add_(d)
    return mag


def _loss_grad_magnitudes(f, inp, loss):
    """(tensor, |S * weight * dloss / dtensor|) at each place a filter's loss looks at: the lookup's input; the edge-match
    strips of the wallpaper's input and, for both axes, of the column-cropped tensor the row strips are taken from."""
    if not loss.requires_grad:
        return []
    if f["kind"] == LOOKUP:
        (gl,) = torch.autograd.grad(GS * loss, inp, retain_graph=True)
        return [(inp, gl.abs())]
    t, em = f["params"]
    em2, w = em // 2, GS * f["weight"]
    if t == WP["horizontal"]:
        return [(inp, w * _edge_magnitude(inp, 3, em))]
    if t == WP["vertical"]:
        return [(inp, w * _edge_magnitude(inp, 2, em))]
    cropped = inp[:, :, :, em2:-em2]
    return [(inp, w * _edge_magnitude(inp, 3, em)), (cropped, w * _edge_magnitude(cropped, 2, em))]


def _roundings(filters):
    """How many fp32 roundings the copy of the upstream gradient in one element can go through: one per "shift" wallpaper
    (two terms summed), two per edge-match strip pair (a term from each strip where they overlap), one per lookup (its
    loss gradient added); at least one."""
    m = 0
    for f in filters:
        if f["kind"] == LOOKUP:
            m += 1
        elif f["kind"] == WALL:
            t, em = f["params"]
            m += 1 if t == WP["shift"] else (2 * (2 if t == WP["both"] else 1) if em else 0)
    return max(1, m)


@pytest.mark.parametrize("case", list(CASES))
def test_filter_chain_against_float64(case):
    hw, filters, shifts = CASES[case]
    H, W = hw
    seed = list(CASES).index(case) + 120
    g = torch.Generator().manual_seed(seed + 3)
    z = _latent(H, W, filters, g)
    eng = _engine(hw, seed)
    try:
        for i, (f, (rh, rw)) in enumerate(zip(filters, shifts)):
            assert eng.add_filter(f["kind"], f["weight"], f["params"]) == i
            eng.set_filter_shifts(i, rh, rw)
        x, out, ref_losses, inputs = _reference(z, filters, shifts)  # the drawer image is the latent
        out_hw = tuple(out.shape[2:])
        n_f = len(filters)
        a = _iterate(eng, z, n_f + 2, hw, out_hw)
        b = _iterate(eng, z, n_f + 2, hw, out_hw)
    finally:
        eng.close()
    assert torch.equal(a["img"], z)
    if any(f.get("table") is DEFAULT_TABLE for f in filters):  # the doubled colour is used, through its first entry
        d = torch.cdist(z.permute(0, 2, 3, 1).reshape(-1, 3).double(), torch.tensor(DEFAULT_TABLE, dtype=torch.float64))
        assert (d.argmin(1) == 11).sum() >= 3

    # forward: the chain's output is a copy of image values or table entries, exactly
    mism = (a["filtered"].double() != out.detach()).sum().item()
    print(f"[filters] {case}: filtered {out_hw}, {mism} mismatches")
    assert mism == 0

    # the losses, one slot per filter at the front of the loss vector
    for i, lr in enumerate(ref_losses):
        e, r = float(a["losses"][i]), lr.item()
        print(f"[filters] {case}: loss[{i}] engine {e:.9g} float64 {r:.9g}")
        assert abs(e - r) <= 1e-6 * abs(r)

    # g_img: the VJP at the engine's g_filtered plus every filter's scaled loss gradient
    gf = a["g_filtered"].double()
    L = (out * gf).sum() + GS * sum(ref_losses)
    (ref,) = torch.autograd.grad(L, x, retain_graph=True)
    (C,) = torch.autograd.grad(out, x, grad_outputs=gf.abs(), retain_graph=True)
    T = torch.zeros_like(ref)
    for f, inp, lf in zip(filters, inputs, ref_losses):
        for t, mag in _loss_grad_magnitudes(f, inp, lf):
            T += mag if t is x else torch.autograd.grad(t, x, grad_outputs=mag, retain_graph=True)[0]
    err = (a["g_img"].double() - ref).abs()
    excess = (err - 2.0 ** -24 * _roundings(filters) * C).clamp(min=0)
    tau = torch.where(excess > 0, excess / T, torch.zeros_like(excess)).max().item()
    print(f"[filters] {case}: g_img max err {err.max().item():.3e}  max|ref| {ref.abs().max().item():.3e}  "
          f"max T {T.max().item():.3e}  measured tau {tau:.3e} (<= {TAU:g})")
    assert tau <= TAU

    # a second identical iteration: bit-identical (one writer per element everywhere, fixed-order reductions)
    for key in ("filtered", "g_filtered", "g_img"):
        assert torch.equal(a[key], b[key]), key
    assert np.array_equal(a["losses"], b["losses"])


@pytest.mark.parametrize("wp_type,hw,em,size_msg", [
    ("horizontal", (33, 45), 46, "width"),   # em > W
    ("horizontal", (33, 45), 1, "width"),    # em2 = 0
    ("horizontal", (32, 40), 40, "width"),   # em = W on an even width crops to nothing
    ("vertical", (33, 45), 34, "height"),
    ("vertical", (33, 45), 1, "height"),
    ("both", (32, 40), 33, "height"),        # fits the width, not the height
])
def test_edge_match_refuses_what_does_not_fit(wp_type, hw, em, size_msg):
    """em > size is refused, and so is em = 1 (em2 = 0: the reference's [em2:-em2] slices to nothing) and an em that crops
    an even size to nothing; the refused filter leaves the chain as it was."""
    eng = _engine(hw, 7)
    try:
        with pytest.raises(E.EngineError, match=f"wallpaper_edge_match does not fit the image {size_msg}"):
            eng.add_filter(WALL, 1.0, [WP[wp_type], em])
        assert eng.num_losses() == 2
    finally:
        eng.close()
