"""The line-sketch drawer (`line_sketch`, LineDrawer) on the CPU: the plugin against the real reference's recorded start
geometry, rates, clip_z and composite (tests/golden/line_sketch.npz, oracle/make_golden_line.py); the float64 oracle's
self-checks (areas, flattening bound, boundary gradient against finite differences); and the session's control flow
against a recording stand-in for the engine."""
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from oracle import polygon_ref as PR
from oracle import stroke_ref as SR
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import plugins as P

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "line_sketch.npz"))
CASES = {c["name"]: c for c in json.loads(str(GOLD["cases"]))}


def _settings(case):
    s = dict(size=case["size"], strokes=24, stroke_length=8, min_stroke_width=0.5, max_stroke_width=2,
             allow_paper_color=False)
    s.update(case["settings"])
    return SimpleNamespace(**s)


def _drawer(settings):
    w, h = settings.size
    eng = SimpleNamespace(image_hw=(h, w), device=torch.device("cpu"))
    return P.LineDrawer(settings, P.Session(eng))


@pytest.mark.parametrize("name", sorted(CASES))
def test_start_geometry_rates_and_clip_match_the_reference(name):
    case = CASES[name]
    st = _settings(case)
    d = _drawer(st)
    random.seed(case["seed"])
    d.load_model(st, "cpu")
    assert np.array_equal(d.points().numpy(), GOLD[name + "_points"])   # bit for bit
    assert np.array_equal(d.widths().numpy(), GOLD[name + "_widths"])
    assert np.array_equal(d.paper().numpy(), np.float32(P.PAPER_RGBA))
    assert d.max_width == case["max_width"]
    for div, key in ((1, "_rates1"), (10, "_rates10")):
        rates = np.array([o["lr"] for o in d.get_opts(div)])
        assert rates.shape == GOLD[name + key].shape and np.abs(rates - GOLD[name + key]).max() <= 1e-7
    d.widths().copy_(torch.from_numpy(GOLD[name + "_clip_in"]))
    d.clip_z()
    assert np.abs(d.widths().numpy() - GOLD[name + "_clip_out"]).max() <= 1e-7
    assert d.get_z_copy() is None


def test_synth_composite_matches_the_reference():
    names = [n for n in CASES if n + "_render" in GOLD]
    assert names
    for name in names:
        out = SR.synth_composite(torch.from_numpy(GOLD[name + "_render"]))
        assert (out - torch.from_numpy(GOLD[name + "_synth"])).abs().max().item() <= 1e-7


def _lattice_area(points, w, H, W, n):
    z = np.concatenate([np.asarray(points, dtype=np.float64).reshape(-1), np.full(len(points), w), [1, 1, 1, 1]])
    sc = SR.Scene(z, len(points), (len(points[0]) - 1) // 3, H, W)
    return SR.coverage(sc.winners(PR.regular_samples(H, W, n))).sum(), sc


def test_covered_area_converges_to_the_capsule_union():
    # one straight segment: area 2 w L + pi w^2, and d area / dw (the boundary integral with G = 1) is the perimeter
    a, b, w = np.array([6.3, 7.1]), np.array([21.7, 15.9]), 2.2
    pts = [[a + (b - a) * t for t in (0, 1 / 3, 2 / 3, 1)]]
    L = float(np.hypot(*(b - a)))
    exact = 2 * w * L + np.pi * w * w
    errs = []
    for n in (4, 8, 16, 32):
        area, sc = _lattice_area(pts, w, 24, 28, n)
        errs.append(abs(area - exact))
    print(f"[oracle] straight stroke area error by lattice {errs}")
    assert max(errs[2:]) < 1e-3 * exact
    g = SR.capsule_gradients(sc, np.ones((24, 28)))
    gp, gw = SR.fold(sc, g)
    assert abs(gw[0] - (2 * L + 2 * np.pi * w)) < 1e-6 * L  # tangent end disks leave roundoff-sized gaps
    # a curved stroke: the lattice areas converge (differences shrink as the lattice refines)
    curved = [[[4.0, 20.0], [8.0, 2.0], [22.0, 26.0], [26.0, 6.0]]]
    areas = [_lattice_area(curved, 1.7, 28, 30, n)[0] for n in (4, 8, 16, 32, 64)]
    diffs = np.abs(np.diff(areas))
    print(f"[oracle] curved stroke areas {areas}")
    assert diffs[-1] < diffs[0] and diffs[-1] < 1e-3 * areas[-1]


def test_flattening_error_is_within_the_sagitta_bound():
    random.seed(3)
    pts = P.line_start_points(384, 216, 24, 8).double().numpy()
    err, bound = SR.cubic_flattening_error(pts)
    print(f"[oracle] default start geometry: flattening error {err:.4g} px, bound max|B''|/(8 S^2) = {bound:.4g} px")
    assert err <= bound and bound < 0.5
    curved = np.array([[[4.0, 20.0], [8.0, 2.0], [22.0, 26.0], [26.0, 6.0]]])
    err, bound = SR.cubic_flattening_error(curved)
    assert err <= bound


def _fd_scene():
    """Three one-segment strokes crossing each other; the last one leaves the canvas on the right."""
    pts = np.array([[[2.0, 3.0], [9.0, 8.0], [14.0, 4.0], [21.5, 15.0]],
                    [[3.0, 16.5], [8.0, 5.0], [15.0, 17.0], [19.0, 2.5]],
                    [[6.0, 10.0], [13.0, 12.5], [20.0, 8.5], [27.0, 11.0]]])
    widths = np.array([1.6, 1.2, 2.1])
    return pts, widths


def test_boundary_gradient_matches_finite_differences():
    """d/dtheta of sum_p h(p) c(p) from the boundary integral against central differences of the coverage of a 48 x 48
    lattice per pixel.  Measured: max error 0.42 % of the largest gradient component, mean 0.08 %; the tolerance is 2 %."""
    H, W, n, eps = 20, 24, 48, 0.05
    pts, widths = _fd_scene()
    h = np.random.default_rng(0).uniform(0.5, 1.5, (H, W))
    samples = PR.regular_samples(H, W, n)

    def F(z):
        sc = SR.Scene(z, 3, 1, H, W)
        return float((SR.coverage(sc.winners(samples)) * h).sum())

    z0 = np.concatenate([pts.reshape(-1), widths, [1, 1, 1, 1]])
    sc = SR.Scene(z0, 3, 1, H, W)
    gp, gw = SR.fold(sc, SR.capsule_gradients(sc, h))
    grad = np.concatenate([gp.reshape(-1), gw])
    fd = np.empty_like(grad)
    for i in range(len(grad)):
        zp, zm = z0.copy(), z0.copy()
        zp[i] += eps
        zm[i] -= eps
        fd[i] = (F(zp) - F(zm)) / (2 * eps)
    err = np.abs(grad - fd)
    print(f"[oracle] boundary gradient vs finite differences: max {err.max() / np.abs(fd).max():.3e}, "
          f"mean {err.mean() / np.abs(fd).max():.3e} of max|grad| {np.abs(fd).max():.3f}")
    assert err.max() <= 2e-2 * np.abs(fd).max()


# ------------------------------------------------------------------------------------------------ session control flow
class StrokeFake(FakeEngine):
    def __init__(self, *, drawer=E.DRAWER_VQGAN, strokes=None, **kw):
        super().__init__(drawer=drawer, grid=(1, 1), strokes=strokes, **kw)
        self.z_shape = (sum(E.stroke_z_layout(strokes[0], strokes[1])),)

    def set_synth_iteration(self, it):
        self._log("set_synth_iteration", it=it)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", StrokeFake)
    FakeEngine.loss_script = staticmethod(lambda it, n: np.full(n, 1.0 / (1 + it), dtype=np.float32))
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(prompts="a sketch", drawer="line_sketch", clip_models="ViT-B/16", outdir="", seed="5",
                b200_allow_synthetic=True, vector_prompts="none")
    base.update(kw)
    api.add_settings(**base)
    args = api.apply_settings()
    api.do_init(args)
    return args


def test_options_resolve_and_reach_the_engine(fake, tmp_path):
    args = _init(tmp_path)
    assert (args.strokes, args.stroke_length, args.min_stroke_width, args.max_stroke_width, args.allow_paper_color) == \
        (24, 8, 0.5, 2, False)
    eng = api._state.engine
    W, H = args.size
    assert eng.kw["drawer"] == E.DRAWER_STROKES and eng.kw["strokes"] == (24, 8, 2 * H / 100, False)
    d = api._state.drawer
    assert isinstance(d, P.LineDrawer) and tuple(d.get_z().shape) == eng.z_shape == (24 * 25 * 2 + 24 + 4,)
    # no start image: the reference's init_from_tensor is a no-op, and load_model drew the points after random.seed
    assert "vqgan_encode" not in eng.names()
    random.seed(api._state.seed)
    assert torch.equal(d.points(), P.line_start_points(W, H, 24, 8))
    api.reset_settings()
    args = _init(tmp_path, strokes=5, stroke_length=3, max_stroke_width=4.0, allow_paper_color=True, size=[100, 50])
    assert api._state.engine.kw["strokes"] == (5, 3, 2.0, True)


def test_three_rates_and_their_drops(fake, tmp_path):
    args = _init(tmp_path, iterations=20, learning_rate_drops=[50, 25], allow_paper_color=True)
    d = api._state.drawer
    assert [o["lr"] for o in d.get_opts(1)] == [1.0, 0.1, 0.01]
    assert [o["lr"] for o in d.get_opts(10)] == [0.1, 0.01, 0.001]
    z0 = d.get_z().clone()
    assert api.do_run(args) is True
    eng = api._state.engine
    # the engine takes the points' rate; the widths and the paper run at 1/10 and 1/100 of it inside the fused Adam
    lrs = [round(c[1]["lr"], 9) for c in eng.calls if c[0] == "iterate"]
    assert lrs == [1.0] * 5 + [0.1] * 5 + [0.01] * 10
    assert eng.names().count("reset_optimizer") == 3
    # no best state is kept or restored (get_z_copy is None): z is only ever what the engine stepped
    assert d.get_z_copy() is None and torch.equal(d.get_z(), z0)


@pytest.mark.parametrize("kw", [dict(init_weight=0.5), dict(init_weight_dist=0.5), dict(init_weight_cos=0.5),
                                dict(init_weight_pix=0.5)], ids=lambda kw: next(iter(kw)))
def test_anchors_are_refused(fake, tmp_path, kw):
    with pytest.raises(ValueError, match="line_sketch"):
        _init(tmp_path, **kw)
