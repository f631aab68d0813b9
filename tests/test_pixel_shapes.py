"""The pixel drawer's shaped cells on the host: the geometry against the reference (tests/golden/pixel_shapes.npz, written
by oracle/make_golden_pixel.py from the unmodified PixelDrawer), the float64 rasteriser of oracle/polygon_ref.py against
exact areas, and the API routing with a recording engine.  No GPU."""
import json
import os

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from fake_engine import FakeEngine
from oracle import polygon_ref as PR
from oracle.make_golden_pixel import init_image
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import pixel_shapes as PS
from pixray_b200 import plugins as P

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "pixel_shapes.npz"))
CASES = json.loads(str(GOLD["cases"]))


def _grid(case, verbose=False):
    s = case["settings"]
    return PS.grid_for(case["size"], case["pixel_type"], s.get("pixel_size"), s.get("pixel_scale"),
                       s.get("pixel_edge_check", True), s.get("pixel_iso_check", True), verbose=verbose)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_geometry_and_colours_match_the_reference(case):
    rows, cols = _grid(case)
    assert (rows, cols) == (case["rows"], case["cols"])
    if case["seed"] is None:
        return
    name, (w, h) = case["name"], case["size"]
    xy, off = PS.polygons((w, h), rows, cols, case["pixel_type"])
    assert np.array_equal(off, GOLD[name + "_off"])
    assert np.array_equal(xy.view(np.uint32), GOLD[name + "_xy"].view(np.uint32))  # every vertex, bit for bit
    rgba = PS.init_colours(torch.from_numpy(init_image(case["seed"], w, h)), rows, cols, case["pixel_type"])
    assert rgba.shape == GOLD[name + "_rgba"].shape
    np.testing.assert_allclose(rgba, GOLD[name + "_rgba"], rtol=0, atol=1e-7)


def test_the_fixture_covers_every_type_and_the_grid_rules():
    types = {c["pixel_type"] for c in CASES if c["seed"] is not None}
    assert types == set(PS.PIXEL_TYPES)
    seen = {(c["pixel_type"], tuple(c["size"])): (c["rows"], c["cols"]) for c in CASES if not c["settings"]}
    assert seen[("hex", (256, 256))] == (57, 41)
    assert seen[("hex", (384, 216))] == (63, 81)
    xy, off = PS.polygons((256, 256), 57, 41, "hex")
    assert len(off) - 1 == 2308
    xy, off = PS.polygons((384, 216), 63, 81, "hex")
    assert len(off) - 1 == 5071


def test_announced_grid_is_the_one_before_the_edge_check(capsys):
    assert PS.grid_for((256, 256), "hex") == (57, 41)
    assert capsys.readouterr().out.strip() == "Running pixeldrawer with 40x56 grid"


def test_unknown_pixel_type_is_refused():
    with pytest.raises(ValueError, match="rect, rectshift, hex, tri, diamond, knit"):
        PS.grid_for((64, 64), "hexagon")
    with pytest.raises(ValueError, match="rect, rectshift, hex, tri, diamond, knit"):
        PS.polygons((64, 64), 4, 4, "square")


def test_colours_need_a_start_image():
    with pytest.raises(ValueError, match="init_image or use init_noise"):
        PS.init_colours(None, 4, 4, "hex")


# ---------------------------------------------------------------------------------------------------- oracle rasteriser
def _clip_to_canvas(v, w, h):
    """Sutherland-Hodgman clip of a convex-or-not simple polygon against [0, w] x [0, h]."""
    def clip(poly, inside, cut):
        out = []
        for i in range(len(poly)):
            a, b = poly[i - 1], poly[i]
            if inside(b):
                if not inside(a):
                    out.append(cut(a, b))
                out.append(b)
            elif inside(a):
                out.append(cut(a, b))
        return out

    def at_x(x0):
        return lambda a, b: (x0, a[1] + (b[1] - a[1]) * (x0 - a[0]) / (b[0] - a[0]))

    def at_y(y0):
        return lambda a, b: (a[0] + (b[0] - a[0]) * (y0 - a[1]) / (b[1] - a[1]), y0)

    p = [tuple(q) for q in v]
    p = clip(p, lambda q: q[0] >= 0, at_x(0.0))
    p = clip(p, lambda q: q[0] <= w, at_x(float(w)))
    p = clip(p, lambda q: q[1] >= 0, at_y(0.0))
    p = clip(p, lambda q: q[1] <= h, at_y(float(h)))
    return np.array(p, dtype=np.float64).reshape(-1, 2)


def _shoelace(p):
    if len(p) < 3:
        return 0.0, 0.0
    x, y = p[:, 0], p[:, 1]
    area = 0.5 * abs(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))
    perim = np.sum(np.hypot(np.roll(x, -1) - x, np.roll(y, -1) - y))
    return area, perim


@pytest.mark.parametrize("pixel_type", ["rect", "rectshift", "tri"])
def test_oracle_sample_counts_converge_to_the_visible_area(pixel_type):
    """For the tilings (no overlaps), the samples a shape wins on a dense n x n lattice per pixel estimate its area inside
    the canvas to within one lattice spacing times its perimeter."""
    w, h, n = 37, 29, 12
    rows, cols = PS.grid_for((w, h), pixel_type, pixel_size=[6, 5], verbose=False)
    xy, off = PS.polygons((w, h), rows, cols, pixel_type)
    win = PR.polygon_winners(xy, off, h, w, PR.regular_samples(h, w, n))
    counts = np.bincount(win[win >= 0].ravel(), minlength=len(off) - 1) / (n * n)
    total = 0.0
    for k in range(len(off) - 1):
        area, perim = _shoelace(_clip_to_canvas(xy[off[k]:off[k + 1]].astype(np.float64), w, h))
        assert abs(counts[k] - area) <= perim / n + 1e-9, (k, counts[k], area)
        total += area
    assert abs(counts.sum() - total) <= 1e-9 + 2 * (w + h) / n


def test_oracle_rect_grid_with_integer_cells_is_the_nearest_upsample():
    """A rect grid whose cells are whole pixels renders exactly the fast pixel drawer's image (F.interpolate nearest)."""
    w, h, cols, rows = 24, 20, 6, 5
    xy, off = PS.polygons((w, h), rows, cols, "rect")
    g = torch.Generator().manual_seed(3)
    rgb = torch.rand(rows * cols, 3, generator=g, dtype=torch.float64)
    colours = torch.cat([rgb, torch.ones(rows * cols, 1, dtype=torch.float64)], dim=1)
    rng = np.random.default_rng(0)
    samples = PR.regular_samples(h, w, 2) + rng.uniform(-0.2, 0.2, (h, w, 4, 2))  # jittered, still inside their pixel
    img = PR.polygon_render(xy, off, colours, h, w, samples)
    grid = rgb.T.reshape(1, 3, rows, cols)
    want = F.interpolate(grid, size=(h, w), mode="nearest")[0]
    assert torch.equal(img, want)


def test_oracle_render_is_linear_and_differentiable_in_the_colours():
    w, h = 20, 16
    rows, cols = PS.grid_for((w, h), "hex", pixel_size=[5, 6], verbose=False)
    xy, off = PS.polygons((w, h), rows, cols, "hex")
    n = len(off) - 1
    c = torch.rand(n, 4, dtype=torch.float64, requires_grad=True)
    samples = PR.regular_samples(h, w, 2)
    img = PR.polygon_render(xy, off, c, h, w, samples)
    g = torch.randn_like(img)
    (img * g).sum().backward()
    win = PR.polygon_winners(xy, off, h, w, samples)
    want = torch.zeros(n, 4, dtype=torch.float64)
    for s in range(4):
        for k in np.unique(win[s][win[s] >= 0]):
            want[k, :3] += 0.25 * g[:, torch.as_tensor(win[s] == k)].sum(dim=1)
    assert torch.allclose(c.grad, want, atol=1e-12, rtol=0)


# ---------------------------------------------------------------------------------------------------- API routing
class PolygonFakeEngine(FakeEngine):
    """FakeEngine plus the polygon drawer's surface: z = [n, 4] RGBA fills of the polygons it was built with."""

    def __init__(self, *, drawer=E.DRAWER_VQGAN, polygons=None, grid=None, **kw):
        super().__init__(drawer=drawer, grid=grid if grid is not None else (1, 1), **kw)
        if drawer == E.DRAWER_POLYGON:
            self.kw["polygons"] = polygons
            self.kw["grid"] = grid
            self.z_shape = (len(polygons[1]) - 1, 4)

    def set_synth_iteration(self, it):
        self._log("set_synth_iteration", it=it)

    def synth(self, z):
        """A flat image of the mean RGB of z (the default drawer's grid: 0.5), so a test can see which z was rendered."""
        self._log("synth", shape=tuple(z.shape))
        v = float(z[:, :3].mean()) if self.z_shape[1] == 4 else 0.5
        return torch.full((1, 3, *self.image_hw), v)


@pytest.fixture
def fake(monkeypatch, tmp_path):
    monkeypatch.setattr(api, "_engine_factory", PolygonFakeEngine)
    PolygonFakeEngine.loss_script = staticmethod(lambda it, n: np.full(n, 1.0 / (1 + it), dtype=np.float32))
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps({"ViT-B/16": [[0.1] * 512], "ViT-B/32": [[0.2] * 512]}))
    monkeypatch.setenv("PIXRAY_ROOT", str(tmp_path))
    api.reset_settings()
    yield
    api.reset_settings()


def _init(**kw):
    base = dict(prompts="x", clip_models="ViT-B/32", num_cuts=8, outdir="", seed="7", b200_allow_synthetic=True)
    base.update(kw)
    api.add_settings(**base)
    args = api.apply_settings()
    api.do_init(args)
    return args


def test_hex_reaches_the_engine_as_polygons_with_the_drawers_rate(fake, capsys):
    case = next(c for c in CASES if c["name"] == "hex_square_scale")
    _init(drawer="pixel", pixel_type="hex", size=case["size"], iterations=5, **case["settings"])
    assert "Running pixeldrawer with 16x22 grid" in capsys.readouterr().out
    eng = api._state.engine
    assert eng.kw["drawer"] == E.DRAWER_POLYGON
    xy, off = eng.kw["polygons"]
    assert np.array_equal(off, GOLD["hex_square_scale_off"])
    assert np.array_equal(xy.view(np.uint32), GOLD["hex_square_scale_xy"].view(np.uint32))
    d = api._state.drawer
    assert isinstance(d, P.PixelDrawer) and tuple(d.get_z().shape) == (len(off) - 1, 4)
    assert torch.all(d.get_z()[:, 3] == 1.0)
    assert api._state.lr == pytest.approx(0.03)
    assert d.get_opts(10) == [{"lr": pytest.approx(0.003)}]


def test_learning_rate_drops_divide_the_drawers_rate(fake):
    args = _init(drawer="pixel", pixel_type="diamond", size=[64, 64], pixel_scale=4.0, iterations=20,
                 learning_rate_drops=[50, 25])
    assert api.do_run(args) is True
    its = [round(c[1]["lr"], 8) for c in api._state.engine.calls if c[0] == "iterate"]
    assert its == [0.03] * 5 + [0.003] * 5 + [0.0003] * 10
    # the final checkin renders iteration 20's samples
    assert api._state.engine.calls[-2:] == [("set_synth_iteration", {"it": 20}), ("synth", {"shape": tuple(api._state.engine.z_shape)})]


def test_default_pixel_drawer_is_unchanged(fake):
    """pixel_type rect (the default) keeps the square-grid fast path: the same engine calls as before the shaped cells
    existed (recorded from the previous release: FastPixelDrawer, DRAWER_PIXEL, the global learning rate)."""
    args = _init(drawer="pixel", size=[64, 48], iterations=3)
    api.do_run(args)
    eng = api._state.engine
    assert isinstance(api._state.drawer, P.FastPixelDrawer)
    assert {k: v for k, v in eng.kw.items() if k != "clip"} == dict(
        drawer=E.DRAWER_PIXEL, image_hw=(48, 64), cutn=8, seed=798386561, grid=(45, 64), cut_aspect=4 / 3)
    assert eng.calls == [
        ("load_module", {"module": 1, "n": 152}), ("finalize", {}), ("set_prompts", {"clip": 0, "n": 2}),
        ("reset_optimizer", {}), ("iterate", {"lr": 0.2, "it": 0, "params": False}),
        ("iterate", {"lr": 0.2, "it": 1, "params": False}), ("reset_optimizer", {}),
        ("iterate", {"lr": 0.02, "it": 2, "params": False}), ("synth", {"shape": (1, 3, 45, 64)})]
    assert api._state.lr == pytest.approx(0.02)


def test_fast_pixel_does_not_gain_the_shape_options():
    api.reset_settings()
    api.add_settings(prompts="x", drawer="fast_pixel", pixel_type="hex")
    with pytest.raises(ValueError, match="Requested setting not found, aborting: pixel_type=hex"):
        api.apply_settings()
    api.reset_settings()
    api.add_settings(prompts="x", drawer="pixel", pixel_type="hex", pixel_edge_check=False)
    a = api.apply_settings()
    assert a.pixel_type == "hex" and a.pixel_edge_check is False and a.pixel_iso_check is True
    api.reset_settings()


def test_shaped_cells_need_a_start_image(fake):
    with pytest.raises(ValueError, match="init_image or use init_noise"):
        _init(drawer="pixel", pixel_type="hex", size=[32, 32], init_noise="none", iterations=2)


def test_unknown_pixel_type_is_refused_before_the_engine_is_built(fake, monkeypatch):
    built = []
    monkeypatch.setattr(api, "_engine_factory", lambda **kw: built.append(kw))
    with pytest.raises(ValueError, match="rect, rectshift, hex, tri, diamond, knit"):
        _init(drawer="pixel", pixel_type="octagon", size=[32, 32], iterations=2)
    assert built == []


def test_to_image_and_overlays_render_the_current_colours(fake):
    """to_image renders the current z (the fused iteration never calls drawer.synth, so a cached render would go stale),
    and every overlay re-encodes that current image (api.re_average_z: to_image -> reapply_from_tensor)."""
    _init(drawer="pixel", pixel_type="hex", size=[32, 24], pixel_scale=4.0, iterations=4)
    d = api._state.drawer
    with torch.no_grad():
        d.get_z()[:, :3] = 0.2
    assert np.asarray(d.to_image())[0, 0, 0] == int(0.2 * 255)
    with torch.no_grad():
        d.get_z()[:, :3] = 0.7
    assert np.asarray(d.to_image())[0, 0, 0] == int(0.7 * 255)       # the new colours, not the first render
    api.re_average_z(None)                                           # first overlay: re-encodes the 0.7 image
    assert torch.allclose(d.get_z()[:, :3], torch.tensor(int(0.7 * 255) / 255.0))
    with torch.no_grad():
        d.get_z()[:, :3] = 0.4                                       # optimisation moves the colours on
    api.re_average_z(None)                                           # second overlay: re-encodes the CURRENT image
    assert torch.allclose(d.get_z()[:, :3], torch.tensor(int(0.4 * 255) / 255.0))
    assert torch.all(d.get_z()[:, 3] == 1.0)
