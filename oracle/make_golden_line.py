"""Generate tests/golden/line_sketch.npz by running the REAL reference LineDrawer (linedrawer.py) (container-only).

    python -m oracle.make_golden_line

diffvg, ttools and skimage are not installed here; they are registered as stub modules before the reference is
imported.  The pydiffvg stub renders whatever RGBA image the case sets (colours are kept as float32, see
shape_group); the render itself is the engine's job and is checked against oracle/stroke_ref.py, not against this
fixture.
tests/test_line_sketch.py requires plugins.LineDrawer to reproduce, per case: the start points (bit for bit after
random.seed), the start widths, the rates of get_opts(1) and get_opts(10), clip_z on out-of-range widths, and synth's
composite of a recorded RGBA render (on the small canvas).
"""
import json
import os
import random
import sys
import types
from types import SimpleNamespace

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "line_sketch.npz")


class _Recorder:
    def __init__(self):
        self.render = None


REC = _Recorder()


def _install_stubs():
    def path(num_control_points, points, stroke_width, is_closed):
        return SimpleNamespace(num_control_points=num_control_points, points=points, stroke_width=stroke_width,
                               is_closed=is_closed)

    def rect(p_min, p_max):
        return SimpleNamespace(p_min=p_min, p_max=p_max)

    def shape_group(shape_ids, fill_color=None, stroke_color=None):
        # linedrawer.py:97 builds the stroke colour from ints (an int64 tensor), on which its own clip_z fails in
        # current torch ("result type Float can't be cast"); the stub keeps colours as float32, the type diffvg renders
        to_f = lambda c: None if c is None else c.float()  # noqa: E731
        return SimpleNamespace(shape_ids=shape_ids, fill_color=to_f(fill_color), stroke_color=to_f(stroke_color))

    class RenderFunction:
        @staticmethod
        def serialize_scene(*a, **k):
            return []

        @staticmethod
        def apply(width, height, *a):
            return REC.render.clone() if REC.render is not None else torch.zeros(height, width, 4)

    m = types.ModuleType("pydiffvg")
    m.Path, m.Rect, m.ShapeGroup, m.RenderFunction = path, rect, shape_group, RenderFunction
    m.set_use_gpu = m.set_device = lambda *a, **k: None
    m.get_device = lambda: torch.device("cpu")
    sys.modules["pydiffvg"] = m
    ttools = types.ModuleType("ttools")
    ttools.modules = types.ModuleType("ttools.modules")
    sys.modules["ttools"], sys.modules["ttools.modules"] = ttools, ttools.modules
    sk = types.ModuleType("skimage")
    sk.io = types.ModuleType("skimage.io")
    sys.modules["skimage"], sys.modules["skimage.io"] = sk, sk.io


# (name, (width, height), settings beyond the defaults, random seed)
CASES = [
    ("default_landscape", (384, 216), {}, 11),
    ("default_square", (256, 256), {}, 12),
    ("portrait_short", (120, 200), dict(strokes=5, stroke_length=3), 13),
    ("wide_thick_paper", (300, 100), dict(strokes=7, stroke_length=2, max_stroke_width=5.0, allow_paper_color=True), 14),
    ("one_segment", (64, 48), dict(strokes=3, stroke_length=1, min_stroke_width=1.0, max_stroke_width=10.0), 15),
]


def main():
    _install_stubs()
    from oracle import shim
    shim.install()
    from linedrawer import LineDrawer

    G, meta = {}, []
    for name, (w, h), extra, seed in CASES:
        s = dict(size=[w, h], strokes=24, stroke_length=8, min_stroke_width=0.5, max_stroke_width=2,
                 allow_paper_color=False)
        s.update(extra)
        settings = SimpleNamespace(**s)
        d = LineDrawer(settings)
        REC.render = None
        random.seed(seed)
        d.load_model(settings, None)
        G[name + "_points"] = torch.stack([p.points.detach() for p in d.shapes[1:]]).numpy()
        G[name + "_widths"] = torch.stack([p.stroke_width.detach() for p in d.shapes[1:]]).numpy()
        G[name + "_rates1"] = np.array([o.param_groups[0]["lr"] for o in d.get_opts(1)])
        G[name + "_rates10"] = np.array([o.param_groups[0]["lr"] for o in d.get_opts(10)])
        gen = torch.Generator().manual_seed(seed)
        wild = (torch.rand(len(d.shapes) - 1, generator=gen) * 3 - 1) * d.max_width  # below 1, inside, above max_width
        with torch.no_grad():
            for p, v in zip(d.shapes[1:], wild):
                p.stroke_width.copy_(v)
        d.clip_z()
        G[name + "_clip_in"] = wild.numpy()
        G[name + "_clip_out"] = torch.stack([p.stroke_width.detach() for p in d.shapes[1:]]).numpy()
        if w * h <= 4096:  # the composite is per pixel: one small canvas pins it (and keeps the fixture small)
            REC.render = torch.rand(h, w, 4, generator=gen) * 1.2 - 0.1  # any RGBA, alpha outside [0, 1] included
            G[name + "_render"] = REC.render.numpy()
            G[name + "_synth"] = d.synth(3).detach().numpy()
        meta.append(dict(name=name, size=[w, h], settings=extra, seed=seed, max_width=d.max_width))
    G["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **G)
    print(f"wrote {OUT}: {len(meta)} cases")


if __name__ == "__main__":
    main()
