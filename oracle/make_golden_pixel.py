"""Generate tests/golden/pixel_shapes.npz by running the REAL reference PixelDrawer (pixeldrawer.py) (container-only).

    python -m oracle.make_golden_pixel

PixelDrawer.__init__ derives the grid and encode_image builds one diffvg Polygon + ShapeGroup per cell.  diffvg,
ttools and skimage are not installed here; they are registered as stub modules before the reference is imported.  The
pydiffvg stub records every Polygon's points and every ShapeGroup's fill colour and renders nothing -- the render is the
engine's job and is checked against oracle/polygon_ref.py, not against this fixture.  tests/test_pixel_shapes.py
requires pixray_b200/pixel_shapes.py to reproduce the recorded grid counts, vertices (bit for bit) and colours.

Init images come from numpy's PCG64 (stable across versions), so the fixture stores seeds, not pixels.
"""
import json
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "pixel_shapes.npz")
TYPES = ("rect", "rectshift", "hex", "tri", "diamond", "knit")


def init_image(seed, width, height):
    """The start image of a case: [1, 3, height, width] float32 in [-1, 1)."""
    return np.random.default_rng(seed).random((1, 3, height, width), dtype=np.float32) * np.float32(2.0) - np.float32(1.0)


class _Recorder:
    def __init__(self):
        self.points, self.fills = [], []


REC = _Recorder()


def _install_stubs():
    def polygon(points, is_closed):
        REC.points.append(points.detach().clone())
        return SimpleNamespace(points=points, is_closed=is_closed)

    def shape_group(shape_ids, stroke_color=None, fill_color=None):
        REC.fills.append(fill_color.detach().clone())
        return SimpleNamespace(shape_ids=shape_ids, fill_color=fill_color)

    class RenderFunction:
        @staticmethod
        def serialize_scene(*a, **k):
            return []

        @staticmethod
        def apply(width, height, *a):
            return torch.zeros(height, width, 4)

    m = types.ModuleType("pydiffvg")
    m.Polygon, m.ShapeGroup, m.RenderFunction = polygon, shape_group, RenderFunction
    m.set_use_gpu = m.set_device = lambda *a, **k: None
    sys.modules["pydiffvg"] = m
    ttools = types.ModuleType("ttools")
    ttools.modules = types.ModuleType("ttools.modules")
    sys.modules["ttools"], sys.modules["ttools.modules"] = ttools, ttools.modules
    sk = types.ModuleType("skimage")
    sk.io = types.ModuleType("skimage.io")
    sys.modules["skimage"], sys.modules["skimage.io"] = sk, sk.io


# (name, (width, height), settings beyond the defaults, init seed or None for a grid-only case)
def _cases():
    out = []
    for t in TYPES:
        out += [
            (f"{t}_square_scale", (100, 100), dict(pixel_scale=2.5), 11),
            (f"{t}_portrait_scale", (90, 130), dict(pixel_scale=3.0), 12),
            (f"{t}_landscape_size", (150, 84), dict(pixel_size=[17, 9]), 13),
            (f"{t}_landscape_checks_off", (120, 70), dict(pixel_scale=4.0, pixel_edge_check=False, pixel_iso_check=False), 14),
            (f"{t}_square_default", (256, 256), {}, None),
            (f"{t}_portrait_default", (200, 250), {}, None),
            (f"{t}_landscape_default", (384, 216), {}, None),
            (f"{t}_clamped", (30, 20), dict(pixel_size=[50, 40]), None),
        ]
    return out


def main():
    _install_stubs()
    from oracle import shim
    shim.install()
    from pixeldrawer import PixelDrawer

    G, meta = {}, []
    for name, (w, h), extra, seed in _cases():
        s = dict(size=[w, h], pixel_size=None, pixel_scale=None, pixel_type=name.split("_")[0], pixel_edge_check=True,
                 pixel_iso_check=True, transparent=False)
        s.update(extra)
        d = PixelDrawer(SimpleNamespace(**s))
        meta.append(dict(name=name, size=[w, h], settings=extra, pixel_type=s["pixel_type"], rows=d.num_rows,
                         cols=d.num_cols, seed=seed))
        if seed is None:
            continue
        REC.points.clear()
        REC.fills.clear()
        d.encode_image(torch.from_numpy(init_image(seed, w, h)))
        G[name + "_xy"] = torch.cat(REC.points).numpy().astype(np.float32)
        G[name + "_off"] = np.cumsum([0] + [p.shape[0] for p in REC.points]).astype(np.int32)
        G[name + "_rgba"] = torch.stack(REC.fills).numpy().astype(np.float32)
    G["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **G)
    print(f"wrote {OUT}: {len(meta)} cases")


if __name__ == "__main__":
    main()
