"""The vdiff drawer at any canvas size, on the host: the U-Net size and margins (pixray_b200.util.vdiff_gen_size), the
centre crop of synth, VdiffDrawer.init_from_tensor's reverse crop and what api.do_init hands the engine, against
tests/golden/vdiff_canvas.npz, which oracle/make_golden_vdiff_canvas.py records from the reference's own VdiffDrawer
(vdiff.py:55-58, 131-143, 159-170).  The engine does the crop itself on the GPU; tests/test_vdiff_canvas_gpu.py ties it
to the same margins."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import plugins as P
from pixray_b200 import util as U

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "vdiff_canvas.npz"))
CASES = json.loads(str(GOLD["cases"]))
IDS = [c["name"] for c in CASES]


def pattern(shape, a, b, c):
    """oracle/make_golden_vdiff_canvas.py's inputs: ((a ch + b row + c col) mod 97) / 48 - 1."""
    _, ch, h, w = shape
    k = torch.arange(ch).view(1, ch, 1, 1) * a + torch.arange(h).view(1, 1, h, 1) * b + torch.arange(w).view(1, 1, 1, w) * c
    return (k % 97).float() / 48 - 1


def _crop(img, w, h):
    gw, gh, mx, my = U.vdiff_gen_size(w, h)
    if mx or my:
        return img[:, :, my:my + h, mx:mx + w]
    return img


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_gen_size_and_margins(case):
    w, h = case["size"]
    gw, gh, mx, my = U.vdiff_gen_size(w, h)
    assert [gw, gh] == case["gen"] and [mx, my] == case["margins"]
    assert gw % 128 == 0 and gh % 128 == 0
    want = (w, h) if (mx or my) else (gw, gh)
    assert U.vdiff_image_size(w, h) == want
    assert list(GOLD[case["name"] + "_synth_last_row"].shape[-1:]) == [want[0]]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_synth_crop(case):
    """clamp((x alpha - v sigma + 1) / 2) cropped at the helper's margins is the reference's synth output."""
    name, (w, h), (gw, gh) = case["name"], case["size"], case["gen"]
    alpha, sigma = (torch.tensor(c, dtype=torch.float32) for c in GOLD[name + "_coefs"][:2])
    x = pattern((1, 3, gh, gw), 31, 11, 19) * sigma
    v = pattern((1, 3, gh, gw), 29, 13, 5)
    out = _crop(((x * alpha - v * sigma).add(1).div(2)).clamp(0, 1), w, h)
    assert list(out.shape) == case["synth_shape"]
    s = case["synth_stride"]
    np.testing.assert_allclose(out[:, :, ::s, ::s].numpy(), GOLD[name + "_synth"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(out[:, :, -1, :].numpy(), GOLD[name + "_synth_last_row"], rtol=0, atol=1e-6)
    np.testing.assert_allclose(out[:, :, :, -1].numpy(), GOLD[name + "_synth_last_col"], rtol=0, atol=1e-6)


class _StandIn:
    """The engine surface VdiffDrawer.init_from_tensor uses: z_shape (gen), image_hw (canvas), the schedule setter."""

    def __init__(self, image_hw, gen_hw):
        self.device = torch.device("cpu")
        self.image_hw = tuple(image_hw)
        self.z_shape = (1, 3, gen_hw[0], gen_hw[1])
        self.schedule = None

    def vdiff_set_schedule(self, steps, alphas, sigmas):
        self.schedule = (steps, alphas, sigmas)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_init_from_tensor_reverse_crop(case):
    """x = frame * alpha_0 + noise * sigma_0 with the start image placed at the margins of a zero gen-size frame."""
    name, (w, h), (gw, gh) = case["name"], case["size"], case["gen"]
    iw, ih = U.vdiff_image_size(w, h)
    eng = _StandIn((ih, iw), (gh, gw))
    d = P.VdiffDrawer(SimpleNamespace(iterations=case["iterations"], vdiff_skip=0), SimpleNamespace(engine=eng))
    start = pattern((1, 3, ih, iw), 41, 7, 3)
    d.init_from_tensor(start, seed=5)
    noise = torch.randn(eng.z_shape, generator=torch.Generator().manual_seed(5))
    a0, s0 = float(d.alphas[0]), float(d.sigmas[0])
    assert abs(a0 - GOLD[name + "_coefs"][2]) <= 1e-7 and abs(s0 - GOLD[name + "_coefs"][3]) <= 1e-7
    assert tuple(d.x.shape) == (1, 3, gh, gw)
    np.testing.assert_allclose((d.x - noise * s0).numpy(), GOLD[name + "_init_x"], rtol=0, atol=1e-6)
    frame = d.gen_frame(start)
    a0_ref = torch.tensor(GOLD[name + "_coefs"][2], dtype=torch.float32)  # the reference's own alpha_0, to the bit
    np.testing.assert_array_equal((frame * a0_ref).numpy(), GOLD[name + "_init_x"])


def _default_init(tmp_path, monkeypatch, **kw):
    monkeypatch.setattr(api, "_engine_factory", FakeEngine)
    api.reset_settings()
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps({"ViT-B/16": [[0.1] * 512]}))
    monkeypatch.setenv("PIXRAY_ROOT", str(tmp_path))
    api.add_settings(prompts="a lighthouse", drawer="vdiff", clip_models="ViT-B/16", outdir="", seed="7",
                     b200_allow_synthetic=True, **kw)
    try:
        return api.do_init(api.apply_settings())
    finally:
        api.reset_settings()


def test_do_init_hands_the_engine_canvas_and_gen_size(tmp_path, monkeypatch):
    """Default settings (384 x 216): the canvas is the image, the U-Net runs at 384 x 256."""
    _default_init(tmp_path, monkeypatch)
    eng = api._state.engine
    assert eng.kw["drawer"] == E.DRAWER_VDIFF
    assert eng.kw["image_hw"] == (216, 384)
    assert eng.kw["vdiff_gen_hw"] == (256, 384)


@pytest.mark.parametrize("size,image_hw,gen_hw", [([255, 255], (256, 256), (256, 256)), ([64, 64], (64, 64), (128, 128)),
                                                   ([256, 256], (256, 256), (256, 256))])
def test_do_init_edges(tmp_path, monkeypatch, size, image_hw, gen_hw):
    """No margin to cut: the image is the gen-size frame.  A 64-pixel side runs the U-Net at 128 and crops."""
    _default_init(tmp_path, monkeypatch, size=size)
    eng = api._state.engine
    assert eng.kw["image_hw"] == image_hw and eng.kw["vdiff_gen_hw"] == gen_hw
