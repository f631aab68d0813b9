"""Generate tests/golden/vdiff_canvas.npz by running the REAL reference VdiffDrawer (vdiff.py) (container-only).

    python -m oracle.make_golden_vdiff_canvas

The drawer is built through its own __init__ from a settings namespace; load_model (which downloads a checkpoint) is
replaced by setting a stub model that returns a fixed v, so synth's arithmetic and its centre crop, and
init_from_tensor's reverse crop, are the reference's own code.  Per canvas the fixture records:
  gen size and margins (VdiffDrawer.gen_width / gen_height, the int((gen - canvas) / 2) of synth);
  synth's output for a known x / v at one step (the clamped prediction, cropped when a margin is non-zero), on canvases
  above 4096 pixels every 4th row and column of it and its full last row and column;
  the gen-size frame init_from_tensor builds from a known start tensor, before it is noised: the call runs with its
  noise draw returning zeros, so it records frame * alpha_0 (+ 0 * sigma_0) and alpha_0.
x, v and the start tensor are integer patterns over the pixel index (no random numbers: the fixture stays small and
the tests can rebuild them), each a different residue mod 97 per pixel, so a shifted crop cannot match.
When both margins are zero the reference does not crop: its image is the whole gen-size frame, and so is the start
tensor it takes (a canvas-size one would not broadcast against x), which is what the case records.
tests/test_vdiff_canvas.py checks pixray_b200.util's gen size / margins, the crop and VdiffDrawer.init_from_tensor.
"""
import json
import os
from types import SimpleNamespace

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "vdiff_canvas.npz")

# (name, (width, height)): pixray's quality x aspect presets, then the edges of the round-up
CANVASES = [
    ("normal_widescreen", (384, 216)),
    ("normal_square", (288, 288)),
    ("normal_portrait", (256, 320)),
    ("draft_widescreen", (192, 108)),
    ("draft_square", (144, 144)),
    ("better_widescreen", (576, 324)),
    ("best_widescreen", (768, 432)),
    ("square_512", (512, 512)),
    ("tiny_64", (64, 64)),
    ("odd_127", (127, 127)),
    ("odd_129x100", (129, 100)),
    ("no_crop_255", (255, 255)),
    ("wide_200x100", (200, 100)),
    ("tall_100x200", (100, 200)),
]
ITERATIONS, STEP = 20, 7


def pattern(shape, a, b, c):
    """[1, 3, h, w] float32 in [-1, 1): ((a ch + b row + c col) mod 97) / 48 - 1 (tests/test_vdiff_canvas.py rebuilds it)."""
    _, ch, h, w = shape
    k = torch.arange(ch).view(1, ch, 1, 1) * a + torch.arange(h).view(1, 1, h, 1) * b + torch.arange(w).view(1, 1, 1, w) * c
    return (k % 97).float() / 48 - 1


class _FixedV(torch.nn.Module):
    """Stands in for the diffusion model: returns the case's v whatever it is given."""

    def __init__(self, v):
        super().__init__()
        self.v = v

    def forward(self, x, t, **kw):
        return self.v.clone()


def main():
    from oracle import shim
    shim.install()
    from vdiff import VdiffDrawer

    G, meta = {}, []
    for k, (name, (w, h)) in enumerate(CANVASES):
        settings = SimpleNamespace(vdiff_model="cc12m_1", size=[w, h], iterations=ITERATIONS, vdiff_schedule="default",
                                   clip_models=["ViT-B/16"], vdiff_skip=0)
        d = VdiffDrawer(settings)
        gw, gh = d.gen_width, d.gen_height
        mx, my = int((gw - w) / 2), int((gh - h) / 2)
        v = pattern((1, 3, gh, gw), 29, 13, 5)
        d.model, d.device, d.pred, d.v = _FixedV(v), torch.device("cpu"), None, None
        # init_from_tensor with its noise draw returning zeros: x = frame * alpha_0
        cropped = mx != 0 or my != 0
        start = pattern((1, 3, h, w) if cropped else (1, 3, gh, gw), 41, 7, 3)
        randn = torch.randn
        torch.randn = lambda *a, **kw: torch.zeros(*a, **{q: u for q, u in kw.items() if q != "generator"})
        try:
            d.init_from_tensor(start)
        finally:
            torch.randn = randn
        init_x = d.x.detach().clone()
        a0 = float(d.sample_state[5][0])
        # synth at one step for a known x
        x = pattern((1, 3, gh, gw), 31, 11, 19) * float(d.sample_state[6][STEP])
        d.x = x.clone().requires_grad_(True)
        out = d.synth(STEP).detach()
        # large canvases keep every 4th row and column, plus the full last row and column (the window's far edges)
        stride = 4 if w * h > 4096 else 1
        G[name + "_synth"] = out[:, :, ::stride, ::stride].numpy()
        G[name + "_synth_last_row"] = out[:, :, -1, :].numpy()
        G[name + "_synth_last_col"] = out[:, :, :, -1].numpy()
        G[name + "_init_x"] = init_x.numpy()
        G[name + "_coefs"] = np.array([float(d.sample_state[5][STEP]), float(d.sample_state[6][STEP]), a0,
                                       float(d.sample_state[6][0])], dtype=np.float64)
        meta.append(dict(name=name, size=[w, h], gen=[gw, gh], margins=[mx, my], step=STEP, iterations=ITERATIONS,
                         synth_shape=list(out.shape), synth_stride=stride))
    G["cases"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **G)
    print(f"wrote {OUT}: {len(meta)} cases")


if __name__ == "__main__":
    main()
