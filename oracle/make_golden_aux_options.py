"""Generate tests/golden/aux_loss_options.npz (and the two PNGs it reads) by running the REAL reference SmoothnessLoss
and EdgeLoss (container-only) on the options beyond make_golden_aux.py's: the smoothness pre-blur and edge_order 2,
and the edge loss's target and mask images.

    python -m oracle.make_golden_aux_options

Each case holds one get_loss call of the unmodified class (imported under oracle/shim.py) with its value and autograd
gradient; tests/test_aux_loss_options.py requires oracle/aux_ref.py to reproduce them and pixray_b200.losses to
reproduce the resized target and mask.  EdgeLoss.get_loss calls `torch.tensor(0.0).cuda()`; Tensor.cuda is patched to
the identity for those calls, as in make_golden_aux.py.
"""
import os
import types

import numpy as np
import torch
from PIL import Image

from oracle import shim

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
OUT = os.path.join(GOLDEN, "aux_loss_options.npz")
TARGET_PNG = os.path.join(GOLDEN, "edge_target.png")
MASK_PNG = os.path.join(GOLDEN, "edge_mask.png")

# (tag, type, kernel, std, spacing, edge_order)
SMOOTH_CASES = [(f"smooth_k{k}_s{s}".replace(".", "p"), "default", k, s, 1, 1) for k in (3, 4.5, 7) for s in (1, 2.5)] + [
    ("smooth_clipped_k4p5", "clipped", 4.5, 1.0, 1, 1),
    ("smooth_log_k4p5", "log", 4.5, 1.0, 1, 1),
    ("smooth_o2_sp1", "default", 0, 1.0, 1, 2),
    ("smooth_o2_sp2", "log", 0, 1.0, 2, 2),
    ("smooth_o2_sp1_k5", "default", 5, 1.5, 1, 2),
    ("smooth_o2_sp2_k4p5", "clipped", 4.5, 1.0, 2, 2),
]
# (tag, out H, W, margins (percent), image?, mask?)
EDGE_CASES = [
    ("edge_image", 24, 24, (10, 20, 15, 0), True, False),
    ("edge_mask", 24, 24, (10, 10, 10, 10), False, True),
    ("edge_image_mask", 24, 24, (10, 10, 10, 10), True, True),
    ("edge_nonsquare", 20, 28, (5, 15, 10, 25), True, False),
    ("edge_nonsquare_mask", 20, 28, (5, 5, 5, 5), True, True),
]


def _write_pngs():
    yy, xx = np.mgrid[0:29, 0:37].astype(np.float64)
    rgb = np.stack([128 + 120 * np.sin(xx / 5.0), 128 + 120 * np.cos(yy / 4.0 + xx / 9.0),
                    np.where((xx // 6 + yy // 5) % 2 == 0, 230.0, 20.0)], -1)
    Image.fromarray(np.clip(rgb, 0, 255).astype(np.uint8), "RGB").save(TARGET_PNG)
    yy, xx = np.mgrid[0:23, 0:31].astype(np.float64)
    m = np.where((xx - 15) ** 2 / 100.0 + (yy - 11) ** 2 / 49.0 < 1.0, 0, 255).astype(np.float64)
    m[:, :3] = 0
    m[20:, :] = 128  # a grey band: the threshold is > 0 of the resized values, ringing included
    Image.fromarray(m.astype(np.uint8), "L").save(MASK_PNG)


def main():
    shim.install()
    from Losses.EdgeLoss import EdgeLoss
    from Losses.SmoothnessLoss import SmoothnessLoss

    _write_pngs()
    G = {}
    g = torch.Generator().manual_seed(2468)
    cut = torch.rand(4, 3, 16, 16, generator=g) * 1.2 - 0.1
    G["cut"] = cut.numpy()
    for tag, kind, k, s, sp, order in SMOOTH_CASES:
        c = cut.clone().requires_grad_(True)
        args = types.SimpleNamespace(smoothness_weight=0.9, smoothness_type=kind, smoothness_gaussian_kernel=k,
                                     smoothness_gaussian_std=s, smoothness_spacing=sp, smoothness_edge_order=order)
        val = sum(SmoothnessLoss(device="cpu").get_loss({16: c}, None, args))
        val.backward()
        G[tag + "_val"], G[tag + "_grad"] = val.detach().numpy(), c.grad.numpy()
        G[tag + "_cfg"] = np.array([{"default": 0, "clipped": 1, "log": 2}[kind], k, s, sp, order], dtype=np.float64)

    orig_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **kw: self
    try:
        for tag, H, W, margins, use_img, use_mask in EDGE_CASES:
            out = torch.rand(1, 3, H, W, generator=g)
            el = EdgeLoss(device="cpu")
            args = types.SimpleNamespace(edge_thickness=5, edge_margins=list(margins), edge_color="[0.2+0.6+0.9]",
                                         edge_color_weight=0.1, global_color_weight=0.05,
                                         edge_input_image=TARGET_PNG if use_img else "",
                                         edge_mask_image=MASK_PNG if use_mask else "")
            args = el.parse_settings(args)
            o = out.clone().requires_grad_(True)
            val = el.get_loss({}, o, args)
            val.backward()
            G[tag + "_out"], G[tag + "_val"], G[tag + "_grad"] = out.numpy(), val.detach().numpy(), o.grad.numpy()
            G[tag + "_cfg"] = np.array(list(margins) + [int(use_img), int(use_mask)], dtype=np.int32)
            if use_img:
                G[tag + "_target"] = el.resized.numpy()
            if use_mask:
                G[tag + "_mask"] = el.resized_mask.numpy()
    finally:
        torch.Tensor.cuda = orig_cuda
    G["edge_color"] = np.array([0.2, 0.6, 0.9], dtype=np.float32)
    np.savez_compressed(OUT, **G)
    print("wrote", OUT, "with", len(G), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
