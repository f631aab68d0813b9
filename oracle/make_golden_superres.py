"""Generate tests/golden/super_resolution.npz by running the REAL reference SuperResolutionDrawer (super_resolution.py,
real_esrganer.py) (container-only).

    python -m oracle.make_golden_superres

basicsr is not vendored: basicsr.archs.rrdbnet_arch is registered as a stub module whose RRDBNet holds the checkpoint's
tensors and evaluates oracle/rrdbnet_ref.py, and basicsr.utils.download_util as an empty stub.  The stubs go in before
the reference is imported (pixray's class_table drops the drawer otherwise).  The drawer loads the seeded full-depth
weights (pixray_b200.synthetic.rrdbnet_state_dict) from models/super_resolution_RealESRGAN_x4plus.ckpt in a scratch
working directory, under params_ema as Real-ESRGAN ships them, and runs init_from_tensor, synth, backward and clip_z as
written.  The fixture pins the drawer's own steps (the bilinear quarter-size init, enhance at tile 0 / pre_pad 0 being
exactly model(z), clamp_with_grad, the [0, 1] clip); the 67 MB of weights are regenerated from the seed, and a few
slices of them are stored so that a change of the generator is caught.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "super_resolution.npz")
SEED = 0
CASES = {"a": (34, 48, 11), "b": (37, 50, 12)}  # init tensor height, width, numpy seed


def _install_stubs():
    from oracle import rrdbnet_ref as RR

    class RRDBNet(nn.Module):
        def __init__(self, num_in_ch, num_out_ch, num_feat=64, num_block=23, num_grow_ch=32, scale=4):
            super().__init__()
            assert (num_in_ch, num_out_ch, scale) == (3, 3, 4)
            conv = lambda cin, cout: nn.Conv2d(cin, cout, 3, 1, 1)  # noqa: E731
            nf, gc = num_feat, num_grow_ch
            self.conv_first = conv(3, nf)
            self.body = nn.ModuleList()
            for _ in range(num_block):
                rrdb = nn.Module()
                for j in (1, 2, 3):
                    rdb = nn.Module()
                    for k in range(1, 6):
                        setattr(rdb, f"conv{k}", conv(nf + gc * (k - 1), gc if k < 5 else nf))
                    setattr(rrdb, f"rdb{j}", rdb)
                self.body.append(rrdb)
            self.conv_body, self.conv_up1, self.conv_up2, self.conv_hr = (conv(nf, nf) for _ in range(4))
            self.conv_last = conv(nf, 3)

        def forward(self, x):
            return RR.rrdbnet(x, dict(self.named_parameters()))

    basicsr = types.ModuleType("basicsr")
    archs = types.ModuleType("basicsr.archs")
    arch = types.ModuleType("basicsr.archs.rrdbnet_arch")
    arch.RRDBNet = RRDBNet
    utils = types.ModuleType("basicsr.utils")
    dl = types.ModuleType("basicsr.utils.download_util")
    dl.load_file_from_url = lambda *a, **k: None
    for name, m in (("basicsr", basicsr), ("basicsr.archs", archs), ("basicsr.archs.rrdbnet_arch", arch),
                    ("basicsr.utils", utils), ("basicsr.utils.download_util", dl)):
        sys.modules[name] = m


def main():
    from pixray_b200 import synthetic as S
    sys.path.insert(0, ROOT)
    _install_stubs()
    from oracle import shim
    shim.install()
    import super_resolution as SR

    sd = S.rrdbnet_state_dict(SEED)
    out = {"seed": np.int64(SEED)}
    for k in ("conv_first.weight", "body.0.rdb1.conv1.weight", "body.22.rdb3.conv5.weight", "conv_last.bias",
              "conv_hr.weight"):
        out["w:" + k] = sd[k].numpy().ravel()[:64].copy()
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            os.makedirs("models")
            torch.save({"params_ema": sd}, "models/super_resolution_RealESRGAN_x4plus.ckpt")
            drawer = SR.SuperResolutionDrawer(types.SimpleNamespace(super_resolution_model="RealESRGAN_x4plus"))
            drawer.load_model(None, torch.device("cpu"))
            for case, (h, w, seed) in CASES.items():
                init = np.random.default_rng(seed).random((1, 3, h, w), dtype=np.float32) * np.float32(2) - np.float32(1)
                drawer.init_from_tensor(torch.from_numpy(init))
                z = drawer.get_z().detach().clone()
                img = drawer.synth(0)
                g = torch.from_numpy(np.random.default_rng(seed + 100).standard_normal(img.shape).astype(np.float32))
                img.backward(g)
                out[f"{case}_init"] = init
                out[f"{case}_z"] = z.numpy()
                out[f"{case}_image"] = img.detach().numpy()
                out[f"{case}_g"] = g.numpy()
                out[f"{case}_zgrad"] = drawer.get_z().grad.numpy()
                drawer.clip_z()
                out[f"{case}_clip_z"] = drawer.get_z().detach().numpy()
                print(f"case {case}: init {h}x{w} -> z {tuple(z.shape[-2:])} -> image {tuple(img.shape[-2:])}")
        finally:
            os.chdir(cwd)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
