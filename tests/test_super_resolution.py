"""The super-resolution drawer on the CPU: the restated RRDBNet (oracle/rrdbnet_ref.py) and the settings / init / weight
plumbing of api.py and plugins.SuperResolutionDrawer, against a recording stand-in for the engine."""
import os

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from oracle import rrdbnet_ref as RR
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import plugins as P
from pixray_b200 import synthetic as S

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "super_resolution.npz")


class SuperResFakeEngine(FakeEngine):
    """The recording engine with the super-resolution drawer's latent: z = [1, 3, H/4, W/4]."""

    def __init__(self, *, drawer=E.DRAWER_VQGAN, image_hw=(256, 256), grid=None, **kw):
        super().__init__(drawer=drawer, image_hw=image_hw, grid=grid or (1, 1), **kw)
        if drawer == E.DRAWER_SUPERRES:
            self.z_shape = (1, 3, image_hw[0] // 4, image_hw[1] // 4)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", SuperResFakeEngine)
    api.reset_settings()
    yield
    api.reset_settings()


def _settings(tmp_path, **kw):
    from PIL import Image
    rgb = (np.random.default_rng(4).random((38, 50, 3)) * 255).astype(np.uint8)
    Image.fromarray(rgb).save(tmp_path / "init.png")
    base = dict(prompts="a cat", drawer="super_resolution", size=[50, 38], clip_models="ViT-B/32", num_cuts=4, outdir="",
                seed="3", b200_allow_synthetic=True, vector_prompts="none", init_image=str(tmp_path / "init.png"))
    base.update(kw)
    return base


def _init(tmp_path, **kw):
    api.add_settings(**_settings(tmp_path, **kw))
    args = api.apply_settings()
    api.do_init(args)
    return args


# ---------------------------------------------------------------------------------------------- the restated network
def test_oracle_reproduces_the_reference_drawer():
    """tests/golden/super_resolution.npz, written by oracle/make_golden_superres.py from the unmodified reference drawer
    with the seeded full-depth weights: z after the bilinear init bit for bit, the image and z.grad to 1e-5."""
    d = np.load(GOLDEN)
    sd = S.rrdbnet_state_dict(int(d["seed"]))
    for k in [k for k in d.files if k.startswith("w:")]:
        assert np.array_equal(sd[k[2:]].numpy().ravel()[:d[k].size], d[k]), k
    for case in ("a", "b"):
        init = torch.from_numpy(d[f"{case}_init"])
        z = RR.latent_from_tensor(init)
        assert np.array_equal(z.numpy(), d[f"{case}_z"])
        z = z.clone().requires_grad_(True)
        img = RR.superres_synth(z, sd)
        assert np.abs(img.detach().numpy() - d[f"{case}_image"]).max() <= 1e-5
        img.backward(torch.from_numpy(d[f"{case}_g"]))
        g_ref = d[f"{case}_zgrad"]
        assert np.abs(z.grad.numpy() - g_ref).max() <= 1e-5 * max(1.0, np.abs(g_ref).max())
        assert np.array_equal(z.detach().clip(0, 1).numpy(), d[f"{case}_clip_z"])


def test_matched_rounding_oracle_stays_close_to_fp32():
    sd = S.rrdbnet_state_dict(1, num_block=2)
    z = torch.rand(1, 3, 6, 5, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    a, b = RR.rrdbnet(z, sd), RR.rrdbnet(z, sd, matched=True)
    assert a.shape == (1, 3, 24, 20) and 0 < (a - b).abs().max().item() <= 5e-3


def test_synthetic_weights_land_inside_the_clamp():
    sd = S.rrdbnet_state_dict(0, num_block=2)
    out = RR.rrdbnet(torch.rand(1, 3, 8, 8, generator=torch.Generator().manual_seed(0)), sd)
    assert ((out > 0) & (out < 1)).float().mean().item() >= 0.9
    assert abs(S.superres_fwd_flops(1, 1) / 1e6 - 35.85) < 0.01


# ---------------------------------------------------------------------------------------------- settings and plumbing
def test_settings_and_model_names(fake, tmp_path):
    api.add_settings(**_settings(tmp_path))
    assert api.apply_settings().super_resolution_model == "RealESRGAN_x4plus"
    api.reset_settings()
    api.add_settings(**_settings(tmp_path, super_resolution_model="RealESRGAN_x2plus"))
    with pytest.raises(ValueError, match="checkpoint table"):
        api.do_init(api.apply_settings())
    api.reset_settings()
    api.add_settings(**_settings(tmp_path, vqgan_model="imagenet_f16_16384"))
    with pytest.raises(ValueError, match="Requested setting not found"):
        api.apply_settings()


def test_canvas_is_truncated_to_a_multiple_of_4(fake, tmp_path):
    _init(tmp_path)
    st = api._state
    assert st.engine.kw["drawer"] == E.DRAWER_SUPERRES and st.engine.kw["image_hw"] == (36, 48)
    assert st.engine.kw["cut_aspect"] == pytest.approx(50 / 38)  # global_aspect_width from the requested size
    assert tuple(st.drawer.get_z().shape) == (1, 3, 9, 12)
    assert float(st.drawer.get_z().min()) >= 0.0 and float(st.drawer.get_z().max()) <= 1.0
    assert st.drawer.get_opts(1) is None and st.drawer.get_num_resolutions() is None


def test_start_image_is_required(fake, tmp_path):
    with pytest.raises(ValueError, match="starts from an image"):
        _init(tmp_path, init_image=None, init_noise="none")


def test_init_is_the_bilinear_quarter(fake, tmp_path):
    _init(tmp_path)
    t = torch.rand(1, 3, 38, 50, generator=torch.Generator().manual_seed(3)) * 2 - 1
    d = api._state.drawer
    assert torch.equal(d.get_z_from_tensor(t), RR.latent_from_tensor(t))
    d.reapply_from_tensor(t)
    assert torch.equal(d.get_z(), RR.latent_from_tensor(t))
    d.z += 2.0
    d.clip_z()
    assert float(d.get_z().max()) == 1.0


def test_synthetic_weights_need_the_opt_in(fake, tmp_path):
    with pytest.raises(ValueError, match="b200_allow_synthetic"):
        _init(tmp_path, b200_allow_synthetic=False, b200_text_encoder=lambda m, t: torch.zeros(1, 512))
    api.reset_settings()
    _init(tmp_path)
    sd = api._state.engine.modules[E.MOD_VQGAN]
    assert sd["conv_first.weight"].shape == (64, 3, 3, 3) and "body.22.rdb3.conv5.bias" in sd


@pytest.mark.parametrize("wrap", ["params_ema", "params", None])
def test_checkpoint_wrappers_are_unwrapped(fake, tmp_path, wrap):
    sd = {"conv_first.weight": torch.ones(2)}
    obj = {wrap: sd, "other": {"x": torch.zeros(1)}} if wrap else sd
    if wrap == "params":
        obj = {"params": sd}
    path = tmp_path / "net.pth"
    torch.save(obj, path)
    assert api._load_state_dict(str(path)).keys() == sd.keys()
    assert api._load_state_dict(obj).keys() == sd.keys()
    if wrap == "params_ema":
        both = {"params": {"wrong": torch.zeros(1)}, "params_ema": sd}
        assert api._load_state_dict(both).keys() == sd.keys()


def test_given_weights_reach_the_engine(fake, tmp_path):
    sd = {"conv_first.weight": torch.ones(2)}
    _init(tmp_path, b200_weights={"super_resolution": {"params_ema": sd}})
    assert api._state.engine.modules[E.MOD_VQGAN].keys() == sd.keys()
    assert isinstance(api._state.drawer, P.SuperResolutionDrawer)
