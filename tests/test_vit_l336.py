"""ViT-L/14@336px as a perceptor, on the CPU: do_init against the recording stand-in for the engine (tests/fake_engine.py)
-- the name is accepted, the 336-pixel cutouts and the tower's architecture reach the engine, a 224-pixel tower beside
it is refused, a vector prompt without an entry for it warns and continues -- and the synthetic state_dict's shapes."""
import json
import os

import numpy as np
import pytest

from fake_engine import FakeEngine
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

NAME = "ViT-L/14@336px"
ARCH = E.CLIP_ARCH[NAME]


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", FakeEngine)
    FakeEngine.loss_script = staticmethod(lambda it, n: np.full(n, 1.0 / (1 + it), dtype=np.float32))
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    """do_init with a textoff.json that has vectors for the 224-pixel ViT-B towers only (as the default one), and an
    empty stand-in state_dict for every perceptor (the fake engine only records it)."""
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps({"ViT-B/16": [[0.1] * 512], "ViT-B/32": [[0.2] * 512]}))
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    models = kw.get("clip_models", NAME).split(",")
    base = dict(size=[64, 64], num_cuts=8, outdir="", seed="7", b200_allow_synthetic=True,
                b200_weights={m: {} for m in models})
    base.update(kw)
    api.add_settings(**base)
    return api.do_init(api.apply_settings())


def test_arch_is_vit_l14_at_336_pixels():
    assert ARCH == dict(width=1024, layers=24, heads=16, patch=14, image_res=336, out_dim=768)
    assert {k: v for k, v in ARCH.items() if k != "image_res"} == \
        {k: v for k, v in E.CLIP_ARCH["ViT-L/14"].items() if k != "image_res"}
    assert (ARCH["image_res"] // ARCH["patch"]) ** 2 + 1 == 577


def test_the_name_is_accepted_and_cut_size_336_reaches_the_engine(fake, tmp_path, capsys):
    _init(tmp_path, prompts="a cat", clip_models=NAME)
    eng = api._state.engine
    assert eng.cut_size == 336
    assert eng.kw["clip"] == [ARCH]
    assert api._state.make_cutouts.cut_size == 336
    assert E.MOD_CLIP0 in eng.modules
    # 768-wide text embedding for the tower's Prompt (seeded, b200_allow_synthetic)
    emb, w, _ = eng.prompts[0]
    assert np.asarray(emb).shape[-1] == 768
    # the default vector prompt (textoff) has no entry for this tower: warned, the session continues
    assert f"WARNING: no vector for {NAME} in textoff!" in capsys.readouterr().out
    assert len(w) == 1


def test_the_224_pixel_towers_keep_cut_size_224(fake, tmp_path):
    _init(tmp_path, prompts="a cat", clip_models="ViT-B/32,ViT-L/14")
    assert api._state.engine.cut_size == 224 and api._state.make_cutouts.cut_size == 224


@pytest.mark.parametrize("models", [f"{NAME},ViT-B/16", f"ViT-B/32,{NAME}", f"{NAME},SLIP_VITB16"])
def test_mixing_with_a_224_pixel_tower_is_refused(fake, tmp_path, models):
    with pytest.raises(NotImplementedError, match="different resolutions"):
        _init(tmp_path, prompts="a cat", clip_models=models)


def test_two_336_pixel_towers_are_one_resolution(fake, tmp_path):
    _init(tmp_path, prompts="a cat", clip_models=f"{NAME},{NAME}")
    assert api._state.engine.cut_size == 336 and len(api._state.engine.kw["clip"]) == 2


def test_synthetic_state_dict_shapes():
    """openai-CLIP's visual.* keys at the tower's shapes (one layer: the other 23 repeat its keys)."""
    sd = S.clip_state_dict(dict(ARCH, layers=1), 1)
    W, P, D, T = 1024, 14, 768, 577
    want = {"visual.conv1.weight": (W, 3, P, P), "visual.class_embedding": (W,), "visual.positional_embedding": (T, W),
            "visual.proj": (W, D), "visual.ln_pre.weight": (W,), "visual.ln_post.bias": (W,),
            "visual.transformer.resblocks.0.attn.in_proj_weight": (3 * W, W),
            "visual.transformer.resblocks.0.attn.in_proj_bias": (3 * W,),
            "visual.transformer.resblocks.0.attn.out_proj.weight": (W, W),
            "visual.transformer.resblocks.0.mlp.c_fc.weight": (4 * W, W),
            "visual.transformer.resblocks.0.mlp.c_proj.weight": (W, 4 * W)}
    for k, shape in want.items():
        assert tuple(sd[k].shape) == shape, k
    assert len(sd) == 8 + 12
