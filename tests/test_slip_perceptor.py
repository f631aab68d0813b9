"""SLIP perceptors on the CPU: the timm ViT restatement (oracle/slip_ref.py) against transformers and against the golden of
the unmodified slip.py, the checkpoint loading, the synthetic weights, and do_init's handling of SLIP model names."""
import argparse
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fake_engine import FakeEngine  # noqa: E402
from oracle import ref_path as R  # noqa: E402
from oracle import slip_ref as SR  # noqa: E402
from pixray_b200 import api  # noqa: E402
from pixray_b200 import engine as E  # noqa: E402
from pixray_b200 import synthetic as S  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "slip_perceptor.npz")
SMALL = dict(width=64, layers=2, heads=2, patch=8, image_res=32, out_dim=16)


def close(a, b, tol):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    err = (a - b).abs().max().item()
    assert err <= tol, f"max abs err {err:.3e} > {tol:.1e}"


def test_timm_vit_restatement_matches_transformers_vit():
    """Un-vendored leaf: timm 0.5 VisionTransformer.  Cross-check against HF ViTModel (exact GELU, eps 1e-6, qkv bias)."""
    tr = pytest.importorskip("transformers")
    cfg = tr.ViTConfig(hidden_size=64, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, image_size=32,
                       patch_size=8, hidden_act="gelu", layer_norm_eps=1e-6, qkv_bias=True, attn_implementation="eager")
    hf = tr.ViTModel(cfg, add_pooling_layer=False).eval()
    mine = SR.make_model(SMALL, S.slip_state_dict(SMALL, 9))
    v = mine.visual
    sd = hf.state_dict()
    with torch.no_grad():
        sd["embeddings.cls_token"].copy_(v.cls_token)
        sd["embeddings.position_embeddings"].copy_(v.pos_embed)
        sd["embeddings.patch_embeddings.projection.weight"].copy_(v.patch_embed.proj.weight)
        sd["embeddings.patch_embeddings.projection.bias"].copy_(v.patch_embed.proj.bias)
        sd["layernorm.weight"].copy_(v.norm.weight)
        sd["layernorm.bias"].copy_(v.norm.bias)
        for i, blk in enumerate(v.blocks):
            p = f"encoder.layer.{i}."
            W, b = blk.attn.qkv.weight, blk.attn.qkv.bias
            for j, nm in enumerate(("query", "key", "value")):
                sd[p + f"attention.attention.{nm}.weight"].copy_(W[j * 64:(j + 1) * 64])
                sd[p + f"attention.attention.{nm}.bias"].copy_(b[j * 64:(j + 1) * 64])
            for dst, src in (("attention.output.dense", blk.attn.proj), ("intermediate.dense", blk.mlp.fc1),
                             ("output.dense", blk.mlp.fc2), ("layernorm_before", blk.norm1),
                             ("layernorm_after", blk.norm2)):
                sd[p + dst + ".weight"].copy_(src.weight)
                sd[p + dst + ".bias"].copy_(src.bias)
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        a = v(x)
        b = hf(pixel_values=x).last_hidden_state[:, 0]
    close(a, b, 1e-5)


def _golden_model(G):
    w, layers, heads, patch, res, out = (int(t) for t in G["arch"])
    arch = dict(width=w, layers=layers, heads=heads, patch=patch, image_res=res, out_dim=out)
    return SR.make_model(arch, S.slip_state_dict(arch, int(G["seed"])))


def test_golden_of_the_reference_slip_base_is_reproduced():
    """slip.py's SLIP_Base (preprocess, encode_image, `module.` stripping) run on the restatement: the oracle's
    slip_preprocess / encode_image give the same input, unit embeddings and input gradient."""
    G = np.load(GOLDEN)
    model = _golden_model(G)
    x = torch.from_numpy(G["imgs"]).requires_grad_(True)
    close(SR.slip_preprocess(x.detach()), G["preprocessed"], 1e-6)
    e = SR.encode_image(model, x)
    close(e.detach(), G["embeds"], 1e-6)
    (e * torch.from_numpy(G["direction"])).sum().backward()
    close(x.grad, G["grad"], 1e-6 * max(1.0, float(np.abs(G["grad"]).max())))


def test_clip_normalised_adaptor_equals_the_direct_slip_path():
    """ref_path.encode_image hands a model CLIP-normalised input; SlipPerceptor re-normalises it affinely to ImageNet."""
    model = SR.make_model(SMALL, S.slip_state_dict(SMALL, 4))
    g = torch.Generator().manual_seed(2)
    x = (torch.rand(3, 3, 32, 32, generator=g) * 1.4 - 0.2).requires_grad_(True)
    direct = SR.encode_image(model, x)
    (direct * torch.arange(16.0)).sum().backward()
    g_direct = x.grad.clone()
    x.grad = None
    via = R.encode_image(SR.SlipPerceptor(model), x)
    (via * torch.arange(16.0)).sum().backward()
    close(via.detach(), direct.detach(), 1e-6)
    close(x.grad, g_direct, 1e-6 * max(1.0, g_direct.abs().max().item()))


def test_synthetic_slip_weights_load_strictly_into_the_restatement():
    for arch in (SMALL, E.SLIP_ARCH["SLIP_VITB16"]):
        sd = S.slip_state_dict(arch, 1)
        m = SR.make_model(arch, sd)
        assert set(m.state_dict()) == set(sd)


def test_load_state_dict_strips_the_module_prefix_of_a_slip_checkpoint(tmp_path):
    sd = S.slip_state_dict(SMALL, 2)
    extra = {"transformer.resblocks.0.ln_1.weight": torch.ones(4), "logit_scale": torch.tensor(2.0)}
    ckpt = {"state_dict": {"module." + k: v for k, v in {**sd, **extra}.items()},
            "args": argparse.Namespace(model="SLIP_VITB16", ssl_mlp_dim=8, ssl_emb_dim=4)}
    path = tmp_path / "slip_base_100ep.pt"
    torch.save(ckpt, path)
    got = api._load_state_dict(str(path))
    assert set(got) == set(sd) | set(extra)
    for k, v in sd.items():
        assert torch.equal(got[k], v)


@pytest.fixture
def fake(monkeypatch, tmp_path):
    monkeypatch.setattr(api, "_engine_factory", FakeEngine)
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps({"ViT-B/16": [[0.1] * 512]}))
    monkeypatch.setenv("PIXRAY_ROOT", str(tmp_path))
    api.reset_settings()
    yield
    api.reset_settings()


def _init(clip_models):
    api.add_settings(prompts="a cat|a dog:0.5", clip_models=clip_models, drawer="vqgan", num_cuts=8, outdir="",
                     seed="7", b200_allow_synthetic=True)
    args = api.apply_settings()
    api.do_init(args)
    return api._state.engine


@pytest.mark.parametrize("models", ["SLIP_VITB16", "ViT-B/16,SLIP_VITB16"])
def test_do_init_hands_the_tower_kind_to_the_engine(fake, models):
    names = models.split(",")
    eng = _init(models)
    assert [c.get("tower", E.TOWER_OPENAI_CLIP) for c in eng.kw["clip"]] == \
        [E.SLIP_ARCH[m]["tower"] if m in E.SLIP_ARCH else E.TOWER_OPENAI_CLIP for m in names]
    assert E.SLIP_ARCH["SLIP_VITB16"]["tower"] == E.TOWER_TIMM_VIT
    for i, m in enumerate(names):
        sd = eng.modules[E.MOD_CLIP0 + i]
        if m in E.SLIP_ARCH:
            assert set(sd) == set(S.slip_state_dict(E.SLIP_ARCH[m]))
        else:
            assert "visual.conv1.weight" in sd
    # prompts of every perceptor in the reference's order: the text prompts, then (openai-CLIP only here) the vector
    synth = argparse.Namespace(b200_text_encoder=None, b200_allow_synthetic=True)
    for i, m in enumerate(names):
        emb, w, _ = eng.prompts[i]
        texts = [api._text_embed(synth, m, t, 512) for t in ("a cat", "a dog")]
        assert np.allclose(emb[:2], torch.cat(texts).numpy())
        assert w[:2] == [1.0, 0.5]
        assert len(w) == (3 if m == "ViT-B/16" else 2)


@pytest.mark.parametrize("model", ["SLIP_VITS16", "CLIP_VITS16", "SIMCLR_VITS16"])
def test_unsupported_slip_models_are_refused_with_the_reason(fake, model):
    with pytest.raises(NotImplementedError) as ex:
        _init(model)
    msg = str(ex.value)
    assert model in msg
    if model == "SIMCLR_VITS16":
        assert "image_projection" in msg and "text tower" in msg
    else:
        assert "32-wide heads" in msg
