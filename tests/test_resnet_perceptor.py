"""CPU side of the CLIP ResNet perceptors: the float64 oracle (oracle/resnet_ref.py) against independent torch code, the
BatchNorm fold, the shape derivation from a state_dict for all five towers, and do_init with an engine that reports the
ResNet tower kind (the plain FakeEngine reports none, so tests/test_api.py keeps RN50 refused)."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from fake_engine import FakeEngine
from oracle.resnet_ref import ResnetRef, fold_conv
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

TINY = dict(width=16, layers=4, heads=8, patch=0, image_res=64, out_dim=32, tower=E.TOWER_CLIP_RESNET, blocks=(1, 1, 1, 1))


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + ".running_mean"].double(), sd[p + ".running_var"].double(), sd[p + ".weight"].double(),
                        sd[p + ".bias"].double(), training=False, eps=1e-5)


def test_block_matches_conv2d_and_batch_norm():
    sd = S.clip_resnet_state_dict(TINY, 0)
    ref = ResnetRef(sd)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 64, 8, 8, generator=g, dtype=torch.float64)  # the input of layer2.0: 4 w channels, a ReLU output
    v = {k: t.double() for k, t in sd.items() if t.is_floating_point()}
    p = "visual.layer2.0."
    h = torch.relu(_bn(F.conv2d(x, v[p + "conv1.weight"]), v, p + "bn1"))
    h = torch.relu(_bn(F.conv2d(h, v[p + "conv2.weight"], padding=1), v, p + "bn2"))
    h = _bn(F.conv2d(F.avg_pool2d(h, 2), v[p + "conv3.weight"]), v, p + "bn3")
    idn = _bn(F.conv2d(F.avg_pool2d(x, 2), v[p + "downsample.0.weight"]), v, p + "downsample.1")
    want = torch.relu(h + idn)
    assert torch.allclose(ref.block(x, 1, 0), want, rtol=1e-12, atol=1e-12)


def test_attnpool_matches_multi_head_attention_row0():
    sd = S.clip_resnet_state_dict(TINY, 2)
    ref = ResnetRef(sd)
    g = torch.Generator().manual_seed(3)
    x = torch.rand(3, 32 * 16, 2, 2, generator=g, dtype=torch.float64)
    t = ref.tokens(x)                                   # [B, T, C]
    a = "visual.attnpool."
    v = {k: sd[a + k].double() for k in ("q_proj.weight", "k_proj.weight", "v_proj.weight", "q_proj.bias", "k_proj.bias",
                                         "v_proj.bias", "c_proj.weight", "c_proj.bias")}
    tt = t.transpose(0, 1)                              # [T, B, C]
    full, _ = F.multi_head_attention_forward(
        tt, tt, tt, t.shape[-1], ref.heads, in_proj_weight=None,
        in_proj_bias=torch.cat([v["q_proj.bias"], v["k_proj.bias"], v["v_proj.bias"]]), bias_k=None, bias_v=None,
        add_zero_attn=False, dropout_p=0.0, out_proj_weight=v["c_proj.weight"], out_proj_bias=v["c_proj.bias"],
        use_separate_proj_weight=True, q_proj_weight=v["q_proj.weight"], k_proj_weight=v["k_proj.weight"],
        v_proj_weight=v["v_proj.weight"], need_weights=False)
    assert torch.allclose(ref.attnpool(t), full[0], rtol=1e-12, atol=1e-12)


def test_fold_equals_unfolded_batch_norm():
    sd = S.clip_resnet_state_dict(TINY, 4)
    x = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(5), dtype=torch.float64) - 0.5
    a, b = ResnetRef(sd).encode_image(x), ResnetRef(sd, folded=True).encode_image(x)
    assert ((a - b).norm() / a.norm()).item() < 5e-3  # the fold's fp16 weight rounding only
    # the fold itself is exact in float64 before the rounding
    w, bias = fold_conv(sd, "visual.layer1.0.conv2", "visual.layer1.0.bn2")
    y = torch.rand(1, 16, 5, 5, dtype=torch.float64)
    v = {k: t.double() for k, t in sd.items() if t.is_floating_point()}
    want = _bn(F.conv2d(y, v["visual.layer1.0.conv2.weight"], padding=1), v, "visual.layer1.0.bn2")
    got = F.conv2d(y, w, bias, padding=1)
    assert ((got - want).norm() / want.norm()).item() < 2e-3


@pytest.mark.parametrize("name", sorted(E.RESNET_ARCH))
def test_shapes_and_keys_derive_from_the_state_dict(name):
    arch = E.RESNET_ARCH[name]
    sd = S.clip_resnet_state_dict(arch, 0)
    assert E.resnet_arch_of(sd) == arch
    E.check_resnet_state_dict(name, sd)
    assert arch["heads"] * 64 == 32 * arch["width"] and arch["layers"] == sum(arch["blocks"])
    assert sd["visual.layer1.0.bn1.num_batches_tracked"].dtype == torch.int64
    side = arch["image_res"] // 32
    assert sd["visual.attnpool.positional_embedding"].shape == (side * side + 1, 32 * arch["width"])
    assert S.resnet_fwd_flops(arch) > 0


def test_block_count_mismatch_is_refused():
    sd = S.clip_resnet_state_dict(E.RESNET_ARCH["RN50"], 0)
    sd = {k: v for k, v in sd.items() if not k.startswith("visual.layer3.5.")}
    with pytest.raises(E.EngineError, match="blocks per stage"):
        E.check_resnet_state_dict("RN50", sd)


def test_activations_stay_bounded_at_full_depth():
    """The synthetic weights keep RN50x64's 36-block stage inside fp16's comfortable range."""
    arch = E.RESNET_ARCH["RN50x64"]
    ref = ResnetRef(S.clip_resnet_state_dict(arch, 0))
    x = torch.rand(1, 3, 448, 448, generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 4 - 2
    _, outs = ref.features(x)
    peak = max(o.abs().max().item() for o in outs)
    assert 1e-2 < peak < 1e3


class ResnetFakeEngine(FakeEngine):
    TOWERS = E.B200Engine.TOWERS


@pytest.fixture
def rfake(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", ResnetFakeEngine)
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    rows = {"RN50": [[0.3] * 1024], "RN101": [[0.4] * 512], "RN50x4": [[0.5] * 640], "RN50x16": [[0.6] * 768],
            "ViT-B/16": [[0.1] * 512], "ViT-B/32": [[0.2] * 512]}
    (tmp_path / "vectors" / "textoff.json").write_text(json.dumps(rows))
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(size=[64, 64], num_cuts=8, outdir="", seed="7", b200_allow_synthetic=True)
    base.update(kw)
    api.add_settings(**base)
    return api.do_init(api.apply_settings())


@pytest.mark.parametrize("model", ["RN50", "RN50x4"])
def test_do_init_builds_a_resnet_perceptor(rfake, tmp_path, model):
    _init(tmp_path, prompts="a cat", clip_models=model)
    eng = api._state.engine
    arch = E.RESNET_ARCH[model]
    assert eng.kw["clip"] == [arch] and eng.cut_size == arch["image_res"]
    assert eng.modules[E.MOD_CLIP0]["visual.attnpool.c_proj.weight"].shape == (arch["out_dim"], 32 * arch["width"])
    assert api._state.perceptors[0].family == "clip"


def test_quality_better_runs_three_perceptors(rfake, tmp_path):
    _init(tmp_path, prompts="a cat", quality="better", vector_prompts="textoff")
    eng = api._state.engine
    names = ["RN50", "ViT-B/32", "ViT-B/16"]
    assert [c["out_dim"] for c in eng.kw["clip"]] == [1024, 512, 512]
    assert set(eng.modules) == {E.MOD_VQGAN, E.MOD_CLIP0, E.MOD_CLIP1, E.MOD_CLIP2}
    want_row = {"RN50": 0.3, "ViT-B/32": 0.2, "ViT-B/16": 0.1}
    for i, m in enumerate(names):
        table = api._state.prompt_tables[i]
        assert len(table) == 2  # the text prompt, then the vector prompt
        assert torch.allclose(table[1].embed, torch.full_like(table[1].embed, want_row[m]))


def test_four_perceptors_are_refused(rfake, tmp_path):
    with pytest.raises(NotImplementedError, match="at most three"):
        _init(tmp_path, prompts="a cat", clip_models="RN50,RN101,ViT-B/32,ViT-B/16")


def test_plain_fake_engine_still_refuses_resnet(monkeypatch, tmp_path):
    monkeypatch.setattr(api, "_engine_factory", FakeEngine)
    api.reset_settings()
    with pytest.raises(NotImplementedError, match="no ResNet image towers"):
        _init(tmp_path, prompts="a cat", clip_models="RN50")
    api.reset_settings()


def test_full_depth_backward_bound_catches_a_dropped_branch():
    """The full-depth backward bounds of tests/test_resnet_tower_gpu.py (against the VJP at the engine's forward values:
    rel-L2 1e-2 / cosine 0.9999, and 5e-2 / 0.999 for RN50x64) against planted bugs: RN50 with the main or the identity
    branch's gradient dropped in any one block moves the float64 VJP by at least 0.17 rel-L2 (cosine at most 0.99)."""
    arch = E.RESNET_ARCH["RN50"]
    ref = ResnetRef(S.clip_resnet_state_dict(arch, 21), folded=True)
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(1, 3, 224, 224, generator=g, dtype=torch.float64) - 0.45) / 0.27
    de = torch.randn(1, arch["out_dim"], generator=g, dtype=torch.float64)
    clean = ref.vjp_at(None, x, de).flatten()
    rel_bound, cos_bound = 5e-2, 0.999  # the loosest of the bounds
    for s, n in enumerate(arch["blocks"]):
        for i in range(n):
            for branch in ("main", "identity"):
                bug = ref.vjp_at(None, x, de, drop=(s, i, branch)).flatten()
                rel = ((bug - clean).norm() / clean.norm()).item()
                cos = (bug @ clean / (bug.norm() * clean.norm())).item()
                assert rel > 3 * rel_bound and cos < cos_bound, (s, i, branch, rel, cos)
