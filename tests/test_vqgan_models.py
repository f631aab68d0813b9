"""The VQGAN drawer's checkpoints on the CPU: engine.vqgan_config reads the architecture of every form pixray's vqgan_model
table ships (taming VQModel with its loss.* tensors, GumbelVQ, a Net2NetTransformer's first_stage_model) from the tensor
shapes; the oracle's GumbelQuantize restatement picks what F.gumbel_softmax picks; do_init hands the engine the derived
config (against a recording stand-in); a run without a checkpoint issues the engine calls it always did."""
import json
import os

import pytest
import torch
from torch.nn import functional as F

from fake_engine import FakeEngine
from oracle import gumbel_ref as G
from oracle import ref_path as R
from pixray_b200 import api
from pixray_b200 import engine as E

GOLDEN_DEFAULT = os.path.join(os.path.dirname(__file__), "golden", "vqgan_default_calls.json")

# small stand-ins of the table's f16 models: the shapes vqgan_config reads, at a width the CPU builds in a second
F16 = dict(z_channels=256, ch=128, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2, attn_resolution=16, resolution=256)
NARROW = dict(z_channels=64, ch=64, ch_mult=(1, 2), num_res_blocks=1, attn_resolution=128, resolution=256)
CASES = [("vqmodel", 1024, NARROW), ("gumbel", 8192, NARROW), ("net2net", 16384, NARROW), ("vqmodel", 8192, F16)]


def _oracle(cfg, gumbel):
    kw = dict(n_embed=cfg["n_embed"], embed_dim=cfg["z_channels"], with_encoder=True, ch=cfg["ch"], ch_mult=cfg["ch_mult"],
              num_res_blocks=cfg["num_res_blocks"], attn_resolutions=(cfg["attn_resolution"],),
              resolution=cfg["resolution"], z_channels=cfg["z_channels"])
    return G.GumbelVQModel(**kw) if gumbel else R.VQModel(**kw)


def _checkpoint(form, cfg):
    """A checkpoint of `form` around the oracle model built with `cfg`, as torch.load returns it."""
    sd = _oracle(cfg, form == "gumbel").state_dict()
    if form == "net2net":
        out = {"first_stage_model." + k: v for k, v in sd.items()}
        out["cond_stage_model.encoder.conv_in.weight"] = torch.zeros(8, 3, 3, 3)
        out["transformer.tok_emb.weight"] = torch.zeros(cfg["n_embed"], 16)
        out["transformer.blocks.0.attn.key.weight"] = torch.zeros(16, 16)
        return {"state_dict": out}
    sd["loss.discriminator.main.0.weight"] = torch.zeros(64, 3, 4, 4)  # VQLPIPSWithDiscriminator
    sd["loss.perceptual_loss.net.slice1.0.weight"] = torch.zeros(64, 3, 3, 3)
    return {"state_dict": sd}


@pytest.mark.parametrize("form,n_embed,arch", CASES)
def test_config_from_the_shapes_of_every_checkpoint_form(form, n_embed, arch):
    cfg = dict(arch, n_embed=n_embed)
    sd = api._vqgan_state_dict(_checkpoint(form, cfg))
    assert not [k for k in sd if k.startswith(("loss.", "first_stage_model.", "cond_stage_model.", "transformer."))]
    assert E.vqgan_config(sd) == dict(cfg, gumbel=form == "gumbel")


def _refusal(sd, edit, match):
    sd = dict(sd)
    edit(sd)
    with pytest.raises(E.EngineError, match=match):
        E.vqgan_config(sd)


def test_inconsistent_or_unsupported_shapes_are_refused_naming_the_tensor():
    cfg = dict(NARROW, n_embed=1024)
    sd = api._vqgan_state_dict(_checkpoint("vqmodel", cfg))
    E.vqgan_config(sd)

    def put(name, *shape):
        return lambda d: d.__setitem__(name, torch.zeros(*shape))

    def drop(name):
        return lambda d: d.pop(name)

    _refusal(sd, drop("quantize.embedding.weight"), "neither")
    _refusal(sd, put("quantize.embed.weight", 1024, 64), "both")
    _refusal(sd, drop("post_quant_conv.weight"), "'post_quant_conv.weight' is missing")
    _refusal(sd, put("post_quant_conv.weight", 64, 32, 1, 1), r"'post_quant_conv.weight' has shape \[64, 32, 1, 1\]")
    # embed_dim != z_channels: both numbers in the message
    _refusal(sd, lambda d: (d.__setitem__("quantize.embedding.weight", torch.zeros(1024, 128)),
                            d.__setitem__("post_quant_conv.weight", torch.zeros(64, 128, 1, 1))),
             "'quantize.embedding.weight' has embed_dim 128 but post_quant_conv.weight has z_channels 64")
    _refusal(sd, put("decoder.conv_in.weight", 128, 32, 3, 3), "'decoder.conv_in.weight' has shape")
    _refusal(sd, put("decoder.up.1.block.0.conv1.weight", 96, 64, 3, 3), "'decoder.up.1.block.0.conv1.weight' has 96")
    _refusal(sd, put("decoder.up.0.block.2.conv1.weight", 64, 64, 3, 3), "blocks per level")
    _refusal(sd, put("decoder.up.0.attn.0.q.weight", 64, 64, 1, 1), "attn.* keys at levels")
    _refusal(sd, put("encoder.conv_in.weight", 32, 3, 3, 3), "'encoder.conv_in.weight' has 32 output channels")
    # the tensor-core nearest-code search's limits
    _refusal(sd, lambda d: d.__setitem__("quantize.embedding.weight", torch.zeros(32768, 64)),
             "'quantize.embedding.weight' has 32768 codes")
    _refusal(sd, lambda d: d.__setitem__("quantize.embedding.weight", torch.zeros(1020, 64)), "has 1020 codes")
    narrow = api._vqgan_state_dict(_checkpoint("vqmodel", dict(NARROW, z_channels=32, n_embed=64)))
    with pytest.raises(E.EngineError, match="'post_quant_conv.weight' gives z_channels 32"):
        E.vqgan_config(narrow)
    gsd = api._vqgan_state_dict(_checkpoint("gumbel", dict(NARROW, n_embed=1024)))
    _refusal(gsd, drop("quantize.proj.weight"), "'quantize.proj.weight' is missing")
    _refusal(gsd, put("quantize.proj.weight", 512, 64, 1, 1), r"'quantize.proj.weight' has shape \[512, 64, 1, 1\]")


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_gumbel_quantize_equals_torch_gumbel_softmax(seed):
    """The restatement with noise -Exp(1).log() drawn after manual_seed(s) picks the code F.gumbel_softmax(hard=True)
    picks after the same seed, and its straight-through value is that code's row within one rounding."""
    n_embed, zc, hw = 512, 64, (4, 6)
    g = torch.Generator().manual_seed(100 + seed)
    h = torch.randn(1, zc, *hw, generator=g)
    w, b = torch.randn(n_embed, zc, 1, 1, generator=g) * zc ** -0.5, 0.05 * torch.randn(n_embed, generator=g)
    embed = torch.randn(n_embed, zc, generator=g)
    logits = F.conv2d(h, w, b)
    torch.manual_seed(seed)
    want = F.gumbel_softmax(logits, tau=1.0, dim=1, hard=True)
    torch.manual_seed(seed)
    noise = -torch.empty_like(logits).exponential_().log()
    z_q, idx, got_logits = G.gumbel_quantize(h, w, b, embed, noise)
    assert torch.equal(got_logits, logits)
    assert torch.equal(idx, want.argmax(dim=1).reshape(-1))
    assert torch.allclose(z_q, embed[idx].T.reshape(1, zc, *hw), rtol=0, atol=1e-5)
    assert torch.allclose(z_q, torch.einsum("bnhw,nd->bdhw", want, embed), rtol=0, atol=1e-5)


# ------------------------------------------------------------------------------------------------ do_init
class RecordingEngine(FakeEngine):
    """FakeEngine that keeps its constructor's vqgan argument and encodes GumbelVQs the way B200Engine does."""

    def __init__(self, *, vqgan=None, **kw):
        super().__init__(vqgan=vqgan, **kw)
        self.vqgan = vqgan
        v = E.VQGAN_F16_16384 if vqgan is None else vqgan
        self.gumbel = bool(v.get("gumbel", False))
        self.cfg.n_embed = v["n_embed"]

    def vqgan_encode_gumbel(self, img, noise):
        self._log("vqgan_encode_gumbel", shape=tuple(img.shape), noise=tuple(noise.shape), noise_sum=float(noise.sum()))
        return torch.zeros(self.z_shape)


@pytest.fixture
def rec(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", RecordingEngine)
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    base = dict(prompts="x", clip_models="ViT-B/16", size=[72, 40], num_cuts=8, outdir="", seed="7",
                b200_allow_synthetic=True, vector_prompts="none")
    base.update(kw)
    api.add_settings(**base)
    args = api.apply_settings()
    api.do_init(args)
    return args


@pytest.mark.parametrize("form,n_embed,arch", CASES[:3])
def test_do_init_builds_the_engine_from_the_checkpoint(rec, tmp_path, form, n_embed, arch):
    cfg = dict(arch, n_embed=n_embed)
    path = tmp_path / f"vqgan_{form}.ckpt"
    torch.save(_checkpoint(form, cfg), path)
    _init(tmp_path, b200_weights={"vqgan": str(path)}, vqgan_model="openimages_f16_8192", init_noise="none")
    eng = api._state.engine
    assert eng.vqgan == dict(cfg, gumbel=form == "gumbel")
    f = 2 ** (len(arch["ch_mult"]) - 1)
    assert eng.image_hw == (40 // f * f, 72 // f * f)                              # _side with the checkpoint's levels
    loaded = eng.modules[E.MOD_VQGAN]
    assert not [k for k in loaded if k.startswith(("loss.", "first_stage_model.", "cond_stage_model.", "transformer."))]
    # the random start (vqgan.py:162-171) draws rows of the checkpoint's own codebook
    code = loaded["quantize.embed.weight" if form == "gumbel" else "quantize.embedding.weight"]
    z = api._state.drawer.get_z()
    assert tuple(z.shape) == eng.z_shape
    rows = z[0].reshape(arch["z_channels"], -1).T
    assert all(bool((code == r).all(dim=1).any()) for r in rows)


def test_a_gumbel_checkpoint_encodes_with_fresh_gumbel_noise(rec, tmp_path):
    cfg = dict(NARROW, n_embed=1024)
    _init(tmp_path, b200_weights={"vqgan": _checkpoint("gumbel", cfg)}, size=[64, 64])
    eng = api._state.engine
    enc = [c for c in eng.calls if c[0].startswith("vqgan_encode")]
    assert [c[0] for c in enc] == ["vqgan_encode_gumbel"]
    assert enc[0][1]["noise"] == (1024, 32, 32)
    noise_sum = enc[0][1]["noise_sum"]
    assert abs(noise_sum / (1024 * 32 * 32) - 0.5772) < 0.01                      # E[-log Exp(1)] = Euler's gamma
    api._state.drawer.reapply_from_tensor(torch.zeros(1, 3, 64, 64))
    assert eng.calls[-1][0] == "vqgan_encode_gumbel" and eng.calls[-1][1]["noise_sum"] != noise_sum


def _default_run_log(tmp_path, **kw):
    """The engine calls (with their arguments) of a default-weights session: do_init and three iterations, for the
    encoded noise start and the random-codebook start."""
    logs = []
    for start in ("pixels", "none"):
        api.reset_settings()
        args = _init(tmp_path, init_noise=start, iterations=3, **kw)
        api.do_run(args)
        eng = api._state.engine
        logs.append(dict(ctor=dict(eng.kw, vqgan=eng.vqgan, image_hw=list(eng.image_hw)),
                         calls=[[n, {k: (list(v) if isinstance(v, tuple) else v) for k, v in a.items()}] for n, a in eng.calls],
                         z0_sum=float(api._state.drawer.get_z().double().sum()) if start == "none" else None))
    return json.loads(json.dumps(logs))


@pytest.mark.parametrize("label", [None, "imagenet_f16_1024", "openimages_f16_8192", "coco"])
def test_the_default_run_is_unchanged(rec, tmp_path, label):
    """No b200_weights['vqgan']: the seeded imagenet_f16_16384 stand-in, built with vqgan=None as before, whatever
    vqgan_model says.  tests/golden/vqgan_default_calls.json is this log as the engine calls were issued before the
    drawer read its architecture from the checkpoint."""
    got = _default_run_log(tmp_path, **({} if label is None else dict(vqgan_model=label)))
    with open(GOLDEN_DEFAULT) as f:
        want = json.load(f)
    assert got == want


@pytest.mark.parametrize("dest", ["vqgan_config", "vqgan_checkpoint"])
def test_vqgan_config_and_checkpoint_are_known_and_refused_when_set(rec, tmp_path, dest):
    api.add_settings(prompts="x")
    assert getattr(api.apply_settings(), dest) is None
    api.reset_settings()
    with pytest.raises(ValueError, match=rf"{dest}=.*b200_weights\['vqgan'\]"):
        _init(tmp_path, **{dest: "models/vqgan_coco.yaml"})
