"""CPU: the text towers' host side.  The tokenizer against the ids the reference's own tokenizer gives
(tests/golden/text_tokens.json, oracle/make_golden_text.py), the float64 oracle of encode_text against an independent
implementation (transformers.CLIPTextModelWithProjection), and the api's routing of prompt texts to the engine's tower
(a recording stand-in with a tower)."""
import json
import os

import numpy as np
import pytest
import torch

from fake_engine import FakeEngine
from oracle import text_ref
from pixray_b200 import api
from pixray_b200 import plugins as P
from pixray_b200 import synthetic as S
from pixray_b200 import tokenizer as TK

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VOCAB = os.path.join(GOLDEN, "bpe_vocab_used_merges.txt.gz")
GOLD = json.load(open(os.path.join(GOLDEN, "text_tokens.json"), encoding="utf-8"))


@pytest.fixture(scope="module")
def tok():
    return TK.get(VOCAB)


def test_tokenizer_reproduces_the_reference_ids(tok):
    """SLIP's SimpleTokenizer.__call__ truncates to 77 ids; clip.tokenize raises on the same over-length inputs."""
    assert len(GOLD["strings"]) >= 40 and any(GOLD["overflows"])
    for s, ids, over in zip(GOLD["strings"], GOLD["ids"], GOLD["overflows"]):
        got = tok(s, "slip")
        assert got.shape == (1, 77) and got.dtype == np.int32
        assert got[0].tolist() == ids, s
        if over:
            with pytest.raises(RuntimeError, match="too long for context length 77"):
                tok(s, "clip")
        else:
            assert tok(s, "clip")[0].tolist() == ids, s
    batch = tok(GOLD["strings"][:3], "clip")
    assert batch.shape == (3, 77) and [r.tolist() for r in batch] == GOLD["ids"][:3]


def test_truncated_slip_sequence_loses_its_eot(tok):
    """The over-length string keeps 77 ids without the EOT: encode_text's argmax then reads the largest remaining id."""
    s = next(s for s, o in zip(GOLD["strings"], GOLD["overflows"]) if o)
    ids = tok(s, "slip")[0]
    assert ids[0] == TK.SOT and TK.EOT not in ids.tolist() and ids.min() > 0


def test_vocab_lookup_names_the_setting(monkeypatch, tmp_path):
    assert TK.find_vocab(VOCAB) == VOCAB
    with pytest.raises(FileNotFoundError, match="b200_bpe_vocab"):
        TK.find_vocab(str(tmp_path / "missing.txt.gz"))
    monkeypatch.setenv("PIXRAY_ROOT", str(tmp_path))
    monkeypatch.setitem(__import__("sys").modules, "clip", None)  # no installed clip package
    with pytest.raises(FileNotFoundError, match="b200_bpe_vocab"):
        TK.find_vocab()
    (tmp_path / "SLIP").mkdir()
    (tmp_path / "SLIP" / TK.VOCAB_NAME).write_bytes(open(VOCAB, "rb").read())
    assert TK.find_vocab() == str(tmp_path / "SLIP" / TK.VOCAB_NAME)


@pytest.mark.parametrize("width", [512, 768])
def test_oracle_matches_transformers_clip_text_model(width, tok):
    """oracle/text_ref.py against transformers' CLIPTextModelWithProjection with the same seeded weights, float64."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    D, L = 512 if width == 512 else 768, 2
    sd = S.clip_text_state_dict(width, L, D, seed=width)
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=width, intermediate_size=4 * width, num_hidden_layers=L,
                         num_attention_heads=width // 64, max_position_embeddings=77, hidden_act="quick_gelu",
                         layer_norm_eps=1e-5, projection_dim=D, eos_token_id=2, attn_implementation="sdpa")
    m = CLIPTextModelWithProjection(cfg).double().eval()  # sdpa: the eager path takes the softmax in float32
    hf = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
          "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
          "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
          "text_projection.weight": sd["text_projection"].T}
    for i in range(L):
        p, q = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
            hf[q + f"self_attn.{nm}.weight"] = sd[p + "attn.in_proj_weight"][j * width:(j + 1) * width]
            hf[q + f"self_attn.{nm}.bias"] = sd[p + "attn.in_proj_bias"][j * width:(j + 1) * width]
        for a, b in (("attn.out_proj", "self_attn.out_proj"), ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2"),
                     ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2")):
            hf[q + b + ".weight"], hf[q + b + ".bias"] = sd[p + a + ".weight"], sd[p + a + ".bias"]
    missing, unexpected = m.load_state_dict({k: v.double() for k, v in hf.items()}, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing)
    ids = torch.from_numpy(tok(["a cat", "an apple in the style of Cézanne", GOLD["strings"][-1]], "slip")).long()
    with torch.no_grad():
        want = m(input_ids=ids).text_embeds
    got = text_ref.encode_text(sd, ids)
    rel = ((got - want).norm(dim=-1) / want.norm(dim=-1)).max().item()
    assert rel <= 1e-10, rel


# ---------------------------------------------------------------------------------------------- api routing
class TowerEngine(FakeEngine):
    """FakeEngine whose perceptors have text towers: encode_text logs the ids and returns seeded rows per sequence."""

    def text_tower(self, clip_idx=0):
        return dict(width=512, layers=12, ctx=77, out_dim=self.clip_dims[clip_idx])

    def encode_text(self, clip_idx, tokens):
        t = np.asarray(tokens)
        self._log("encode_text", clip=clip_idx, tokens=t.copy())
        rows = [torch.randn(self.clip_dims[clip_idx], generator=torch.Generator().manual_seed(int(r.sum()) + 7 * clip_idx))
                for r in t]
        return torch.stack(rows)

    def vdiff_set_clip_embed(self, e):
        self.clip_embed = np.asarray(e).copy()
        super().vdiff_set_clip_embed(e)


@pytest.fixture
def tower(monkeypatch):
    monkeypatch.setattr(api, "_engine_factory", TowerEngine)
    api.reset_settings()
    yield
    api.reset_settings()


def _init(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(size=[64, 64], num_cuts=8, outdir="", seed="7", b200_allow_synthetic=False, vector_prompts="none",
                b200_bpe_vocab=VOCAB)
    base.update(kw)
    api.add_settings(**base)
    return api.do_init(api.apply_settings())


def _encoded(eng):
    return [(c[1]["clip"], c[1]["tokens"]) for c in eng.calls if c[0] == "encode_text"]


def test_prompts_and_spot_prompts_go_to_the_tower_in_the_reference_order(tower, tmp_path, tok):
    (tmp_path / "inputs").mkdir()
    (tmp_path / "inputs" / "spot_square.png").write_bytes(open(os.path.join(GOLDEN, "spot_square.png"), "rb").read())
    _init(tmp_path, prompts="a cat:2|a dog:-0.5:0.3", clip_models="ViT-B/16,SLIP_VITB16", spot_prompts="a red circle",
          spot_prompts_off="the sky|a dot")
    eng = api._state.engine
    fam = ["clip", "slip"]
    # pixray.py:859-870, 917-931: for each prompt, for each perceptor; prompts, then spot, then spot-off
    want = [(i, t) for t in ("a cat", "a dog", "a red circle", "the sky", "a dot") for i in (0, 1)]
    got = _encoded(eng)
    assert len(got) == len(want)
    for (ci, ids), (wi, txt) in zip(got, want):
        assert ci == wi and np.array_equal(ids, tok(txt, fam[wi]))
    for i in (0, 1):  # the registered rows are the tower's embeddings (normalised by the engine, not here)
        emb, w, stops = eng.prompts[i]
        assert w == pytest.approx([2.0, -0.5]) and stops[1] == pytest.approx(0.3)
        for j, txt in enumerate(("a cat", "a dog")):
            assert np.allclose(emb[j], eng.encode_text(i, tok(txt, fam[i]))[0].numpy())


def test_vdiff_clip_embed_comes_from_the_tower(tower, tmp_path, tok):
    _init(tmp_path, prompts="a cat:2|a dog", drawer="vdiff", clip_models="ViT-B/16", iterations=2,
          b200_weights={"vdiff": {"dummy": torch.zeros(1)}})
    eng = api._state.engine
    e = torch.cat([eng.encode_text(0, tok(t, "clip")) for t in ("a cat", "a dog")])
    want = torch.nn.functional.normalize((e * torch.tensor([2.0, 1.0])[:, None]).sum(0, keepdim=True), dim=-1)
    assert np.allclose(eng.clip_embed.reshape(-1), want.numpy().reshape(-1), atol=1e-6)


def test_text_encoder_still_wins(tower, tmp_path):
    seen = []

    def enc(model, txt):
        seen.append((model, txt))
        return torch.ones(1, 512)
    _init(tmp_path, prompts="a cat|=a dog", clip_models="ViT-B/16", b200_text_encoder=enc)
    assert seen == [("ViT-B/16", "a cat"), ("ViT-B/16", "=a dog")] and not _encoded(api._state.engine)


def test_equals_prompt_on_the_tower_raises(tower, tmp_path):
    with pytest.raises(ValueError, match="'='"):
        _init(tmp_path, prompts="=a cat", clip_models="ViT-B/16")


def test_no_encoder_no_tower_no_synthetic_raises(monkeypatch, tmp_path):
    monkeypatch.setattr(api, "_engine_factory", FakeEngine)
    api.reset_settings()
    try:
        with pytest.raises(ValueError, match="text tower"):
            _init(tmp_path, prompts="a cat", clip_models="ViT-B/16")
        api.reset_settings()
        _init(tmp_path, prompts="a cat", clip_models="ViT-B/16", b200_allow_synthetic=True)  # synthetic still allowed
        with pytest.raises(NotImplementedError, match="no text tower"):
            api._state.perceptors[0].encode_text("a cat")
    finally:
        api.reset_settings()


def test_perceptor_encode_text_tokenises_per_family(tower, tmp_path, tok):
    _init(tmp_path, prompts="x", clip_models="ViT-B/16,SLIP_VITB16", b200_allow_synthetic=True)
    eng = api._state.engine
    per = api._state.perceptors
    assert isinstance(per[1], P.Perceptor) and per[0].family == "clip" and per[1].family == "slip"
    long = GOLD["strings"][-1]
    with pytest.raises(RuntimeError, match="too long"):
        per[0].encode_text(long)
    out = per[1].encode_text(["a cat", long])
    assert tuple(out.shape) == (2, 512)
    assert np.array_equal(_encoded(eng)[-1][1], tok(["a cat", long], "slip"))
