"""The text towers on the engine (engine_text.inc) against float64: the causal attention on both of its paths, full-depth
towers at the real widths, causality and chunking through the public call, a pixray run that encodes its prompts on
the engine, and the memory of a session without text keys.

The float64 reference is oracle/text_ref.py with the tensors the engine uploads as fp16 (token embedding, the four
GEMM weights of every block, text_projection) rounded to fp16 first, as openai-CLIP's fp16 model holds them.

Full-depth bounds: per-embedding rel-L2 <= REL_L2_BOUND and cosine >= COS_BOUND.  Measured on an H100 80GB HBM3 (SXM)
at its 700 W power limit: rel-L2 1.05e-3 .. 1.59e-3 (MEASURED_REL_L2) and cosine >= 0.9999987 over both widths, both
attention paths, every batch and the pixray run, so the rel-L2 bound keeps a 2.5x margin."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import text_ref
from pixray_b200 import _lib
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from pixray_b200 import tokenizer as TK

pytestmark = pytest.mark.gpu

VOCAB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpe_vocab_used_merges.txt.gz")
U = 2.0 ** -11
REL_L2_BOUND = 4e-3   # 2.5x MEASURED_REL_L2
COS_BOUND = 1 - 1e-5
MEASURED_REL_L2 = 1.6e-3
# device memory a pixel-drawer session with one 128-wide image tower and no text keys takes at pxr_finalize, as the
# parent commit measured it on an H100 80GB HBM3 (cudaMemGetInfo before / after: 10 MiB in every session after the first);
# a session without text keys builds no tower and allocates nothing more
FINALIZE_BYTES_PARENT = 10485760
F16_KEYS = ("token_embedding.weight", "attn.in_proj_weight", "attn.out_proj.weight", "mlp.c_fc.weight",
            "mlp.c_proj.weight", "text_projection")


def _causal_hook(qkv, B, T, H):
    W = 64 * H
    o = torch.zeros(B * T, W, device="cuda", dtype=torch.float16)
    err = (C.c_char * 256)()
    rc = _lib.load().pxr_test_attention_causal(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), B, T, H, W,
                                               C.c_float(0.125), err, 256)
    assert rc == 0, err.value
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("T,B,H", [(1, 3, 8), (16, 12, 8), (77, 8, 12), (77, 1, 8), (128, 4, 16), (240, 8, 12)])
def test_causal_attention_hook_against_float64(monkeypatch, fused, T, B, H):
    """Element budget C u (sum_j P_ij |v_j| (1 + |S_ij| + sum_k P_ik |S_ik|) + |o_i|) + 2^-24: fp16 P / scores (the chain
    stores S in fp16) carried through the softmax and the PV product, and the fp16 output.  Then rows <= t0 are
    bit-identical when every token after t0 changes."""
    monkeypatch.setenv("PXR_FUSED_ATTN", "1" if fused else "0")
    g = torch.Generator().manual_seed(T * 1000 + B * 10 + H)
    qkv = torch.randn(B * T, 3 * 64 * H, generator=g).half()
    o = _causal_hook(qkv.cuda(), B, T, H).cpu().double()
    ref = text_ref.causal_attention(qkv, B, T, H)
    x = qkv.double().reshape(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    S_ = (x[0] @ x[1].transpose(-1, -2)) / 8.0
    mask = torch.full((T, T), float("-inf"), dtype=torch.float64).triu(1)
    P = torch.softmax(S_ + mask, dim=-1)
    aS = S_.abs().masked_fill(mask.isinf(), 0)
    spread = 1 + aS + (P * aS).sum(-1, keepdim=True)
    pv = ((P * spread) @ x[2].abs()).transpose(1, 2).reshape(B * T, 64 * H)
    budget = 4 * U * (pv + ref.abs()) + 2.0 ** -24
    ratio = ((o - ref).abs() / budget).max().item()
    print(f"causal attn fused={fused} T={T} B={B} H={H}: max err / budget {ratio:.3f}")
    assert ratio <= 1.0
    if T > 1:
        t0 = T // 2
        q2 = qkv.clone().reshape(B, T, -1)
        q2[:, t0 + 1:] = torch.randn(B, T - t0 - 1, q2.shape[-1], generator=g).half()
        o2 = _causal_hook(q2.reshape(B * T, -1).cuda(), B, T, H).cpu().reshape(B, T, -1)
        assert torch.equal(o2[:, :t0 + 1], o.half().reshape(B, T, -1)[:, :t0 + 1])


def _sd(width, out_dim, seed):
    vis = S.clip_state_dict(dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=out_dim), seed)
    return {**vis, **S.clip_text_state_dict(width, 12, out_dim, seed + 1)}


def _engine(sd, out_dim):
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(8, 8), cutn=2,
                       clip=[dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=out_dim)])
    eng.load_module(E.MOD_CLIP0, sd)
    eng.finalize()
    return eng


def _f16(sd):
    return {k: (v.half().double() if k.endswith(F16_KEYS) else v.double()) for k, v in sd.items()
            if not k.startswith("visual.")}


def _sequences(n, seed):
    """n id rows of 77: SOT, random ids below SOT, EOT, zeros; the last one 77 ids with no EOT (SLIP's truncation)."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 77), dtype=np.int32)
    for b in range(n):
        L = int(rng.integers(0, 76))
        out[b, :L + 2] = [TK.SOT] + list(rng.integers(1, TK.SOT, L)) + [TK.EOT]
    out[-1] = [TK.SOT] + list(rng.integers(1, TK.SOT, 76))
    return out


def _compare(got, want, what):
    got, want = got.double().cpu(), want.double()
    rel = ((got - want).norm(dim=-1) / want.norm(dim=-1))
    cos = torch.nn.functional.cosine_similarity(got, want, dim=-1)
    print(f"{what}: rel-L2 max {rel.max().item():.3e} mean {rel.mean().item():.3e}, cosine min {cos.min().item():.8f}")
    assert rel.max().item() <= REL_L2_BOUND and cos.min().item() >= COS_BOUND
    return rel.max().item()


@pytest.fixture(scope="module", params=[(512, 512), (768, 768)], ids=["512x12", "768x12"])
def tower(request):
    width, D = request.param
    sd = _sd(width, D, width)
    ids = _sequences(80, width)
    want = text_ref.encode_text(_f16(sd), ids)
    return sd, D, ids, want


@pytest.mark.parametrize("fused", [True, False])
def test_full_depth_tower_against_float64(monkeypatch, tower, fused):
    sd, D, ids, want = tower
    monkeypatch.setenv("PXR_FUSED_ATTN", "1" if fused else "0")
    eng = _engine(sd, D)
    assert eng.text_tower(0) == dict(width=sd["token_embedding.weight"].shape[1], layers=12, ctx=77, out_dim=D)
    w = sd["token_embedding.weight"].shape[1]
    for n in (1, 3, 80):
        _compare(eng.encode_text(0, ids[:n]), want[:n], f"W={w} fused={fused} n={n}")
    # chunking: 80 sequences in one call are the rows of the calls on each 32-sequence chunk, and of single calls
    all80 = eng.encode_text(0, ids)
    parts = torch.cat([eng.encode_text(0, ids[c:c + 32]) for c in range(0, 80, 32)])
    assert torch.equal(all80, parts)
    for b in (0, 33, 79):
        assert torch.equal(all80[b:b + 1], eng.encode_text(0, ids[b:b + 1]))
    # causality through the public call: after the EOT, zeros or random ids below EOT give the same embedding bits
    rng = np.random.default_rng(5)
    a = np.zeros((4, 77), dtype=np.int32)
    for b, L in enumerate((0, 7, 40, 74)):
        a[b, :L + 2] = [TK.SOT] + list(rng.integers(1, TK.SOT, L)) + [TK.EOT]
    z = a.copy()
    for b, L in enumerate((0, 7, 40, 74)):
        z[b, L + 2:] = rng.integers(0, TK.EOT, 77 - L - 2)
    assert torch.equal(eng.encode_text(0, a), eng.encode_text(0, z))
    eng.close()


def test_malformed_input_is_refused():
    sd = _sd(512, 512, 3)
    eng = _engine(sd, 512)
    ok = np.zeros((1, 77), dtype=np.int32)
    for bad, msg in ((np.full((1, 77), 49408, dtype=np.int32), "outside the vocabulary"),
                     (np.zeros((1, 76), dtype=np.int32), "context")):
        with pytest.raises(E.EngineError, match=msg):
            eng.encode_text(0, bad)
    assert eng.encode_text(0, ok).shape == (1, 512)
    assert eng.encode_text(0, np.zeros((0, 77), dtype=np.int32)).shape == (0, 512)
    eng.close()
    # a perceptor without text keys has no tower; a text_projection of another width is refused at finalize
    vis = {k: v for k, v in sd.items() if k.startswith("visual.")}
    eng = _engine(vis, 512)
    assert eng.text_tower(0) is None
    with pytest.raises(E.EngineError, match="no text tower"):
        eng.encode_text(0, ok)
    eng.close()
    with pytest.raises(E.EngineError, match="out_dim"):
        _engine({**vis, **S.clip_text_state_dict(512, 1, 256, 4)}, 512)


def test_pixray_run_encodes_prompts_on_the_engine(tmp_path):
    """pixray.run with full synthetic state_dicts (visual + text) for a CLIP and a SLIP perceptor, no text encoder, no
    synthetic embeddings: the registered prompt embeddings are the oracle's."""
    from pixray_b200 import api
    clip_arch, slip_arch = E.CLIP_ARCH["ViT-B/32"], E.SLIP_ARCH["SLIP_VITB16"]
    sd_c = {**S.clip_state_dict(clip_arch, 11), **S.clip_text_state_dict(512, 12, 512, 12)}
    sd_s = {**S.slip_state_dict(slip_arch, 13), **S.clip_text_state_dict(512, 12, 512, 14)}
    prompts = ["a cat:2", "an apple in the style of Cézanne", "rock 'n' roll, isn't it?"]
    api.run("|".join(prompts), "pixel", clip_models="ViT-B/32,SLIP_VITB16", size=[64, 64], num_cuts=4, iterations=3,
            outdir="", seed="1", b200_allow_synthetic=False, b200_bpe_vocab=VOCAB, vector_prompts="none",
            b200_weights={"ViT-B/32": sd_c, "SLIP_VITB16": sd_s})
    tok = TK.get(VOCAB)
    texts = ["a cat", prompts[1], prompts[2]]
    for i, (sd, fam) in enumerate(((sd_c, "clip"), (sd_s, "slip"))):
        got = torch.cat([p.embed for p in api._state.prompt_tables[i]])
        want = text_ref.encode_text(_f16(sd), tok(texts, fam))
        _compare(got, want, f"pixray.run perceptor {i} ({fam})")
    assert api._state.cur_iteration == 3
    api._state.engine.close()
    api.reset_settings()


def _finalize_bytes():
    sd = S.clip_state_dict(dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=64), 1)
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(8, 8), cutn=2,
                       clip=[dict(width=128, layers=1, heads=2, patch=32, image_res=224, out_dim=64)])
    eng.load_module(E.MOD_CLIP0, sd)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    eng.finalize()
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    eng.close()
    return used


def test_session_without_text_keys_allocates_what_the_parent_did():
    _finalize_bytes()  # first session: module loading and context growth
    used = min(_finalize_bytes() for _ in range(2))  # the smaller of two: other processes share the device
    print(f"finalize without text keys: {used} bytes (parent {FINALIZE_BYTES_PARENT})")
    assert used <= FINALIZE_BYTES_PARENT
