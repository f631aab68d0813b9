"""SLIP perceptors on the GPU: the exact-GELU GEMM epilogue against float64, the timm ViT tower through the whole
iteration against the CPU oracle (oracle/slip_ref.py behind oracle/ref_path.iterate), the full SLIP_VITB16 /
SLIP_VITL16 shapes, and a session through pixray_b200.run.

Stated tolerances (fp16 tensor-core operands, fp32 accumulation, against SLIP's fp32 reference) are those of
tests/test_pipeline_gpu.py and tests/test_big_shapes_gpu.py."""
import hashlib

import numpy as np
import pytest
import torch

from gemm_util import run_gemm
from oracle import ref_path as R
from oracle import slip_ref as SR
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_big_shapes_gpu import check_subset
from test_pipeline_gpu import (SMALL_CLIP, SMALL_VQ, _assert_pipeline_tolerances, plant_extremes, random_transforms,
                               report, vqgan_synth_with_engine_clamp_sides)

pytestmark = pytest.mark.gpu

ACT_QUICKGELU, ACT_QUICKGELU_BWD, ACT_GELU, ACT_GELU_BWD = 1, 2, 6, 7
SMALL_SLIP = dict(SMALL_CLIP, tower=E.TOWER_TIMM_VIT)


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def _ulp16(v):
    return torch.from_numpy(np.spacing(np.abs(v.detach().cpu().numpy().astype(np.float16)))).double()


def _check_gelu(u16, out16, acc64, bias, name):
    """u16: the saved pre-activation, out16 = gelu(u16); u16 within the GEMM's bound of float64 A B^T + bias, out16 within
    one fp16 ulp of float64 gelu(u16)."""
    u64 = acc64 + (0 if bias is None else bias.double().cpu())
    e_u = (u16.double().cpu() - u64).abs().max().item()
    assert e_u <= 3e-3 * max(u64.abs().max().item(), 1.0), f"{name}: pre-activation err {e_u}"
    ref, _ = SR.gelu(u16.cpu())
    err = (out16.double().cpu() - ref).abs()
    assert (err <= _ulp16(ref)).all(), f"{name}: gelu out err {err.max().item():.3e} exceeds one fp16 ulp"


def _check_gelu_bwd(g16, prod32, u16, name):
    """g16 = fp16(prod * (Phi(u) + u phi(u))) with prod the same GEMM's fp32 product: the factor to 2^-11 rel + 2^-24."""
    _, f = SR.gelu(u16.cpu())
    y = prod32.double().cpu() * f
    err = (g16.double().cpu() - y).abs()
    bound = 2.0 ** -11 * y.abs() * (1 + 2.0 ** -20) + 2.0 ** -24
    assert (err <= bound).all(), f"{name}: backward factor err {(err - bound).max().item():.3e} over the bound"


@pytest.mark.parametrize("te", [0, -1])
@pytest.mark.parametrize("N,ld,bias", [(384, 400, True), (200, 208, False)])
def test_gelu_epilogue_against_float64(te, N, ld, bias):
    """fc1 forward (bias, GELU, pre-activation to aux_out) and fc2 dgrad (MN-major B, times gelu'(u)) on both epilogue
    paths (te=0: tensor-map epilogue where the shape allows it; -1: the generic one), with an M tail and a ragged N."""
    g = torch.Generator().manual_seed(61)
    M, K = 1000, 256
    A, B = _rand(g, M, K, scale=0.2), _rand(g, N, K, scale=0.2)
    b = (torch.randn(N, generator=g)).cuda() if bias else None
    acc64 = A.double().cpu() @ B.double().cpu().T
    aux = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    out = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, bias=b, act=ACT_GELU, aux_out=aux, out_f16=out, ldc=ld, tma_epi=te)
    _check_gelu(aux[:, :N], out[:, :N], acc64, b, f"gelu fwd te={te} N={N}")
    # backward: same product twice, once plain in fp32, once through the GELU-backward epilogue
    Bt = B.t().contiguous()
    prod = torch.zeros(M, ld, device="cuda")
    run_gemm(A, Bt, M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, out_f32=prod, ldc=ld, tma_epi=te)
    gout = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, Bt, M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, act=ACT_GELU_BWD, aux_in=aux, out_f16=gout, ldc=ld,
             tma_epi=te)
    _check_gelu_bwd(gout[:, :N], prod[:, :N], aux[:, :N], f"gelu bwd te={te} N={N}")
    with pytest.raises(RuntimeError, match="saved pre-activation"):
        run_gemm(A, Bt, M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, act=ACT_GELU_BWD, out_f16=gout, ldc=ld)


@pytest.mark.parametrize("te", [0, -1])
def test_gelu_epilogue_batched(te):
    """The batched form: 3 x 4 independent [197, 200] GEMMs (row pitch 208), rows of one batch never spill into the next."""
    g = torch.Generator().manual_seed(62)
    imgs, heads, T, d, N, ldp = 3, 4, 197, 64, 200, 208
    A = _rand(g, imgs * heads * T, d, scale=0.4)
    B = _rand(g, imgs * heads * N, d, scale=0.4)
    aux = torch.full((imgs, heads, T, ldp), 9.0, device="cuda", dtype=torch.half)
    out = torch.full((imgs, heads, T, ldp), 9.0, device="cuda", dtype=torch.half)
    kw = dict(lda=d, ldb=d, nb0=heads, nb1=imgs, a_bs=(T * d, heads * T * d), b_bs=(N * d, heads * N * d), b_batched=1,
              block_n=128, ldc=ldp, c_bs=(T * ldp, heads * T * ldp), tma_epi=te)
    run_gemm(A, B, T, N, d, act=ACT_GELU, aux_out=aux, out_f16=out, **kw)
    acc64 = torch.einsum("ihtd,ihnd->ihtn", A.double().cpu().view(imgs, heads, T, d), B.double().cpu().view(imgs, heads, N, d))
    _check_gelu(aux[..., :N], out[..., :N], acc64, None, f"batched gelu te={te}")
    prod = torch.zeros(imgs, heads, T, ldp, device="cuda")
    run_gemm(A, B, T, N, d, out_f32=prod, **kw)
    gout = torch.zeros(imgs, heads, T, ldp, device="cuda", dtype=torch.half)
    run_gemm(A, B, T, N, d, act=ACT_GELU_BWD, aux_in=aux, out_f16=gout, **kw)
    _check_gelu_bwd(gout[..., :N], prod[..., :N], aux[..., :N], f"batched gelu bwd te={te}")


# sha256 of the QuickGELU epilogue outputs (aux, out, dgrad) of _quickgelu_outputs per epilogue path, as the GEMM computed
# them before the exact-GELU codes existed: adding those codes left the QuickGELU results bit-identical
QUICKGELU_SHA256 = {
    0: "4eefe0add9d13e3e859e79dd1c59fec18ecf3bb6aa8b03303cf78c9f9fe497c8",
    -1: "5cd45e778ce09bf40e87f946d5a7d74e9db780fb0fd5fbfbff7a1003d4274f87",
}


def _quickgelu_outputs(te):
    g = torch.Generator().manual_seed(63)
    M, N, K, ld = 1000, 384, 256, 400
    A, B = _rand(g, M, K, scale=0.2), _rand(g, N, K, scale=0.2)
    b = torch.randn(N, generator=g).cuda()
    aux = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    out = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, bias=b, act=ACT_QUICKGELU, aux_out=aux, out_f16=out, ldc=ld,
             tma_epi=te)
    gout = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, B.t().contiguous(), M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, act=ACT_QUICKGELU_BWD, aux_in=aux,
             out_f16=gout, ldc=ld, tma_epi=te)
    h = hashlib.sha256()
    for t in (aux, out, gout):
        h.update(t.cpu().numpy().tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("te", [0, -1])
def test_quickgelu_epilogue_is_bit_identical(te):
    assert _quickgelu_outputs(te) == QUICKGELU_SHA256[te]


# ------------------------------------------------------------------------------------------------ the timm ViT tower
def build(seed, clips=(SMALL_SLIP,), cutn=8, image=32):
    """Engine + oracle models for a VQGAN session with the given perceptors (openai-CLIP or timm towers)."""
    torch.manual_seed(seed)
    vq_cfg = SMALL_VQ
    vq = R.init_vqgan_weights(R.VQModel(n_embed=vq_cfg["n_embed"], embed_dim=vq_cfg["z_channels"], ch=vq_cfg["ch"],
                                        ch_mult=vq_cfg["ch_mult"], num_res_blocks=vq_cfg["num_res_blocks"],
                                        attn_resolutions=(vq_cfg["attn_resolution"],), resolution=vq_cfg["resolution"],
                                        z_channels=vq_cfg["z_channels"]), seed)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(image, image), vqgan=vq_cfg, cutn=cutn, clip=list(clips),
                       noise_fac=0.1, seed=seed)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    models, prompt_sets = [], []
    g = torch.Generator().manual_seed(seed + 2)
    for i, c in enumerate(clips):
        if c.get("tower") == E.TOWER_TIMM_VIT:
            sd = S.slip_state_dict(c, seed + 1 + i)
            models.append(SR.SlipPerceptor(SR.make_model(c, sd)))
        else:
            sd = S.clip_state_dict(c, seed + 1 + i)
            m = R.ClipVisual(c["image_res"], c["patch"], c["width"], c["layers"], c["heads"], c["out_dim"])
            m.load_state_dict(sd)
            models.append(m.eval().requires_grad_(False))
        eng.load_module(E.MOD_CLIP0 + i, sd)
        pm = [(torch.randn(1, c["out_dim"], generator=g), w, float("-inf")) for w in (1.0, -0.3)]
        prompt_sets.append(pm)
    eng.finalize()
    for i, pm in enumerate(prompt_sets):
        eng.set_prompts(i, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
    hw = image // 2
    idx = torch.randint(vq_cfg["n_embed"], (hw * hw,), generator=g)
    z = vq.quantize.embedding.weight[idx].T.reshape(1, vq_cfg["z_channels"], hw, hw).contiguous()
    z = (z + 0.05 * torch.randn(z.shape, generator=g)).contiguous()
    return vq, models, eng, prompt_sets, z


def _stagewise(vq, models, eng, prompt_sets, z, seed, image_prompts=()):
    cutn, cs = 8, 224
    T = random_transforms(cutn, cs, seed)
    g = torch.Generator().manual_seed(seed + 9)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    if image_prompts:
        eng.set_image_prompts([t for t, _ in image_prompts], [w for _, w in image_prompts])
    img = eng.synth(z)
    synth, _ = vqgan_synth_with_engine_clamp_sides(vq, eng, (32, 32))
    ref = R.iterate(synth, z, list(models), list(prompt_sets), torch.from_numpy(T), cs, "reflection", 0.37, facs, noise,
                    image_prompts=list(image_prompts))
    eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.37, noise_facs=facs.numpy(), noise=noise)
    embs = [eng.encode_image(i).clone() for i in range(len(models))]
    losses = torch.cat([eng.prompt_loss(i).clone() for i in range(len(models))])
    zg = eng.backward().clone()
    assert torch.isfinite(zg).all()
    err = dict(image=report("image", img, ref["image"])[0],
               embeds=max(report(f"unit embeds {i}", e, ref["embeds"][i])[0] for i, e in enumerate(embs)),
               losses=report("prompt losses", losses, torch.stack([l.reshape(()) for l in ref["losses"]]))[0])
    err["z_grad"], err["z_grad_max"] = report("z.grad", zg, ref["z_grad"])
    return (embs, zg), err


PATHS = {"fused": {}, "batched_gemms_row_softmax": {"PXR_FUSED_ATTN": "0"}, "fp32_stream": {"PXR_CLIP_STREAM": "32"}}


def _env(monkeypatch, settings):
    for k in ("PXR_FUSED_ATTN", "PXR_CLIP_STREAM", "PXR_CLIP_LAST_CLS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in settings.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("path", sorted(PATHS))
def test_timm_tower_matches_the_oracle(path, monkeypatch):
    """A small timm tower (width 128, 2 layers, 2 heads, patch 32) on every attention / residual-stream path."""
    _env(monkeypatch, PATHS[path])
    vq, models, eng, prompt_sets, z = build(71)
    _, err = _stagewise(vq, models, eng, prompt_sets, z, 71)
    eng.close()
    _assert_pipeline_tolerances(err)


def test_timm_tower_with_image_prompts(monkeypatch):
    _env(monkeypatch, {})
    vq, models, eng, prompt_sets, z = build(73)
    g = torch.Generator().manual_seed(74)
    tp = [(torch.rand(1, 3, 32, 32, generator=g), 0.8), (torch.rand(1, 3, 40, 24, generator=g) * 0.5 + 0.25, -0.4)]
    _, err = _stagewise(vq, models, eng, prompt_sets, z, 73, image_prompts=tp)
    assert eng.num_losses() == 4
    eng.close()
    _assert_pipeline_tolerances(err)


def test_mixed_clip_and_slip_share_the_cutout_batch(monkeypatch):
    """An openai-CLIP and a timm perceptor encode the same cutouts; their gradients add into d loss / d batch."""
    _env(monkeypatch, {})
    vq, models, eng, prompt_sets, z = build(75, clips=(SMALL_CLIP, SMALL_SLIP))
    _, err = _stagewise(vq, models, eng, prompt_sets, z, 75)
    eng.close()
    _assert_pipeline_tolerances(err)


def test_timm_tower_last_layer_on_all_rows_is_bit_identical(monkeypatch):
    outs = {}
    for last_cls in ("1", "0"):
        _env(monkeypatch, {"PXR_CLIP_LAST_CLS": last_cls})
        vq, models, eng, prompt_sets, z = build(77)
        outs[last_cls], err = _stagewise(vq, models, eng, prompt_sets, z, 77)
        eng.close()
        _assert_pipeline_tolerances(err)
    (e1, g1), (e0, g0) = outs["1"], outs["0"]
    assert torch.equal(e1[0], e0[0])
    assert torch.equal(g1, g0)


def test_timm_tower_is_refused_after_finalize_and_for_unknown_kinds():
    vq, models, eng, prompt_sets, z = build(79)
    with pytest.raises(E.EngineError, match="after pxr_finalize"):
        eng._check(eng.lib.pxr_set_clip_tower(eng.h, 0, E.TOWER_TIMM_VIT), "pxr_set_clip_tower")
    eng.close()
    with pytest.raises(E.EngineError, match="unknown tower kind"):
        E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=8, clip=[dict(SMALL_CLIP, tower=5)])


@pytest.mark.slow
@pytest.mark.parametrize("name", ["SLIP_VITB16", "SLIP_VITL16"])
def test_full_slip_shapes(name, monkeypatch):
    """SLIP_VITB16 / SLIP_VITL16 at their full shapes, synthetic weights, cutn 8: embeddings and d loss / d cutout against
    the oracle (the subset check of test_big_shapes_gpu.py, here on every cutout)."""
    _env(monkeypatch, {})
    cutn, cs, seed = 8, 224, 81
    arch = E.SLIP_ARCH[name]
    sd = S.slip_state_dict(arch, seed)
    model = SR.SlipPerceptor(SR.make_model(arch, sd))
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=cutn, clip=[arch], seed=seed)
    vq = R.init_vqgan_weights(R.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1,
                                        attn_resolutions=(16,), resolution=32, z_channels=128), seed)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    eng.load_module(E.MOD_CLIP0, sd)
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 1)
    pm = [(torch.randn(1, 512, generator=g), 1.0, float("-inf")), (torch.randn(1, 512, generator=g), -0.2, float("-inf"))]
    eng.set_prompts(0, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
    img = torch.rand(1, 3, 32, 32, generator=g)
    T = random_transforms(cutn, cs, 7)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    batch_ref = R.make_cutouts(img, torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
    eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    check_subset(eng, [model], [pm], batch_ref, list(range(cutn)), cutn, cs)
    eng.close()


def test_run_mixed_clip_and_slip_end_to_end(tmp_path, monkeypatch):
    """pixray_b200.run with clip_models='ViT-B/16,SLIP_VITB16' (synthetic weights and prompts): it runs, and the loss falls."""
    _env(monkeypatch, {})
    from pixray_b200 import api
    api.reset_settings()
    api.add_settings(prompts="a cat", drawer="vqgan", clip_models="ViT-B/16,SLIP_VITB16", size=[64, 64], num_cuts=16,
                     iterations=40, b200_allow_synthetic=True, outdir="", seed="3", vector_prompts="none",
                     b200_device_checkdrop=False)
    args = api.apply_settings()
    api.do_init(args)
    assert api._state.engine.num_losses() == 2
    losses = []
    for it in range(30):
        api.train(args, it)
        losses.append(float(np.sum(api._state.losses)))
    api.reset_settings()
    print("[slip run] loss sums", losses[0], losses[-1])
    assert np.isfinite(losses).all()
    assert np.mean(losses[-5:]) < np.mean(losses[:5])
