"""The VQGAN drawer at the real f16 architecture (ch 128, ch_mult (1, 1, 2, 2, 4), 2 res blocks, z_channels 256, 256 x 256
canvas) with 1024, 8192 and 8192-Gumbel codebooks, seeded synthetic weights, against the float64 oracle: synth and its
gradient, the GumbelVQ encoder, and whole runs through do_init / do_run from each checkpoint form.

Tolerances of synth and z.grad are test_big_shapes_gpu.py::test_config3_shape_vqgan512_two_perceptors_cutn128's for the
16384-code decoder: image max-abs-err < 5e-3, z.grad max-abs-err <= 3e-2 * max|z.grad|."""
import numpy as np
import pytest
import torch

from oracle import gumbel_ref as G
from oracle import ref_path as R
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_pipeline_gpu import SMALL_CLIP, plant_extremes, random_transforms, report

pytestmark = pytest.mark.gpu

F16 = dict(z_channels=256, ch=128, ch_mult=(1, 1, 2, 2, 4), num_res_blocks=2, attn_resolution=16, resolution=256)
GRAD_SCALE = 4096.0  # the engine's default loss scale: g_img is stored scaled by it
MODELS = [(1024, False), (8192, False), (8192, True)]


def _models(n_embed, gumbel, seed, with_encoder=False):
    cfg = dict(F16, n_embed=n_embed)
    sd = S.vqgan_state_dict(cfg, seed, with_encoder=with_encoder, gumbel=gumbel)
    assert E.vqgan_config(sd) == dict(cfg, gumbel=gumbel)
    kw = dict(n_embed=n_embed, embed_dim=256, with_encoder=with_encoder, ch=128, ch_mult=F16["ch_mult"], num_res_blocks=2,
              attn_resolutions=(16,), resolution=256, z_channels=256)
    vq = (G.GumbelVQModel if gumbel else R.VQModel)(**kw)
    vq.load_state_dict(sd)
    vq.eval().requires_grad_(False)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(256, 256), vqgan=E.vqgan_config(sd), cutn=8, clip=[SMALL_CLIP],
                       seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, seed + 1))
    eng.finalize()
    return sd, vq, eng


def _codebook(vq):
    return vq.codebook if isinstance(vq, G.GumbelVQModel) else vq.quantize.embedding.weight


@pytest.mark.parametrize("n_embed,gumbel", MODELS)
def test_synth_and_gradient_match_the_float64_oracle(n_embed, gumbel):
    seed = 11
    sd, vq, eng = _models(n_embed, gumbel, seed)
    # the tensor-core nearest-code search is on: its counters exist only on that path
    eng.debug_read("vq_stats", (2,), dtype=torch.int32)
    vq64 = vq.double()
    cb = _codebook(vq64)
    g = torch.Generator().manual_seed(seed + 2)
    idx = torch.randint(n_embed, (256,), generator=g)
    z = (cb[idx].T.reshape(1, 256, 16, 16).float() + 0.05 * torch.randn(1, 256, 16, 16, generator=g)).contiguous()
    prompts = [(torch.randn(1, 64, generator=g), w, float("-inf")) for w in (1.0, -0.3)]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])

    img = eng.synth(z)
    idx_eng = eng.debug_read("vq_idx", (256,), dtype=torch.int32).cpu().long()
    assert torch.equal(idx_eng, R.vector_quantize(z.double().movedim(1, 3), cb)[1].reshape(-1))
    T = random_transforms(8, 224, seed)
    facs, noise = plant_extremes(torch.rand(8, generator=g) * 0.1, torch.randn(8, 3, 224, 224, generator=g))
    eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    eng.prompt_loss(0)
    eng.backward()
    g_img = eng.debug_read("g_img", (1, 3, 256, 256)).cpu().double() / GRAD_SCALE
    zg = eng.debug_read("z_grad", z.shape).cpu()
    # the oracle's synth on the side of clamp_with_grad's [0, 1] each pixel is on in the engine (test_pipeline_gpu.py,
    # vqgan_synth_with_engine_clamp_sides), fed the engine's own d loss / d image
    pre = eng.debug_read("img_pre", (1, 3, 256, 256)).cpu().double()
    side = (pre > 1).double() - (pre < 0).double()
    zr = z.double().requires_grad_(True)
    zq, _ = R.vector_quantize(zr.movedim(1, 3), cb)
    x = vq64.decode(zq.movedim(3, 1)).add(1).div(2)
    ref = x.clamp(0, 1)
    e_img, _ = report(f"{n_embed}{'-gumbel' if gumbel else ''} image 256x256", img, ref.detach())
    assert e_img < 5e-3
    kept = g_img * ((g_img * side) >= 0)
    x.backward(kept)
    e_g, m_g = report(f"{n_embed}{'-gumbel' if gumbel else ''} z.grad", zg, zr.grad)
    assert torch.isfinite(zg).all() and m_g > 0 and e_g <= 3e-2 * m_g


def test_gumbel_encode_picks_the_oracles_codes():
    """pxr_vqgan_encode_gumbel at 256 x 256 with 8192 codes.  The oracle takes the engine's own quant_conv output (exact in
    fp16, so the encoder's rounding stays out of the comparison; test_vqgan_encoder_gpu.py covers the encoder) and forms
    the logits in float64.  The engine's logits come from an fp16 GEMM: the projection weight rounded to fp16 (relative
    2^-11) and fp32 accumulation over 256 terms, so each logit is within b = (2^-11 + 256 * 2^-24) * sum_k |h_k W_jk| of
    the oracle's, and the pick can only differ where the oracle's top-two margin is below 2 b (bounded here by 4 b)."""
    seed = 21
    sd, vq, eng = _models(8192, True, seed, with_encoder=True)
    g = torch.Generator().manual_seed(seed + 5)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, 256), torch.linspace(-1, 1, 256), indexing="ij")
    img = (torch.stack([yy, xx, yy * xx])[None] * 0.6 + 0.3 * torch.randn(1, 3, 256, 256, generator=g)).clamp(-1, 1)
    torch.manual_seed(seed)
    noise = -torch.empty(1, 8192, 16, 16).exponential_().log()
    z = eng.vqgan_encode_gumbel(img, noise).cpu()
    h_eng = eng.debug_read("enc_h", (256, 256)).cpu()
    idx_eng = eng.debug_read("enc_idx", (256,), dtype=torch.int32).cpu().long()
    # the encoder itself: the same bound as test_vqgan_encoder_gpu.py
    _, _, h_ref, _ = vq.encode(img, noise)
    e_h = (h_eng - h_ref[0].reshape(256, 256)).abs().max().item() / h_ref.abs().max().item()
    assert e_h < 1e-2

    h64 = h_eng.double().reshape(1, 256, 16, 16)
    w64, b64 = vq.quantize.proj.weight.double(), vq.quantize.proj.bias.double()
    _, idx_ref, logits = G.gumbel_quantize(h64, w64, b64, vq.codebook.double(), noise.double())
    top2 = (logits + noise.double()).reshape(8192, 256).topk(2, dim=0).values
    margin = top2[0] - top2[1]
    mag = (h64.abs().reshape(256, 256).T @ w64.abs().reshape(8192, 256).T).max(dim=1).values  # max_j sum_k |h_k W_jk|
    bound = 4 * (2.0 ** -11 + 256 * 2.0 ** -24) * mag
    decided = margin > bound
    print(f"[gumbel encode] codes compared at {int(decided.sum())}/256 positions; {int((~decided).sum())} excluded as "
          f"near-ties (margin <= bound); smallest margin {margin.min().item():.3e}, largest bound {bound.max().item():.3e}")
    assert decided.float().mean().item() >= 0.9
    assert torch.equal(idx_eng[decided], idx_ref[decided])
    assert torch.equal(z[0].reshape(256, 256), vq.codebook[idx_eng].T)                   # exactly the code rows
    # fixed reduction order: the same noise gives the same latent
    assert torch.equal(z, eng.vqgan_encode_gumbel(img, noise).cpu())
    with pytest.raises(E.EngineError, match="pxr_vqgan_encode_gumbel"):
        eng.vqgan_encode(img)


def test_nearest_code_engine_refuses_gumbel_encode():
    from test_pipeline_gpu import SMALL_VQ
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=8, clip=[SMALL_CLIP], seed=0)
    eng.load_module(E.MOD_VQGAN, S.vqgan_state_dict(SMALL_VQ, 0, with_encoder=True))
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    with pytest.raises(E.EngineError, match="call pxr_vqgan_encode"):
        eng.vqgan_encode_gumbel(torch.zeros(1, 3, 32, 32), torch.zeros(1024, 16, 16))


def _checkpoint(form, n_embed, seed):
    sd = S.vqgan_state_dict(dict(F16, n_embed=n_embed), seed, with_encoder=True, gumbel=form == "gumbel")
    if form == "net2net":
        sd = {"first_stage_model." + k: v for k, v in sd.items()}
        sd["cond_stage_model.encoder.conv_in.weight"] = torch.zeros(8, 3, 3, 3)
        sd["transformer.tok_emb.weight"] = torch.zeros(n_embed, 16)
    else:
        sd["loss.discriminator.main.0.weight"] = torch.zeros(64, 3, 4, 4)
    return {"state_dict": sd}


@pytest.mark.parametrize("form,n_embed,init_image", [("vqmodel", 1024, False), ("gumbel", 8192, False),
                                                     ("gumbel", 8192, True), ("net2net", 16384, False)])
def test_three_steps_through_the_api_from_each_checkpoint_form(tmp_path, form, n_embed, init_image):
    from PIL import Image
    path = tmp_path / "vqgan.ckpt"
    torch.save(_checkpoint(form, n_embed, 3), path)
    extra = {}
    if init_image:
        rng = np.random.default_rng(0)
        Image.fromarray(rng.integers(0, 255, (256, 256, 3), dtype=np.uint8)).save(tmp_path / "init.png")
        extra["init_image"] = str(tmp_path / "init.png")
    api.reset_settings()
    api.add_settings(prompts="a red square", clip_models="ViT-B/16", size=[256, 256], num_cuts=8, iterations=3, outdir="",
                     seed="5", b200_allow_synthetic=True, vector_prompts="none", b200_device_checkdrop=False,
                     b200_weights={"vqgan": str(path)}, vqgan_model="openimages_f16_8192" if form == "gumbel" else "coco",
                     **extra)
    args = api.apply_settings()
    api.do_init(args)
    eng, drawer = api._state.engine, api._state.drawer
    assert eng.gumbel == (form == "gumbel") and eng.cfg.n_embed == n_embed
    z0 = drawer.get_z_copy()
    api.do_run(args)
    z = drawer.get_z()
    lo, hi = eng.z_bounds()
    assert api._state.losses is not None and np.isfinite(api._state.losses).all()
    assert torch.isfinite(z).all() and not torch.equal(z, z0)
    assert (z >= lo[None, :, None, None]).all() and (z <= hi[None, :, None, None]).all()
    api.reset_settings()


def test_the_default_run_is_bit_identical_with_the_derived_config():
    """The seeded imagenet_f16_16384 stand-in built the old way (vqgan=None) and with the config vqgan_config derives from
    the same weights: identical losses, bit for bit, over three fused iterations."""
    sd = S.vqgan_state_dict(E.VQGAN_F16_16384, 0, with_encoder=True)
    cfg = E.vqgan_config(sd)
    assert cfg == dict(E.VQGAN_F16_16384, gumbel=False)
    clip = E.CLIP_ARCH["ViT-B/16"]
    clip_sd = S.clip_state_dict(clip, 1)
    prompts = S.prompts(512, (1.0, 0.1), 2)
    z0 = S.z0_vqgan(sd["quantize.embedding.weight"], (16, 16), 3)
    runs = []
    for vqgan in (None, cfg):
        eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(256, 256), vqgan=vqgan, cutn=64, clip=[clip], seed=0)
        eng.load_module(E.MOD_VQGAN, sd)
        eng.load_module(E.MOD_CLIP0, clip_sd)
        eng.finalize()
        eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
        z = z0.clone().cuda().contiguous()
        out = []
        for it in range(3):
            losses = np.zeros(2, dtype=np.float32)
            eng.iterate(z, 0.1, it, losses_out=losses)
            out.append(losses)
        runs.append((np.stack(out), z.cpu()))
        eng.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
