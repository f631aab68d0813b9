"""model.encode (VqganDrawer.init_from_tensor / reapply_from_tensor / get_z_from_tensor, vqgan.py:174-185): taming Encoder +
quant_conv + nearest code on the engine (pxr_vqgan_encode) against the oracle's restatement.  The encoder output feeds an
arg-min over the codebook, so the comparison is: the pre-quantisation features to fp16 accuracy, the chosen codes equal
wherever the oracle's own decision is not a near-tie, and the returned latent EXACTLY the codebook rows of the chosen codes."""
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _check(cfg, image_hw, seed, clip_cfg):
    H, W = image_hw
    sd = S.vqgan_state_dict(cfg, seed, with_encoder=True)
    vq = R.VQModel(n_embed=cfg["n_embed"], embed_dim=cfg["z_channels"], with_encoder=True, ch=cfg["ch"], ch_mult=cfg["ch_mult"],
                   num_res_blocks=cfg["num_res_blocks"], attn_resolutions=(cfg["attn_resolution"],),
                   resolution=cfg["resolution"], z_channels=cfg["z_channels"])
    vq.load_state_dict(sd)
    vq.eval().requires_grad_(False)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(H, W), vqgan=cfg, cutn=8, clip=[clip_cfg], seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(clip_cfg, 1))
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 5)
    # a smooth image plus noise, in [-1, 1] like init_tensor * 2 - 1 (pixray.py:718-727)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    img = (torch.stack([yy, xx, yy * xx])[None] * 0.6 + 0.3 * torch.randn(1, 3, H, W, generator=g)).clamp(-1, 1)
    quant, idx, h = vq.encode(img)
    z = eng.vqgan_encode(img).cpu()
    C, hw = quant.shape[1], quant.shape[2] * quant.shape[3]
    h_eng = eng.debug_read("enc_h", (C, hw)).cpu()
    idx_eng = eng.debug_read("enc_idx", (hw,), dtype=torch.int32).cpu().long()
    h_ref = h[0].reshape(C, hw)
    e_h = (h_eng - h_ref).abs().max().item() / h_ref.abs().max().item()
    same = idx_eng == idx
    # where the codes differ the oracle's own decision must be a near-tie: the engine's code is (almost) as close
    cb = vq.quantize.embedding.weight
    flat = h_ref.t()
    d_ref = (flat - cb[idx]).pow(2).sum(1)
    d_eng = (flat - cb[idx_eng]).pow(2).sum(1)
    slack = ((d_eng - d_ref) / d_ref.clamp_min(1e-12))[~same]
    print(f"[parity] encoder features rel err {e_h:.2e}; codes equal {int(same.sum())}/{hw}; worst distance slack of the "
          f"differing ones {float(slack.max()) if slack.numel() else 0.0:.2e}")
    assert e_h < 1e-2
    assert same.float().mean().item() >= 0.9
    assert slack.numel() == 0 or slack.max().item() < 2e-2
    assert torch.equal(z[0].reshape(C, hw), cb[idx_eng].t())               # exactly the codebook rows
    assert torch.equal(z.cuda().cpu(), eng.vqgan_encode(img).cpu())         # deterministic
    return eng, vq, z


def test_encoder_small_matches_the_oracle():
    from test_pipeline_gpu import SMALL_CLIP, SMALL_VQ
    _check(SMALL_VQ, (32, 32), 3, SMALL_CLIP)
    _check(SMALL_VQ, (32, 48), 4, SMALL_CLIP)   # non-square latent


def test_encoder_attention_rows_longer_than_1024():
    """96 x 96: the encoder's mid and down-block attention run at the 48 x 48 latent, T = 2304 tokens per row."""
    from test_pipeline_gpu import SMALL_CLIP, SMALL_VQ
    _check(SMALL_VQ, (96, 96), 6, SMALL_CLIP)


def test_encoder_full_size_and_drawer_init():
    """imagenet_f16_16384 at 256 x 256, then VqganDrawer.init_from_tensor -> synth round trip through the plugin classes."""
    from test_pipeline_gpu import SMALL_CLIP
    from pixray_b200 import plugins as P
    eng, vq, z = _check(E.VQGAN_F16_16384, (256, 256), 0, SMALL_CLIP)
    session = P.Session(eng)
    drawer = P.VqganDrawer(None, session)
    drawer.load_model(None, eng.device)
    img = torch.rand(1, 3, 256, 256) * 2 - 1
    drawer.init_from_tensor(img)
    assert tuple(drawer.get_z().shape) == (1, 256, 16, 16)
    out = drawer.synth(0)
    assert torch.isfinite(out).all() and 0.0 <= float(out.min()) and float(out.max()) <= 1.0
    z_before = drawer.get_z_copy()
    drawer.reapply_from_tensor(torch.rand(1, 3, 256, 256) * 2 - 1)
    assert not torch.equal(z_before, drawer.get_z())
