"""The ViT-L/14@336px image tower on the engine (577 tokens: its attention runs on the streaming kernels, attn_long.cu).

(a) Full depth at the real shape, layer by layer against float64, and the patch gradient by norm: the checks and budgets
    of tests/test_vit_tower_gpu.py (imported), on 336-pixel cutouts.
(b) Two layers at full width, T and heads: forward and backward per element, as (a)'s module does for the other towers.
(c) One whole iteration (synth -> make_cutouts -> encode -> Prompt loss -> backward) against oracle/ref_path.iterate on a
    two-layer tower with four cutouts, with smoke()'s tolerances.
(d) The built engine runs the streaming kernels for this tower and no row softmax; PXR_FUSED_ATTN=0 gives the chain."""
import csv
import os

import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import cutouts
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_pipeline_gpu import random_transforms
from test_vit_tower_gpu import (COS_BOUND, REL_L2_BOUND, Report, Tower, _env, _round_up, _state_dict,
                                check_backward_elementwise, check_forward, rel_l2_cos, vjp)

pytestmark = pytest.mark.gpu

NAME = "ViT-L/14@336px"
ARCH = E.CLIP_ARCH[NAME]
CS = ARCH["image_res"]


def run_engine(arch, settings, monkeypatch, seed, cutn):
    """tests/test_vit_tower_gpu.run_engine at 336-pixel cutouts: the tower's taps after make_cutouts -> encode_image ->
    backward, in float64 on the CPU."""
    _env(monkeypatch, settings)
    sd = _state_dict(arch, seed, False)
    tw = Tower(arch, sd)
    W, H, L, T, D = tw.W, tw.H, tw.L, tw.T, tw.D
    M = cutn * T
    fused = settings.get("PXR_FUSED_ATTN", "1") != "0"
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=cutn, cut_size=CS, clip=[arch],
                       seed=seed)
    try:
        eng.load_module(E.MOD_CLIP0, sd)
        eng.finalize()
        pm = S.prompts(D, (1.0, -0.3), seed)
        eng.set_prompts(0, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
        g = torch.Generator().manual_seed(seed)
        img = eng.synth(torch.rand(eng.z_shape, generator=g))
        facs, noise = torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, CS, CS, generator=g)
        eng.make_cutouts(img, transforms=random_transforms(cutn, CS, seed), zoom_padding=E.PAD_REFLECTION, fill=0.4,
                         noise_facs=facs.numpy(), noise=noise)
        eng.encode_image(0)
        eng.backward()

        def rd(name, shape, dtype=torch.half):
            return eng.debug_read(f"clip0.{name}", shape, dtype).double().cpu()

        tp = dict(patches=rd("patches", (cutn, tw.np, tw.Kp)), t=rd("t", (M, W), torch.float32),
                  hcls=rd("hcls", (cutn, W)), e=rd("e", (cutn, D), torch.float32), de16=rd("de16", (cutn, D)),
                  gx16=rd("gx16", (M, W)), g_patches=rd("g_patches", (cutn, tw.np, tw.Kp)))
        for l in range(L + 1):
            tp[f"x{l}"] = rd(f"x{l}", (M, W))
        for l in range(L):
            tp[f"x_mid{l}"] = rd(f"x_mid{l}", (M, W))
            tp[f"qkv{l}"] = rd(f"qkv{l}", (M, 3 * W))
            tp[f"u{l}"] = rd(f"u{l}", (M, 4 * W))
            if fused:
                tp[f"o{l}"] = rd(f"o{l}", (M, W))
            else:
                tp[f"P{l}"] = rd(f"P{l}", (cutn, H, T, _round_up(T, 8)))
    finally:
        eng.close()
    return tw, tp, dict(B=cutn, cls_only=True, stream32=False, fused=fused)


def test_full_depth_tower_step_by_step_and_gradient_norm(monkeypatch):
    tw, tp, kw = run_engine(ARCH, {}, monkeypatch, seed=11, cutn=2)
    assert tw.T == 577
    rep = Report(f"{NAME} full depth")
    check_forward(rep, tw, tp, **kw)
    _, _, gp, _ = vjp(tw, tp, tp["de16"], cls_only=True, stream32=False, fused=True, var=False)
    rel, cos = rel_l2_cos(tp["g_patches"], gp)
    rep.lines.append(f"  g_patches vs float64 VJP: rel-L2 {rel:.3e} (bound {REL_L2_BOUND:.0e}), cosine {cos:.8f}")
    rep.finish()
    assert rel <= REL_L2_BOUND and cos >= COS_BOUND


def test_two_layer_tower_forward_and_backward_per_element(monkeypatch):
    tw, tp, kw = run_engine(dict(ARCH, layers=2), {}, monkeypatch, seed=13, cutn=3)
    rep = Report(f"{NAME} two layers")
    check_forward(rep, tw, tp, **kw)
    check_backward_elementwise(rep, tw, tp, **kw)
    rep.finish()


def test_whole_iteration_matches_the_oracle(monkeypatch):
    """smoke()'s pipeline (VQGAN drawer -> cutouts -> tower -> Prompt -> z.grad) at 336-pixel cutouts, two layers."""
    monkeypatch.delenv("PXR_FUSED_ATTN", raising=False)
    vq_cfg = dict(z_channels=128, n_embed=1024, ch=128, ch_mult=(1, 2), num_res_blocks=1, attn_resolution=16,
                  resolution=32)
    arch = dict(ARCH, layers=2)
    cutn = 4
    vq_sd, clip_sd = S.vqgan_state_dict(vq_cfg, 0), S.clip_state_dict(arch, 1)
    prompts = S.prompts(arch["out_dim"], (1.0, 0.1), 2)
    z = S.z0_vqgan(vq_sd["quantize.embedding.weight"], (16, 16), 3)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=vq_cfg, cutn=cutn, cut_size=CS, clip=[arch],
                       seed=0)
    try:
        eng.load_module(E.MOD_VQGAN, vq_sd)
        eng.load_module(E.MOD_CLIP0, clip_sd)
        eng.finalize()
        eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
        T = cutouts.sample_transforms(cutn, CS, 4)
        g = torch.Generator().manual_seed(5)
        facs = torch.rand(cutn, generator=g) * 0.1
        noise = torch.randn(cutn, 3, CS, CS, generator=g)
        facs[0] = facs[1] = 0.1  # unmistakable extremes, as smoke() plants them
        noise[0, 0, 5, 7], noise[1, 2, 100, 50] = 30.0, -30.0
        img = eng.synth(z)
        eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.5, noise_facs=facs.numpy(), noise=noise)
        emb = eng.encode_image(0).cpu()
        zg = eng.backward().cpu()
    finally:
        eng.close()
    vq = R.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1, attn_resolutions=(16,),
                   resolution=32, z_channels=128)
    vq.load_state_dict(vq_sd)
    clip = R.ClipVisual(CS, arch["patch"], arch["width"], arch["layers"], arch["heads"], arch["out_dim"])
    clip.load_state_dict(clip_sd)
    ref = R.iterate(lambda zz: R.vqgan_synth(vq.eval().requires_grad_(False), zz), z, [clip.eval().requires_grad_(False)],
                    [prompts], torch.from_numpy(T), CS, "reflection", 0.5, facs, noise)
    e_emb = (emb - ref["embeds"][0]).abs().max().item()
    e_g = (zg - ref["z_grad"]).abs().max().item()
    m_g = ref["z_grad"].abs().max().item()
    print(f"[vit-l336] embeds max_abs_err {e_emb:.3e}; z.grad max_abs_err {e_g:.3e} (max |grad| {m_g:.3e})")
    assert torch.isfinite(zg).all() and e_emb < 5e-3 and e_g <= 3e-2 * m_g


def _op_names(settings, monkeypatch, tmp_path):
    _env(monkeypatch, settings)
    arch = dict(ARCH, layers=2)
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=2, cut_size=CS, clip=[arch], seed=0)
    try:
        eng.load_module(E.MOD_CLIP0, S.clip_state_dict(arch, 1))
        eng.finalize()
        pm = S.prompts(arch["out_dim"], (1.0,), 2)
        eng.set_prompts(0, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
        z = torch.rand(eng.z_shape, generator=torch.Generator().manual_seed(1)).cuda()
        path = str(tmp_path / "ops.csv")
        monkeypatch.setenv("PXR_PROFILE_DUMP", path)
        eng.profile_iteration(z, 0.1, 0)
        monkeypatch.delenv("PXR_PROFILE_DUMP")
        return [r["op"] for r in csv.DictReader(open(path))]
    finally:
        eng.close()


def test_the_tower_runs_the_streaming_kernels_and_no_row_softmax(monkeypatch, tmp_path):
    ops = _op_names({}, monkeypatch, tmp_path)
    assert sum(op.startswith("attn_long_fwd B=2 T=577 heads=16") for op in ops) == 2
    assert sum(op.startswith("attn_long_bwd B=2 T=577 heads=16") for op in ops) == 2
    assert not any(op.startswith("softmax_forward") or op.startswith("softmax_backward") for op in ops)
    chain = _op_names({"PXR_FUSED_ATTN": "0"}, monkeypatch, tmp_path)
    assert sum(op.startswith("softmax_forward") for op in chain) == 2
    assert not any(op.startswith("attn_long") for op in chain)
    assert os.path.exists(tmp_path / "ops.csv")
