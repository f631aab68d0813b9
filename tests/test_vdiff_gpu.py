"""GPU parity of the vdiff drawer (row a6: VdiffDrawer.synth over the cc12m_1 U-Net, vdiff.py:159-172) against
oracle/ref_path.py's VDiffCC12M1, which tests/test_oracle_golden.py pins bit-exactly to the reference's own
v-diffusion-pytorch model (same seeded initialisation, same outputs and gradients).

The 603 M-parameter model is built from torch.manual_seed(0) on the CPU and its state_dict handed to the engine under the
checkpoint's keys.  Tolerances (fp16 tensor-core operands / fp32 accumulation vs fp32 CPU): v and pred 2e-2 of max|v|
(measured 1.7e-3), image 1e-2 abs, d loss / d image 3e-2.

z.grad: the U-Net's 111 ReLUs make its backward DISCONTINUOUS in the forward activations: a pre-activation within the
fp16 forward error (~1e-3 of the activation scale) of zero takes the other branch than in the fp32 oracle, and every such
element changes its gradient entry by O(1).  tools/vdiff_layers.py shows this entering block by block
(forward taps agree to 1e-3 everywhere; gradient taps drift to ~5e-2 rel-L2 through the 56 blocks), independent of the
gradient scale.  The smooth drawers (swish / QuickGELU) do not have this effect and keep 3e-2; here the stated bound is
max-abs-err <= 8e-2 max|z.grad|, relative L2 error <= 0.12 and cosine similarity >= 0.99 -- the reference's own CUDA path
runs this U-Net under fp16 autocast (sampling.py:9-10) and differs from an fp32 evaluation in the same way.  At 256 x 256,
where the direct alpha * g_pred term dominates z.grad, the measured error is 2.9e-3.  The matched-rounding test below
removes the branch flips and brings the 64 x 64 gradient to 6.5e-3 max-abs / 1.0e-2 rel-L2.
"""
import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import engine as E
from pixray_b200 import util as U
from test_pipeline_gpu import SMALL_CLIP, plant_extremes, random_transforms, report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    return R.VDiffCC12M1().eval().requires_grad_(False)


def _engine(model, hw, cutn=8, seed=3):
    clip = R.init_clip_weights(R.ClipVisual(224, SMALL_CLIP["patch"], SMALL_CLIP["width"], SMALL_CLIP["layers"],
                                            SMALL_CLIP["heads"], SMALL_CLIP["out_dim"]), seed + 1)
    eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(hw, hw), cutn=cutn, clip=[SMALL_CLIP], noise_fac=0.1, seed=seed)
    eng.load_module(E.MOD_VQGAN, model.ref_state_dict())
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, SMALL_CLIP["out_dim"], generator=g), w, float("-inf")) for w in (1.0, -0.3)]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
    steps, alphas, sigmas = U.vdiff_schedule(20)
    rs, ra, rsg = R.vdiff_schedule(20)
    assert np.allclose(steps, rs.numpy(), atol=1e-6) and np.allclose(alphas, ra.numpy(), atol=1e-6)
    eng.vdiff_set_schedule(steps, alphas, sigmas)
    ce = torch.randn(1, 512, generator=g)
    eng.vdiff_set_clip_embed(ce.numpy())
    return eng, clip, prompts, ce, torch.from_numpy(steps), torch.from_numpy(alphas), torch.from_numpy(sigmas), g


def _check(model, hw, it, cutn=8):
    eng, clip, prompts, ce, steps, alphas, sigmas, g = _engine(model, hw, cutn)
    x = torch.randn(1, 3, hw, hw, generator=g) * float(sigmas[it]) + 0.3 * torch.rand(1, 3, hw, hw, generator=g)
    t = steps[it:it + 1]
    synth = lambda zz: R.vdiff_synth(model, zz, t, ce, alphas[it], sigmas[it])[0]  # noqa: E731
    cs = 224
    T = random_transforms(cutn, cs, 5)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    ref = R.iterate(synth, x, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
    _, ref_pred, ref_v = R.vdiff_synth(model, x, t, ce, alphas[it], sigmas[it])
    eng.vdiff_set_iteration(it)
    img = eng.synth(x)
    v = eng.debug_read("vd_v", (1, 3, hw, hw))
    pred = eng.debug_read("vd_pred", (1, 3, hw, hw))
    e_v, m_v = report(f"vdiff {hw}^2 it {it}: v", v, ref_v)
    e_p, _ = report("pred", pred, ref_pred)
    e_i, _ = report("image", img, ref["image"])
    eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    zg = eng.backward()
    e_gi, m_gi = report("d/d image", eng.debug_read("g_img", (1, 3, hw, hw)) / 4096.0, ref["image_grad"])
    e_g, m_g = report("z.grad", zg, ref["z_grad"])
    d = (zg.cpu() - ref["z_grad"])
    idx = d.abs().reshape(-1).argmax().item()
    c_, y_, x_ = idx // (hw * hw), (idx // hw) % hw, idx % hw
    frac = (d.abs() > 1e-2 * m_g).float().mean().item()
    print(f"[parity] z.grad rel-L2 err {d.norm().item() / ref['z_grad'].norm().item():.3e}; max err at (c={c_}, y={y_}, x={x_}); "
          f"{100 * frac:.2f}% of elements off by more than 1% of max|grad|")
    # the U-Net term alone: z.grad = alpha * g_pred + dv/dx^T (-sigma g_pred)
    pre = (ref_pred + 1) / 2
    gi = ref["image_grad"]
    gp = 0.5 * gi * ((gi * (pre - pre.clamp(0, 1))) >= 0)
    un_ref = ref["z_grad"] - float(alphas[it]) * gp
    un_eng = zg.cpu() - float(alphas[it]) * gp
    report("U-Net term of z.grad", un_eng, un_ref)
    assert torch.isfinite(zg).all()
    assert e_v <= 2e-2 * m_v and e_p <= 2e-2 * max(m_v, 1.0) and e_i <= 1e-2
    assert e_gi <= 3e-2 * m_gi
    cos = torch.nn.functional.cosine_similarity(zg.cpu().reshape(1, -1), ref["z_grad"].reshape(1, -1)).item()
    l2 = d.norm().item() / ref["z_grad"].norm().item()
    print(f"[parity] z.grad cosine similarity {cos:.5f}")
    assert e_g <= 8e-2 * m_g and l2 <= 0.12 and cos >= 0.99
    return eng, x, alphas, sigmas


def test_vdiff_synth_and_gradient_64(model):
    """64 x 64: levels 64 ... 1, so the implicit-GEMM convs (64, 32, 16, 8), the im2col path (4, 2, 1), the fused
    attention (T = 16, 4, 1), avg-pool / bilinear adjoints and the skip concatenations are all exercised."""
    eng, x, alphas, sigmas = _check(model, 64, it=6)
    # makenoise (sampling.sample_step_noise) on the pred / v of the synth above
    pred = eng.debug_read("vd_pred", (1, 3, 64, 64)).cpu()
    v = eng.debug_read("vd_v", (1, 3, 64, 64)).cpu()
    noise = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(9))
    xr = R.vdiff_renoise(x, pred, v, alphas, sigmas, 6, noise)
    xe = eng.vdiff_renoise(x.clone().cuda(), 6, noise)
    e, m = report("renoise", xe, xr)
    assert e <= 1e-5 * max(m, 1.0)


def test_vdiff_gradient_with_matched_rounding_points(model):
    """The decisive check of the backward chain: the SAME comparison against the oracle evaluated with fp16-rounded
    weights and fp16 rounding (straight-through) at the tensors the engine stores as fp16, so that the ReLU branches are
    decided on (nearly) the same pre-activations.  The forward then agrees to ~1e-4 and z.grad to the 3e-2 bound of the
    smooth drawers -- what remains of the 64 x 64 gap above is the branch flips, not the kernels."""
    import copy
    mq = copy.deepcopy(model).round_weights_to_fp16_()
    mq.quant = True
    hw, it, cutn, cs = 64, 6, 8, 224
    eng, clip, prompts, ce, steps, alphas, sigmas, g = _engine(mq, hw, cutn)
    x = torch.randn(1, 3, hw, hw, generator=g) * float(sigmas[it]) + 0.3 * torch.rand(1, 3, hw, hw, generator=g)
    t = steps[it:it + 1]
    T = random_transforms(cutn, cs, 5)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    ref = R.iterate(lambda zz: R.vdiff_synth(mq, zz, t, ce, alphas[it], sigmas[it])[0], x, [clip], [prompts],
                    torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
    eng.vdiff_set_iteration(it)
    img = eng.synth(x)
    e_i, _ = report("matched rounding: image", img, ref["image"])
    eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    zg = eng.backward()
    e_g, m_g = report("matched rounding: z.grad", zg, ref["z_grad"])
    l2 = (zg.cpu() - ref["z_grad"]).norm().item() / ref["z_grad"].norm().item()
    print(f"[parity] matched rounding: z.grad rel-L2 err {l2:.3e}")
    assert e_i <= 2e-3
    assert e_g <= 3e-2 * m_g


@pytest.mark.slow
def test_vdiff_synth_and_gradient_256(model):
    """BASELINE config 4's canvas: adds the 16 x 16 attention (T = 256: batched-GEMM chain), split-K convs at 8 x 8 and
    the 256 x 256 / 128-channel layers."""
    _check(model, 256, it=12)
