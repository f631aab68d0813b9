"""GPU parity of the whole hot path against the CPU oracle (oracle/ref_path.py), stage by stage, at a size the
oracle finishes in seconds: synth -> cutouts -> encode_image -> Prompt loss -> backward (z.grad) -> Adam/clip_z.

Tolerances (stated, fp16 tensor-core operands with fp32 accumulation vs an fp32 CPU oracle):
  image 5e-3 abs, cutout batch 1e-4 abs given the same image, embeddings 5e-3 abs, losses 2e-3 abs,
  z.grad max-abs-err <= 3e-2 * max|z.grad_oracle|.
"""
import numpy as np
import pytest
import torch

from oracle import ref_path as R
from pixray_b200 import engine as E

pytestmark = pytest.mark.gpu

SMALL_VQ = dict(z_channels=128, n_embed=1024, ch=128, ch_mult=(1, 2), num_res_blocks=1, attn_resolution=16,
                resolution=32)
SMALL_CLIP = dict(width=128, layers=2, heads=2, patch=32, image_res=224, out_dim=64)


def random_transforms(cutn, cs, seed):
    g = np.random.default_rng(seed)
    T = np.zeros((cutn, 3, 3), dtype=np.float32)
    for n in range(cutn):
        a, d = g.uniform(0.9, 1.8, 2)
        b, c = g.uniform(-0.15, 0.15, 2)
        tx, ty = g.uniform(-0.5 * cs, 0.15 * cs, 2)
        p, q = g.uniform(-4e-4, 4e-4, 2)
        if n >= int(0.6 * cutn):  # wide group: shrink so the fill colour shows
            a, d = g.uniform(0.8, 0.98, 2)
            tx, ty = g.uniform(0.0, 0.1 * cs, 2)
        T[n] = [[a, b, tx], [c, d, ty], [p, q, 1.0]]
    return T


def build(cutn=8, image=32, seed=0, clip_cfg=SMALL_CLIP, vq_cfg=SMALL_VQ, n_prompts=2):
    torch.manual_seed(seed)
    vq = R.init_vqgan_weights(R.VQModel(n_embed=vq_cfg["n_embed"], embed_dim=vq_cfg["z_channels"], ch=vq_cfg["ch"],
                                        ch_mult=vq_cfg["ch_mult"], num_res_blocks=vq_cfg["num_res_blocks"],
                                        attn_resolutions=(vq_cfg["attn_resolution"],), resolution=vq_cfg["resolution"],
                                        z_channels=vq_cfg["z_channels"]), seed)
    clip = R.init_clip_weights(R.ClipVisual(224, clip_cfg["patch"], clip_cfg["width"], clip_cfg["layers"],
                                            clip_cfg["heads"], clip_cfg["out_dim"]), seed + 1)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(image, image), vqgan=vq_cfg, cutn=cutn, clip=[clip_cfg],
                       noise_fac=0.1, seed=seed)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, clip_cfg["out_dim"], generator=g), w, float("-inf")) for w in [1.0, -0.3, 0.1][:n_prompts]]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
    f = 2 ** (len(vq_cfg["ch_mult"]) - 1)
    hw = image // f
    idx = torch.randint(vq_cfg["n_embed"], (hw * hw,), generator=g)
    z = vq.quantize.embedding.weight[idx].T.reshape(1, vq_cfg["z_channels"], hw, hw).contiguous()
    z = (z + 0.05 * torch.randn(z.shape, generator=g)).contiguous()
    return vq, clip, eng, prompts, z


def plant_extremes(facs, noise):
    """The d/dmin, d/dmax terms of the global range normalise (slip.py:21-36) land on ONE element each and carry a
    large share of z.grad.  Which element is the extreme is decided by the noise tails, and a 1e-3 forward difference
    (fp16 decoder vs fp32 oracle) can flip a near-tie.  Parity runs therefore plant two unmistakable extremes so both
    sides route those terms to the same element (asserted through the engine's `irange`)."""
    facs, noise = facs.clone(), noise.clone()
    facs[0] = facs[1] = 0.1
    noise[0, 0, 5, 7] = 30.0
    noise[1, 2, 100, 50] = -30.0
    return facs, noise


class _ClampSided(torch.autograd.Function):
    """clamp_with_grad (vqgan.py:66-79) whose BACKWARD takes the side of [0, 1] each pixel is on from `side` (-1 / 0 / +1)
    instead of from its own unclamped value; the forward value is the oracle's own."""

    @staticmethod
    def forward(ctx, x, side):
        ctx.save_for_backward(side)
        return x.clamp(0, 1)

    @staticmethod
    def backward(ctx, g):
        (side,) = ctx.saved_tensors
        return g * (g * side >= 0), None   # g * (g * (x - clamp(x)) >= 0): only the sign of x - clamp(x) matters


def vqgan_synth_with_engine_clamp_sides(vq, eng, image_hw):
    """ClampWithGrad's backward is discontinuous in the unclamped image: a pixel within the engine's fp16 forward error
    (~1.5e-3) of 0 or 1 can sit on the other side of the clamp in the engine, and then a whole pixel's gradient is kept
    on one side and dropped on the other (on the 48x32 canvas ONE such pixel moves z.grad by 3e-2 of its maximum;
    tests/diag_aspect.py).  Returns (synth, n_flipped): the oracle's synth evaluated on the piece of the
    function the engine is on -- identical to R.vqgan_synth wherever the sides agree."""
    H, W = image_hw
    pre_e = eng.debug_read("img_pre", (1, 3, H, W)).cpu()
    side_e = ((pre_e > 1).float() - (pre_e < 0).float())

    def synth(zz):
        zq, _ = R.vector_quantize(zz.movedim(1, 3), vq.quantize.embedding.weight)
        return _ClampSided.apply(vq.decode(zq.movedim(3, 1)).add(1).div(2), side_e)

    return synth, side_e


def report(name, got, ref):
    err = (got.float().cpu() - ref).abs().max().item()
    mag = ref.abs().max().item()
    print(f"[parity] {name}: max_abs_err={err:.3e}  ref_max={mag:.3e}  rel={err / max(mag, 1e-30):.3e}")
    return err, mag


def test_pipeline_stagewise_small():
    cutn, cs = 8, 224
    vq, clip, eng, prompts, z = build(cutn=cutn)
    T = random_transforms(cutn, cs, 3)
    g = torch.Generator().manual_seed(9)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    fill = 0.37
    ref = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z, [clip], [prompts], torch.from_numpy(T), cs, "reflection",
                    fill, facs, noise)

    # z.grad of the oracle must not be degenerate for the comparison to mean anything
    assert ref["z_grad"].abs().max() > 0

    img = eng.synth(z)
    e_img, _ = report("synth image", img, ref["image"])
    # cutouts on the oracle's image isolate the gather kernel from decoder rounding
    batch = eng.make_cutouts(ref["image"], transforms=T, zoom_padding=E.PAD_REFLECTION, fill=fill,
                             noise_facs=facs.numpy(), noise=noise)
    e_batch, _ = report("cutout batch (oracle image in)", batch, ref["batch"])
    # border padding variant
    ref_b = R.make_cutouts(ref["image"], torch.from_numpy(T), cs, "border", fill, facs, noise)
    batch_b = eng.make_cutouts(ref["image"], transforms=T, zoom_padding=E.PAD_BORDER, fill=fill,
                               noise_facs=facs.numpy(), noise=noise)
    e_batch_b, _ = report("cutout batch border", batch_b, ref_b)

    # now the engine's own chain: image -> cutouts -> embeds -> loss -> backward
    batch2 = eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=fill, noise_facs=facs.numpy(),
                              noise=noise)
    report("cutout batch (engine image in)", batch2, ref["batch"])
    emb = eng.encode_image(0)
    e_emb, _ = report("unit embeds", emb, ref["embeds"][0])
    losses = eng.prompt_loss(0)
    ref_losses = torch.stack([l.reshape(()) for l in ref["losses"]])
    e_loss, _ = report("prompt losses", losses, ref_losses)
    zg = eng.backward()
    e_g, m_g = report("z.grad", zg, ref["z_grad"])
    assert torch.isfinite(zg).all()

    assert e_img < 5e-3
    assert e_batch < 1e-4 and e_batch_b < 1e-4
    assert e_emb < 5e-3
    assert e_loss < 2e-3
    assert e_g <= 3e-2 * m_g


def test_a_nan_gradient_is_not_swallowed_by_the_fixed_point_sums():
    """The scatters of the cutout backward accumulate in 64-bit fixed point (order-independent); a NaN contribution has no
    integer representation and must still surface as a NaN gradient, as it does in the reference -- and the next, clean
    iteration must be clean again."""
    cutn, cs = 8, 224
    vq, clip, eng, prompts, z = build(cutn=cutn, seed=2)
    T = random_transforms(cutn, cs, 6)
    g = torch.Generator().manual_seed(3)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    losses = np.zeros(2, dtype=np.float32)
    zc = z.clone().cuda()
    eng.iterate(zc, 0.0, 0, params=dict(transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise),
                losses_out=losses)
    clean = eng.debug_read("z_grad", z.shape).cpu()
    assert torch.isfinite(clean).all()
    bad = noise.clone()
    bad[3, 1, 17, 40] = float("nan")
    zc = z.clone().cuda()
    eng.iterate(zc, 0.0, 1, params=dict(transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=bad),
                losses_out=losses)
    poisoned = eng.debug_read("z_grad", z.shape).cpu()
    assert torch.isnan(poisoned).any(), "a NaN in the cutout batch must reach z.grad"
    zc = z.clone().cuda()
    eng.iterate(zc, 0.0, 2, params=dict(transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise),
                losses_out=losses)
    again = eng.debug_read("z_grad", z.shape).cpu()
    assert torch.equal(again, clean), "the pass after a poisoned one is clean and bit-identical to the first"


def test_intermediate_gradients_small():
    """d loss / d image and d loss / d cutout-batch against autograd on the oracle (finer than z.grad)."""
    cutn, cs = 8, 224
    vq, clip, eng, prompts, z = build(cutn=cutn, seed=5)
    T = torch.from_numpy(random_transforms(cutn, cs, 4))
    g = torch.Generator().manual_seed(11)
    facs = torch.rand(cutn, generator=g) * 0.1
    noise = torch.randn(cutn, 3, cs, cs, generator=g)
    img0 = R.vqgan_synth(vq, z).detach()
    img_r = img0.clone().requires_grad_(True)
    batch_r = R.make_cutouts(img_r, T, cs, "border", 0.6, facs, noise)
    batch_r.retain_grad()
    emb = R.encode_image(clip, batch_r).float()
    loss = sum(R.prompt_loss(emb, *p) for p in prompts)
    loss.backward()

    eng.synth(z)
    eng.make_cutouts(img0, transforms=T.numpy(), zoom_padding=E.PAD_BORDER, fill=0.6, noise_facs=facs.numpy(),
                     noise=noise)
    eng.encode_image(0)
    eng.backward()
    S = 4096.0
    g_batch = eng.debug_read("g_batch", (cutn, 3, cs, cs)) / S
    g_img = eng.debug_read("g_img", (1, 3, 32, 32)) / S
    # direct term only lives in g_batch; the argmin/argmax terms are added inside cutout_backward, so compare away
    # from those two elements
    ref_gb = batch_r.grad.clone()
    flat = batch_r.detach().reshape(-1)
    i_min, i_max = flat.argmin().item(), flat.argmax().item()
    ir = eng.debug_read("irange", (4,), dtype=torch.int32).cpu()
    print("[parity] argmin/argmax element index engine", ir[:2].tolist(), "oracle", [i_min, i_max])
    assert ir[0].item() == i_min and ir[1].item() == i_max  # index bookkeeping: bit-exact
    mask = torch.ones_like(flat, dtype=torch.bool)
    mask[i_min] = False
    mask[i_max] = False
    e1 = (g_batch.cpu().reshape(-1)[mask] - ref_gb.reshape(-1)[mask]).abs().max().item()
    m1 = ref_gb.abs().max().item()
    print(f"[parity] d/d batch: err={e1:.3e} ref_max={m1:.3e}")
    e2, m2 = report("d/d image", g_img, img_r.grad)
    assert e1 <= 3e-2 * m1
    assert e2 <= 3e-2 * m2


def test_adam_clip_and_iterate_small():
    """pxr_iterate = forward + backward + Adam + clip_z.  The VQ argmin makes the optimisation trajectory chaotic
    (one flipped code changes the image), so each iteration is checked from the SAME z: losses and z.grad against the
    oracle, and the fused Adam/clip_z update exactly against torch-semantics Adam fed the engine's own gradient."""
    cutn, cs, lr = 8, 224, 0.05
    vq, clip, eng, prompts, z = build(cutn=cutn, seed=7)
    T = random_transforms(cutn, cs, 8)
    zmin, zmax = R.vqgan_z_bounds(vq)
    lo, hi = eng.z_bounds()
    assert torch.equal(lo.cpu(), zmin.reshape(-1)) and torch.equal(hi.cpu(), zmax.reshape(-1))
    adam = R.AdamState(z)
    z_ref = z.clone()
    losses = np.zeros(2, dtype=np.float32)
    for it in range(3):
        pad = "reflection" if it % 2 == 0 else "border"
        g = torch.Generator().manual_seed(100 + it)
        facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
        r = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z_ref, [clip], [prompts], torch.from_numpy(T), cs, pad, 0.5,
                      facs, noise)
        z_eng = z_ref.clone().cuda()
        torch.cuda.synchronize()
        eng.iterate(z_eng, lr, it, params=dict(transforms=T, zoom_padding=it % 2, fill=0.5, noise_facs=facs.numpy(),
                                               noise=noise), losses_out=losses)
        g_eng = eng.debug_read("z_grad", z.shape).cpu()
        ir = eng.debug_read("irange", (4,), dtype=torch.int32).cpu()
        flat = r["batch"].reshape(-1)
        assert ir[0].item() == flat.argmin().item() and ir[1].item() == flat.argmax().item()
        ref_l = np.array([float(l) for l in r["losses"]], dtype=np.float32)
        print(f"[parity] iter {it}: losses engine {losses} oracle {ref_l}")
        assert np.abs(losses - ref_l).max() < 5e-3
        report(f"iter {it} image", eng.debug_read("img", (1, 3, 32, 32)), r["image"])
        report(f"iter {it} batch", eng.debug_read("batch", (cutn, 3, cs, cs)), r["batch"])
        gb = eng.debug_read("g_batch", (cutn, 3, cs, cs)).cpu().reshape(-1) / 4096.0
        rb = r["batch_grad"].reshape(-1).clone()
        for i in (int(ir[0]), int(ir[1])):
            gb[i] = rb[i] = 0.0  # the range terms are added to these two elements inside cutout_backward
        report(f"iter {it} d/d batch (direct term)", gb, rb)
        report(f"iter {it} d/d pooled", eng.debug_read("g_pooled", (1, 3, cs, cs)) / 4096.0,
               torch.zeros(1, 3, cs, cs))  # magnitude only
        report(f"iter {it} d/d image", eng.debug_read("g_img", (1, 3, 32, 32)) / 4096.0, r["image_grad"])
        # the same inputs through the per-op entry points must give the same gradient as pxr_iterate
        img_it = eng.debug_read("img", (1, 3, 32, 32)).cpu()
        img_op = eng.synth(z_ref).cpu()
        report(f"iter {it} image: per-op synth vs pxr_iterate (same engine)", img_it, img_op)
        eng.make_cutouts(None, transforms=T, zoom_padding=it % 2, fill=0.5, noise_facs=facs.numpy(), noise=noise, it=it)
        eng.encode_image(0)
        g_ops = eng.backward().cpu()
        report(f"iter {it} z.grad per-op path vs pxr_iterate", g_ops, g_eng)
        e_g, m_g = report(f"iter {it} z.grad", g_eng, r["z_grad"])
        # this seed has a tiny, cancellation-dominated gradient (max 3e-4) behind two discontinuities of the path
        # (max-pool argmax and ClampWithGrad's sign mask flip on 1e-3 forward differences): 5e-2 here, 3e-2 elsewhere
        assert e_g <= 5e-2 * m_g
        z_next = torch.maximum(torch.minimum(adam.step(z_ref, g_eng, lr), zmax), zmin)  # clip_z, vqgan.py:202-204
        e_z, _ = report(f"iter {it} z after Adam+clip_z", z_eng, z_next)
        assert e_z < 2e-5
        z_ref = z_next
    assert eng.num_launches() > 0


def test_two_perceptors_share_the_cutout_batch():
    """BASELINE config 3 shape of the path: two CLIP models (patch 16 and patch 32) encode the SAME cutout batch
    (one MakeCutouts per input_resolution, pixray.py:643-649); their gradients add into d loss / d batch."""
    cutn, cs, seed = 8, 224, 31
    torch.manual_seed(seed)
    vq = R.init_vqgan_weights(R.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1,
                                        attn_resolutions=(16,), resolution=32, z_channels=128), seed)
    cfg_a = dict(width=128, layers=2, heads=2, patch=32, image_res=224, out_dim=64)
    cfg_b = dict(width=128, layers=1, heads=2, patch=16, image_res=224, out_dim=64)
    clip_a = R.init_clip_weights(R.ClipVisual(224, 32, 128, 2, 2, 64), seed + 1)
    clip_b = R.init_clip_weights(R.ClipVisual(224, 16, 128, 1, 2, 64), seed + 2)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=cutn, clip=[cfg_a, cfg_b],
                       noise_fac=0.1, seed=seed)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    eng.load_module(E.MOD_CLIP0, clip_a.state_dict())
    eng.load_module(E.MOD_CLIP1, clip_b.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 3)
    pa = [(torch.randn(1, 64, generator=g), 1.0, float("-inf"))]
    pb = [(torch.randn(1, 64, generator=g), 0.5, float("-inf")), (torch.randn(1, 64, generator=g), -0.2, float("-inf"))]
    eng.set_prompts(0, pa[0][0].numpy(), [1.0], [float("-inf")])
    eng.set_prompts(1, torch.cat([p[0] for p in pb]).numpy(), [0.5, -0.2], [float("-inf")] * 2)
    idx = torch.randint(1024, (256,), generator=g)
    z = (vq.quantize.embedding.weight[idx].T.reshape(1, 128, 16, 16) + 0.05 * torch.randn(1, 128, 16, 16, generator=g)).contiguous()
    T = random_transforms(cutn, cs, 6)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    ref = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z, [clip_a, clip_b], [pa, pb], torch.from_numpy(T), cs, "border", 0.3,
                    facs, noise)
    zc = z.clone().cuda()
    losses = np.zeros(3, dtype=np.float32)
    eng.iterate(zc, 0.05, 1, params=dict(transforms=T, zoom_padding=E.PAD_BORDER, fill=0.3, noise_facs=facs.numpy(),
                                         noise=noise), losses_out=losses)
    ref_l = np.array([float(l) for l in ref["losses"]], dtype=np.float32)
    print(f"[parity] two perceptors: losses engine {losses} oracle {ref_l}")
    assert np.abs(losses - ref_l).max() < 5e-3
    e_g, m_g = report("two perceptors z.grad", eng.debug_read("z_grad", z.shape), ref["z_grad"])
    assert e_g <= 3e-2 * m_g


def test_fft_drawer_and_patch14_perceptor():
    """BASELINE config 5 shape of the path at a small size: FftDrawer.synth (fftdrawer.py:78-84; spectrum -> irfft2 ->
    /std -> colour decorrelation -> sigmoid) feeding a patch-14 ViT (T = 257 tokens, the ViT-L/14 token count)."""
    cutn, cs, seed, H = 8, 224, 41, 64
    clip_cfg = dict(width=128, layers=1, heads=2, patch=14, image_res=224, out_dim=64)
    clip = R.init_clip_weights(R.ClipVisual(224, 14, 128, 1, 2, 64), seed)
    eng = E.B200Engine(drawer=E.DRAWER_FFT, image_hw=(H, H), cutn=cutn, clip=[clip_cfg], noise_fac=0.1, seed=seed)
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 1)
    prompts = [(torch.randn(1, 64, generator=g), 1.0, float("-inf")), (torch.randn(1, 64, generator=g), -0.3, float("-inf"))]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    z = (torch.randn(1, 3, H, H // 2 + 1, 2, generator=g) * 0.01).contiguous()  # fft_image(sd=0.01), fftdrawer.py:57
    T = random_transforms(cutn, cs, 7)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    ref = R.iterate(lambda zz: R.fft_synth(zz), z, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.45, facs,
                    noise)
    img = eng.synth(z)
    e_img, _ = report("fft image", img, ref["image"])
    eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.45, noise_facs=facs.numpy(), noise=noise)
    emb = eng.encode_image(0)
    e_emb, _ = report("fft/patch14 embeds", emb, ref["embeds"][0])
    zg = eng.backward()
    e_g, m_g = report("fft spectrum grad", zg, ref["z_grad"])
    assert e_img < 2e-4 and e_emb < 5e-3
    assert e_g <= 3e-2 * m_g
    # Adam without clip_z (FftDrawer.clip_z is a no-op, fftdrawer.py:100-101), lr 0.3 (fftdrawer.py:21)
    zc = z.clone().cuda()
    eng.step(zc, 0.3, 0)
    exp = R.AdamState(z).step(z, zg.cpu(), 0.3)
    e_z, _ = report("fft z after Adam", zc, exp)
    assert e_z < 1e-5


def _stagewise(vq, clip, eng, prompts, z, image, seed):
    """synth -> cutouts -> embeds -> losses -> z.grad on the engine, against the oracle evaluated on the engine's side of
    the clamp (vqgan_synth_with_engine_clamp_sides: the same forward).  Returns the engine's (image, embeds, losses,
    z.grad) and the errors against the stated tolerances' quantities."""
    cutn, cs = 8, 224
    T = random_transforms(cutn, cs, seed)
    g = torch.Generator().manual_seed(seed + 9)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    img = eng.synth(z)
    synth, _ = vqgan_synth_with_engine_clamp_sides(vq, eng, (image, image))
    ref = R.iterate(synth, z, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.37, facs, noise)
    eng.make_cutouts(img, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.37, noise_facs=facs.numpy(), noise=noise)
    emb = eng.encode_image(0).clone()
    losses = eng.prompt_loss(0).clone()
    zg = eng.backward().clone()
    assert torch.isfinite(zg).all()
    err = dict(image=report(f"{image}x{image} image", img, ref["image"])[0],
               embeds=report("unit embeds", emb, ref["embeds"][0])[0],
               losses=report("prompt losses", losses, torch.stack([l.reshape(()) for l in ref["losses"]]))[0])
    err["z_grad"], err["z_grad_max"] = report("z.grad", zg, ref["z_grad"])
    return (img, emb, losses, zg), err


def _assert_pipeline_tolerances(err):
    assert err["image"] < 5e-3
    assert err["embeds"] < 5e-3
    assert err["losses"] < 2e-3
    assert err["z_grad"] <= 3e-2 * err["z_grad_max"]


def test_decoder_attention_rows_longer_than_1024():
    """A 96 x 96 canvas: the 48 x 48 latent gives T = 2304 tokens in the decoder's mid and up-block attention, rows the
    unfused row softmax must cover in full (a 640 x 480 or 1024 x 1024 canvas of the full-size model has T = 1200 / 4096)."""
    vq, clip, eng, prompts, z = build(image=96, seed=13)
    assert z.shape[-1] * z.shape[-2] == 2304
    _, err = _stagewise(vq, clip, eng, prompts, z, 96, 13)
    eng.close()
    _assert_pipeline_tolerances(err)


ATTENTION_PATHS = {
    "fused": {},
    "batched_gemms_row_softmax": {"PXR_FUSED_ATTN": "0"},
    "fp32_stream": {"PXR_CLIP_STREAM": "32"},
}


@pytest.mark.parametrize("path", sorted(ATTENTION_PATHS))
def test_every_attention_path_matches_the_oracle(path, monkeypatch):
    """Each attention / residual-stream path a session can select (read at session create) on the small pipeline."""
    for k in ("PXR_FUSED_ATTN", "PXR_CLIP_STREAM", "PXR_CLIP_LAST_CLS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in ATTENTION_PATHS[path].items():
        monkeypatch.setenv(k, v)
    vq, clip, eng, prompts, z = build(seed=21)
    _, err = _stagewise(vq, clip, eng, prompts, z, 32, 21)
    eng.close()
    _assert_pipeline_tolerances(err)


def test_last_layer_on_all_rows_is_bit_identical(monkeypatch):
    """The last ViT layer restricted to the class rows (default) and run on all rows (PXR_CLIP_LAST_CLS=0) compute the
    class rows with the same operations: embeddings, loss values and z.grad are bit-identical (the prompt-loss kernel
    sums the losses over the cutouts in a fixed order)."""
    outs = {}
    for last_cls in ("1", "0"):
        for k in ("PXR_FUSED_ATTN", "PXR_CLIP_STREAM"):
            monkeypatch.delenv(k, raising=False)
        monkeypatch.setenv("PXR_CLIP_LAST_CLS", last_cls)
        vq, clip, eng, prompts, z = build(seed=23)
        outs[last_cls], err = _stagewise(vq, clip, eng, prompts, z, 32, 23)
        eng.close()
        _assert_pipeline_tolerances(err)
    (img1, emb1, l1, g1), (img0, emb0, l0, g0) = outs["1"], outs["0"]
    assert torch.equal(img1, img0)
    assert torch.equal(emb1, emb0)
    assert torch.equal(l1, l0)
    assert torch.equal(g1, g0)


@pytest.mark.parametrize("width", [384, 640])
def test_vit_width_not_a_multiple_of_256(width):
    """Widths 128 k with odd k have LayerNorm kernels (8-byte vectors only) and match the oracle."""
    clip_cfg = dict(width=width, layers=1, heads=width // 64, patch=32, image_res=224, out_dim=64)
    vq, clip, eng, prompts, z = build(seed=width, clip_cfg=clip_cfg)
    _, err = _stagewise(vq, clip, eng, prompts, z, 32, width)
    eng.close()
    _assert_pipeline_tolerances(err)


@pytest.mark.parametrize("width", [320, 576])
def test_vit_width_without_layernorm_kernel_is_refused(width):
    clip_cfg = dict(width=width, layers=1, heads=width // 64, patch=32, image_res=224, out_dim=64)
    with pytest.raises(E.EngineError, match="multiple of 128"):
        build(clip_cfg=clip_cfg)
