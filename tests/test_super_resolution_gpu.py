"""The super-resolution drawer (PXR_DRAWER_SUPERRES: SuperResolutionDrawer over Real-ESRGAN's RRDBNet x4) on the GPU:
the LeakyReLU epilogue of the dense-block convolutions against torch, the image and z.grad against the restated network
(oracle/rrdbnet_ref.py) in fp32 and at the engine's rounding points, one whole iteration against the oracle pipeline,
repeatability, checkpoint resume, api.run in managed and host mode, and two ranks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ref_path as R
from oracle import rrdbnet_ref as RR
from pixray_b200 import _lib
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_pipeline_gpu import SMALL_CLIP, _ClampSided, plant_extremes, random_transforms, report

pytestmark = pytest.mark.gpu

SHALLOW = dict(num_feat=64, num_block=2, num_grow_ch=32)


def run_conv(x, lda, c_in, wt, n_out, cout_pad, *, bias=None, out_f16=None, res_f16=None, ldc=None, act=0, aux_in=None,
             act_col0=0):
    """pxr_test_conv on an NHWC fp16 tensor x [1, H, W, >= c_in] of pixel stride lda whose first c_in channels are read."""
    _, H, W, _ = x.shape
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    d = _lib.TestGemmDesc()
    d.a, d.lda, d.b = p(x), lda, p(wt)
    d.N, d.block_n, d.alpha = n_out, min(128, cout_pad), 1.0
    d.bias, d.act, d.aux_in, d.act_col0 = p(bias), act, p(aux_in), act_col0
    d.res_f16, d.out_f16, d.ldc = p(res_f16), p(out_f16), ldc
    err = C.create_string_buffer(512)
    rc = _lib.load().pxr_test_conv(C.byref(d), 1, H, W, c_in, cout_pad, 3, err, 512)
    assert rc == 0, err.value.decode()
    torch.cuda.synchronize()


def _conv_weights(w, cin_k, cout_pad):
    """[cout, cin, 3, 3] -> the implicit-GEMM layout [9 * cout_pad, cin_k] (fp16, zero padded)."""
    cout, cin = w.shape[:2]
    out = torch.zeros(9, cout_pad, cin_k)
    out[:, :cout, :cin] = w.permute(2, 3, 0, 1).reshape(9, cout, cin)
    return out.reshape(9 * cout_pad, cin_k).half().cuda()


def _nchw(t, C):
    return t[..., :C].permute(0, 3, 1, 2).float().cpu()


@pytest.mark.parametrize("k", [1, 2, 4])
def test_dense_conv_forward_epilogue(k):
    """conv_k of a dense block: reads the first round_up(64 + 32 (k-1), 64) channels of the 224-channel buffer (weights
    zero beyond the real inputs) and writes lrelu(conv + bias) into its own 32-channel slice, leaving the rest intact."""
    g = torch.Generator().manual_seed(k)
    H, W, Cd, cin = 13, 19, 224, 64 + 32 * (k - 1)
    cin_k = (cin + 63) // 64 * 64
    buf = torch.randn(1, H, W, Cd, generator=g).half().cuda()
    before = buf.clone()
    w = torch.randn(32, cin, 3, 3, generator=g) * 0.05
    b = torch.randn(32, generator=g) * 0.1
    off = cin
    run_conv(buf, Cd, cin_k, _conv_weights(w, cin_k, 32), 32, 32, bias=b.cuda(), out_f16=buf[..., off:], ldc=Cd, act=4)
    want = F.leaky_relu(F.conv2d(_nchw(before, cin), w.half().float(), b, padding=1), 0.2)
    got = _nchw(buf[..., off:off + 32], 32)
    assert (got - want).abs().max().item() <= 2e-3 * want.abs().max().item() + 1e-3
    keep = torch.ones(Cd, dtype=torch.bool)
    keep[off:off + 32] = False
    assert torch.equal(buf[..., keep], before[..., keep])


@pytest.mark.parametrize("col0", [0, 96])
def test_dense_conv_backward_epilogue(col0):
    """The dgrad with the LeakyReLU backward epilogue: in place over the residual (the accumulated gradient), the sum
    multiplied by 1 or 0.2 by the sign of the saved post-activation in the columns >= col0 only."""
    g = torch.Generator().manual_seed(7 + col0)
    H, W, Cd, N = 11, 17, 224, 128
    gy = torch.randn(1, H, W, 64, generator=g).half().cuda()
    w = torch.randn(N, 64, 3, 3, generator=g) * 0.05
    act = torch.randn(1, H, W, Cd, generator=g).half().cuda()
    acc = torch.randn(1, H, W, Cd, generator=g).half().cuda()
    before = acc.clone()
    run_conv(gy, 64, 64, _conv_weights(w, 64, N), N, N, out_f16=acc[..., 64:], res_f16=acc[..., 64:], ldc=Cd, act=5,
             aux_in=act[..., 64:], act_col0=col0)
    s = F.conv2d(_nchw(gy, 64), w.half().float(), padding=1) + _nchw(before[..., 64:], N)
    mask = torch.where(_nchw(act[..., 64:], N) > 0, 1.0, 0.2)
    mask[:, :col0] = 1.0
    want = s * mask
    got = _nchw(acc[..., 64:64 + N], N)
    assert (got - want).abs().max().item() <= 2e-3 * want.abs().max().item() + 2e-3
    assert torch.equal(acc[..., :64], before[..., :64]) and torch.equal(acc[..., 64 + N:], before[..., 64 + N:])


def _engine(sd, hw, arch=None, cutn=8, seed=3):
    clip = R.init_clip_weights(R.ClipVisual(224, SMALL_CLIP["patch"], SMALL_CLIP["width"], SMALL_CLIP["layers"],
                                            SMALL_CLIP["heads"], SMALL_CLIP["out_dim"]), seed + 1)
    eng = E.B200Engine(drawer=E.DRAWER_SUPERRES, image_hw=hw, superres=arch, cutn=cutn, clip=[SMALL_CLIP], seed=seed)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, SMALL_CLIP["out_dim"], generator=g), w, float("-inf")) for w in (1.0, -0.3)]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [p[1] for p in prompts], [p[2] for p in prompts])
    return eng, clip, prompts


def _latent(hw, seed):
    return torch.rand(1, 3, hw[0] // 4, hw[1] // 4, generator=torch.Generator().manual_seed(seed))


@pytest.fixture(scope="module")
def full_sd():
    return S.rrdbnet_state_dict(0)


@pytest.mark.parametrize("case", ["full_32x48", "shallow_52x36"])
def test_forward_image_matches_the_oracle(case, full_sd):
    if case == "full_32x48":
        sd, arch, hw = full_sd, None, (32, 48)
    else:
        sd, arch, hw = S.rrdbnet_state_dict(1, **SHALLOW), SHALLOW, (52, 36)
    eng, _, _ = _engine(sd, hw, arch)
    z = _latent(hw, 4)
    img = eng.synth(z)
    ref = RR.superres_synth(z.double(), sd).float()
    e, _ = report(f"superres image {case}", img, ref)
    pre = RR.rrdbnet(z.double(), sd)
    print(f"[parity] {case}: pre-clamp range [{pre.min().item():.3f}, {pre.max().item():.3f}], "
          f"{((pre < 0) | (pre > 1)).double().mean().item():.3%} of the pixels clamped")
    assert tuple(img.shape) == (1, 3) + hw and e <= 5e-3


def _zgrad_case(sd, hw, arch, matched, seed=5, cutn=8, cs=224):
    eng, clip, prompts = _engine(sd, hw, arch, cutn)
    g = torch.Generator().manual_seed(seed)
    z = _latent(hw, seed)
    T = random_transforms(cutn, cs, seed)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    img = eng.synth(z)
    pre_e = eng.debug_read("img_pre", (1, 3) + hw).cpu()
    side_e = (pre_e > 1).float() - (pre_e < 0).float()
    synth = lambda zz: _ClampSided.apply(RR.rrdbnet(zz, sd, matched), side_e)  # noqa: E731
    ref = R.iterate(synth, z, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
    eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    zg = eng.backward()
    return img, zg, ref


def test_zgrad_with_matched_rounding_points(full_sd):
    """The decisive check of the backward chain: the oracle evaluated with the engine's fp16 weights (0.2 folded into
    conv5) and straight-through fp16 rounding at every tensor the engine stores in fp16, so the LeakyReLU kinks and the
    clamp are decided on (nearly) the same values."""
    img, zg, ref = _zgrad_case(full_sd, (32, 48), None, True)
    e_i, _ = report("superres matched: image", img, ref["image"])
    e_g, m_g = report("superres matched: z.grad", zg, ref["z_grad"])
    assert e_i <= 2e-3 and e_g <= 3e-2 * m_g


@pytest.mark.parametrize("case", ["full_32x48", "shallow_52x36"])
def test_zgrad_against_pure_fp32(case, full_sd):
    """Against the fp32 network with no rounding at all: the bound DESIGN states for the drawer."""
    if case == "full_32x48":
        sd, arch, hw = full_sd, None, (32, 48)
    else:
        sd, arch, hw = S.rrdbnet_state_dict(1, **SHALLOW), SHALLOW, (52, 36)
    img, zg, ref = _zgrad_case(sd, hw, arch, False)
    report(f"superres fp32 {case}: image", img, ref["image"])
    e_g, m_g = report(f"superres fp32 {case}: z.grad", zg, ref["z_grad"])
    l2 = (zg.cpu() - ref["z_grad"]).norm().item() / ref["z_grad"].norm().item()
    print(f"[parity] superres fp32 {case}: z.grad rel-L2 err {l2:.3e}")
    assert e_g <= 3e-2 * m_g


def _iterate_once(sd, hw, arch, it=2, seed=6):
    eng, clip, prompts = _engine(sd, hw, arch)
    z = _latent(hw, seed).cuda()
    eng.iterate(z, 0.05, it)
    eng.sync()
    return eng, z, eng.debug_read("z_grad", eng.z_shape).cpu()


def test_one_iteration_matches_the_oracle():
    """pxr_iterate (synth -> cutouts -> ViT -> prompts -> backward -> Adam with clip_z to [0, 1]) against ref_path.iterate
    with the restated drawer, on explicit cutout parameters."""
    sd, hw, cutn, cs = S.rrdbnet_state_dict(2, **SHALLOW), (48, 32), 8, 224
    eng, clip, prompts = _engine(sd, hw, SHALLOW, cutn)
    g = torch.Generator().manual_seed(9)
    z = _latent(hw, 9)
    T = random_transforms(cutn, cs, 9)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    eng.synth(z)
    pre_e = eng.debug_read("img_pre", (1, 3) + hw).cpu()
    side_e = (pre_e > 1).float() - (pre_e < 0).float()
    ref = R.iterate(lambda zz: _ClampSided.apply(RR.rrdbnet(zz, sd, True), side_e), z, [clip], [prompts],
                    torch.from_numpy(T), cs, "reflection", 0.4, facs, noise)
    zc = z.clone().cuda()
    losses = np.zeros(eng.num_losses(), dtype=np.float32)
    eng.iterate(zc, 0.05, 0, params=dict(transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(),
                                          noise=noise), losses_out=losses)
    zg = eng.debug_read("z_grad", eng.z_shape).cpu()
    e_g, m_g = report("superres iterate: z.grad", zg, ref["z_grad"])
    assert e_g <= 3e-2 * m_g
    assert np.allclose(losses, np.array([float(v) for v in ref["losses"]]), rtol=2e-3, atol=1e-4)
    zn = zc.cpu()
    assert float(zn.min()) >= 0.0 and float(zn.max()) <= 1.0 and not torch.equal(zn, z)


def test_repeated_runs_are_bit_identical(full_sd):
    _, z1, g1 = _iterate_once(full_sd, (32, 48), None)
    _, z2, g2 = _iterate_once(full_sd, (32, 48), None)
    assert torch.equal(g1, g2) and torch.equal(z1.cpu(), z2.cpu())


def _settings(tmp_path, **kw):
    from PIL import Image
    rgb = (np.random.default_rng(4).random((38, 50, 3)) * 255).astype(np.uint8)
    Image.fromarray(rgb).save(tmp_path / "init.png")
    base = dict(prompts="a cat", drawer="super_resolution", size=[50, 38], clip_models="ViT-B/32", num_cuts=4,
                outdir="", seed="3", b200_allow_synthetic=True, vector_prompts="none",
                init_image=str(tmp_path / "init.png"))
    base.update(kw)
    return base


@pytest.mark.parametrize("managed", [True, False], ids=["managed", "host"])
def test_api_run_completes_on_the_engine(tmp_path, managed):
    api.run(**_settings(tmp_path, iterations=3, b200_device_checkdrop=managed))
    st = api._state
    assert isinstance(st.drawer, api.P.SuperResolutionDrawer)
    assert st.engine.image_hw == (36, 48) and st.engine.z_shape == (1, 3, 9, 12)
    z = st.drawer.get_z().cpu()
    assert float(z.min()) >= 0.0 and float(z.max()) <= 1.0 and st.cur_iteration == 3
    assert st.drawer.to_image().size == (48, 36)


def test_checkpoint_continues_bit_identically(tmp_path):
    def start():
        api.reset_settings()
        api.add_settings(**_settings(tmp_path, iterations=8))
        args = api.apply_settings()
        api.do_init(args)
        return args

    args = start()
    for it in range(2):
        api.train(args, it)
        api._state.cur_iteration = it + 1
    path = str(tmp_path / "ckpt.bin")
    api.save_checkpoint(path)
    for it in range(2, 4):
        api.train(args, it)
    api._state.engine.sync()
    z_a = api._state.drawer.get_z().cpu().clone()
    args = start()
    assert api.load_checkpoint(path) == 2
    for it in range(2, 4):
        api.train(args, it)
    api._state.engine.sync()
    assert torch.equal(api._state.drawer.get_z().cpu(), z_a)


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    sd = S.rrdbnet_state_dict(3, **SHALLOW)
    eng = E.B200Engine(drawer=E.DRAWER_SUPERRES, image_hw=(48, 32), superres=SHALLOW, cutn=8, clip=[SMALL_CLIP], seed=9,
                       device=rank, rank=rank, world=world)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    eng.init_comm()
    g = torch.Generator().manual_seed(2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    z = _latent((48, 32), 5).cuda()
    eng.iterate(z, 0.05, 0)
    eng.sync()
    torch.save(dict(z=z.cpu(), zg=eng.debug_read("z_grad", eng.z_shape).cpu()), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_match_the_single_gpu_gradient(tmp_path):
    import torch.multiprocessing as mp
    from test_multigpu import _free_port
    mp.spawn(_rank_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in (0, 1))
    assert torch.equal(r0["zg"], r1["zg"]) and torch.equal(r0["z"], r1["z"])
    sd = S.rrdbnet_state_dict(3, **SHALLOW)
    eng = E.B200Engine(drawer=E.DRAWER_SUPERRES, image_hw=(48, 32), superres=SHALLOW, cutn=8, clip=[SMALL_CLIP], seed=9)
    eng.load_module(E.MOD_VQGAN, sd)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    g = torch.Generator().manual_seed(2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    z = _latent((48, 32), 5).cuda()
    eng.iterate(z, 0.05, 0)
    eng.sync()
    zg = eng.debug_read("z_grad", eng.z_shape).cpu()
    e, m = report("superres two ranks vs one GPU: z.grad", r0["zg"], zg)
    assert e <= 1e-3 * m
