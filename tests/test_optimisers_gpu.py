"""GPU: the optimiser update rules of pxr_set_optimizer (Adam, AdamW, Adagrad, Adamax, DiffGrad) against the float64
oracle (oracle/optim_ref.py) on the latents of three drawers; the managed step against the plain one; checkpoints of
every rule; pixray.run with each rule; and the replicated step across two ranks."""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import optim_ref as R
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_pipeline_gpu import SMALL_CLIP, build

pytestmark = pytest.mark.gpu

KINDS = list(E.OPTIMISERS)
# the rates the reference suggests beside each constructor (pixray.py:538-546)
LR = {"Adam": 0.1, "AdamW": 0.2, "Adagrad": 0.5, "Adamax": 0.5, "DiffGrad": 2.0}
HEADER = 64  # sizeof(StateHeader) in engine.cu


def gradients(steps, n, seed):
    """float32 gradients with magnitudes from 1e-6 to 1e3, exact zeros and sign flips between consecutive steps."""
    rng = np.random.default_rng(seed)
    g = 10.0 ** rng.uniform(-6, 3, size=(steps, n)) * np.where(rng.random((steps, n)) < 0.5, -1.0, 1.0)
    g[:, : n // 8] = 0.0
    g[1::2, n // 8: n // 4] = -g[0::2, n // 8: n // 4]  # steps is even
    g[rng.random((steps, n)) < 0.05] = 0.0
    return g.astype(np.float32)


def set_z(eng, z):
    """Load z into the engine through its state blob (an Adam session's version-1 layout: header, z, m, v)."""
    blob = bytearray(eng.save_state())
    zb = z.numel() * 4
    assert len(blob) == HEADER + 3 * zb
    blob[HEADER:HEADER + zb] = z.detach().cpu().float().contiguous().numpy().tobytes()
    eng.load_state(bytes(blob))


@pytest.fixture(scope="module")
def vdiff_sd():
    return S.vdiff_state_dict(0)


def _clip_sd(seed):
    return S.clip_state_dict(SMALL_CLIP, seed)


def drawer_case(name, vdiff_sd=None):
    """(engine, z0, lo, hi): lo / hi broadcast against z (None: no clamp)."""
    g = torch.Generator().manual_seed(11)
    if name == "vqgan":
        _, _, eng, _, z = build(cutn=8, seed=29)
        lo, hi = eng.z_bounds()
        return eng, z.detach(), lo.cpu().view(1, -1, 1, 1).double(), hi.cpu().view(1, -1, 1, 1).double()
    if name == "fast_pixel":
        eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(16, 16), cutn=8, clip=[SMALL_CLIP], seed=3)
        z = torch.rand(1, 3, 16, 16, generator=g)
        lo, hi = torch.zeros(()).double(), torch.ones(()).double()
    else:
        eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(64, 64), cutn=8, clip=[SMALL_CLIP], seed=3)
        eng.load_module(E.MOD_VQGAN, vdiff_sd)
        z = torch.randn(1, 3, 64, 64, generator=g)
        lo = hi = None
    eng.load_module(E.MOD_CLIP0, _clip_sd(4))
    eng.finalize()
    return eng, z, lo, hi


@pytest.mark.parametrize("drawer", ["vqgan", "fast_pixel", "vdiff"])
@pytest.mark.parametrize("kind", KINDS)
def test_step_matches_the_float64_oracle(kind, drawer, vdiff_sd):
    """30 pxr_step calls on given gradients with a reset at step 15, against the oracle + clip_z from the same fp32 z."""
    eng, z0, lo, hi = drawer_case(drawer, vdiff_sd)
    lr, n, steps = LR[kind], z0.numel(), 30
    set_z(eng, z0)
    eng.set_optimizer(E.OPTIMISERS[kind])
    G = gradients(steps, n, 7)
    ref = R.Optimizer(kind, float(np.float32(lr)), n)
    zr = z0.double().reshape(-1).numpy()
    zc = z0.clone().cuda()
    clamp = (lambda t: t) if lo is None else (lambda t: torch.maximum(torch.minimum(t, hi), lo))
    for k in range(steps):
        if k == 15:
            eng.reset_optimizer()
            ref.reset()
        eng.set_z_grad(torch.from_numpy(G[k]).reshape(z0.shape).cuda())
        eng.step(zc, lr, k)
        pre = torch.from_numpy(ref.step(zr, G[k].astype(np.float64))).reshape(z0.shape)
        zr = clamp(pre).reshape(-1).numpy()
    zz = zc.cpu().double()
    zref = torch.from_numpy(zr).reshape(z0.shape)
    tol = 1e-5 * (zref.abs().max().item() + steps * lr)
    err = (zz - zref).abs().max().item()
    print(f"[optimiser] {kind} on {drawer}: max|z - z_ref| {err:.3e} (bound {tol:.3e})")
    assert err <= tol
    if lo is not None:
        lo32, hi32 = lo.float().double().expand_as(zz), hi.float().double().expand_as(zz)
        assert bool(((zz >= lo32) & (zz <= hi32)).all())
        below, above = pre < lo - tol, pre > hi + tol  # clamped by the oracle, clear of the rounding band
        assert bool(below.any() or above.any()) or drawer == "vqgan"
        assert torch.equal(zz[below], lo32[below]) and torch.equal(zz[above], hi32[above])


@pytest.mark.parametrize("kind", KINDS)
def test_managed_step_equals_the_plain_step(kind):
    """The managed kernel on the gradient its own iteration produced equals pxr_step on that gradient, through a scheduled
    drop that leaves a fresh instance of the rule behind: identical bits."""
    from test_pipeline_gpu import random_transforms
    _, _, eng_a, _, z = build(cutn=8, seed=17)
    _, _, eng_b, _, _ = build(cutn=8, seed=17)
    T = random_transforms(8, 224, 3)
    for e in (eng_a, eng_b):
        e.set_optimizer(E.OPTIMISERS[kind])
    base = 0.05
    eng_a.set_schedule(base, iter_drop_delay=12, max_loss_drops=1, auto_stop=False, drops=[2])
    za, zb = z.clone().cuda(), z.clone().cuda()
    eng_b.synth(zb)  # loads z into the plain engine
    lr = float(np.float32(base))
    for it in range(6):
        eng_a.iterate(za, 0.0, it, params=dict(transforms=T, zoom_padding=it % 2, fill=0.4))
        eng_a.sync()
        eng_b.set_z_grad(eng_a.debug_read("z_grad", z.shape).contiguous())
        eng_b.step(zb, lr, it)
        assert torch.equal(za, zb), (kind, it, (za - zb).abs().max().item())
        if it == 2:  # learning_rate / 10 (pixray.py:522-539), in the managed kernel's arithmetic
            lr = float(np.float32(np.float64(np.float32(base)) / 10))
            eng_b.reset_optimizer()
    assert eng_a.poll_status()["num_loss_drop"] == 1


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "Adam"])
def test_checkpoint_resume_follows_the_uninterrupted_run(kind):
    """As tests/test_train_control_gpu.py checks for Adam: save after 3 managed iterations, load into a fresh engine of the
    same rule and continue."""
    _, _, eng_a, _, z = build(cutn=8, seed=23)
    _, _, eng_b, _, _ = build(cutn=8, seed=23)
    for e in (eng_a, eng_b):
        e.set_optimizer(E.OPTIMISERS[kind])
        e.set_schedule(0.05, iter_drop_delay=12, max_loss_drops=2, auto_stop=False, drops=[1])
    za = z.clone().cuda()
    for it in range(3):
        eng_a.iterate(za, 0.0, it)
    eng_a.sync()
    blob = eng_a.save_state()
    arrays = 3 if kind == "DiffGrad" else 2
    assert len(blob) == HEADER + 8 + (1 + arrays) * 4 * z.numel()
    for it in range(3, 7):
        eng_a.iterate(za, 0.0, it)
    eng_a.sync()
    eng_b.load_state(blob)
    zb = eng_b.read_z()
    for it in range(3, 7):
        eng_b.iterate(zb, 0.0, it)
    eng_b.sync()
    ra, rb = eng_a.poll_status(), eng_b.poll_status()
    assert ra["num_loss_drop"] == rb["num_loss_drop"] == 1 and abs(ra["lr"] - rb["lr"]) < 1e-9
    moved = (za - z.cuda()).abs().max().item()
    diff = (za - zb).abs()
    assert moved > 0.02 and diff.median().item() < 1e-3 * moved and (diff > 0.1 * moved).float().mean().item() < 0.02


def test_checkpoints_name_their_rule():
    _, _, eng_a, _, z = build(cutn=8, seed=31)
    _, _, eng_b, _, _ = build(cutn=8, seed=31)
    assert len(eng_b.save_state()) == HEADER + 3 * 4 * z.numel()  # Adam: version 1, unchanged
    eng_a.set_optimizer(E.OPT_DIFFGRAD)
    blob = eng_a.save_state()
    with pytest.raises(E.EngineError, match="DiffGrad.*Adam"):
        eng_b.load_state(blob)
    eng_b.set_optimizer(E.OPT_ADAMAX)
    with pytest.raises(E.EngineError, match="DiffGrad.*Adamax"):
        eng_b.load_state(blob)
    eng_b.set_optimizer(E.OPT_DIFFGRAD)
    eng_b.load_state(blob)
    with pytest.raises(E.EngineError, match="unknown optimiser kind 5"):
        eng_b.set_optimizer(5)


@pytest.mark.parametrize("kind", KINDS)
def test_api_run_with_each_rule(kind):
    """pixray's loop on vqgan at 128x128 with one scheduled drop, device-managed and host-driven: both move z, report
    finite losses and take the same control decisions."""
    from pixray_b200 import api
    seen = {}
    for managed in (True, False):
        api.reset_settings()
        api.add_settings(prompts="a cat", drawer="vqgan", size=[128, 128], clip_models="ViT-B/16", iterations=12,
                         num_cuts=8, outdir="", vector_prompts="none", b200_allow_synthetic=True, seed="5",
                         learning_rate_drops=[50], optimiser=kind, b200_device_checkdrop=managed)
        args = api.apply_settings()
        api.do_init(args)
        st = api._state
        z0 = st.drawer.get_z_copy().clone()
        assert api.do_run(args) is True
        st.engine.sync()
        moved = (st.engine.read_z().cpu() - z0.cpu()).abs().max().item()
        assert np.isfinite(st.losses).all() and moved > 0
        seen[managed] = (st.num_loss_drop, st.cur_iteration)
    assert seen[True] == seen[False] == (1, 12)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from test_pipeline_gpu import SMALL_VQ, random_transforms
    from oracle import ref_path as Rp
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    seed = 21
    vq = Rp.init_vqgan_weights(Rp.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1,
                                          attn_resolutions=(16,), resolution=32, z_channels=128), seed)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=8, clip=[SMALL_CLIP], seed=seed,
                       device=rank, rank=rank, world=world)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    eng.load_module(E.MOD_CLIP0, _clip_sd(seed + 1))
    eng.finalize()
    eng.init_comm()
    g = torch.Generator().manual_seed(seed + 2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    idx = torch.randint(1024, (256,), generator=g)
    z = (vq.quantize.embedding.weight[idx].T.reshape(1, 128, 16, 16) + 0.05 * torch.randn(1, 128, 16, 16, generator=g)).contiguous()
    eng.set_optimizer(E.OPT_DIFFGRAD)
    T = random_transforms(8, 224, 3)
    zc = z.clone().cuda()
    for it in range(4):
        eng.iterate(zc, 0.5, it, params=dict(transforms=T, zoom_padding=it % 2, fill=0.4))
    eng.sync()
    torch.save(dict(z=zc.cpu(), z0=z), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_diffgrad_is_bit_identical_across_ranks(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_rank_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / n, weights_only=False) for n in ("rank0.pt", "rank1.pt"))
    assert torch.equal(r0["z"], r1["z"]) and not torch.equal(r0["z"], r0["z0"])
