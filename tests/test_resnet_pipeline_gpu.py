"""The CLIP ResNet perceptors through the rest of the engine, against the oracle pipeline (oracle/ref_path.iterate with
oracle/resnet_ref.py as the tower), with smoke()'s tolerances (losses 5e-3, z.grad 3e-2 of its largest element):

  * one fused iteration with RN50 on the VQGAN and the pixel drawers, with text prompts, image prompts (two targets,
    encode_image_prompts) and spot prompts of both kinds (spot_pass);
  * the three perceptors of quality="better" (RN50 beside two ViTs sharing the cutout batch) in one iteration;
  * an RN50 checkpoint's own text tower against oracle/text_ref.py;
  * a 2-rank cutout-sharded iteration matching the oracle and bit-identical across ranks (skipped with fewer than 2 GPUs).
"""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import ref_path as R
from oracle import text_ref
from oracle.resnet_ref import ResnetRef
from pixray_b200 import cutouts
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_pipeline_gpu import SMALL_CLIP, SMALL_VQ, plant_extremes, report

pytestmark = pytest.mark.gpu
RN50 = E.RESNET_ARCH["RN50"]
CS = 224


class RefClip(torch.nn.Module):
    """ResnetRef on the engine's folded weights, as oracle/ref_path.iterate calls a perceptor"""

    def __init__(self, sd):
        super().__init__()
        self.ref = ResnetRef(sd, folded=True)

    def encode_image(self, x):
        return self.ref.encode_image(x).to(x.dtype)


def _vq(seed):
    return R.init_vqgan_weights(R.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1,
                                          attn_resolutions=(16,), resolution=32, z_channels=128), seed)


def _set(eng, i, table, which=None):
    args = (torch.cat([p[0] for p in table]).numpy(), [p[1] for p in table], [p[2] for p in table])
    if which is None:
        eng.set_prompts(i, *args)
    else:
        eng.set_spot_prompts(i, which, *args)


def run_pipeline(drawer, models, cutn=8, seed=5, extras=True, rank=0, world=1):
    """One pxr_iterate on explicit cutout parameters against ref_path.iterate; returns (engine losses, z.grad, oracle)."""
    g = torch.Generator().manual_seed(seed)
    archs, refs, sds = [], [], []
    for i, m in enumerate(models):
        if m == "RN50":
            sd = S.clip_resnet_state_dict(RN50, seed + 1 + i)
            archs.append(RN50)
            refs.append(RefClip(sd))
        else:
            clip = R.init_clip_weights(R.ClipVisual(224, 32, 128, 2, 2, 64), seed + 1 + i)
            sd = clip.state_dict()
            archs.append(SMALL_CLIP)
            refs.append(clip)
        sds.append(sd)
    if drawer == "vqgan":
        vq = _vq(seed)
        kw = dict(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ)
        idx = torch.randint(1024, (16 * 16,), generator=g)
        z = (vq.quantize.embedding.weight[idx].T.reshape(1, 128, 16, 16) + 0.05 * torch.randn(1, 128, 16, 16, generator=g))
        synth = lambda zz: R.vqgan_synth(vq, zz)  # noqa: E731
    else:
        kw = dict(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(12, 12))
        z = torch.rand(1, 3, 12, 12, generator=g)
        synth = lambda zz: R.pixel_synth(zz, (48, 48))  # noqa: E731
    z = z.contiguous()
    eng = E.B200Engine(cutn=cutn, clip=archs, seed=seed, noise_fac=0.1, rank=rank, world=world, **kw)
    try:
        if drawer == "vqgan":
            eng.load_module(E.MOD_VQGAN, vq.state_dict())
        for i, sd in enumerate(sds):
            eng.load_module(E.MOD_CLIP0 + i, sd)
        eng.finalize()
        if world > 1:
            eng.init_comm()
        rnd = lambda D: torch.randn(1, D, generator=g)  # noqa: E731
        prompts = [[(rnd(a["out_dim"]), 1.0, float("-inf")), (rnd(a["out_dim"]), -0.3, float("-inf"))] for a in archs]
        for i, t in enumerate(prompts):
            _set(eng, i, t)
        kwr, n_spot = {}, 0
        if extras:
            yy, xx = torch.meshgrid(torch.arange(CS), torch.arange(CS), indexing="ij")
            mask = (((yy - 100) ** 2 + (xx - 130) ** 2) < 60 ** 2)[None].expand(3, -1, -1).contiguous()
            spot_on = [[(rnd(a["out_dim"]), 0.8, float("-inf"))] for a in archs]
            spot_off = [[(rnd(a["out_dim"]), 0.5, -0.1)] for a in archs]
            eng.set_spot_mask(mask)
            for i in range(len(archs)):
                _set(eng, i, spot_on[i], 1)
                _set(eng, i, spot_off[i], 0)
            targets = [torch.rand(1, 3, 32, 32, generator=g), torch.rand(1, 3, 60, 40, generator=g) * 0.5 + 0.25]
            eng.set_image_prompts(targets, [0.7, -0.4])
            kwr = dict(image_prompts=list(zip(targets, [0.7, -0.4])), spot_mask=mask, spot_prompts=spot_on,
                       spot_prompts_off=spot_off)
            n_spot = 2
        T = cutouts.sample_transforms(cutn, CS, seed + 11)
        facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, CS, CS, generator=g))
        n_loss = eng.num_losses()
        assert n_loss == len(archs) * (2 + n_spot + (2 if extras else 0))
        zc = z.clone().cuda()
        losses = np.zeros(n_loss, dtype=np.float32)
        eng.iterate(zc, 0.05, 1, params=dict(transforms=T, zoom_padding=E.PAD_BORDER, fill=0.35, noise_facs=facs.numpy(),
                                             noise=noise), losses_out=losses)
        zg = eng.debug_read("z_grad", z.shape).cpu()
    finally:
        eng.close()
    ref = None
    if rank == 0:
        ref = R.iterate(synth, z, refs, prompts, torch.from_numpy(T), CS, "border", 0.35, facs, noise, **kwr)
    return losses, zg, ref


def _compare(label, losses, zg, ref):
    ref_l = np.array([float(l) for l in ref["losses"]], dtype=np.float32)
    print(f"[resnet pipeline] {label}: losses engine {losses} oracle {ref_l}")
    assert len(ref_l) == len(losses) and np.abs(losses - ref_l).max() < 5e-3
    e_g, m_g = report(f"{label} z.grad", zg, ref["z_grad"])
    assert torch.isfinite(zg).all() and e_g <= 3e-2 * m_g


@pytest.mark.parametrize("drawer", ["vqgan", "pixel"])
def test_rn50_iteration_with_image_and_spot_prompts(drawer):
    losses, zg, ref = run_pipeline(drawer, ["RN50"])
    _compare(f"RN50 {drawer}, image + spot prompts", losses, zg, ref)
    l2, zg2, _ = run_pipeline(drawer, ["RN50"])
    assert np.array_equal(losses, l2) and torch.equal(zg, zg2), "two runs differ"


def test_three_perceptors_share_the_cutout_batch():
    losses, zg, ref = run_pipeline("vqgan", ["RN50", "ViT", "ViT"], extras=False)
    _compare("RN50 + two ViTs", losses, zg, ref)


def test_rn50_checkpoint_text_tower():
    sd = S.clip_resnet_state_dict(RN50, 3, text=(512, 12))
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(12, 12), cutn=2, clip=[RN50], seed=0)
    try:
        eng.load_module(E.MOD_CLIP0, sd)
        eng.finalize()
        assert eng.text_tower(0) == dict(width=512, layers=12, ctx=77, out_dim=1024)
        ids = torch.randint(1, 49405, (5, 77), generator=torch.Generator().manual_seed(4))
        ids[:, 0] = 49406
        for r, n in enumerate((3, 10, 40, 76, 20)):
            ids[r, n] = 49407
            ids[r, n + 1:] = 0
        got = eng.encode_text(0, ids).double().cpu()
    finally:
        eng.close()
    want = text_ref.encode_text(sd, ids)
    rel = ((got - want).norm() / want.norm()).item()
    print(f"[resnet pipeline] RN50 text tower rel-L2 {rel:.3e}")
    assert rel <= 4e-3  # the bound of tests/test_text_tower_gpu.py's full-depth towers


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    losses, zg, ref = run_pipeline("vqgan", ["RN50"], rank=rank, world=world)
    torch.save(dict(zg=zg, losses=losses, ref=ref), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_match_one(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in (0, 1))
    assert torch.equal(r0["zg"], r1["zg"]), "the replicated drawer backward must be bit-identical across ranks"
    _compare("RN50, 2 ranks", r0["losses"], r0["zg"], r0["ref"])
