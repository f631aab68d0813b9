"""Cutout sets on the engine: perceptors of different input resolutions in one session (pixray.py:642-649, 1266-1336).

  * additivity: d loss / d image of a two-set session is, bit for bit, the fp32 sum of two one-set sessions (one per
    resolution, same perceptors, prompts and cutout parameters), and every loss entry equals theirs, with the
    cutout-space saturation loss once per set;
  * set 0 is unchanged: with engine-drawn parameters its batch is bit-identical to a one-set session's, while set 1
    draws from Philox streams of its own;
  * the per-op path (pxr_make_cutouts_set / pxr_encode_image / pxr_prompt_loss / pxr_backward) equals pxr_iterate_sets
    bit for bit, and two runs give identical bits;
  * quality "best" and "supreme" at full depth (seeded synthetic weights) through the public API, managed and host mode;
  * parity with oracle/multires_ref.iterate_sets (float64; pinned to the reference's ascend_txt by
    tests/golden/multires_ascend.npz) at DESIGN.md 3's tolerances -- cutouts 1e-4, embeddings 5e-3, losses 5e-3, z.grad
    3e-2 of its largest element -- for RN50x4's widths (one block per stage) at 288 beside a 2-layer ViT-B/32, and a
    2-layer ViT-L/14@336px-shaped tower beside a 2-layer ViT-B/16, on a square and a non-square canvas, with an image
    prompt and the saturation, palette and smoothness losses; and on two ranks (two GPUs only).
"""
import os
import socket

import numpy as np
import pytest
import torch

from oracle import multires_ref as MR
from oracle import ref_path as R
from oracle.resnet_ref import ResnetRef
from pixray_b200 import api
from pixray_b200 import cutouts
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu

V224 = dict(width=128, layers=2, heads=2, patch=32, image_res=224, out_dim=64)
V288 = dict(width=128, layers=2, heads=2, patch=32, image_res=288, out_dim=64)
CUTN = 8


def _params(cs, seed, noise=True, canvas=(48, 48)):
    g = torch.Generator().manual_seed(seed)
    p = dict(transforms=cutouts.sample_transforms(CUTN, cs, seed, aspect=canvas[1] / canvas[0]), zoom_padding=E.PAD_BORDER,
             fill=0.35)
    if noise:
        p.update(noise_facs=(torch.rand(CUTN, generator=g) * 0.1).numpy(),
                 noise=torch.randn(CUTN, 3, cs, cs, generator=g).cuda())
    return p


def _engine(archs, seed=3, aux=True, canvas=(48, 48)):
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=canvas, grid=(12, 12), cutn=CUTN, cut_size=archs[0]["image_res"],
                       clip=archs, seed=seed, noise_fac=0.1, cut_aspect=canvas[1] / canvas[0])
    for i, a in enumerate(archs):
        eng.load_module(E.MOD_CLIP0 + i, S.clip_state_dict(a, 11 + a["image_res"] + 7 * a["layers"]))
    eng.finalize()
    for i, a in enumerate(archs):
        g = torch.Generator().manual_seed(100 + a["image_res"])
        eng.set_prompts(i, torch.randn(2, a["out_dim"], generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    if aux:
        eng.add_aux_loss(E.LOSS_SATURATION, 1.0, [0.7])
    return eng


def _z(seed=1):
    return torch.rand(1, 3, 12, 12, generator=torch.Generator().manual_seed(seed)).cuda()


def _iterate(eng, params):
    z = _z()
    losses = np.zeros(eng.num_losses(), dtype=np.float32)
    eng.iterate(z, 0.05, 1, params=params, losses_out=losses)
    g_img = eng.debug_read("g_img", (3, *eng.image_hw)).cpu()
    zg = eng.debug_read("z_grad", eng.z_shape).cpu()
    return losses, g_img, zg


@pytest.mark.parametrize("canvas", [(48, 48), (40, 64)])
def test_two_sets_add_up_bit_for_bit(canvas):
    p224, p288 = _params(224, 5, canvas=canvas), _params(288, 6, canvas=canvas)
    two = _engine([V224, V288], canvas=canvas)
    try:
        assert two.cutout_sets() == [224, 288] and two.num_losses() == 4 + 2
        l2, g2, _ = _iterate(two, [p224, p288])
    finally:
        two.close()
    outs = []
    for arch, p in ((V224, p224), (V288, p288)):
        one = _engine([arch], canvas=canvas)
        try:
            outs.append(_iterate(one, [p]))
        finally:
            one.close()
    (la, ga, _), (lb, gb, _) = outs
    print(f"[multires] canvas {canvas}: losses {l2}; max |d loss / d image| {g2.abs().max():.3e}")
    assert np.isfinite(l2).all() and torch.isfinite(g2).all() and g2.abs().max() > 0
    # loss vector: prompts of perceptor 0, of perceptor 1, then saturation of set 0 and of set 1
    assert np.array_equal(l2, np.concatenate([la[:2], lb[:2], la[2:], lb[2:]]))
    assert torch.equal(g2, ga + gb)


def test_set0_is_unchanged_and_set1_has_its_own_streams():
    two, one0, one1 = _engine([V224, V288], aux=False), _engine([V224], aux=False), _engine([V288], aux=False)
    try:
        for e in (two, one0, one1):
            e.iterate(_z(), 0.05, 4)
        b_two = two.debug_read("batch", (CUTN, 3, 224, 224)).cpu()
        b_one = one0.debug_read("batch", (CUTN, 3, 224, 224)).cpu()
        assert torch.equal(b_two, b_one)
        s1 = two.debug_read("set1.batch", (CUTN, 3, 288, 288)).cpu()
        s1_alone = one1.debug_read("batch", (CUTN, 3, 288, 288)).cpu()
        assert torch.isfinite(s1).all() and not torch.equal(s1, s1_alone)
        m1 = two.debug_read("set1.minv", (CUTN, 9)).cpu()
        m1_alone = one1.debug_read("minv", (CUTN, 9)).cpu()
        assert not torch.equal(m1, m1_alone)
    finally:
        for e in (two, one0, one1):
            e.close()


def _per_op(eng, params):
    img = eng.synth(_z())
    for s, p in enumerate(params):
        eng.make_cutouts(img, it=1, cut_set=s, **p)
    losses = []
    for i in range(2):
        eng.encode_image(i)
        losses.append(eng.prompt_loss(i).cpu())
    zg = eng.backward().cpu()
    return torch.cat(losses), zg


def test_per_op_path_equals_iterate_sets():
    params = [_params(224, 8, noise=False), _params(288, 9, noise=False)]
    runs = []
    for _ in range(2):
        eng = _engine([V224, V288], aux=False)
        try:
            lo, zo = _per_op(eng, params)
            lf, _, zf = _iterate(eng, params)
        finally:
            eng.close()
        assert torch.equal(zo, zf) and np.array_equal(lo.numpy(), lf)
        runs.append((lf, zf))
    assert np.array_equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_iterate_with_one_params_struct_names_iterate_sets():
    eng = _engine([V224, V288], aux=False)
    try:
        with pytest.raises(E.EngineError, match="pxr_iterate_sets"):
            eng.iterate(_z(), 0.05, 1, params=_params(224, 1, noise=False))
        with pytest.raises(E.EngineError, match="spot prompts"):
            eng.set_spot_prompts(0, 1, np.ones((1, 64), np.float32), [1.0], [float("-inf")])
    finally:
        eng.close()


def _preset_run(tmp_path, quality, managed):
    api.reset_settings()
    api.add_settings(prompts="a red boat", quality=quality, size=[64, 64], iterations=3, seed="3", outdir=str(tmp_path),
                     b200_allow_synthetic=True, vector_prompts="none", save_every=0, display_every=0,
                     custom_loss="saturation", b200_device_checkdrop=managed)
    args = api.apply_settings()
    api.do_init(args)
    st = api._state
    eng = st.engine
    assert eng.cutout_sets() == [288, 224]
    out = []
    for it in range(2):
        losses = np.zeros(eng.num_losses(), dtype=np.float32)
        eng.iterate(st.drawer.get_z(), st.lr, it, losses_out=losses)
        out.append(losses)
    eng.sync()
    z = st.drawer.get_z().detach().cpu().clone()
    eng.close()
    api.reset_settings()
    return np.stack(out), z


@pytest.mark.parametrize("quality,n_perc", [("best", 3), ("supreme", 4)])
def test_best_and_supreme_presets_run(tmp_path, quality, n_perc):
    (l_host, z_host), (l_man, z_man) = _preset_run(tmp_path, quality, False), _preset_run(tmp_path, quality, True)
    print(f"[multires] {quality}: losses {l_host[0]}")
    assert l_host.shape[1] == n_perc + 2  # a prompt per perceptor, saturation per set
    assert np.isfinite(l_host).all() and torch.isfinite(z_host).all()
    assert np.array_equal(l_host, l_man)


class _RefResnet(torch.nn.Module):
    def __init__(self, sd):
        super().__init__()
        self.ref = ResnetRef(sd, folded=True)

    def encode_image(self, x):
        return self.ref.encode_image(x).to(x.dtype)


PAL = [0.9, 0.1, 0.1, 0.1, 0.8, 0.2, 0.2, 0.2, 0.9]
CASES = {
    "rn50x4+vitb32": [dict(E.RESNET_ARCH["RN50x4"], blocks=(1, 1, 1, 1), layers=4),
                      dict(E.CLIP_ARCH["ViT-B/32"], layers=2)],
    "vitl336+vitb16": [dict(E.CLIP_ARCH["ViT-L/14@336px"], layers=2), dict(E.CLIP_ARCH["ViT-B/16"], layers=2)],
}


def run_parity(case, canvas, cutn=4, seed=21, rank=0, world=1):
    """One pxr_iterate_sets on explicit per-set parameters and, on rank 0, multires_ref.iterate_sets in float64."""
    archs = CASES[case]
    g = torch.Generator().manual_seed(seed)
    sds, refs = [], []
    for i, a in enumerate(archs):
        if a.get("tower") == E.TOWER_CLIP_RESNET:
            sd = S.clip_resnet_state_dict(a, seed + 1 + i)
            refs.append(_RefResnet(sd))
        else:
            m = R.init_clip_weights(R.ClipVisual(a["image_res"], a["patch"], a["width"], a["layers"], a["heads"],
                                                 a["out_dim"]), seed + 1 + i)
            sd = m.state_dict()
            refs.append(m.double())
        sds.append(sd)
    aspect = canvas[1] / canvas[0]
    sizes, set_of = E.cutout_sets(archs[0]["image_res"], [a["image_res"] for a in archs])
    sets = []
    for k, cs in enumerate(sizes):
        T = cutouts.sample_transforms(cutn, cs, seed + 40 + k, aspect=aspect)
        facs = torch.rand(cutn, generator=g) * 0.1
        noise = torch.randn(cutn, 3, cs, cs, generator=g)
        facs[0] = facs[1] = 0.1  # unmistakable extremes: both sides route the d/dmin, d/dmax terms to one element
        noise[0, 0, 5, 7], noise[1, 2, 100, 50] = 30.0, -30.0
        sets.append(dict(cs=cs, transforms=T, facs=facs, noise=noise))
    z = torch.rand(1, 3, 12, 12, generator=g)
    prompts = [[(torch.randn(1, a["out_dim"], generator=g), 1.0, float("-inf")),
                (torch.randn(1, a["out_dim"], generator=g), -0.3, float("-inf"))] for a in archs]
    timg = torch.rand(1, 3, 30, 26, generator=g)
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=canvas, grid=(12, 12), cutn=cutn, cut_size=sizes[0], clip=archs,
                       seed=seed, noise_fac=0.1, cut_aspect=aspect, rank=rank, world=world)
    try:
        for i, sd in enumerate(sds):
            eng.load_module(E.MOD_CLIP0 + i, sd)
        eng.finalize()
        if world > 1:
            eng.init_comm()
        for i, t in enumerate(prompts):
            eng.set_prompts(i, torch.cat([p[0] for p in t]).numpy(), [p[1] for p in t], [p[2] for p in t])
        eng.set_image_prompts([timg], [0.6])
        eng.add_aux_loss(E.LOSS_SATURATION, 1.0, [1.3])
        eng.add_aux_loss(E.LOSS_PALETTE, 1.0, [0.8] + PAL)
        eng.add_aux_loss(E.LOSS_SMOOTHNESS, 1.0, [0.9, 0, 1])
        params = [dict(transforms=s_["transforms"], zoom_padding=E.PAD_BORDER, fill=0.35, noise_facs=s_["facs"].numpy(),
                       noise=s_["noise"].cuda()) for s_ in sets]
        losses = np.zeros(eng.num_losses(), dtype=np.float32)
        eng.iterate(z.clone().cuda(), 0.05, 1, params=params, losses_out=losses)
        zg = eng.debug_read("z_grad", z.shape).cpu()
        lo = rank * (cutn // world)
        batches = [eng.debug_read("batch" if k == 0 else f"set{k}.batch", (cutn // world, 3, cs, cs)).cpu()
                   for k, cs in enumerate(sizes)]
        embeds = [eng.debug_read(f"clip{i}.e", (cutn // world, a["out_dim"])).cpu() for i, a in enumerate(archs)]
    finally:
        eng.close()
    ref = None
    if rank == 0:
        d = torch.float64
        oset = [dict(cs=s_["cs"], transforms=torch.from_numpy(s_["transforms"]).to(d), noise_facs=s_["facs"].to(d),
                     noise=s_["noise"].to(d)) for s_ in sets]
        pal = np.array(PAL, dtype=np.float32).reshape(3, 3)
        aux = [(1.0, "cutouts", lambda b: R.saturation_loss(b, 1.3)),
               (1.0, "cutouts", lambda b: R.palette_loss(b.float(), pal, 0.8)[0].to(b.dtype)),
               (1.0, "cutouts", lambda b: R.smoothness_loss(b, 0.9))]
        ref = MR.iterate_sets(z.to(d), oset, list(zip(refs, set_of)),
                              [[(e.to(d), w, st) for (e, w, st) in t] for t in prompts],
                              image_prompts=[(timg.to(d), 0.6)], aux=aux, zoom_padding="border", fill=0.35, aspect=aspect,
                              synth_fn=lambda zz: R.pixel_synth(zz, canvas))
        ref["lo"] = lo
    return dict(losses=losses, zg=zg, batches=batches, embeds=embeds, lo=lo), ref


def _check(label, got, ref, cutn=4):
    n = got["batches"][0].shape[0]
    lo = got["lo"]
    for k, b in enumerate(got["batches"]):
        e = (b.double() - ref["batches"][k][lo:lo + n]).abs().max().item()
        print(f"[multires parity] {label} set {k} cutouts max_abs_err {e:.3e}")
        assert e < 1e-4
    for i, emb in enumerate(got["embeds"]):
        r = ref["embeds"][i][lo:lo + n]
        u = emb.double() / emb.double().norm(dim=-1, keepdim=True)
        e = (u - r).abs().max().item()
        print(f"[multires parity] {label} perceptor {i} embeddings max_abs_err {e:.3e}")
        assert e < 5e-3
    ref_l = np.array([float(x) for x in ref["losses"]])
    print(f"[multires parity] {label} losses engine {got['losses']} oracle {ref_l}")
    assert got["losses"].shape == ref_l.shape and np.abs(got["losses"] - ref_l).max() < 5e-3
    e_g = (got["zg"].double() - ref["z_grad"]).abs().max().item()
    m_g = ref["z_grad"].abs().max().item()
    print(f"[multires parity] {label} z.grad max_abs_err {e_g:.3e} (max |grad| {m_g:.3e})")
    assert torch.isfinite(got["zg"]).all() and e_g <= 3e-2 * m_g


@pytest.mark.parametrize("canvas", [(48, 48), (40, 64)])
@pytest.mark.parametrize("case", list(CASES))
def test_parity_with_the_multires_oracle(case, canvas):
    got, ref = run_parity(case, canvas)
    n_sets = len(got["batches"])
    assert n_sets == 2 and got["losses"].size == 2 * (2 + 1) + 3 * n_sets
    _check(f"{case} {canvas}", got, ref)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    got, ref = run_parity("rn50x4+vitb32", (40, 64), rank=rank, world=world)
    torch.save(dict(got=got, ref=ref), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_match_one(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in (0, 1))
    assert torch.equal(r0["got"]["zg"], r1["got"]["zg"]), "the replicated drawer backward must be bit-identical across ranks"
    assert np.array_equal(r0["got"]["losses"], r1["got"]["losses"])
    one, _ = run_parity("rn50x4+vitb32", (40, 64))
    e = (r0["got"]["zg"] - one["zg"]).abs().max().item()
    print(f"[multires] 2 ranks vs 1 GPU: z.grad max_abs_err {e:.3e} (max |grad| {one['zg'].abs().max():.3e})")
    assert e <= 3e-2 * one["zg"].abs().max().item()
    _check("rn50x4+vitb32 (40, 64), rank 0 of 2", r0["got"], r0["ref"])
