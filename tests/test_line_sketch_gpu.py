"""The line-sketch drawer (PXR_DRAWER_STROKES) on the GPU: the rasteriser's winners and image against the float64 oracle
(oracle/stroke_ref.py) at the engine's own sample positions, the boundary backward against the oracle on the engine's
own chords, one whole iteration against the oracle pipeline, bit-identical repeats, the three-rate Adam + width clamp
against three torch.optim.Adam + clip_z, managed and host runs of api.run, and two ranks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import ref_path as R
from oracle import stroke_ref as SR
from pixray_b200 import _lib
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import plugins as P
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def hook_samples(seed, it, H, W):
    lib = _lib.load()
    f = lib.pxr_test_raster_samples
    f.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p]
    out = torch.empty(H, W, 4, 2, device="cuda")
    assert f(seed, it, H, W, out.data_ptr()) == 0
    return out.cpu().numpy()


def build(W, H, N, L, max_width, paper=False, seed=5, clip_sd=None, cutn=8, rank=0, world=1):
    from test_pipeline_gpu import SMALL_CLIP
    eng = E.B200Engine(drawer=E.DRAWER_STROKES, image_hw=(H, W), strokes=(N, L, max_width, paper), cutn=cutn,
                       clip=[SMALL_CLIP], seed=seed, device=rank, rank=rank, world=world)
    eng.load_module(E.MOD_CLIP0, clip_sd if clip_sd is not None else S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    return eng


def scene_z(W, H, N, L, max_width, seed, paper=P.PAPER_RGBA, off_canvas=False):
    """Start points as the drawer draws them, widths spread over [1, max_width], the given paper RGBA."""
    import random
    rng = random.Random(seed)
    pts = P.line_start_points(W, H, N, L, rng=rng)
    if off_canvas:
        pts[0, :, 0] += 0.6 * W  # the first path runs off the right edge
    g = torch.Generator().manual_seed(seed)
    widths = 1 + torch.rand(N, generator=g) * (max_width - 1)
    return torch.cat([pts.reshape(-1), widths, torch.tensor(paper, dtype=torch.float32)]).contiguous()


@pytest.mark.parametrize("case", [(384, 216, 24, 8, 4.32, P.PAPER_RGBA, False),
                                  (96, 64, 6, 3, 3.0, (0.9, 0.3, 0.5, 0.7), True)], ids=["384x216", "96x64_paper"])
def test_forward_matches_the_oracle_at_the_engines_samples(case):
    W, H, N, L, mw, paper, off = case
    eng = build(W, H, N, L, mw, paper=True, seed=11)
    z = scene_z(W, H, N, L, mw, 2, paper, off)
    eng.set_synth_iteration(3)
    img = eng.synth(z)[0].cpu().double()
    win = eng.debug_read("stroke_winner", (4, H, W), dtype=torch.int32).cpu().numpy()
    caps = eng.debug_read("stroke_caps", (N * L * SR.S, 4)).cpu().numpy()
    sc = SR.Scene(z.numpy(), N, L, H, W, caps)
    ref_win, dist = sc.winners(hook_samples(11, 3, H, W), edge_distance=True)
    near = dist <= 1e-4
    flat = np.abs(caps - SR.flatten(sc.points)).max()
    print(f"[parity] strokes {W}x{H}: {N}x{L} paths, {int(near.sum())} of {near.size} samples within 1e-4 px of an "
          f"outline excluded, {int((win >= 0).sum())} covered; fp32 chords vs float64 flattening {flat:.2e} px")
    assert flat < 1e-3
    assert np.array_equal(win[~near], ref_win[~near])
    ref = SR.composite(SR.coverage(ref_win), sc.paper)
    clean = torch.as_tensor(~near.any(axis=0))
    assert (img - ref).abs()[:, clean].max().item() <= 1e-6
    assert torch.equal(eng.synth(z)[0].cpu().double(), img)


def _iteration_case(paper):
    from test_pipeline_gpu import SMALL_CLIP, plant_extremes, random_transforms
    W, H, N, L, mw, cutn, cs, seed, it = 64, 48, 5, 2, 3.0, 8, 224, 4, 1
    clip = R.init_clip_weights(R.ClipVisual(224, SMALL_CLIP["patch"], SMALL_CLIP["width"], SMALL_CLIP["layers"],
                                            SMALL_CLIP["heads"], SMALL_CLIP["out_dim"]), seed + 1)
    eng = build(W, H, N, L, mw, paper=paper, seed=seed, clip_sd=clip.state_dict(), cutn=cutn)
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, 64, generator=g), 1.0, float("-inf")), (torch.randn(1, 64, generator=g), -0.3, float("-inf"))]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    z = scene_z(W, H, N, L, mw, 7, (0.95, 0.9, 0.8, 0.85) if paper else P.PAPER_RGBA)
    T = random_transforms(cutn, cs, 3 + seed)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    params = dict(transforms=T, zoom_padding=E.PAD_BORDER, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    return locals()


@pytest.mark.parametrize("paper", [False, True], ids=["paper_fixed", "paper_trainable"])
def test_backward_and_one_iteration_match_the_oracle(paper):
    """The backward alone against the float64 oracle on the engine's chords, winners and image gradient: measured on an
    H100, max-abs error 1.3e-3 of max|grad| for the points (tolerance 3e-3); then the whole iteration (3e-2)."""
    from test_pipeline_gpu import report
    c = _iteration_case(paper)
    eng, z, W, H, N, L, it, seed = c["eng"], c["z"], c["W"], c["H"], c["N"], c["L"], c["it"], c["seed"]

    def run():
        zc = z.clone().cuda()
        losses = np.zeros(2, dtype=np.float32)
        eng.reset_optimizer()
        eng.iterate(zc, 1.0, it, params=c["params"], losses_out=losses)
        return (zc.cpu(), losses, eng.debug_read("z_grad", z.shape).cpu(), eng.debug_read("g_img", (3, H, W)).cpu(),
                eng.debug_read("stroke_winner", (4, H, W), dtype=torch.int32).cpu().numpy(),
                eng.debug_read("stroke_caps", (N * L * SR.S, 4)).cpu().numpy())

    zc, losses, zg, g_img, win, caps = run()
    n_pts, n_w, _ = E.stroke_z_layout(N, L)
    # the backward alone, on the engine's chords, winners and image gradient (default grad scale 4096)
    ref_g = torch.from_numpy(SR.gradient(z.numpy(), N, L, H, W, win, g_img.double().numpy() / 4096.0, paper, caps))
    for name, sl in (("points", slice(0, n_pts)), ("widths", slice(n_pts, n_pts + n_w)), ("paper", slice(n_pts + n_w, None))):
        e, m = report(f"strokes backward {name}", zg[sl], ref_g[sl].float())
        if name == "paper" and not paper:
            assert torch.all(zg[sl] == 0)
        else:
            assert m > 0 and e <= 3e-3 * m
    # the whole iteration against the oracle pipeline over the float64 render at the engine's samples
    meta = (N, L, H, W, hook_samples(seed, it, H, W), paper)
    ref = R.iterate(lambda zz: SR.StrokeRender.apply(zz, meta)[None].float(), z, [c["clip"]], [c["prompts"]],
                    torch.from_numpy(c["T"]), c["cs"], "border", 0.4, c["facs"], c["noise"])
    ref_l = np.array([float(l) for l in ref["losses"]], dtype=np.float32)
    assert np.abs(losses - ref_l).max() < 5e-3
    e_g, m_g = report("strokes z.grad (whole iteration)", zg, ref["z_grad"])
    assert e_g <= 3e-2 * m_g
    # bit-identical repeats
    zc2, _, zg2, g_img2, win2, _ = run()
    assert torch.equal(g_img2, g_img) and torch.equal(zg2, zg) and torch.equal(zc2, zc) and np.array_equal(win2, win)


def test_three_rate_adam_and_width_clamp_match_torch():
    """pxr_step on given gradients, several steps and a drop, against the reference's three torch.optim.Adam + clip_z."""
    W, H, N, L, mw = 64, 48, 4, 2, 3.0
    eng = build(W, H, N, L, mw, paper=True)
    n_pts, n_w, _ = E.stroke_z_layout(N, L)
    z = scene_z(W, H, N, L, mw, 3, (0.9, 0.8, 0.7, 1.0))
    ref = z.clone().double()
    parts = [ref[:n_pts].clone().requires_grad_(True), ref[n_pts:n_pts + n_w].clone().requires_grad_(True),
             ref[n_pts + n_w:].clone().requires_grad_(True)]
    g = torch.Generator().manual_seed(9)
    zc = z.clone().cuda()
    eng.synth(zc)  # loads z into the engine
    eng.reset_optimizer()
    div = 1
    opts = [torch.optim.Adam([p], lr=r / div) for p, r in zip(parts, (1.0, 0.1, 0.01))]
    for step in range(8):
        if step == 4:  # a drop: fresh optimisers at a tenth of the rates
            div = 10
            eng.reset_optimizer()
            opts = [torch.optim.Adam([p], lr=r / div) for p, r in zip(parts, (1.0, 0.1, 0.01))]
        grad = torch.randn(z.numel(), generator=g) * 3
        eng.set_z_grad(grad.cuda())
        eng.step(zc, 1.0 / div, step)
        for p, sl in zip(parts, (slice(0, n_pts), slice(n_pts, n_pts + n_w), slice(n_pts + n_w, None))):
            p.grad = grad[sl].double()
        for o in opts:
            o.step()
        with torch.no_grad():
            parts[1].clamp_(1.0, mw)
    want = torch.cat([p.detach() for p in parts])
    got = zc.cpu().double()
    err = ((got - want).abs() / want.abs().clamp_min(1.0)).max().item()
    print(f"[parity] three-rate Adam + width clamp after 8 steps and a drop: max rel err {err:.3e}")
    assert err <= 1e-6
    assert float(got[n_pts:n_pts + n_w].min()) >= 1.0 and float(got[n_pts:n_pts + n_w].max()) <= mw


def _settings(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(prompts="a line drawing", drawer="line_sketch", size=[96, 64], strokes=6, stroke_length=3,
                clip_models="ViT-B/32", num_cuts=4, outdir="", seed="3", b200_allow_synthetic=True, vector_prompts="none")
    base.update(kw)
    return base


def test_managed_and_host_runs_make_the_same_decisions(tmp_path):
    out = {}
    for managed in (True, False):
        api.run(**_settings(tmp_path, iterations=40, learning_rate_drops=[20, 60], auto_stop=True,
                            allow_paper_color=True, b200_device_checkdrop=managed))
        st = api._state
        z = st.drawer.get_z().cpu()
        n_pts, n_w, _ = E.stroke_z_layout(6, 3)
        assert float(z[n_pts:n_pts + n_w].min()) >= 1.0 and float(z[n_pts:n_pts + n_w].max()) <= 0.02 * 64 + 1e-6
        assert st.drawer.to_image().size == (96, 64)
        out[managed] = (st.cur_iteration, st.num_loss_drop, round(float(st.lr), 6), st.best_iter)
        print(f"[parity] line_sketch api.run managed={managed}: iteration {st.cur_iteration}, drops {st.num_loss_drop}, "
              f"lr {st.lr}, best_iter {st.best_iter}")
    assert out[True] == out[False]


def test_checkpoint_continues_bit_identically(tmp_path):
    def start():
        api.reset_settings()
        api.add_settings(**_settings(tmp_path, iterations=8, allow_paper_color=True))
        args = api.apply_settings()
        api.do_init(args)
        return args

    args = start()
    for it in range(4):
        api.train(args, it)
        api._state.cur_iteration = it + 1
    api.save_checkpoint(tmp_path / "ck.bin")
    for it in range(4, 8):
        api.train(args, it)
    api._state.engine.sync()
    z_a = api._state.drawer.get_z().cpu().clone()
    args = start()
    assert api.load_checkpoint(tmp_path / "ck.bin") == 4
    for it in range(4, 8):
        api.train(args, it)
    api._state.engine.sync()
    assert torch.equal(api._state.drawer.get_z().cpu(), z_a)


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    c = _iteration_case(True)
    eng = build(c["W"], c["H"], c["N"], c["L"], c["mw"], paper=True, seed=c["seed"], clip_sd=c["clip"].state_dict(),
                cutn=c["cutn"], rank=rank, world=world)
    eng.init_comm()
    eng.set_prompts(0, torch.cat([p[0] for p in c["prompts"]]).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    zc = c["z"].clone().cuda(rank)
    eng.iterate(zc, 1.0, c["it"], params=c["params"], losses_out=np.zeros(2, dtype=np.float32))
    torch.save(dict(zg=eng.debug_read("z_grad", c["z"].shape).cpu(), z=zc.cpu()), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_are_bit_identical(tmp_path):
    import torch.multiprocessing as mp
    from test_multigpu import _free_port
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / n, weights_only=False) for n in ("rank0.pt", "rank1.pt"))
    assert torch.equal(r0["zg"], r1["zg"]) and torch.equal(r0["z"], r1["z"])
