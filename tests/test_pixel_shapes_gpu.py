"""The polygon drawer (PXR_DRAWER_POLYGON: PixelDrawer's hex / tri / diamond / knit / rectshift cells) on the GPU: the
sample positions, the rasteriser's winners and image against the float64 oracle (oracle/polygon_ref.py) at those same
positions, the gather backward against float64 autograd, one whole iteration against the oracle pipeline, the round
trips (checkpoint, api.run in managed and host mode, two ranks), polygons far off the canvas, and the session features
that work on any drawer's z / image (filters, image prompts, spot prompts, the init_weight family on [n, 4])."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import polygon_ref as PR
from oracle import ref_path as R
from pixray_b200 import _lib
from pixray_b200 import api
from pixray_b200 import engine as E
from pixray_b200 import pixel_shapes as PS
from pixray_b200 import synthetic as S

pytestmark = pytest.mark.gpu

TYPES = ("rect", "rectshift", "hex", "tri", "diamond", "knit")


def hook_samples(seed, it, H, W):
    lib = _lib.load()
    f = lib.pxr_test_raster_samples
    f.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p]
    out = torch.empty(H, W, 4, 2, device="cuda")
    assert f(seed, it, H, W, out.data_ptr()) == 0
    return out.cpu().numpy()


def build(pixel_type, W, H, seed=5, clip_sd=None, cutn=8, **grid_kw):
    from test_pipeline_gpu import SMALL_CLIP
    rows, cols = PS.grid_for((W, H), pixel_type, verbose=False, **grid_kw)
    xy, off = PS.polygons((W, H), rows, cols, pixel_type)
    eng = E.B200Engine(drawer=E.DRAWER_POLYGON, image_hw=(H, W), polygons=(xy, off), cutn=cutn, clip=[SMALL_CLIP],
                       seed=seed)
    eng.load_module(E.MOD_CLIP0, clip_sd if clip_sd is not None else S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    return eng, xy, off


def colours(n, seed, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    z = torch.ones(n, 4)
    z[:, :3] = torch.rand(n, 3, generator=g) * (hi - lo) + lo
    return z.contiguous()


def test_sample_positions_are_stratified_jittered_and_keyed_by_iteration():
    H = W = 256
    s0, s0b, s1 = hook_samples(7, 0, H, W), hook_samples(7, 0, H, W), hook_samples(7, 1, H, W)
    assert np.array_equal(s0, s0b)                                     # same (seed, iteration): same positions
    assert np.mean(s0 != s1) > 0.999                                   # the next iteration draws new ones
    assert np.mean(s0 != hook_samples(8, 0, H, W)) > 0.999             # so does another seed
    px = np.arange(W, dtype=np.float64)[None, :, None]
    py = np.arange(H, dtype=np.float64)[:, None, None]
    ox, oy = s0[..., 0] - px, s0[..., 1] - py                          # [H, W, 4] offsets inside the pixel
    dx, dy = np.array([0, 1, 0, 1]) / 2.0, np.array([0, 0, 1, 1]) / 2.0
    # sample s lies in its stratum [dx/2, (dx+1)/2] x [dy/2, (dy+1)/2] (the upper edge only through fp32 rounding)
    assert np.all(ox >= dx) and np.all(ox <= dx + 0.5) and np.all(oy >= dy) and np.all(oy <= dy + 0.5)
    for o in (ox, oy):
        m, sigma = o.mean(), o.std() / np.sqrt(o.size)
        print(f"[parity] raster sample offset mean {m:.6f} (sigma {sigma:.2e})")
        assert abs(m - 0.5) <= 5 * sigma


@pytest.mark.parametrize("pixel_type", TYPES)
@pytest.mark.parametrize("canvas", [(77, 53, dict(pixel_scale=4.0)), (384, 216, {})], ids=["77x53", "384x216"])
def test_forward_matches_the_oracle_at_the_engines_samples(pixel_type, canvas):
    W, H, grid_kw = canvas
    eng, xy, off = build(pixel_type, W, H, seed=11, **grid_kw)
    n = len(off) - 1
    z = colours(n, 3)
    eng.set_synth_iteration(3)
    img = eng.synth(z)[0].cpu().double()
    win = eng.debug_read("poly_winner", (4, H, W), dtype=torch.int32).cpu().numpy()
    ref_win, dist = PR.polygon_winners(xy, off, H, W, hook_samples(11, 3, H, W), edge_distance=True)
    near = dist <= 1e-4
    print(f"[parity] {pixel_type} {W}x{H}: {n} polygons, {int(near.sum())} of {near.size} samples within 1e-4 px of an "
          f"edge excluded, {int((win == -1).sum())} uncovered")
    assert np.array_equal(win[~near], ref_win[~near])
    ref = PR.polygon_render(xy, off, z, H, W, None, winners=ref_win)
    clean = torch.as_tensor(~near.any(axis=0))
    assert (img - ref).abs()[:, clean].max().item() <= 1e-6
    # the same image again: the render is a pure function of (z, seed, iteration)
    assert torch.equal(eng.synth(z)[0].cpu().double(), img)


@pytest.mark.parametrize("pixel_type", TYPES)
def test_one_iteration_matches_the_oracle(pixel_type):
    """As test_pixel_drawer_matches_the_oracle: one whole iteration on explicit cutout parameters against R.iterate over
    the float64 rasteriser at the engine's samples; the gather backward against float64 autograd on the engine's own
    image gradient; Adam + clip_z (RGB to [0, 1], alpha to 1); bit-identical repeats."""
    from test_pipeline_gpu import SMALL_CLIP, plant_extremes, random_transforms, report
    W, H, cutn, cs, seed, it = 64, 48, 8, 224, 4, 1
    clip = R.init_clip_weights(R.ClipVisual(224, SMALL_CLIP["patch"], SMALL_CLIP["width"], SMALL_CLIP["layers"],
                                            SMALL_CLIP["heads"], SMALL_CLIP["out_dim"]), seed + 1)
    eng, xy, off = build(pixel_type, W, H, seed=seed, clip_sd=clip.state_dict(), cutn=cutn, pixel_scale=4.0)
    n = len(off) - 1
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, 64, generator=g), 1.0, float("-inf")), (torch.randn(1, 64, generator=g), -0.3, float("-inf"))]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    z = colours(n, seed, -0.2, 1.2)                                    # some colours outside [0, 1]
    T = random_transforms(cutn, cs, 3 + seed)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    params = dict(transforms=T, zoom_padding=E.PAD_BORDER, fill=0.4, noise_facs=facs.numpy(), noise=noise)

    def run():
        zc = z.clone().cuda()
        losses = np.zeros(2, dtype=np.float32)
        eng.reset_optimizer()
        eng.iterate(zc, 0.03, it, params=params, losses_out=losses)
        return (zc.cpu(), losses, eng.debug_read("z_grad", (n, 4)).cpu(), eng.debug_read("g_img", (3, H, W)).cpu(),
                eng.debug_read("poly_winner", (4, H, W), dtype=torch.int32).cpu().numpy())

    zc, losses, zg, g_img, win = run()
    ref_win = PR.polygon_winners(xy, off, H, W, hook_samples(seed, it, H, W))
    ref = R.iterate(lambda zz: PR.polygon_render(xy, off, zz, H, W, None, winners=ref_win)[None].float(), z, [clip],
                    [prompts], torch.from_numpy(T), cs, "border", 0.4, facs, noise)
    ref_l = np.array([float(l) for l in ref["losses"]], dtype=np.float32)
    assert np.abs(losses - ref_l).max() < 5e-3
    e_g, m_g = report(f"{pixel_type} z.grad", zg, ref["z_grad"])
    assert e_g <= 3e-2 * m_g
    assert torch.all(zg[:, 3] == 0)                                    # alpha gets no gradient
    # the backward alone: float64 autograd of <render(z), g_img> with the engine's winners and image gradient
    gi = g_img.double() / 4096.0                                       # the engine's default grad scale
    c = z.double().requires_grad_(True)
    (PR.polygon_render(xy, off, c, H, W, None, winners=win) * gi).sum().backward()
    ca = z.double().requires_grad_(True)
    (PR.polygon_render(xy, off, ca, H, W, None, winners=win) * gi.abs()).sum().backward()  # 0.25 sum |g| per polygon
    err = (zg.double() - c.grad)[:, :3].abs()
    assert torch.all(err <= 1e-5 * ca.grad[:, :3] + 1e-30), float((err / (ca.grad[:, :3] + 1e-30)).max())
    # Adam + clip_z on the engine's own gradient
    z_next = R.AdamState(z).step(z, zg, 0.03)
    z_next[:, :3] = z_next[:, :3].clamp(0, 1)
    z_next[:, 3] = 1.0
    e_z, _ = report(f"{pixel_type} z after Adam + clip_z", zc, z_next)
    assert e_z < 2e-5 and torch.all(zc[:, 3] == 1.0)
    zc2, _, zg2, g_img2, _ = run()
    assert torch.equal(g_img2, g_img) and torch.equal(zg2, zg) and torch.equal(zc2, zc)


def _settings(tmp_path, **kw):
    (tmp_path / "vectors").mkdir(exist_ok=True)
    (tmp_path / "vectors" / "textoff.json").write_text('{"ViT-B/32": [[0.2]]}')
    os.environ["PIXRAY_ROOT"] = str(tmp_path)
    base = dict(prompts="a red hexagon", drawer="pixel", pixel_type="hex", size=[64, 48], clip_models="ViT-B/32",
                num_cuts=4, outdir="", seed="3", b200_allow_synthetic=True, vector_prompts="none")
    base.update(kw)
    return base


@pytest.mark.parametrize("managed", [True, False], ids=["managed", "host"])
def test_api_run_completes_on_the_engine(tmp_path, managed):
    api.run(**_settings(tmp_path, iterations=4, b200_device_checkdrop=managed))
    st = api._state
    assert isinstance(st.drawer, api.P.PixelDrawer) and st.engine.z_shape[1] == 4
    z = st.drawer.get_z().cpu()
    assert torch.all(z[:, 3] == 1.0) and float(z[:, :3].min()) >= 0.0 and float(z[:, :3].max()) <= 1.0
    # the default learning_rate_drops=[75] drops once, after iteration 2: the drawer's 0.03 divided by 10
    assert st.cur_iteration == 4 and api.get_image() is not None and st.lr == pytest.approx(0.003)
    assert st.drawer.to_image().size == (64, 48)


def test_checkpoint_continues_bit_identically(tmp_path):
    def start():
        api.reset_settings()
        api.add_settings(**_settings(tmp_path, iterations=8))
        args = api.apply_settings()
        api.do_init(args)
        return args

    args = start()
    for it in range(3):
        api.train(args, it)
        api._state.cur_iteration = it + 1
    path = str(tmp_path / "ckpt.bin")
    api.save_checkpoint(path)
    for it in range(3, 6):
        api.train(args, it)
    api._state.engine.sync()
    z_a = api._state.drawer.get_z().cpu().clone()
    args = start()
    assert api.load_checkpoint(path) == 3
    for it in range(3, 6):
        api.train(args, it)
    api._state.engine.sync()
    assert torch.equal(api._state.drawer.get_z().cpu(), z_a)


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from test_pipeline_gpu import SMALL_CLIP
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    rows, cols = PS.grid_for((64, 48), "hex", pixel_scale=4.0, verbose=False)
    xy, off = PS.polygons((64, 48), rows, cols, "hex")
    eng = E.B200Engine(drawer=E.DRAWER_POLYGON, image_hw=(48, 64), polygons=(xy, off), cutn=8, clip=[SMALL_CLIP], seed=9,
                       device=rank, rank=rank, world=world)
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    eng.finalize()
    eng.init_comm()
    g = torch.Generator().manual_seed(2)
    eng.set_prompts(0, torch.randn(2, 64, generator=g).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    zc = colours(len(off) - 1, 5).cuda()
    for it in range(3):
        eng.iterate(zc, 0.03, it)
    eng.sync()
    torch.save(dict(z=zc.cpu(), zg=eng.debug_read("z_grad", (len(off) - 1, 4)).cpu()), os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_keep_identical_colours(tmp_path):
    import torch.multiprocessing as mp
    from test_multigpu import _free_port
    mp.spawn(_rank_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in (0, 1))
    assert torch.equal(r0["zg"], r1["zg"]) and torch.equal(r0["z"], r1["z"])


def test_polygons_far_off_the_canvas_never_win():
    """Finite coordinates far outside the canvas are accepted: a polygon entirely off the canvas gets no tiles and never
    covers a sample, and one spanning +-1e30 is drawn over the canvas where it crosses it.  Everything else renders as
    without them, and the backward stays finite."""
    from test_pipeline_gpu import SMALL_CLIP
    W, H = 64, 48
    rows, cols = PS.grid_for((W, H), "hex", pixel_scale=4.0, verbose=False)
    xy, off = PS.polygons((W, H), rows, cols, "hex")
    far = np.array([[1e30, 1e30], [2e30, 1e30], [1e30, 2e30], [-1e30, -1e30], [-2e30, -1e30], [-1e30, -2e30],
                    [-1e30, 10.0], [1e30, 10.0], [1e30, 20.0]], dtype=np.float32)
    xy2 = np.concatenate([xy, far])
    off2 = np.concatenate([off, off[-1] + np.array([3, 6, 9])]).astype(np.int32)
    n0 = len(off) - 1
    out = []
    for pts, offs in ((xy, off), (xy2, off2)):
        eng = E.B200Engine(drawer=E.DRAWER_POLYGON, image_hw=(H, W), polygons=(pts, offs), cutn=8, clip=[SMALL_CLIP], seed=2)
        eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
        eng.finalize()
        eng.set_prompts(0, torch.randn(1, 64, generator=torch.Generator().manual_seed(1)).numpy(), [1.0], [float("-inf")])
        z = colours(len(offs) - 1, 1)
        eng.set_synth_iteration(0)
        img = eng.synth(z)[0].cpu()
        win = eng.debug_read("poly_winner", (4, H, W), dtype=torch.int32).cpu()
        zc = z.clone().cuda()
        eng.iterate(zc, 0.03, 0)
        out.append((img, win, eng.debug_read("z_grad", tuple(eng.z_shape)).cpu()))
    (img0, win0, _), (img1, win1, zg1) = out
    assert not bool(((win1 == n0) | (win1 == n0 + 1)).any())
    assert float(zg1[n0:n0 + 2].abs().max()) == 0.0 and bool(torch.isfinite(zg1).all())
    covered = (win1 == n0 + 2).any(dim=0)
    assert bool(covered.any()) and not bool(covered.all())
    assert torch.equal(win1[:, ~covered], win0[:, ~covered])
    assert torch.equal(img1[:, ~covered], img0[:, ~covered])


def _run_feature(tmp_path, **kw):
    api.reset_settings()
    api.add_settings(**_settings(tmp_path, iterations=6, **kw))
    args = api.apply_settings()
    api.do_init(args)
    z0 = api._state.drawer.get_z_copy().cpu()
    api.do_run(args)
    st = api._state
    st.engine.sync()
    z = st.drawer.get_z().cpu()
    assert st.cur_iteration == 6 and st.losses is not None and np.all(np.isfinite(st.losses))
    assert torch.all(z[:, 3] == 1.0) and float(z[:, :3].min()) >= 0.0 and float(z[:, :3].max()) <= 1.0
    assert not torch.equal(z, z0)
    return st


def test_filters_run_on_the_polygon_drawer(tmp_path):
    st = _run_feature(tmp_path, filters="tiler:0.5,wallpaper", wallpaper_type="shift")
    assert st.engine.num_losses() == len(st.losses) == 3              # two filters, one prompt


def test_image_prompts_run_on_the_polygon_drawer(tmp_path):
    st = _run_feature(tmp_path, image_prompts=[torch.rand(1, 3, 40, 30, generator=torch.Generator().manual_seed(1))])
    assert st.engine.num_losses() == len(st.losses) == 2              # prompt, image prompt


def test_spot_prompts_run_on_the_polygon_drawer(tmp_path):
    mask = np.zeros((224, 224), dtype=bool)
    mask[50:150, 60:170] = True
    st = _run_feature(tmp_path, spot_prompts="a spot", spot_prompts_off="no spot", spot_file=mask)
    assert st.engine.num_losses() == len(st.losses) == 3              # spot, spot off, prompt


def test_init_weight_family_runs_on_the_polygon_drawer(tmp_path):
    from PIL import Image
    rgb = (np.random.default_rng(4).random((48, 64, 3)) * 255).astype(np.uint8)
    Image.fromarray(rgb).save(tmp_path / "init.png")
    st = _run_feature(tmp_path, init_image=str(tmp_path / "init.png"), init_weight=0.5, init_weight_dist=0.3,
                      init_weight_cos=0.2, init_weight_pix=0.4)
    assert st.engine.num_losses() == len(st.losses) == 5              # prompt, four anchors
    assert tuple(st.z_orig.shape) == st.engine.z_shape


def test_latent_anchor_gradient_on_the_rgba_colours():
    """init_weight_dist on z = [n, 4]: the anchor adds weight * (z - z_orig) / numel to z.grad after the raster backward,
    over all four columns, and reports weight / 2 * mean((z - z_orig)^2)."""
    from test_pipeline_gpu import plant_extremes, random_transforms
    W, H, cutn, cs = 64, 48, 8, 224
    eng, xy, off = build("knit", W, H, seed=6, cutn=cutn, pixel_scale=4.0)
    n = len(off) - 1
    g = torch.Generator().manual_seed(8)
    eng.set_prompts(0, torch.randn(1, 64, generator=g).numpy(), [1.0], [float("-inf")])
    z, ref = colours(n, 2), colours(n, 3)
    T = random_transforms(cutn, cs, 5)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    params = dict(transforms=T, zoom_padding=E.PAD_BORDER, fill=0.4, noise_facs=facs.numpy(), noise=noise)

    def grad(n_losses):
        eng.reset_optimizer()
        losses = np.zeros(n_losses, dtype=np.float32)
        eng.iterate(z.clone().cuda(), 0.03, 2, params=params, losses_out=losses)
        return eng.debug_read("z_grad", (n, 4)).cpu(), losses

    g0, l0 = grad(1)
    w = 0.7
    eng.add_anchor(E.ANCHOR_MSE, w, ref)
    g1, l1 = grad(2)
    want = w * (z - ref) / z.numel()
    assert (g1 - g0 - want).abs().max().item() <= 1e-6 * want.abs().max().item() + 1e-9
    # the prompt loss is unchanged
    assert abs(float(l1[0]) - float(l0[0])) <= 1e-6 * abs(float(l0[0]))
    assert abs(float(l1[1]) - w / 2 * float(((z.double() - ref.double()) ** 2).mean())) <= 1e-6
