"""GPU parity of the auxiliary-loss options: SmoothnessLoss's pre-blur (smoothness_gaussian_kernel) and edge_order 2,
EdgeLoss's target and mask images (kernels_losses.cu: blur_axis_kernel / blur_axis_adjoint_kernel, smooth_*_kernel,
edge_kernel).  The oracle is oracle/aux_ref.py, which tests/test_aux_loss_options.py pins to vectors produced by the
real reference classes.

Isolation as in tests/test_aux_losses_gpu.py: each case runs the same inputs without and with the loss and compares the
difference of the gradient buffers with torch autograd of the oracle loss on the ENGINE's own tensor.  Bounds as
there: gradients 1e-4 of the largest entry (plus the run-to-run floor), values 1e-5 relative.
"""
import os
import socket
import types

import numpy as np
import pytest
import torch

from oracle import aux_ref as A
from oracle import ref_path as R
from pixray_b200 import engine as E
from pixray_b200 import losses as L
from test_pipeline_gpu import build, plant_extremes, random_transforms

pytestmark = pytest.mark.gpu
S = 4096.0
CUTN, CS, IMG = 8, 224, 32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G = np.load(os.path.join(GOLDEN, "aux_loss_options.npz"))
TARGET_PNG, MASK_PNG = os.path.join(GOLDEN, "edge_target.png"), os.path.join(GOLDEN, "edge_mask.png")
TYPES = ("default", "clipped", "log")
SMOOTH = sorted(k[:-4] for k in G.files if k.startswith("smooth") and k.endswith("_cfg"))
EDGE = sorted(k[:-4] for k in G.files if k.startswith("edge_") and k.endswith("_cfg"))
COLOR = [0.2, 0.6, 0.9]


def _run(eng, z, T, facs, noise):
    eng.synth(z)
    eng.make_cutouts(None, transforms=T, zoom_padding=E.PAD_REFLECTION, fill=0.4, noise_facs=facs.numpy(), noise=noise)
    eng.encode_image(0)
    eng.backward()
    return dict(g_img=eng.debug_read("g_img", (1, 3, IMG, IMG)).cpu() / S,
                g_batch=eng.debug_read("g_batch", (CUTN, 3, CS, CS)).cpu() / S,
                img=eng.debug_read("img", (1, 3, IMG, IMG)).cpu(), batch=eng.debug_read("batch", (CUTN, 3, CS, CS)).cpu(),
                losses=eng.read_losses().copy())


@pytest.fixture(scope="module")
def setup():
    vq, clip, eng, prompts, z = build(cutn=CUTN, seed=13)
    T = random_transforms(CUTN, CS, 6)
    g = torch.Generator().manual_seed(17)
    facs, noise = plant_extremes(torch.rand(CUTN, generator=g) * 0.1, torch.randn(CUTN, 3, CS, CS, generator=g))
    base = _run(eng, z, T, facs, noise)
    return dict(vq=vq, clip=clip, eng=eng, prompts=prompts, z=z, T=T, facs=facs, noise=noise, base=base)


def _smooth_args(tag):
    kind, k, s, sp, order = G[tag + "_cfg"]
    return types.SimpleNamespace(smoothness_weight=0.9, smoothness_type=TYPES[int(kind)], smoothness_gaussian_kernel=float(k),
                                 smoothness_gaussian_std=float(s), smoothness_spacing=int(sp), smoothness_edge_order=int(order))


def _smooth_oracle(args):
    return lambda x: A.smoothness_loss(x, args.smoothness_weight, args.smoothness_type, spacing=args.smoothness_spacing,
                                       edge_order=args.smoothness_edge_order, gaussian_kernel=args.smoothness_gaussian_kernel,
                                       gaussian_std=args.smoothness_gaussian_std)


def _edge_loss(tag):
    cfg = G[tag + "_cfg"]
    el = L.EdgeLoss(device="cuda")
    args = types.SimpleNamespace(edge_thickness=5, edge_margins=[int(v) for v in cfg[:4]], edge_color="[0.2+0.6+0.9]",
                                 edge_color_weight=0.1, global_color_weight=0.05,
                                 edge_input_image=TARGET_PNG if cfg[4] else "", edge_mask_image=MASK_PNG if cfg[5] else "")
    args = el.parse_settings(args)
    target, mask = el.resized((IMG, IMG))
    m = R.edge_margins_px(args.edge_margins, IMG, IMG)
    return el, args, (lambda x: A.edge_loss(x, COLOR, m, 0.1, 0.05, target=target, mask=mask))


def _check(setup, loss, args, weight, which, fn, name):
    eng, base = setup["eng"], setup["base"]
    eng.clear_aux_losses()
    loss.attach(types.SimpleNamespace(engine=eng), args, weight)
    cur = _run(eng, setup["z"], setup["T"], setup["facs"], setup["noise"])
    eng.clear_aux_losses()
    x = base[which].clone().requires_grad_(True)
    ref = weight * fn(x)
    ref.backward()
    key = "g_img" if which == "img" else "g_batch"
    delta = cur[key] - base[key]
    err, mag = (delta - x.grad).abs().max().item(), x.grad.abs().max().item()
    print(f"[aux-opt] {name}: loss engine {cur['losses'][2]:.7f} oracle {ref.item():.7f}; grad max_abs_err {err:.3e} (max {mag:.3e})")
    assert np.isfinite(cur["losses"]).all()
    assert abs(cur["losses"][2] - ref.item()) <= 1e-5 * max(1.0, abs(ref.item()))
    assert np.allclose(cur["losses"][:2], base["losses"][:2], atol=0)
    floor = 1e-5 * base[key].abs().max().item()
    assert mag > 0 and err <= 1e-4 * mag + floor


@pytest.mark.parametrize("tag", SMOOTH)
def test_smoothness_option(setup, tag):
    args = _smooth_args(tag)
    _check(setup, L.SmoothnessLoss(device="cuda"), args, 1.3, "batch", _smooth_oracle(args), tag)


@pytest.mark.parametrize("tag", EDGE)
def test_edge_option(setup, tag):
    el, args, fn = _edge_loss(tag)
    _check(setup, el, args, 2.0, "img", fn, tag)


@pytest.mark.parametrize("params,msg", [
    ([0.9, 0, 1, 3], "edge_order"),
    ([0.9, 0, 1, 1, -1], "tap count"),
    ([0.9, 0, 1, 1, 2, 0.25, 0.25, 0.25], "n \\* n taps"),
    ([0.9, 0, 1, 1, 2, 0.5, 0.0, 0.0, 0.5], "separable"),
    ([0.9, 0, 1, 1, 2, 0.25, 0.25, 0.25, float("nan")], "finite"),
    ([0.9, 0, 1, 2, 223] + [1.0 / 223 ** 2] * 223 ** 2, "at least 3"),
    ([0.9, 0, 1, 1, 224] + [1.0 / 224 ** 2] * 224 ** 2, "at least 2"),
])
def test_smoothness_refusals(setup, params, msg):
    eng = setup["eng"]
    eng.clear_aux_losses()
    with pytest.raises(E.EngineError, match=msg):
        eng.add_aux_loss(E.LOSS_SMOOTHNESS, 1.0, params)
    assert eng.num_losses() == 2


@pytest.mark.parametrize("extra,msg", [([1] + [0.5] * (3 * IMG * IMG - 1), "edge target"), ([2] + [1.0] * (IMG * IMG + 1), "edge target"),
                                       ([4], "edge mode")])
def test_edge_refusals(setup, extra, msg):
    eng = setup["eng"]
    eng.clear_aux_losses()
    with pytest.raises(E.EngineError, match=msg):
        eng.add_aux_loss(E.LOSS_EDGE, 1.0, [0.1, 0.05, 3, 3, 3, 3] + COLOR + extra)
    assert eng.num_losses() == 2


def _iterate(setup, z):
    eng = setup["eng"]
    zc = z.clone().cuda()
    losses = np.zeros(eng.num_losses(), dtype=np.float32)
    n0 = eng.num_launches()
    eng.iterate(zc, 0.05, 0, params=dict(transforms=setup["T"], zoom_padding=0, fill=0.4, noise_facs=setup["facs"].numpy(),
                                         noise=setup["noise"]), losses_out=losses)
    return eng.debug_read("z_grad", z.shape).cpu(), losses, eng.num_launches() - n0


def test_options_through_the_whole_iteration(setup):
    """pxr_iterate with a 7-tap blur + edge_order 2 smoothness and an image + mask edge loss: the loss vector and z.grad
    against the oracle's autograd of ascend_txt, and two runs bit-identical."""
    eng = setup["eng"]
    eng.clear_aux_losses()
    sargs = types.SimpleNamespace(smoothness_weight=0.9, smoothness_type="default", smoothness_gaussian_kernel=7,
                                  smoothness_gaussian_std=2.0, smoothness_spacing=1, smoothness_edge_order=2)
    session = types.SimpleNamespace(engine=eng)
    L.SmoothnessLoss(device="cuda").attach(session, sargs, 2.0)
    el, eargs, efn = _edge_loss("edge_image_mask")
    el.attach(session, eargs, 2.0)
    zg, losses, _ = _iterate(setup, setup["z"])
    zg2, losses2, _ = _iterate(setup, setup["z"])
    eng.clear_aux_losses()
    assert torch.equal(zg, zg2) and np.array_equal(losses, losses2)
    aux = [(2.0, lambda o, b, e: _smooth_oracle(sargs)(b)), (2.0, lambda o, b, e: efn(o))]
    ref = R.iterate(lambda zz: R.vqgan_synth(setup["vq"], zz), setup["z"], [setup["clip"]], [setup["prompts"]],
                    torch.from_numpy(setup["T"]), CS, "reflection", 0.4, setup["facs"], setup["noise"], aux=aux)
    ref_l = np.array([float(l) for l in ref["losses"]], dtype=np.float32)
    print("[aux-opt] losses engine", losses, "\n          oracle", ref_l)
    assert losses.shape == ref_l.shape == (4,)
    assert np.abs(losses - ref_l).max() < 5e-3
    err, mag = (zg - ref["z_grad"]).abs().max().item(), ref["z_grad"].abs().max().item()
    print(f"[aux-opt] z.grad: max_abs_err {err:.3e} (max {mag:.3e})")
    assert err <= 3e-2 * mag


def test_default_options_keep_the_launch_list_and_values(setup):
    """The defaults (kernel 0, edge_order 1, no images) issue the launches the 3- and 9-value calls always issued, and the
    explicit long forms of the same settings give bit-identical values."""
    eng = setup["eng"]
    eng.clear_aux_losses()
    _, _, n_none = _iterate(setup, setup["z"])
    runs = []
    for sp, ep in [([0.9, 0, 1], [0.1, 0.05, 3, 6, 4, 0] + COLOR), ([0.9, 0, 1, 1, 0], [0.1, 0.05, 3, 6, 4, 0] + COLOR + [0])]:
        eng.clear_aux_losses()
        eng.add_aux_loss(E.LOSS_SMOOTHNESS, 1.0, sp)
        eng.add_aux_loss(E.LOSS_EDGE, 1.0, ep)
        runs.append(_iterate(setup, setup["z"]))
    eng.clear_aux_losses()
    assert runs[0][2] == n_none + 3 + 2 == runs[1][2]  # smoothness: sharp + final + grad; edge: kernel + final
    assert np.array_equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][0], runs[1][0])
    # the product's defaults take the short form
    d = L.SmoothnessLoss(device="cuda").engine_params(types.SimpleNamespace(
        smoothness_weight=0.9, smoothness_type="default", smoothness_gaussian_kernel=0, smoothness_gaussian_std=1,
        smoothness_spacing=1, smoothness_edge_order=1), None)
    assert d == [0.9, 0, 1]


# ---- two ranks over NCCL (the spawn pattern of tests/test_multigpu.py)
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from test_pipeline_gpu import SMALL_CLIP, SMALL_VQ
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    cutn, cs, seed = 8, 224, 21
    vq = R.init_vqgan_weights(R.VQModel(n_embed=1024, embed_dim=128, ch=128, ch_mult=(1, 2), num_res_blocks=1,
                                        attn_resolutions=(16,), resolution=32, z_channels=128), seed)
    clip = R.init_clip_weights(R.ClipVisual(224, 32, 128, 2, 2, 64), seed + 1)
    eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=(32, 32), vqgan=SMALL_VQ, cutn=cutn, clip=[SMALL_CLIP], seed=seed,
                       device=rank, rank=rank, world=world)
    eng.load_module(E.MOD_VQGAN, vq.state_dict())
    eng.load_module(E.MOD_CLIP0, clip.state_dict())
    eng.finalize()
    eng.init_comm()
    g = torch.Generator().manual_seed(seed + 2)
    prompts = [(torch.randn(1, 64, generator=g), 1.0, float("-inf")), (torch.randn(1, 64, generator=g), -0.3, float("-inf"))]
    eng.set_prompts(0, torch.cat([p[0] for p in prompts]).numpy(), [1.0, -0.3], [float("-inf")] * 2)
    idx = torch.randint(1024, (256,), generator=g)
    z = (vq.quantize.embedding.weight[idx].T.reshape(1, 128, 16, 16) + 0.05 * torch.randn(1, 128, 16, 16, generator=g)).contiguous()
    T = random_transforms(cutn, cs, 3)
    facs, noise = plant_extremes(torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g))
    sargs = types.SimpleNamespace(smoothness_weight=0.9, smoothness_type="log", smoothness_gaussian_kernel=5,
                                  smoothness_gaussian_std=1.5, smoothness_spacing=1, smoothness_edge_order=2)
    L.SmoothnessLoss(device="cuda").attach(types.SimpleNamespace(engine=eng), sargs, 2.0)
    zc = z.clone().cuda()
    losses = np.zeros(3, dtype=np.float32)
    eng.iterate(zc, 0.05, 0, params=dict(transforms=T, zoom_padding=0, fill=0.4, noise_facs=facs.numpy(), noise=noise),
                losses_out=losses)
    zg = eng.debug_read("z_grad", z.shape).cpu()
    torch.save(dict(zg=zg, losses=losses.copy(), z=zc.cpu()), os.path.join(out_dir, f"rank{rank}.pt"))
    if rank == 0:
        ref = R.iterate(lambda zz: R.vqgan_synth(vq, zz), z, [clip], [prompts], torch.from_numpy(T), cs, "reflection", 0.4,
                        facs, noise, aux=[(2.0, lambda o, b, e: _smooth_oracle(sargs)(b))])
        torch.save(dict(zg=ref["z_grad"], losses=torch.stack([l.reshape(()) for l in ref["losses"]])),
                   os.path.join(out_dir, "ref.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_blurred_smoothness_two_ranks(tmp_path):
    """The halo exchange carries the neighbours' BLURRED boundary rows: z.grad as on one GPU, ranks bit-identical."""
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1, ref = (torch.load(tmp_path / n, weights_only=False) for n in ("rank0.pt", "rank1.pt", "ref.pt"))
    assert torch.equal(r0["zg"], r1["zg"]) and torch.equal(r0["z"], r1["z"])
    assert np.array_equal(r0["losses"], r1["losses"])
    err, mag = (r0["zg"] - ref["zg"]).abs().max().item(), ref["zg"].abs().max().item()
    print(f"[aux-opt] 2-rank blurred smoothness z.grad: max_abs_err={err:.3e} ref_max={mag:.3e}")
    assert err <= 3e-2 * mag
    assert np.abs(r0["losses"] - ref["losses"].numpy()).max() < 5e-3
