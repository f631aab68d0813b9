"""CPU: the auxiliary-loss options SmoothnessLoss pre-blur / edge_order 2 and EdgeLoss target / mask images.

- oracle/aux_ref.py reproduces tests/golden/aux_loss_options.npz (the unmodified reference classes' values and autograd
  gradients, oracle/make_golden_aux_options.py);
- pixray_b200.losses turns the settings into the engine's parameters: the reference's blur taps, and the reference's
  resized target and mask bit for bit from the golden PNGs; URLs and invalid values are refused;
- the cutout-sharded smoothness algorithm with the blur (each rank blurs its cutouts, exchanges two BLURRED boundary
  rows with each neighbour, and gathers its gradient from rows -1 .. rows of the stack) run over gloo on two ranks
  equals the single-process gradient.
"""
import os
import socket
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import aux_ref as A
from pixray_b200 import losses as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G = np.load(os.path.join(GOLDEN, "aux_loss_options.npz"))
TARGET_PNG, MASK_PNG = os.path.join(GOLDEN, "edge_target.png"), os.path.join(GOLDEN, "edge_mask.png")
TYPES = ("default", "clipped", "log")
SMOOTH = sorted(k[:-4] for k in G.files if k.startswith("smooth") and k.endswith("_cfg"))
EDGE = sorted(k[:-4] for k in G.files if k.startswith("edge_") and k.endswith("_cfg"))


def _close(val, grad, ref_val, ref_grad):
    assert abs(float(val) - float(ref_val)) <= 1e-6 * abs(float(ref_val))
    assert np.abs(grad - ref_grad).max() <= 2e-6 * np.abs(ref_grad).max()


def test_golden_has_every_case():
    assert len(SMOOTH) == 12 and len(EDGE) == 5
    cfgs = [G[t + "_cfg"] for t in SMOOTH]
    assert {(c[1], c[2]) for c in cfgs} >= {(k, s) for k in (3, 4.5, 7) for s in (1, 2.5)}
    assert {int(c[0]) for c in cfgs} == {0, 1, 2}
    assert {(c[1] > 0, c[3], c[4]) for c in cfgs} >= {(b, sp, 2) for b in (False, True) for sp in (1, 2)}


@pytest.mark.parametrize("tag", SMOOTH)
def test_smoothness_restatement_matches_reference(tag):
    kind, k, s, sp, order = G[tag + "_cfg"]
    x = torch.from_numpy(G["cut"]).double().requires_grad_(True)
    val = A.smoothness_loss(x, 0.9, TYPES[int(kind)], spacing=int(sp), edge_order=int(order), gaussian_kernel=float(k),
                            gaussian_std=float(s))
    val.backward()
    _close(val.item(), x.grad.numpy(), G[tag + "_val"], G[tag + "_grad"])


@pytest.mark.parametrize("tag", EDGE)
def test_edge_restatement_matches_reference(tag):
    cfg = G[tag + "_cfg"]
    out = torch.from_numpy(G[tag + "_out"]).double().requires_grad_(True)
    H, W = out.shape[2:]
    target = torch.from_numpy(G[tag + "_target"]).double() if cfg[4] else None
    mask = torch.from_numpy(G[tag + "_mask"]).double() if cfg[5] else None
    val = A.edge_loss(out, G["edge_color"].tolist(), _margins_px(cfg[:4], H, W), 0.1, 0.05, target=target, mask=mask)
    val.backward()
    _close(val.item(), out.grad.numpy(), G[tag + "_val"], G[tag + "_grad"])


def _margins_px(m, H, W):
    return (int(m[0] / 100.0 * W), int(m[1] / 100.0 * W), int(m[2] / 100.0 * H), int(m[3] / 100.0 * H))


def _edge_args(img="", mask="", margins=(10, 10, 10, 10)):
    return types.SimpleNamespace(edge_thickness=5, edge_margins=list(margins), edge_color="[0.2+0.6+0.9]",
                                 edge_color_weight=0.1, global_color_weight=0.05, edge_input_image=img,
                                 edge_mask_image=mask)


@pytest.mark.parametrize("tag", EDGE)
def test_edge_parse_settings_resizes_like_the_reference(tag):
    cfg = G[tag + "_cfg"]
    H, W = G[tag + "_out"].shape[2:]
    el = L.EdgeLoss(device="cpu")
    el.parse_settings(_edge_args(TARGET_PNG if cfg[4] else "", MASK_PNG if cfg[5] else ""))
    target, mask = el.resized((H, W))
    if cfg[4]:
        assert np.array_equal(target.numpy(), G[tag + "_target"])
    else:
        assert target is None
    if cfg[5]:
        assert np.array_equal(mask.numpy(), G[tag + "_mask"])
        assert (mask > 0).any() and (mask <= 0).any()
    else:
        assert mask is None


def test_edge_engine_params_layout():
    el = L.EdgeLoss(device="cpu")
    # brace expansion and a sorted glob, first file (util.real_glob)
    args = el.parse_settings(_edge_args(os.path.join(GOLDEN, "edge_{target,mask}.png"), MASK_PNG))
    session = types.SimpleNamespace(engine=types.SimpleNamespace(image_hw=(20, 28)))
    p = el.engine_params(args, session)
    hw = 20 * 28
    assert p.dtype == np.float32 and p.size == 10 + 4 * hw and p[9] == 3
    t, m = el.resized((20, 28))
    assert np.array_equal(p[10:10 + 3 * hw], t.reshape(-1).numpy()) and np.array_equal(p[10 + 3 * hw:], m.reshape(-1).numpy())
    # the mask pattern edge_{target,mask}.png expands to [edge_target, edge_mask]; sorted, the first is edge_mask.png
    assert el.image.mode == "RGB" and el.image.size == (31, 23)
    plain = L.EdgeLoss(device="cpu")
    q = plain.engine_params(plain.parse_settings(_edge_args()), session)
    assert len(q) == 9  # no images: today's parameter list


def test_edge_refuses_urls_and_missing_files():
    for field in ("img", "mask"):
        with pytest.raises(ValueError, match="URL"):
            L.EdgeLoss(device="cpu").parse_settings(_edge_args(**{field: "https://example.com/a.png"}))
        with pytest.raises(FileNotFoundError):
            L.EdgeLoss(device="cpu").parse_settings(_edge_args(**{field: os.path.join(GOLDEN, "no_such_*.png")}))


def _smooth_args(**kw):
    a = dict(smoothness_weight=0.9, smoothness_type="default", smoothness_gaussian_kernel=0, smoothness_gaussian_std=1,
             smoothness_spacing=1, smoothness_edge_order=1)
    a.update(kw)
    return types.SimpleNamespace(**a)


def test_smoothness_engine_params():
    s = L.SmoothnessLoss(device="cpu")
    assert s.engine_params(_smooth_args(), None) == [0.9, 0, 1]  # the defaults keep the 3-value call
    assert s.engine_params(_smooth_args(smoothness_edge_order=2, smoothness_type="log"), None) == [0.9, 2, 1, 2, 0]
    p = s.engine_params(_smooth_args(smoothness_gaussian_kernel=4.5, smoothness_gaussian_std=2.5), None)
    assert p[:5] == [0.9, 0, 1, 1, 5] and len(p) == 5 + 25
    K = torch.tensor(p[5:]).reshape(5, 5)
    assert torch.allclose(K.double(), A.gaussian_kernel2d(4.5, 2.5), rtol=1e-6, atol=0)
    assert not torch.allclose(K, K.flip(0))  # ceil(4.5) taps centred at 1.75: off-centre
    # the separable form the engine applies (row sums) reproduces the 2-D kernel
    u = K.double().sum(1)
    assert torch.allclose(u[:, None] * u[None, :], K.double(), rtol=1e-6, atol=0)


@pytest.mark.parametrize("kw,msg", [(dict(smoothness_edge_order=3), "edge_order=1 and edge_order=2"),
                                    (dict(smoothness_edge_order=0), "edge_order=1 and edge_order=2"),
                                    (dict(smoothness_gaussian_kernel=-3), "smoothness_gaussian_kernel"),
                                    (dict(smoothness_gaussian_kernel=5, smoothness_gaussian_std=0), "smoothness_gaussian_std"),
                                    (dict(smoothness_gaussian_kernel=5, smoothness_gaussian_std=-1), "smoothness_gaussian_std")])
def test_smoothness_refuses_invalid_values(kw, msg):
    with pytest.raises(ValueError, match=msg):
        L.SmoothnessLoss(device="cpu").engine_params(_smooth_args(**kw), None)


def test_torch_refuses_the_same_edge_orders():
    with pytest.raises(RuntimeError, match="edge_order"):
        torch.gradient(torch.rand(5, 5), edge_order=3)


# ---- two ranks over gloo: the engine's blurred-halo algorithm (engine.cu aux_on_cutouts) in float64
CUTN, CS = 4, 14


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_grad(rank, world, port, out, k, std, order, spacing):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    cut = torch.from_numpy(G["cut"][:CUTN, :, :CS, :CS]).double()
    n_local = CUTN // world
    x = cut[rank * n_local:(rank + 1) * n_local].clone().requires_grad_(True)
    w = A.gaussian_kernel2d(k, std)
    b = F.conv2d(x, w[None, None].repeat(3, 1, 1, 1), groups=3)           # this rank's blurred cutouts
    cs2 = b.shape[2]
    rows = b.permute(0, 2, 3, 1).reshape(-1, cs2, 3)                      # [n_local * cs', cs', 3]
    # halo: the previous rank's last two and the next rank's first two BLURRED rows, through one allreduce(sum)
    xbuf = torch.zeros(world, 2, 2, cs2, 3, dtype=torch.float64)
    xbuf[rank, 0], xbuf[rank, 1] = rows[:2].detach(), rows[-2:].detach()
    dist.all_reduce(xbuf)
    parts = ([xbuf[rank - 1, 1]] if rank > 0 else []) + [rows] + ([xbuf[rank + 1, 0]] if rank < world - 1 else [])
    ext = torch.cat(parts)
    off = 2 if rank > 0 else 0
    sq = 0
    for c in range(3):
        gy, gx = torch.gradient(ext[:, :, c], spacing=spacing, edge_order=order)
        sq = sq + gy ** 2 + gx ** 2
    sharp = torch.sqrt(sq)
    n_glob = CUTN * cs2 * cs2
    lo, hi = off - (1 if rank > 0 else 0), off + rows.shape[0] + (1 if rank < world - 1 else 0)
    # rows -1 .. rows of the local stack carry every term that reads a local element; the value sums the local rows
    (sharp[lo:hi].sum() * 0.9 / n_glob).backward()
    val = (sharp[off:off + rows.shape[0]].detach().sum() * 0.9 / n_glob).reshape(1)
    dist.all_reduce(val)
    full = torch.zeros(CUTN, 3, CS, CS, dtype=torch.float64)
    full[rank * n_local:(rank + 1) * n_local] = x.grad
    dist.all_reduce(full)
    if rank == 0:
        torch.save(dict(grad=full, val=val), out)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("k,std,order,spacing", [(5, 1.5, 1, 1), (4.5, 1.0, 2, 2)])
def test_blurred_halo_two_ranks_matches_single_process(tmp_path, k, std, order, spacing):
    import torch.multiprocessing as mp
    out = str(tmp_path / "ranks.pt")
    mp.spawn(_rank_grad, args=(2, _free_port(), out, k, std, order, spacing), nprocs=2, join=True)
    got = torch.load(out)
    x = torch.from_numpy(G["cut"][:CUTN, :, :CS, :CS]).double().requires_grad_(True)
    ref = A.smoothness_loss(x, 0.9, "default", spacing=spacing, edge_order=order, gaussian_kernel=k, gaussian_std=std)
    ref.backward()
    err, mag = (got["grad"] - x.grad).abs().max().item(), x.grad.abs().max().item()
    assert mag > 0 and err <= 2e-5 * mag, (err, mag)
    assert abs(got["val"].item() - ref.item()) <= 1e-12
