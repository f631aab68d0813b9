"""The CLIP ResNet towers op by op at their real shapes: every op of the forward and of the data backward is fed the
engine's own tapped fp16 input (clipN.rn.*) and checked per element against float64.

Budget of a GEMM / conv output: C_GEMM u sum |a||b| (fp32 accumulation of exact fp16 products, u = 2^-11) plus the
rounding of the stored value (u |y| for fp16, 2^-24 |y| for fp32).  Row kernels (pools, token build, mean-token spread, the
stem's preprocess + im2col and its gather) carry their fp32 arithmetic relative to the sum of the magnitudes they combine
plus the output rounding.  ReLU masks are the engine's: each backward op masks with the stored activation > 0, as the
engine does, so a flipped mask near 0 is not an error here.  The padded channels (zero weights) must be exactly 0.

(a) Forward: RN50 and RN50x4 (40-, 80-, 160-wide layers padded) at full depth, the stem's input stage against the float64
    preprocess + stride-2 im2col, every conv, pool and block sum, and the attention pool (tokens, q / k / v, the
    single-query attention, c_proj).
(b) Backward per element: the same, op by op from the engine's de16 back to d loss / d cutouts, on RN50 at full depth and
    on a tower with one block per stage at RN50x4's widths with 3 cutouts (ragged tiles)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ref_path as R
from oracle.resnet_ref import ResnetRef
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_attn_gpu import FLOOR, TINY, U
from test_pipeline_gpu import random_transforms

pytestmark = pytest.mark.gpu

C_GEMM = 2.0
U32 = 2.0 ** -20  # a row kernel's fp32 arithmetic, relative to the magnitudes it combines


def _pad(c):
    return (c + 63) // 64 * 64


class Report:
    def __init__(self, label):
        self.label, self.lines, self.bad = label, [], []

    def check(self, name, got, ref, budget):
        err = (got - ref).abs()
        ratio = (err / budget).max().item()
        self.lines.append(f"  {name}: max err/budget {ratio:.3f}")
        over = ~(err <= budget)
        if over.any():
            i = tuple(over.nonzero()[0].tolist())
            self.bad.append(f"{self.label} {name}: {int(over.sum())} elements over budget, first at {i}: got "
                            f"{got[i].item():.6e} ref {ref[i].item():.6e} budget {budget[i].item():.3e}")

    def zero(self, name, t):
        if t.numel() and t.abs().max().item() != 0:
            self.bad.append(f"{self.label} {name}: padded channels are not 0")

    def finish(self):
        print(f"[resnet ops] {self.label}\n" + "\n".join(self.lines))
        assert not self.bad, "\n".join(self.bad)


def run(arch, cutn, seed):
    """make_cutouts -> encode_image -> prompt loss -> backward on a pixel-drawer engine; every tap as float64 NCHW-able
    [B, H, W, Cp] tensors"""
    sd = S.clip_resnet_state_dict(arch, seed)
    cs = arch["image_res"]
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=cutn, cut_size=cs, clip=[arch],
                       seed=seed)
    tp = {}
    try:
        eng.load_module(E.MOD_CLIP0, sd)
        eng.finalize()
        pm = S.prompts(arch["out_dim"], (1.0, -0.3), seed)
        eng.set_prompts(0, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
        g = torch.Generator().manual_seed(seed)
        img = eng.synth(torch.rand(eng.z_shape, generator=g))
        facs, noise = torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, cs, cs, generator=g)
        eng.make_cutouts(img, transforms=random_transforms(cutn, cs, seed), zoom_padding=E.PAD_REFLECTION, fill=0.4,
                         noise_facs=facs.numpy(), noise=noise)
        eng.encode_image(0)
        eng.backward()

        def rd(name, shape, dt=torch.half):
            full = name if name.startswith("clip0.") or name in ("batch", "g_batch", "range") else "clip0.rn." + name
            tp[name] = eng.debug_read(full, shape, dt).double().cpu()

        B, w, h0 = cutn, arch["width"], cs // 2
        c1, c3 = _pad(w // 2), _pad(w)
        rd("cols", (B, h0, h0, 64))
        rd("g_cols", (B, h0, h0, 64))
        for n, c in (("a1", c1), ("a2", c1), ("a3", c3), ("g_a1", c1), ("g_a2", c1), ("g_a3", c3)):
            rd("stem." + n, (B, h0, h0, c))
        rd("stem.out", (B, h0 // 2, h0 // 2, c3))
        rd("stem.g_out", (B, h0 // 2, h0 // 2, c3))
        h, cin = h0 // 2, c3
        for s, nb in enumerate(arch["blocks"]):
            pp, co = _pad(w << s), 4 * (w << s)
            for k in range(nb):
                stride = 2 if (s > 0 and k == 0) else 1
                ho = h // stride
                t = f"{s + 1}.{k}."
                for n in ("a", "b", "g_a", "g_b"):
                    rd(t + n, (B, h, h, pp))
                for n in ("y", "g_sum"):
                    rd(t + n, (B, ho, ho, co))
                down = stride > 1 or cin != co
                if stride > 1:
                    rd(t + "b_pool", (B, ho, ho, pp))
                    rd(t + "g_b_pool", (B, ho, ho, pp))
                if down:
                    rd(t + "identity", (B, ho, ho, co))
                    rd(t + "g_identity", (B, ho, ho, cin))
                    if stride > 1:
                        rd(t + "x_pool", (B, ho, ho, cin))
                        rd(t + "g_identity_in", (B, h, h, cin))
                h, cin = ho, co
        Ce, T = 32 * w, h * h + 1
        for n, shape in (("tokens", (B, T, Ce)), ("kv", (B, T, 2 * Ce)), ("o", (B, Ce)), ("g_o", (B, Ce)),
                         ("g_q", (B, Ce)), ("g_kv", (B, T, 2 * Ce)), ("g_tokens", (B, T, Ce)), ("g_token0", (B, Ce))):
            rd("pool." + n, shape)
        rd("pool.q", (B, Ce), torch.float32)
        rd("pool.p", (B, Ce // 64, T), torch.float32)
        for n, shape, dt in (("clip0.e", (B, arch["out_dim"]), torch.float32), ("clip0.de16", (B, arch["out_dim"]), torch.half),
                             ("batch", (B, 3, cs, cs), torch.float32), ("g_batch", (B, 3, cs, cs), torch.float32),
                             ("range", (4,), torch.float32)):
            rd(n, shape, dt)
    finally:
        eng.close()
    return sd, tp


def nchw(t, c):
    return t[..., :c].permute(0, 3, 1, 2)


def conv(x, w, b=None, transpose=False):
    if transpose:  # the data gradient of a stride-1 "same" conv
        return F.conv_transpose2d(x, w, None, padding=w.shape[-1] // 2)
    return F.conv2d(x, w, b, padding=w.shape[-1] // 2)


def gemm_budget(sabs, y, out32=False):
    return C_GEMM * U * sabs + (2.0 ** -24 * y.abs() + FLOOR if out32 else U * (y.abs() + TINY))


def row_budget(mag, y):
    return U32 * mag + U * (y.abs() + TINY)


def pool_bwd(g):
    return F.interpolate(g, scale_factor=2, mode="nearest") * 0.25


def check_act(rep, name, got, ref, budget):
    """got [B, H, W, Cp] engine tap; ref / budget NCHW with the real channels"""
    c = ref.shape[1]
    rep.check(name, nchw(got, c), ref, budget)
    rep.zero(name + " (padding)", got[..., c:])


def check_tower(label, arch, cutn, seed):
    sd, tp = run(arch, cutn, seed)
    ref = ResnetRef(sd, folded=True)
    fw = ref._fold
    rep = Report(label)
    w = arch["width"]
    mask = lambda t, c: (nchw(t, c) > 0).double()  # noqa: E731
    # ---- stem input stage: the float64 preprocess of the engine's cutouts (its global range), stride-2 im2col
    mn, rng = tp["range"][0], tp["range"][1]
    mean = torch.tensor(R.CLIP_MEAN, dtype=torch.float64).view(1, 3, 1, 1)
    std = torch.tensor(R.CLIP_STD, dtype=torch.float64).view(1, 3, 1, 1)
    xn = ((tp["batch"] - mn) / rng - mean) / std
    B, cs = xn.shape[0], xn.shape[-1]
    h0 = cs // 2
    cols = F.unfold(xn, 3, padding=1, stride=2).view(B, 27, h0, h0)
    mag = (tp["batch"].abs() + mn.abs()) / rng / std + mean.abs() / std
    check_act(rep, "stem cols (preprocess + im2col)", tp["cols"], cols,
              row_budget(F.unfold(mag, 3, padding=1, stride=2).view(B, 27, h0, h0), cols))
    # ---- forward, every op from the engine's own input
    w1, b1 = fw["conv1"]
    w1f = w1.reshape(w1.shape[0], 27, 1, 1)
    x = nchw(tp["cols"], 27)
    y = torch.relu(conv(x, w1f, b1))
    check_act(rep, "stem conv1", tp["stem.a1"], y, gemm_budget(conv(x.abs(), w1f.abs(), b1.abs()), y))
    for i, (src, dst) in enumerate((("stem.a1", "stem.a2"), ("stem.a2", "stem.a3")), start=2):
        wi, bi = fw[f"conv{i}"]
        x = nchw(tp[src], wi.shape[1])
        y = torch.relu(conv(x, wi, bi))
        check_act(rep, f"stem conv{i}", tp[dst], y, gemm_budget(conv(x.abs(), wi.abs(), bi.abs()), y))
    x = nchw(tp["stem.a3"], w)
    y = F.avg_pool2d(x, 2)
    check_act(rep, "stem avgpool", tp["stem.out"], y, row_budget(F.avg_pool2d(x.abs(), 2), y))
    xin, cin = "stem.out", w
    for s, nb in enumerate(arch["blocks"]):
        p_ = w << s
        for k in range(nb):
            t, pre = f"{s + 1}.{k}.", f"layer{s + 1}.{k}"
            stride = 2 if (s > 0 and k == 0) else 1
            x = nchw(tp[xin], cin)
            wa, ba = fw[pre + ".conv1"]
            y = torch.relu(conv(x, wa, ba))
            check_act(rep, t + "conv1", tp[t + "a"], y, gemm_budget(conv(x.abs(), wa.abs(), ba.abs()), y))
            a = nchw(tp[t + "a"], p_)
            wb, bb = fw[pre + ".conv2"]
            y = torch.relu(conv(a, wb, bb))
            check_act(rep, t + "conv2", tp[t + "b"], y, gemm_budget(conv(a.abs(), wb.abs(), bb.abs()), y))
            bmain = t + "b"
            if stride > 1:
                bt = nchw(tp[t + "b"], p_)
                y = F.avg_pool2d(bt, 2)
                check_act(rep, t + "avgpool", tp[t + "b_pool"], y, row_budget(F.avg_pool2d(bt.abs(), 2), y))
                bmain = t + "b_pool"
            idn, idn_abs = x, x.abs()
            if pre + ".downsample" in fw:
                xs = x
                if stride > 1:
                    y = F.avg_pool2d(x, 2)
                    check_act(rep, t + "downsample avgpool", tp[t + "x_pool"], y, row_budget(F.avg_pool2d(x.abs(), 2), y))
                    xs = nchw(tp[t + "x_pool"], cin)
                wd, bd = fw[pre + ".downsample"]
                y = conv(xs, wd, bd)
                check_act(rep, t + "downsample", tp[t + "identity"], y, gemm_budget(conv(xs.abs(), wd.abs(), bd.abs()), y))
                idn = nchw(tp[t + "identity"], 4 * p_)
                idn_abs = idn.abs()
            bm = nchw(tp[bmain], p_)
            wc, bc = fw[pre + ".conv3"]
            y = torch.relu(conv(bm, wc, bc) + idn)
            check_act(rep, t + "conv3 + identity, ReLU", tp[t + "y"], y,
                      gemm_budget(conv(bm.abs(), wc.abs(), bc.abs()) + idn_abs, y))
            xin, cin = t + "y", 4 * p_
    # ---- attention pool
    Ce = 32 * w
    a = "visual.attnpool."
    W16 = lambda n: sd[a + n + ".weight"].float().half().double()  # noqa: E731
    bias = lambda n: sd[a + n + ".bias"].float().double()  # noqa: E731
    pos = sd[a + "positional_embedding"].float().double()
    xl = nchw(tp[xin], Ce)
    pix = xl.flatten(2).transpose(1, 2)
    tok = torch.cat([pix.mean(1, keepdim=True), pix], 1) + pos
    tmag = torch.cat([pix.abs().mean(1, keepdim=True), pix.abs()], 1) + pos.abs()
    rep.check("pool tokens (mean + positions)", tp["pool.tokens"], tok, row_budget(tmag, tok))
    tk = tp["pool.tokens"]
    wkv = torch.cat([W16("k_proj"), W16("v_proj")])
    bkv = torch.cat([bias("k_proj"), bias("v_proj")])
    kv = tk @ wkv.T + bkv
    rep.check("pool k | v", tp["pool.kv"], kv, gemm_budget(tk.abs() @ wkv.abs().T + bkv.abs(), kv))
    q = tk[:, 0] @ W16("q_proj").T + bias("q_proj")
    rep.check("pool q", tp["pool.q"], q, gemm_budget(tk[:, 0].abs() @ W16("q_proj").abs().T + bias("q_proj").abs(), q, True))
    H, T = Ce // 64, tk.shape[1]
    qh = (tp["pool.q"] * 0.125).view(B, H, 1, 64)
    kh = tp["pool.kv"][..., :Ce].view(B, T, H, 64).transpose(1, 2)
    vh = tp["pool.kv"][..., Ce:].view(B, T, H, 64).transpose(1, 2)
    sc = (qh @ kh.transpose(-1, -2)).squeeze(2)
    pr = torch.softmax(sc, -1)
    smag = (qh.abs() @ kh.abs().transpose(-1, -2)).squeeze(2)
    rep.check("pool softmax", tp["pool.p"], pr, pr * (2.0 ** -18 + 2.0 ** -21 * (smag + sc.abs()).amax(-1, keepdim=True)) + FLOOR)
    pe = tp["pool.p"]
    o = (pe.unsqueeze(2) @ vh).squeeze(2).reshape(B, Ce)
    omag = (pe.unsqueeze(2) @ vh.abs()).squeeze(2).reshape(B, Ce)
    rep.check("pool attention o", tp["pool.o"], o, row_budget(omag, o))
    ov = tp["pool.o"]
    e = ov @ W16("c_proj").T + bias("c_proj")
    rep.check("c_proj", tp["clip0.e"], e, gemm_budget(ov.abs() @ W16("c_proj").abs().T + bias("c_proj").abs(), e, True))

    # ---- backward, op by op from the engine's de16
    de = tp["clip0.de16"]
    go = de @ W16("c_proj")
    rep.check("d c_proj", tp["pool.g_o"], go, gemm_budget(de.abs() @ W16("c_proj").abs(), go))
    gov = tp["pool.g_o"].view(B, H, 64)
    dp = (vh @ gov.unsqueeze(-1)).squeeze(-1)                        # [B, H, T]
    dpm = (vh.abs() @ gov.abs().unsqueeze(-1)).squeeze(-1)
    dsum = (pe * dp).sum(-1, keepdim=True)
    ds = pe * (dp - dsum)
    dsm = pe * (dpm + (pe * dpm).sum(-1, keepdim=True))
    gk = ds.unsqueeze(-1) * qh                                       # [B, H, T, 64]
    gv = pe.unsqueeze(-1) * gov.unsqueeze(2)
    gkv = torch.cat([gk.transpose(1, 2).reshape(B, T, Ce), gv.transpose(1, 2).reshape(B, T, Ce)], -1)
    gkvm = torch.cat([(dsm.unsqueeze(-1) * qh.abs()).transpose(1, 2).reshape(B, T, Ce),
                      gv.abs().transpose(1, 2).reshape(B, T, Ce)], -1)
    rep.check("d attention k | v", tp["pool.g_kv"], gkv, row_budget(16 * gkvm, gkv))
    gq = 0.125 * (ds.unsqueeze(-2) @ kh).squeeze(-2).reshape(B, Ce)
    gqm = 0.125 * (dsm.unsqueeze(-2) @ kh.abs()).squeeze(-2).reshape(B, Ce)
    rep.check("d attention q", tp["pool.g_q"], gq, row_budget(16 * gqm, gq))
    g = tp["pool.g_kv"]
    gt = g @ wkv
    rep.check("d k | v projections", tp["pool.g_tokens"], gt, gemm_budget(g.abs() @ wkv.abs(), gt))
    g0 = tp["pool.g_q"] @ W16("q_proj")
    rep.check("d q projection", tp["pool.g_token0"], g0, gemm_budget(tp["pool.g_q"].abs() @ W16("q_proj").abs(), g0))
    gtk, g0e = tp["pool.g_tokens"], tp["pool.g_token0"]
    hw = T - 1
    side = int(round(hw ** 0.5))
    spread = gtk[:, 1:] + (gtk[:, :1] + g0e.unsqueeze(1)) / hw
    smag2 = gtk[:, 1:].abs() + (gtk[:, :1].abs() + g0e.abs().unsqueeze(1)) / hw
    m = mask(tp[xin], Ce).flatten(2).transpose(1, 2)
    gs = (spread * m).transpose(1, 2).reshape(B, Ce, side, side)
    check_act(rep, "d tokens (mean spread, last ReLU)", tp[xin.replace("y", "g_sum")], gs,
              row_budget((smag2 * m).transpose(1, 2).reshape(B, Ce, side, side), gs))
    blocks = [(s, k) for s, nb in enumerate(arch["blocks"]) for k in range(nb)]
    for j in range(len(blocks) - 1, -1, -1):
        s, k = blocks[j]
        p_ = w << s
        t, pre = f"{s + 1}.{k}.", f"layer{s + 1}.{k}"
        stride = 2 if (s > 0 and k == 0) else 1
        first = j == 0
        prev = "stem.out" if first else f"{blocks[j - 1][0] + 1}.{blocks[j - 1][1]}.y"
        cin = w if first else 4 * (w << blocks[j - 1][0])
        gsum = nchw(tp[t + "g_sum"], 4 * p_)
        wc, _ = fw[pre + ".conv3"]
        mb = mask(tp[t + "b"], p_)
        y = conv(gsum, wc, transpose=True)
        ym = conv(gsum.abs(), wc.abs(), transpose=True)
        if stride > 1:
            check_act(rep, t + "d conv3", tp[t + "g_b_pool"], y, gemm_budget(ym, y))
            gbp = nchw(tp[t + "g_b_pool"], p_)
            y = pool_bwd(gbp) * mb
            check_act(rep, t + "d avgpool, ReLU", tp[t + "g_b"], y, row_budget(pool_bwd(gbp.abs()), y))
        else:
            check_act(rep, t + "d conv3, ReLU", tp[t + "g_b"], y * mb, gemm_budget(ym * mb, y * mb))
        gb = nchw(tp[t + "g_b"], p_)
        wb, _ = fw[pre + ".conv2"]
        ma = mask(tp[t + "a"], p_)
        y = conv(gb, wb, transpose=True) * ma
        check_act(rep, t + "d conv2, ReLU", tp[t + "g_a"], y, gemm_budget(conv(gb.abs(), wb.abs(), transpose=True) * ma, y))
        gid, gidm = gsum, gsum.abs()
        if pre + ".downsample" in fw:
            wd, _ = fw[pre + ".downsample"]
            y = conv(gsum, wd, transpose=True)
            check_act(rep, t + "d downsample", tp[t + "g_identity"], y, gemm_budget(conv(gsum.abs(), wd.abs(), transpose=True), y))
            gid = nchw(tp[t + "g_identity"], cin)
            if stride > 1:
                y = pool_bwd(gid)
                check_act(rep, t + "d downsample avgpool", tp[t + "g_identity_in"], y, row_budget(pool_bwd(gid.abs()), y))
                gid = nchw(tp[t + "g_identity_in"], cin)
            gidm = gid.abs()
        ga = nchw(tp[t + "g_a"], p_)
        wa, _ = fw[pre + ".conv1"]
        mx = 1.0 if first else mask(tp[prev], cin)
        y = (conv(ga, wa, transpose=True) + gid) * mx
        dst = "stem.g_out" if first else prev.replace("y", "g_sum")
        check_act(rep, t + "d conv1 + identity" + ("" if first else ", ReLU"), tp[dst], y,
                  gemm_budget((conv(ga.abs(), wa.abs(), transpose=True) + gidm) * mx, y))
    go_ = nchw(tp["stem.g_out"], w)
    y = pool_bwd(go_) * mask(tp["stem.a3"], w)
    check_act(rep, "stem d avgpool, ReLU", tp["stem.g_a3"], y, row_budget(pool_bwd(go_.abs()), y))
    for i, (src, dst, mk, c) in enumerate((("stem.g_a3", "stem.g_a2", "stem.a2", w // 2),
                                            ("stem.g_a2", "stem.g_a1", "stem.a1", w // 2))):
        wi, _ = fw[f"conv{3 - i}"]
        gi = nchw(tp[src], wi.shape[0])
        mm = mask(tp[mk], c)
        y = conv(gi, wi, transpose=True) * mm
        check_act(rep, f"stem d conv{3 - i}, ReLU", tp[dst], y, gemm_budget(conv(gi.abs(), wi.abs(), transpose=True) * mm, y))
    g1 = nchw(tp["stem.g_a1"], w // 2)
    y = conv(g1, w1f, transpose=True)
    check_act(rep, "stem d conv1 (im2col rows)", tp["g_cols"], y, gemm_budget(conv(g1.abs(), w1f.abs(), transpose=True), y))
    gc = nchw(tp["g_cols"], 27).reshape(B, 27, -1)
    gx = F.fold(gc, (cs, cs), 3, padding=1, stride=2) / (std * rng)
    gxm = F.fold(gc.abs(), (cs, cs), 3, padding=1, stride=2) / (std * rng)
    rep.check("stem input stage backward (gather)", tp["g_batch"], gx, U32 * gxm + 2.0 ** -24 * gx.abs() + FLOOR)
    rep.finish()


@pytest.mark.parametrize("name", ["RN50", "RN50x4"])
def test_full_depth_op_by_op(name):
    check_tower(f"{name} full depth", E.RESNET_ARCH[name], cutn=4, seed=31)


def test_one_block_per_stage_op_by_op():
    arch = dict(E.RESNET_ARCH["RN50x4"], blocks=(1, 1, 1, 1), layers=4)
    check_tower("RN50x4 widths, one block per stage, 3 cutouts", arch, cutn=3, seed=33)
