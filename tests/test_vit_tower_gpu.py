"""The ViT image towers (Engine::build_clip) layer by layer against float64, at the real shapes, on every attention and
residual-stream path.

The reference is float64 on the CPU, built from the oracle modules (oracle/ref_path.py ClipVisual, oracle/slip_ref.py
SlipVisual) in double precision with the engine's weights: the GEMM weights (patch embedding, qkv, out_proj, c_fc /
fc1, c_proj / fc2, proj) rounded to fp16 as the engine uploads them, biases, LayerNorm parameters, class and position
embeddings in fp32.  The engine runs make_cutouts -> encode_image -> backward; the tower's input is the engine's own
`clipN.patches`, so the cutouts and the preprocess (tested elsewhere) drop out.

(a) Forward, one step at a time, at full depth: every step is fed the engine's own stored input (its debug taps) and
    compared with the engine's stored output, element by element.  u = 2^-11, c = 2 (C_GEMM), every |.| product in
    float64 over the fp16 operands:
      GEMM output          c u sum|a||b| + one rounding of the stored output (u (|y| + 2^-14) fp16, 2^-24 |y| fp32)
      LN -> GEMM           + sum_k amb_k (2u |h_k| + 2^-24) |w_k|: the reference rounds the float64 LayerNorm output h
                           to fp16 itself; where h lies within the LN kernel's fp32 error (4 2^-18 (|gamma||x^| + |beta|))
                           of an fp16 rounding boundary (amb_k), the engine's h may sit one fp16 ulp away
      MLP second GEMM      + u sum_k (|act'(u_k)| (|u_k| + 2^-14) + |act_k| + 2^-14) |w_k|: the activation is evaluated
                           on the fp32 pre-activation, not on the stored fp16 u, and then rounded to fp16
      LayerNorm outputs    4 u (|gamma| |x^| + |beta|) + 2^-24   (4 2^-18 on the fp32 stream), as tests/test_row_kernels_gpu.py
      fused attention o    the budget of tests/test_attn_gpu.py (imported)
      row-softmax P        P (e_ij + sum_k P_ik e_ik) + u (P + 2^-14) + 2^-20 P, e = u |S| + c u scale |q||k|: the fp16
                           scores and their GEMM error carried through the softmax; pad columns exactly 0
    In the class-rows-only last layer (PXR_CLIP_LAST_CLS=1) only the B class rows, at pitch T W, are compared.

(b) Backward per element on two-layer towers at full width, T and heads (layer 0 a full layer, layer 1 the class-rows
    tail): the float64 VJP from the engine's de16, taken at the engine's own forward values, through proj, ln_post, both
    layers, ln_pre and the patch-embed dgrad, against gx16 (d/dt, all rows) and g_patches, both scaled by the 4096
    gradient scale.  Over a chain of a dozen fp16 roundings a worst-case (|.|-propagated) bound grows ~sqrt(K) per GEMM
    and says nothing, so every element carries a statistical budget instead: every rounding of a stored fp16 / fp32
    tensor is an independent error of standard deviation (its bound) / sqrt(3), the attention backward's own error one
    of u mag (tests/test_attn_gpu.py's magnitudes), every GEMM's accumulation one of 2^-20 sum|a||b|, every LayerNorm
    backward's 2^-18 times the row-kernel test's magnitude; variances are carried through the exact Jacobians squared,
    and the budget is K_SIGMA = 6 standard deviations + 2^-24.  g_patches is also checked against the engine's own gx16
    with the single-GEMM budget of (a).

(c) Backward at full depth by norm: g_patches against the float64 VJP at the engine's forward values,
    rel-L2 <= REL_L2_BOUND = 4e-3 and cosine >= COS_BOUND = 1 - 1e-5.  Measured on an H100 SXM at its default power
    limit: rel-L2 7.9e-4 .. 1.6e-3 (MEASURED_REL_L2) and cosine >= 0.9999987 over the six full-depth cases, so the rel-L2
    bound has a 2.5x margin.  The CPU tests plant bugs in the float64 reference and measure what they move:
      one head's dV dropped in layer 6 of ViT-B/32      g_patches rel-L2 5.1e-2, over ten times the full-depth bound;
                                                        in a two-layer tower, 100x the per-element budget of (b)
      the mean term of one ln_1 backward dropped        rel-L2 4.3e-3 at full depth (about the bound: the norm check
                                                        cannot see it); in a two-layer tower 2-8x the per-element budget
                                                        of (b), which is the check that catches it
      the QuickGELU slope 1.702 taken as 1.7            rel-L2 2.2e-4, half of one fp16 rounding (u = 4.9e-4): below
                                                        the resolution of any comparison with an fp16 backward, so no
                                                        test here asserts on it; the constant itself is pinned by
                                                        test_slip_gpu.py's bit-identity test of the QuickGELU epilogue

(d) Residual-stream outliers: two channels of a few hundred, planted through layer 0's c_proj / fc2 bias, on the fp16
    stream; (a) and (b) hold, and every value of gx16 and g_patches is finite (the largest |4096 g| is printed against the
    fp16 limit 65504).

Every tensor prints its largest err / budget; with cutn 3, M = B T is ragged."""
import pytest
import torch

from oracle import ref_path as R
from oracle import slip_ref as SR
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S
from test_attn_gpu import C_BUDGET, FLOOR, TINY, U, _reference, _split
from test_pipeline_gpu import random_transforms

U32 = 2.0 ** -18    # the LayerNorm kernels' fp32 arithmetic, as in tests/test_row_kernels_gpu.py
C_GEMM = 2.0        # c of the GEMM budgets
C_LN = 4.0          # c of the LayerNorm budgets (tests/test_row_kernels_gpu.py)
ACC = 2.0 ** -20    # standard deviation of a GEMM's fp32 accumulation error, relative to sum |a||b|
K_SIGMA = 6.0
GRAD_SCALE = 4096.0
FP16_MAX = 65504.0
REL_L2_BOUND = 4e-3   # 2.5x the largest measured, MEASURED_REL_L2
COS_BOUND = 1 - 1e-5
MEASURED_REL_L2 = 1.6e-3
SCALE = 0.125       # 1 / sqrt(64)


def f16(t):
    """What upload_f16 makes of an fp32 weight, in float64."""
    return t.detach().float().half().double()


def r16v(y):
    """Variance of the rounding of y to fp16 (uniform within +-u (|y| + 2^-14))."""
    return (U * (y.abs() + TINY)) ** 2 / 3


def r32v(y):
    return (2.0 ** -24 * y.abs()) ** 2 / 3


def _round_up(n, m):
    return (n + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ the float64 tower
class _Layer:
    def __init__(self, ln1, wqkv, bqkv, wo, bo, ln2, wfc, bfc, wproj, bproj):
        self.ln1, self.ln2 = ln1, ln2
        self.wqkv, self.wo, self.wfc, self.wproj = wqkv, wo, wfc, wproj       # [out, in], fp16 values
        self.bqkv, self.bo, self.bfc, self.bproj = bqkv, bo, bfc, bproj


class Tower:
    """The oracle image tower in float64 with the engine's weights (fp16 where the engine uploads fp16)."""

    def __init__(self, arch, sd):
        self.timm = arch.get("tower") == E.TOWER_TIMM_VIT
        W, P = arch["width"], arch["patch"]
        self.W, self.H, self.L, self.P, self.D = W, arch["heads"], arch["layers"], P, arch["out_dim"]
        self.np = (arch["image_res"] // P) ** 2
        self.T, self.Kp = self.np + 1, _round_up(3 * P * P, 64)
        if self.timm:
            m = SR.make_model(arch, sd).double()
            v = m.visual
            conv, self.conv_b = v.patch_embed.proj.weight, v.patch_embed.proj.bias.detach()
            self.cls, self.pos = v.cls_token.detach().reshape(W), v.pos_embed.detach().reshape(-1, W)
            self.ln_pre, self.ln_post, proj = None, v.norm, m.image_projection
            blocks = [(b.norm1, b.attn.qkv, b.attn.proj, b.norm2, b.mlp.fc1, b.mlp.fc2) for b in v.blocks]
        else:
            m = R.ClipVisual(arch["image_res"], P, W, arch["layers"], arch["heads"], arch["out_dim"])
            m.load_state_dict(sd)
            m = m.double()
            v = m.visual
            conv, self.conv_b = v.conv1.weight, None
            self.cls, self.pos = v.class_embedding.detach(), v.positional_embedding.detach()
            self.ln_pre, self.ln_post, proj = v.ln_pre, v.ln_post, v.proj
            blocks = [(b.ln_1, None, b.attn.out_proj, b.ln_2, b.mlp.c_fc, b.mlp.c_proj) for b in v.transformer.resblocks]
            mha = [b.attn for b in v.transformer.resblocks]
        m.requires_grad_(False)
        with torch.no_grad():  # the engine's fp16 weights, in the module itself
            conv.copy_(f16(conv))
            proj.copy_(f16(proj))
            self.layers = []
            for i, (n1, qkv, po, n2, fc, pr) in enumerate(blocks):
                if qkv is None:
                    wq, bq = mha[i].in_proj_weight, mha[i].in_proj_bias
                else:
                    wq, bq = qkv.weight, qkv.bias
                for w in (wq, po.weight, fc.weight, pr.weight):
                    w.copy_(f16(w))
                self.layers.append(_Layer(n1, wq.detach(), bq.detach(), po.weight.detach(), po.bias.detach(), n2,
                                          fc.weight.detach(), fc.bias.detach(), pr.weight.detach(), pr.bias.detach()))
        self.model = m
        self.conv = torch.zeros(W, self.Kp, dtype=torch.float64)
        self.conv[:, :3 * P * P] = conv.detach().reshape(W, -1)
        self.proj = proj.detach()   # [W, D]

    def act(self, u, slope=1.702):
        """The MLP activation and its derivative (QuickGELU, or timm's exact GELU)."""
        if self.timm:
            return SR.gelu(u)
        s = torch.sigmoid(slope * u)
        return u * s, s + slope * u * s * (1 - s)

    def pos_rows(self, B):
        return self.pos.repeat(B, 1)


def _ln(x, ln):
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + ln.eps)
    xh = (x - mean) * rstd
    ga, be = ln.weight.detach(), ln.bias.detach()
    return xh * ga + be, xh, rstd, ga.abs() * xh.abs() + be.abs()


def _merge(t, B, T):
    """[n, B, H, T, 64] -> [B*T, n*H*64] (inverse of test_attn_gpu._split)."""
    n, _, H = t.shape[:3]
    return t.permute(1, 3, 0, 2, 4).reshape(B * T, n * H * 64)


def forward64(tw, patches, cls_only=False):
    """The exact float64 forward from patches [B, np, Kp]: the engine's taps (u of a class-rows-only last layer compact)
    and the embeddings."""
    B, T, W = patches.shape[0], tw.T, tw.W
    t = torch.zeros(B, T, W, dtype=torch.float64)
    t[:, 0] = tw.cls
    t[:, 1:] = patches @ tw.conv.T + (0 if tw.conv_b is None else tw.conv_b)
    t = t.reshape(B * T, W)
    x = t + tw.pos_rows(B)
    if tw.ln_pre is not None:
        x = _ln(x, tw.ln_pre)[0]
    taps = dict(t=t, x0=x)
    cls = torch.arange(B) * T
    for l, ly in enumerate(tw.layers):
        qkv = _ln(x, ly.ln1)[0] @ ly.wqkv.T + ly.bqkv
        o = _merge(_reference(qkv, None, B, T, tw.H, SCALE)[0]["o"][None], B, T)
        xm = x + o @ ly.wo.T + ly.bo
        u = _ln(xm, ly.ln2)[0] @ ly.wfc.T + ly.bfc
        x = xm + tw.act(u)[0] @ ly.wproj.T + ly.bproj
        taps.update({f"qkv{l}": qkv, f"o{l}": o, f"x_mid{l}": xm, f"x{l + 1}": x,
                     f"u{l}": u[cls] if cls_only and l == tw.L - 1 else u})
    taps["hcls"] = _ln(x[cls], tw.ln_post)[0]
    taps["e"] = taps["hcls"] @ tw.proj
    return taps


# ------------------------------------------------------------------------------------------------ float64 VJP
def _mm(a, va, w):
    """y = a @ w and, with va, the variance of the engine's y: the inputs' errors through w plus the accumulation."""
    y = a @ w
    if va is None:
        return y, None
    return y, va @ (w * w) + (ACC * (a.abs() @ w.abs())) ** 2


def _lnb(dy, vdy, x, ln, drop_mean=False):
    """LayerNorm backward (rows of x) and, with vdy, the variance of the engine's result."""
    _, xh, rstd, _ = _ln(x, ln)
    ga = ln.weight.detach()
    gg = dy * ga
    m1, m2 = gg.mean(-1, keepdim=True), (gg * xh).mean(-1, keepdim=True)
    d = rstd * (gg - (0 if drop_mean else m1) - xh * m2)
    if vdy is None:
        return d, None
    W = x.shape[-1]
    vg = vdy * ga * ga
    var = rstd ** 2 * (vg + vg.mean(-1, keepdim=True) / W + xh ** 2 * (vg * xh ** 2).mean(-1, keepdim=True) / W)
    bmag = rstd * (gg.abs() + gg.abs().mean(-1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(-1, keepdim=True))
    return d, var + (U32 * bmag) ** 2


def _attn_bwd(qkv, go, vgo, B, T, H, fused, drop_dv_head=False):
    """gqkv = the attention's VJP (tests/test_attn_gpu.py's float64 reference) and its variance: dO's error through the
    exact Jacobian squared plus the kernel's own error, of standard deviation u mag (mag that test's magnitudes; the
    row-softmax path also rounds dP to fp16, which adds P o sum_j P_j |dO||V_j|)."""
    ref, mag = _reference(qkv, go, B, T, H, SCALE)
    if drop_dv_head:
        ref["dv"] = ref["dv"].clone()
        ref["dv"][:, 0] = 0
    g = _merge(torch.stack([ref["dq"], ref["dk"], ref["dv"]]), B, T)
    if vgo is None:
        return g, None
    x = _split(qkv.double(), B, T, H)
    q, k, v = x[0], x[1], x[2]
    p = torch.softmax((q @ k.transpose(-1, -2)) * SCALE, -1)
    vg = _split(vgo, B, T, H)[0]
    pp = p * p
    vdv = pp.transpose(-1, -2) @ vg
    vdp = vg @ (v * v).transpose(-1, -2)
    vds = pp * (vdp + (pp * vdp).sum(-1, keepdim=True))
    vdq = SCALE ** 2 * vds @ (k * k)
    vdk = SCALE ** 2 * vds.transpose(-1, -2) @ (q * q)
    lq, lk, lv = mag["dq"], mag["dk"], mag["dv"]
    if not fused:
        ga = _split(go.double(), B, T, H)[0].abs()
        dpa = ga @ v.abs().transpose(-1, -2)
        extra = p * (p * dpa).sum(-1, keepdim=True)
        lq, lk = lq + SCALE * extra @ k.abs(), lk + SCALE * extra.transpose(-1, -2) @ q.abs()
    local = torch.stack([lq, lk, lv]) * U
    return g, _merge(torch.stack([vdq, vdk, vdv]) + local ** 2, B, T)


def vjp(tw, taps, de, *, cls_only, stream32, fused, var=True, mutate=None, mutate_layer=None):
    """d/dt (gx16's content after the ln_pre backward) and d/d patches from de [B, D] at the forward values `taps`,
    following the engine's backward op by op; with var, also the variances of the engine's gx16 and g_patches."""
    B, T, W, L = de.shape[0], tw.T, tw.W, tw.L
    M = B * T
    cls = torch.arange(B) * T
    z = (lambda t: torch.zeros_like(t)) if var else (lambda t: None)
    gcls, v = _mm(de, z(de), tw.proj.T)
    d, vd = _lnb(gcls, v + r16v(gcls) if var else None, taps[f"x{L}"][cls], tw.ln_post)
    gx = torch.zeros(M, W, dtype=torch.float64)
    gx[cls] = d
    v16 = v32 = None
    if var:
        v32 = torch.zeros_like(gx)
        v32[cls] = vd + (r32v(d) if stream32 else r16v(d))
        v16 = v32 + r16v(gx) if stream32 else v32.clone()

    def accumulate(rows, d, vd):
        gx[rows] += d
        if var:
            if stream32:
                v32[rows] += vd + r32v(gx[rows])
                v16[rows] = v32[rows] + r16v(gx[rows])
            else:
                v16[rows] += vd + r16v(gx[rows])

    for l in reversed(range(L)):
        ly = tw.layers[l]
        rows = cls if cls_only and l == L - 1 else torch.arange(M)
        p, vp = _mm(gx[rows], v16[rows] if var else None, ly.wproj)
        slope = 1.7 if mutate == "gelu_slope" else 1.702
        da = tw.act(taps[f"u{l}"][:len(rows)], slope)[1]   # compact in a class-rows-only layer
        g4 = p * da
        vg4 = vp * da * da + (2.0 ** -20 * g4) ** 2 + r16v(g4) if var else None
        gh, vgh = _mm(g4, vg4, ly.wfc)
        d, vd = _lnb(gh, vgh + r16v(gh) if var else None, taps[f"x_mid{l}"][rows], ly.ln2)
        accumulate(rows, d, vd)
        go = torch.zeros(M, W, dtype=torch.float64)
        vgo = torch.zeros_like(go) if var else None
        go[rows], vr = _mm(gx[rows], v16[rows] if var else None, ly.wo)
        if var:
            vgo[rows] = vr + r16v(go[rows])
        gqkv, vq = _attn_bwd(taps[f"qkv{l}"], go, vgo, B, T, tw.H, fused,
                             drop_dv_head=mutate == "dv_head" and l == mutate_layer)
        gh, vgh = _mm(gqkv, vq, ly.wqkv)
        d, vd = _lnb(gh, vgh + r16v(gh) if var else None, taps[f"x{l}"], ly.ln1,
                     drop_mean=mutate == "ln_mean" and l == mutate_layer)
        accumulate(torch.arange(M), d, vd)
    if tw.ln_pre is not None:  # overwrites gx16 (and the fp32 gx) with d/dt
        d, vd = _lnb(gx, v16, taps["t"] + tw.pos_rows(B), tw.ln_pre)
        gx, v16 = d, (vd + r16v(d) if var else None)
    tok = gx.view(B, T, W)[:, 1:]
    gp, vgp = _mm(tok, v16.view(B, T, W)[:, 1:] if var else None, tw.conv)
    return gx, v16, gp, (vgp + r16v(gp) if var else None)


# ------------------------------------------------------------------------------------------------ checks
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

    def finish(self):
        print(f"[vit tower] {self.label}\n" + "\n".join(self.lines))
        assert not self.bad, "\n".join(self.bad)


def _gemm_budget(a, w, y, out32):
    return C_GEMM * U * (a.abs() @ w.abs().T) + (2.0 ** -24 * y.abs() + FLOOR if out32 else U * (y.abs() + TINY))


def _ln_gemm(x, ln, w, b):
    """fp16(LN(x)) @ w^T + b and the tie term of the fp16 rounding of the LN output."""
    h, _, _, fmag = _ln(x, ln)
    h16 = h.float().half().double()
    delta = C_LN * U32 * fmag + FLOOR
    amb = ((h - delta).float().half() != (h + delta).float().half()).double()
    return h16, h16 @ w.T + b, (amb * (2 * U * h16.abs() + 2.0 ** -24)) @ w.abs().T


def _stream_round(y, stream32):
    """One rounding to the stream's type (after the fp32 sum the kernel forms first)."""
    return 2.0 ** -24 * y.abs() + FLOOR + (0 if stream32 else U * (y.abs() + TINY))


def check_forward(rep, tw, tp, *, B, cls_only, stream32, fused):
    T, W, H, L = tw.T, tw.W, tw.H, tw.L
    cls = torch.arange(B) * T
    # stem: t = patches conv1^T (+ bias), class rows the class embedding; x0 = ln_pre(t + pos) or t + pos
    pt = tp["patches"].reshape(B * tw.np, tw.Kp)
    ref = pt @ tw.conv.T + (0 if tw.conv_b is None else tw.conv_b)
    t = tp["t"].view(B, T, W)
    rep.check("t (patch rows)", t[:, 1:].reshape(-1, W), ref, _gemm_budget(pt, tw.conv, ref, True))
    assert torch.equal(t[:, 0], tw.cls.float().double().expand(B, W)), "t: class rows are not the class embedding"
    xin = tp["t"] + tw.pos_rows(B)
    if tw.ln_pre is not None:
        y, _, _, fmag = _ln(xin, tw.ln_pre)
        rep.check("x0 = ln_pre(t + pos)", tp["x0"], y, C_LN * (U32 if stream32 else U) * fmag + FLOOR)
    else:
        rep.check("x0 = t + pos", tp["x0"], xin, _stream_round(xin, stream32))
    ldT = _round_up(T, 8)
    for l, ly in enumerate(tw.layers):
        tail = cls if cls_only and l == L - 1 else torch.arange(B * T)
        x = tp[f"x{l}"]
        h16, ref, tie = _ln_gemm(x, ly.ln1, ly.wqkv, ly.bqkv)
        rep.check(f"qkv{l}", tp[f"qkv{l}"], ref, _gemm_budget(h16, ly.wqkv, ref, False) + tie)
        qkv = tp[f"qkv{l}"]
        if fused:
            r, mag = _reference(qkv, None, B, T, H, SCALE)
            rep.check(f"o{l}", _split(tp[f"o{l}"], B, T, H)[0], r["o"], C_BUDGET * U * mag["o"] + FLOOR)
            o, o_err = tp[f"o{l}"], 0
        else:
            x3 = _split(qkv, B, T, H)
            q, k, v = x3[0], x3[1], x3[2]
            s = (q @ k.transpose(-1, -2)) * SCALE
            e = U * (s.abs() + TINY) + C_GEMM * U * SCALE * (q.abs() @ k.abs().transpose(-1, -2))
            p = torch.softmax(s, -1)
            bud = p * (e + (p * e).sum(-1, keepdim=True)) + U * (p + TINY) + 2.0 ** -20 * p
            P = tp[f"P{l}"]
            rep.check(f"P{l}", P[..., :T], p, bud)
            assert torch.equal(P[..., T:], torch.zeros_like(P[..., T:])), f"P{l}: pad columns are not 0"
            P16 = P[..., :T]
            o4 = P16 @ v   # the engine's O = P V from its own fp16 P, rounded to fp16
            o = _merge(o4[None], B, T)
            o_err = _merge((U * (o4.abs() + TINY) + C_GEMM * U * (P16 @ v.abs()))[None], B, T)
        xm = x[tail] + o[tail] @ ly.wo.T + ly.bo
        bud = C_GEMM * U * (o[tail].abs() @ ly.wo.abs().T) + _stream_round(xm, stream32)
        if not fused:
            bud = bud + o_err[tail] @ ly.wo.abs().T
        rep.check(f"x_mid{l}", tp[f"x_mid{l}"][tail], xm, bud)
        h16, ref, tie = _ln_gemm(tp[f"x_mid{l}"][tail], ly.ln2, ly.wfc, ly.bfc)
        u16 = tp[f"u{l}"][:len(tail)]
        rep.check(f"u{l}", u16, ref, _gemm_budget(h16, ly.wfc, ref, False) + tie)
        a, da = tw.act(u16)
        xn = tp[f"x_mid{l}"][tail] + a @ ly.wproj.T + ly.bproj
        act_err = U * (da.abs() * (u16.abs() + TINY) + a.abs() + TINY)
        bud = (C_GEMM * U * (a.abs() @ ly.wproj.abs().T) + act_err @ ly.wproj.abs().T + _stream_round(xn, stream32))
        rep.check(f"x{l + 1}", tp[f"x{l + 1}"][tail], xn, bud)
    hc, _, _, fmag = _ln(tp[f"x{L}"][cls], tw.ln_post)
    rep.check("hcls = ln_post(x_out class rows)", tp["hcls"], hc, C_LN * U * fmag + FLOOR)
    ref = tp["hcls"] @ tw.proj
    rep.check("e = hcls proj", tp["e"], ref, _gemm_budget(tp["hcls"], tw.proj.T, ref, True))


def check_backward_elementwise(rep, tw, tp, *, B, cls_only, stream32, fused):
    gx, v16, gp, vgp = vjp(tw, tp, tp["de16"], cls_only=cls_only, stream32=stream32, fused=fused)
    rep.check("gx16 = d/dt (x4096)", tp["gx16"], gx, K_SIGMA * v16.sqrt() + FLOOR)
    g_eng = tp["g_patches"]
    rep.check("g_patches (x4096), chain", g_eng, gp, K_SIGMA * vgp.sqrt() + FLOOR)
    tok = tp["gx16"].view(B, tw.T, tw.W)[:, 1:]
    ref = tok @ tw.conv
    rep.check("g_patches from the engine's gx16", g_eng, ref, _gemm_budget(tok, tw.conv.T, ref, False))


def rel_l2_cos(got, ref):
    a, b = got.flatten(), ref.flatten()
    return ((a - b).norm() / b.norm()).item(), (a @ b / (a.norm() * b.norm())).item()


# ------------------------------------------------------------------------------------------------ engine runs
def _env(monkeypatch, settings):
    for k in ("PXR_FUSED_ATTN", "PXR_CLIP_STREAM", "PXR_CLIP_LAST_CLS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in settings.items():
        monkeypatch.setenv(k, v)


def _state_dict(arch, seed, outliers):
    timm = arch.get("tower") == E.TOWER_TIMM_VIT
    sd = S.slip_state_dict(arch, seed) if timm else S.clip_state_dict(arch, seed)
    if outliers:  # two residual-stream channels of a few hundred from layer 0 on
        key = "visual.blocks.0.mlp.fc2.bias" if timm else "visual.transformer.resblocks.0.mlp.c_proj.bias"
        sd[key][7] += 300.0
        sd[key][100] -= 200.0
    return sd


def run_engine(arch, settings, monkeypatch, seed, cutn=3, outliers=False):
    """The tower's taps after make_cutouts -> encode_image -> backward, in float64 on the CPU."""
    _env(monkeypatch, settings)
    sd = _state_dict(arch, seed, outliers)
    tw = Tower(arch, sd)
    W, H, L, T, D = tw.W, tw.H, tw.L, tw.T, tw.D
    M = cutn * T
    stream32 = settings.get("PXR_CLIP_STREAM") == "32"
    fused = T <= 240 and settings.get("PXR_FUSED_ATTN", "1") != "0"
    xdt = torch.float32 if stream32 else torch.half
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(16, 16), cutn=cutn, clip=[arch], seed=seed)
    try:
        eng.load_module(E.MOD_CLIP0, sd)
        eng.finalize()
        pm = S.prompts(D, (1.0, -0.3), seed)
        eng.set_prompts(0, torch.cat([p[0] for p in pm]).numpy(), [p[1] for p in pm], [p[2] for p in pm])
        g = torch.Generator().manual_seed(seed)
        img = eng.synth(torch.rand(eng.z_shape, generator=g))
        facs, noise = torch.rand(cutn, generator=g) * 0.1, torch.randn(cutn, 3, 224, 224, generator=g)
        eng.make_cutouts(img, transforms=random_transforms(cutn, 224, seed), zoom_padding=E.PAD_REFLECTION, fill=0.4,
                         noise_facs=facs.numpy(), noise=noise)
        eng.encode_image(0)
        eng.backward()

        def rd(name, shape, dtype=torch.half):
            return eng.debug_read(f"clip0.{name}", shape, dtype).double().cpu()

        tp = dict(patches=rd("patches", (cutn, tw.np, tw.Kp)), t=rd("t", (M, W), torch.float32),
                  hcls=rd("hcls", (cutn, W)), e=rd("e", (cutn, D), torch.float32), de16=rd("de16", (cutn, D)),
                  gx16=rd("gx16", (M, W)), g_patches=rd("g_patches", (cutn, tw.np, tw.Kp)))
        for l in range(L + 1):
            tp[f"x{l}"] = rd(f"x{l}", (M, W), xdt)
        for l in range(L):
            tp[f"x_mid{l}"] = rd(f"x_mid{l}", (M, W), xdt)
            tp[f"qkv{l}"] = rd(f"qkv{l}", (M, 3 * W))
            tp[f"u{l}"] = rd(f"u{l}", (M, 4 * W))
            if fused:
                tp[f"o{l}"] = rd(f"o{l}", (M, W))
            else:
                tp[f"P{l}"] = rd(f"P{l}", (cutn, H, T, _round_up(T, 8)))
        assert torch.equal(rd(f"x{L}", (M, W), xdt), rd("x_out", (M, W), xdt))
    finally:
        eng.close()
    return tw, tp, dict(B=cutn, cls_only=settings.get("PXR_CLIP_LAST_CLS", "1") != "0", stream32=stream32, fused=fused)


B32, B16, L14 = E.CLIP_ARCH["ViT-B/32"], E.CLIP_ARCH["ViT-B/16"], E.CLIP_ARCH["ViT-L/14"]
SB16, SL16 = E.SLIP_ARCH["SLIP_VITB16"], E.SLIP_ARCH["SLIP_VITL16"]
F32, UNFUSED, ALL_ROWS = {"PXR_CLIP_STREAM": "32"}, {"PXR_FUSED_ATTN": "0"}, {"PXR_CLIP_LAST_CLS": "0"}

# full depth: forward step by step (a) and g_patches by norm (c)
FULL = {
    "ViT-B/32": (B32, {}),
    "ViT-B/32 row-softmax fp32-stream": (B32, {**UNFUSED, **F32}),
    "ViT-B/16 all-rows": (B16, ALL_ROWS),
    "SLIP_VITB16 fp32-stream": (SB16, F32),
    "ViT-L/14": (L14, {}),
    "SLIP_VITL16 all-rows": (SL16, ALL_ROWS),
}
SLOW = {"ViT-L/14", "SLIP_VITL16 all-rows"}

# two layers at full width, T and heads: forward (a) and backward per element (b)
TWO = {
    "ViT-B/32": (B32, {}),
    "ViT-B/32 row-softmax all-rows": (B32, {**UNFUSED, **ALL_ROWS}),
    "ViT-B/16 fp32-stream": (B16, F32),
    "ViT-L/14": (L14, {}),
    "SLIP_VITB16": (SB16, {}),
    "SLIP_VITL16 fp32-stream all-rows": (SL16, {**F32, **ALL_ROWS}),
}


def _params(cases):
    return [pytest.param(k, marks=[pytest.mark.slow] if k in SLOW else []) for k in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _params(FULL))
def test_full_depth_tower_step_by_step_and_gradient_norm(case, monkeypatch):
    arch, settings = FULL[case]
    tw, tp, kw = run_engine(arch, settings, monkeypatch, seed=11)
    rep = Report(f"{case} full depth")
    check_forward(rep, tw, tp, **kw)
    _, _, gp, _ = vjp(tw, tp, tp["de16"], cls_only=kw["cls_only"], stream32=kw["stream32"], fused=kw["fused"], var=False)
    rel, cos = rel_l2_cos(tp["g_patches"], gp)
    rep.lines.append(f"  g_patches vs float64 VJP: rel-L2 {rel:.3e} (bound {REL_L2_BOUND:.0e}), cosine {cos:.8f}")
    rep.finish()
    assert rel <= REL_L2_BOUND and cos >= COS_BOUND


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TWO))
def test_two_layer_tower_forward_and_backward_per_element(case, monkeypatch):
    arch, settings = TWO[case]
    tw, tp, kw = run_engine(dict(arch, layers=2), settings, monkeypatch, seed=13)
    rep = Report(f"{case} two layers")
    check_forward(rep, tw, tp, **kw)
    check_backward_elementwise(rep, tw, tp, **kw)
    rep.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("arch", [B32, SB16], ids=["ViT-B/32", "SLIP_VITB16"])
def test_residual_stream_outliers(arch, monkeypatch):
    tw, tp, kw = run_engine(dict(arch, layers=2), {}, monkeypatch, seed=17, outliers=True)
    peak = tp["x1"].abs().amax(0)
    assert peak[7] > 100 and peak[100] > 100, "the planted channels did not reach the stream"
    rep = Report(f"outliers {'timm' if tw.timm else 'openai'} two layers (stream peak {peak.max().item():.0f})")
    check_forward(rep, tw, tp, **kw)
    check_backward_elementwise(rep, tw, tp, **kw)
    for name in ("gx16", "g_patches"):
        m = tp[name].abs().max().item()
        rep.lines.append(f"  largest |4096 g| in {name}: {m:.1f} (fp16 limit {FP16_MAX:.0f})")
        assert torch.isfinite(tp[name]).all(), f"{name}: not finite"
    rep.finish()


# ------------------------------------------------------------------------------------------------ CPU tests
def _toy_patches(tw, B, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(B, tw.np, tw.Kp, dtype=torch.float64)
    p[..., :3 * tw.P ** 2] = torch.randn(B, tw.np, 3 * tw.P ** 2, generator=g, dtype=torch.float64)
    return p, torch.randn(B, tw.D, generator=g, dtype=torch.float64) * GRAD_SCALE * 1e-3


@pytest.mark.parametrize("timm", [False, True], ids=["openai", "timm"])
@pytest.mark.parametrize("cls_only", [True, False])
def test_reference_vjp_matches_the_oracle_module_autograd(timm, cls_only):
    """The float64 forward / VJP restated above against autograd through the oracle module itself."""
    arch = dict(width=128, layers=3, heads=2, patch=32, image_res=224, out_dim=64)
    if timm:
        arch["tower"] = E.TOWER_TIMM_VIT
    tw = Tower(arch, _state_dict(arch, 5, False))
    B, P, gp_ = 3, tw.P, 224 // tw.P
    patches, de = _toy_patches(tw, B, 6)
    taps = forward64(tw, patches, cls_only)
    img = patches[..., :3 * P * P].reshape(B, gp_, gp_, 3, P, P).permute(0, 3, 1, 4, 2, 5).reshape(B, 3, 224, 224)
    img = img.clone().requires_grad_(True)
    e = tw.model.encode_image(img)
    assert torch.allclose(e, taps["e"], rtol=1e-10, atol=1e-12)
    (e * de).sum().backward()
    gimg = img.grad.reshape(B, 3, gp_, P, gp_, P).permute(0, 2, 4, 1, 3, 5).reshape(B, tw.np, 3 * P * P)
    _, _, gp, _ = vjp(tw, taps, de, cls_only=cls_only, stream32=False, fused=True, var=False)
    assert torch.allclose(gp[..., :3 * P * P], gimg, rtol=1e-9, atol=1e-9 * gimg.abs().max().item())
    assert torch.equal(gp[..., 3 * P * P:], torch.zeros_like(gp[..., 3 * P * P:]))


def _mutated(arch, mutation, layer, var):
    tw = Tower(arch, _state_dict(arch, 11, False))
    patches, de = _toy_patches(tw, 3, 12)
    taps = forward64(tw, patches, cls_only=True)
    kw = dict(cls_only=True, stream32=False, fused=True)
    ref = vjp(tw, taps, de, var=var, **kw)
    mut = vjp(tw, taps, de, var=False, mutate=mutation, mutate_layer=layer, **kw)
    return ref, mut


def test_dropped_head_gradient_exceeds_the_full_depth_bound_tenfold():
    """One head's dV dropped in layer 6 of the float64 reference of full-depth ViT-B/32 moves g_patches by at least ten
    times the full-depth rel-L2 bound."""
    (_, _, ref, _), (_, _, mut, _) = _mutated(B32, "dv_head", 6, False)
    rel, cos = rel_l2_cos(mut, ref)
    print(f"[vit tower] dV of one head dropped in layer 6: rel-L2 change {rel:.3e}, cosine {cos:.8f}")
    assert rel >= 10 * REL_L2_BOUND and cos < COS_BOUND


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("mutation,least", [("dv_head", 10.0), ("ln_mean", 1.5)])
def test_mutations_exceed_the_two_layer_element_budgets(mutation, least, layer):
    """A two-layer ViT-B/32 reference with one head's dV dropped, or with the mean term of ln_1's backward dropped, in
    layer 0 (a full layer) or layer 1 (the class-rows tail) leaves elements of gx16 and g_patches outside their budgets
    by the factor `least`."""
    (gx, v16, gp, vgp), (mx, _, mp, _) = _mutated(dict(B32, layers=2), mutation, layer, True)
    r = ((mx - gx).abs() / (K_SIGMA * v16.sqrt() + FLOOR)).max().item()
    r2 = ((mp - gp).abs() / (K_SIGMA * vgp.sqrt() + FLOOR)).max().item()
    print(f"[vit tower] {mutation} in layer {layer}: largest change / budget {r:.2f} in gx16, {r2:.2f} in g_patches")
    assert r >= least and r2 >= least
