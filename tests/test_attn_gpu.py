"""Fused tensor-core attention (pixray_b200/csrc/attn_tc.cu) against a float64 restatement of nn.MultiheadAttention's
core (SLIP/models.py:18-64 residual blocks call it with need_weights=False): S = scale q k^T, P = softmax(S), O = P v,
and its backward, computed on the CPU from the same fp16 qkv / dO the kernel reads.

Every output element has its own error budget (u = 2^-11, the fp16 unit roundoff; P the float64 probabilities; every
|.| product in float64; c = 4):
  o    c u (P |V|) + 2^-24                 dv   c u (P^T |dO|) + 2^-24
  dq   c u scale (M |K|) + 2^-24           dk   c u scale (M^T |Q|) + 2^-24
  lse  2^-16 (1 + scale max_j sum_d |q_id| |k_jd|)
with M = P o (|dO| |V|^T + (|dO| . |O|) 1^T), which bounds the fp16 rounding of dS = P o (dP - D) (D = dO . O is
formed from the fp16 O the forward stored).  P and dS enter the MMAs as fp16, whose rounding error below the smallest
normal 2^-14 is an absolute 2^-25 = u 2^-14 rather than u relative: wherever P or dS is rounded to fp16, the budget
uses P + 2^-14 and M + 2^-14 (on rows of near-one-hot P, most of P is subnormal in fp16).
Every case prints the largest err / (u magnitude) of each output; with PXR_ATTN_TEST_LOG set to a file path, these
lines (and the throughput report) are also appended to that file."""
import ctypes as C
import os

import pytest
import torch

from pixray_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -11
C_BUDGET = 4.0
FLOOR = 2.0 ** -24
TINY = 2.0 ** -14    # smallest normal fp16: below it an fp16 value is rounded to 2^-25 = u TINY absolute, not u relative
GUARD = 64           # sentinel rows before and after every output
SENTINEL = 1234.0    # exact in fp16 and fp32


def _log(lines):
    """Print the report lines, and append them to the file PXR_ATTN_TEST_LOG names, if set."""
    text = "\n".join(lines)
    print(text)
    path = os.environ.get("PXR_ATTN_TEST_LOG")
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "a") as f:
            f.write(text + "\n")


def _guarded(rows, cols, dtype):
    """[GUARD + rows + GUARD, cols] buffer: guards hold SENTINEL, the interior NaN (every element must be written)."""
    buf = torch.full((rows + 2 * GUARD, cols), SENTINEL, dtype=dtype, device="cuda")
    buf[GUARD:GUARD + rows] = float("nan")
    return buf


def _run(qkv, d_o, B, T, H, scale, repeat=1, check=True):
    lib = _lib.load()
    W = 64 * H
    o_buf = _guarded(B * T, W, torch.half)
    lse_buf = _guarded(B * H * T, 1, torch.float32)
    g_buf = _guarded(B * T, 3 * W, torch.half) if d_o is not None else None
    o, lse = o_buf[GUARD:-GUARD], lse_buf[GUARD:-GUARD, 0]
    gqkv = g_buf[GUARD:-GUARD] if g_buf is not None else None
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_attention(C.c_void_p(qkv.data_ptr()), C.c_void_p(o.data_ptr()), C.c_void_p(lse.data_ptr()),
                                C.c_void_p(d_o.data_ptr()) if d_o is not None else None,
                                C.c_void_p(gqkv.data_ptr()) if gqkv is not None else None, B, T, H, W,
                                C.c_float(scale), repeat, err, 512)
    assert rc == 0, err.value.decode()
    torch.cuda.synchronize()
    for name, buf in (("o", o_buf), ("lse", lse_buf), ("gqkv", g_buf)):
        if buf is None or not check:
            continue
        assert (buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all(), f"{name}: write outside the tensor"
        assert not torch.isnan(buf[GUARD:-GUARD]).any(), f"{name}: element left unwritten (or NaN)"
    return o, lse, gqkv


def _split(t, B, T, H, d=64):
    """[B*T, n*d*H] -> [n, B, H, T, d]"""
    n = t.shape[1] // (d * H)
    return t.reshape(B, T, n, H, d).permute(2, 0, 3, 1, 4)


def _reference(qkv, d_o, B, T, H, scale, d=64, causal=False, device="cpu"):
    """float64 outputs and per-element magnitudes, all [B, H, T, d] (lse [B, H, T]), on `device`.  causal: row t
    attends to keys <= t (the forward only)."""
    x = _split(qkv.to(device).double(), B, T, H, d)
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * scale
    keep = torch.ones(T, T, dtype=torch.bool, device=device).tril() if causal else None
    if causal:
        s = s.masked_fill(~keep, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    ref = dict(o=o, lse=lse)
    pf = p + (TINY * keep if causal else TINY)  # P as an fp16 MMA operand (masked keys take no part)
    sa = q.abs() @ k.abs().transpose(-1, -2)
    mag = dict(o=pf @ v.abs(), lse=1 + scale * (sa.masked_fill(~keep, 0) if causal else sa).amax(-1))
    if d_o is not None:
        g = _split(d_o.to(device).double(), B, T, H, d)[0]
        dp = g @ v.transpose(-1, -2)
        ds = p * (dp - (g * o).sum(-1, keepdim=True))
        ref.update(dq=scale * ds @ k, dk=scale * ds.transpose(-1, -2) @ q, dv=p.transpose(-1, -2) @ g)
        m = p * (g.abs() @ v.abs().transpose(-1, -2) + (g.abs() * o.abs()).sum(-1, keepdim=True)) + TINY
        mag.update(dq=scale * m @ k.abs(), dk=scale * m.transpose(-1, -2) @ q.abs(), dv=pf.transpose(-1, -2) @ g.abs())
    return ref, mag


def _check(label, o, lse, gqkv, ref, mag, B, T, H):
    """Asserts every element within its budget; logs the largest err / (u magnitude) per output."""
    got = dict(o=_split(o.cpu().double(), B, T, H)[0], lse=lse.cpu().double().reshape(B, H, T))
    if gqkv is not None:
        gq = _split(gqkv.cpu().double(), B, T, H)
        got.update(dq=gq[0], dk=gq[1], dv=gq[2])
    line, bad = [label], []
    for name in ("o", "lse", "dq", "dk", "dv"):
        if name not in got:
            continue
        err = (got[name] - ref[name]).abs()
        if name == "lse":
            bound = 2.0 ** -16 * mag[name]
            ratio = (err / bound).max().item()
            line.append(f"lse err/bound {ratio:.3f}")
        else:
            bound = C_BUDGET * U * mag[name] + FLOOR
            excess = (err - FLOOR).clamp_min(0)
            ratio = (excess / (U * mag[name])).nan_to_num(0.0, posinf=float("inf")).max().item()
            line.append(f"{name} err/(u mag) {ratio:.3f}")
        over = err > bound
        if over.any():
            i = over.nonzero()[0].tolist()
            bad.append(f"{name}: {int(over.sum())} elements over budget, first at {i}: got {got[name][tuple(i)].item():.6e} "
                       f"ref {ref[name][tuple(i)].item():.6e} bound {bound[tuple(i)].item():.3e}")
    _log(["  ".join(line)])
    assert not bad, "\n".join(bad)


def _inputs(B, T, H, seed, qkv_std=1.5, d=64):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = d * H
    qkv = (torch.randn(B * T, 3 * W, generator=g, device="cuda") * qkv_std).half()
    d_o = torch.randn(B * T, W, generator=g, device="cuda").half()
    return qkv, d_o


def _case(label, qkv, d_o, B, T, H, scale):
    o, lse, gqkv = _run(qkv, d_o, B, T, H, scale)
    ref, mag = _reference(qkv, d_o, B, T, H, scale)
    _check(label, o, lse, gqkv, ref, mag, B, T, H)
    return o, lse, gqkv


@pytest.mark.parametrize("B,T,H", [(2, 197, 12), (3, 50, 4), (1, 240, 2), (2, 130, 3), (5, 64, 2), (1, 16, 1), (150, 197, 1),
                                   # many (image, head) pairs, one per CTA (ViT-B/32 with many cutouts)
                                   (40, 50, 12), (13, 128, 12)])
def test_attention_matches_torch(B, T, H):
    qkv, d_o = _inputs(B, T, H, B * 1000 + T)
    _case(f"B={B} T={T} H={H} scale=0.125", qkv, d_o, B, T, H, 0.125)


# the edges of the 64-row query / key blocks, and the production sequence lengths (ViT-B/32, ViT-B/16, vdiff 4^2 / 8^2)
@pytest.mark.parametrize("T", [1, 2, 8, 63, 64, 65, 127, 128, 129, 191, 192, 193, 239, 240, 50, 197, 16])
@pytest.mark.parametrize("B,H", [(1, 1), (1, 12), (3, 1), (3, 12)])
def test_attention_block_edges(T, B, H):
    qkv, d_o = _inputs(B, T, H, 7 * T + B + H)
    _case(f"edges B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("scale", [1.0, 0.03])
@pytest.mark.parametrize("B,T,H", [(2, 197, 12), (3, 50, 4), (1, 240, 2), (2, 65, 1)])
def test_attention_any_scale(B, T, H, scale):
    qkv, d_o = _inputs(B, T, H, 31 * T + H)
    _case(f"B={B} T={T} H={H} scale={scale}", qkv, d_o, B, T, H, scale)


def _peaked(B, T, H, target, seed, d=64, scale=0.125):
    """Every query's largest score is at key `target` (per head), about 8 above the rest: P ~ 0.94 there."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = d * H
    qkv = torch.randn(B * T, 3 * W, generator=g, device="cuda") * 0.5
    x = qkv.view(B, T, 3, H, d)
    x[:, :, 0, :, 0] = 4.0
    x[:, :, 1, :, 0] = 0.5 * torch.randn(B, T, H, generator=g, device="cuda")
    x[:, target, 1, :, 0] = 2.0 / scale
    return qkv.half(), torch.randn(B * T, W, generator=g, device="cuda").half()


@pytest.mark.parametrize("T", [129, 197, 240])
@pytest.mark.parametrize("where", ["first", "last"])
def test_attention_row_max_in_first_or_last_key_block(T, where):
    """The online softmax meets the row maximum in its first key block (never rescales) or in its last (rescales the
    whole running sum and output at the end)."""
    B, H = 2, 3
    target = 0 if where == "first" else T - 1
    qkv, d_o = _peaked(B, T, H, target, T)
    _case(f"row max in the {where} key block B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("T", [50, 197])
def test_attention_near_one_hot_rows(T):
    """Scores spanning about +-80: most rows put nearly all their weight on one key."""
    B, H = 2, 4
    qkv, d_o = _inputs(B, T, H, 5 + T, qkv_std=5.0)
    _case(f"near one-hot B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("T", [1, 65, 197])
def test_attention_tied_scores(T):
    """Identical K rows: every score of a row ties, P is uniform and O is the mean of V."""
    B, H = 2, 2
    W = 64 * H
    qkv, d_o = _inputs(B, T, H, 77 + T)
    qkv.view(B, T, 3, W)[:, :, 1] = qkv.view(B, T, 3, W)[:, :1, 1]
    _case(f"tied scores B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("B,T,H", [(3, 50, 12), (2, 197, 12), (4, 65, 2)])
def test_attention_class_row_gradient(B, T, H):
    """dO zero except on the class row (row 0) of each image -- what the last layer's class-token restriction hands
    the attention.  dq of every other row is exactly 0 (P (0 - 0)); dk and dv still meet their budgets."""
    qkv, d_o = _inputs(B, T, H, 3 * T + B)
    d_o.view(B, T, -1)[:, 1:] = 0
    _, _, gqkv = _case(f"class-row dO B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)
    W = 64 * H
    dq_rest = gqkv.view(B, T, 3 * W)[:, 1:, :W]
    assert torch.equal(dq_rest, torch.zeros_like(dq_rest))


@pytest.mark.parametrize("g_scale", [4096.0, 2.0 ** -8])
def test_attention_gradient_dynamic_range(g_scale):
    """dO at the engine's loss scale (4096) and at 2^-8: dS must neither overflow nor underflow in fp16."""
    B, T, H = 2, 197, 12
    qkv, d_o = _inputs(B, T, H, 11)
    d_o = (d_o.float() * g_scale).half()
    _case(f"dO x {g_scale} B={B} T={T} H={H}", qkv, d_o, B, T, H, 0.125)


@pytest.mark.parametrize("B,T,H", [(3, 197, 12), (2, 65, 2), (40, 50, 12)])
def test_attention_is_deterministic(B, T, H):
    """One writer per output element: two calls give the same bits, and the forward alone gives the same o / lse as
    the forward of a forward + backward call."""
    qkv, d_o = _inputs(B, T, H, 123 + T)
    o1, l1, g1 = _run(qkv, d_o, B, T, H, 0.125)
    o2, l2, g2 = _run(qkv, d_o, B, T, H, 0.125)
    o3, l3, _ = _run(qkv, None, B, T, H, 0.125)
    assert torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(g1, g2)
    assert torch.equal(o1, o3) and torch.equal(l1, l3)


def test_attention_throughput_report():
    """Config-2 shape (64 images x 12 heads x 197 tokens): time per call, reported (not asserted)."""
    B, T, H = 64, 197, 12
    W = 64 * H
    qkv = torch.randn(B * T, 3 * W, device="cuda").half()
    d_o = torch.randn(B * T, W, device="cuda").half()
    _run(qkv, None, B, T, H, 0.125, repeat=3)
    _run(qkv, d_o, B, T, H, 0.125, repeat=3)
    lines = []
    for name, g in (("fwd", None), ("fwd+bwd", d_o)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        _run(qkv, g, B, T, H, 0.125, repeat=20, check=False)
        e1.record()
        torch.cuda.synchronize()
        lines.append(f"attention {name} B={B} T={T} H={H}: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us per call")
    _log(lines)
