"""Every plain GEMM plan the engine builds, replayed against float64 with the engine's own operand layouts.

The ViT / text / ResNet linear layers and their dgrads, the batched attention chain, the VQ score GEMM and the U-Net's
tiny-level GEMMs all go through `add_gemm` / `add_gemm_splitk`, which record each plan: both operands as planned (mode,
pitch, extents, batch strides), M / N / K, the whole epilogue and the plan's choices (pxr_test_gemm_records).  The engine
also reports its device allocations (pxr_test_allocations).  These tests build each engine at real widths (finalize()
makes the plans; nothing runs) and check

- footprint, statically: every range a plan addresses lies inside one allocation, at most one operand reads past K, and
  the pad columns a tensor-map store may write past a ragged N belong to no other plan's data;
- routing: what the wide kernel and split-K may combine, and that each engine still reaches the plan kinds it is here for;
- replay: each distinct plan, rebuilt by the test hook from the record (the hook must report the engine's own choices), on
  random fp16 operands whose elements inside the extents but past M / N / K are +-1e4 and whose pitch padding is NaN,
  against float64: |err| <= 2^-11 |ref| + 2^-16 S for fp16 outputs, 2^-22 |ref| + 2^-16 S for fp32 ones
  (S = |alpha| sum |a||b| + |bias| + |res|), activations against float64 of the activation of the kernel's own saved
  pre-activation with constants derived from the code below; canaries untouched, two runs bit-identical;
- the VQ score plan against the bound vq_select relies on;
- that the bound rejects a dropped k-block, a batch slice read from its neighbour and a ragged last column taken from
  another column (CPU).
"""
import bisect
import ctypes as C
import math
import os
import re

import pytest
import torch

from pixray_b200 import _lib
from pixray_b200 import engine as E
from pixray_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OP_K, OP_MN = 0, 1
ACT_NONE, ACT_QG, ACT_QG_BWD, ACT_GELU, ACT_GELU_BWD, ACT_RELU, ACT_RELU_BWD = 0, 1, 2, 6, 7, 8, 9
TE_NONE, TE_GELU, TE_GELU_BWD = 0, 2, 3
REL16, REL32, ABS = 2.0 ** -11, 2.0 ** -22, 2.0 ** -16
BIG = 1.0e4
CANARY = -7.0
SMALL_CLIP = dict(width=128, layers=2, heads=2, patch=32, image_res=224, out_dim=64)


# ------------------------------------------------------------------------------------------------------- the hooks
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def gemm_records(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_gemm_records(eng.h, None, 0, C.byref(n)), "pxr_test_gemm_records")
    recs = (_lib.TestGemmRec * n.value)()
    eng._check(lib.pxr_test_gemm_records(eng.h, recs, n.value, C.byref(n)), "pxr_test_gemm_records")
    return list(recs)


def allocations(eng):
    lib, n = _lib.load(), C.c_int()
    eng._check(lib.pxr_test_allocations(eng.h, None, None, 0, C.byref(n)), "pxr_test_allocations")
    ptrs, sizes = (C.c_void_p * n.value)(), (C.c_longlong * n.value)()
    eng._check(lib.pxr_test_allocations(eng.h, ptrs, sizes, n.value, C.byref(n)), "pxr_test_allocations")
    return sorted((p, s) for p, s in zip(ptrs, sizes))


# ------------------------------------------------------------------------------------------------------- engines
# the engine's A/B switches that change which GEMMs it plans: every engine starts from their defaults, whatever the
# caller's environment holds, and sets only the ones it names
SWITCHES = ("PXR_FUSED_ATTN", "PXR_CLIP_STREAM", "PXR_CLIP_LAST_CLS", "PXR_CONV_SPLITK", "PXR_GEMM_BN", "PXR_GEMM_TMA_EPI",
            "PXR_VQ_TC")


def _with_env(env, make):
    old = {k: os.environ.get(k) for k in SWITCHES + tuple(env)}
    for k in SWITCHES:
        os.environ.pop(k, None)
    os.environ.update(env)
    try:
        eng = make()
        eng.finalize()
        return eng
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _vit(arch, cutn, sd, text=None):
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=cutn, cut_size=arch["image_res"],
                       clip=[arch], seed=0)
    eng.load_module(E.MOD_CLIP0, {**sd, **(text or {})})
    return eng


def _vitb32():
    arch = dict(E.CLIP_ARCH["ViT-B/32"], layers=2)
    return _vit(arch, 32, S.clip_state_dict(arch, 0), S.clip_text_state_dict(512, 2, 512, 1))


def _vitb32_chain():
    arch = dict(E.CLIP_ARCH["ViT-B/32"], layers=2)
    return _vit(arch, 32, S.clip_state_dict(arch, 0))


def _slip():
    arch = dict(E.SLIP_ARCH["SLIP_VITB16"], layers=2)
    return _vit(arch, 8, S.slip_state_dict(arch, 0))


def _vitl14():
    arch = dict(E.CLIP_ARCH["ViT-L/14"], layers=2)
    return _vit(arch, 8, S.clip_state_dict(arch, 0))


def _resnet():
    arch = E.RESNET_ARCH["RN50x4"]
    eng = E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(48, 48), grid=(16, 16), cutn=4, cut_size=arch["image_res"],
                       clip=[arch], seed=0)
    eng.load_module(E.MOD_CLIP0, S.clip_resnet_state_dict(arch, 0))
    return eng


def _vdiff():
    eng = E.B200Engine(drawer=E.DRAWER_VDIFF, image_hw=(256, 256), cutn=8, clip=[SMALL_CLIP], seed=0)
    eng.load_module(E.MOD_VQGAN, S.vdiff_state_dict(0, c=128))
    eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
    return eng


def _vqgan(hw):
    def make():
        eng = E.B200Engine(drawer=E.DRAWER_VQGAN, image_hw=hw, vqgan=E.VQGAN_F16_16384, cutn=8, clip=[SMALL_CLIP], seed=0)
        eng.load_module(E.MOD_VQGAN, S.vqgan_state_dict(E.VQGAN_F16_16384, 0, with_encoder=True))
        eng.load_module(E.MOD_CLIP0, S.clip_state_dict(SMALL_CLIP, 1))
        return eng
    return make


# name: (constructor, environment, the plan kinds the engine must reach)
ENGINES = {
    "vitb32": (_vitb32, {}, {"wide192", "wide256", "act1", "act2", "te_act1", "te_act2", "res16", "batchedA", "cls_rows",
                             "o32", "mnB", "text77"}),
    "vitb32_stream32_chain": (_vitb32_chain, {"PXR_CLIP_STREAM": "32", "PXR_FUSED_ATTN": "0"},
                              {"res32", "batched_both", "mnA", "chain50", "ragged"}),
    "slipb16_chain": (_slip, {"PXR_FUSED_ATTN": "0"}, {"act6", "act7", "te_act6", "te_act7", "batched_both", "chain197",
                                                       "ragged"}),
    "vitl14": (_vitl14, {}, {"batched_both", "mnA", "chain257", "ragged"}),
    "rn50x4": (_resnet, {}, {"act8", "act9", "res16", "mnB", "o32", "cls_rows"}),
    "vdiff256": (_vdiff, {}, {"splitk", "splitk_bias", "batched_both", "chain256", "mnB"}),
    "vqgan256": (_vqgan((256, 256)), {}, {"chain256", "mnA", "o32", "vq_score"}),
    "vqgan288x432": (_vqgan((288, 432)), {}, {"chain486", "mnA", "vq_score", "ragged"}),
}
SLOW = {"vqgan288x432"}


class Built:
    def __init__(self, name):
        self.name = name
        make, env, self.expect = ENGINES[name]
        self.eng = _with_env(env, make)
        self.recs = gemm_records(self.eng)
        self.allocs = allocations(self.eng)
        self.starts = [a for a, _ in self.allocs]

    def alloc_of(self, lo, hi):
        """The allocation holding the byte range [lo, hi), or None."""
        i = bisect.bisect_right(self.starts, lo) - 1
        if i < 0:
            return None
        a, n = self.allocs[i]
        return (a, n) if hi <= a + n else None

    def close(self):
        self.eng.close()


def _params():
    return [pytest.param(n, marks=[pytest.mark.gpu] + ([pytest.mark.slow] if n in SLOW else [])) for n in ENGINES]


@pytest.fixture(scope="module", params=_params())
def built(request):
    b = Built(request.param)
    yield b
    b.close()


def _name(b, r):
    return f"{b.name}: {r.label.decode()}"


# ------------------------------------------------------------------------------------------------------- geometry
def operands(r):
    """(name, ptr, mode, ld, mn_extent, k_extent, (nb0, bs0), (nb1, bs1), rows used, 2 bytes) of A and B."""
    return [("A", r.a, r.a_mode, r.lda, r.a_mn_extent, r.a_k_extent, (r.a_nb0, r.a_bs0), (r.a_nb1, r.a_bs1), r.M),
            ("B", r.b, r.b_mode, r.ldb, r.b_mn_extent, r.b_k_extent, (r.b_nb0, r.b_bs0), (r.b_nb1, r.b_bs1), r.N)]


def op_span(mode, ld, mn, k, nb0, bs0, nb1, bs1):
    """Elements from the operand's pointer to one past the last element its extents address."""
    inner = (k - 1) * ld + mn if mode == OP_MN else (mn - 1) * ld + k
    return (nb1 - 1) * bs1 + (nb0 - 1) * bs0 + inner


def epilogue_tensors(r):
    """(name, ptr, bytes per element, ldc, bs0, bs1, nb0, nb1, rows, cols, written) of every epilogue tensor, the split-K
    reduce's included."""
    nb0, nb1 = r.a_nb0, r.a_nb1
    t = []
    split = r.k_splits > 1
    for name, ptr, eb, written in (("out_f16", r.out_f16, 2, True), ("out_f32", r.out_f32, 4, True),
                                   ("aux_out", r.aux_out, 2, True), ("aux_in", r.aux_in, 2, False),
                                   ("res_f16", r.res_f16, 2, False), ("res_f32", r.res_f32, 4, False)):
        if ptr:
            if split and name == "out_f32":  # the partial-sum slabs [k_splits][M][ldc]
                t.append((name, ptr, eb, r.ldc, r.M * r.ldc, 0, r.k_splits, 1, r.M, r.N, True))
            else:
                t.append((name, ptr, eb, r.ldc, r.c_bs0, r.c_bs1, nb0, nb1, r.M, r.N, written))
    if split:
        t.append(("red_out", r.red_out, 2, r.ld_out, 0, 0, 1, 1, r.M, r.N, True))
        if r.red_res:
            t.append(("red_res", r.red_res, 2, r.ld_out, 0, 0, 1, 1, r.M, r.N, False))
    return t


def _intervals(ptr, eb, ld, bs0, bs1, nb0, nb1, rows, c0, c1):
    """Byte intervals [lo, hi) of columns [c0, c1) of every row of every batch."""
    b0 = torch.arange(nb0, dtype=torch.int64) * bs0
    b1 = torch.arange(nb1, dtype=torch.int64) * bs1
    rr = torch.arange(rows, dtype=torch.int64) * ld
    lo = (b1.view(-1, 1, 1) + b0.view(1, -1, 1) + rr.view(1, 1, -1)).flatten() + c0
    return ptr + lo * eb, ptr + (lo + (c1 - c0)) * eb


def _valid_intervals(r):
    """Byte intervals of the data every part of plan r reads or writes inside M x N x K (operands and epilogue)."""
    out = []
    for _, ptr, mode, ld, _, _, (nb0, bs0), (nb1, bs1), used in operands(r):
        if mode == OP_MN:  # rows are k, columns the used mn
            out.append(_intervals(ptr, 2, ld, bs0 if nb0 > 1 else 0, bs1 if nb1 > 1 else 0, nb0, nb1, r.K, 0, used))
        else:
            out.append(_intervals(ptr, 2, ld, bs0 if nb0 > 1 else 0, bs1 if nb1 > 1 else 0, nb0, nb1, used, 0, r.K))
    for _, ptr, eb, ld, bs0, bs1, nb0, nb1, rows, cols, _ in epilogue_tensors(r):
        out.append(_intervals(ptr, eb, ld, bs0, bs1, nb0, nb1, rows, 0, cols))
    return out


class Cover:
    """Whether a byte lies in any of a set of intervals: max end over the intervals starting at or before it."""

    def __init__(self, ivs):
        lo = torch.cat([a for a, _ in ivs]) if ivs else torch.zeros(0, dtype=torch.int64)
        hi = torch.cat([b for _, b in ivs]) if ivs else torch.zeros(0, dtype=torch.int64)
        order = torch.argsort(lo)
        self.lo = lo[order]
        self.hi_max = torch.cummax(hi[order], 0).values if len(hi) else hi

    def hits(self, addr):
        i = torch.searchsorted(self.lo, addr, right=True) - 1
        ok = i >= 0
        return ok & (self.hi_max[i.clamp_min(0)] > addr)


# ------------------------------------------------------------------------------------------------------- footprint
def check_footprint(b, r, others=None):
    """Static: operands and epilogue tensors inside one allocation each, K covered by one side, pad columns private."""
    name = _name(b, r)
    for op, ptr, mode, ld, mn, k, (nb0, bs0), (nb1, bs1), used in operands(r):
        assert mn >= used and k >= 1 and ld >= (mn if mode == OP_MN else k), f"{name}: {op} extents {mn} x {k} at ld {ld}"
        span = op_span(mode, ld, mn, k, nb0, bs0, nb1, bs1)
        assert b.alloc_of(ptr, ptr + 2 * span), f"{name}: {op} [{ptr:#x}, +{2 * span}) lies in no allocation"
    assert min(r.a_k_extent, r.b_k_extent) == r.K, \
        f"{name}: k extents A {r.a_k_extent}, B {r.b_k_extent} for K = {r.K}: both sides read past K"
    for t, ptr, eb, ld, bs0, bs1, nb0, nb1, rows, cols, written in epilogue_tensors(r):
        gran = 16 // eb
        pad = -(-cols // gran) * gran if (written and r.tma_epi != TE_NONE) else cols
        assert ld >= pad, f"{name}: {t} pitch {ld} below {pad}"
        span = (nb1 - 1) * bs1 + (nb0 - 1) * bs0 + (rows - 1) * ld + pad
        assert b.alloc_of(ptr, ptr + eb * span), f"{name}: {t} [{ptr:#x}, +{eb * span}) lies in no allocation"
    return pad_is_private(b, r, others)


def pad_is_private(b, r, others):
    """Whether the columns [N, round_up(N, 16 bytes)) a tensor-map store may write hold no other plan's data."""
    if others is None or r.tma_epi == TE_NONE:
        return True
    for t, ptr, eb, ld, bs0, bs1, nb0, nb1, rows, cols, written in epilogue_tensors(r):
        gran = 16 // eb
        if not written or cols % gran == 0:
            continue
        lo, _ = _intervals(ptr, eb, ld, bs0, bs1, nb0, nb1, rows, cols, -(-cols // gran) * gran)
        addr = torch.cat([lo + eb * j for j in range(-(-cols // gran) * gran - cols)])
        if others.hits(addr).any():
            return False
    return True


def _others_cover(b, skip):
    return Cover([iv for i, q in enumerate(b.recs) if i != skip for iv in _valid_intervals(q)])


def test_footprint(built):
    b = built
    assert b.recs, "no GEMM plans recorded"
    ragged = [i for i, r in enumerate(b.recs) if r.tma_epi != TE_NONE and r.N % 8]
    for i, r in enumerate(b.recs):
        private = check_footprint(b, r, _others_cover(b, i) if i in ragged else None)
        assert private, f"{_name(b, r)}: the pad columns past N = {r.N} hold another plan's data"
    print(f"[gemm plans] {b.name}: {len(b.recs)} plans inside {len(b.allocs)} allocations, {len(ragged)} with a ragged "
          f"tensor-map store")


# ------------------------------------------------------------------------------------------------------- routing
def features(r):
    f = set()
    batched_a = r.a_nb0 * r.a_nb1 > 1
    batched_b = r.b_nb0 * r.b_nb1 > 1
    if batched_a and batched_b:
        f.add("batched_both")
    if batched_a and not batched_b:
        f.add("batchedA")
    if r.a_mode == OP_MN:
        f.add("mnA")
    if r.b_mode == OP_MN:
        f.add("mnB")
    if r.act:
        f.add(f"act{r.act}")
        if r.tma_epi != TE_NONE:
            f.add(f"te_act{r.act}")  # the activation on the tensor-map epilogue
    if r.res_f32:
        f.add("res32")
    if r.res_f16 or r.red_res:
        f.add("res16")
    if r.in_place:
        f.add("in_place")
    if r.wide:
        f.add(f"wide{r.block_n}")
    if r.k_splits > 1:
        f.add("splitk")
        if r.red_bias:
            f.add("splitk_bias")  # the reduce carries the bias
    if r.out_f32 and r.k_splits == 1:
        f.add("o32")
    if r.a_mode == OP_K and r.a_nb0 * r.a_nb1 == 1 and r.lda >= 16 * r.a_k_extent:
        f.add("cls_rows")  # rows a whole sequence apart: one row per image (class / token-0 rows)
    if r.alpha != 1.0 and r.M == r.N and r.a_mode == OP_K and r.b_mode == OP_K:  # S = scale q k^T of the chain
        f.add(f"chain{r.M}")
    if r.N % 8:
        f.add("ragged")
    if r.out_f32 and r.K == 256 and r.N == 16384:
        f.add("vq_score")
    if r.M % 77 == 0 and r.N == 3 * r.K and r.a_nb0 * r.a_nb1 == 1:
        f.add("text77")  # the qkv GEMM of a text tower's 77-token chunk
    return f


def test_routing(built):
    b = built
    seen = set()
    for r in b.recs:
        name = _name(b, r)
        assert r.k_blocks == -(-r.K // 64), f"{name}: the plan runs {r.k_blocks} k-blocks for K = {r.K}"
        if r.block_n > 128:
            assert r.wide and r.block_n in (192, 256), name
        if r.wide:
            assert r.a_mode == OP_K and r.a_nb0 == r.a_nb1 == 1, f"{name}: a wide plan with a batched or MN-major A"
            assert r.tma_epi != TE_NONE and r.out_f16 and not r.out_f32 and not r.res_f32, \
                f"{name}: a wide plan needs a tensor-map epilogue with an fp16 output"
            assert r.k_splits == 1, name
        if r.k_splits > 1:
            assert r.alpha == 1.0 and r.a_nb0 == r.a_nb1 == 1 and r.b_nb0 == r.b_nb1 == 1, name
            assert r.out_f32 and not r.out_f16 and not r.bias and not r.res_f16 and not r.res_f32 and not r.act, name
            assert r.tma_epi == TE_NONE and r.ldc == r.N, f"{name}: split-K partial sums on the generic epilogue"
            assert r.red_out and r.ld_out >= r.N, name
            assert r.k_splits <= r.k_blocks, name
        else:
            assert not (r.red_out or r.red_bias or r.red_res), name
        # the replay checks one main output, and forms the backward activations' bound without a residual
        assert not (r.out_f16 and r.out_f32), f"{name}: both an fp16 and an fp32 output"
        assert not (r.act in (ACT_QG_BWD, ACT_GELU_BWD) and (r.res_f16 or r.res_f32)), \
            f"{name}: an activation backward with a residual"
        seen |= features(r)
    missing = b.expect - seen
    print(f"[gemm plans] {b.name}: {len(b.recs)} plans, {sum(r.wide for r in b.recs)} wide, "
          f"{sum(r.k_splits > 1 for r in b.recs)} split-K, {sum(r.in_place for r in b.recs)} in place; kinds {sorted(seen)}")
    assert not missing, f"{b.name}: no plan of the kinds {sorted(missing)} any more"


# ------------------------------------------------------------------------------------------------------- the bound
def gemm_bound(ref, s, f32=False):
    return (REL32 if f32 else REL16) * ref.abs() + ABS * s


def ratio(err, bound):
    return (err.abs() / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0


def worst_at(err, bound, ref):
    """(err / bound, ref, err, bound) at the element where err / bound is largest."""
    q = err.abs() / bound.clamp_min(1e-300)
    i = int(q.flatten().argmax())
    return q.flatten()[i].item(), ref.flatten()[i].item(), err.abs().flatten()[i].item(), bound.flatten()[i].item()


def ulp16(v):
    """One fp16 ulp at |v| (the subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -24)))
    return torch.exp2(e.clamp_min(-14) - 10)


# Activation constants, from gemm_tc.cu.
# Tensor-map QuickGELU (sigmoid1702_h2): z = fp16(u * fp16(0.851)), t = tanh.approx.f16x2(z), s = fp16(0.5 t + 0.5).
#   fp16(0.851) = 0.85107421875 is 8.7e-5 = 2^-13.5 off 1.702 / 2, and z's rounding adds 2^-11 relative; through tanh
#   (max over z of |z| sech^2 z = 0.45) that moves t by at most 0.45 (2^-11 + 2^-13.5) absolute.  tanh.approx.f16 is
#   within 2^-10.987 relative (PTX ISA), |t| <= 1.  The hfma rounds s in [0, 1] by at most 2^-12.
TANH_ERR = 2.0 ** -10.987 + 0.45 * (2.0 ** -11 + 2.0 ** -13.5)
S_ERR_TE = 0.5 * TANH_ERR + 2.0 ** -12
#   a = fp16(u * fp16(1.702)): fp16(1.702) = 1.7021484375, 1.5e-4 absolute off, plus 2^-11 relative rounding.
A_REL_TE = 2.0 ** -11 + 0.00015 / 1.702
# Generic QuickGELU (fast_sigmoid = __fdividef(1, 1 + __expf(-x)) in fp32): __expf is within 2 + 1.16 |x| ulp (CUDA
# programming guide, fast intrinsics), __fdividef 2 ulp; the sigmoid's relative error is at most their sum.
def _fast_sigmoid_rel(z):
    return (4.0 + 1.16 * z.abs()) * 2.0 ** -23


def sigmoid1702(u):
    return torch.sigmoid(1.702 * u)


def quickgelu(u):
    return u * sigmoid1702(u)


def quickgelu_grad(u):
    s = sigmoid1702(u)
    return s * (1 + 1.702 * u * (1 - s))


def gelu(u):
    return 0.5 * u * torch.erfc(-u / math.sqrt(2.0))


def gelu_grad(u):
    return 0.5 * torch.erfc(-u / math.sqrt(2.0)) + u * torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)


def act_forward_bound(act, te, aux, out_ref):
    """|out - act(aux)| allowed for the forward activations, aux = the kernel's own fp16 pre-activation."""
    if act == ACT_GELU:  # stated within one fp16 ulp (erfcf in fp32 of exactly the fp16 u)
        return ulp16(out_ref) + 2.0 ** -24
    if te == TE_GELU:  # out = fp16(u s~), |s~ - s| <= S_ERR_TE
        return aux.abs() * S_ERR_TE * (1 + REL16) + REL16 * out_ref.abs() + 2.0 ** -25
    # generic: out = fp16(x sigmoid~(1.702 x)) of the fp32 pre-activation x, |x - aux| <= 2^-11 |aux|, |qg'| <= 1.13
    return (REL16 + _fast_sigmoid_rel(1.702 * aux)) * out_ref.abs() + 1.13 * REL16 * aux.abs() + 2.0 ** -25


def act_grad_bound(act, te, u, x):
    """(g, dg): the derivative factor at the saved fp16 u and the absolute error the kernel may make in it."""
    if act in (ACT_GELU_BWD,):
        g = gelu_grad(u)
        # 2^-11 relative, and the fp32 cancellation of Phi(u) + u phi(u) near its zero (u = -0.75): erfcf is within
        # 4 ulp, expf within 2 (CUDA programming guide), the argument products and the final add round by 1/2 ulp
        # each -- at most 8 fp32 ulp of Phi(u) + |u| phi(u)
        pos = 0.5 * torch.erfc(-u / math.sqrt(2.0)) + u.abs() * torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)
        return g, REL16 * g.abs() + 8 * 2.0 ** -24 * pos
    s = sigmoid1702(u)
    g = quickgelu_grad(u)
    a = 1.702 * u
    if te == TE_GELU_BWD:
        # g~ = fp16(s~ b~ + s~), b~ = fp16(a~ (1 - s~)): g = s + a s - a s^2 moves by eps (|1 + a (1 - 2 s)| + |a| eps)
        # for |s~ - s| <= eps, by s (1 - s) |a~ - a| for a~, plus the two roundings
        es = S_ERR_TE
        dg = es * ((1 + a * (1 - 2 * s)).abs() + a.abs() * es) + (s * (1 - s) + es) * A_REL_TE * a.abs() \
            + REL16 * (s + es) * (a * (1 - s)).abs() * (1 + A_REL_TE) + REL16 * (g.abs() + es * (1 + 2 * a.abs()))
        return g, dg
    es = s * _fast_sigmoid_rel(a)  # generic, fp32
    dg = es * ((1 + a * (1 - 2 * s)).abs() + a.abs() * es) + 8 * 2.0 ** -24 * (g.abs() + s * a.abs())
    return g, dg


# ------------------------------------------------------------------------------------------------------- replay
def _strided(buf, ptr_off, shape, strides):
    return torch.as_strided(buf, shape, strides, buf.storage_offset() + ptr_off)


def aligned(n, dtype, like, fill):
    """n elements filled with `fill`, at the address of the engine pointer `like` modulo 256 (the tensor-map and vector
    epilogue paths depend on 16-byte alignment; the caching allocator hands out 512-byte aligned blocks)."""
    eb = torch.tensor([], dtype=dtype).element_size()
    off = (like % 256) // eb if like else 0
    buf = torch.full((n + 256 // eb,), fill, device="cuda", dtype=dtype)[off:off + n]
    assert not like or buf.data_ptr() % 256 == like % 256
    return buf


def aligned_copy(t, like):
    out = aligned(t.numel(), t.dtype, like, 0)
    out.copy_(t)
    return out


def make_operand(g, ptr, mode, ld, mn, k, nb0, bs0, nb1, bs1, used, K, scale, device="cuda"):
    """A flat fp16 buffer laid out like the operand: NaN outside its extents, +-1e4 inside them past `used` rows / K,
    scale * N(0, 1) in the used part.  Returns (buffer, the used part as float64 [nb1, nb0, used, K])."""
    span = op_span(mode, ld, mn, k, nb0, bs0, nb1, bs1)
    buf = aligned(span, torch.half, ptr, float("nan"))
    s0, s1 = (bs0 if nb0 > 1 else 0), (bs1 if nb1 > 1 else 0)
    if mode == OP_MN:  # element (r, k) at k ld + r
        full = _strided(buf, 0, (nb1, nb0, k, mn), (s1, s0, ld, 1))
    else:
        full = _strided(buf, 0, (nb1, nb0, mn, k), (s1, s0, ld, 1))
    sign = torch.randint(0, 2, full.shape, device=device, generator=g).half() * 2 - 1
    full.copy_(sign * BIG)
    if mode == OP_MN:
        part = full[:, :, :K, :used]
    else:
        part = full[:, :, :used, :K]
    part.copy_((torch.randn(part.shape, device=device, generator=g) * scale).half())
    val = part.double()
    return buf, (val.transpose(-1, -2) if mode == OP_MN else val)


def epilogue_buffer(like, eb, ld, bs0, bs1, nb0, nb1, rows, cols, fill):
    span = (nb1 - 1) * bs1 + (nb0 - 1) * bs0 + (rows - 1) * ld + ld + 64  # a whole last row and a canary tail
    return aligned(span, torch.float32 if eb == 4 else torch.half, like, fill)


def epi_view(buf, ld, bs0, bs1, nb0, nb1, rows, cols, c0=0):
    return torch.as_strided(buf, (nb1, nb0, rows, cols), (bs1 if nb1 > 1 else 0, bs0 if nb0 > 1 else 0, ld, 1),
                            buf.storage_offset() + c0)


def _desc(r, A, B, bufs):
    d = _lib.TestGemmDesc()
    d.a, d.a_mode, d.lda, d.a_mn_extent, d.a_k_extent = _p(A), r.a_mode, r.lda, r.a_mn_extent, r.a_k_extent
    d.a_bs0, d.a_bs1 = r.a_bs0, r.a_bs1
    d.b, d.b_mode, d.ldb, d.b_mn_extent, d.b_k_extent = _p(B), r.b_mode, r.ldb, r.b_mn_extent, r.b_k_extent
    d.b_bs0, d.b_bs1 = r.b_bs0, r.b_bs1
    d.b_batched = int(r.b_nb0 * r.b_nb1 > 1)
    assert not d.b_batched or (r.b_nb0, r.b_nb1) == (r.a_nb0, r.a_nb1)
    d.nb0, d.nb1 = r.a_nb0, r.a_nb1
    d.M, d.N, d.K, d.block_n, d.fmt = r.M, r.N, r.K, r.block_n, 0
    d.alpha, d.bias_per_row, d.act, d.act_col0 = r.alpha, r.bias_per_row, r.act, r.act_col0
    for f in ("bias", "aux_in", "aux_out", "res_f32", "res_f16", "out_f32", "out_f16"):
        setattr(d, f, _p(bufs.get(f)))
    d.ldc, d.c_bs0, d.c_bs1 = r.ldc, r.c_bs0, r.c_bs1
    # the epilogue path the engine's plan took: the tensor-map one, or the generic one (add_gemm_splitk forces it)
    d.tma_epi = 0 if r.tma_epi != TE_NONE else -1
    if r.k_splits > 1:
        d.k_splits = r.k_splits
    return d


def _run(r, A, B, inputs, init):
    """One run of the plan (+ the split-K reduce) on fresh copies of the initial epilogue buffers."""
    lib = _lib.load()
    bufs = {k: aligned_copy(v, v.data_ptr()) for k, v in init.items()}
    bufs.update(inputs)
    if r.in_place:  # the residual is the output buffer itself
        if r.k_splits > 1:
            bufs["red_res"] = bufs["red_out"]
        elif r.res_f16:
            bufs["res_f16"] = bufs["out_f16"]
        else:
            bufs["res_f32"] = bufs["out_f32"]
    d = _desc(r, A, B, bufs)
    info = (C.c_int * 6)()
    assert lib.pxr_test_gemm_plan_info(C.byref(d), info) == 0
    got = dict(zip(("wide", "block_n", "stages", "tma_epi", "grid", "k_splits"), list(info)))
    want = {k: getattr(r, k) for k in got}
    assert got == want, f"{r.label.decode()}: the hook plans {got}, the engine planned {want}"
    err = C.create_string_buffer(512)
    rc = lib.pxr_test_gemm(C.byref(d), err, 512)
    assert rc == 0, f"pxr_test_gemm rc={rc}: {err.value.decode()}"
    if r.k_splits > 1:
        rc = lib.pxr_test_splitk_reduce(_p(bufs["out_f32"]), r.k_splits, C.c_longlong(r.M), r.N, int(r.ldc),
                                        _p(bufs.get("red_bias")), _p(bufs.get("red_res")), _p(bufs["red_out"]),
                                        int(r.ld_out))
        assert rc == 0, "pxr_test_splitk_reduce"
    torch.cuda.synchronize()
    return bufs


def replay(b, r, seed, others):
    """Worst err / bound of plan r over its outputs; asserts plan identity, canaries and determinism."""
    name = _name(b, r)
    private = check_footprint(b, r, others)  # static: nothing is launched on an out-of-range descriptor
    g = torch.Generator(device="cuda").manual_seed(seed)
    fwd_act = r.act in (ACT_QG, ACT_GELU)
    # pre-activations over about [-12, 12] for the forward activations, O(1) sums elsewhere
    sa, sb = 1.0, (4.0 if fwd_act else 1.0) / math.sqrt(r.K)
    A, Av = make_operand(g, r.a, r.a_mode, r.lda, r.a_mn_extent, r.a_k_extent, r.a_nb0, r.a_bs0, r.a_nb1, r.a_bs1, r.M, r.K, sa)
    B, Bv = make_operand(g, r.b, r.b_mode, r.ldb, r.b_mn_extent, r.b_k_extent, r.b_nb0, r.b_bs0, r.b_nb1, r.b_bs1, r.N, r.K, sb)
    nb0, nb1 = r.a_nb0, r.a_nb1
    split = r.k_splits > 1
    geo = (r.ldc, r.c_bs0, r.c_bs1, nb0, nb1, r.M, r.N)
    inputs, init = {}, {}
    bias = r.red_bias if split else r.bias
    if bias:
        n_bias = r.M if r.bias_per_row else r.N
        inputs["red_bias" if split else "bias"] = aligned_copy(torch.randn(n_bias, device="cuda", generator=g) * 0.5, bias)
    if r.aux_in:  # the saved (pre-)activation: over [-12, 12], NaN outside the M x N output
        aux = epilogue_buffer(r.aux_in, 2, *geo, float("nan"))
        epi_view(aux, *geo).copy_((torch.rand((nb1, nb0, r.M, r.N), device="cuda", generator=g) * 24 - 12).half())
        inputs["aux_in"] = aux
    res_name = "red_res" if split and r.red_res else ("res_f16" if r.res_f16 else ("res_f32" if r.res_f32 else None))
    rgeo = (r.ld_out, 0, 0, 1, 1, r.M, r.N) if split else geo
    res = None
    if res_name:
        eb = 4 if res_name == "res_f32" else 2
        res = epilogue_buffer(getattr(r, res_name), eb, *rgeo, float("nan"))
        epi_view(res, *rgeo).copy_(torch.randn((nb1, nb0, r.M, r.N), device="cuda", generator=g) * 0.5)
    outs = []  # (name, bytes per element, geometry) of the written tensors that are checked
    if split:
        init["out_f32"] = aligned(r.k_splits * r.M * r.ldc, torch.float32, r.out_f32, 0.0)
        init["red_out"] = epilogue_buffer(r.red_out, 2, *rgeo, CANARY)
        outs.append(("red_out", 2, rgeo))
    else:
        for f, eb in (("out_f16", 2), ("out_f32", 4), ("aux_out", 2)):
            if getattr(r, f):
                init[f] = epilogue_buffer(getattr(r, f), eb, *geo, CANARY)
                outs.append((f, eb, geo))
    if res is not None:
        if r.in_place:
            tgt = "red_out" if split else ("out_f16" if res_name == "res_f16" else "out_f32")
            epi_view(init[tgt], *(rgeo if split else geo)).copy_(epi_view(res, *(rgeo if split else geo)))
        else:
            inputs[res_name] = res
    got = _run(r, A, B, inputs, init)
    again = _run(r, A, B, inputs, init)
    for f, _, _ in outs:
        assert torch.equal(got[f].view(torch.uint8), again[f].view(torch.uint8)), f"{name}: two runs differ in {f}"

    # untouched: everything outside each batch's M x N, except the pad columns a private tensor-map store may write
    for f, eb, (ld, bs0, bs1, n0, n1, rows, cols) in outs:
        gran = 16 // eb
        touched = torch.zeros(got[f].shape, device="cuda", dtype=torch.bool)
        epi_view(touched, ld, bs0, bs1, n0, n1, rows, cols).fill_(True)
        pad = -(-cols // gran) * gran - cols
        if pad and r.tma_epi != TE_NONE and not split:
            assert private, f"{name}: the pad columns of {f} are not the output's own"
            epi_view(touched, ld, bs0, bs1, n0, n1, rows, pad, cols).fill_(True)
        keep = ~touched
        assert torch.equal(got[f][keep].view(torch.uint8 if eb == 2 else torch.int32),
                           init[f][keep].view(torch.uint8 if eb == 2 else torch.int32)), \
            f"{name}: {f} written outside the output"

    # float64 reference, in the epilogue's order
    acc = Av @ Bv.transpose(-1, -2)
    s = abs(r.alpha) * (Av.abs() @ Bv.abs().transpose(-1, -2))
    y = r.alpha * acc
    if bias:
        bv = inputs["red_bias" if split else "bias"].double()
        bv = bv.view(-1, 1) if r.bias_per_row else bv
        y = y + bv
        s = s + bv.abs()
    if fwd_act:
        aux_k = epi_view(got["aux_out"], *geo).double()
        wa = worst_at(aux_k - y, gemm_bound(y, s), y)
        assert wa[0] <= 1.0, f"{name}: saved pre-activation err / bound {wa[0]:.3f}"
        ref = (gelu if r.act == ACT_GELU else quickgelu)(aux_k)
        out = epi_view(got["out_f16"], *geo).double()
        w = worst_at(out - ref, act_forward_bound(r.act, r.tma_epi, aux_k, ref), ref)
        assert w[0] <= 1.0, f"{name}: activation err / bound {w[0]:.3f}"
        return max(w, wa)
    bound_extra = None
    if r.act in (ACT_QG_BWD, ACT_GELU_BWD):
        u = epi_view(inputs["aux_in"], *geo).double()
        gfac, dg = act_grad_bound(r.act, r.tma_epi, u, y)
        ref = y * gfac
        # the sum's own error through the factor, the factor's error, the fp16 store (and the tensor-map QuickGELU's
        # fp16 rounding of the sum before its half-precision product)
        rel = 2 * REL16 if r.tma_epi == TE_GELU_BWD else REL16
        bound_extra = gfac.abs() * ABS * s + y.abs() * dg + rel * ref.abs() + 2.0 ** -25
    else:
        ref = y
    if res is not None:
        rv = epi_view(res, *(rgeo if split else geo)).double()
        ref = ref + rv
        s = s + rv.abs()
    if r.act == ACT_RELU:
        ref = ref.clamp_min(0)
    f, eb, og = outs[0]
    out = epi_view(got[f], *og).double()
    assert torch.isfinite(out).all(), f"{name}: non-finite outputs (padding or +-1e4 elements were read)"
    if r.act == ACT_RELU_BWD:
        u = epi_view(inputs["aux_in"], *geo).double()
        assert torch.equal(out[u <= 0], torch.zeros_like(out[u <= 0])), f"{name}: the ReLU mask does not follow aux_in"
        ref = torch.where(u > 0, ref, torch.zeros_like(ref))
        s = torch.where(u > 0, s, torch.zeros_like(s))
    bound = bound_extra if bound_extra is not None else gemm_bound(ref, s, f32=(eb == 4))
    w = worst_at(out - ref, bound, ref)
    assert w[0] <= 1.0, f"{name}: err / bound {w[0]:.3f}"
    if r.out_f32 and r.K == 256 and r.N == 16384 and not split:
        vq_score_check(name, r, g)
    return w


SIG_SKIP = {"label", "a", "b", "bias", "aux_in", "aux_out", "res_f32", "res_f16", "out_f32", "out_f16", "red_bias",
            "red_res", "red_out"}
SIG_FIELDS = [f for f, _ in _lib.TestGemmRec._fields_ if f not in SIG_SKIP]


def _signature(r):
    # which pointers are set, and their alignment (it decides the vector and tensor-map epilogue paths)
    ptrs = [getattr(r, f) for f in sorted(SIG_SKIP - {"label"})]
    return tuple(getattr(r, f) for f in SIG_FIELDS) + tuple((bool(p), (p or 0) % 256) for p in ptrs)


def test_replay_every_plan(built):
    b = built
    first = {}
    for i, r in enumerate(b.recs):
        first.setdefault(_signature(r), i)
    worst, worst_name = (0.0, 0.0, 0.0, 0.0), ""
    for k, i in enumerate(first.values()):
        r = b.recs[i]
        others = _others_cover(b, i) if (r.tma_epi != TE_NONE and r.N % 8) else None
        w = replay(b, r, seed=k, others=others)
        if w[0] > worst[0]:
            worst, worst_name = w, r.label.decode()
    q, ref, err, bound = worst
    print(f"[gemm plans] {b.name}: {len(b.recs)} plans, {len(first)} signatures replayed; worst err/bound {q:.3f} "
          f"({worst_name}; there ref {ref:.4e}, |err| {err:.4e}, bound {bound:.4e})")


# ------------------------------------------------------------------------------------------------------- VQ scores
def vq_score_check(name, r, g):
    """scores = x~ . c~ of fp16-rounded fp32 operands (vq_prep's power-of-two scaling puts max |x|, |c| in [0.5, 1))
    within vq_select's 2^-9 |x|_2 |c|_2 + 2^-22 (|x|_1 + |c|_1) of the exact fp32 x . c."""
    x = torch.rand(r.M, r.K, device="cuda", generator=g) * 2 - 1
    c = torch.rand(r.N, r.K, device="cuda", generator=g) * 2 - 1
    x[:, :3] *= 1e-6  # some operands in fp16's subnormal range
    out = torch.full((r.M, r.ldc), CANARY, device="cuda")
    d = _lib.TestGemmDesc()
    d.a, d.lda, d.a_mn_extent, d.a_k_extent = _p(x16 := x.half()), r.K, r.M, r.K  # contiguous [M, K] / [N, K]
    d.b, d.ldb, d.b_mn_extent, d.b_k_extent = _p(c16 := c.half()), r.K, r.N, r.K
    d.nb0 = d.nb1 = 1
    d.M, d.N, d.K, d.block_n, d.alpha = r.M, r.N, r.K, r.block_n, 1.0
    d.out_f32, d.ldc = _p(out), r.ldc
    err = C.create_string_buffer(256)
    assert _lib.load().pxr_test_gemm(C.byref(d), err, 256) == 0, err.value
    torch.cuda.synchronize()
    del x16, c16
    xd, cd = x.double(), c.double()
    ref = xd @ cd.T
    bound = 2.0 ** -9 * xd.norm(dim=1, keepdim=True) * cd.norm(dim=1) + 2.0 ** -22 * (
        xd.abs().sum(1, keepdim=True) + cd.abs().sum(1))
    q = ratio(out[:, :r.N].double() - ref, bound)
    print(f"[gemm plans] {name}: VQ scores err / vq_select bound {q:.3e}")
    assert q <= 1.0


# ------------------------------------------------------------------------------------------------------- the bound
def test_bound_rejects_planted_defects():
    """Pure float64 on the CPU: a perfectly rounded fp16 output passes, and references with one 64-deep k-block dropped
    from one 128 x 128 tile, one head's keys read from its neighbour, or the last ragged column of a T = 257 score
    matrix taken from column 255 all fail."""
    g = torch.Generator().manual_seed(3)
    M, N, K = 384, 768, 768
    a = torch.randn(M, K, generator=g).half().double()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half().double()
    acc, s = a @ w.T, a.abs() @ w.abs().T
    out = acc.half().double()
    assert ratio(out - acc, gemm_bound(acc, s)) <= 1.0
    w_drop = w.clone()
    w_drop[:, 64:128] = 0
    bad = acc.clone()
    bad[128:256, 128:256] = (a @ w_drop.T)[128:256, 128:256]
    assert ratio(out - bad, gemm_bound(bad, s)) > 1.0, "a dropped k-block passes the bound"

    heads, T, d = 4, 50, 64
    q = torch.randn(heads, T, d, generator=g).half().double()
    k = torch.randn(heads, T, d, generator=g).half().double()
    acc, s = 0.125 * q @ k.transpose(1, 2), 0.125 * q.abs() @ k.abs().transpose(1, 2)
    out = acc.half().double()
    assert ratio(out - acc, gemm_bound(acc, s)) <= 1.0
    bad = acc.clone()
    bad[1] = 0.125 * q[1] @ k[2].T
    assert ratio(out - bad, gemm_bound(bad, s)) > 1.0, "a batch slice read from its neighbour passes the bound"

    T = 257
    q = torch.randn(T, d, generator=g).half().double()
    k = torch.randn(T, d, generator=g).half().double()
    acc, s = 0.125 * q @ k.T, 0.125 * q.abs() @ k.abs().T
    out = acc.half().double()
    assert ratio(out - acc, gemm_bound(acc, s)) <= 1.0
    bad = acc.clone()
    bad[:, 256] = acc[:, 255]
    assert ratio(out - bad, gemm_bound(bad, s)) > 1.0, "a ragged last column taken from column 255 passes the bound"


def test_activation_bounds_reject_a_wrong_derivative():
    """Pure float64: the tensor-map QuickGELU backward's bound admits the exact derivative rounded to fp16 and rejects
    s (1 + 1.702 u s), the derivative with s in place of 1 - s."""
    u = torch.linspace(-12, 12, 4097, dtype=torch.float64).half().double()
    x = torch.ones_like(u)
    g, dg = act_grad_bound(ACT_QG_BWD, TE_GELU_BWD, u, x)
    bound = x.abs() * dg + 2 * REL16 * (x * g).abs() + 2.0 ** -25
    assert ratio((x * g).half().double() - x * g, bound) <= 1.0
    s = sigmoid1702(u)
    wrong = s * (1 + 1.702 * u * s)
    assert ratio(wrong - x * g, bound) > 1.0


def test_record_struct_follows_the_header():
    """ctypes lays the record out by its field list: it must name the header's fields in its order."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pixray_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} pxr_test_gemm_rec;", src).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        first, *rest = decl.split(",")
        names += [re.sub(r"\[.*\]$", "", re.sub(r"^.*[\s*]", "", first.strip()))] + [r.strip() for r in rest]
    assert [f[0] for f in _lib.TestGemmRec._fields_] == names
