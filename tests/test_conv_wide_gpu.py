"""Implicit-GEMM convolutions on the 384-thread kernel (gemm_wide_kernel) against the 288-thread one on the same plan.

A convolution with bias and / or an fp16 residual and no split-K runs its 128-, 192- and 256-column tiles in the
384-thread kernel; `narrow_kernel` runs the same plan on the 288-thread kernel (at most 128 columns).  Both accumulate
every output in the same k order (tap-major, then 64-channel blocks) and share the per-element epilogue arithmetic, so
their outputs must agree bit for bit.  Channels past N inside a wider pixel pitch and pixels past the last image must
stay untouched, two runs must give the same bits, and the result is held against torch fp32 conv2d at the tolerances
of test_gemm_gpu.py, so that a mistake both kernels share is caught too."""
import pytest
import torch
import torch.nn.functional as F

from conv_kernel_util import run_conv_on

pytestmark = pytest.mark.gpu

CANARY = 3.0
PAD_CH, PAD_PIX = 64, 37

# (batch, H, W, Cin, Cout, ksize, tile widths): the VQGAN decoder's 256^2 and 128^2 convolutions (ResBlock conv,
# conv with a 256-channel input, the upsample conv, the 1x1 nin_shortcut), ragged latents at tile_w 16 (9x9, 18x27)
# and tile_w 8 (5x36, 24x8), several images, and one tile (fewer tiles than SMs).
SHAPES = [
    (1, 256, 256, 128, 128, 3, (128,)),
    (1, 128, 128, 256, 128, 3, (128,)),
    (1, 128, 128, 256, 256, 3, (128, 192, 256)),
    (1, 128, 128, 256, 128, 1, (128,)),
    (1, 9, 9, 128, 128, 3, (128,)),
    (1, 18, 27, 128, 256, 3, (128, 192, 256)),
    (1, 5, 36, 64, 128, 3, (128,)),
    (1, 24, 8, 128, 256, 3, (256,)),
    (3, 18, 27, 128, 128, 3, (128,)),
    (2, 24, 8, 64, 256, 1, (192,)),
]

# name -> (bias, residual, in place)
MODES = {
    "f16 bias": (True, False, False),
    "f16": (False, False, False),
    "res16 bias": (True, True, False),
    "res16 in place": (True, True, True),
}


def _inputs(B, H, W, Cin, Cout, ks, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(B, H, W, Cin, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(Cout, Cin, ks, ks, device="cuda", generator=g) * (0.4 / (Cin * ks * ks) ** 0.5)).half()
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B * H * W + PAD_PIX, Cout + PAD_CH, device="cuda", generator=g).half()
    wt = w.permute(2, 3, 0, 1).reshape(ks * ks, Cout, Cin).contiguous()  # [tap][cout][cin], tap = 3 (dy + 1) + dx + 1
    return x, w, wt, bias, res


def _run(x, wt, Cout, ks, bn, mode, bias, res, narrow):
    has_bias, has_res, in_place = MODES[mode]
    B, H, W, _ = x.shape
    ld = Cout + PAD_CH
    if in_place:
        out = res.clone()
        r = out
    else:
        out = torch.full((B * H * W + PAD_PIX, ld), CANARY, device="cuda", dtype=torch.half)
        r = res if has_res else None
    run_conv_on(x, wt, Cout, Cout, ks, block_n=bn, bias=bias if has_bias else None, res_f16=r, out_f16=out, ldc=ld,
                narrow_kernel=narrow)
    return out


def _check_ref(out, ref, name):
    err = (out.float() - ref).abs().max().item()
    mag = ref.abs().max().item()
    assert err <= 3e-3 * max(mag, 1.0), f"{name}: err {err} vs ref max {mag}"


@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,bns", SHAPES)
def test_conv_wide_matches_narrow(B, H, W, Cin, Cout, ks, bns):
    x, w, wt, bias, res = _inputs(B, H, W, Cin, Cout, ks, seed=H + 7 * W + 13 * Cin + Cout + ks + B)
    px = B * H * W
    acc = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), padding=ks // 2).permute(0, 2, 3, 1).reshape(px, Cout)
    for bn in bns:
        for mode, (has_bias, has_res, in_place) in MODES.items():
            name = f"{mode} bn={bn} {B}x{H}x{W} {Cin}->{Cout} k{ks}"
            o_w = _run(x, wt, Cout, ks, bn, mode, bias, res, 0)
            o_w2 = _run(x, wt, Cout, ks, bn, mode, bias, res, 0)
            o_n = _run(x, wt, Cout, ks, min(bn, 128), mode, bias, res, 1)
            assert torch.equal(o_w, o_w2), f"{name}: two runs differ"
            assert torch.equal(o_w, o_n), f"{name}: 384-thread output differs from the 288-thread kernel's " \
                f"(max {(o_w.float() - o_n.float()).abs().max().item():.3e})"
            untouched = res if in_place else torch.full_like(res, CANARY)
            assert torch.equal(o_w[:px, Cout:], untouched[:px, Cout:]), f"{name}: channels past N written"
            assert torch.equal(o_w[px:], untouched[px:]), f"{name}: pixels past the output written"
            ref = acc + (bias if has_bias else 0.0) + (res[:px, :Cout].float() if has_res else 0.0)
            _check_ref(o_w[:px, :Cout], ref, name)
