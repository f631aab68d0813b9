"""GPU parity of the wgmma GEMM / implicit-GEMM conv kernel against torch fp32 matmul of the same fp16 inputs.

`cg` is the C ABI's cta_group request: sm_90 has no CTA-pair MMA, so cg=2 must be accepted and runs the same single-CTA
tiles as cg=1 (the axis checks that the request stays harmless).  Tiles are at most 128 columns wide: a
requested block_n of 192 or 256 runs as 128.  Widths other than 64 / 128 (e.g. 16, 80, 112) take the generic
fragment path."""
import pytest
import torch
import torch.nn.functional as F

from gemm_util import run_conv, run_gemm

pytestmark = pytest.mark.gpu


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).half()


def _check(out, ref, tol, name):
    err = (out.float() - ref).abs().max().item()
    mag = ref.abs().max().item()
    print(f"{name}: max_abs_err={err:.3e} ref_max={mag:.3e}")
    assert err <= tol * max(mag, 1.0), f"{name}: err {err} vs ref max {mag}"


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("M,N,K,bn", [(300, 256, 192, 128), (128, 64, 64, 64), (197, 197, 64, 208), (1000, 768, 768, 256),
                                      (1000, 768, 768, 192), (2000, 100, 320, 64), (700, 400, 448, 80),
                                      (500, 336, 320, 112)])
def test_gemm_kmajor(M, N, K, bn, cg):
    """One CTA per 128 x bn tile (bn clamped to 128 for this epilogue); cg=2 runs the same tiles."""
    torch.manual_seed(0)
    A, B = _rand(M, K), _rand(N, K)
    out = torch.full((M, N), 7.0, device="cuda")
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, out_f32=out, ldc=N, cta_group=cg)
    _check(out, A.float() @ B.float().T, 2e-3, f"kmajor cg{cg} {M}x{N}x{K}")


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_epilogue_bias_gelu_residual(cg):
    torch.manual_seed(1)
    M, N, K = 520, 384, 256
    A, B = _rand(M, K, scale=0.2), _rand(N, K, scale=0.2)
    bias = torch.randn(N, device="cuda")
    res = torch.randn(M, N, device="cuda")
    out16 = torch.zeros(M, N, device="cuda", dtype=torch.half)
    out32 = torch.zeros(M, N, device="cuda")
    aux = torch.zeros(M, N, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, alpha=0.5, bias=bias, act=1, aux_out=aux, res_f32=res,
             out_f32=out32, out_f16=out16, ldc=N, cta_group=cg)
    u = 0.5 * (A.float() @ B.float().T) + bias
    ref = u * torch.sigmoid(1.702 * u) + res
    _check(aux, u, 2e-3, "aux(pre-act)")
    _check(out32, ref, 2e-3, "gelu+res f32")
    _check(out16, ref, 4e-3, "gelu+res f16")
    # backward epilogue: multiply by quickgelu'(u)
    g = torch.zeros(M, N, device="cuda")
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, act=2, aux_in=aux, out_f32=g, ldc=N, cta_group=cg)
    uf = aux.float()
    s = torch.sigmoid(1.702 * uf)
    ref_g = (A.float() @ B.float().T) * (s * (1 + 1.702 * uf * (1 - s)))
    _check(g, ref_g, 2e-3, "gelu bwd")
    # an activation code past QuickGELU backward is refused, not run as a plain epilogue
    with pytest.raises(RuntimeError, match="unknown epilogue activation"):
        run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, act=3, out_f32=g, ldc=N, cta_group=cg)


def test_gemm_bias_per_row_and_tail():
    torch.manual_seed(2)
    M, N, K = 512, 250, 128
    A, B = _rand(M, K), _rand(N, K)
    bias = torch.randn(M, device="cuda")
    out = torch.zeros(M, 256, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, bias=bias, bias_per_row=1, out_f16=out, ldc=256)
    ref = A.float() @ B.float().T + bias[:, None]
    _check(out[:, :N], ref, 4e-3, "row-bias tail")
    assert out[:, N:].abs().max().item() == 0.0


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_mn_major_b(cg):
    torch.manual_seed(3)
    M, N, K = 260, 256, 200
    A = _rand(M, K)
    Bt = _rand(K, N)  # stored [K, N]: n contiguous -> MN-major B
    out = torch.zeros(M, N, device="cuda")
    run_gemm(A, Bt, M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, out_f32=out, ldc=N, cta_group=cg)
    _check(out, A.float() @ Bt.float(), 2e-3, f"MN-major B cg{cg}")


def test_gemm_mn_major_a():
    torch.manual_seed(4)
    M, N, K = 197, 64, 197
    At = _rand(K, 208)  # stored [K, M(ld 208)]: m contiguous -> MN-major A
    At[:, M:] = 0
    B = _rand(N, K + 11)[:, :K]  # ld = K+11?  needs ld % 8 == 0 -> use 208
    Bp = torch.zeros(N, 208, device="cuda", dtype=torch.half)
    Bp[:, :K] = B
    out = torch.zeros(M, N, device="cuda")
    run_gemm(At, Bp, M, N, K, a_mode=1, lda=208, ldb=208, block_n=64, out_f32=out, ldc=N)
    _check(out, At[:, :M].float().T @ Bp[:, :K].float().T, 2e-3, "MN-major A")


@pytest.mark.parametrize("cg", [1, 2])
def test_gemm_both_mn_major_batched_attention_shapes(cg):
    """dK = dS^T Q per (image, head): A = dS stored [q, k] (MN-major), B = Q stored [q, d] (MN-major)."""
    torch.manual_seed(5)
    imgs, heads, T, d, ldp = 3, 4, 197, 64, 208
    dS = torch.zeros(imgs, heads, T, ldp, device="cuda", dtype=torch.half)
    dS[..., :T] = _rand(imgs, heads, T, T, scale=0.1)
    qkv = _rand(imgs, T, 3 * heads * d)
    out = torch.zeros(imgs, T, heads * d, device="cuda", dtype=torch.half)
    run_gemm(dS, qkv, T, d, T, a_mode=1, lda=ldp, a_mn=T, a_k=T, b_mode=1, ldb=3 * heads * d, b_mn=d, b_k=T,
             nb0=heads, nb1=imgs, a_bs=(T * ldp, heads * T * ldp), b_bs=(d, T * 3 * heads * d), b_batched=1,
             block_n=64, out_f16=out, ldc=heads * d, c_bs=(d, T * heads * d), cta_group=cg)
    q = qkv[..., : heads * d].reshape(imgs, T, heads, d).permute(0, 2, 1, 3).float()
    ref = torch.einsum("bhqk,bhqd->bhkd", dS[..., :T].float(), q).permute(0, 2, 1, 3).reshape(imgs, T, heads * d)
    _check(out, ref, 4e-3, "batched both-MN")


def test_gemm_batched_qk():
    torch.manual_seed(6)
    imgs, heads, T, d, ldp = 2, 12, 197, 64, 208
    qkv = _rand(imgs, T, 3 * heads * d)
    S = torch.zeros(imgs, heads, T, ldp, device="cuda", dtype=torch.half)
    k_off = qkv.view(-1)[heads * d:]
    run_gemm(qkv, k_off, T, T, d, lda=3 * heads * d, a_mn=T, a_k=d, ldb=3 * heads * d, b_mn=T, b_k=d, nb0=heads,
             nb1=imgs, a_bs=(d, T * 3 * heads * d), b_bs=(d, T * 3 * heads * d), b_batched=1, block_n=208,
             alpha=0.125, out_f16=S, ldc=ldp, c_bs=(T * ldp, heads * T * ldp))
    q = qkv[..., : heads * d].reshape(imgs, T, heads, d).permute(0, 2, 1, 3).float()
    k = qkv[..., heads * d: 2 * heads * d].reshape(imgs, T, heads, d).permute(0, 2, 1, 3).float()
    ref = 0.125 * q @ k.transpose(-1, -2)
    _check(S[..., :T], ref, 4e-3, "batched QK^T")
    assert S[..., T:].abs().max().item() == 0.0


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("H,W,Cin,Cout,ks,bn", [(32, 32, 128, 128, 3, 128), (16, 16, 256, 512, 3, 128),
                                                  (64, 64, 64, 3, 3, 16), (16, 16, 256, 256, 1, 64),
                                                  # ragged widths / heights (pixray's preset latents: 9x9, 18x18, 6x12 ...)
                                                  (9, 9, 128, 128, 3, 128), (18, 26, 64, 128, 3, 64), (6, 12, 128, 64, 3, 64),
                                                  (4, 4, 64, 64, 3, 64), (27, 27, 64, 64, 1, 64), (13, 24, 128, 3, 3, 16)])
def test_conv_implicit_gemm(H, W, Cin, Cout, ks, bn, cg):
    torch.manual_seed(7)
    x = _rand(1, H, W, Cin, scale=0.5)
    w = _rand(Cout, Cin, ks, ks, scale=0.05)
    bias = torch.randn(Cout, device="cuda")
    cout_pad = max(16, (Cout + 15) // 16 * 16)
    wt = torch.zeros(ks * ks, cout_pad, Cin, device="cuda", dtype=torch.half)
    wt[:, :Cout] = w.permute(2, 3, 0, 1).reshape(ks * ks, Cout, Cin)
    out = torch.zeros(1, H, W, cout_pad, device="cuda")
    run_conv(x, wt, Cout, cout_pad, ks, block_n=bn, bias=bias, out_f32=out, ldc=cout_pad, cta_group=cg)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, padding=ks // 2).permute(0, 2, 3, 1)
    _check(out[..., :Cout], ref, 2e-3, f"conv{ks}x{ks} {H}x{W} {Cin}->{Cout}")


@pytest.mark.parametrize("te,cg", [(0, 1), (-1, 1), (0, 2)])
def test_gemm_tensor_map_epilogue_modes(te, cg):
    """The five tensor-map epilogue shapes (te=0: chosen automatically; te=-1: the generic epilogue on the same
    problem) on a GEMM with an M tail, several N tiles and a padded row pitch."""
    torch.manual_seed(21)
    M, N, K, ld = 1000, 384, 256, 400
    A, B = _rand(M, K, scale=0.2), _rand(N, K, scale=0.2)
    bias = torch.randn(N, device="cuda")
    acc = A.float() @ B.float().T
    # TE_F16 (alpha, bias)
    o = torch.full((M, ld), 3.0, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, alpha=0.5, bias=bias, out_f16=o, ldc=ld, tma_epi=te, cta_group=cg)
    _check(o[:, :N], 0.5 * acc + bias, 3e-3, "f16 out")
    assert (o[:, N:] == 3.0).all(), "columns past N must stay untouched"
    # TE_GELU
    o = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    aux = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=192, bias=bias, act=1, aux_out=aux, out_f16=o, ldc=ld, tma_epi=te, cta_group=cg)
    u = acc + bias
    _check(aux[:, :N], u, 3e-3, "gelu aux")
    _check(o[:, :N], u * torch.sigmoid(1.702 * u), 3e-3, "gelu out")
    # TE_GELU_BWD with an MN-major B (the fc2 dgrad shape)
    Bt = B.t().contiguous()  # [K, N]
    g = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, Bt, M, N, K, lda=K, b_mode=1, ldb=N, block_n=128, act=2, aux_in=aux, out_f16=g, ldc=ld, tma_epi=te, cta_group=cg)
    uf = aux[:, :N].float()
    sg = torch.sigmoid(1.702 * uf)
    _check(g[:, :N], acc * (sg * (1 + 1.702 * uf * (1 - sg))), 3e-3, "gelu bwd")
    # TE_RES32
    res = torch.randn(M, ld, device="cuda")
    o32 = torch.full((M, ld), 5.0, device="cuda")
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=192, bias=bias, res_f32=res, out_f32=o32, ldc=ld, tma_epi=te, cta_group=cg)
    _check(o32[:, :N], acc + bias + res[:, :N], 2e-3, "res32")
    assert (o32[:, N:] == 5.0).all()
    # in place (out == res), as the residual stream does
    r2 = res.clone()
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=192, bias=bias, res_f32=r2, out_f32=r2, ldc=ld, tma_epi=te, cta_group=cg)
    _check(r2[:, :N], acc + bias + res[:, :N], 2e-3, "res32 in place")
    # TE_RES16
    r16 = _rand(M, ld)
    o = torch.zeros(M, ld, device="cuda", dtype=torch.half)
    run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=128, res_f16=r16, out_f16=o, ldc=ld, tma_epi=te, cta_group=cg)
    _check(o[:, :N], acc + r16[:, :N].float(), 3e-3, "res16")


@pytest.mark.parametrize("te,cg", [(0, 1), (-1, 1), (0, 2)])
def test_gemm_tensor_map_epilogue_batched_ragged(te, cg):
    """Attention-score shape: 197 x 197 per (image, head), row pitch 200, rows of one batch must not spill into the next."""
    torch.manual_seed(22)
    imgs, heads, T, d, ldp = 3, 4, 197, 64, 200
    qkv = _rand(imgs * T, 3 * heads * d, scale=0.3)
    S = torch.full((imgs, heads, T, ldp), 9.0, device="cuda", dtype=torch.half)
    run_gemm(qkv, qkv[:, heads * d:], T, T, d, lda=3 * heads * d, ldb=3 * heads * d, nb0=heads, nb1=imgs,
             a_bs=(d, T * 3 * heads * d), b_bs=(d, T * 3 * heads * d), b_batched=1, block_n=208, alpha=0.125, out_f16=S,
             ldc=ldp, c_bs=(T * ldp, heads * T * ldp), tma_epi=te, cta_group=cg)
    x = qkv.float().view(imgs, T, 3, heads, d)
    ref = 0.125 * torch.einsum("ithd,ishd->ihts", x[:, :, 0], x[:, :, 1])
    _check(S[..., :T], ref, 3e-3, "batched scores")
    # TMA stores clip at 16-byte granularity: the pad columns up to the next 16-byte boundary (inside the row pitch)
    # receive the accumulator's zeros; the generic epilogue leaves them untouched
    pad = S[..., T:]
    assert ((pad == 9.0) | (pad == 0.0)).all()


@pytest.mark.parametrize("te,cg", [(0, 1), (-1, 1), (0, 2)])
@pytest.mark.parametrize("H,W,Cin,Cout,bn", [(32, 32, 128, 128, 128), (16, 16, 256, 512, 64), (24, 8, 64, 64, 64),
                                             (9, 9, 64, 64, 64), (18, 27, 128, 128, 128), (5, 36, 64, 128, 64)])
def test_conv_tensor_map_epilogue(H, W, Cin, Cout, bn, te, cg):
    torch.manual_seed(23)
    x = _rand(1, H, W, Cin, scale=0.5)
    w = _rand(Cout, Cin, 3, 3, scale=0.05)
    bias = torch.randn(Cout, device="cuda")
    res = _rand(1, H, W, Cout)
    wt = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, padding=1).permute(0, 2, 3, 1)
    out = torch.zeros(1, H, W, Cout, device="cuda", dtype=torch.half)
    run_conv(x, wt, Cout, Cout, 3, block_n=bn, bias=bias, out_f16=out, ldc=Cout, tma_epi=te, cta_group=cg)
    _check(out, ref, 3e-3, f"conv f16 {H}x{W}")
    run_conv(x, wt, Cout, Cout, 3, block_n=bn, bias=bias, res_f16=res, out_f16=out, ldc=Cout, tma_epi=te, cta_group=cg)
    _check(out, ref + res.float(), 3e-3, f"conv res16 {H}x{W}")


def test_gemm_throughput_report():
    """Not an assertion on speed: prints achieved TFLOP/s for the CLIP-sized GEMMs so the first GPU run is informative."""
    torch.manual_seed(8)
    for (M, N, K) in [(12608, 2304, 768), (12608, 3072, 768), (12608, 768, 3072), (12608, 768, 768)]:
        A, B = _rand(M, K, scale=0.1), _rand(N, K, scale=0.1)
        ref = A.float() @ B.float().T
        for cg, bn in [(1, 256), (2, 256), (2, 192)]:
            out = torch.zeros(M, N, device="cuda", dtype=torch.half)
            run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, out_f16=out, ldc=N, repeat=3, cta_group=cg)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            run_gemm(A, B, M, N, K, lda=K, ldb=K, block_n=bn, out_f16=out, ldc=N, repeat=20, cta_group=cg)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 20
            _check(out, ref, 4e-3, f"big {M}x{N}x{K} cg{cg} bn{bn}")
            print(f"GEMM {M}x{N}x{K} cta_group {cg} bn {bn}: {ms * 1e3:.1f} us  {2 * M * N * K / ms / 1e9:.1f} TFLOP/s")


def _time(fn, reps=20):
    fn(3)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn(reps)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def test_gemm_epilogue_throughput_report():
    """Prints us per launch of the CLIP ViT-B/16 (64 cutouts) GEMMs with their pipeline epilogues, generic vs tensor-map."""
    torch.manual_seed(9)
    M = 64 * 197
    A768, A3072 = _rand(M, 768, scale=0.1), _rand(M, 3072, scale=0.1)
    W1, W2, Wp = _rand(3072, 768, scale=0.1), _rand(768, 3072, scale=0.1), _rand(768, 768, scale=0.1)
    o3072 = torch.zeros(M, 3072, device="cuda", dtype=torch.half)
    aux = torch.zeros(M, 3072, device="cuda", dtype=torch.half)
    o768 = torch.zeros(M, 768, device="cuda", dtype=torch.half)
    res32, o32 = torch.randn(M, 768, device="cuda"), torch.zeros(M, 768, device="cuda")
    b3072, b768 = torch.randn(3072, device="cuda"), torch.randn(768, device="cuda")
    qkv = _rand(M, 2304, scale=0.3)
    S = torch.zeros(64 * 12 * 197, 200, device="cuda", dtype=torch.half)
    cases = {
        "fc1 bias+gelu+aux": lambda te, r, cg=1: run_gemm(A768, W1, M, 3072, 768, lda=768, ldb=768, block_n=192, bias=b3072, act=1,
                                                    aux_out=aux, out_f16=o3072, ldc=3072, repeat=r, tma_epi=te, cta_group=cg),
        "fc2 dgrad gelu-bwd (B mn)": lambda te, r, cg=1: run_gemm(A768, W2, M, 3072, 768, lda=768, b_mode=1, ldb=3072, block_n=192,
                                                            act=2, aux_in=aux, out_f16=o3072, ldc=3072, repeat=r, tma_epi=te, cta_group=cg),
        "fc2 bias+res32": lambda te, r, cg=1: run_gemm(A3072, W2, M, 768, 3072, lda=3072, ldb=3072, block_n=192, bias=b768,
                                                 res_f32=res32, out_f32=o32, ldc=768, repeat=r, tma_epi=te, cta_group=cg),
        "proj bias+res32": lambda te, r, cg=1: run_gemm(A768, Wp, M, 768, 768, lda=768, ldb=768, block_n=192, bias=b768,
                                                  res_f32=res32, out_f32=o32, ldc=768, repeat=r, tma_epi=te, cta_group=cg),
        "proj dgrad f16 (B mn)": lambda te, r, cg=1: run_gemm(A768, Wp, M, 768, 768, lda=768, b_mode=1, ldb=768, block_n=192,
                                                        out_f16=o768, ldc=768, repeat=r, tma_epi=te, cta_group=cg),
        "scores 197x197x64 x768": lambda te, r, cg=1: run_gemm(qkv, qkv[:, 768:], 197, 197, 64, lda=2304, ldb=2304, nb0=12, nb1=64,
                                                         a_bs=(64, 197 * 2304), b_bs=(64, 197 * 2304), b_batched=1,
                                                         block_n=208, alpha=0.125, out_f16=S, ldc=200,
                                                         c_bs=(197 * 200, 12 * 197 * 200), repeat=r, tma_epi=te, cta_group=cg),
    }
    for name, fn in cases.items():
        t_gen = _time(lambda r: fn(-1, r))
        t_tma = _time(lambda r: fn(0, r))
        t_pair = _time(lambda r: fn(0, r, 2))
        print(f"{name:32s} generic {t_gen:7.1f} us   tensor-map {t_tma:7.1f} us   tensor-map + CTA pairs {t_pair:7.1f} us")
