// attn_bwd_wg: the fused attention backward on wgmma, for one (image, head) pair per CTA and T <= 208 (see attn_tc.cuh
// for the tensors and the forward).  Two warpgroups of 128 threads; every score product is formed once.
//
// Staging.  Thread 0 issues every TMA load of the pair up front (there is no ring to refill, so no producer warps): per
// 64-row block i one mbarrier covers K and V rows [64 i, 64 i + 64) (64-row boxes) and Q rows [64 i, 64 i + 64) up to
// QP = round16(T) (16-row boxes); one more covers dO (16-row boxes), requested first.  Rows >= T of the image are
// zero-filled by the tensor map.  As soon as dO has landed, every thread forms D_i = dO_i . O_i (from the fp16 O the
// forward stored) and lse_i log2(e) into shared memory, while K, V and Q still arrive.  Tiles are
// [rows][64] fp16 with 128-byte rows and the 128-byte swizzle (attn_frag's swz), read by wgmma through descriptors.
//
// Phase 1 (dK, dV): warpgroup wg owns the 64-key tiles kt = wg, wg + 2, ... and walks the queries in 64-row chunks (the
// last one 16, 32 or 48 rows):  S^T = K_kt Q^T and dP^T = V_kt dO^T (both operands K-major, shared memory),
// P^T = exp2(c S^T - L), dS^T = P^T o (dP^T - D) in registers, then dV += P^T dO and dK += dS^T Q with P^T / dS^T as the
// fp16 register A operand and dO / Q read MN-major.  dS^T is also stored (stmatrix.trans) as dS into the shared buffer
// dS_kt = [QP query rows][64 keys of tile kt], the K-major A layout of phase 2.
// Phase 2 (dQ), after one CTA barrier: warpgroup wg owns the 64-query tiles qt = wg, wg + 2, ...: dQ = sum_kt dS_kt K_kt
// over the key tiles in order (K read MN-major).  Rows of a 64-row query tile past QP read finite rows of the next buffer
// (dS_kt+1, or K after the last one) and are not stored.
//
// Rounding is that of attn_bwd_kernel: P (ex2.approx.ftz, which parts from exp2f only for results below 2^-126, where
// the fp16 operand is 0 either way) and dS are rounded to fp16 only as MMA operands, scale multiplies the fp32 dK / dQ
// accumulators before the fp16 store, and P, dS are exactly zero for keys >= T or queries >= T, so the zero rows add
// exact zeros.  Every output element has one writer and the sums run in a fixed order: no atomics, the same bits every run.
#include "attn_tc.cuh"
#include "attn_frag.cuh"
#include "gemm_tc.cuh"
#include "launch.cuh"
#include "ptx.cuh"
#include <cstdio>
#include <mutex>

namespace pxr {
namespace {

using namespace attn_frag;
using namespace ptx;

constexpr int WG_THREADS = 256;
constexpr int WG_MAX_T = 208;
constexpr int TILE = 64 * ROW_BYTES;  // one 64-row staged tile

__host__ __device__ int round16(int T) { return (T + 15) & ~15; }
__host__ __device__ int round64(int T) { return (T + 63) & ~63; }
// dS buffers, K, V, Q, dO, then L and D (QP floats each), one mbarrier per 64-row block and one for dO; 1024 bytes for the
// alignment
int wg_smem(int T) {
  const int QP = round16(T), KP = round64(T), NB = KP / 64;
  return (NB * QP + 2 * KP + 2 * QP) * ROW_BYTES + 2 * QP * 4 + (NB + 1) * 8 + 1024;
}

__device__ __forceinline__ uint64_t desc_k(uint32_t addr) { return make_smem_desc_sw128(addr, 0, 1024); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t addr) { return make_smem_desc_sw128(addr, 8192, 1024); }

template <int N>
__device__ __forceinline__ void fence_acc(float (&x)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) wgmma_fence_operand(x[i]);
}

// S = A B^T over the 64 head columns (four k16 steps), A a 64-row K-major tile, B NJ 16-row slices of a K-major tile
// (one m64n64 instruction per step for a full chunk, NJ m64n16 ones otherwise: the n16 fragments tile the n64 one)
template <int NJ>
__device__ __forceinline__ void scores(float (&s)[8 * NJ], uint32_t a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint64_t ad = desc_k(a) + 2 * k, bd = desc_k(b) + 2 * k;  // k16 step: 32 bytes along the row
    if (NJ == 4) {
      wgmma_m64n64<0, 0>(s, ad, bd, k > 0, 0);
    } else {
#pragma unroll
      for (int j = 0; j < NJ; ++j) wgmma_m64n16<0, 0>(s + 8 * j, ad, bd + j * (2048 >> 4), k > 0, 0);
    }
  }
}

// A fragment of query slice j (16 columns) of a transposed-score fragment
template <int N>
__device__ __forceinline__ void to_a(uint32_t (&a)[4], const float (&x)[N], int j) {
  a[0] = pack(x[8 * j], x[8 * j + 1]);
  a[1] = pack(x[8 * j + 2], x[8 * j + 3]);
  a[2] = pack(x[8 * j + 4], x[8 * j + 5]);
  a[3] = pack(x[8 * j + 6], x[8 * j + 7]);
}

struct Smem {
  uint32_t dS, K, V, Q, dO;  // shared addresses
  const float *L, *D;
  int QP;
};

// Phase 1 on one query chunk: rows [q0, q0 + 16 NJ) against key tile kt.  key0: this thread's first key row (absolute);
// its second is key0 + 8; acc = 0 on the tile's first chunk (its wgmmas overwrite dK, dV: zeroing them with ordinary
// instructions would make ptxas serialise every wgmma).  Leaves the dV and dK groups in flight; the next chunk's first wait
// retires them.
template <int NJ>
__device__ __forceinline__ void dkdv_chunk(float (&dk)[32], float (&dv)[32], const Smem& sm, int kt, int q0, int key0,
                                           int T, float c, uint32_t acc) {
  const int t = threadIdx.x & 127, lane = t & 31, w = t >> 5;
  float s[8 * NJ], dp[8 * NJ];
  wgmma_fence();
  scores<NJ>(s, sm.K + kt * TILE, sm.Q + q0 * ROW_BYTES);
  wgmma_commit();
  scores<NJ>(dp, sm.V + kt * TILE, sm.dO + q0 * ROW_BYTES);
  wgmma_commit();
  wgmma_wait<1>();  // S^T (and the previous chunk's dV, dK) done; dP^T may still run
  fence_acc(s);
  const bool k0_live = key0 < T, k1_live = key0 + 8 < T;
  uint32_t pa[NJ][4];
#pragma unroll
  for (int i = 0; i < 2 * NJ; ++i) {  // 8-query column group i: queries q0 + 8 i + 2 (lane % 4) + {0, 1}
    const int q = q0 + 8 * i + 2 * (lane & 3);
    const float2 L = *reinterpret_cast<const float2*>(sm.L + q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const bool live = (e < 2 ? k0_live : k1_live) && q + (e & 1) < T;
      float& x = s[4 * i + e];
      x = live ? ex2_approx(x * c - ((e & 1) ? L.y : L.x)) : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) to_a(pa[j], s, j);
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < NJ; ++j) wgmma_m64n64_rs<1>(dv, pa[j], desc_mn(sm.dO + (q0 + 16 * j) * ROW_BYTES), acc | j);
  wgmma_commit();
  wgmma_wait<1>();  // dP^T done; dV may still run
  fence_acc(dp);
  uint32_t sa[NJ][4];
#pragma unroll
  for (int i = 0; i < 2 * NJ; ++i) {
    const int q = q0 + 8 * i + 2 * (lane & 3);
    const float2 D = *reinterpret_cast<const float2*>(sm.D + q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float& x = dp[4 * i + e];
      x = s[4 * i + e] * (x - ((e & 1) ? D.y : D.x));
    }
  }
  // dS_kt rows q0 + 16 j + 8 (m / 2) + i, key chunk 2 w + m % 2 <- matrix m = register m of the slice, transposed
  const int m = lane >> 3, r = lane & 7;
  const uint32_t dst = sm.dS + kt * sm.QP * ROW_BYTES;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    to_a(sa[j], dp, j);
    stmatrix_x4_trans(dst + swz(q0 + 16 * j + 8 * (m >> 1) + r, 2 * w + (m & 1)), sa[j][0], sa[j][1], sa[j][2], sa[j][3]);
  }
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < NJ; ++j) wgmma_m64n64_rs<1>(dk, sa[j], desc_mn(sm.Q + (q0 + 16 * j) * ROW_BYTES), acc | j);
  wgmma_commit();
}

__global__ void __launch_bounds__(WG_THREADS, 1) attn_bwd_wg(const __grid_constant__ AttnWgArgs a) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  const AttnParams& p = a.p;
  const int h = blockIdx.x, b = blockIdx.y;
  const int T = p.T, W = p.W, ld3 = 3 * W, QP = round16(T), KP = round64(T), NB = KP / 64;
  const uint32_t raw = ptx::smem_u32(smem_raw), base = (raw + 1023u) & ~1023u;
  Smem sm;
  sm.QP = QP;
  sm.dS = base;
  sm.K = sm.dS + NB * QP * ROW_BYTES;
  sm.V = sm.K + KP * ROW_BYTES;
  sm.Q = sm.V + KP * ROW_BYTES;
  sm.dO = sm.Q + QP * ROW_BYTES;
  float* Ls = reinterpret_cast<float*>(smem_raw + (sm.dO + QP * ROW_BYTES - raw));
  float* Ds = Ls + QP;
  sm.L = Ls;
  sm.D = Ds;
  uint64_t* bar = reinterpret_cast<uint64_t*>(Ds + QP);

  if (threadIdx.x == 0) {
    prefetch_tmap(&a.kv);
    prefetch_tmap(&a.q);
    prefetch_tmap(&a.d_o);
    for (int i = 0; i <= NB; ++i) mbar_init(&bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  // Every SM asks for its whole pair at once, so what the first MMAs wait for is requested first: dO and O (D = dO . O is
  // needed before any dS), then K, V and Q block by block.  O goes to registers, all loads before any use (one memory
  // latency for the pair).
  uint8_t* gen = smem_raw - raw;  // generic pointer of shared address 0 for the TMA helpers
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar[NB], QP * ROW_BYTES);
    for (int r = 0; r < QP; r += 16) tma_load_4d(&a.d_o, &bar[NB], gen + sm.dO + r * ROW_BYTES, 64 * h, r, b, 0);
  }
  constexpr int PRO = (WG_MAX_T + 15) / 16 * 16 * 8 / WG_THREADS + 1;  // 16-byte chunks per thread at QP = 208 (6.5)
  uint4 o16[PRO];
  float lse[PRO];
#pragma unroll
  for (int k = 0; k < PRO; ++k) {
    const int i = threadIdx.x + k * WG_THREADS, r = i >> 3;
    o16[k] = make_uint4(0, 0, 0, 0);
    lse[k] = 0.f;
    if (r < T) {
      o16[k] = *reinterpret_cast<const uint4*>(p.o + (size_t)(b * T + r) * W + h * 64 + (i & 7) * 8);
      if ((i & 7) == 0) lse[k] = p.lse[(size_t)(b * p.H + h) * T + r];
    }
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < NB; ++i) {
      const int r1 = min(64 * i + 64, QP);
      mbar_arrive_expect_tx(&bar[i], 2 * TILE + (r1 - 64 * i) * ROW_BYTES);
      tma_load_4d(&a.kv, &bar[i], gen + sm.K + i * TILE, W + 64 * h, 64 * i, b, 0);
      tma_load_4d(&a.kv, &bar[i], gen + sm.V + i * TILE, 2 * W + 64 * h, 64 * i, b, 0);
      for (int r = 64 * i; r < r1; r += 16) tma_load_4d(&a.q, &bar[i], gen + sm.Q + r * ROW_BYTES, 64 * h, r, b, 0);
    }
  }
  // D and L; the 8 lanes of a row are adjacent: shuffle-reduce.  dO rows >= T are the tensor map's zeros, as O's.
  mbar_wait(&bar[NB], 0);
#pragma unroll
  for (int k = 0; k < PRO; ++k) {
    const int i = threadIdx.x + k * WG_THREADS, r = i >> 3;
    if (i >= QP * 8) break;  // warp-uniform: QP * 8 is a multiple of 128
    const uint4 dv16 = *reinterpret_cast<const uint4*>(gen + sm.dO + swz(r, i & 7));
    const __half* hv = reinterpret_cast<const __half*>(&dv16);
    const __half* ho = reinterpret_cast<const __half*>(&o16[k]);
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) d += __half2float(hv[j]) * __half2float(ho[j]);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    if ((i & 7) == 0) {
      Ds[r] = d;
      Ls[r] = lse[k] * LOG2E;
    }
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, lane = t & 31, w = t >> 5;
  const float c = p.scale * LOG2E;
  const int row0 = 16 * w + (lane >> 2), col0 = h * 64 + 2 * (lane & 3);  // fragment row / column of register 0
  const int nfull = QP / 64, tail = (QP % 64) / 16;

  for (int kt = wg; kt < NB; kt += 2) {  // phase 1: dK, dV of 64 keys
    mbar_wait(&bar[kt], 0);
    float dk[32], dv[32];
    const int key0 = 64 * kt + row0;
    for (int qc = 0; qc < nfull; ++qc) {
      mbar_wait(&bar[qc], 0);
      dkdv_chunk<4>(dk, dv, sm, kt, 64 * qc, key0, T, c, qc > 0);
    }
    if (tail) {
      mbar_wait(&bar[nfull], 0);
      if (tail == 1) dkdv_chunk<1>(dk, dv, sm, kt, 64 * nfull, key0, T, c, nfull > 0);
      else if (tail == 2) dkdv_chunk<2>(dk, dv, sm, kt, 64 * nfull, key0, T, c, nfull > 0);
      else dkdv_chunk<3>(dk, dv, sm, kt, 64 * nfull, key0, T, c, nfull > 0);
    }
    wgmma_wait<0>();
    fence_acc(dk);
    fence_acc(dv);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int key = key0 + 8 * half;
      if (key >= T) continue;
      __half* row = p.gqkv + (size_t)(b * T + key) * ld3 + col0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = 4 * i + 2 * half;
        *reinterpret_cast<uint32_t*>(row + W + 8 * i) = pack(dk[r] * p.scale, dk[r + 1] * p.scale);
        *reinterpret_cast<uint32_t*>(row + 2 * W + 8 * i) = pack(dv[r], dv[r + 1]);
      }
    }
  }
  fence_proxy_async_smem();  // the stmatrix stores of dS, before phase 2's wgmma reads them
  __syncthreads();

  for (int qt = wg; qt * 64 < QP; qt += 2) {  // phase 2: dQ of 64 queries
    float dq[32];
    wgmma_fence();
    for (int kt = 0; kt < NB; ++kt) {
      const uint64_t ad = desc_k(sm.dS + (kt * QP + qt * 64) * ROW_BYTES), bd = desc_mn(sm.K + kt * TILE);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 1>(dq, ad + 2 * k, bd + k * (2048 >> 4), (kt | k) != 0, 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(dq);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int q = 64 * qt + row0 + 8 * half;
      if (q >= T) continue;
      __half* row = p.gqkv + (size_t)(b * T + q) * ld3 + col0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = 4 * i + 2 * half;
        *reinterpret_cast<uint32_t*>(row + 8 * i) = pack(dq[r] * p.scale, dq[r + 1] * p.scale);
      }
    }
  }
}

}  // namespace

bool attn_bwd_wg_fits(int T) { return T >= 1 && T <= WG_MAX_T && wg_smem(T) <= 227 * 1024; }

int attn_bwd_wg_prepare(AttnPlan* plan, char* err, int errlen) {
  const AttnParams& p = plan->p;
  if (!attn_bwd_wg_fits(p.T) || !p.d_o || !p.gqkv || p.causal) {
    if (err && errlen > 0) snprintf(err, errlen, "attn_bwd_wg needs a non-causal backward with T <= %d", WG_MAX_T);
    return -1;
  }
  plan->wg.p = p;
  const uint64_t B = p.B, T = p.T, W = p.W;
  const uint64_t qkv_dims[4] = {3 * W, T, B, 1}, qkv_str[3] = {3 * W, T * 3 * W, B * T * 3 * W};
  const uint64_t do_dims[4] = {W, T, B, 1}, do_str[3] = {W, T * W, B * T * W};
  const uint32_t box64[4] = {64, 64, 1, 1}, box16[4] = {64, 16, 1, 1};
  int rc = tmap_encode_4d(&plan->wg.kv, p.qkv, 0, qkv_dims, qkv_str, box64, err, errlen);
  if (!rc) rc = tmap_encode_4d(&plan->wg.q, p.qkv, 0, qkv_dims, qkv_str, box16, err, errlen);
  if (!rc) rc = tmap_encode_4d(&plan->wg.d_o, p.d_o, 0, do_dims, do_str, box16, err, errlen);
  if (rc) return rc;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncSetAttribute(attn_bwd_wg, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_smem(WG_MAX_T));
  });
  plan->smem_bwd = wg_smem(p.T);
  return 0;
}

void attn_bwd_wg_launch(const AttnPlan& plan, cudaStream_t st) {
  launch_pdl(attn_bwd_wg, dim3(plan.p.H, plan.p.B), dim3(WG_THREADS), plan.smem_bwd, st, plan.wg);
}

}  // namespace pxr
