// Nearest codebook row (vqgan.py:60-64) with the distance matrix on the tensor cores and the decision in exact fp32.
//
// vq_partial_kernel (kernels_decoder.cu) evaluates |x|^2 + |c|^2 - 2 x.c for all hw x n_e pairs with fp32 FMAs: 1.07 G FMAs =
// slow at config 2 (256 positions, 16384 codes, 256 channels) for 2 GFLOP.  Here:
//   1. vq_prep: z [C, hw] fp32 -> zh [hw, C] fp16, each position scaled by a power of two into fp16's normal range;
//      |x|^2 and the error-bound terms |x|_2, |x|_1 per position;
//   2. one wgmma GEMM (gemm_tc.cu): scores[p, j] = zh[p, :] . cbh[j, :]  (fp16 operands, fp32 accumulate, 2 GFLOP);
//   3. vq_select: per position the approximate distances d~ = |c|^2 - 2 x.c~, their minimum, every code whose d~ lies
//      within the ROUNDING BOUND of that minimum (a handful), and for those candidates the exact fp32 evaluation -- the
//      same FMA chain over k = 0 .. C-1 and the same expression as vq_partial_kernel -- with first-index ties.  The true
//      fp32 arg-min is always among the candidates (bound below), so the chosen index is the one the all-fp32 search picks.
//      If a position ever collects more candidates than the list holds, it falls back to the exact search over all codes.
// Bound: operands rounded to fp16 (relative 2^-11 in the normal range, absolute 2^-25 below it), products exact, fp32
// accumulation over K terms:  |x.c~ - x.c| <= 2^-9 |x|_2 |c|_2 + 2^-22 (|x|_1 + |c|_1) in the scaled units -- twice the
// worst case, deliberately.  With e that bound, d~(j*) <= min_j d~(j) + 4 e for the exact minimiser j*.
#include <cfloat>

#include "kernels.cuh"
#include "launch.cuh"

namespace pxr {
namespace {

constexpr int VQS_THREADS = 256;
constexpr int VQS_MAX_PER_THREAD = 64;  // n_e <= 256 * 64 = 16384 codes per position row kept in registers
constexpr int VQS_CAND = 256;

// one block per position
__global__ void __launch_bounds__(256) vq_prep_kernel(const float* __restrict__ z, int C, int hw, act_t* __restrict__ zh,
                                                      float* __restrict__ pinfo) {
  pdl_prologue();
  const int p = blockIdx.x;
  __shared__ float red[3][8];
  float amax = 0.f, l1 = 0.f;
  for (int k = threadIdx.x; k < C; k += blockDim.x) {
    const float v = fabsf(z[(size_t)k * hw + p]);
    amax = fmaxf(amax, v);
    l1 += v;
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    l1 += __shfl_xor_sync(0xffffffffu, l1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = amax;
    red[1][threadIdx.x >> 5] = l1;
  }
  __syncthreads();
  amax = 0.f;
  l1 = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
    amax = fmaxf(amax, red[0][w]);
    l1 += red[1][w];
  }
  // power-of-two scale bringing the largest |x_k| into [0.5, 1): exact to apply and to undo
  int e = 0;
  if (amax > 0.f && amax < FLT_MAX) frexpf(amax, &e);
  const float scale = ldexpf(1.f, -e);
  for (int k = threadIdx.x; k < C; k += blockDim.x)
    zh[(size_t)p * C + k] = __float2half_rn(z[(size_t)k * hw + p] * scale);
  if (threadIdx.x == 0) {
    // |x|^2 exactly as vq_partial_kernel sums it (one thread, k ascending), and |x|_2 for the bound
    float s = 0.f;
    for (int k = 0; k < C; ++k) {
      const float v = z[(size_t)k * hw + p];
      s += v * v;
    }
    pinfo[4 * p + 0] = s;
    pinfo[4 * p + 1] = scale;
    pinfo[4 * p + 2] = sqrtf(s) * 1.0000002f;  // |x|_2 (unscaled), rounded up
    pinfo[4 * p + 3] = l1 * 1.0001f;           // |x|_1 (unscaled), rounded up (fp32 sum of <= 1024 terms)
  }
}

__device__ __forceinline__ bool vq_better(float d, int j, float bd, int bj) { return d < bd || (d == bd && j < bj); }

// exact fp32 distance of position p (column xs[0..C)) to code j: the FMA chain and the expression of vq_partial_kernel
__device__ __forceinline__ float vq_exact(const float* __restrict__ xs, const float* __restrict__ cb_row, int C, float x2,
                                          float c2j) {
  float acc = 0.f;
  for (int k = 0; k < C; ++k) acc = fmaf(xs[k], cb_row[k], acc);
  return (x2 + c2j) - 2.f * acc;
}

// scores: [hw, ld] fp32 = (scale_p * x_p) . (cb_scale * c_j); cb: [n_e, C] fp32; bound terms: cmax2 = max_j |c_j|_2,
// cmax1 = max_j |c_j|_1 (unscaled).  One block per position.
__global__ void __launch_bounds__(VQS_THREADS) vq_select_kernel(const float* __restrict__ scores, int ld,
                                                                const float* __restrict__ z, const float* __restrict__ cb,
                                                                const float* __restrict__ c2, const float* __restrict__ pinfo,
                                                                float cb_scale, float cmax2, float cmax1, int C, int hw,
                                                                int n_e, int* __restrict__ idx, act_t* __restrict__ zq,
                                                                int* __restrict__ stats) {
  pdl_prologue();
  extern __shared__ float xs[];  // [C]
  __shared__ float rmin[VQS_THREADS / 32];
  __shared__ float rd[VQS_THREADS / 32];
  __shared__ int rj[VQS_THREADS / 32];
  __shared__ int cand[VQS_CAND];
  __shared__ int ncand;
  __shared__ int s_best;
  const int p = blockIdx.x, tid = threadIdx.x;
  const float x2 = pinfo[4 * p], scale = pinfo[4 * p + 1], xn2 = pinfo[4 * p + 2], xn1 = pinfo[4 * p + 3];
  for (int k = tid; k < C; k += VQS_THREADS) xs[k] = z[(size_t)k * hw + p];
  if (tid == 0) ncand = 0;
  // unscale factor of the scores (both scales are powers of two: exact)
  const float inv = 1.f / (scale * cb_scale);
  // the bound in unscaled units: the absolute (sub-normal) term was incurred on the scaled operands
  const float eps_dot = 0.001953125f * xn2 * cmax2 + 2.3841858e-07f * inv * (xn1 * scale + cmax1 * cb_scale);
  const float slack = 4.f * eps_dot + 1e-5f * (x2 + cmax2 * cmax2);
  float dt[VQS_MAX_PER_THREAD];
  float lmin = FLT_MAX;
  const float* row = scores + (size_t)p * ld;
#pragma unroll
  for (int u = 0; u < VQS_MAX_PER_THREAD / 4; ++u) {
    const int j = 4 * (tid + u * VQS_THREADS);
    if (j < n_e) {  // n_e % 4 == 0 (checked by the launcher)
      const float4 s = __ldcs(reinterpret_cast<const float4*>(row + j));
      const float4 c = *reinterpret_cast<const float4*>(c2 + j);
      dt[4 * u + 0] = c.x - 2.f * (s.x * inv);
      dt[4 * u + 1] = c.y - 2.f * (s.y * inv);
      dt[4 * u + 2] = c.z - 2.f * (s.z * inv);
      dt[4 * u + 3] = c.w - 2.f * (s.w * inv);
      lmin = fminf(lmin, fminf(fminf(dt[4 * u], dt[4 * u + 1]), fminf(dt[4 * u + 2], dt[4 * u + 3])));
    } else {
      dt[4 * u] = dt[4 * u + 1] = dt[4 * u + 2] = dt[4 * u + 3] = FLT_MAX;
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
  if ((tid & 31) == 0) rmin[tid >> 5] = lmin;
  __syncthreads();
  float gmin = rmin[0];
#pragma unroll
  for (int w = 1; w < VQS_THREADS / 32; ++w) gmin = fminf(gmin, rmin[w]);
  const float thr = gmin + slack;
#pragma unroll
  for (int u = 0; u < VQS_MAX_PER_THREAD / 4; ++u) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (dt[4 * u + i] <= thr) {
        const int slot = atomicAdd(&ncand, 1);
        if (slot < VQS_CAND) cand[slot] = 4 * (tid + u * VQS_THREADS) + i;
      }
    }
  }
  __syncthreads();
  const int nc = ncand;
  float bd = FLT_MAX;
  int bj = 0x7fffffff;
  if (nc <= VQS_CAND) {
    for (int i = tid; i < nc; i += VQS_THREADS) {
      const int j = cand[i];
      const float d = vq_exact(xs, cb + (size_t)j * C, C, x2, c2[j]);
      if (vq_better(d, j, bd, bj)) {
        bd = d;
        bj = j;
      }
    }
  } else {  // the list overflowed (a flat neighbourhood): exact search over every code
    for (int j = tid; j < n_e; j += VQS_THREADS) {
      const float d = vq_exact(xs, cb + (size_t)j * C, C, x2, c2[j]);
      if (vq_better(d, j, bd, bj)) {
        bd = d;
        bj = j;
      }
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const float od = __shfl_xor_sync(0xffffffffu, bd, o);
    const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (vq_better(od, oj, bd, bj)) {
      bd = od;
      bj = oj;
    }
  }
  if ((tid & 31) == 0) {
    rd[tid >> 5] = bd;
    rj[tid >> 5] = bj;
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < VQS_THREADS / 32; ++w)
      if (vq_better(rd[w], rj[w], bd, bj)) {
        bd = rd[w];
        bj = rj[w];
      }
    s_best = bj;
    idx[p] = bj;
    if (stats) {  // diagnostics: total candidates, overflowed positions
      atomicAdd(&stats[0], nc);
      if (nc > VQS_CAND) atomicAdd(&stats[1], 1);
    }
  }
  __syncthreads();
  const float* best = cb + (size_t)s_best * C;
  for (int k = tid; k < C; k += VQS_THREADS) zq[(size_t)p * C + k] = __float2half_rn(best[k]);
}

}  // namespace

bool vq_tc_supported(int C, int n_e) { return C % 64 == 0 && n_e % 8 == 0 && n_e <= VQS_THREADS * VQS_MAX_PER_THREAD; }

void vq_prep(const float* z, int C, int hw, act_t* zh, float* pinfo, cudaStream_t st) {
  launch_pdl(vq_prep_kernel, dim3(hw), dim3(256), 0, st, z, C, hw, zh, pinfo);
}

void vq_select(const float* scores, int ld, const float* z, const float* cb, const float* c2, const float* pinfo,
               float cb_scale, float cmax2, float cmax1, int C, int hw, int n_e, int* idx, act_t* zq, int* stats,
               cudaStream_t st) {
  launch_pdl(vq_select_kernel, dim3(hw), dim3(VQS_THREADS), C * sizeof(float), st, scores, ld, z, cb, c2, pinfo, cb_scale,
             cmax2, cmax1, C, hw, n_e, idx, zq, stats);
}

}  // namespace pxr
