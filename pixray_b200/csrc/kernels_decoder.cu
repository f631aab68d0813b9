// VQGAN-drawer side kernels: nearest-code search, GroupNorm(+swish) fwd/bwd, nearest upsample and its adjoint,
// image finish (clamp_with_grad) and the pixel drawer.  All HBM/L2-bound; vectorised 16-byte accesses on NHWC fp16.
#include "kernels.cuh"
#include "launch.cuh"
#include <cooperative_groups.h>
#include <cfloat>

namespace pxr {

namespace {

constexpr int VQ_POS = 16;    // latent positions per block
constexpr int VQ_CODES = 1024;  // codes per block (4 per thread)

// grid (n_e / VQ_CODES, ceil(hw / VQ_POS)), block 256.
__global__ void __launch_bounds__(256) vq_partial_kernel(const float* __restrict__ z, const float* __restrict__ cbT,
                                                         const float* __restrict__ c2, int C, int hw, int n_e,
                                                         int n_chunks, float* __restrict__ part_d,
                                                         int* __restrict__ part_i) {
  pdl_prologue();
  extern __shared__ float xs[];  // [C][VQ_POS]
  __shared__ float x2[VQ_POS];
  __shared__ float red_d[8][VQ_POS];
  __shared__ int red_i[8][VQ_POS];
  const int p0 = blockIdx.y * VQ_POS;
  const int j0 = blockIdx.x * VQ_CODES;
  for (int i = threadIdx.x; i < C * VQ_POS; i += 256) {
    int k = i / VQ_POS, p = i % VQ_POS;
    xs[i] = (p0 + p < hw) ? z[(size_t)k * hw + p0 + p] : 0.f;
  }
  __syncthreads();
  if (threadIdx.x < VQ_POS) {
    float s = 0.f;
    for (int k = 0; k < C; ++k) s += xs[k * VQ_POS + threadIdx.x] * xs[k * VQ_POS + threadIdx.x];
    x2[threadIdx.x] = s;
  }
  float acc[4][VQ_POS];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int p = 0; p < VQ_POS; ++p) acc[c][p] = 0.f;
#pragma unroll 4  // four k-slices of codebook loads in flight per thread: the loop is L2-latency bound otherwise
  for (int k = 0; k < C; ++k) {
    float cv[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      int j = j0 + threadIdx.x + 256 * c;
      cv[c] = j < n_e ? cbT[(size_t)k * n_e + j] : 0.f;
    }
    const float4* xr = reinterpret_cast<const float4*>(xs + k * VQ_POS);
#pragma unroll
    for (int p4 = 0; p4 < VQ_POS / 4; ++p4) {
      float4 xv = xr[p4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc[c][4 * p4 + 0] = fmaf(xv.x, cv[c], acc[c][4 * p4 + 0]);
        acc[c][4 * p4 + 1] = fmaf(xv.y, cv[c], acc[c][4 * p4 + 1]);
        acc[c][4 * p4 + 2] = fmaf(xv.z, cv[c], acc[c][4 * p4 + 2]);
        acc[c][4 * p4 + 3] = fmaf(xv.w, cv[c], acc[c][4 * p4 + 3]);
      }
    }
  }
  __syncthreads();
  // d = (|x|^2 + |c|^2) - 2 x.c   (vqgan.py:61), first-minimum wins ties like argmin
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int p = 0; p < VQ_POS; ++p) {
    float best = FLT_MAX;
    int bi = 0x7fffffff;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      int j = j0 + threadIdx.x + 256 * c;
      if (j < n_e) {
        float d = (x2[p] + c2[j]) - 2.f * acc[c][p];
        if (d < best || (d == best && j < bi)) {
          best = d;
          bi = j;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float od = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (od < best || (od == best && oi < bi)) {
        best = od;
        bi = oi;
      }
    }
    if (lane == 0) {
      red_d[warp][p] = best;
      red_i[warp][p] = bi;
    }
  }
  __syncthreads();
  if (threadIdx.x < VQ_POS && p0 + threadIdx.x < hw) {
    float best = red_d[0][threadIdx.x];
    int bi = red_i[0][threadIdx.x];
    for (int w = 1; w < 8; ++w) {
      float od = red_d[w][threadIdx.x];
      int oi = red_i[w][threadIdx.x];
      if (od < best || (od == best && oi < bi)) {
        best = od;
        bi = oi;
      }
    }
    part_d[(size_t)(p0 + threadIdx.x) * n_chunks + blockIdx.x] = best;
    part_i[(size_t)(p0 + threadIdx.x) * n_chunks + blockIdx.x] = bi;
  }
}

// one block per position: final argmin over chunks, gather the code row as fp16
__global__ void vq_final_kernel(const float* __restrict__ part_d, const int* __restrict__ part_i, int n_chunks,
                                const float* __restrict__ cb, int C, int* __restrict__ idx, act_t* __restrict__ zq) {
  pdl_prologue();
  const int p = blockIdx.x;
  __shared__ int s_idx;
  if (threadIdx.x == 0) {
    float best = part_d[(size_t)p * n_chunks];
    int bi = part_i[(size_t)p * n_chunks];
    for (int c = 1; c < n_chunks; ++c) {
      float od = part_d[(size_t)p * n_chunks + c];
      int oi = part_i[(size_t)p * n_chunks + c];
      if (od < best || (od == best && oi < bi)) {
        best = od;
        bi = oi;
      }
    }
    s_idx = bi;
    idx[p] = bi;
  }
  __syncthreads();
  const float* row = cb + (size_t)s_idx * C;
  for (int k = threadIdx.x; k < C; k += blockDim.x) zq[(size_t)p * C + k] = __float2half_rn(row[k]);
}

__global__ void vq_backward_kernel(const act_t* __restrict__ dzq, float inv_scale, int C, int hw,
                                   float* __restrict__ z_grad) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // over [C, hw]
  if (i >= C * hw) return;
  int k = i / hw, p = i % hw;
  z_grad[i] = __half2float(dzq[(size_t)p * C + k]) * inv_scale;
}

// ------------------------------------------------------------------ GroupNorm
constexpr int GN_G = 32;
constexpr int GN_TARGET_BLOCKS = 592;  // ~4 per SM
__host__ __device__ inline int gn_rows_per_block(int pixels) {
  int r = (pixels + GN_TARGET_BLOCKS - 1) / GN_TARGET_BLOCKS;
  r = (r + 31) / 32 * 32;
  return r < 32 ? 32 : r;
}

__device__ __forceinline__ void load8(const act_t* p, float (&f)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ void store8(act_t* p, const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

// The shift gn_partial_kernel subtracts for its pivoted sums: x at pixel 0 in group g's first channel, one value per group
// that every block reads alike.
__device__ __forceinline__ float gn_pivot(const act_t* x, int C, int g) { return __half2float(x[g * (C / GN_G)]); }

// Fixed-order block reduction of the thread sums s[half][a/b] to out[32 groups][2] (no atomics: every rank of the
// cutout-sharded mode must produce the same bits, and so must every run): pixel lanes -> channel vector -> group.
__device__ __forceinline__ void gn_block_reduce(const float (&s)[2][2], float (*red)[256], float (*acc)[2], int vecs, int cpg,
                                                float* __restrict__ out) {
  const int vc = threadIdx.x % vecs, pl = threadIdx.x / vecs, plane = 256 / vecs;
  red[0][threadIdx.x] = s[0][0];
  red[1][threadIdx.x] = s[0][1];
  red[2][threadIdx.x] = s[1][0];
  red[3][threadIdx.x] = s[1][1];
  __syncthreads();
  if (pl == 0) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    for (int l = 0; l < plane; ++l)
#pragma unroll
      for (int k = 0; k < 4; ++k) t[k] += red[k][l * vecs + vc];
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][vc] = t[k];  // slot vc belongs to lane pl == 0 of this vector: no hazard
  }
  __syncthreads();
  if (threadIdx.x < GN_G * 2) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    float t = 0.f;
    if (cpg >= 8) {
      const int vpg = cpg / 8;
      for (int v = g * vpg; v < (g + 1) * vpg; ++v) t += red[which][v] + red[2 + which][v];
    } else {  // cpg == 4: a vector holds two groups
      t = red[(g & 1) * 2 + which][g >> 1];
    }
    acc[g][which] = t;
  }
  __syncthreads();
  if (threadIdx.x < GN_G * 2) out[threadIdx.x] = (&acc[0][0])[threadIdx.x];
}

// Accumulates, per group, sum(a) and sum(b) where (a, b) = F(element).  MODE 0: (x, x^2) into part[block], and
// (d, d^2) with d = x - pivot into part[gridDim.x + block], the pivot of a group being x at pixel 0 in the group's first
// channel (gn_pivot): gn_final_kernel takes the statistics from the second set where the first loses its precision
// (gn_refine_variance).  MODE 1: backward sums (dxh, dxh * xh).  Block: 256 threads = (256 / (C/8)) pixel lanes x (C/8)
// channel vectors.  one_group (GroupNorm(1, C)): every group's pivot is x[0, 0], so gn_final_kernel can merge the groups'
// pivoted sums; act: 0 none, 1 swish, 2 ReLU (its mask in the backward); gamma_add is added to gamma (null gamma / beta: 0).
template <int MODE>
__global__ void __launch_bounds__(256) gn_partial_kernel(const act_t* __restrict__ x, const act_t* __restrict__ dy,
                                                         const float* __restrict__ stats,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, int pixels, int C, int swish,
                                                         float* __restrict__ part, float gamma_add, int one_group) {
  pdl_prologue();
  __shared__ float acc[GN_G][2];
  const int vecs = C / 8, cpg = C / GN_G;
  const int vc = threadIdx.x % vecs, pl = threadIdx.x / vecs, plane = 256 / vecs;
  const int c0 = vc * 8;
  const int rpb = gn_rows_per_block(pixels);
  const int p_begin = blockIdx.x * rpb;
  const int p_end = min(pixels, p_begin + rpb);
  float s[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // [half][a/b] : halves of the 8-vector (cpg == 4 splits groups)
  float sp[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // MODE 0: the pivoted sums
  float g8[8], b8[8], mean8[8], rstd8[8], pv[2];
  if (MODE == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) pv[h] = gn_pivot(x, C, one_group ? 0 : (c0 + 4 * h) / cpg);
  }
  if (MODE == 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      g8[i] = gamma ? gamma[c0 + i] : 0.f;
      if (gamma_add != 0.f) g8[i] += gamma_add;
      b8[i] = beta ? beta[c0 + i] : 0.f;
      int g = (c0 + i) / cpg;
      mean8[i] = stats[2 * g];
      rstd8[i] = stats[2 * g + 1];
    }
  }
  for (int p = p_begin + pl; p < p_end; p += plane) {
    float xv[8];
    load8(x + (size_t)p * C + c0, xv);
    if (MODE == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i >> 2][0] += xv[i];
        s[i >> 2][1] += xv[i] * xv[i];
        const float d = xv[i] - pv[i >> 2];
        sp[i >> 2][0] += d;
        sp[i >> 2][1] += d * d;
      }
    } else {
      float dv[8];
      load8(dy + (size_t)p * C + c0, dv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float xh = (xv[i] - mean8[i]) * rstd8[i];
        float d = dv[i];
        if (swish == 1) {
          float a = g8[i] * xh + b8[i];
          float sg = 1.f / (1.f + __expf(-a));
          d *= sg * (1.f + a * (1.f - sg));
        } else if (swish == 2) {
          d = (g8[i] * xh + b8[i]) > 0.f ? d : 0.f;
        }
        float dxh = d * g8[i];
        s[i >> 2][0] += dxh;
        s[i >> 2][1] += dxh * xh;
      }
    }
  }
  __shared__ float red[4][256];
  gn_block_reduce(s, red, acc, vecs, cpg, part + (size_t)blockIdx.x * GN_G * 2);
  if (MODE == 0) gn_block_reduce(sp, red, acc, vecs, cpg, part + (size_t)(gridDim.x + blockIdx.x) * GN_G * 2);
}

// MODE 0: stats[g] = (mean, rstd), from the plain sums or, where those lose their precision, from the pivoted ones
// (x: the tensor, for the pivots).  MODE 1: gstats[g] = (mean dxh, mean dxh*xh).  One block of 256 threads.
// one_group: the 32 equal-sized groups' means are averaged into the whole tensor's before anything is derived from them.
template <int MODE>
__global__ void gn_final_kernel(const float* __restrict__ part, int nblk, double count, float eps, const act_t* x, int C,
                                float* __restrict__ out, int one_group) {
  pdl_prologue();
  const int t = threadIdx.x & 63, q = threadIdx.x >> 6;  // 256 threads: slot (group, which) x quarter of the partials
  double s = 0.0, sp = 0.0;
  for (int b = q; b < nblk; b += 4) s += (double)part[(size_t)b * GN_G * 2 + t];
  if (MODE == 0)
    for (int b = q; b < nblk; b += 4) sp += (double)part[(size_t)(nblk + b) * GN_G * 2 + t];
  __shared__ double acc4[4][GN_G * 2], acc4p[4][GN_G * 2];
  __shared__ double sh[GN_G * 2], shp[GN_G * 2];
  acc4[q][t] = s;
  acc4p[q][t] = sp;
  __syncthreads();
  if (q == 0) {
    sh[t] = (acc4[0][t] + acc4[1][t] + acc4[2][t] + acc4[3][t]) / count;
    shp[t] = (acc4p[0][t] + acc4p[1][t] + acc4p[2][t] + acc4p[3][t]) / count;
  }
  __syncthreads();
  if (one_group && threadIdx.x < 4) {  // thread k merges one of sh[even], sh[odd], shp[even], shp[odd]: fixed order
    double* v = threadIdx.x < 2 ? sh : shp;
    const int which = threadIdx.x & 1;
    double a = 0.0;
    for (int g = 0; g < GN_G; ++g) a += v[2 * g + which];
    a /= GN_G;
    for (int g = 0; g < GN_G; ++g) v[2 * g + which] = a;
  }
  __syncthreads();
  if (q != 0) return;
  if (MODE == 0) {
    if ((t & 1) == 0) {
      double mean = sh[t], var = sh[t + 1] - mean * mean;
      if (var < 0) var = 0;
      if (gn_refine_variance(mean, var)) {
        const double md = shp[t];
        mean = gn_pivot(x, C, one_group ? 0 : t >> 1) + md;
        var = shp[t + 1] - md * md;
        if (var < 0) var = 0;
      }
      out[t] = (float)mean;
      out[t + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  } else {
    out[t] = (float)sh[t];
  }
}

__global__ void __launch_bounds__(256) gn_apply_kernel(const act_t* __restrict__ x, const float* __restrict__ stats,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       long long nvec, int C, int swish, act_t* __restrict__ y,
                                                       float gamma_add, const act_t* __restrict__ res) {
  pdl_prologue();
  const int cpg = C / GN_G, vecs = C / 8;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < nvec;
       v += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(v % vecs) * 8;
    float xv[8], rv[8];
    load8(x + v * 8, xv);
    if (res) load8(res + v * 8, rv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int g = (c0 + i) / cpg;
      float ga = gamma ? gamma[c0 + i] : 0.f;
      if (gamma_add != 0.f) ga += gamma_add;
      float a = (xv[i] - stats[2 * g]) * stats[2 * g + 1] * ga + (beta ? beta[c0 + i] : 0.f);
      a = swish == 1 ? a / (1.f + __expf(-a)) : (swish == 2 ? fmaxf(a, 0.f) : a);
      xv[i] = res ? a + rv[i] : a;
    }
    store8(y + v * 8, xv);
  }
}

__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const act_t* __restrict__ dy, const act_t* __restrict__ x,
                                                           const float* __restrict__ stats,
                                                           const float* __restrict__ gstats,
                                                           const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, long long nvec, int C,
                                                           int swish, const act_t* __restrict__ dres,
                                                           act_t* __restrict__ dx, float gamma_add) {
  pdl_prologue();
  const int cpg = C / GN_G, vecs = C / 8;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < nvec;
       v += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(v % vecs) * 8;
    float xv[8], dv[8], rv[8];
    load8(x + v * 8, xv);
    load8(dy + v * 8, dv);
    if (dres) load8(dres + v * 8, rv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int g = (c0 + i) / cpg;
      float rstd = stats[2 * g + 1];
      float xh = (xv[i] - stats[2 * g]) * rstd;
      float d = dv[i];
      float ga = gamma ? gamma[c0 + i] : 0.f;
      if (gamma_add != 0.f) ga += gamma_add;
      const float be = beta ? beta[c0 + i] : 0.f;
      if (swish == 1) {
        float a = ga * xh + be;
        float sg = 1.f / (1.f + __expf(-a));
        d *= sg * (1.f + a * (1.f - sg));
      } else if (swish == 2) {
        d = (ga * xh + be) > 0.f ? d : 0.f;
      }
      float dxh = d * ga;
      float r = rstd * (dxh - gstats[2 * g] - xh * gstats[2 * g + 1]);
      xv[i] = dres ? r + rv[i] : r;
    }
    store8(dx + v * 8, xv);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm in ONE cooperative kernel per direction (replaces partial + final + apply: 3 launches, 2 passes over x).
// The grid (<= one 1024-thread block per SM) splits the pixels into contiguous slabs; a block keeps its slab of x
// (and dy when it fits) in shared memory, so every tensor is read from HBM once.  Statistics: block partials in a fixed
// order -> global scratch -> grid-wide barrier -> every block folds all partials in the same fixed order (double
// accumulation).  No atomics anywhere: identical bits on every run and on every rank of the cutout-sharded mode.
constexpr int GNC_THREADS = 1024;

// Grid-wide barrier for a grid of at most one block per SM.  INVARIANT (the launchers enforce it: gnc_rows_per_block gives grid <= num_sms): gridDim.x
// <= num_sms with 1024-thread blocks whose shared memory leaves room for one of them per SM, and nothing else that could pin
// an SM forever runs on the device -- the engine's stream runs one kernel at a time; under programmatic dependent launch the
// previous kernel's blocks may still hold SMs when the first blocks of this one start, but they finish on their own, and
// this kernel's own dependents are only released once every one of its blocks is resident (griddepcontrol.launch_dependents
// is issued per block).  A plain launch plus this barrier avoids the extra launch cost of cudaLaunchCooperativeKernel +
// grid.sync(), which matters at 78 GroupNorm calls per iteration.  `counter` only ever
// grows: the launcher passes the value it must reach (count before the launch + gridDim.x), so no reset and no generation
// bit is needed.  The spin is bounded: ~2 s of SM clocks (2^32) without progress traps the kernel, so a violated invariant
// (a debugger or sanitizer serialising blocks, a foreign persistent kernel on the device) surfaces as a launch failure on
// the next CUDA call instead of a hang.  compute-sanitizer runs use PXR_GN_COOP=0 (the three-kernel variant).
__device__ __forceinline__ void gnc_grid_barrier(unsigned long long* counter, unsigned long long target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1ULL);
    unsigned long long v;
    const long long t0 = clock64();
    unsigned spins = 0;
    do {
      asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(counter) : "memory");
      if (v < target && (++spins & 0x3ffu) == 0 && clock64() - t0 > (1LL << 32)) __trap();
    } while (v < target);
  }
  __syncthreads();
}

// per-block fixed-order reduction of the thread partials s[half][a/b] to part_out[32 groups][2].
// Threads (vc, pl) hold the sums of vector column vc over the pixels of plane pl: a fixed-shape binary tree over the
// planes (plane = GNC_THREADS / vecs is a power of two for every supported C) -- log2(plane) barriers instead of a
// serial walk over up to 64 planes by `vecs` threads (a chain of dependent shared-memory loads).
__device__ __forceinline__ void gnc_block_partials(const float (&s)[2][2], float* red, int vecs, int cpg,
                                                   float* __restrict__ part_out) {
  const int tid = threadIdx.x, vc = tid % vecs, pl = tid / vecs, plane = GNC_THREADS / vecs;
  red[0 * GNC_THREADS + tid] = s[0][0];
  red[1 * GNC_THREADS + tid] = s[0][1];
  red[2 * GNC_THREADS + tid] = s[1][0];
  red[3 * GNC_THREADS + tid] = s[1][1];
  for (int stride = plane >> 1; stride >= 1; stride >>= 1) {
    __syncthreads();
    if (pl < stride) {
#pragma unroll
      for (int k = 0; k < 4; ++k) red[k * GNC_THREADS + tid] += red[k * GNC_THREADS + tid + stride * vecs];
    }
  }
  __syncthreads();
  if (tid < GN_G * 2) {
    const int g = tid >> 1, which = tid & 1;
    float t = 0.f;
    if (cpg >= 8) {
      const int vpg = cpg / 8;
      for (int v = g * vpg; v < (g + 1) * vpg; ++v) t += red[which * GNC_THREADS + v] + red[(2 + which) * GNC_THREADS + v];
    } else {  // cpg == 4: a vector holds two groups
      t = red[((g & 1) * 2 + which) * GNC_THREADS + (g >> 1)];
    }
    part_out[tid] = t;
  }
}

// Thread-block-cluster variant for the small layers (the whole tensor fits the shared memory of <= 16 SMs): the block
// partials stay in shared memory, the hardware cluster barrier replaces the global-memory grid barrier and every block
// folds its peers' partials through distributed shared memory -- no global round trips between the two phases.
__device__ __forceinline__ void gnc_cluster_fold(float* cpart, int nblk, double count, double* acc4, double* sh) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync();  // every block's cpart is written
  const int tid = threadIdx.x;
  if (tid < 256) {
    const int slot = tid & 63, qd = tid >> 6;
    double a = 0.0;
    for (int b = qd; b < nblk; b += 4) a += (double)cluster.map_shared_rank(cpart, b)[slot];  // fixed order
    acc4[qd * 64 + slot] = a;
  }
  __syncthreads();
  if (tid < 64) sh[tid] = (acc4[tid] + acc4[64 + tid] + acc4[128 + tid] + acc4[192 + tid]) / count;
  cluster.sync();  // nobody leaves (or rewrites cpart) while a peer still reads it
}

// every block: fold the nblk (<= GNC_FOLD_MAX) block partials -> sh[64] = per-(group, which) mean.  All 1024 threads
// take part: thread (slot, lane16) loads partials lane16, lane16 + 16, ... with every load issued before the first add
// (ONE L2 round trip after the grid barrier, where the previous 256-thread version paid ~37 dependent ones), then the 16
// lane sums are added in a fixed order in double.
constexpr int GNC_FOLD_LANES = GNC_THREADS / 64;                        // 16
constexpr int GNC_FOLD_MAX = 160;                                       // >= blocks per grid (<= num_sms)
constexpr int GNC_FOLD_PER = (GNC_FOLD_MAX + GNC_FOLD_LANES - 1) / GNC_FOLD_LANES;  // 10
__device__ __forceinline__ void gnc_fold(const float* part, int nblk, double count, double* acc16, double* sh) {
  const int tid = threadIdx.x;
  const int slot = tid & 63, ln = tid >> 6;
  float v[GNC_FOLD_PER];
#pragma unroll
  for (int u = 0; u < GNC_FOLD_PER; ++u) {
    const int b = ln + u * GNC_FOLD_LANES;
    v[u] = b < nblk ? __ldcg(part + (size_t)b * GN_G * 2 + slot) : 0.f;
  }
  double a = 0.0;
#pragma unroll
  for (int u = 0; u < GNC_FOLD_PER; ++u) a += (double)v[u];
  acc16[ln * 64 + slot] = a;
  __syncthreads();
  if (tid < 64) {
    double t = 0.0;
#pragma unroll
    for (int l = 0; l < GNC_FOLD_LANES; ++l) t += acc16[l * 64 + tid];
    sh[tid] = t / count;
  }
  __syncthreads();
}

// GroupNorm(1, C): the 32 equal-sized groups' means (of x, x^2 or of the backward sums) average to the whole-tensor mean
__device__ __forceinline__ void gnc_merge_groups(double* sh) {
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int g = 0; g < GN_G; ++g) {
      a += sh[2 * g];
      b += sh[2 * g + 1];
    }
    a /= GN_G;
    b /= GN_G;
    for (int g = 0; g < GN_G; ++g) {
      sh[2 * g] = a;
      sh[2 * g + 1] = b;
    }
  }
  __syncthreads();
}

template <bool CLUSTER>
__global__ void __launch_bounds__(GNC_THREADS, 1)
    gn_coop_fwd_kernel(const act_t* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                       int pixels, int C, int swish, float eps, int rpb, float* part, float* __restrict__ stats_out,
                       act_t* y, unsigned long long* bar, unsigned long long bar_target, GnOpts o) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t gnc_smem[];
  float* red = reinterpret_cast<float*>(gnc_smem);                       // [4][1024]
  act_t* cx = reinterpret_cast<act_t*>(gnc_smem + 4 * GNC_THREADS * 4);  // slab of x
  __shared__ double acc4[GNC_THREADS];  // gnc_fold: [16 lanes][64 slots]
  __shared__ double sh[64];
  __shared__ float st[64];
  const int vecs = C / 8, cpg = C / GN_G;
  const int vc = threadIdx.x % vecs, pl = threadIdx.x / vecs, plane = GNC_THREADS / vecs;
  const int c0 = vc * 8;
  const int p_begin = blockIdx.x * rpb, p_end = min(pixels, p_begin + rpb);
  float ga8[8], be8[8];  // loaded before the grid barrier: one dependent global round trip less after it
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ga8[i] = (gamma ? gamma[c0 + i] : 0.f) + o.gamma_add;
    be8[i] = beta ? beta[c0 + i] : 0.f;
  }
  float s[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll 4
  for (int p = p_begin + pl; p < p_end; p += plane) {
    const uint4 u = *reinterpret_cast<const uint4*>(x + (size_t)p * C + c0);
    *reinterpret_cast<uint4*>(cx + (size_t)(p - p_begin) * C + c0) = u;
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(h[i]);
      s[i >> 1][0] += t.x + t.y;
      s[i >> 1][1] += t.x * t.x + t.y * t.y;
    }
  }
  __shared__ float cpart[GN_G * 2];
  if (CLUSTER) {
    gnc_block_partials(s, red, vecs, cpg, cpart);
    gnc_cluster_fold(cpart, gridDim.x, (double)pixels * cpg, acc4, sh);
  } else {
    gnc_block_partials(s, red, vecs, cpg, part + (size_t)blockIdx.x * GN_G * 2);
    gnc_grid_barrier(bar, bar_target);
    gnc_fold(part, gridDim.x, (double)pixels * cpg, acc4, sh);
  }
  if (o.one_group) gnc_merge_groups(sh);  // GroupNorm(1, C): every group takes the statistics of the whole tensor
  __shared__ int refine;
  if (threadIdx.x == 0) refine = 0;
  __syncthreads();
  if (threadIdx.x < GN_G) {
    const double mean = sh[2 * threadIdx.x], ex2 = sh[2 * threadIdx.x + 1];
    double var = ex2 - mean * mean;
    if (var < 0) var = 0;
    if (gn_refine_variance(mean, var)) refine = 1;
    st[2 * threadIdx.x] = (float)mean;
    st[2 * threadIdx.x + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  // Every block folded the same partials, so `refine` is the same in the whole grid.  The second pass sums x - mean (the
  // first pass's fp32 mean) over the slab in shared memory; its partials replace the first ones in `part` once every block
  // has read those (second barrier), and are read after the third.  Without it a block adds its two arrivals at once.
  if (refine) {
    float m2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) m2[h] = st[2 * ((c0 + 4 * h) / cpg)];
    float s2[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int p = p_begin + pl; p < p_end; p += plane) {
      float xv[8];
      load8(cx + (size_t)(p - p_begin) * C + c0, xv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = xv[i] - m2[i >> 2];
        s2[i >> 2][0] += d;
        s2[i >> 2][1] += d * d;
      }
    }
    __shared__ float cpart2[GN_G * 2];
    gnc_block_partials(s2, red, vecs, cpg, cpart2);
    if (CLUSTER) {
      gnc_cluster_fold(cpart2, gridDim.x, (double)pixels * cpg, acc4, sh);
    } else {
      gnc_grid_barrier(bar, bar_target + gridDim.x);
      if (threadIdx.x < GN_G * 2) part[(size_t)blockIdx.x * GN_G * 2 + threadIdx.x] = cpart2[threadIdx.x];
      gnc_grid_barrier(bar, bar_target + 2 * gridDim.x);
      gnc_fold(part, gridDim.x, (double)pixels * cpg, acc4, sh);
    }
    if (o.one_group) gnc_merge_groups(sh);
    if (threadIdx.x < GN_G) {
      const double md = sh[2 * threadIdx.x];
      double var = sh[2 * threadIdx.x + 1] - md * md;
      if (var < 0) var = 0;
      st[2 * threadIdx.x] = (float)((double)st[2 * threadIdx.x] + md);
      st[2 * threadIdx.x + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __syncthreads();
  } else if (!CLUSTER && threadIdx.x == 0) {
    atomicAdd(bar, 2ULL);
  }
  if (blockIdx.x == 0 && threadIdx.x < GN_G * 2) stats_out[threadIdx.x] = st[threadIdx.x];
  float sc8[8], sh8[8];  // y = x * sc + sh
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c0 + i) / cpg;
    sc8[i] = st[2 * g + 1] * ga8[i];
    sh8[i] = be8[i] - st[2 * g] * st[2 * g + 1] * ga8[i];
  }
#pragma unroll 4
  for (int p = p_begin + pl; p < p_end; p += plane) {
    float xv[8], rv[8];
    load8(cx + (size_t)(p - p_begin) * C + c0, xv);
    if (o.res) load8(o.res + (size_t)p * C + c0, rv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = xv[i] * sc8[i] + sh8[i];
      const float r = swish == 1 ? a / (1.f + __expf(-a)) : (swish == 2 ? fmaxf(a, 0.f) : a);
      xv[i] = o.res ? r + rv[i] : r;
    }
    store8(y + (size_t)p * C + c0, xv);
  }
}

template <bool CLUSTER>
__global__ void __launch_bounds__(GNC_THREADS, 1)
    gn_coop_bwd_kernel(const act_t* __restrict__ dy, const act_t* __restrict__ x, const float* __restrict__ stats,
                       const float* __restrict__ gamma, const float* __restrict__ beta, int pixels, int C, int swish,
                       const act_t* dres, int rpb, int cache_dy, float* part, act_t* dx, unsigned long long* bar,
                       unsigned long long bar_target, GnOpts o) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t gnc_smem[];
  float* red = reinterpret_cast<float*>(gnc_smem);
  // The slab kept in shared memory between the two phases is dxh = dy * act'(a) * gamma (fp16), NOT x: the activation's
  // derivative (exp + reciprocal per element) is then evaluated once instead of once per phase -- at the 256^2 level the
  // kernel is bound by exactly those instructions -- and phase 2 re-reads x from L2
  // in place of dy: the same bytes.  (cache_dy is ignored; kept in the signature for the launcher.)
  act_t* cg = reinterpret_cast<act_t*>(gnc_smem + 4 * GNC_THREADS * 4);
  __shared__ double acc4[GNC_THREADS];  // gnc_fold: [16 lanes][64 slots]
  __shared__ double sh[64];
  const int vecs = C / 8, cpg = C / GN_G;
  const int vc = threadIdx.x % vecs, pl = threadIdx.x / vecs, plane = GNC_THREADS / vecs;
  const int c0 = vc * 8;
  const int p_begin = blockIdx.x * rpb, p_end = min(pixels, p_begin + rpb);
  float g8[8], b8[8], mean2[2], rstd2[2];  // cpg >= 4: elements 0..3 and 4..7 of the vector each sit in one group
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    g8[i] = (gamma ? gamma[c0 + i] : 0.f) + o.gamma_add;
    b8[i] = beta ? beta[c0 + i] : 0.f;
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int g = (c0 + 4 * i) / cpg;
    mean2[i] = stats[2 * g];
    rstd2[i] = stats[2 * g + 1];
  }
  float s[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll 2
  for (int p = p_begin + pl; p < p_end; p += plane) {
    const uint4 ux = *reinterpret_cast<const uint4*>(x + (size_t)p * C + c0);
    const uint4 ud = *reinterpret_cast<const uint4*>(dy + (size_t)p * C + c0);
    const __half2* hx = reinterpret_cast<const __half2*>(&ux);
    const __half2* hd = reinterpret_cast<const __half2*>(&ud);
    float t8[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 tx = __half22float2(hx[i]), td = __half22float2(hd[i]);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = 2 * i + k;
        const float xh = ((k ? tx.y : tx.x) - mean2[e >> 2]) * rstd2[e >> 2];
        float d = k ? td.y : td.x;
        if (swish == 1) {
          const float a = g8[e] * xh + b8[e];
          const float sg = 1.f / (1.f + __expf(-a));
          d *= sg * (1.f + a * (1.f - sg));
        } else if (swish == 2) {
          d = (g8[e] * xh + b8[e]) > 0.f ? d : 0.f;
        }
        t8[e] = d * g8[e];
      }
    }
    // the sums see the fp16-rounded dxh: phase 2 subtracts the means from exactly these values
    uint4 ut;
    __half2* ht = reinterpret_cast<__half2*>(&ut);
#pragma unroll
    for (int i = 0; i < 4; ++i) ht[i] = __floats2half2_rn(t8[2 * i], t8[2 * i + 1]);
    *reinterpret_cast<uint4*>(cg + (size_t)(p - p_begin) * C + c0) = ut;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 tx = __half22float2(hx[i]), tt = __half22float2(ht[i]);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int e = 2 * i + k;
        const float xh = ((k ? tx.y : tx.x) - mean2[e >> 2]) * rstd2[e >> 2];
        const float dxh = k ? tt.y : tt.x;
        s[e >> 2][0] += dxh;
        s[e >> 2][1] += dxh * xh;
      }
    }
  }
  __shared__ float cpart[GN_G * 2];
  if (CLUSTER) {
    gnc_block_partials(s, red, vecs, cpg, cpart);
    gnc_cluster_fold(cpart, gridDim.x, (double)pixels * cpg, acc4, sh);
  } else {
    gnc_block_partials(s, red, vecs, cpg, part + (size_t)blockIdx.x * GN_G * 2);
    gnc_grid_barrier(bar, bar_target);
    gnc_fold(part, gridDim.x, (double)pixels * cpg, acc4, sh);
  }
  if (o.one_group) gnc_merge_groups(sh);
  float gs0[2], gs1[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int g = (c0 + 4 * i) / cpg;
    gs0[i] = (float)sh[2 * g];
    gs1[i] = (float)sh[2 * g + 1];
  }
#pragma unroll 2
  for (int p = p_begin + pl; p < p_end; p += plane) {
    float xv[8], tv[8], rv[8];
    load8(x + (size_t)p * C + c0, xv);
    load8(cg + (size_t)(p - p_begin) * C + c0, tv);
    if (dres) load8(dres + (size_t)p * C + c0, rv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xh = (xv[i] - mean2[i >> 2]) * rstd2[i >> 2];
      const float r = rstd2[i >> 2] * (tv[i] - gs0[i >> 2] - xh * gs1[i >> 2]);
      xv[i] = dres ? r + rv[i] : r;
    }
    store8(dx + (size_t)p * C + c0, xv);
  }
}

__global__ void __launch_bounds__(256) upsample2x_kernel(const act_t* __restrict__ x, int H, int W, int C, int ld_in,
                                                         act_t* __restrict__ y) {
  pdl_prologue();
  const int vecs = C / 8;
  const long long n = (long long)4 * H * W * vecs;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    int vc = (int)(v % vecs);
    long long p = v / vecs;
    int ox = (int)(p % (2 * W)), oy = (int)(p / (2 * W));
    const uint4* src = reinterpret_cast<const uint4*>(x + ((size_t)(oy >> 1) * W + (ox >> 1)) * ld_in) + vc;
    reinterpret_cast<uint4*>(y)[v] = *src;
  }
}

__global__ void __launch_bounds__(256) downsum2x_kernel(const act_t* __restrict__ gy, int H, int W, int C,
                                                        act_t* __restrict__ gx) {
  pdl_prologue();
  const int vecs = C / 8;
  const long long n = (long long)H * W * vecs;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    int vc = (int)(v % vecs);
    long long p = v / vecs;
    int ix = (int)(p % W), iy = (int)(p / W);
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        float t[8];
        load8(gy + ((size_t)(2 * iy + dy) * (2 * W) + 2 * ix + dx) * C + vc * 8, t);
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += t[i];
      }
    store8(gx + v * 8, s);
  }
}

__global__ void image_to_nhwc64_kernel(const float* __restrict__ img, int pixels, act_t* __restrict__ out) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // one 16-byte chunk (8 channels) per thread
  if (i >= pixels * 8) return;
  const int p = i >> 3, ch = i & 7;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (ch == 0) {
    v[0] = img[p];
    v[1] = img[(size_t)pixels + p];
    v[2] = img[(size_t)2 * pixels + p];
  }
  store8(out + (size_t)p * 64 + ch * 8, v);
}

__global__ void subsample_odd_kernel(const act_t* __restrict__ full, int H, int W, int C, act_t* __restrict__ y) {
  pdl_prologue();
  const int Ho = H / 2, Wo = W / 2, vecs = C / 8;
  const long long n = (long long)Ho * Wo * vecs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vecs);
    const long long px = i / vecs;
    const int ox = (int)(px % Wo), oy = (int)(px / Wo);
    const uint4 u = *reinterpret_cast<const uint4*>(full + ((size_t)(2 * oy + 1) * W + 2 * ox + 1) * C + v * 8);
    *reinterpret_cast<uint4*>(y + (size_t)px * C + v * 8) = u;
  }
}

__global__ void gather_codes_kernel(const float* __restrict__ cb, const int* __restrict__ idx, int C, int hw,
                                    float* __restrict__ z) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over [C, hw]
  if (i >= C * hw) return;
  const int k = i / hw, p = i % hw;
  z[i] = cb[(size_t)idx[p] * C + k];
}

__global__ void image_finish_kernel(const float* __restrict__ conv_out, int ld, int pixels, float* __restrict__ pre,
                                    float* __restrict__ img, int shift) {
  pdl_prologue();
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pixels) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = conv_out[(size_t)p * ld + c];
    const float v = shift ? (x + 1.f) / 2.f : x;  // decode(z_q).add(1).div(2), vqgan.py:195
    pre[(size_t)c * pixels + p] = v;
    img[(size_t)c * pixels + p] = fminf(fmaxf(v, 0.f), 1.f);
  }
}

__global__ void image_finish_bwd_kernel(const float* __restrict__ g_img, const float* __restrict__ pre, int pixels,
                                        int ld, act_t* __restrict__ g_out, int shift) {
  pdl_prologue();
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pixels) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float g = g_img[(size_t)c * pixels + p];
    float v = pre[(size_t)c * pixels + p];
    float cl = fminf(fmaxf(v, 0.f), 1.f);
    float keep = (g * (v - cl) >= 0.f) ? 1.f : 0.f;  // vqgan.py:79
    g_out[(size_t)p * ld + c] = __float2half_rn((shift ? 0.5f * g : g) * keep);
  }
}

__global__ void pixel_synth_kernel(const float* __restrict__ z, int rows, int cols, int H, int W,
                                   float* __restrict__ pre, float* __restrict__ img) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H * W) return;
  int x = i % W, y = (i / W) % H, c = i / (W * H);
  // F.interpolate(mode="nearest"): src = floor(dst * in / out)  (fast_pixeldrawer.py:90)
  int sy = min((int)floorf(y * ((float)rows / H)), rows - 1);
  int sx = min((int)floorf(x * ((float)cols / W)), cols - 1);
  float v = z[((size_t)c * rows + sy) * cols + sx];
  pre[i] = v;
  img[i] = fminf(fmaxf(v, 0.f), 1.f);
}

__global__ void pixel_synth_bwd_kernel(const float* __restrict__ g_img, const float* __restrict__ pre, int rows,
                                       int cols, int H, int W, float inv_scale, float* __restrict__ z_grad) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // over [3, rows, cols]
  if (i >= 3 * rows * cols) return;
  int sx = i % cols, sy = (i / cols) % rows, c = i / (cols * rows);
  // all output pixels whose nearest source is (sy, sx)
  float s = 0.f;
  int y0 = (int)ceilf(sy * ((float)H / rows)) - 1, y1 = (int)ceilf((sy + 1) * ((float)H / rows)) + 1;
  int x0 = (int)ceilf(sx * ((float)W / cols)) - 1, x1 = (int)ceilf((sx + 1) * ((float)W / cols)) + 1;
  for (int y = max(0, y0); y < min(H, y1); ++y) {
    if (min((int)floorf(y * ((float)rows / H)), rows - 1) != sy) continue;
    for (int x = max(0, x0); x < min(W, x1); ++x) {
      if (min((int)floorf(x * ((float)cols / W)), cols - 1) != sx) continue;
      size_t o = ((size_t)c * H + y) * W + x;
      float g = g_img[o], v = pre[o];
      float cl = fminf(fmaxf(v, 0.f), 1.f);
      if (g * (v - cl) >= 0.f) s += g;
    }
  }
  z_grad[i] = s * inv_scale;
}

inline int grid_for(long long n, int block, int cap = 148 * 16) {
  long long g = (n + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

void vq_nearest(const float* z, const float* cbT, const float* c2, const float* cb, int C, int hw, int n_e,
                float* part_d, int* part_i, int* idx, act_t* zq, cudaStream_t st) {
  const int n_chunks = (n_e + VQ_CODES - 1) / VQ_CODES;
  dim3 grid(n_chunks, (hw + VQ_POS - 1) / VQ_POS);
  launch_pdl(vq_partial_kernel, dim3(grid), dim3(256), C * VQ_POS * sizeof(float), st, z, cbT, c2, C, hw, n_e, n_chunks, part_d, part_i);
  launch_pdl(vq_final_kernel, dim3(hw), dim3(128), 0, st, part_d, part_i, n_chunks, cb, C, idx, zq);
}

void vq_backward(const act_t* dzq, float inv_scale, int C, int hw, float* z_grad, cudaStream_t st) {
  launch_pdl(vq_backward_kernel, dim3((C * hw + 255) / 256), dim3(256), 0, st, dzq, inv_scale, C, hw, z_grad);
}

int gn_num_partials(int pixels, int C) {
  const int rpb = gn_rows_per_block(pixels);
  return (pixels + rpb - 1) / rpb;
}

void gn_stats(const act_t* x, int pixels, int C, float eps, float* part, float* stats, cudaStream_t st, GnOpts o) {
  const int nblk = gn_num_partials(pixels, C);
  launch_pdl(gn_partial_kernel<0>, dim3(nblk), dim3(256), 0, st, x, nullptr, nullptr, nullptr, nullptr, pixels, C, 0, part,
             0.f, o.one_group);
  launch_pdl(gn_final_kernel<0>, dim3(1), dim3(256), 0, st, part, nblk, (double)pixels * (C / GN_G), eps, x, C, stats,
             o.one_group);
}

void gn_apply(const act_t* x, const float* stats, const float* gamma, const float* beta, int pixels, int C, int swish,
              act_t* y, cudaStream_t st, GnOpts o) {
  const long long nvec = (long long)pixels * C / 8;
  launch_pdl(gn_apply_kernel, dim3(grid_for(nvec, 256)), dim3(256), 0, st, x, stats, gamma, beta, nvec, C, swish, y,
             o.gamma_add, o.res);
}

void gn_backward(const act_t* dy, const act_t* x, const float* stats, const float* gamma, const float* beta,
                 int pixels, int C, int swish, const act_t* dres, float* part, float* gstats, act_t* dx,
                 cudaStream_t st, GnOpts o) {
  const int nblk = gn_num_partials(pixels, C);
  launch_pdl(gn_partial_kernel<1>, dim3(nblk), dim3(256), 0, st, x, dy, stats, gamma, beta, pixels, C, swish, part,
             o.gamma_add, o.one_group);
  launch_pdl(gn_final_kernel<1>, dim3(1), dim3(256), 0, st, part, nblk, (double)pixels * (C / GN_G), 0.f,
             (const act_t*)nullptr, C, gstats, o.one_group);
  const long long nvec = (long long)pixels * C / 8;
  launch_pdl(gn_bwd_apply_kernel, dim3(grid_for(nvec, 256)), dim3(256), 0, st, dy, x, stats, gstats, gamma, beta, nvec, C, swish, dres,
                                                           dx, o.gamma_add);
}

namespace {
constexpr int GNC_SMEM_MAX = 216 * 1024;
int gnc_rows_per_block(int pixels, int num_sms) {
  int r = (pixels + num_sms - 1) / num_sms;
  return r < 16 ? 16 : r;
}
bool g_gn_cluster = false;  // PXR_GN_CLUSTER=1 enables the cluster variant (measured 1 % slower than the grid barrier at config 2)
void gnc_init() {
  static bool done = false;
  if (done) return;
  cudaFuncSetAttribute(gn_coop_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GNC_SMEM_MAX);
  cudaFuncSetAttribute(gn_coop_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GNC_SMEM_MAX);
  cudaFuncSetAttribute(gn_coop_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GNC_SMEM_MAX);
  cudaFuncSetAttribute(gn_coop_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GNC_SMEM_MAX);
  cudaFuncSetAttribute(gn_coop_fwd_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  cudaFuncSetAttribute(gn_coop_bwd_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (const char* e = getenv("PXR_GN_CLUSTER")) g_gn_cluster = atoi(e) != 0;
  done = true;
}
// one cluster of 8 or 16 blocks when the tensor is small enough for their shared memory (slabs bytes: fwd 1x, bwd 2x)
int gnc_cluster_blocks(int pixels, int C, int slabs) {
  if (!g_gn_cluster) return 0;
  for (int nb : {8, 16}) {
    const int rpb = (pixels + nb - 1) / nb;
    if (4 * GNC_THREADS * 4 + (size_t)slabs * rpb * C * 2 <= (size_t)GNC_SMEM_MAX && rpb * nb >= pixels) return nb;
  }
  return 0;
}
template <class K, class... Args>
void gnc_launch_cluster(K kernel, int nb, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nb);
  cfg.blockDim = dim3(GNC_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = nb;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, args...);
}
}  // namespace

bool gn_coop_supported(int pixels, int C, int num_sms) {
  if (C % 8 || (C / 8) > GNC_THREADS || GNC_THREADS % (C / 8) || (C % GN_G) || (C / GN_G != 4 && (C / GN_G) % 8)) return false;
  if (num_sms > GNC_FOLD_MAX) return false;  // gnc_fold's register array covers grids of <= GNC_FOLD_MAX blocks
  const int rpb = gnc_rows_per_block(pixels, num_sms);
  return 4 * GNC_THREADS * 4 + (size_t)rpb * C * 2 <= (size_t)GNC_SMEM_MAX;
}

void gn_forward_coop(const act_t* x, const float* gamma, const float* beta, int pixels, int C, int swish, float eps,
                     float* part, float* stats, act_t* y, int num_sms, GridBarrier* gb, cudaStream_t st, GnOpts o) {
  gnc_init();
  if (const int nb = gnc_cluster_blocks(pixels, C, 1)) {
    const int rpb = (pixels + nb - 1) / nb;
    gnc_launch_cluster(gn_coop_fwd_kernel<true>, nb, 4 * GNC_THREADS * 4 + (size_t)rpb * C * 2, st, x, gamma, beta, pixels,
                       C, swish, eps, rpb, part, stats, y, (unsigned long long*)nullptr, 0ULL, o);
    return;
  }
  int rpb = gnc_rows_per_block(pixels, num_sms);
  const int grid = (pixels + rpb - 1) / rpb;
  const size_t smem = 4 * GNC_THREADS * 4 + (size_t)rpb * C * 2;
  launch_pdl(gn_coop_fwd_kernel<false>, dim3(grid), dim3(GNC_THREADS), smem, st, x, gamma, beta, pixels, C, swish, eps, rpb, part, stats, y,
                                                             gb->counter, gb->issued + grid, o);
  // three barriers' worth of arrivals per block (the second pass's two are added at once when it is not needed)
  if (cudaPeekAtLastError() == cudaSuccess) gb->issued += 3 * grid;  // a rejected launch must not move the target
}

void gn_backward_coop(const act_t* dy, const act_t* x, const float* stats, const float* gamma, const float* beta,
                      int pixels, int C, int swish, const act_t* dres, float* part, act_t* dx, int num_sms,
                      GridBarrier* gb, cudaStream_t st, GnOpts o) {
  gnc_init();
  if (const int nb = gnc_cluster_blocks(pixels, C, 2)) {
    const int rpb = (pixels + nb - 1) / nb;
    gnc_launch_cluster(gn_coop_bwd_kernel<true>, nb, 4 * GNC_THREADS * 4 + (size_t)2 * rpb * C * 2, st, dy, x, stats, gamma,
                       beta, pixels, C, swish, dres, rpb, 1, part, dx, (unsigned long long*)nullptr, 0ULL, o);
    return;
  }
  int rpb = gnc_rows_per_block(pixels, num_sms);
  const int grid = (pixels + rpb - 1) / rpb;
  const size_t slab = (size_t)rpb * C * 2;
  const int cache_dy = 0;  // the kernel keeps ONE slab (dxh) since round 2
  const size_t smem = 4 * GNC_THREADS * 4 + slab;
  launch_pdl(gn_coop_bwd_kernel<false>, dim3(grid), dim3(GNC_THREADS), smem, st, dy, x, stats, gamma, beta, pixels, C, swish, dres, rpb,
                                                             cache_dy, part, dx, gb->counter, gb->issued + grid, o);
  if (cudaPeekAtLastError() == cudaSuccess) gb->issued += grid;
}

void upsample2x(const act_t* x, int H, int W, int C, act_t* y, cudaStream_t st, int ld_in) {
  launch_pdl(upsample2x_kernel, dim3(grid_for((long long)4 * H * W * C / 8, 256)), dim3(256), 0, st, x, H, W, C,
             ld_in > 0 ? ld_in : C, y);
}
void downsum2x(const act_t* gy, int H, int W, int C, act_t* gx, cudaStream_t st) {
  launch_pdl(downsum2x_kernel, dim3(grid_for((long long)H * W * C / 8, 256)), dim3(256), 0, st, gy, H, W, C, gx);
}

void image_to_nhwc64(const float* img, int pixels, act_t* out, cudaStream_t st) {
  launch_pdl(image_to_nhwc64_kernel, dim3((pixels * 8 + 255) / 256), dim3(256), 0, st, img, pixels, out);
}
void subsample_odd(const act_t* full, int H, int W, int C, act_t* y, cudaStream_t st) {
  launch_pdl(subsample_odd_kernel, dim3(grid_for((long long)(H / 2) * (W / 2) * C / 8, 256)), dim3(256), 0, st, full, H, W, C, y);
}
void gather_codes(const float* cb, const int* idx, int C, int hw, float* z, cudaStream_t st) {
  launch_pdl(gather_codes_kernel, dim3((C * hw + 255) / 256), dim3(256), 0, st, cb, idx, C, hw, z);
}

void image_finish(const float* conv_out, int ld, int pixels, float* pre, float* img, cudaStream_t st, int shift) {
  launch_pdl(image_finish_kernel, dim3((pixels + 255) / 256), dim3(256), 0, st, conv_out, ld, pixels, pre, img, shift);
}
void image_finish_backward(const float* g_img, const float* pre, int pixels, int ld, act_t* g_out, cudaStream_t st,
                           int shift) {
  launch_pdl(image_finish_bwd_kernel, dim3((pixels + 255) / 256), dim3(256), 0, st, g_img, pre, pixels, ld, g_out, shift);
}

void pixel_synth(const float* z, int rows, int cols, int H, int W, float* pre, float* img, cudaStream_t st) {
  launch_pdl(pixel_synth_kernel, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, z, rows, cols, H, W, pre, img);
}
void pixel_synth_backward(const float* g_img, const float* pre, int rows, int cols, int H, int W, float inv_scale,
                          float* z_grad, cudaStream_t st) {
  launch_pdl(pixel_synth_bwd_kernel, dim3((3 * rows * cols + 255) / 256), dim3(256), 0, st, g_img, pre, rows, cols, H, W, inv_scale,
                                                                        z_grad);
}

}  // namespace pxr
