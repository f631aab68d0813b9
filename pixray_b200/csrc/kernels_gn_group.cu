// GroupNorm(32, C) for the small-spatial decoder levels, one thread-block CLUSTER per group (no grid-wide barrier).
//
// The single-kernel GroupNorm of kernels_decoder.cu splits the PIXELS over the grid, so every block owns a piece of every
// group and the statistics need a grid-wide barrier (launch + barrier latency on every call; 52 such calls per config-2
// iteration on tensors of 256 KB ... 2 MB).  Here the split is by GROUP: the cluster (1 ... 8 CTAs) of group g reads only
// that group's channels, reduces (sum, sum of squares) over its own CTAs through distributed shared memory and applies --
// nothing crosses clusters, so there is no global synchronisation at all.
//
// The same kernels also absorb the epilogue of a split-K convolution (gemm_tc.cu: fp32 partial sums [splits][px][ld]):
//   forward : x = fp16(sum_s ws[s] + bias + res) is written (the residual stream / the saved GN input) AND normalised
//             in the same pass -- replaces splitk_reduce + gn_forward (2 launches, 1 barrier, 1 re-read of x);
//   backward: dy = fp16(sum_s ws[s]) never reaches memory -- replaces splitk_reduce + gn_backward.
// Arithmetic order matches the unfused kernels (partials summed in split order after the bias, then the residual, one
// rounding to fp16 before the statistics), reductions are fixed-order (warp tree -> warps -> cluster ranks): bit-identical
// on every run and on every rank of the cutout-sharded mode.
//
// Work unit: (pixel, 8-channel vector) = 16 B of fp16 / 32 B of fp32.  A group has px * (cpg / 8) units; CTA r of the
// cluster owns a contiguous range of them and each thread keeps its <= UPT units in registers between the two phases.
#include <cooperative_groups.h>

#include "kernels.cuh"
#include "launch.cuh"

namespace cg = cooperative_groups;

namespace pxr {
namespace {

constexpr int GG_MAX_THREADS = 512;
constexpr int GG_G = 32;

__device__ __forceinline__ void gg_unpack8(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 gg_pack8(const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// sum over the split-K partials of one unit, in split order, starting from the bias (the order of splitk_reduce_kernel)
__device__ __forceinline__ void gg_sum_splits(const float* __restrict__ src, int splits, size_t slab, float (&acc)[8]) {
  int s0 = 0;
  for (; s0 + 4 <= splits; s0 += 4) {
    float4 a[4], b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      a[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * slab));
      b[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * slab + 4));
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      acc[0] += a[u].x;
      acc[1] += a[u].y;
      acc[2] += a[u].z;
      acc[3] += a[u].w;
      acc[4] += b[u].x;
      acc[5] += b[u].y;
      acc[6] += b[u].z;
      acc[7] += b[u].w;
    }
  }
  for (; s0 < splits; ++s0) {
    const float4 a = __ldcg(reinterpret_cast<const float4*>(src + s0 * slab));
    const float4 b = __ldcg(reinterpret_cast<const float4*>(src + s0 * slab + 4));
    acc[0] += a.x;
    acc[1] += a.y;
    acc[2] += a.z;
    acc[3] += a.w;
    acc[4] += b.x;
    acc[5] += b.y;
    acc[6] += b.z;
    acc[7] += b.w;
  }
}

// (a, b) summed over the whole cluster in a fixed order; every thread of every CTA returns the same two doubles.
// red: [2][16] doubles of shared memory, cpart: [2] doubles (read by the cluster peers through DSMEM).
__device__ __forceinline__ void gg_cluster_sum(double a, double b, double* red, double* cpart, double& ta, double& tb) {
  cg::cluster_group cluster = cg::this_cluster();
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[warp] = a;
    red[16 + warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb = 0.0;
    for (int w = 0; w < nwarp; ++w) {
      sa += red[w];
      sb += red[16 + w];
    }
    cpart[0] = sa;
    cpart[1] = sb;
  }
  cluster.sync();  // every CTA's cpart is written (and visible cluster-wide)
  ta = 0.0;
  tb = 0.0;
  const unsigned nb = cluster.num_blocks();
  for (unsigned r = 0; r < nb; ++r) {
    const double* p = cluster.map_shared_rank(cpart, r);
    ta += p[0];
    tb += p[1];
  }
}

struct GgGeom {
  int g, c0, vpg, u_begin, u_end;
};
__device__ __forceinline__ GgGeom gg_geometry(int px, int C) {
  cg::cluster_group cluster = cg::this_cluster();
  const int cs = (int)cluster.num_blocks(), r = (int)cluster.block_rank();
  GgGeom q;
  q.g = blockIdx.x / cs;
  const int cpg = C / GG_G;
  q.vpg = cpg / 8;
  const int upg = px * q.vpg, upc = upg / cs;  // the launcher guarantees px % cs == 0
  q.u_begin = r * upc;
  q.u_end = q.u_begin + upc;
  q.c0 = q.g * cpg + ((q.u_begin + threadIdx.x) % q.vpg) * 8;  // blockDim.x % vpg == 0: the same vector for all units
  return q;
}

template <int UPT>
__global__ void __launch_bounds__(GG_MAX_THREADS)
    gn_group_fwd_kernel(const act_t* __restrict__ x, const float* __restrict__ ws, int splits, int ld_ws,
                        const float* __restrict__ bias, const act_t* res, act_t* x_out,  // res may alias x_out
                       
                        const float* __restrict__ gamma, const float* __restrict__ beta, int px, int C, int swish,
                        float eps, float* __restrict__ stats_out, act_t* __restrict__ y) {
  pdl_launch_dependents();
  __shared__ double red[32];
  __shared__ double cpart[2], cpart2[2];
  const GgGeom q = gg_geometry(px, C);
  float ga[8], be[8], bi[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {  // constant weights: may be read ahead of the dependency wait
    ga[i] = gamma[q.c0 + i];
    be[i] = beta[q.c0 + i];
    bi[i] = (ws && bias) ? bias[q.c0 + i] : 0.f;
  }
  pdl_wait();
  const size_t slab = (size_t)px * ld_ws;
  float xv[UPT][8];
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int k = 0; k < UPT; ++k) {
    const int u = q.u_begin + threadIdx.x + k * blockDim.x;
    if (u < q.u_end) {
      const int p = u / q.vpg;
      if (ws) {
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = bi[i];
        uint4 r16 = make_uint4(0, 0, 0, 0);
        if (res) r16 = *reinterpret_cast<const uint4*>(res + (size_t)p * C + q.c0);
        gg_sum_splits(ws + (size_t)p * ld_ws + q.c0, splits, slab, acc);
        if (res) {
          float rv[8];
          gg_unpack8(r16, rv);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[i] += rv[i];
        }
        const uint4 o = gg_pack8(acc);  // the statistics see the fp16-rounded tensor, like the unfused path
        *reinterpret_cast<uint4*>(x_out + (size_t)p * C + q.c0) = o;
        gg_unpack8(o, xv[k]);
      } else {
        gg_unpack8(*reinterpret_cast<const uint4*>(x + (size_t)p * C + q.c0), xv[k]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s0 += xv[k][i];
        s1 += xv[k][i] * xv[k][i];
      }
    }
  }
  double ta, tb;
  gg_cluster_sum((double)s0, (double)s1, red, cpart, ta, tb);
  const double n = (double)px * (C / GG_G);
  double mean = ta / n;
  double var = tb / n - mean * mean;
  if (var < 0) var = 0;
  if (gn_refine_variance(mean, var)) {  // every CTA of the cluster holds the same sums: a cluster-uniform branch
    const float m0 = (float)mean;
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int k = 0; k < UPT; ++k) {
      if (q.u_begin + threadIdx.x + k * blockDim.x < q.u_end) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = xv[k][i] - m0;
          d0 += d;
          d1 += d * d;
        }
      }
    }
    double ua, ub;
    gg_cluster_sum((double)d0, (double)d1, red, cpart2, ua, ub);
    const double md = ua / n;
    mean = (double)m0 + md;
    var = ub / n - md * md;
    if (var < 0) var = 0;
  }
  const float m = (float)mean, rs = (float)(1.0 / sqrt(var + (double)eps));
  if (cg::this_cluster().block_rank() == 0 && threadIdx.x == 0) {
    stats_out[2 * q.g] = m;
    stats_out[2 * q.g + 1] = rs;
  }
#pragma unroll
  for (int k = 0; k < UPT; ++k) {
    const int u = q.u_begin + threadIdx.x + k * blockDim.x;
    if (u < q.u_end) {
      const int p = u / q.vpg;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float sc = rs * ga[i];
        const float a = xv[k][i] * sc + (be[i] - m * sc);
        o[i] = swish ? a / (1.f + __expf(-a)) : a;
      }
      *reinterpret_cast<uint4*>(y + (size_t)p * C + q.c0) = gg_pack8(o);
    }
  }
  cg::this_cluster().sync();  // no CTA may exit (and release its shared memory) while a peer still reads its partials
}

template <int UPT>
__global__ void __launch_bounds__(GG_MAX_THREADS)
    gn_group_bwd_kernel(const act_t* __restrict__ dy, const float* __restrict__ ws, int splits, int ld_ws,
                        const act_t* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                        const float* __restrict__ beta, int px, int C, int swish, const act_t* dres,
                        act_t* dx) {  // dres may alias dx
  pdl_launch_dependents();
  __shared__ double red[32];
  __shared__ double cpart[2];
  const GgGeom q = gg_geometry(px, C);
  float ga[8], be[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ga[i] = gamma[q.c0 + i];
    be[i] = beta[q.c0 + i];
  }
  pdl_wait();
  const float mean = stats[2 * q.g], rstd = stats[2 * q.g + 1];
  const size_t slab = (size_t)px * ld_ws;
  float xh[UPT][8], dxh[UPT][8];
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int k = 0; k < UPT; ++k) {
    const int u = q.u_begin + threadIdx.x + k * blockDim.x;
    if (u < q.u_end) {
      const int p = u / q.vpg;
      float xv[8], dv[8];
      gg_unpack8(*reinterpret_cast<const uint4*>(x + (size_t)p * C + q.c0), xv);
      if (ws) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        gg_sum_splits(ws + (size_t)p * ld_ws + q.c0, splits, slab, acc);
        gg_unpack8(gg_pack8(acc), dv);  // the unfused path stores dy as fp16 between the two kernels
      } else {
        gg_unpack8(*reinterpret_cast<const uint4*>(dy + (size_t)p * C + q.c0), dv);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float h = (xv[i] - mean) * rstd;
        float d = dv[i];
        if (swish) {
          const float a = ga[i] * h + be[i];
          const float sg = 1.f / (1.f + __expf(-a));
          d *= sg * (1.f + a * (1.f - sg));
        }
        const float t = d * ga[i];
        xh[k][i] = h;
        dxh[k][i] = t;
        s0 += t;
        s1 += t * h;
      }
    }
  }
  double ta, tb;
  gg_cluster_sum((double)s0, (double)s1, red, cpart, ta, tb);
  const double n = (double)px * (C / GG_G);
  const float m0 = (float)(ta / n), m1 = (float)(tb / n);
#pragma unroll
  for (int k = 0; k < UPT; ++k) {
    const int u = q.u_begin + threadIdx.x + k * blockDim.x;
    if (u < q.u_end) {
      const int p = u / q.vpg;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = rstd * (dxh[k][i] - m0 - xh[k][i] * m1);
      if (dres) {
        float rv[8];
        gg_unpack8(*reinterpret_cast<const uint4*>(dres + (size_t)p * C + q.c0), rv);
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] += rv[i];
      }
      *reinterpret_cast<uint4*>(dx + (size_t)p * C + q.c0) = gg_pack8(o);
    }
  }
  cg::this_cluster().sync();
}

struct GgLaunch {
  int cs = 0, threads = 0, upt = 0;
};
int gg_target_units() {
  static const int t = [] {
    const char* e = getenv("PXR_GN_GROUP_UNITS");
    const int v = e ? atoi(e) : 0;
    return v > 0 ? v : 128;
  }();
  return t;
}
// cluster size / block size / units per thread for a tensor, or cs == 0 when the shape is not covered
GgLaunch gg_plan(int px, int C, bool any_size) {
  GgLaunch l;
  if (C % GG_G || (C / GG_G) % 8) return l;
  const int vpg = C / GG_G / 8;
  if (vpg != 1 && vpg != 2 && vpg != 4) return l;
  const long long upg = (long long)px * vpg;
  // The group split is used while a group is <= 2048 units (16^2 / 32^2 latents); beyond that the 16-byte reads at a
  // pixel stride of C and the scheduling of 8-CTA clusters of 512 threads cost more than the grid barrier saves
  // (tests/test_groupnorm_gpu.py::test_groupnorm_timing_report times both).
  static const long long max_units = [] {
    const char* e = getenv("PXR_GN_GROUP_MAX_UNITS");
    const long long v = e ? atoll(e) : 0;
    return v > 0 ? v : 2048LL;
  }();
  if (!any_size && upg > max_units) return l;
  int cs = 1;
  while (cs < 8 && upg / cs > gg_target_units() && px % (cs * 2) == 0) cs *= 2;
  if (px % cs) return l;
  const long long upc = upg / cs;
  if (upc > (long long)GG_MAX_THREADS * 4) return l;
  l.threads = (int)std::min<long long>(GG_MAX_THREADS, (upc + 31) / 32 * 32);
  const int upt = (int)((upc + l.threads - 1) / l.threads);
  l.upt = upt <= 1 ? 1 : (upt <= 2 ? 2 : 4);
  l.cs = cs;
  return l;
}

template <class K, class... Args>
cudaError_t gg_launch(K kernel, const GgLaunch& l, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(GG_G * l.cs);
  cfg.blockDim = dim3(l.threads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = l.cs;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[1].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = at;
  cfg.numAttrs = 2;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

}  // namespace

bool gn_group_supported(int pixels, int C) { return gg_plan(pixels, C, false).cs > 0; }
bool gn_group_possible(int pixels, int C) { return gg_plan(pixels, C, true).cs > 0; }

void gn_forward_group(const act_t* x, const GnSplitK* sk, const float* gamma, const float* beta, int pixels, int C,
                      int swish, float eps, float* stats, act_t* y, cudaStream_t st) {
  const GgLaunch l = gg_plan(pixels, C, true);
  const float* ws = sk ? sk->ws : nullptr;
  const int splits = sk ? sk->splits : 0, ld_ws = sk ? sk->ld_ws : 0;
  const float* bias = sk ? sk->bias : nullptr;
  const act_t* res = sk ? sk->res : nullptr;
  act_t* x_out = sk ? sk->out : nullptr;
  switch (l.upt) {
    case 1: gg_launch(gn_group_fwd_kernel<1>, l, st, x, ws, splits, ld_ws, bias, res, x_out, gamma, beta, pixels, C, swish, eps, stats, y); break;
    case 2: gg_launch(gn_group_fwd_kernel<2>, l, st, x, ws, splits, ld_ws, bias, res, x_out, gamma, beta, pixels, C, swish, eps, stats, y); break;
    default: gg_launch(gn_group_fwd_kernel<4>, l, st, x, ws, splits, ld_ws, bias, res, x_out, gamma, beta, pixels, C, swish, eps, stats, y); break;
  }
}

void gn_backward_group(const act_t* dy, const GnSplitK* sk, const act_t* x, const float* stats, const float* gamma,
                       const float* beta, int pixels, int C, int swish, const act_t* dres, act_t* dx, cudaStream_t st) {
  const GgLaunch l = gg_plan(pixels, C, true);
  const float* ws = sk ? sk->ws : nullptr;
  const int splits = sk ? sk->splits : 0, ld_ws = sk ? sk->ld_ws : 0;
  switch (l.upt) {
    case 1: gg_launch(gn_group_bwd_kernel<1>, l, st, dy, ws, splits, ld_ws, x, stats, gamma, beta, pixels, C, swish, dres, dx); break;
    case 2: gg_launch(gn_group_bwd_kernel<2>, l, st, dy, ws, splits, ld_ws, x, stats, gamma, beta, pixels, C, swish, dres, dx); break;
    default: gg_launch(gn_group_bwd_kernel<4>, l, st, dy, ws, splits, ld_ws, x, stats, gamma, beta, pixels, C, swish, dres, dx); break;
  }
}

}  // namespace pxr
