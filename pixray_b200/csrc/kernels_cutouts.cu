// MakeCutouts as fused gather kernels (pixray.py:445-511, cached-transform semantics 480-486):
//   pool_forward    : (AdaptiveAvgPool2d + AdaptiveMaxPool2d)/2 of the whole image, once instead of cutn times
//   cutout_forward  : per-cutout homography resample (reflection / border padding for the zoom group, constant grey
//                     fill for the wide group) + noise, emitting block partials of the global min / max
//   patchify_*      : CLIP_Base.preprocess (global range normalise + mean/std, slip.py:21-60) fused with the
//                     im2col of the ViT patch embedding, and its adjoint
//   cutout_backward : adjoint of the resample (scatter-add through the bilinear taps) incl. the d/dmin, d/dmax terms
#include "kernels.cuh"
#include "launch.cuh"
#include "color_jitter.cuh"
#include "philox.cuh"
#include "pool_bounds.cuh"
#include <cfloat>

namespace pxr {
namespace {


// ATen adaptive pooling window [floor(i*in/out), ceil((i+1)*in/out)): pool_start / pool_end of pool_bounds.cuh

__global__ void pool_fwd_kernel(const float* __restrict__ img, int H, int W, int cs, float* __restrict__ pooled,
                                int* __restrict__ argmax) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * cs * cs) return;
  int ox = i % cs, oy = (i / cs) % cs, c = i / (cs * cs);
  int y0 = pool_start(oy, H, cs), y1 = pool_end(oy, H, cs);
  int x0 = pool_start(ox, W, cs), x1 = pool_end(ox, W, cs);
  const float* p = img + (size_t)c * H * W;
  float s = 0.f, m = -FLT_MAX;
  int mi = y0 * W + x0;
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x) {
      float v = p[y * W + x];
      s += v;
      if (v > m) {  // first maximum wins, like ATen's adaptive_max_pool2d
        m = v;
        mi = y * W + x;
      }
    }
  float avg = s / (float)((y1 - y0) * (x1 - x0));
  pooled[i] = (avg + m) / 2.f;  // pixray.py:463
  argmax[i] = mi;
}

__global__ void spot_mask_kernel(const float* __restrict__ x, const unsigned char* __restrict__ mask, int zero_where_set,
                                 int n, float* __restrict__ y) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool set = mask[i] != 0;
  y[i] = (set != (zero_where_set != 0)) ? x[i] : 0.f;
}

__global__ void pool_bwd_kernel(const float* __restrict__ g_pooled, const int* __restrict__ argmax, int H, int W,
                                int cs, float* __restrict__ g_img, int accumulate) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H * W) return;
  int x = i % W, y = (i / W) % H, c = i / (W * H);
  // candidate output rows / cols whose window may contain (y, x)
  int oy_lo = max(0, (int)(((long long)y * cs) / H) - 2), oy_hi = min(cs - 1, (int)((((long long)(y + 1)) * cs) / H) + 2);
  int ox_lo = max(0, (int)(((long long)x * cs) / W) - 2), ox_hi = min(cs - 1, (int)((((long long)(x + 1)) * cs) / W) + 2);
  float s = 0.f;
  for (int oy = oy_lo; oy <= oy_hi; ++oy) {
    int y0 = pool_start(oy, H, cs), y1 = pool_end(oy, H, cs);
    if (y < y0 || y >= y1) continue;
    for (int ox = ox_lo; ox <= ox_hi; ++ox) {
      int x0 = pool_start(ox, W, cs), x1 = pool_end(ox, W, cs);
      if (x < x0 || x >= x1) continue;
      size_t o = ((size_t)c * cs + oy) * cs + ox;
      float g = g_pooled[o] * 0.5f;
      s += g / (float)((y1 - y0) * (x1 - x0));
      if (argmax[o] == y * W + x) s += g;
    }
  }
  g_img[i] = accumulate ? g_img[i] + s : s;
}

// ------------------------------------------------------------------ coordinate helpers (ATen grid_sampler semantics)
__device__ __forceinline__ float clip_coord(float x, int size) { return fminf((float)(size - 1), fmaxf(x, 0.f)); }
__device__ __forceinline__ float reflect_coord(float x, int twice_low, int twice_high) {
  if (twice_low == twice_high) return 0.f;
  float mn = (float)twice_low / 2.f;
  float span = (float)(twice_high - twice_low) / 2.f;
  x = fabsf(x - mn);
  float extra = fmodf(x, span);
  int flips = (int)floorf(x / span);
  return (flips % 2 == 0) ? extra + mn : span - extra + mn;
}
// padding: 0 reflection, 1 border, 2 zeros (align_corners=True: coordinates are already in pixels)
__device__ __forceinline__ float pad_coord(float x, int size, int padding) {
  if (padding == 1) return clip_coord(x, size);
  if (padding == 0) return clip_coord(reflect_coord(x, 0, 2 * (size - 1)), size);
  return x;
}

struct Taps {
  int x0, y0;     // north-west tap; the others are +1
  float w[4];     // nw, ne, sw, se
  bool in[4];
};
__device__ __forceinline__ Taps make_taps(float xs, float ys, int sw, int sh) {
  Taps t;
  float fx = floorf(xs), fy = floorf(ys);
  t.x0 = (int)fx;
  t.y0 = (int)fy;
  float ax = xs - fx, ay = ys - fy;
  t.w[0] = (1.f - ax) * (1.f - ay);
  t.w[1] = ax * (1.f - ay);
  t.w[2] = (1.f - ax) * ay;
  t.w[3] = ax * ay;
  bool xin0 = t.x0 >= 0 && t.x0 < sw, xin1 = t.x0 + 1 >= 0 && t.x0 + 1 < sw;
  bool yin0 = t.y0 >= 0 && t.y0 < sh, yin1 = t.y0 + 1 >= 0 && t.y0 + 1 < sh;
  t.in[0] = xin0 && yin0;
  t.in[1] = xin1 && yin0;
  t.in[2] = xin0 && yin1;
  t.in[3] = xin1 && yin1;
  return t;
}
__device__ __forceinline__ void src_coord(const float* m, int u, int v, float& xs, float& ys) {
  float X = m[0] * u + m[1] * v + m[2];
  float Y = m[3] * u + m[4] * v + m[5];
  float Z = m[6] * u + m[7] * v + m[8];
  float s = fabsf(Z) > 1e-8f ? 1.f / Z : 1.f;  // kornia transform_points
  xs = X * s;
  ys = Y * s;
}

// one warped pixel, all three channels: bilinear taps (+ the wide group's fill under the uncovered weight)
__device__ __forceinline__ void warp_sample(const float* __restrict__ pooled, const Taps& t, int sw, int sh, bool zoom,
                                            float fill, float rgb[3]) {
  float cover = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) cover += t.in[k] ? t.w[k] : 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* p = pooled + (size_t)c * sh * sw;
    float val = 0.f;
    if (t.in[0]) val += t.w[0] * p[t.y0 * sw + t.x0];
    if (t.in[1]) val += t.w[1] * p[t.y0 * sw + t.x0 + 1];
    if (t.in[2]) val += t.w[2] * p[(t.y0 + 1) * sw + t.x0];
    if (t.in[3]) val += t.w[3] * p[(t.y0 + 1) * sw + t.x0 + 1];
    if (!zoom) val += (1.f - cover) * fill;  // kornia _fill_and_warp
    rgb[c] = val;
  }
}

// F.interpolate(mode='bilinear', align_corners=False) source coordinate and taps along one axis (ATen
// area_pixel_compute_source_index: scale * (dst + 0.5) - 0.5, clamped at 0; the high tap clamps at in - 1)
__device__ __forceinline__ void lin_taps(int o, int in, int out, int& i0, int& i1, float& l1) {
  const float scale = (float)in / (float)out;
  float src = scale * ((float)o + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = (int)src;
  if (i0 > in - 1) i0 = in - 1;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = src - (float)i0;
}

__global__ void rescale_fwd_kernel(const float* __restrict__ x, int in_h, int in_w, int out_h, int out_w,
                                   float* __restrict__ y) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * out_h * out_w) return;
  const int ox = i % out_w, oy = (i / out_w) % out_h, c = i / (out_w * out_h);
  int x0, x1, y0, y1;
  float lx, ly;
  lin_taps(ox, in_w, out_w, x0, x1, lx);
  lin_taps(oy, in_h, out_h, y0, y1, ly);
  const float* p = x + (size_t)c * in_h * in_w;
  // ATen: h0lambda * (w0lambda * a + w1lambda * b) + h1lambda * (w0lambda * c + w1lambda * d)
  const float top = (1.f - lx) * p[y0 * in_w + x0] + lx * p[y0 * in_w + x1];
  const float bot = (1.f - lx) * p[y1 * in_w + x0] + lx * p[y1 * in_w + x1];
  y[i] = (1.f - ly) * top + ly * bot;
}

// ---------------------------------------------------------------------------------------------------------------
// Order-independent accumulation.  The scatter of the warp adjoint, the un-stretch adjoint and the two range sums add
// many contributions to one address from many blocks; float atomics would make the result depend on the arrival order (a
// last-bit difference that flips fp16 roundings further down the drawer backward: measured as a two-state jitter of 7e-4 of
// max|z.grad| between identical runs).  They accumulate in 64-bit FIXED POINT instead -- integer addition is associative,
// so the sum is the same bits on every run and on every rank -- and one small kernel converts to fp32 (and clears the
// accumulator for the next pass).  Scales: 2^36 for gradient images (range +-1.3e8, step 1.5e-11: finer than an fp32 add at
// the magnitudes that occur, grad_scale * dL ~ 1e-2 ... 1e2), 2^30 for the two range sums (range +-8.6e9).
constexpr float FX_GRAD = 68719476736.f;       // 2^36
constexpr float FX_GRAD_INV = 1.f / 68719476736.f;
constexpr float FX_GRAD_MAX = 67108864.f;      // 2^26: half the range; beyond it (or NaN / Inf) the pass is poisoned
constexpr float FX_SUM = 1073741824.f;         // 2^30
constexpr float FX_SUM_INV = 1.f / 1073741824.f;
constexpr float FX_SUM_MAX = 4294967296.f;     // 2^32
// A NaN / Inf / out-of-range contribution cannot be represented in the integer sum (and must not vanish into it: the
// reference's blow-ups surface as NaN gradients).  It marks the pass instead -- `poison` keeps the id of the last pass that
// saw one -- and the conversion kernel writes NaN for the whole tensor of such a pass.
__device__ __forceinline__ void fx_add(long long* p, float v, float scale, float vmax, unsigned int* poison, unsigned int pass) {
  if (fabsf(v) < vmax) atomicAdd(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(__float2ll_rn(v * scale)));
  else atomicMax(poison, pass);
}
__global__ void __launch_bounds__(256) fx_to_float_kernel(long long* __restrict__ acc, float* __restrict__ out, int n,
                                                          float inv_scale, const unsigned int* __restrict__ poison,
                                                          unsigned int pass) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = (*poison == pass) ? __int_as_float(0x7fc00000) : (float)acc[i] * inv_scale;
  acc[i] = 0;
}

__global__ void rescale_bwd_kernel(const float* __restrict__ gy, int in_h, int in_w, int out_h, int out_w,
                                   long long* __restrict__ gx, unsigned int* poison, unsigned int pass) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * out_h * out_w) return;
  const int ox = i % out_w, oy = (i / out_w) % out_h, c = i / (out_w * out_h);
  int x0, x1, y0, y1;
  float lx, ly;
  lin_taps(ox, in_w, out_w, x0, x1, lx);
  lin_taps(oy, in_h, out_h, y0, y1, ly);
  long long* p = gx + (size_t)c * in_h * in_w;
  const float g = gy[i];
  fx_add(p + y0 * in_w + x0, (1.f - ly) * (1.f - lx) * g, FX_GRAD, FX_GRAD_MAX, poison, pass);
  fx_add(p + y0 * in_w + x1, (1.f - ly) * lx * g, FX_GRAD, FX_GRAD_MAX, poison, pass);
  fx_add(p + y1 * in_w + x0, ly * (1.f - lx) * g, FX_GRAD, FX_GRAD_MAX, poison, pass);
  fx_add(p + y1 * in_w + x1, ly * lx * g, FX_GRAD, FX_GRAD_MAX, poison, pass);
}

constexpr int CUT_THREADS = 256;

// grid (ceil(cs*cs/4 / 256), n_local); each thread: 4 consecutive u of one row v, all 3 channels
__global__ void __launch_bounds__(CUT_THREADS) cutout_fwd_kernel(CutoutArgs a, float* __restrict__ batch,
                                                                 float* __restrict__ part_min,
                                                                 float* __restrict__ part_max,
                                                                 int* __restrict__ part_imin,
                                                                 int* __restrict__ part_imax) {
  pdl_prologue();
  const int n = blockIdx.y;
  const int n_global = a.first_global + n;
  const int cs = a.cs;
  const int grp = blockIdx.x * CUT_THREADS + threadIdx.x;
  const int groups = cs * cs / 4;
  float tmin = FLT_MAX, tmax = -FLT_MAX;
  int imin = 0x7fffffff, imax = 0x7fffffff;
  if (grp < groups) {
    const int v = (grp * 4) / cs, u0 = (grp * 4) % cs;
    const bool zoom = n_global < a.cutn_zoom;
    const int padding = zoom ? a.zoom_padding : 2;
    float m[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) m[i] = a.minv[n * 9 + i];
    float fac = 0.f;
    float nz[3][4];
    const bool have_noise = a.noise_mode != 0;
    if (a.noise_mode == 1) {  // explicit facs + noise tensor (parity tests replay the oracle's draws)
      fac = a.noise_facs[n];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float4 t = *reinterpret_cast<const float4*>(a.noise + (((size_t)n * 3 + c) * cs + v) * cs + u0);
        nz[c][0] = t.x;
        nz[c][1] = t.y;
        nz[c][2] = t.z;
        nz[c][3] = t.w;
      }
    } else if (a.noise_mode == 2) {
      // engine RNG: Philox keyed by (seed, iter), counted by the GLOBAL element index -> shard invariant.
      // facs ~ U(0, noise_fac) per cutout (pixray.py:509), noise ~ N(0,1) per element (pixray.py:510)
      fac = philox_uniform(a.seed, (uint32_t)a.iter, 1u + a.rng_stream, (uint64_t)n_global) * a.noise_fac;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        uint64_t e = (((uint64_t)n_global * 3 + c) * cs + v) * cs + u0;
        philox_normal4(a.seed, (uint32_t)a.iter, a.rng_stream, e >> 2, nz[c]);
      }
    }
    int cj_code = 0;
    float cj_sat = 1.f, cj_hue = 0.f;
    if (a.jitter) {  // K.ColorJitter, last stage of the stack (pixray.py:416, 436)
      cj_code = (int)a.jitter[n * 3];
      cj_sat = a.jitter[n * 3 + 1];
      cj_hue = a.jitter[n * 3 + 2];
    }
    float out[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float xs, ys;
      src_coord(m, u0 + j, v, xs, ys);
      xs = pad_coord(xs, a.src_w, padding);
      ys = pad_coord(ys, a.src_h, padding);
      Taps t = make_taps(xs, ys, a.src_w, a.src_h);
      float rgb[3];
      warp_sample(a.pooled, t, a.src_w, a.src_h, zoom, a.fill, rgb);
      cj_apply(rgb, cj_code, cj_sat, cj_hue);
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c][j] = have_noise ? rgb[c] + fac * nz[c][j] : rgb[c];  // pixray.py:508-510
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      size_t o = (((size_t)n * 3 + c) * cs + v) * cs + u0;
      *reinterpret_cast<float4*>(batch + o) = make_float4(out[c][0], out[c][1], out[c][2], out[c][3]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float val = out[c][j];
        int e = (int)(o + j);
        if (val < tmin || (val == tmin && e < imin)) {
          tmin = val;
          imin = e;
        }
        if (val > tmax || (val == tmax && e < imax)) {
          tmax = val;
          imax = e;
        }
      }
    }
  }
  // block reduce
  __shared__ float smin[CUT_THREADS / 32], smax[CUT_THREADS / 32];
  __shared__ int simin[CUT_THREADS / 32], simax[CUT_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float om = __shfl_xor_sync(0xffffffffu, tmin, o);
    int oi = __shfl_xor_sync(0xffffffffu, imin, o);
    if (om < tmin || (om == tmin && oi < imin)) {
      tmin = om;
      imin = oi;
    }
    float oM = __shfl_xor_sync(0xffffffffu, tmax, o);
    int oI = __shfl_xor_sync(0xffffffffu, imax, o);
    if (oM > tmax || (oM == tmax && oI < imax)) {
      tmax = oM;
      imax = oI;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    smin[threadIdx.x >> 5] = tmin;
    simin[threadIdx.x >> 5] = imin;
    smax[threadIdx.x >> 5] = tmax;
    simax[threadIdx.x >> 5] = imax;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < CUT_THREADS / 32; ++w) {
      if (smin[w] < tmin || (smin[w] == tmin && simin[w] < imin)) {
        tmin = smin[w];
        imin = simin[w];
      }
      if (smax[w] > tmax || (smax[w] == tmax && simax[w] < imax)) {
        tmax = smax[w];
        imax = simax[w];
      }
    }
    int b = blockIdx.y * gridDim.x + blockIdx.x;
    part_min[b] = tmin;
    part_max[b] = tmax;
    part_imin[b] = imin;
    part_imax[b] = imax;
  }
}

// block partial min / max (+ first element index) of an arbitrary fp32 buffer -- used when a caller hands
// pxr_encode_image its own batch (CLIP_Base.preprocess recomputes the global range, slip.py:21-36)
__global__ void __launch_bounds__(256) minmax_partial_kernel(const float* __restrict__ x, long long n,
                                                             float* __restrict__ part_min,
                                                             float* __restrict__ part_max,
                                                             int* __restrict__ part_imin,
                                                             int* __restrict__ part_imax) {
  pdl_prologue();
  float tmin = FLT_MAX, tmax = -FLT_MAX;
  int imin = 0x7fffffff, imax = 0x7fffffff;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (v < tmin || (v == tmin && (int)i < imin)) {
      tmin = v;
      imin = (int)i;
    }
    if (v > tmax || (v == tmax && (int)i < imax)) {
      tmax = v;
      imax = (int)i;
    }
  }
  __shared__ float smin[256], smax[256];
  __shared__ int simin[256], simax[256];
  smin[threadIdx.x] = tmin;
  smax[threadIdx.x] = tmax;
  simin[threadIdx.x] = imin;
  simax[threadIdx.x] = imax;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 256; ++i) {
      if (smin[i] < tmin || (smin[i] == tmin && simin[i] < imin)) {
        tmin = smin[i];
        imin = simin[i];
      }
      if (smax[i] > tmax || (smax[i] == tmax && simax[i] < imax)) {
        tmax = smax[i];
        imax = simax[i];
      }
    }
    part_min[blockIdx.x] = tmin;
    part_max[blockIdx.x] = tmax;
    part_imin[blockIdx.x] = imin;
    part_imax[blockIdx.x] = imax;
  }
}

// One block folds the per-block partial extremes.  (value, then the smaller element index on ties) is a total order, so the
// fold is associative and commutative: any tree gives the same result.  1024 threads keep <= 4 partials each in flight
// (all loads issued before the first compare) and finish with warp shuffles; the previous 256-thread version walked the
// partials with dependent loads and folded 256 shared-memory slots serially in thread 0.
constexpr int MMR_THREADS = 1024;
__device__ __forceinline__ void mmr_take_min(float& v, int& i, float ov, int oi) {
  if (ov < v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}
__device__ __forceinline__ void mmr_take_max(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}
__global__ void __launch_bounds__(MMR_THREADS) minmax_reduce_kernel(const float* __restrict__ part_min,
                                                                    const float* __restrict__ part_max,
                                                                    const int* __restrict__ part_imin,
                                                                    const int* __restrict__ part_imax, int nparts,
                                                                    float* __restrict__ range, int* __restrict__ irange) {
  pdl_prologue();
  __shared__ float smin[32], smax[32];
  __shared__ int simin[32], simax[32];
  float tmin = FLT_MAX, tmax = -FLT_MAX;
  int imin = 0x7fffffff, imax = 0x7fffffff;
  for (int base = threadIdx.x; base < nparts; base += 4 * MMR_THREADS) {
    float a[4], b[4];
    int ia[4], ib[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = base + u * MMR_THREADS;
      const bool ok = i < nparts;
      a[u] = ok ? part_min[i] : FLT_MAX;
      b[u] = ok ? part_max[i] : -FLT_MAX;
      ia[u] = ok ? part_imin[i] : 0x7fffffff;
      ib[u] = ok ? part_imax[i] : 0x7fffffff;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      mmr_take_min(tmin, imin, a[u], ia[u]);
      mmr_take_max(tmax, imax, b[u], ib[u]);
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    mmr_take_min(tmin, imin, __shfl_xor_sync(0xffffffffu, tmin, o), __shfl_xor_sync(0xffffffffu, imin, o));
    mmr_take_max(tmax, imax, __shfl_xor_sync(0xffffffffu, tmax, o), __shfl_xor_sync(0xffffffffu, imax, o));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    smin[warp] = tmin;
    smax[warp] = tmax;
    simin[warp] = imin;
    simax[warp] = imax;
  }
  __syncthreads();
  if (warp == 0) {
    tmin = smin[lane];
    tmax = smax[lane];
    imin = simin[lane];
    imax = simax[lane];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      mmr_take_min(tmin, imin, __shfl_xor_sync(0xffffffffu, tmin, o), __shfl_xor_sync(0xffffffffu, imin, o));
      mmr_take_max(tmax, imax, __shfl_xor_sync(0xffffffffu, tmax, o), __shfl_xor_sync(0xffffffffu, imax, o));
    }
    if (lane == 0) {
      float R = tmax - tmin;  // max of (img - minv), slip.py:26-31
      range[0] = tmin;
      range[1] = (R != 0.f) ? R : 1.f;  // `if maxv != 0` (slip.py:33)
      range[2] = tmax;
      range[3] = (R != 0.f) ? 1.f : 0.f;  // whether the division (and so d/dmax) happened
      irange[0] = imin;
      irange[1] = imax;
    }
  }
}

// Cutout-sharded ranks: exchange buffer {min, -max} goes through one allreduce(min); afterwards every rank holds the
// global range, and only the rank that owns the extreme element keeps its index (others get -1).
__global__ void range_pack_kernel(const float* __restrict__ range, float* __restrict__ xbuf) {
  pdl_prologue();
  xbuf[0] = range[0];
  xbuf[1] = -range[2];
}
__global__ void range_unpack_kernel(const float* __restrict__ xbuf, float* __restrict__ range,
                                    int* __restrict__ irange) {
  pdl_prologue();
  const float gmin = xbuf[0], gmax = -xbuf[1];
  if (range[0] != gmin) irange[0] = -1;
  if (range[2] != gmax) irange[1] = -1;
  const float R = gmax - gmin;
  range[0] = gmin;
  range[1] = (R != 0.f) ? R : 1.f;
  range[2] = gmax;
  range[3] = (R != 0.f) ? 1.f : 0.f;
}

// channel c's entry of a per-channel kernel argument, by selects: a dynamic index would copy the argument to local memory
__device__ __forceinline__ float by_channel(const float (&v)[3], int c) { return c == 0 ? v[0] : (c == 1 ? v[1] : v[2]); }

// thread: 8 consecutive k of one patch row (ix..ix+7), requires P % 8 == 0
__global__ void __launch_bounds__(256) patchify_fwd_kernel(const float* __restrict__ batch,
                                                           const float* __restrict__ range, int n, int cs, int P,
                                                           int ld, act_t* __restrict__ patches, ChannelNorm nrm) {
  pdl_prologue();
  const int gp = cs / P;
  const int vec_per_row = 3 * P * P / 8;
  const long long total = (long long)n * gp * gp * vec_per_row;
  const float mn = range[0], R = range[1];
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    int kv = (int)(t % vec_per_row);
    long long row = t / vec_per_row;
    int px = (int)(row % gp), py = (int)((row / gp) % gp), b = (int)(row / (gp * gp));
    int k0 = kv * 8;
    int ix = k0 % P, iy = (k0 / P) % P, c = k0 / (P * P);
    const float* src = batch + (((size_t)b * 3 + c) * cs + py * P + iy) * cs + px * P + ix;
    float4 a = reinterpret_cast<const float4*>(src)[0], b4 = reinterpret_cast<const float4*>(src)[1];
    float v[8] = {a.x, a.y, a.z, a.w, b4.x, b4.y, b4.z, b4.w};
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
    const float mean = by_channel(nrm.mean, c), stdv = by_channel(nrm.std, c);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float y0 = (((v[2 * i] - mn) / R) - mean) / stdv;
      float y1 = (((v[2 * i + 1] - mn) / R) - mean) / stdv;
      h[i] = __floats2half2_rn(y0, y1);
    }
    *reinterpret_cast<uint4*>(patches + (size_t)row * ld + k0) = u;
  }
}

__global__ void __launch_bounds__(256) patchify_bwd_kernel(const act_t* __restrict__ g_patches,
                                                           const float* __restrict__ batch,
                                                           const float* __restrict__ range, int n, int cs, int P,
                                                           int ld, int accumulate, float* __restrict__ g_batch,
                                                           long long* __restrict__ sums, unsigned int* poison,
                                                           unsigned int pass, ChannelNorm nrm) {
  pdl_prologue();
  const int gp = cs / P;
  const int vec_per_row = 3 * P * P / 8;
  const long long total = (long long)n * gp * gp * vec_per_row;
  const float mn = range[0], R = range[1];
  float s1 = 0.f, s2 = 0.f;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    int kv = (int)(t % vec_per_row);
    long long row = t / vec_per_row;
    int px = (int)(row % gp), py = (int)((row / gp) % gp), b = (int)(row / (gp * gp));
    int k0 = kv * 8;
    int ix = k0 % P, iy = (k0 / P) % P, c = k0 / (P * P);
    size_t o = (((size_t)b * 3 + c) * cs + py * P + iy) * cs + px * P + ix;
    uint4 u = *reinterpret_cast<const uint4*>(g_patches + (size_t)row * ld + k0);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    float4 xa = reinterpret_cast<const float4*>(batch + o)[0], xb = reinterpret_cast<const float4*>(batch + o)[1];
    float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
    float g[8];
    const float k = 1.f / (by_channel(nrm.std, c) * R);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __half22float2(h[i]);
      g[2 * i] = f.x * k;
      g[2 * i + 1] = f.y * k;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1 += g[i];
      s2 += g[i] * (xv[i] - mn) / R;
    }
    float4* dst = reinterpret_cast<float4*>(g_batch + o);
    if (accumulate) {
      float4 p0 = dst[0], p1 = dst[1];
      dst[0] = make_float4(p0.x + g[0], p0.y + g[1], p0.z + g[2], p0.w + g[3]);
      dst[1] = make_float4(p1.x + g[4], p1.y + g[5], p1.z + g[6], p1.w + g[7]);
    } else {
      dst[0] = make_float4(g[0], g[1], g[2], g[3]);
      dst[1] = make_float4(g[4], g[5], g[6], g[7]);
    }
  }
  __shared__ float r1[8], r2[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) {
    r1[threadIdx.x >> 5] = s1;
    r2[threadIdx.x >> 5] = s2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < 8; ++i) {
      a += r1[i];
      b += r2[i];
    }
    fx_add(&sums[0], a, FX_SUM, FX_SUM_MAX, poison, pass);
    fx_add(&sums[1], b, FX_SUM, FX_SUM_MAX, poison, pass);
  }
}

// The block's share of the two range sums of the preprocess backward (sum g, sum g (x - min) / R): a fixed-order warp and
// block reduction, then one fixed-point add each.  256-thread blocks.
__device__ __forceinline__ void range_sums_block_add(float s1, float s2, long long* sums, unsigned int* poison,
                                                     unsigned int pass) {
  __shared__ float r1[8], r2[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) {
    r1[threadIdx.x >> 5] = s1;
    r2[threadIdx.x >> 5] = s2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b2 = 0.f;
    for (int i = 0; i < 8; ++i) {
      a += r1[i];
      b2 += r2[i];
    }
    fx_add(&sums[0], a, FX_SUM, FX_SUM_MAX, poison, pass);
    fx_add(&sums[1], b2, FX_SUM, FX_SUM_MAX, poison, pass);
  }
}

// Any patch size (e.g. ViT-L/14: P = 14): one thread per patch element, coalesced over k.
__global__ void __launch_bounds__(256) patchify_fwd_generic_kernel(const float* __restrict__ batch,
                                                                   const float* __restrict__ range, int n, int cs,
                                                                   int P, int ld, act_t* __restrict__ patches,
                                                                   ChannelNorm nrm) {
  pdl_prologue();
  const int gp = cs / P, K = 3 * P * P;
  const long long total = (long long)n * gp * gp * K;
  const float mn = range[0], R = range[1];
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(t % K);
    const long long row = t / K;
    const int px = (int)(row % gp), py = (int)((row / gp) % gp), b = (int)(row / (gp * gp));
    const int ix = k % P, iy = (k / P) % P, c = k / (P * P);
    const float v = batch[(((size_t)b * 3 + c) * cs + py * P + iy) * cs + px * P + ix];
    patches[(size_t)row * ld + k] = __float2half_rn((((v - mn) / R) - by_channel(nrm.mean, c)) / by_channel(nrm.std, c));
  }
}

// one thread per batch element (coalesced over x), gathers its gradient from the patch matrix
__global__ void __launch_bounds__(256) patchify_bwd_generic_kernel(const act_t* __restrict__ g_patches,
                                                                   const float* __restrict__ batch,
                                                                   const float* __restrict__ range, int n, int cs,
                                                                   int P, int ld, int accumulate,
                                                                   float* __restrict__ g_batch,
                                                                   long long* __restrict__ sums, unsigned int* poison,
                                                           unsigned int pass, ChannelNorm nrm) {
  pdl_prologue();
  const int gp = cs / P;
  const long long total = (long long)n * 3 * cs * cs;
  const float mn = range[0], R = range[1];
  float s1 = 0.f, s2 = 0.f;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % cs), y = (int)((t / cs) % cs), c = (int)((t / ((long long)cs * cs)) % 3);
    const int b = (int)(t / ((long long)3 * cs * cs));
    float g = 0.f;
    if (y < gp * P && x < gp * P) {
      const long long row = ((long long)b * gp + y / P) * gp + x / P;
      const int k = (c * P + y % P) * P + x % P;
      g = __half2float(g_patches[(size_t)row * ld + k]) / (by_channel(nrm.std, c) * R);
    }
    s1 += g;
    s2 += g * (batch[t] - mn) / R;
    g_batch[t] = accumulate ? g_batch[t] + g : g;
  }
  range_sums_block_add(s1, s2, sums, poison, pass);
}

// CLIP ResNet stem input: the stride-2, pad-1 3x3 im2col of the normalised cutouts, one thread per 8 of the 64 columns of
// an output pixel's row.  Column k < 27 = (c * 3 + ky) * 3 + kx (conv1.weight's [cout, 3, 3, 3] order); taps outside the
// image and columns 27..63 are 0 (the conv pads the normalised image with zeros).
__global__ void __launch_bounds__(256) rn_stem_fwd_kernel(const float* __restrict__ batch, const float* __restrict__ range,
                                                          int n, int cs, act_t* __restrict__ cols, ChannelNorm nrm) {
  pdl_prologue();
  const int ho = cs / 2;
  const long long total = (long long)n * ho * ho * 8;
  const float mn = range[0], R = range[1];
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int kv = (int)(t & 7);
    const long long row = t >> 3;
    const int ox = (int)(row % ho), oy = (int)((row / ho) % ho), b = (int)(row / ((long long)ho * ho));
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int k = kv * 8 + i;
      v[i] = 0.f;
      if (k < 27) {
        const int c = k / 9, ky = (k / 3) % 3, kx = k % 3;
        const int y = 2 * oy - 1 + ky, x = 2 * ox - 1 + kx;
        if (y >= 0 && y < cs && x >= 0 && x < cs) {
          const float a = batch[(((size_t)b * 3 + c) * cs + y) * cs + x];
          v[i] = (((a - mn) / R) - by_channel(nrm.mean, c)) / by_channel(nrm.std, c);
        }
      }
    }
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(cols + (size_t)row * 64 + kv * 8) = u;
  }
}

// its adjoint as a gather: one thread per batch element sums the (at most 4) column entries that read it, in a fixed tap
// order, so repeated runs give the same bits; the range sums as patchify_bwd_generic_kernel
__global__ void __launch_bounds__(256) rn_stem_bwd_kernel(const act_t* __restrict__ g_cols, const float* __restrict__ batch,
                                                          const float* __restrict__ range, int n, int cs, int accumulate,
                                                          float* __restrict__ g_batch, long long* __restrict__ sums,
                                                          unsigned int* poison, unsigned int pass, ChannelNorm nrm) {
  pdl_prologue();
  const int ho = cs / 2;
  const long long total = (long long)n * 3 * cs * cs;
  const float mn = range[0], R = range[1];
  float s1 = 0.f, s2 = 0.f;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % cs), y = (int)((t / cs) % cs), c = (int)((t / ((long long)cs * cs)) % 3);
    const int b = (int)(t / ((long long)3 * cs * cs));
    float g = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y + 1 - ky;  // = 2 oy
      if (yy < 0 || (yy & 1) || (yy >> 1) >= ho) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = x + 1 - kx;
        if (xx < 0 || (xx & 1) || (xx >> 1) >= ho) continue;
        const long long row = ((long long)b * ho + (yy >> 1)) * ho + (xx >> 1);
        g += __half2float(g_cols[(size_t)row * 64 + (c * 3 + ky) * 3 + kx]);
      }
    }
    g /= by_channel(nrm.std, c) * R;
    s1 += g;
    s2 += g * (batch[t] - mn) / R;
    g_batch[t] = accumulate ? g_batch[t] + g : g;
  }
  range_sums_block_add(s1, s2, sums, poison, pass);
}

__global__ void __launch_bounds__(CUT_THREADS) cutout_bwd_kernel(CutoutArgs a, const float* __restrict__ g_batch,
                                                                 const float* __restrict__ range,
                                                                 const int* __restrict__ irange,
                                                                 const float* __restrict__ sums,
                                                                 long long* __restrict__ g_pooled, unsigned int* poison,
                                                                 unsigned int pass) {
  pdl_prologue();
  const int n = blockIdx.y;
  const int n_global = a.first_global + n;
  const int cs = a.cs;
  const int grp = blockIdx.x * CUT_THREADS + threadIdx.x;
  if (grp >= cs * cs / 4) return;
  const int v = (grp * 4) / cs, u0 = (grp * 4) % cs;
  const bool zoom = n_global < a.cutn_zoom;
  const int padding = zoom ? a.zoom_padding : 2;
  float m[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) m[i] = a.minv[n * 9 + i];
  int cj_code = 0;
  float cj_sat = 1.f, cj_hue = 0.f;
  if (a.jitter) {
    cj_code = (int)a.jitter[n * 3];
    cj_sat = a.jitter[n * 3 + 1];
    cj_hue = a.jitter[n * 3 + 2];
  }
  // global range normalise: dL/dR = -sum g_a * a / R ; argmax gets +dR, argmin gets -(sum g_a + dR)
  const float dR = (range[3] != 0.f) ? -sums[1] : 0.f;
  const float dMin = -(sums[0] + dR);
  float g[3][4];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    size_t o = (((size_t)n * 3 + c) * cs + v) * cs + u0;
    float4 t = *reinterpret_cast<const float4*>(g_batch + o);
    g[c][0] = t.x;
    g[c][1] = t.y;
    g[c][2] = t.z;
    g[c][3] = t.w;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int e = (int)(o + j);
      if (e == irange[1]) g[c][j] += dR;
      if (e == irange[0]) g[c][j] += dMin;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float xs, ys;
    src_coord(m, u0 + j, v, xs, ys);
    xs = pad_coord(xs, a.src_w, padding);
    ys = pad_coord(ys, a.src_h, padding);
    Taps t = make_taps(xs, ys, a.src_w, a.src_h);
    float gpre[3] = {g[0][j], g[1][j], g[2][j]};
    if (cj_code) {  // through the ColorJitter Jacobian at the recomputed pre-jitter colour
      float rgb[3];
      warp_sample(a.pooled, t, a.src_w, a.src_h, zoom, a.fill, rgb);
      const float gout[3] = {gpre[0], gpre[1], gpre[2]};
      cj_vjp(rgb, cj_code, cj_sat, cj_hue, gout, gpre);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      long long* p = g_pooled + (size_t)c * a.src_h * a.src_w;
      const int sw = a.src_w;
      float gv = gpre[c];
      if (t.in[0]) fx_add(p + t.y0 * sw + t.x0, t.w[0] * gv, FX_GRAD, FX_GRAD_MAX, poison, pass);
      if (t.in[1]) fx_add(p + t.y0 * sw + t.x0 + 1, t.w[1] * gv, FX_GRAD, FX_GRAD_MAX, poison, pass);
      if (t.in[2]) fx_add(p + (t.y0 + 1) * sw + t.x0, t.w[2] * gv, FX_GRAD, FX_GRAD_MAX, poison, pass);
      if (t.in[3]) fx_add(p + (t.y0 + 1) * sw + t.x0 + 1, t.w[3] * gv, FX_GRAD, FX_GRAD_MAX, poison, pass);
    }
  }
}

}  // namespace

void pool_forward(const float* img, int H, int W, int cs, float* pooled, int* argmax, cudaStream_t st) {
  launch_pdl(pool_fwd_kernel, dim3((3 * cs * cs + 255) / 256), dim3(256), 0, st, img, H, W, cs, pooled, argmax);
}
void pool_backward(const float* g_pooled, const int* argmax, int H, int W, int cs, float* g_img, cudaStream_t st,
                   int accumulate) {
  launch_pdl(pool_bwd_kernel, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, g_pooled, argmax, H, W, cs, g_img, accumulate);
}
void spot_mask_apply(const float* x, const unsigned char* mask, int zero_where_set, int n, float* y, cudaStream_t st) {
  launch_pdl(spot_mask_kernel, dim3((n + 255) / 256), dim3(256), 0, st, x, mask, zero_where_set, n, y);
}

void rescale_bilinear(const float* x, int in_h, int in_w, int out_h, int out_w, float* y, cudaStream_t st) {
  launch_pdl(rescale_fwd_kernel, dim3((3 * out_h * out_w + 255) / 256), dim3(256), 0, st, x, in_h, in_w, out_h, out_w, y);
}
void rescale_bilinear_backward(const float* gy, int in_h, int in_w, int out_h, int out_w, long long* acc, FxPass fx, float* gx,
                               cudaStream_t st) {
  launch_pdl(rescale_bwd_kernel, dim3((3 * out_h * out_w + 255) / 256), dim3(256), 0, st, gy, in_h, in_w, out_h, out_w, acc, fx.poison,
             fx.pass);
  launch_pdl(fx_to_float_kernel, dim3((3 * in_h * in_w + 255) / 256), dim3(256), 0, st, acc, gx, 3 * in_h * in_w, FX_GRAD_INV,
             static_cast<const unsigned int*>(fx.poison), fx.pass);
}
void range_sums_finish(long long* acc, FxPass fx, float* sums, cudaStream_t st) {
  launch_pdl(fx_to_float_kernel, dim3(1), dim3(256), 0, st, acc, sums, 2, FX_SUM_INV, static_cast<const unsigned int*>(fx.poison),
             fx.pass);
}

int cutout_num_blocks(int n_local, int cs) { return n_local * ((cs * cs / 4 + CUT_THREADS - 1) / CUT_THREADS); }

void cutout_forward(const CutoutArgs& a, float* batch, float* part_min, float* part_max, int* part_imin,
                    int* part_imax, cudaStream_t st) {
  dim3 grid((a.cs * a.cs / 4 + CUT_THREADS - 1) / CUT_THREADS, a.n_local);
  launch_pdl(cutout_fwd_kernel, dim3(grid), dim3(CUT_THREADS), 0, st, a, batch, part_min, part_max, part_imin, part_imax);
}

void range_pack(const float* range, float* xbuf, cudaStream_t st) { launch_pdl(range_pack_kernel, dim3(1), dim3(1), 0, st, range, xbuf); }
void range_unpack(const float* xbuf, float* range, int* irange, cudaStream_t st) {
  launch_pdl(range_unpack_kernel, dim3(1), dim3(1), 0, st, xbuf, range, irange);
}

void minmax_partials(const float* x, long long n, int nparts, float* part_min, float* part_max, int* part_imin,
                     int* part_imax, cudaStream_t st) {
  launch_pdl(minmax_partial_kernel, dim3(nparts), dim3(256), 0, st, x, n, part_min, part_max, part_imin, part_imax);
}

void minmax_reduce(const float*, const float* part_min, const float* part_max, const int* part_imin,
                   const int* part_imax, int nparts, float* range, int* irange, cudaStream_t st) {
  launch_pdl(minmax_reduce_kernel, dim3(1), dim3(MMR_THREADS), 0, st, part_min, part_max, part_imin, part_imax, nparts, range, irange);
}

static int patch_grid(long long total) {
  long long g = (total + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  return (int)(g < 1 ? 1 : g);
}

void patchify_forward(const float* batch, const float* range, int n, int cs, int P, int ld, act_t* patches,
                      const ChannelNorm& nrm, cudaStream_t st) {
  if (P % 8) {
    const long long tot = (long long)n * (cs / P) * (cs / P) * 3 * P * P;
    launch_pdl(patchify_fwd_generic_kernel, dim3(patch_grid(tot)), dim3(256), 0, st, batch, range, n, cs, P, ld, patches, nrm);
    return;
  }
  const long long total = (long long)n * (cs / P) * (cs / P) * (3 * P * P / 8);
  launch_pdl(patchify_fwd_kernel, dim3(patch_grid(total)), dim3(256), 0, st, batch, range, n, cs, P, ld, patches, nrm);
}
void patchify_backward(const act_t* g_patches, const float* batch, const float* range, int n, int cs, int P, int ld,
                       int accumulate, float* g_batch, long long* sums, FxPass fx, const ChannelNorm& nrm, cudaStream_t st) {
  if (P % 8) {
    const long long tot = (long long)n * 3 * cs * cs;
    launch_pdl(patchify_bwd_generic_kernel, dim3(patch_grid(tot)), dim3(256), 0, st, g_patches, batch, range, n, cs, P, ld, accumulate,
                                                                 g_batch, sums, fx.poison, fx.pass, nrm);
    return;
  }
  const long long total = (long long)n * (cs / P) * (cs / P) * (3 * P * P / 8);
  launch_pdl(patchify_bwd_kernel, dim3(patch_grid(total)), dim3(256), 0, st, g_patches, batch, range, n, cs, P, ld, accumulate, g_batch,
                                                         sums, fx.poison, fx.pass, nrm);
}
void rn_stem_forward(const float* batch, const float* range, int n, int cs, act_t* cols, const ChannelNorm& nrm,
                     cudaStream_t st) {
  const long long total = (long long)n * (cs / 2) * (cs / 2) * 8;
  launch_pdl(rn_stem_fwd_kernel, dim3(patch_grid(total)), dim3(256), 0, st, batch, range, n, cs, cols, nrm);
}
void rn_stem_backward(const act_t* g_cols, const float* batch, const float* range, int n, int cs, int accumulate,
                      float* g_batch, long long* sums, FxPass fx, const ChannelNorm& nrm, cudaStream_t st) {
  const long long total = (long long)n * 3 * cs * cs;
  launch_pdl(rn_stem_bwd_kernel, dim3(patch_grid(total)), dim3(256), 0, st, g_cols, batch, range, n, cs, accumulate, g_batch,
             sums, fx.poison, fx.pass, nrm);
}
void cutout_backward(const CutoutArgs& a, const float* g_batch, const float* range, const int* irange,
                     const float* sums, long long* acc, FxPass fx, float* g_pooled, cudaStream_t st) {
  dim3 grid((a.cs * a.cs / 4 + CUT_THREADS - 1) / CUT_THREADS, a.n_local);
  launch_pdl(cutout_bwd_kernel, dim3(grid), dim3(CUT_THREADS), 0, st, a, g_batch, range, irange, sums, acc, fx.poison, fx.pass);
  const int n = 3 * a.src_h * a.src_w;
  launch_pdl(fx_to_float_kernel, dim3((n + 255) / 256), dim3(256), 0, st, acc, g_pooled, n, FX_GRAD_INV,
             static_cast<const unsigned int*>(fx.poison), fx.pass);
}

}  // namespace pxr
