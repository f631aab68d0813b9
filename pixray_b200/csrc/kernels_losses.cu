// Auxiliary losses of the reference (Losses/*.py behind LossInterface.get_loss, pixray.py:1384-1393) as fused
// loss + gradient kernels.  Each launcher adds  grad_scale * weight * dL/dx  into the engine's fp32 gradient buffer of
// the tensor the reference loss reads (`out` -> g_img, the cutout batch -> g_batch, the embeddings -> de) and writes the
// weighted loss value.  All of them are single-pass, HBM / L2-bound gather-pointwise kernels with 16-byte-free scalar
// accesses on planar fp32 data (coalesced along x); reductions are block partials in double folded in a fixed order
// (no atomics: the cutout-sharded ranks must agree bit for bit).
//
//   symmetry   Losses/SymmetryLoss.py:14-17     saturation  Losses/SaturationLoss.py:15-30
//   palette    Losses/PaletteLoss.py:25-35      smoothness  Losses/SmoothnessLoss.py:89-108
//   edge       Losses/EdgeLoss.py:60-108        gaussian    Losses/GaussianLoss.py:31-44
//   aesthetic  Losses/AestheticLoss.py:30-33
#include "kernels.cuh"
#include <cstdio>

namespace pxr {

namespace {

constexpr int AUX_THREADS = 256;

// block-wide sum in a fixed order; result valid on thread 0
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double sh[AUX_THREADS / 32];
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < AUX_THREADS / 32; ++w) t += sh[w];
  __syncthreads();
  return t;
}

// out[k] (=|+=) scale * sum_b part[b * stride + k]   for k < nslots; one block
__global__ void aux_final_kernel(const double* __restrict__ part, int nblk, int stride, int nslots, double scale,
                                 float* __restrict__ out_f, double* __restrict__ out_d, int accumulate) {
  for (int k = 0; k < nslots; ++k) {
    double a = 0.0;
    for (int b = threadIdx.x; b < nblk; b += AUX_THREADS) a += part[(size_t)b * stride + k];
    const double t = block_sum(a);
    if (threadIdx.x == 0) {
      if (out_d) out_d[k] = t * scale;
      if (out_f) out_f[k] = (accumulate ? out_f[k] : 0.f) + (float)(t * scale);
    }
  }
}

inline int aux_grid(long long n) {
  long long g = (n + AUX_THREADS - 1) / AUX_THREADS;
  return (int)(g > AUX_MAX_BLOCKS ? AUX_MAX_BLOCKS : (g < 1 ? 1 : g));
}

// ------------------------------------------------------------------ image losses: `out` planar fp32 [3, H, W]
__global__ void __launch_bounds__(AUX_THREADS) symmetry_kernel(const float* __restrict__ img, int H, int W,
                                                               float gcoef, float* __restrict__ g_img,
                                                               double* __restrict__ part) {
  const long long n = 3LL * H * W;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % W);
    const float d = img[i] - img[i - x + (W - 1 - x)];  // out - flip(out, [3])
    acc += (double)d * d;
    g_img[i] += gcoef * d;  // the pair (x, W-1-x) appears twice in the mean: 4 d / N
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

struct EdgeArgs {
  int left, right, upper, lower;
  float color[3];
  float inv_l, inv_r, inv_u, inv_d, gw;  // 1 / element count of each strip (0 when the margin is 0), global weight / N
  const float* target;  // [3, H, W] edge_input_image resized to the image, or null: the flat colour
  const float* mask;    // [H, W] edge_mask_image resized to the image, or null: the margins
  float inv_n;          // 1 / (3 H W): the masked term is a mean over every element, masked ones included
};

__global__ void __launch_bounds__(AUX_THREADS) edge_kernel(const float* __restrict__ img, int H, int W, EdgeArgs a,
                                                           float gcoef, float* __restrict__ g_img,
                                                           double* __restrict__ part) {
  const long long n = 3LL * H * W;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % W), y = (int)((i / W) % H), c = (int)(i / ((long long)W * H));
    float w = a.gw;
    if (a.mask) {
      // mse(where(mask > 0, target, out), target): only the unmasked elements differ from the target (EdgeLoss.py:100-103)
      if (!(a.mask[(size_t)y * W + x] > 0.f)) w += a.inv_n;
    } else {
      const bool mid = x >= a.left && x < W - a.right;  // the upper / lower strips exclude the corner columns (EdgeLoss.py:91-92)
      if (x < a.left) w += a.inv_l;
      if (x >= W - a.right) w += a.inv_r;
      if (mid && y < a.upper) w += a.inv_u;
      if (mid && y >= H - a.lower) w += a.inv_d;
    }
    const float d = img[i] - (a.target ? a.target[i] : a.color[c]);
    acc += (double)(w * d) * d;
    g_img[i] += gcoef * w * d;
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

__global__ void __launch_bounds__(AUX_THREADS) gaussian_kernel(const float* __restrict__ img, int H, int W, float stdy,
                                                               float stdx, float c0, float c1, float c2, float gcoef,
                                                               float* __restrict__ g_img, double* __restrict__ part) {
  const long long n = 3LL * H * W;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % W), y = (int)((i / W) % H), c = (int)(i / ((long long)W * H));
    const float ny = (float)y - (H - 1.0f) / 2.0f, nx = (float)x - (W - 1.0f) / 2.0f;
    const float gaus = expf(-ny * ny / (2.f * stdy * stdy)) * expf(-nx * nx / (2.f * stdx * stdx));
    const float m = fabsf(1.f - gaus);
    const float d = img[i] - (c == 0 ? c0 : (c == 1 ? c1 : c2));
    acc += (double)(fabsf(d) * m);
    g_img[i] += gcoef * m * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

// ------------------------------------------------------------------ cutout losses: batch fp32 [n, 3, cs, cs]
__global__ void __launch_bounds__(AUX_THREADS) palette_kernel(const float* __restrict__ batch, int n_img, int hw,
                                                              const float* __restrict__ palette, int n_colors,
                                                              float gcoef, float* __restrict__ g_batch,
                                                              int* __restrict__ best_out, double* __restrict__ part) {
  const long long n = (long long)n_img * hw;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const long long img = i / hw, p = i % hw;
    const size_t o = (size_t)img * 3 * hw + p;
    const float r = batch[o], g = batch[o + hw], b = batch[o + 2 * (size_t)hw];
    int best = 0;
    float bd = 3.0e38f;
    for (int k = 0; k < n_colors; ++k) {  // argmin over the palette, first minimum wins (torch argmin)
      const float dr = r - palette[3 * k], dg = g - palette[3 * k + 1], db = b - palette[3 * k + 2];
      const float d2 = dr * dr + dg * dg + db * db;
      if (d2 < bd) {
        bd = d2;
        best = k;
      }
    }
    if (best_out) best_out[i] = best;
    const float dr = r - palette[3 * best], dg = g - palette[3 * best + 1], db = b - palette[3 * best + 2];
    const float nrm = sqrtf(dr * dr + dg * dg + db * db);
    acc += (double)nrm;
    const float s = nrm > 0.f ? gcoef / nrm : 0.f;  // d |v| / dv = v / |v| (0 at 0, like torch.norm's subgradient)
    g_batch[o] += s * dr;
    g_batch[o + hw] += s * dg;
    g_batch[o + 2 * (size_t)hw] += s * db;
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

// saturation, phase 1: sums of rg, rg^2, yb, yb^2 over this rank's cutout pixels
__global__ void __launch_bounds__(AUX_THREADS) saturation_moments_kernel(const float* __restrict__ batch, int n_img,
                                                                         int hw, double* __restrict__ part) {
  const long long n = (long long)n_img * hw;
  double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const long long img = i / hw, p = i % hw;
    const size_t o = (size_t)img * 3 * hw + p;
    const float r = batch[o], g = batch[o + hw], b = batch[o + 2 * (size_t)hw];
    const double rg = (double)r - g, yb = 0.5 * ((double)r + g) - b;
    s0 += rg;
    s1 += rg * rg;
    s2 += yb;
    s3 += yb * yb;
  }
  double t = block_sum(s0);
  if (threadIdx.x == 0) part[blockIdx.x * 4 + 0] = t;
  t = block_sum(s1);
  if (threadIdx.x == 0) part[blockIdx.x * 4 + 1] = t;
  t = block_sum(s2);
  if (threadIdx.x == 0) part[blockIdx.x * 4 + 2] = t;
  t = block_sum(s3);
  if (threadIdx.x == 0) part[blockIdx.x * 4 + 3] = t;
}

// saturation, phase 2: per-pixel gradient from the GLOBAL moments (sums over every rank's cutouts), loss on one thread
__global__ void __launch_bounds__(AUX_THREADS) saturation_grad_kernel(const float* __restrict__ batch, int n_img, int hw,
                                                                      const double* __restrict__ sums, double n_glob,
                                                                      float coef /* -w/10 */, float grad_scale,
                                                                      int write_loss, float* __restrict__ g_batch,
                                                                      float* __restrict__ loss_out) {
  const double rg_mean = sums[0] / n_glob, yb_mean = sums[2] / n_glob;
  // torch.std_mean: unbiased variance
  double rg_var = (sums[1] - n_glob * rg_mean * rg_mean) / (n_glob - 1.0), yb_var = (sums[3] - n_glob * yb_mean * yb_mean) / (n_glob - 1.0);
  if (rg_var < 0) rg_var = 0;
  if (yb_var < 0) yb_var = 0;
  const double std_rggb = sqrt(rg_var + yb_var), mean_rggb = sqrt(rg_mean * rg_mean + yb_mean * yb_mean);
  if (write_loss && blockIdx.x == 0 && threadIdx.x == 0) *loss_out += (float)((std_rggb + 0.3 * mean_rggb) * coef);
  // d colourfulness / d rg_i = (rg_i - rg_mean) / ((n-1) std_rggb) + 0.3 rg_mean / (n mean_rggb)
  const float k_std = std_rggb > 0 ? (float)(coef * (double)grad_scale / ((n_glob - 1.0) * std_rggb)) : 0.f;
  const float k_rg = mean_rggb > 0 ? (float)(coef * (double)grad_scale * 0.3 * rg_mean / (n_glob * mean_rggb)) : 0.f;
  const float k_yb = mean_rggb > 0 ? (float)(coef * (double)grad_scale * 0.3 * yb_mean / (n_glob * mean_rggb)) : 0.f;
  const float rgm = (float)rg_mean, ybm = (float)yb_mean;
  const long long n = (long long)n_img * hw;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const long long img = i / hw, p = i % hw;
    const size_t o = (size_t)img * 3 * hw + p;
    const float r = batch[o], g = batch[o + hw], b = batch[o + 2 * (size_t)hw];
    const float d_rg = k_std * ((r - g) - rgm) + k_rg, d_yb = k_std * ((0.5f * (r + g) - b) - ybm) + k_yb;
    g_batch[o] += d_rg + 0.5f * d_yb;
    g_batch[o + hw] += -d_rg + 0.5f * d_yb;
    g_batch[o + 2 * (size_t)hw] += -d_yb;
  }
}

// ---- smoothness.  The reference reshapes the batch to [cutn * cs, cs, 3] and takes torch.gradient over that 2-D
// grid, so the row difference runs across cutout boundaries (and, when the cutouts are sharded, across ranks: the
// two rows either side of this rank's slab come in through `halo`).  With smoothness_gaussian_kernel the grid is the
// blurred batch (side cs' = cs - taps + 1, see blur_axis_kernel), and `cs` below is that side.
struct SmoothArgs {
  const float* batch;  // [n_img, 3, cs, cs]
  const float* halo;   // [2 sides][2 rows][3][cs]: rows (-2, -1) and (rows, rows + 1) of the global stack, or unused
  int n_img, cs;
  long long g0, gt;    // global index of local row 0, total rows of the global stack (cutn * cs)
  float inv_sp;        // 1 / spacing
  int kind;            // 0 default, 1 clipped (max 0.5), 2 log(1 + s)
  int order;           // torch.gradient edge_order: 1 or 2 (only the first / last point of each axis differ)
};

__device__ __forceinline__ float sm_x(const SmoothArgs& a, int c, long long r, int x) {
  const long long rows = (long long)a.n_img * a.cs;
  if (r >= 0 && r < rows) {
    const long long img = r / a.cs, y = r % a.cs;
    return a.batch[((size_t)img * 3 + c) * a.cs * a.cs + (size_t)y * a.cs + x];
  }
  const int side = r < 0 ? 0 : 1;
  const int k = r < 0 ? (int)(r + 2) : (int)(r - rows);
  return a.halo[(((size_t)side * 2 + k) * 3 + c) * a.cs + x];
}
// d/drow at local row r (global row g0 + r must exist), torch.gradient
__device__ __forceinline__ float sm_gy(const SmoothArgs& a, int c, long long r, int x) {
  const long long G = a.g0 + r;
  if (G == 0) {
    if (a.order == 2)  // (-3 f0 + 4 f1 - f2) / 2h
      return (-1.5f * sm_x(a, c, r, x) + 2.f * sm_x(a, c, r + 1, x) - 0.5f * sm_x(a, c, r + 2, x)) * a.inv_sp;
    return (sm_x(a, c, r + 1, x) - sm_x(a, c, r, x)) * a.inv_sp;
  }
  if (G == a.gt - 1) {
    if (a.order == 2)  // (3 fn - 4 fn-1 + fn-2) / 2h
      return (1.5f * sm_x(a, c, r, x) - 2.f * sm_x(a, c, r - 1, x) + 0.5f * sm_x(a, c, r - 2, x)) * a.inv_sp;
    return (sm_x(a, c, r, x) - sm_x(a, c, r - 1, x)) * a.inv_sp;
  }
  return (sm_x(a, c, r + 1, x) - sm_x(a, c, r - 1, x)) * (0.5f * a.inv_sp);
}
__device__ __forceinline__ float sm_gx(const SmoothArgs& a, int c, long long r, int x) {
  if (x == 0) {
    if (a.order == 2) return (-1.5f * sm_x(a, c, r, 0) + 2.f * sm_x(a, c, r, 1) - 0.5f * sm_x(a, c, r, 2)) * a.inv_sp;
    return (sm_x(a, c, r, 1) - sm_x(a, c, r, 0)) * a.inv_sp;
  }
  if (x == a.cs - 1) {
    if (a.order == 2) return (1.5f * sm_x(a, c, r, x) - 2.f * sm_x(a, c, r, x - 1) + 0.5f * sm_x(a, c, r, x - 2)) * a.inv_sp;
    return (sm_x(a, c, r, x) - sm_x(a, c, r, x - 1)) * a.inv_sp;
  }
  return (sm_x(a, c, r, x + 1) - sm_x(a, c, r, x - 1)) * (0.5f * a.inv_sp);
}
// weight of f(o + d) in torch.gradient's derivative at point o (global index Go of n points along the axis)
__device__ __forceinline__ float sm_w(long long Go, long long n, int d, int order, float inv_sp) {
  if (Go == 0) {
    if (order == 2) return d == 0 ? -1.5f * inv_sp : (d == 1 ? 2.f * inv_sp : (d == 2 ? -0.5f * inv_sp : 0.f));
    return d == 0 ? -inv_sp : (d == 1 ? inv_sp : 0.f);
  }
  if (Go == n - 1) {
    if (order == 2) return d == 0 ? 1.5f * inv_sp : (d == -1 ? -2.f * inv_sp : (d == -2 ? 0.5f * inv_sp : 0.f));
    return d == 0 ? inv_sp : (d == -1 ? -inv_sp : 0.f);
  }
  return d == 1 ? 0.5f * inv_sp : (d == -1 ? -0.5f * inv_sp : 0.f);
}

// phase 1: per pixel of rows [-1, rows]: A = coef * f'(s) / s (0 where the global row does not exist); loss partials
// over the local rows only.  A is laid out [(rows + 2), cs] with row -1 first.
__global__ void __launch_bounds__(AUX_THREADS) smooth_sharp_kernel(SmoothArgs a, float coef, float* __restrict__ A,
                                                                   double* __restrict__ part) {
  const long long rows = (long long)a.n_img * a.cs;
  const long long n = (rows + 2) * a.cs;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const long long r = i / a.cs - 1;
    const int x = (int)(i % a.cs);
    const long long G = a.g0 + r;
    float out = 0.f;
    if (G >= 0 && G < a.gt) {
      float sq = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float gy = sm_gy(a, c, r, x), gx = sm_gx(a, c, r, x);
        sq += gy * gy + gx * gx;
      }
      const float s = sqrtf(sq);
      float f = s, df = 1.f;
      if (a.kind == 1) {
        f = fminf(s, 0.5f);
        df = s <= 0.5f ? 1.f : 0.f;
      } else if (a.kind == 2) {
        f = logf(1.f + s);
        df = 1.f / (1.f + s);
      }
      if (r >= 0 && r < rows) acc += (double)f;
      out = s > 0.f ? coef * df / s : 0.f;
    }
    A[i] = out;
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

// phase 2 (gather form of the stencil's adjoint): d loss / d X(c, r, x) for every local element, added into g_out
// (accumulate) or stored (the blurred path's scratch).  An edge_order 2 end point reads two rows / columns inward; the
// global first / last rows are always local (every rank holds >= 3 rows then), so A is only read inside [-1, rows].
__global__ void __launch_bounds__(AUX_THREADS) smooth_grad_kernel(SmoothArgs a, const float* __restrict__ A,
                                                                  float* __restrict__ g_out, int accumulate) {
  const long long rows = (long long)a.n_img * a.cs;
  const long long n = rows * a.cs * 3;
  const int cs = a.cs, R = a.order;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % cs);
    const long long q = i / cs;
    const int y = (int)(q % cs);
    const int c = (int)((q / cs) % 3);
    const long long img = q / ((long long)cs * 3);
    const long long r = img * cs + y;
    float g = 0.f;
    // rows whose d/drow reads X(r): r - R .. r + R
    for (int dr = -R; dr <= R; ++dr) {
      const long long ro = r + dr, G = a.g0 + ro;
      if (G < 0 || G >= a.gt) continue;
      const float w = sm_w(G, a.gt, -dr, a.order, a.inv_sp);
      if (w != 0.f) g += w * A[(ro + 1) * cs + x] * sm_gy(a, c, ro, x);
    }
    // columns whose d/dcol reads X(x) (same row)
    for (int dx = -R; dx <= R; ++dx) {
      const int xo = x + dx;
      if (xo < 0 || xo >= cs) continue;
      const float w = sm_w(xo, cs, -dx, a.order, a.inv_sp);
      if (w != 0.f) g += w * A[(r + 1) * cs + xo] * sm_gx(a, c, r, xo);
    }
    g_out[i] = accumulate ? g_out[i] + g : g;
  }
}

// GaussianSmoothing (SmoothnessLoss.py:9-72) as two 1-D passes: its 2-D kernel is the outer product of one vector with
// itself normalised to sum 1, i.e. u (x) u with u = v / sum(v).  Valid correlation of planes [P, Hs, Ws] along one axis
// (0: rows, 1: columns) with the n taps u; the output loses n - 1 lines along that axis.
__global__ void __launch_bounds__(AUX_THREADS) blur_axis_kernel(const float* __restrict__ src, int P, int Hs, int Ws,
                                                                int axis, const float* __restrict__ u, int n,
                                                                float* __restrict__ dst) {
  const int Ho = axis == 0 ? Hs - n + 1 : Hs, Wo = axis == 1 ? Ws - n + 1 : Ws;
  const long long total = (long long)P * Ho * Wo;
  const int step = axis == 0 ? Ws : 1;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % Wo);
    const long long q = i / Wo;
    const int y = (int)(q % Ho);
    const long long p = q / Ho;
    const float* s = src + ((size_t)p * Hs + y) * Ws + x;
    float acc = 0.f;
    for (int t = 0; t < n; ++t) acc = fmaf(__ldg(u + t), s[(size_t)t * step], acc);
    dst[i] = acc;
  }
}
// its adjoint (full correlation with the flipped taps) as a gather: dst [P, Hd, Wd] (+)= sum_t u[t] src[j - t], one
// writer per element
__global__ void __launch_bounds__(AUX_THREADS) blur_axis_adjoint_kernel(const float* __restrict__ src, int P, int Hd,
                                                                        int Wd, int axis, const float* __restrict__ u,
                                                                        int n, float* __restrict__ dst, int accumulate) {
  const int Hs = axis == 0 ? Hd - n + 1 : Hd, Ws = axis == 1 ? Wd - n + 1 : Wd;
  const int L = axis == 0 ? Hs : Ws;
  const int step = axis == 0 ? Ws : 1;
  const long long total = (long long)P * Hd * Wd;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * AUX_THREADS) {
    const int x = (int)(i % Wd);
    const long long q = i / Wd;
    const int y = (int)(q % Hd);
    const long long p = q / Hd;
    const int j = axis == 0 ? y : x;
    const int t0 = j - (L - 1) > 0 ? j - (L - 1) : 0, t1 = j < n - 1 ? j : n - 1;
    // src element at line j - t of the blurred axis, same position on the other axis
    const float* s = src + (size_t)p * Hs * Ws + (axis == 0 ? (size_t)x : (size_t)y * Ws) + (size_t)j * step;
    float acc = 0.f;
    for (int t = t0; t <= t1; ++t) acc = fmaf(__ldg(u + t), s[-(long long)t * step], acc);
    dst[i] = accumulate ? dst[i] + acc : acc;
  }
}

// first / last two rows of this rank's stack -> slot `rank` of the exchange buffer [world][2 sides][2][3][cs]
__global__ void smooth_pack_halo_kernel(const float* __restrict__ batch, int n_img, int cs, int rank,
                                        float* __restrict__ xbuf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over [2][2][3][cs]
  if (i >= 12 * cs) return;
  const int x = i % cs, c = (i / cs) % 3, k = (i / (3 * cs)) % 2, side = i / (6 * cs);
  const long long rows = (long long)n_img * cs;
  const long long r = side == 0 ? k : rows - 2 + k;
  const long long img = r / cs, y = r % cs;
  xbuf[(size_t)rank * 12 * cs + i] = batch[((size_t)img * 3 + c) * cs * cs + (size_t)y * cs + x];
}
// after the allreduce: halo = {previous rank's last two rows, next rank's first two rows}
__global__ void smooth_unpack_halo_kernel(const float* __restrict__ xbuf, int cs, int rank, int world,
                                          float* __restrict__ halo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over [2 sides][2][3][cs]
  if (i >= 12 * cs) return;
  const int side = i / (6 * cs), rest = i % (6 * cs);
  float v = 0.f;
  if (side == 0 && rank > 0) v = xbuf[(size_t)(rank - 1) * 12 * cs + 6 * cs + rest];
  if (side == 1 && rank < world - 1) v = xbuf[(size_t)(rank + 1) * 12 * cs + rest];
  halo[i] = v;
}

// ------------------------------------------------------------------ aesthetic head on the embeddings
// one block per local cutout: u = e / |e|; rating = w . u + b; loss += c0 (rating - target)^2;
// de += grad_scale * c1 (rating - target) (w - (w . u) u) / |e|   (both F.normalize calls project, the 2nd is idempotent)
__global__ void __launch_bounds__(128) aesthetic_kernel(const float* __restrict__ e, int D, const float* __restrict__ w,
                                                        float bias, float target, float c1_scaled,
                                                        float* __restrict__ de, __half* __restrict__ de16,
                                                        double* __restrict__ part) {
  const int n = blockIdx.x;
  const float* en = e + (size_t)n * D;
  __shared__ float red[2][4];
  float s_ee = 0.f, s_we = 0.f;
  for (int k = threadIdx.x; k < D; k += 128) {
    s_ee += en[k] * en[k];
    s_we += w[k] * en[k];
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s_ee += __shfl_down_sync(0xffffffffu, s_ee, o);
    s_we += __shfl_down_sync(0xffffffffu, s_we, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s_ee;
    red[1][threadIdx.x >> 5] = s_we;
  }
  __syncthreads();
  const float ee = (red[0][0] + red[0][1]) + (red[0][2] + red[0][3]);
  const float we = (red[1][0] + red[1][1]) + (red[1][2] + red[1][3]);
  const float nrm = fmaxf(sqrtf(ee), 1e-12f);
  const float wu = we / nrm;  // w . u
  const float diff = wu + bias - target;
  if (threadIdx.x == 0) part[n] = (double)diff * diff;
  const float k = c1_scaled * diff / nrm;
  for (int j = threadIdx.x; j < D; j += 128) {
    const float u = en[j] / nrm;
    const float v = de[(size_t)n * D + j] + k * (w[j] - wu * u);
    de[(size_t)n * D + j] = v;
    de16[(size_t)n * D + j] = __float2half_rn(v);
  }
}


// ------------------------------------------------------------------ anchors to a stored copy (pixray.py:1344-1375)
// z-space terms between drawer.get_z() and a reference tensor of the same shape, flattened to one row:
//   kind 0  spherical_dist_loss(z, ref) * w            (init_weight, pixray.py:1352-1356; image_labels, 1344-1349)
//   kind 1  F.mse_loss(z, ref) * w / 2                 (init_weight_dist, 1359-1361)
//   kind 2  F.cosine_embedding_loss(z, ref, 1) * w     (init_weight_cos, 1370-1375)
// One block: n is the latent (65536 floats for a 256^2 VQGAN); sums in double, fixed order.  Adds w * dL/dz to z_grad.
constexpr int ANCHOR_THREADS = 1024;

__device__ __forceinline__ double anchor_block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();  // sh may still be read from the previous sum
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < ANCHOR_THREADS / 32; ++w) t += sh[w];  // every thread folds in the same order
  return t;
}

__global__ void __launch_bounds__(ANCHOR_THREADS) anchor_z_kernel(int kind, const float* __restrict__ z,
                                                                  const float* __restrict__ ref, int n, float weight,
                                                                  float* __restrict__ z_grad, float* __restrict__ slot) {
  __shared__ double sh[ANCHOR_THREADS / 32];
  double zz = 0.0, rr = 0.0, zr = 0.0, dd = 0.0;
  for (int i = threadIdx.x; i < n; i += ANCHOR_THREADS) {
    const double a = z[i], b = ref[i];
    zz += a * a;
    rr += b * b;
    zr += a * b;
    dd += (a - b) * (a - b);
  }
  zz = anchor_block_sum(zz, sh);
  rr = anchor_block_sum(rr, sh);
  zr = anchor_block_sum(zr, sh);
  dd = anchor_block_sum(dd, sh);
  if (kind == 1) {
    if (threadIdx.x == 0) *slot = (float)(0.5 * weight * dd / n);
    const float c = weight / (float)n;
    for (int i = threadIdx.x; i < n; i += ANCHOR_THREADS) z_grad[i] += c * (z[i] - ref[i]);
    return;
  }
  if (kind == 2) {
    const double den = sqrt((zz + 1e-12) * (rr + 1e-12));  // torch's cosine_embedding_loss: EPSILON = 1e-12 under the root
    const double cs = zr / den;
    if (threadIdx.x == 0) *slot = (float)(weight * (1.0 - cs));
    const float cr = (float)(weight / den), cz = (float)(weight * cs / (zz + 1e-12));
    for (int i = threadIdx.x; i < n; i += ANCHOR_THREADS) z_grad[i] += cz * z[i] - cr * ref[i];
    return;
  }
  // spherical: x = normalize(z), y = normalize(ref); d = |x - y|; L = 2 asin(d / 2)^2
  const double nz = fmax(sqrt(zz), 1e-12), nr = fmax(sqrt(rr), 1e-12);
  double d2 = 0.0, xs = 0.0;  // |x - y|^2 and x . (x - y), summed from the differences (no 2 - 2 x.y cancellation)
  for (int i = threadIdx.x; i < n; i += ANCHOR_THREADS) {
    const double x = z[i] / nz, y = ref[i] / nr;
    d2 += (x - y) * (x - y);
    xs += x * (x - y);
  }
  d2 = anchor_block_sum(d2, sh);
  xs = anchor_block_sum(xs, sh);
  const double d = sqrt(d2), half = fmin(0.5 * d, 1.0);
  const double as = asin(half);
  if (threadIdx.x == 0) *slot = (float)(weight * 2.0 * as * as);
  // dL/dd = 2 asin(d/2) / sqrt(1 - d^2/4);  dd/dx = (x - y) / d (0 at d == 0, torch's norm backward);  dx/dz = (I - x x^T) / |z|
  const double c = d > 0.0 ? weight * 2.0 * as / sqrt(fmax(1.0 - half * half, 1e-30)) / d / nz : 0.0;
  for (int i = threadIdx.x; i < n; i += ANCHOR_THREADS) {
    const double x = z[i] / nz, y = ref[i] / nr;
    z_grad[i] += (float)(c * ((x - y) - x * xs));
  }
}

// F.l1_loss(out, init_image_tensor) * w / 2 (init_weight_pix, pixray.py:1363-1368): sign() gradient into g_img
__global__ void __launch_bounds__(AUX_THREADS) anchor_pix_kernel(const float* __restrict__ img, const float* __restrict__ ref,
                                                                 long long n, float gcoef, float* __restrict__ g_img,
                                                                 double* __restrict__ part) {
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)AUX_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * AUX_THREADS) {
    const float d = img[i] - ref[i];
    acc += fabsf(d);
    g_img[i] += d > 0.f ? gcoef : (d < 0.f ? -gcoef : 0.f);
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = t;
}

}  // namespace

void anchor_z(int kind, const float* z, const float* ref, int n, float weight, float* z_grad, float* loss_out,
              cudaStream_t st) {
  anchor_z_kernel<<<1, ANCHOR_THREADS, 0, st>>>(kind, z, ref, n, weight, z_grad, loss_out);
}

void anchor_pix(const float* img, const float* ref, long long n, float weight, float grad_scale, float* g_img, double* part,
                float* loss_out, cudaStream_t st) {
  const int grid = aux_grid(n);
  anchor_pix_kernel<<<grid, AUX_THREADS, 0, st>>>(img, ref, n, 0.5f * weight * grad_scale / (float)n, g_img, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 1, 1, 0.5 * (double)weight / (double)n, loss_out, nullptr, 0);
}

void aux_symmetry(const float* img, int H, int W, float weight, float grad_scale, float* g_img, double* part,
                  float* loss_out, cudaStream_t st) {
  const long long n = 3LL * H * W;
  const int grid = aux_grid(n);
  symmetry_kernel<<<grid, AUX_THREADS, 0, st>>>(img, H, W, 4.f * weight * grad_scale / (float)n, g_img, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 1, 1, (double)weight / (double)n, loss_out, nullptr, 0);
}

void aux_edge(const float* img, int H, int W, const int margins[4], const float color[3], const float* target,
              const float* mask, float edge_color_weight, float global_color_weight, float weight, float grad_scale,
              float* g_img, double* part, float* loss_out, cudaStream_t st) {
  EdgeArgs a;
  a.left = margins[0];
  a.right = margins[1];
  a.upper = margins[2];
  a.lower = margins[3];
  for (int c = 0; c < 3; ++c) a.color[c] = color[c];
  const int mid = W - a.left - a.right;
  a.inv_l = a.left > 0 ? 1.f / (3.f * H * a.left) : 0.f;
  a.inv_r = a.right > 0 ? 1.f / (3.f * H * a.right) : 0.f;
  a.inv_u = (a.upper > 0 && mid > 0) ? 1.f / (3.f * a.upper * mid) : 0.f;
  a.inv_d = (a.lower > 0 && mid > 0) ? 1.f / (3.f * a.lower * mid) : 0.f;
  const long long n = 3LL * H * W;
  a.gw = global_color_weight / (float)n;
  a.target = target;
  a.mask = mask;
  a.inv_n = 1.f / (float)n;
  const int grid = aux_grid(n);
  const float k = edge_color_weight * weight;
  edge_kernel<<<grid, AUX_THREADS, 0, st>>>(img, H, W, a, 2.f * k * grad_scale, g_img, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 1, 1, (double)k, loss_out, nullptr, 0);
}

void aux_gaussian(const float* img, int H, int W, float stdy, float stdx, const float color255[3], float weight,
                  float grad_scale, float* g_img, double* part, float* loss_out, cudaStream_t st) {
  const long long n = 3LL * H * W;
  const int grid = aux_grid(n);
  gaussian_kernel<<<grid, AUX_THREADS, 0, st>>>(img, H, W, stdy, stdx, color255[0] / 255.f, color255[1] / 255.f,
                                                color255[2] / 255.f, weight * grad_scale / (float)n, g_img, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 1, 1, (double)weight / (double)n, loss_out, nullptr, 0);
}

void aux_palette(const float* batch, int n_img, int cs, int cutn_global, const float* palette_dev, int n_colors,
                 float weight, float grad_scale, float* g_batch, int* best_out, double* part, float* loss_out,
                 cudaStream_t st) {
  // mean over all cutn_global * cs^2 pixels, times cutn_global, times palette_weight / 10 (weight carries the latter two)
  const int hw = cs * cs;
  const long long n = (long long)n_img * hw;
  const int grid = aux_grid(n);
  const double k = (double)weight / 10.0 / (double)hw;
  (void)cutn_global;
  palette_kernel<<<grid, AUX_THREADS, 0, st>>>(batch, n_img, hw, palette_dev, n_colors, (float)(k * grad_scale), g_batch,
                                               best_out, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 1, 1, k, loss_out, nullptr, 1);
}

void aux_saturation_moments(const float* batch, int n_img, int cs, double* part, double* sums, cudaStream_t st) {
  const int hw = cs * cs;
  const int grid = aux_grid((long long)n_img * hw);
  saturation_moments_kernel<<<grid, AUX_THREADS, 0, st>>>(batch, n_img, hw, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid, 4, 4, 1.0, nullptr, sums, 0);
}

void aux_saturation_grad(const float* batch, int n_img, int cs, int cutn_global, const double* sums, float weight,
                         float grad_scale, int write_loss, float* g_batch, float* loss_out, cudaStream_t st) {
  const int hw = cs * cs;
  const int grid = aux_grid((long long)n_img * hw);
  saturation_grad_kernel<<<grid, AUX_THREADS, 0, st>>>(batch, n_img, hw, sums, (double)cutn_global * hw, -weight / 10.f,
                                                       grad_scale, write_loss, g_batch, loss_out);
}

void aux_smoothness(const float* batch, int n_img, int cs, int first_global, int cutn_global, const float* halo,
                    float spacing, int kind, int edge_order, float weight, float grad_scale, float* A, float* g_batch,
                    int accumulate, double* part, float* loss_out, cudaStream_t st) {
  SmoothArgs a;
  a.batch = batch;
  a.halo = halo;
  a.n_img = n_img;
  a.cs = cs;
  a.g0 = (long long)first_global * cs;
  a.gt = (long long)cutn_global * cs;
  a.inv_sp = 1.f / spacing;
  a.kind = kind;
  a.order = edge_order;
  const double n_glob = (double)cutn_global * cs * cs;
  const long long rows = (long long)n_img * cs;
  const int grid1 = aux_grid((rows + 2) * cs);
  smooth_sharp_kernel<<<grid1, AUX_THREADS, 0, st>>>(a, (float)(weight * grad_scale / n_glob), A, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, grid1, 1, 1, (double)weight / n_glob, loss_out, nullptr, 1);
  smooth_grad_kernel<<<aux_grid(rows * cs * 3), AUX_THREADS, 0, st>>>(a, A, g_batch, accumulate);
}

void aux_smooth_blur(const float* batch, int n_img, int cs, const float* taps, int n, float* tmp, float* out,
                     cudaStream_t st) {
  const int P = 3 * n_img, cs2 = cs - n + 1;
  blur_axis_kernel<<<aux_grid((long long)P * cs * cs2), AUX_THREADS, 0, st>>>(batch, P, cs, cs, 1, taps, n, tmp);
  blur_axis_kernel<<<aux_grid((long long)P * cs2 * cs2), AUX_THREADS, 0, st>>>(tmp, P, cs, cs2, 0, taps, n, out);
}
void aux_smooth_blur_adjoint(const float* g_out, int n_img, int cs, const float* taps, int n, float* tmp, float* g_batch,
                             cudaStream_t st) {
  const int P = 3 * n_img, cs2 = cs - n + 1;
  blur_axis_adjoint_kernel<<<aux_grid((long long)P * cs * cs2), AUX_THREADS, 0, st>>>(g_out, P, cs, cs2, 0, taps, n, tmp, 0);
  blur_axis_adjoint_kernel<<<aux_grid((long long)P * cs * cs), AUX_THREADS, 0, st>>>(tmp, P, cs, cs, 1, taps, n, g_batch, 1);
}

void aux_smooth_pack_halo(const float* batch, int n_img, int cs, int rank, float* xbuf, cudaStream_t st) {
  smooth_pack_halo_kernel<<<(12 * cs + 255) / 256, 256, 0, st>>>(batch, n_img, cs, rank, xbuf);
}
void aux_smooth_unpack_halo(const float* xbuf, int cs, int rank, int world, float* halo, cudaStream_t st) {
  smooth_unpack_halo_kernel<<<(12 * cs + 255) / 256, 256, 0, st>>>(xbuf, cs, rank, world, halo);
}

void aux_aesthetic(const float* e, int n_local, int D, int cutn_global, const float* w_dev, float bias, float target,
                   float weight, float grad_scale, float* de, __half* de16, double* part, float* loss_out,
                   cudaStream_t st) {
  // loss = weight * 0.02 * mean_n (rating_n - target)^2
  const double c0 = (double)weight * 0.02 / (double)cutn_global;
  aesthetic_kernel<<<n_local, 128, 0, st>>>(e, D, w_dev, bias, target, (float)(2.0 * c0 * grad_scale), de, de16, part);
  aux_final_kernel<<<1, AUX_THREADS, 0, st>>>(part, n_local, 1, 1, c0, loss_out, nullptr, 1);
}

}  // namespace pxr
