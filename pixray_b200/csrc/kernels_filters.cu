// Image filters between drawer.synth and MakeCutouts (do_synth_and_filter, pixray.py:1203-1222; filters/tiler.py,
// filters/wallpaper.py, filters/colorlookup.py): rolls, tiling, edge trims with an edge-match loss, and the nearest-palette
// colour lookup (straight-through) -- planar fp32 [3, H, W] images, forward + adjoint + loss gradients.  HBM-trivial
// (one image), launch-latency bound; PDL chained like the rest of the iteration.
#include "kernels.cuh"
#include "launch.cuh"

namespace pxr {
namespace {

// y[c, (i + sh) % H, (j + sw) % W] = x[c, i, j]   (torch.roll(x, shifts=(sh, sw), dims=(2, 3)))
// backward: gx[c, i, j] (=|+=) gy[c, (i + sh) % H, (j + sw) % W]
template <bool BWD>
__global__ void roll_kernel(const float* __restrict__ in, int H, int W, int sh, int sw, int accumulate,
                            float* __restrict__ out) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H * W) return;
  const int x = i % W, y = (i / W) % H, c = i / (W * H);
  const int yy = (y + sh) % H, xx = (x + sw) % W;
  const size_t rolled = ((size_t)c * H + yy) * W + xx;
  if (BWD) out[i] = accumulate ? out[i] + in[rolled] : in[rolled];
  else out[rolled] = in[i];
}

// wallpaper "shift" (wallpaper.py:33-44): two_rows = cat([x, roll(x, W/2 along w)], dim=2), then roll by (sh, sw) over
// the [2H, W] canvas.  y: [3, 2H, W].
__global__ void wallpaper_shift_fwd_kernel(const float* __restrict__ x, int H, int W, int sh, int sw, float* __restrict__ y) {
  pdl_prologue();
  const int H2 = 2 * H;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H2 * W) return;
  const int xo = i % W, yo = (i / W) % H2, c = i / (W * H2);
  // un-roll: position in two_rows
  const int yt = (yo - sh % H2 + H2) % H2, xt = (xo - sw % W + W) % W;
  const int ys = yt < H ? yt : yt - H;
  const int xs = yt < H ? xt : (xt - W / 2 + W) % W;  // row2[x] = x_src[(x - W/2) mod W]
  y[i] = x[((size_t)c * H + ys) * W + xs];
}
__global__ void wallpaper_shift_bwd_kernel(const float* __restrict__ gy, int H, int W, int sh, int sw, int accumulate,
                                           float* __restrict__ gx) {
  pdl_prologue();
  const int H2 = 2 * H;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H * W) return;
  const int xs = i % W, ys = (i / W) % H, c = i / (W * H);
  // the two places source pixel (ys, xs) went: two_rows[ys, xs] and two_rows[H + ys, (xs + W/2) mod W], both rolled
  const int y1 = (ys + sh) % H2, x1 = (xs + sw) % W;
  const int y2 = (H + ys + sh) % H2, x2 = ((xs + W / 2) % W + sw) % W;
  const float g = gy[((size_t)c * H2 + y1) * W + x1] + gy[((size_t)c * H2 + y2) * W + x2];
  gx[i] = accumulate ? gx[i] + g : g;
}

// crop [top, top + Hc) x [left, left + Wc); backward writes zeros outside
__global__ void crop_fwd_kernel(const float* __restrict__ x, int H, int W, int top, int left, int Hc, int Wc,
                                float* __restrict__ y) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * Hc * Wc) return;
  const int xo = i % Wc, yo = (i / Wc) % Hc, c = i / (Wc * Hc);
  y[i] = x[((size_t)c * H + top + yo) * W + left + xo];
}
__global__ void crop_bwd_kernel(const float* __restrict__ gy, int H, int W, int top, int left, int Hc, int Wc,
                                float* __restrict__ gx) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * H * W) return;
  const int xs = i % W, ys = (i / W) % H, c = i / (W * H);
  const int yo = ys - top, xo = xs - left;
  gx[i] = (yo >= 0 && yo < Hc && xo >= 0 && xo < Wc) ? gy[((size_t)c * Hc + yo) * Wc + xo] : 0.f;
}

// edge match (wallpaper.py:47-53, 58-66): loss = mse(x[first em], x[last em]) / em along one axis; single block reduces in
// a fixed order (the strips are small).  axis 0: columns (horizontal wrap), axis 1: rows.  loss_out (=|+=) weight * loss.
__global__ void edge_match_loss_kernel(const float* __restrict__ x, int H, int W, int em, int axis, float weight,
                                       int accumulate_loss, float* __restrict__ loss_out) {
  pdl_prologue();
  const int n = axis == 0 ? 3 * H * em : 3 * em * W;
  const float k = 1.f / ((float)n * (float)em);
  __shared__ double red[256];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    size_t ia, ib;
    if (axis == 0) {
      const int xe = i % em, y = (i / em) % H, c = i / (em * H);
      ia = ((size_t)c * H + y) * W + xe;
      ib = ((size_t)c * H + y) * W + (W - em + xe);
    } else {
      const int xw = i % W, ye = (i / W) % em, c = i / (W * em);
      ia = ((size_t)c * H + ye) * W + xw;
      ib = ((size_t)c * H + (H - em + ye)) * W + xw;
    }
    const float d = x[ia] - x[ib];
    s += (double)d * d;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)blockDim.x; ++i) t += red[i];
    const float l = weight * (float)(t * (double)k);
    *loss_out = accumulate_loss ? *loss_out + l : l;
  }
}
// its gradient, g += grad_scale * weight * dloss/dx, in gather form: one thread per element of the union of the two strips
// (the first em and the last em positions along the axis; the whole axis when 2 em > size, where the strips overlap and an
// element takes both terms), so every element has one writer and its value does not depend on scheduling.
__global__ void edge_match_grad_kernel(const float* __restrict__ x, int H, int W, int em, int axis, float weight,
                                       float grad_scale, float* __restrict__ g) {
  pdl_prologue();
  const int L = axis == 0 ? W : H, other = axis == 0 ? H : W;
  const int nu = 2 * em < L ? 2 * em : L;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * other * nu) return;
  int j, r, c;
  if (axis == 0) {
    j = i % nu, r = (i / nu) % H, c = i / (nu * H);
  } else {
    r = i % W, j = (i / W) % nu, c = i / (W * nu);
  }
  const int n = 3 * other * em, lo = L - em;
  const float k = 1.f / ((float)n * (float)em), coef = grad_scale * weight * 2.f * k;
  auto at = [&](int p) -> size_t { return axis == 0 ? ((size_t)c * H + r) * W + p : ((size_t)c * H + p) * W + r; };
  const int p = j < em ? j : L - nu + j;  // position along the axis
  float v = g[at(p)];
  if (p < em) v += coef * (x[at(p)] - x[at(lo + p)]);            // p in the first strip: + d(p)
  if (p >= lo) v -= coef * (x[at(p - lo)] - x[at(p)]);           // p in the last strip: - d(p - (L - em))
  g[at(p)] = v;
}

// ColorLookup (colorlookup.py:51-86): z_q = nearest palette colour (torch.cdist + argmin: first minimum), value out = z_q,
// gradient straight through; loss = beta * mean((z_q.detach() - z)^2) + mean((z_q - z.detach())^2) -- the second term has no
// gradient (the table is a constant).  partial sums per block in double, fixed order.
__global__ void colorlookup_fwd_kernel(const float* __restrict__ x, int pixels, const float* __restrict__ pal, int n_col,
                                       float* __restrict__ y, int* __restrict__ best_out, double* __restrict__ part) {
  pdl_prologue();
  __shared__ double red[256];
  double s = 0.0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < pixels; p += gridDim.x * blockDim.x) {
    const float r = x[p], gch = x[(size_t)pixels + p], b = x[(size_t)2 * pixels + p];
    float best = 3.0e38f;
    int bi = 0;
    for (int k = 0; k < n_col; ++k) {
      const float dr = r - pal[3 * k], dg = gch - pal[3 * k + 1], db = b - pal[3 * k + 2];
      const float d = sqrtf(dr * dr + dg * dg + db * db);  // cdist is the Euclidean distance; first minimum wins
      if (d < best) {
        best = d;
        bi = k;
      }
    }
    const float qr = pal[3 * bi], qg = pal[3 * bi + 1], qb = pal[3 * bi + 2];
    y[p] = qr;
    y[(size_t)pixels + p] = qg;
    y[(size_t)2 * pixels + p] = qb;
    if (best_out) best_out[p] = bi;
    s += (double)(qr - r) * (qr - r) + (double)(qg - gch) * (qg - gch) + (double)(qb - b) * (qb - b);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)blockDim.x; ++i) t += red[i];
    part[blockIdx.x] = t;
  }
}
__global__ void colorlookup_loss_kernel(const double* __restrict__ part, int nblk, int pixels, float beta, float weight,
                                        float* __restrict__ loss_out) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double t = 0.0;
  for (int i = 0; i < nblk; ++i) t += part[i];
  *loss_out = weight * (beta + 1.f) * (float)(t / (3.0 * pixels));
}
// gx (=|+=) gy (straight through) + grad_scale * weight * beta * 2 (x - z_q) / N
__global__ void colorlookup_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ x, const float* __restrict__ y,
                                       int n, float beta, float weight, float grad_scale, int accumulate,
                                       float* __restrict__ gx) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float g = gy[i] + grad_scale * weight * beta * 2.f * (x[i] - y[i]) / (float)n;
  gx[i] = accumulate ? gx[i] + g : g;
}

}  // namespace

void filter_roll(const float* x, int H, int W, int sh, int sw, float* y, cudaStream_t st) {
  launch_pdl(roll_kernel<false>, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, x, H, W, sh, sw, 0, y);
}
void filter_roll_backward(const float* gy, int H, int W, int sh, int sw, int accumulate, float* gx, cudaStream_t st) {
  launch_pdl(roll_kernel<true>, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, gy, H, W, sh, sw, accumulate, gx);
}
void filter_wallpaper_shift(const float* x, int H, int W, int sh, int sw, float* y, cudaStream_t st) {
  launch_pdl(wallpaper_shift_fwd_kernel, dim3((3 * 2 * H * W + 255) / 256), dim3(256), 0, st, x, H, W, sh, sw, y);
}
void filter_wallpaper_shift_backward(const float* gy, int H, int W, int sh, int sw, int accumulate, float* gx, cudaStream_t st) {
  launch_pdl(wallpaper_shift_bwd_kernel, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, gy, H, W, sh, sw, accumulate, gx);
}
void filter_crop(const float* x, int H, int W, int top, int left, int Hc, int Wc, float* y, cudaStream_t st) {
  launch_pdl(crop_fwd_kernel, dim3((3 * Hc * Wc + 255) / 256), dim3(256), 0, st, x, H, W, top, left, Hc, Wc, y);
}
void filter_crop_backward(const float* gy, int H, int W, int top, int left, int Hc, int Wc, float* gx, cudaStream_t st) {
  launch_pdl(crop_bwd_kernel, dim3((3 * H * W + 255) / 256), dim3(256), 0, st, gy, H, W, top, left, Hc, Wc, gx);
}
void filter_edge_match(const float* x, int H, int W, int em, int axis, float weight, float grad_scale, int accumulate_loss,
                       float* g, float* loss_out, cudaStream_t st) {
  if (loss_out) launch_pdl(edge_match_loss_kernel, dim3(1), dim3(256), 0, st, x, H, W, em, axis, weight, accumulate_loss, loss_out);
  if (g) {
    const int L = axis == 0 ? W : H, n = 3 * (axis == 0 ? H : W) * (2 * em < L ? 2 * em : L);
    launch_pdl(edge_match_grad_kernel, dim3((n + 255) / 256), dim3(256), 0, st, x, H, W, em, axis, weight, grad_scale, g);
  }
}
void filter_colorlookup(const float* x, int pixels, const float* pal, int n_col, float beta, float weight, float* y,
                        int* best_out, double* part, float* loss_out, cudaStream_t st) {
  int nblk = (pixels + 255) / 256;
  if (nblk > AUX_MAX_BLOCKS) nblk = AUX_MAX_BLOCKS;
  launch_pdl(colorlookup_fwd_kernel, dim3(nblk), dim3(256), 0, st, x, pixels, pal, n_col, y, best_out, part);
  launch_pdl(colorlookup_loss_kernel, dim3(1), dim3(32), 0, st, part, nblk, pixels, beta, weight, loss_out);
}
void filter_colorlookup_backward(const float* gy, const float* x, const float* y, int pixels, float beta, float weight,
                                 float grad_scale, int accumulate, float* gx, cudaStream_t st) {
  const int n = 3 * pixels;
  launch_pdl(colorlookup_bwd_kernel, dim3((n + 255) / 256), dim3(256), 0, st, gy, x, y, n, beta, weight, grad_scale, accumulate, gx);
}

}  // namespace pxr
