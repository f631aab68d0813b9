// Polygon rasteriser of the pixel drawer's shaped cells (PixelDrawer.synth, pixeldrawer.py:330-367): the shapes never
// move and only their fill colours are optimised, so the render is linear in z = [n, 4] RGBA and its exact adjoint is a
// gather over the samples each polygon won.  See kernels.cuh for the contract and raster_samples.cuh for the samples.
#include "kernels.cuh"
#include "launch.cuh"
#include "raster_samples.cuh"

namespace pxr {
namespace {

// Even-odd rule by ray casting towards +x.  The crossing test is the sign of a cross product in double precision: the
// differences of fp32 coordinates and their products are exact there, so only the final subtraction rounds and the
// result is the exact answer for every sample that is not within ~1e-12 px of an edge.
__device__ __forceinline__ bool even_odd_contains(const float2* __restrict__ v, int nv, float px, float py) {
  bool in = false;
  const double X = px, Y = py;
  double xj = v[nv - 1].x, yj = v[nv - 1].y;
  for (int i = 0; i < nv; ++i) {
    const double xi = v[i].x, yi = v[i].y;
    if ((yi > Y) != (yj > Y)) {
      // X < crossing x of edge (i, j) at Y  <=>  sign((xj - xi)(Y - yi) - (X - xi)(yj - yi)) == sign(yj - yi)
      const double cr = (xj - xi) * (Y - yi) - (X - xi) * (yj - yi);
      if (yj > yi ? cr > 0.0 : cr < 0.0) in = !in;
    }
    xj = xi;
    yj = yi;
  }
  return in;
}

__global__ void __launch_bounds__(256) raster_fwd_kernel(RasterScene s, const float* __restrict__ z, int H, int W,
                                                         uint64_t seed, int iter, int* __restrict__ winner,
                                                         float* __restrict__ img) {
  pdl_launch_dependents();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int HW = H * W;
  if (p >= HW) return;
  const int x = p % W, y = p / W;
  // the scene (vertices, boxes, tile lists) is uploaded once at finalize: readable before the wait
  const int t = (y / RASTER_TILE) * s.tiles_x + x / RASTER_TILE;
  const int b = s.tile_start[t], e = s.tile_start[t + 1];
  float sx[4], sy[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) raster_sample(seed, iter, x, y, W, k, sx[k], sy[k]);
  pdl_wait();
  float r = 0.f, g = 0.f, bl = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int win = -1;
    for (int i = b; i < e; ++i) {
      const int q = s.tile_list[i];
      const float4 bb = s.bbox[q];
      if (sx[k] < bb.x || sx[k] > bb.z || sy[k] < bb.y || sy[k] > bb.w) continue;
      const int o = s.off[q];
      if (even_odd_contains(s.xy + o, s.off[q + 1] - o, sx[k], sy[k])) {
        win = q;
        break;
      }
    }
    winner[(size_t)k * HW + p] = win;
    if (win >= 0) {
      r += z[4 * win];
      g += z[4 * win + 1];
      bl += z[4 * win + 2];
    }
  }
  img[p] = r * 0.25f;
  img[HW + p] = g * 0.25f;
  img[2 * HW + p] = bl * 0.25f;
}

__global__ void __launch_bounds__(256) raster_bwd_kernel(RasterScene s, const int* __restrict__ winner,
                                                         const float* __restrict__ g_img, int H, int W, float scale,
                                                         float* __restrict__ z_grad) {
  pdl_launch_dependents();
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= s.n) return;
  // a sample of pixel x lies in [x, x + 1] (closed: fp32 rounding), so the pixels whose samples can fall inside the
  // box [x0, x1] are floor(x0) - 1 .. floor(x1)
  // box <- clamped to one pixel around the canvas first, so far-away coordinates convert to int safely
  const float4 bb = s.bbox[k];
  const float cw = (float)W + 1.f, ch = (float)H + 1.f;
  const int px0 = max(0, (int)floorf(fminf(fmaxf(bb.x, -1.f), cw)) - 1), px1 = min(W - 1, (int)floorf(fminf(fmaxf(bb.z, -1.f), cw)));
  const int py0 = max(0, (int)floorf(fminf(fmaxf(bb.y, -1.f), ch)) - 1), py1 = min(H - 1, (int)floorf(fminf(fmaxf(bb.w, -1.f), ch)));
  const int bw = px1 - px0 + 1, cnt = (px1 >= px0 && py1 >= py0) ? bw * (py1 - py0 + 1) : 0;
  const int HW = H * W;
  pdl_wait();
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int i = lane; i < cnt; i += 32) {
    const int p = (py0 + i / bw) * W + px0 + i % bw;
    const int hits = (winner[p] == k) + (winner[HW + p] == k) + (winner[2 * HW + p] == k) + (winner[3 * HW + p] == k);
    if (hits) {
      a0 += (float)hits * g_img[p];
      a1 += (float)hits * g_img[HW + p];
      a2 += (float)hits * g_img[2 * HW + p];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // butterfly: fixed order, every lane ends with the same sums
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
  }
  if (lane == 0) {
    z_grad[4 * k] = a0 * scale;
    z_grad[4 * k + 1] = a1 * scale;
    z_grad[4 * k + 2] = a2 * scale;
    z_grad[4 * k + 3] = 0.f;  // alpha: clip_z pins it to 1 after every step (pixeldrawer.py:382)
  }
}

}  // namespace

void raster_forward(const RasterScene& s, const float* z, int H, int W, uint64_t seed, int iter, int* winner, float* img,
                    cudaStream_t st) {
  launch_pdl(raster_fwd_kernel, dim3((H * W + 255) / 256), dim3(256), 0, st, s, z, H, W, seed, iter, winner, img);
}

void raster_backward(const RasterScene& s, const int* winner, const float* g_img, int H, int W, float inv_scale,
                     float* z_grad, cudaStream_t st) {
  launch_pdl(raster_bwd_kernel, dim3((s.n + 7) / 8), dim3(256), 0, st, s, winner, g_img, H, W, 0.25f * inv_scale, z_grad);
}

}  // namespace pxr
