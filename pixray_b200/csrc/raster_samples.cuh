// Sample positions of the polygon rasteriser (kernels_raster.cu), shared with the test hook pxr_test_raster_samples so
// the tests see exactly the positions the kernels use.
//
// diffvg renders PixelDrawer's scene with 2 x 2 stratified jittered samples per pixel (pixeldrawer.py:342,
// `render(W, H, 2, 2, cur_iteration, ...)`): sample s = dx + 2 dy of pixel (x, y) lies at
// (x + (dx + u) / 2, y + (dy + v) / 2), u, v ~ U[0, 1).  Here u, v come from Philox keyed by (seed, iteration) and counted
// by (pixel, sample) -- not by rank, so every rank renders the same image, and not by the gradient-accumulation pass, so
// every pass of one iteration sees the same render.  u and v carry 23 random bits, so dx + u is exact in fp32; the final
// x + ... rounds to fp32 and can land on the upper edge of the stratum.
#pragma once
#include "philox.cuh"

namespace pxr {

constexpr uint32_t kRasterStream = 7u;  // Philox stream id (0-6 are the cutout noise, transforms, jitter and filters)

__host__ __device__ inline void raster_sample(uint64_t seed, int iter, int x, int y, int W, int s, float& sx, float& sy) {
  const Philox4 r = philox4x32_10((uint32_t)(y * W + x), (uint32_t)s, (uint32_t)iter, kRasterStream, (uint32_t)seed,
                                  (uint32_t)(seed >> 32));
  const float u = (float)(r.v[0] >> 9) * (1.0f / 8388608.0f), v = (float)(r.v[1] >> 9) * (1.0f / 8388608.0f);
  sx = (float)x + ((float)(s & 1) + u) * 0.5f;
  sy = (float)y + ((float)(s >> 1) + v) * 0.5f;
}

}  // namespace pxr
