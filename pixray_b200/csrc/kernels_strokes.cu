// Line-sketch rasteriser (LineDrawer.synth, linedrawer.py:156-166): open cubic Bézier paths stroked in opaque black over
// an opaque paper rectangle.  Unlike the polygon drawer the geometry itself is optimised, so the backward is the
// derivative of the box-filtered coverage with respect to the outline: a boundary integral (kernels.cuh StrokeScene).
#include "kernels.cuh"
#include "launch.cuh"
#include "raster_samples.cuh"

namespace pxr {
namespace {

constexpr int CAP_GRAD = 5;  // per capsule: d/da (x, y), d/db (x, y), d/dw

__device__ __forceinline__ float bernstein(int m, float t) {
  const float u = 1.f - t;
  return m == 0 ? u * u * u : m == 1 ? 3.f * t * u * u : m == 2 ? 3.f * t * t * u : t * t * t;
}

__device__ __forceinline__ float seg_dist2(float px, float py, float4 c) {
  const float ex = c.z - c.x, ey = c.w - c.y, dx = px - c.x, dy = py - c.y, ll = ex * ex + ey * ey;
  const float t = ll > 0.f ? fminf(fmaxf((dx * ex + dy * ey) / ll, 0.f), 1.f) : 0.f;
  const float rx = dx - t * ex, ry = dy - t * ey;
  return rx * rx + ry * ry;
}

__device__ __forceinline__ float cap_width(const StrokeScene& s, const float* __restrict__ z, int c) {
  return z[s.width_offset + c / (s.n_segments * STROKE_CHORDS)];
}

// tile j covers the closed interval [j T, (j + 1) T]; the value is clamped to one tile around the canvas first, so far-away
// coordinates convert to int safely and a box entirely off the canvas gets an empty range
__device__ __forceinline__ int tile_lo(float v, int n) {
  const float T = (float)RASTER_TILE;
  return max(0, (int)ceilf(fminf(fmaxf(v, -T), n * T + T) / T) - 1);
}
__device__ __forceinline__ int tile_hi(float v, int n) {
  const float T = (float)RASTER_TILE;
  return min(n - 1, (int)floorf(fminf(fmaxf(v, -T), n * T + T) / T));
}

// control points -> chord endpoints at t = i / S and the tile range of each capsule's box grown by its width
__global__ void __launch_bounds__(256) stroke_flatten_kernel(StrokeScene s, const float* __restrict__ z) {
  pdl_launch_dependents();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= s.n_caps) return;
  const int i = c % STROKE_CHORDS, seg = c / STROKE_CHORDS, j = seg % s.n_segments, k = seg / s.n_segments;
  pdl_wait();
  const float* P = z + ((size_t)k * (3 * s.n_segments + 1) + 3 * j) * 2;
  const float t0 = (float)i / STROKE_CHORDS, t1 = (float)(i + 1) / STROKE_CHORDS;
  float ax = 0.f, ay = 0.f, bx = 0.f, by = 0.f;
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    const float wa = bernstein(m, t0), wb = bernstein(m, t1);
    ax += wa * P[2 * m];
    ay += wa * P[2 * m + 1];
    bx += wb * P[2 * m];
    by += wb * P[2 * m + 1];
  }
  const float w = z[s.width_offset + k];
  s.caps[c] = make_float4(ax, ay, bx, by);
  s.cap_tiles[c] = make_int4(tile_lo(fminf(ax, bx) - w, s.tiles_x), tile_lo(fminf(ay, by) - w, s.tiles_y),
                             tile_hi(fmaxf(ax, bx) + w, s.tiles_x), tile_hi(fmaxf(ay, by) + w, s.tiles_y));
}

__device__ __forceinline__ bool in_tile(int4 r, int tx, int ty) {
  return tx >= r.x && tx <= r.z && ty >= r.y && ty <= r.w;
}

// one block per tile: tile_start[t + 1] = number of capsules whose range holds tile t
__global__ void __launch_bounds__(256) stroke_bin_count_kernel(StrokeScene s) {
  pdl_launch_dependents();
  __shared__ int part[8];
  const int t = blockIdx.x, tx = t % s.tiles_x, ty = t / s.tiles_x;
  pdl_wait();
  int n = 0;
  for (int c = threadIdx.x; c < s.n_caps; c += blockDim.x) n += in_tile(s.cap_tiles[c], tx, ty);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int sum = 0;
    for (int w = 0; w < 8; ++w) sum += part[w];
    s.tile_start[t + 1] = sum;
    if (t == 0) s.tile_start[0] = 0;
  }
}

// inclusive scan of tile_start[1 .. tiles] in place (one block)
__global__ void __launch_bounds__(1024) stroke_bin_scan_kernel(StrokeScene s) {
  pdl_launch_dependents();
  __shared__ int part[1024];
  const int n = s.tiles_x * s.tiles_y, per = (n + 1023) / 1024, b = 1 + threadIdx.x * per, e = min(n + 1, b + per);
  pdl_wait();
  int sum = 0;
  for (int i = b; i < e; ++i) sum += s.tile_start[i];
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 1; i < 1024; ++i) part[i] += part[i - 1];
  __syncthreads();
  int run = threadIdx.x ? part[threadIdx.x - 1] : 0;
  for (int i = b; i < e; ++i) {
    run += s.tile_start[i];
    s.tile_start[i] = run;
  }
}

// one block per tile: the capsules of the tile in descending index order (topmost path first), by ordered compaction
__global__ void __launch_bounds__(256) stroke_bin_fill_kernel(StrokeScene s) {
  pdl_launch_dependents();
  __shared__ int warp_n[8];
  const int t = blockIdx.x, tx = t % s.tiles_x, ty = t / s.tiles_x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  pdl_wait();
  int out = s.tile_start[t];
  for (int base = 0; base < s.n_caps; base += blockDim.x) {
    const int c = s.n_caps - 1 - (base + (int)threadIdx.x);
    const bool hit = c >= 0 && in_tile(s.cap_tiles[c], tx, ty);
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_n[wid] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < 8; ++w) {
      before += w < wid ? warp_n[w] : 0;
      total += warp_n[w];
    }
    if (hit) s.tile_list[out + before + __popc(m & ((1u << lane) - 1u))] = c;
    out += total;
    __syncthreads();
  }
}

__device__ __forceinline__ void paper_rgba(const StrokeScene& s, const float* __restrict__ z, float P[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) P[q] = z[s.width_offset + s.n_paths + q];
}

// one thread per pixel: the 4 samples' winners (topmost covering path or -1) and the synth composite of the box-filtered
// RGBA: rgb (1 - c) paper_rgb, alpha c + (1 - c) paper_a, out = rgb alpha + (1 - alpha)
__global__ void __launch_bounds__(256) stroke_fwd_kernel(StrokeScene s, const float* __restrict__ z, uint64_t seed, int iter,
                                                         float* __restrict__ img) {
  pdl_launch_dependents();
  const int W = s.W, H = s.H, HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int x = p % W, y = p / W;
  float sx[4], sy[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) raster_sample(seed, iter, x, y, W, k, sx[k], sy[k]);
  pdl_wait();
  const int t = (y / RASTER_TILE) * s.tiles_x + x / RASTER_TILE, b = s.tile_start[t], e = s.tile_start[t + 1];
  int covered = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int win = -1;
    for (int i = b; i < e; ++i) {
      const int c = s.tile_list[i];
      const float w = cap_width(s, z, c);
      if (seg_dist2(sx[k], sy[k], s.caps[c]) <= w * w) {
        win = c / (s.n_segments * STROKE_CHORDS);
        break;
      }
    }
    s.winner[(size_t)k * HW + p] = win;
    covered += win >= 0;
  }
  float P[4];
  paper_rgba(s, z, P);
  const float cv = 0.25f * (float)covered, A = cv + (1.f - cv) * P[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) img[(size_t)q * HW + p] = (1.f - cv) * P[q] * A + 1.f - A;
}

// per pixel: G = sum_ch g_ch d out_ch / d c at the forward's coverage c, and the paper colour's gradient (interior term)
// reduced per block in a fixed order
__global__ void __launch_bounds__(256) stroke_pixel_kernel(StrokeScene s, const float* __restrict__ z,
                                                           const float* __restrict__ g_img) {
  pdl_launch_dependents();
  __shared__ float red[4][256];
  const int HW = s.H * s.W, p = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();
  float gp[4] = {0.f, 0.f, 0.f, 0.f};
  if (p < HW) {
    float P[4];
    paper_rgba(s, z, P);
    int covered = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) covered += s.winner[(size_t)k * HW + p] >= 0;
    const float cv = 0.25f * (float)covered, u = 1.f - cv, A = cv + u * P[3], ia = 1.f - P[3];
    float G = 0.f;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float g = g_img[(size_t)q * HW + p];
      G += g * (-P[q] * A + u * P[q] * ia - ia);
      gp[q] = g * u * A;
      gp[3] += g * (u * u * P[q] - u);
    }
    s.pix_g[p] = G;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) red[q][threadIdx.x] = gp[q];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
#pragma unroll
      for (int q = 0; q < 4; ++q) red[q][threadIdx.x] += red[q][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 4) s.paper_part[(size_t)blockIdx.x * 4 + threadIdx.x] = red[threadIdx.x][0];
}

// the parameter interval (lo, hi) where the line X(s) = o + s d lies strictly inside capsule c (radius r).  A capsule is
// convex, so the union of the intervals of its two end disks and its body is one interval.
__device__ bool line_in_capsule(float ox, float oy, float dx, float dy, float4 c, float r, float& lo, float& hi) {
  lo = INFINITY;
  hi = -INFINITY;
  const float A = dx * dx + dy * dy;
  const float cx[2] = {c.x, c.z}, cy[2] = {c.y, c.w};
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float qx = ox - cx[e], qy = oy - cy[e];
    const float B = qx * dx + qy * dy, C = qx * qx + qy * qy - r * r, disc = B * B - A * C;
    if (disc > 0.f) {
      const float sq = sqrtf(disc);
      lo = fminf(lo, (-B - sq) / A);
      hi = fmaxf(hi, (-B + sq) / A);
    }
  }
  const float ex = c.z - c.x, ey = c.w - c.y, ll = ex * ex + ey * ey;
  if (ll > 0.f) {
    const float len = sqrtf(ll), mx = -ey / len, my = ex / len, qx = ox - c.x, qy = oy - c.y;
    // 0 < (X - a).e < |e|^2 and |(X - a).m| < r, each linear in s
    float l = -INFINITY, h = INFINITY;
    auto clip = [&](float a0, float a1, float vlo, float vhi) {  // vlo < a0 + a1 s < vhi
      if (a1 == 0.f) {
        if (!(a0 > vlo && a0 < vhi)) { l = INFINITY; h = -INFINITY; }
      } else {
        float s0 = (vlo - a0) / a1, s1 = (vhi - a0) / a1;
        if (a1 < 0.f) { const float tmp = s0; s0 = s1; s1 = tmp; }
        l = fmaxf(l, s0);
        h = fminf(h, s1);
      }
    };
    clip(qx * ex + qy * ey, dx * ex + dy * ey, 0.f, ll);
    clip(qx * mx + qy * my, dx * mx + dy * my, -r, r);
    if (l < h) {
      lo = fminf(lo, l);
      hi = fmaxf(hi, h);
    }
  }
  return lo < hi;
}

// integrals of 1 and s over the part of [s0, s1] of the line o + s d that no capsule of the tile list [b, e) other than
// `self` covers: walk the uncovered gaps in order
__device__ void visible_moments(const StrokeScene& s, const float* __restrict__ z, int b, int e, int self, float ox,
                                float oy, float dx, float dy, float s0, float s1, float& i0, float& i1) {
  i0 = i1 = 0.f;
  float cur = s0;
  for (int guard = 0; guard <= 2 * (e - b) + 1 && cur < s1; ++guard) {
    for (bool moved = true; moved;) {  // move cur past every interval that contains it
      moved = false;
      for (int i = b; i < e; ++i) {
        const int c = s.tile_list[i];
        float lo, hi;
        if (c != self && line_in_capsule(ox, oy, dx, dy, s.caps[c], cap_width(s, z, c), lo, hi) && lo <= cur && hi > cur) {
          cur = hi;
          moved = true;
        }
      }
    }
    if (cur >= s1) break;
    float nx = s1;
    for (int i = b; i < e; ++i) {
      const int c = s.tile_list[i];
      float lo, hi;
      if (c != self && line_in_capsule(ox, oy, dx, dy, s.caps[c], cap_width(s, z, c), lo, hi) && lo > cur && lo < nx) nx = lo;
    }
    i0 += nx - cur;
    i1 += 0.5f * (nx - cur) * (nx + cur);
    cur = nx;
  }
}

// one straight side of capsule c: X(s) = a + sig w n + s (b - a), outward normal sig n, v_n = ((1 - s) da + s db).sig n + dw.
// The side is clipped to the canvas and walked pixel by pixel; G is constant per pixel and v_n linear, so each visible
// piece integrates exactly.
__device__ void side_term(const StrokeScene& s, const float* __restrict__ z, int c, float4 cp, float w, float sig,
                          float acc[CAP_GRAD]) {
  const float ex = cp.z - cp.x, ey = cp.w - cp.y, len = sqrtf(ex * ex + ey * ey);
  if (!(len > 0.f)) return;
  const float nx = -ey / len * sig, ny = ex / len * sig;
  const float ox = cp.x + w * nx, oy = cp.y + w * ny;
  // Liang-Barsky against [0, W] x [0, H]
  float c0 = 0.f, c1 = 1.f;
  const float pd[4] = {-ex, ex, -ey, ey}, qd[4] = {ox, (float)s.W - ox, oy, (float)s.H - oy};
  for (int q = 0; q < 4; ++q) {
    if (pd[q] == 0.f) {
      if (qd[q] < 0.f) return;
    } else {
      const float r = qd[q] / pd[q];
      if (pd[q] < 0.f) c0 = fmaxf(c0, r);
      else c1 = fminf(c1, r);
    }
  }
  if (!(c0 < c1)) return;
  // grid walk (Amanatides-Woo) from c0 to c1
  const float s_in = c0 + 1e-4f * (c1 - c0);
  int ix = min(max((int)floorf(ox + s_in * ex), 0), s.W - 1), iy = min(max((int)floorf(oy + s_in * ey), 0), s.H - 1);
  const int stx = ex > 0.f ? 1 : -1, sty = ey > 0.f ? 1 : -1;
  float tmx = ex != 0.f ? ((float)(ix + (ex > 0.f)) - ox) / ex : INFINITY;
  float tmy = ey != 0.f ? ((float)(iy + (ey > 0.f)) - oy) / ey : INFINITY;
  const float tdx = ex != 0.f ? 1.f / fabsf(ex) : INFINITY, tdy = ey != 0.f ? 1.f / fabsf(ey) : INFINITY;
  float cur = c0;
  for (int guard = 0; guard < s.W + s.H + 4 && cur < c1; ++guard) {
    const float nxt = fminf(fminf(tmx, tmy), c1);
    if (nxt > cur && ix >= 0 && ix < s.W && iy >= 0 && iy < s.H) {
      const float G = s.pix_g[iy * s.W + ix];
      if (G != 0.f) {
        const int t = (iy / RASTER_TILE) * s.tiles_x + ix / RASTER_TILE;
        float i0, i1;
        visible_moments(s, z, s.tile_start[t], s.tile_start[t + 1], c, ox, oy, ex, ey, cur, nxt, i0, i1);
        const float fa = G * len * (i0 - i1), fb = G * len * i1;
        acc[0] += fa * nx;
        acc[1] += fa * ny;
        acc[2] += fb * nx;
        acc[3] += fb * ny;
        acc[4] += G * len * i0;
      }
    }
    cur = fmaxf(cur, nxt);
    if (tmx <= tmy) {
      ix += stx;
      tmx += tdx;
    } else {
      iy += sty;
      tmy += tdy;
    }
  }
}

// node q of the circle of radius w around vertex v: visible when the direction u passes the cone test (the part of the
// circle that is boundary of this capsule and, at a joint, of the previous one) and no other capsule strictly covers it
__device__ void arc_node(const StrokeScene& s, const float* __restrict__ z, int self, int prev, float vx, float vy,
                         float w, float e_prev_x, float e_prev_y, float e_x, float e_y, int q, bool end_cap,
                         float acc[CAP_GRAD]) {
  float uy, ux;
  sincospif(2.f * ((float)q + 0.5f) / STROKE_ARC_NODES, &uy, &ux);
  const float de = ux * e_x + uy * e_y;
  if (end_cap ? de < 0.f : (de > 0.f || ux * e_prev_x + uy * e_prev_y < 0.f)) return;
  const float px = vx + w * ux, py = vy + w * uy;
  if (!(px >= 0.f && px < (float)s.W && py >= 0.f && py < (float)s.H)) return;
  const int ix = min((int)px, s.W - 1), iy = min((int)py, s.H - 1);
  const float G = s.pix_g[iy * s.W + ix];
  if (G == 0.f) return;
  const int t = (iy / RASTER_TILE) * s.tiles_x + ix / RASTER_TILE;
  for (int i = s.tile_start[t]; i < s.tile_start[t + 1]; ++i) {
    const int c = s.tile_list[i];
    if (c == self || c == prev) continue;
    const float r = cap_width(s, z, c);
    if (seg_dist2(px, py, s.caps[c]) < r * r) return;
  }
  const float f = G * w * (2.f * 3.14159265358979f / STROKE_ARC_NODES);
  const int o = end_cap ? 2 : 0;
  acc[o] += f * ux;
  acc[o + 1] += f * uy;
  acc[4] += f;
}

__device__ __forceinline__ void unit_dir(float4 c, float& x, float& y) {
  const float ex = c.z - c.x, ey = c.w - c.y, len = sqrtf(ex * ex + ey * ey);
  x = len > 0.f ? ex / len : 0.f;
  y = len > 0.f ? ey / len : 0.f;
}

// one warp per capsule: both sides, the circle at its start vertex (a cap, or the joint with the previous chord) and, for
// a path's last chord, the cap at its end; the lanes' partial sums are combined by a fixed butterfly and one lane writes
__global__ void __launch_bounds__(256) stroke_cap_kernel(StrokeScene s, const float* __restrict__ z) {
  pdl_launch_dependents();
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (c >= s.n_caps) return;
  pdl_wait();
  const int per_path = s.n_segments * STROKE_CHORDS;
  const bool first = c % per_path == 0, last = (c + 1) % per_path == 0;
  const float4 cp = s.caps[c];
  const float w = cap_width(s, z, c);
  float ex, ey, px = 0.f, py = 0.f;
  unit_dir(cp, ex, ey);
  if (!first) unit_dir(s.caps[c - 1], px, py);
  float acc[CAP_GRAD] = {0.f, 0.f, 0.f, 0.f, 0.f};
  const int n_items = 2 + STROKE_ARC_NODES * (last ? 2 : 1);
  for (int it = lane; it < n_items; it += 32) {
    if (it < 2) {
      side_term(s, z, c, cp, w, it == 0 ? 1.f : -1.f, acc);
    } else if (it < 2 + STROKE_ARC_NODES) {
      arc_node(s, z, c, first ? -1 : c - 1, cp.x, cp.y, w, px, py, ex, ey, it - 2, false, acc);
    } else {
      arc_node(s, z, c, -1, cp.z, cp.w, w, 0.f, 0.f, ex, ey, it - 2 - STROKE_ARC_NODES, true, acc);
    }
  }
#pragma unroll
  for (int q = 0; q < CAP_GRAD; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < CAP_GRAD; ++q) s.cap_grad[(size_t)c * CAP_GRAD + q] = acc[q];
}

// z_grad: control point q of path k folds the chord endpoints that are Bernstein combinations of it (fixed order:
// segment, then chord); a width sums its path's capsules; the paper colour sums the per-block partials
__global__ void __launch_bounds__(256) stroke_fold_kernel(StrokeScene s, int paper_blocks, float inv_scale,
                                                          float* __restrict__ z_grad) {
  pdl_launch_dependents();
  const int e = blockIdx.x * blockDim.x + threadIdx.x, L = s.n_segments, per_path = L * STROKE_CHORDS;
  const int n_pts = s.width_offset;
  if (e >= n_pts + s.n_paths + 4) return;
  pdl_wait();
  float sum = 0.f;
  if (e < n_pts) {
    const int per = (3 * L + 1) * 2, k = e / per, q = (e % per) >> 1, d = e & 1;
    for (int j = max(0, (q - 1) / 3); j <= min(L - 1, q / 3); ++j) {
      const int m = q - 3 * j;
      if (m < 0 || m > 3) continue;
      for (int i = 0; i < STROKE_CHORDS; ++i) {
        const float* g = s.cap_grad + ((size_t)(k * L + j) * STROKE_CHORDS + i) * CAP_GRAD;
        sum += bernstein(m, (float)i / STROKE_CHORDS) * g[d] + bernstein(m, (float)(i + 1) / STROKE_CHORDS) * g[2 + d];
      }
    }
  } else if (e < n_pts + s.n_paths) {
    const int k = e - n_pts;
    for (int c = k * per_path; c < (k + 1) * per_path; ++c) sum += s.cap_grad[(size_t)c * CAP_GRAD + 4];
  } else if (s.paper_trainable) {
    const int q = e - n_pts - s.n_paths;
    for (int b = 0; b < paper_blocks; ++b) sum += s.paper_part[(size_t)b * 4 + q];
  }
  z_grad[e] = sum * inv_scale;
}

}  // namespace

void stroke_flatten(const StrokeScene& s, const float* z, cudaStream_t st) {
  launch_pdl(stroke_flatten_kernel, dim3((s.n_caps + 255) / 256), dim3(256), 0, st, s, z);
}

void stroke_bin(const StrokeScene& s, cudaStream_t st) {
  const int tiles = s.tiles_x * s.tiles_y;
  launch_pdl(stroke_bin_count_kernel, dim3(tiles), dim3(256), 0, st, s);
  launch_pdl(stroke_bin_scan_kernel, dim3(1), dim3(1024), 0, st, s);
  launch_pdl(stroke_bin_fill_kernel, dim3(tiles), dim3(256), 0, st, s);
}

void stroke_raster_forward(const StrokeScene& s, const float* z, uint64_t seed, int iter, float* img, cudaStream_t st) {
  launch_pdl(stroke_fwd_kernel, dim3((s.H * s.W + 255) / 256), dim3(256), 0, st, s, z, seed, iter, img);
}

int stroke_paper_blocks(int H, int W) { return (H * W + 255) / 256; }

void stroke_raster_backward(const StrokeScene& s, const float* z, const float* g_img, float inv_scale, float* z_grad,
                            cudaStream_t st) {
  const int blocks = stroke_paper_blocks(s.H, s.W);
  launch_pdl(stroke_pixel_kernel, dim3(blocks), dim3(256), 0, st, s, z, g_img);
  launch_pdl(stroke_cap_kernel, dim3((s.n_caps + 7) / 8), dim3(256), 0, st, s, z);
  const int n = s.width_offset + s.n_paths + 4;
  launch_pdl(stroke_fold_kernel, dim3((n + 255) / 256), dim3(256), 0, st, s, blocks, inv_scale, z_grad);
}

}  // namespace pxr
