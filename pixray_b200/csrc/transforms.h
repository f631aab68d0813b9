// Host side of MakeCutouts' augmentation sampling (SURVEY.md Appendix A; call sites pixray.py:411-437):
// what kornia's RandomPerspective / RandomResizedCrop / RandomAffine draw per cutout, composed into ONE 3x3
// "dst_pix <- src_pix" homography per cutout -- exactly what MakeCutouts.transforms caches (pixray.py:498).
// The distributions are restated, not kornia's RNG stream (the reference mixes three RNG sources per iteration,
// so its stream is not reproducible anyway); draws come from Philox keyed by (seed, iter, GLOBAL cutout index).
#pragma once
#include "philox.cuh"
#include <cmath>
#include <cstdint>
#include <utility>

namespace pxr {

inline bool invert3x3(const double m[9], double inv[9]) {
  const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double det = a * A + b * B + c * C;
  if (std::fabs(det) < 1e-30) return false;
  const double r = 1.0 / det;
  inv[0] = A * r;
  inv[1] = -(b * i - c * h) * r;
  inv[2] = (b * f - c * e) * r;
  inv[3] = B * r;
  inv[4] = (a * i - c * g) * r;
  inv[5] = -(a * f - c * d) * r;
  inv[6] = C * r;
  inv[7] = -(a * h - b * g) * r;
  inv[8] = (a * e - b * d) * r;
  return true;
}

inline void matmul3(const double a[9], const double b[9], double o[9]) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) o[r * 3 + c] = a[r * 3] * b[c] + a[r * 3 + 1] * b[3 + c] + a[r * 3 + 2] * b[6 + c];
}

// kornia get_perspective_transform: homography taking the 4 src points to the 4 dst points (8x8 linear solve)
inline bool perspective_from_points(const double src[4][2], const double dst[4][2], double H[9]) {
  double A[8][9];
  for (int k = 0; k < 4; ++k) {
    const double x = src[k][0], y = src[k][1], u = dst[k][0], v = dst[k][1];
    double r0[9] = {x, y, 1, 0, 0, 0, -u * x, -u * y, u};
    double r1[9] = {0, 0, 0, x, y, 1, -v * x, -v * y, v};
    for (int j = 0; j < 9; ++j) {
      A[2 * k][j] = r0[j];
      A[2 * k + 1][j] = r1[j];
    }
  }
  for (int c = 0; c < 8; ++c) {
    int piv = c;
    for (int r = c + 1; r < 8; ++r)
      if (std::fabs(A[r][c]) > std::fabs(A[piv][c])) piv = r;
    if (std::fabs(A[piv][c]) < 1e-14) return false;
    if (piv != c)
      for (int j = 0; j < 9; ++j) std::swap(A[piv][j], A[c][j]);
    for (int r = 0; r < 8; ++r) {
      if (r == c) continue;
      const double f = A[r][c] / A[c][c];
      for (int j = c; j < 9; ++j) A[r][j] -= f * A[c][j];
    }
  }
  for (int k = 0; k < 8; ++k) H[k] = A[k][8] / A[k][k];
  H[8] = 1.0;
  return true;
}

// Philox stream words of the draws of cutout set s: 0 noise, 1 noise factors, 2 homographies, 4 / 5 ColorJitter, each
// plus cut_rng_stream(s).  Set 0 adds nothing; the other sets get words of their own, above the shared fill (3) and the
// filters' shifts (6).  The image-prompt and spot passes move the iteration word instead (engine.cu), so no two collide.
inline uint32_t cut_rng_stream(int set) { return 16u * (uint32_t)set; }

struct CutRng {
  uint64_t seed;
  uint32_t iter;
  uint64_t base;
  uint32_t stream = 0;  // cut_rng_stream of the set
  uint32_t k = 0;
  double uni() { return (double)philox_uniform(seed, iter, 2u + stream, base + (k++)); }        // (0, 1]
  double uni(double lo, double hi) { return lo + (hi - lo) * uni(); }
};

// RandomPerspective(distortion_scale, p=0.7): corners move inward by U(0,1) * scale * side/2 per axis
inline void sample_perspective(CutRng& r, int size, double distortion, double p, double H[9]) {
  const bool apply = r.uni() <= p;
  const double w1 = size - 1.0, f = distortion * size / 2.0;
  const double start[4][2] = {{0, 0}, {w1, 0}, {w1, w1}, {0, w1}};
  const double sgn[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  double end[4][2];
  for (int k = 0; k < 4; ++k)
    for (int a = 0; a < 2; ++a) end[k][a] = start[k][a] + f * r.uni() * sgn[k][a];  // draws happen regardless of p
  if (!apply || !perspective_from_points(start, end, H)) {
    for (int i = 0; i < 9; ++i) H[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
}

// RandomResizedCrop(size, scale=(0.25,0.95), ratio=(0.85,1.2), cropping_mode='resample')
inline void sample_resized_crop(CutRng& r, int size, double H[9]) {
  double w = size, h = size;
  for (int attempt = 0; attempt < 10; ++attempt) {
    const double area = r.uni(0.25, 0.95) * size * size;
    const double ratio = std::exp(r.uni(std::log(0.85), std::log(1.2)));
    const double cw = std::round(std::sqrt(area * ratio)), ch = std::round(std::sqrt(area / ratio));
    if (cw > 0 && cw <= size && ch > 0 && ch <= size) {
      w = cw;
      h = ch;
      break;
    }
  }
  const double x0 = std::floor(r.uni() * (size - w + 1) * 0.999999), y0 = std::floor(r.uni() * (size - h + 1) * 0.999999);
  const double src[4][2] = {{x0, y0}, {x0 + w - 1, y0}, {x0 + w - 1, y0 + h - 1}, {x0, y0 + h - 1}};
  const double s1 = size - 1.0;
  const double dst[4][2] = {{0, 0}, {s1, 0}, {s1, s1}, {0, s1}};
  if (!perspective_from_points(src, dst, H))
    for (int i = 0; i < 9; ++i) H[i] = (i % 4 == 0) ? 1.0 : 0.0;
}

// MyRandomAffine(degrees=0, translate=(n_t,n_t), scale=(n_s,n_s)) about the image centre (square canvas)
inline void sample_affine(CutRng& r, int size, double n_s, double n_t, double H[9]) {
  const double c = size / 2.0 - 0.5;
  const double tx = r.uni(-n_t * size, n_t * size), ty = r.uni(-n_t * size, n_t * size);
  const double M[9] = {n_s, 0, (1 - n_s) * c + tx, 0, n_s, (1 - n_s) * c + ty, 0, 0, 1};
  for (int i = 0; i < 9; ++i) H[i] = M[i];
}

// ---- non-square canvases (global_aspect_width != 1): the warps sample from an h x w stretch of the pooled image
inline void source_size(int cut_size, double aspect, int& h, int& w) {  // kornia rescale truncates: int(size * factor)
  h = w = cut_size;
  if (aspect > 1.0) w = (int)(cut_size * aspect);
  else if (aspect < 1.0) h = (int)(cut_size * (1.0 / aspect));
}
inline void identity3(double H[9]) {
  for (int i = 0; i < 9; ++i) H[i] = (i % 4 == 0) ? 1.0 : 0.0;
}
inline void sample_perspective_hw(CutRng& r, int h, int w, double distortion, double p, double H[9]) {
  const bool apply = r.uni() <= p;
  const double fx = distortion * w / 2.0, fy = distortion * h / 2.0;
  const double start[4][2] = {{0, 0}, {w - 1.0, 0}, {w - 1.0, h - 1.0}, {0, h - 1.0}};
  const double sgn[4][2] = {{1, 1}, {-1, 1}, {-1, -1}, {1, -1}};
  double end[4][2];
  for (int k = 0; k < 4; ++k) {
    end[k][0] = start[k][0] + fx * r.uni() * sgn[k][0];
    end[k][1] = start[k][1] + fy * r.uni() * sgn[k][1];
  }
  if (!apply || !perspective_from_points(start, end, H)) identity3(H);
}
inline void sample_resized_crop_hw(CutRng& r, int h, int w, int out, double H[9]) {
  double cw = -1, ch = -1;
  for (int attempt = 0; attempt < 10; ++attempt) {
    const double area = r.uni(0.25, 0.95) * h * w;
    const double ratio = std::exp(r.uni(std::log(0.85), std::log(1.2)));
    const double tw = std::round(std::sqrt(area * ratio)), th = std::round(std::sqrt(area / ratio));
    if (tw > 0 && tw <= w && th > 0 && th <= h) {
      cw = tw;
      ch = th;
      break;
    }
  }
  if (cw < 0) {  // the fallback of the ten-tries loop: whole height or width with the ratio clamped
    const double in_ratio = (double)w / h;
    if (in_ratio < 0.85) {
      cw = w;
      ch = std::round(w / 0.85);
    } else if (in_ratio > 1.2) {
      ch = h;
      cw = std::round(h * 1.2);
    } else {
      cw = w;
      ch = h;
    }
  }
  const double x0 = std::floor(r.uni() * (w - cw + 1) * 0.999999), y0 = std::floor(r.uni() * (h - ch + 1) * 0.999999);
  const double src[4][2] = {{x0, y0}, {x0 + cw - 1, y0}, {x0 + cw - 1, y0 + ch - 1}, {x0, y0 + ch - 1}};
  const double s1 = out - 1.0;
  const double dst[4][2] = {{0, 0}, {s1, 0}, {s1, s1}, {0, s1}};
  if (!perspective_from_points(src, dst, H)) identity3(H);
}
// MyRandomAffine(degrees=0, translate=(tfx, tfy), scale=(lo, hi)) about the centre of an h x w image (pixray.py:424-431)
inline void sample_affine_hw(CutRng& r, int h, int w, double lo, double hi, double tfx, double tfy, double H[9]) {
  const double s = r.uni(lo, hi);
  const double cx = w / 2.0 - 0.5, cy = h / 2.0 - 0.5;
  const double tx = tfx > 0 ? r.uni(-tfx * w, tfx * w) : 0.0, ty = tfy > 0 ? r.uni(-tfy * h, tfy * h) : 0.0;
  const double M[9] = {s, 0, (1 - s) * cx + tx, 0, s, (1 - s) * cy + ty, 0, 0, 1};
  for (int i = 0; i < 9; ++i) H[i] = M[i];
}

// out: [cutn, 9] row-major dst<-src homographies; zoom group first (global index < int(0.6 * cutn), pixray.py:407)
inline void sample_cutout_transforms(uint64_t seed, int iter, int cutn, int cut_size, float* out, double aspect = 1.0,
                                     int src_h = 0, int src_w = 0, uint32_t stream = 0) {
  const int cutn_zoom = (int)(0.6 * cutn);
  int sh, sw;
  source_size(cut_size, aspect, sh, sw);
  if (src_h > 0 && src_w > 0) {
    sh = src_h;
    sw = src_w;
  }
  for (int n = 0; n < cutn; ++n) {
    CutRng r{seed, (uint32_t)iter, (uint64_t)n * 64, stream};
    double A[9], B[9], H[9];
    if (aspect != 1.0) {
      if (n < cutn_zoom) {
        sample_perspective_hw(r, sh, sw, 0.40, 0.7, A);
        sample_resized_crop_hw(r, sh, sw, cut_size, B);
        matmul3(B, A, H);
      } else {
        const double n_s = aspect > 1.0 ? 1.0 / aspect : aspect, n_t = (1 - n_s) / 2;
        if (aspect > 1.0) sample_affine_hw(r, sh, sw, 0.9 * n_s, n_s, 0.0, n_t, A);
        else sample_affine_hw(r, sh, sw, 0.9 * n_s, n_s, n_t, 0.0, A);
        // K.CenterCrop(size=cut_size): the central box, a translation
        const double Cc[9] = {1, 0, -(double)((sw - cut_size) / 2), 0, 1, -(double)((sh - cut_size) / 2), 0, 0, 1};
        double CA[9];
        matmul3(Cc, A, CA);
        sample_perspective(r, cut_size, 0.20, 0.7, B);
        matmul3(B, CA, H);
      }
      for (int i = 0; i < 9; ++i) out[(size_t)n * 9 + i] = (float)H[i];
      continue;
    }
    if (n < cutn_zoom) {
      sample_perspective(r, cut_size, 0.40, 0.7, A);  // pixray.py:414
      sample_resized_crop(r, cut_size, B);            // pixray.py:415
      matmul3(B, A, H);
    } else {
      const double n_s = 0.95, n_t = (1 - n_s) / 2;  // pixray.py:420-423
      sample_affine(r, cut_size, n_s, n_t, A);
      sample_perspective(r, cut_size, 0.20, 0.7, B);  // pixray.py:435 (CenterCrop at cs x cs is the identity)
      matmul3(B, A, H);
    }
    for (int i = 0; i < 9; ++i) out[(size_t)n * 9 + i] = (float)H[i];
  }
}

// K.ColorJitter(hue, saturation, p) parameters (pixray.py:416, 436; kornia random_color_jitter_generator):
// per cutout Bernoulli(p), saturation_factor ~ U(1 - s, 1 + s), hue_factor ~ U(-h, h); one randperm(4) application
// order per group (each stack is its own module, called once per iteration).  out: [cutn, 3] rows
// {code, saturation_factor, hue_factor} in the encoding of color_jitter.cuh.
inline void sample_color_jitter(uint64_t seed, int iter, int cutn, float p, float sat, float hue, float* out,
                                uint32_t stream = 0) {
  const int cutn_zoom = (int)(0.6 * cutn);
  int code[2];
  for (int g = 0; g < 2; ++g) {
    int order[4] = {0, 1, 2, 3};
    for (int k = 3; k > 0; --k) {  // Fisher-Yates
      int j = (int)(philox_uniform(seed, (uint32_t)iter, 5u + stream, (uint64_t)g * 4 + k) * 0.999999f * (k + 1));
      std::swap(order[k], order[j]);
    }
    code[g] = 256 + order[0] + 4 * order[1] + 16 * order[2] + 64 * order[3];
  }
  for (int n = 0; n < cutn; ++n) {
    const uint64_t base = (uint64_t)n * 4;
    const bool apply = philox_uniform(seed, (uint32_t)iter, 4u + stream, base) <= p;
    const float u1 = philox_uniform(seed, (uint32_t)iter, 4u + stream, base + 1),
                u2 = philox_uniform(seed, (uint32_t)iter, 4u + stream, base + 2);
    out[n * 3] = apply ? (float)code[n < cutn_zoom ? 0 : 1] : 0.f;
    out[n * 3 + 1] = 1.f - sat + 2.f * sat * u1;
    out[n * 3 + 2] = -hue + 2.f * hue * u2;
  }
}

// global_fill_color = random.random(), once per iteration (pixray.py:1255-1258)
inline float sample_fill(uint64_t seed, int iter) { return philox_uniform(seed, (uint32_t)iter, 3u, 0); }

}  // namespace pxr
