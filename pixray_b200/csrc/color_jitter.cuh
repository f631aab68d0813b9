// K.ColorJitter(hue=0.1, saturation=0.1, p=0.8), the last stage of both augmentation stacks of MakeCutouts
// (pixray.py:416, 436), per pixel.  kornia 0.6.2 is an un-vendored dependency of the reference (requirements.txt);
// this restates its published algorithm:
//   ColorJitter.apply_transform : four transforms applied in the order `params["order"]` (a randperm(4)):
//        0 adjust_brightness(x, factor - 1) = clamp(x + (factor - 1), 0, 1)   factor == 1 with brightness=0
//        1 adjust_contrast(x, factor)       = clamp(x * factor, 0, 1)         factor == 1 with contrast=0
//        2 adjust_saturation(x, f)          = hsv_to_rgb(h, clamp(s * f, 0, 1), v)
//        3 adjust_hue(x, f * 2pi)           = hsv_to_rgb(fmod(h + f * 2pi, 2pi), s, v)
//   rgb_to_hsv (eps 1e-8): v = max, s = (max - min) / (max + eps), h from the arg-max channel, in radians;
//   hsv_to_rgb: sector = floor(6h) mod 6, the usual (v, q, p, t) table.
// One templated body serves the forward (T = float) and the backward: with T = Dual3 (value + the three partials
// d/d{r,g,b}) it yields the 3x3 Jacobian of the whole chain, so the gradient is by construction the derivative of
// the forward that was executed (max / min route to the first arg-max / arg-min channel as torch.max(dim) does on
// ties, floor and the mods have zero / unit derivative, clamp passes the gradient on the closed interval).
// Host-callable so the CPU suite can check the arithmetic against the oracle without a GPU (test_hooks.cu).
//
// VALUES are computed with individually rounded IEEE operations everywhere (cj_add / cj_sub / cj_mul / cj_div: __f*_rn
// on the device, which the compiler neither contracts into FMAs nor replaces by the approximate division; plain
// operators on the host, where x86-64 code has no FMA contraction).  That makes the device body bit-identical to the
// host body and to torch's elementwise arithmetic, which matters because the map is continuous but its JACOBIAN is
// piecewise, and clamped images are full of colours that sit EXACTLY on a piece boundary: two saturated channels
// (1, 1, x) have a hue of exactly 60 degrees, i.e. exactly on the sector boundary of hsv_to_rgb, and whether
// floor(6 h) comes out as 0 or 1 there is decided by the last bit of h / 2pi.  Round 1 used __fdividef and let the
// compiler contract: forward values agreed to 2e-6, but ~2e-4 of the pixels of a clamped image took the other
// one-sided Jacobian, which showed up as a 2.5e-2 error of d loss / d image.
// Derivative parts carry no such constraint.
#pragma once
#include <cmath>
#include <cuda_runtime.h>

namespace pxr {

struct Dual3 {
  float v;
  float d[3];
};

#define PXR_HD __host__ __device__ __forceinline__
#ifdef __CUDA_ARCH__
#define PXR_UNROLL _Pragma("unroll")
#define PXR_NOUNROLL _Pragma("unroll 1")
#else
#define PXR_UNROLL
#define PXR_NOUNROLL
#endif

// ---- exactly rounded scalar operations (see the header comment)
PXR_HD float cj_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
PXR_HD float cj_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
PXR_HD float cj_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
PXR_HD float cj_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
PXR_HD float cj_val(float x) { return x; }
PXR_HD float cj_val(const Dual3& x) { return x.v; }
PXR_HD float cj_const(float, float c) { return c; }
PXR_HD Dual3 cj_const(const Dual3&, float c) { return Dual3{c, {0.f, 0.f, 0.f}}; }

// ---- the same operations on dual numbers: the value through the exact operations, the partials freely
PXR_HD Dual3 cj_add(const Dual3& a, const Dual3& b) { return Dual3{cj_add(a.v, b.v), {a.d[0] + b.d[0], a.d[1] + b.d[1], a.d[2] + b.d[2]}}; }
PXR_HD Dual3 cj_sub(const Dual3& a, const Dual3& b) { return Dual3{cj_sub(a.v, b.v), {a.d[0] - b.d[0], a.d[1] - b.d[1], a.d[2] - b.d[2]}}; }
PXR_HD Dual3 cj_mul(const Dual3& a, const Dual3& b) {
  return Dual3{cj_mul(a.v, b.v), {a.d[0] * b.v + a.v * b.d[0], a.d[1] * b.v + a.v * b.d[1], a.d[2] * b.v + a.v * b.d[2]}};
}
PXR_HD Dual3 cj_div(const Dual3& a, const Dual3& b) {
  const float r = 1.f / b.v, q = a.v * r;
  return Dual3{cj_div(a.v, b.v), {(a.d[0] - q * b.d[0]) * r, (a.d[1] - q * b.d[1]) * r, (a.d[2] - q * b.d[2]) * r}};
}
PXR_HD Dual3 cj_div(const Dual3& a, float b) {
  const float r = 1.f / b;
  return Dual3{cj_div(a.v, b), {a.d[0] * r, a.d[1] * r, a.d[2] * r}};
}
PXR_HD Dual3 cj_add(const Dual3& a, float b) { return Dual3{cj_add(a.v, b), {a.d[0], a.d[1], a.d[2]}}; }
PXR_HD Dual3 cj_mul(const Dual3& a, float b) { return Dual3{cj_mul(a.v, b), {a.d[0] * b, a.d[1] * b, a.d[2] * b}}; }
PXR_HD Dual3 cj_rsub(float a, const Dual3& b) { return Dual3{cj_sub(a, b.v), {-b.d[0], -b.d[1], -b.d[2]}}; }  // a - b
PXR_HD float cj_rsub(float a, float b) { return cj_sub(a, b); }

// replace the value, keep the partials (x mod m, fmod: derivative 1) / drop them (floor: derivative 0)
PXR_HD float cj_with_value(float, float v) { return v; }
PXR_HD Dual3 cj_with_value(const Dual3& x, float v) { return Dual3{v, {x.d[0], x.d[1], x.d[2]}}; }

// torch.remainder(a, b) (the `%` of the reference: fmod, then + b when the sign differs from b's) and torch.fmod(a, b)
// for b > 0 and a in (-b, 2b) -- the only range this chain produces (h/6 in (-1/6, 1), 6h in (-3, 6], h + shift in
// (-pi, 3pi)): one exact subtraction / the same single rounded addition fmodf's result would see, without fmodf's loop.
PXR_HD float cj_pymod(float a, float b) {
  if (a >= b) return cj_sub(a, b);
  if (a < 0.f) return cj_add(a, b);
  return a;
}
PXR_HD float cj_fmod(float a, float b) { return a >= b ? cj_sub(a, b) : a; }
template <class T>
PXR_HD T cj_clamp01(const T& x) {
  const float v = cj_val(x);
  if (v < 0.f) return cj_const(x, 0.f);
  if (v > 1.f) return cj_const(x, 1.f);
  return x;
}

constexpr float CJ_TWO_PI = 6.283185307179586f;

template <class T>
PXR_HD void cj_rgb_to_hsv(const T c[3], T& h, T& s, T& v) {
  int imax = 0, imin = 0;  // first arg-max / arg-min on ties
  {
    const float v0 = cj_val(c[0]), v1 = cj_val(c[1]), v2 = cj_val(c[2]);
    float hi = v0, lo = v0;
    if (v1 > hi) { hi = v1; imax = 1; }
    if (v2 > hi) { imax = 2; }
    if (v1 < lo) { lo = v1; imin = 1; }
    if (v2 < lo) { imin = 2; }
  }
  const T mx = imax == 0 ? c[0] : (imax == 1 ? c[1] : c[2]);
  const T mn = imin == 0 ? c[0] : (imin == 1 ? c[1] : c[2]);
  const T delta = cj_sub(mx, mn);
  v = mx;
  s = cj_div(delta, cj_add(mx, 1e-8f));
  const T dc = (cj_val(delta) == 0.f) ? cj_const(delta, 1.f) : delta;
  const T rc = cj_sub(mx, c[0]), gc = cj_sub(mx, c[1]), bc = cj_sub(mx, c[2]);
  T hh;
  if (imax == 0) hh = cj_sub(bc, gc);
  else if (imax == 1) hh = cj_add(cj_sub(rc, bc), cj_mul(dc, 2.0f));
  else hh = cj_add(cj_sub(gc, rc), cj_mul(dc, 4.0f));
  hh = cj_div(hh, dc);
  hh = cj_div(hh, 6.0f);
  hh = cj_with_value(hh, cj_pymod(cj_val(hh), 1.0f));
  h = cj_mul(hh, CJ_TWO_PI);
}

template <class T>
PXR_HD void cj_hsv_to_rgb(const T& h_rad, const T& s, const T& v, T c[3]) {
  const T h6 = cj_mul(cj_div(h_rad, CJ_TWO_PI), 6.0f);
  const float hi_f = cj_pymod(floorf(cj_val(h6)), 6.0f);
  const T f = cj_with_value(h6, cj_sub(cj_pymod(cj_val(h6), 6.0f), hi_f));
  const T p = cj_mul(v, cj_rsub(1.0f, s));
  const T q = cj_mul(v, cj_rsub(1.0f, cj_mul(f, s)));
  const T t = cj_mul(v, cj_rsub(1.0f, cj_mul(cj_rsub(1.0f, f), s)));
  const int hi = (int)hi_f;
  switch (hi) {
    case 0: c[0] = v; c[1] = t; c[2] = p; break;
    case 1: c[0] = q; c[1] = v; c[2] = p; break;
    case 2: c[0] = p; c[1] = v; c[2] = t; break;
    case 3: c[0] = p; c[1] = q; c[2] = v; break;
    case 4: c[0] = t; c[1] = p; c[2] = v; break;
    default: c[0] = v; c[1] = p; c[2] = q; break;
  }
}

// code: 0 = this cutout is not jittered (Bernoulli(p) miss); else 256 + o0 + 4*o1 + 16*o2 + 64*o3, o_k = the
// transform applied k-th.  sat = saturation_factor, hue = hue_factor (kornia's unit: fraction of a turn).
template <class T>
PXR_HD void cj_apply(T c[3], int code, float sat, float hue) {
  if (code == 0) return;
  const float hue_rad = cj_mul(cj_mul(hue, 2.f), 3.14159274101257324f);
PXR_NOUNROLL
  for (int k = 0; k < 4; ++k) {
    const int op = (code >> (2 * k)) & 3;
    if (op < 2) {
PXR_UNROLL
      for (int i = 0; i < 3; ++i) c[i] = cj_clamp01(c[i]);
    } else {
      T h, s, v;
      cj_rgb_to_hsv(c, h, s, v);
      if (op == 2) {
        s = cj_clamp01(cj_mul(s, sat));
      } else {
        const T hs = cj_add(h, hue_rad);
        h = cj_with_value(hs, cj_fmod(cj_val(hs), CJ_TWO_PI));
      }
      cj_hsv_to_rgb(h, s, v, c);
    }
  }
}

// g_in = J^T g_out at the pre-jitter colour `rgb`
PXR_HD void cj_vjp(const float rgb[3], int code, float sat, float hue, const float g_out[3], float g_in[3]) {
  if (code == 0) {
    g_in[0] = g_out[0];
    g_in[1] = g_out[1];
    g_in[2] = g_out[2];
    return;
  }
  Dual3 c[3];
PXR_UNROLL
  for (int i = 0; i < 3; ++i) c[i] = Dual3{rgb[i], {i == 0 ? 1.f : 0.f, i == 1 ? 1.f : 0.f, i == 2 ? 1.f : 0.f}};
  cj_apply(c, code, sat, hue);
PXR_UNROLL
  for (int i = 0; i < 3; ++i) g_in[i] = c[0].d[i] * g_out[0] + c[1].d[i] * g_out[1] + c[2].d[i] * g_out[2];
}

}  // namespace pxr
