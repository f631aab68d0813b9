// vdiff drawer side kernels (VdiffDrawer.synth, vdiff.py:159-172, over v-diffusion-pytorch's CC12M1Model,
// diffusion/models/cc12m_1.py): everything of the U-Net that is not a convolution, an attention product or a GroupNorm.
// Activations are NHWC fp16 [pixels, C] like the VQGAN decoder's; all kernels are single-pass and HBM/L2-bound with
// 16-byte accesses along the channel axis.
#include "kernels.cuh"

namespace pxr {

namespace {

__device__ __forceinline__ void ld8(const act_t* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ void st8(act_t* p, const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

inline int vgrid(long long n, int block = 256) {
  long long g = (n + block - 1) / block;
  return (int)(g > 148 * 16 ? 148 * 16 : (g < 1 ? 1 : g));
}

// net input: cat([x, timestep_embed planes]) (cc12m_1.py:247-248) as [pixels, 64] fp16: channels 0..2 = x, 3..18 = te, rest 0
__global__ void vd_input_kernel(const float* __restrict__ x, const float* __restrict__ te, int pixels,
                                act_t* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pixels) return;
  float f[8];
#pragma unroll
  for (int v = 0; v < 8; ++v) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = v * 8 + i;
      f[i] = c < 3 ? x[(size_t)c * pixels + p] : (c < 19 ? te[c - 3] : 0.f);
    }
    st8(out + (size_t)p * 64 + v * 8, f);
  }
}

// AvgPool2d(2) (cc12m_1.py:129): [H, W, C] (pixel stride ld_in) -> [H/2, W/2, C]
__global__ void avgpool2x_kernel(const act_t* __restrict__ x, int H, int W, int C, int ld_in, act_t* __restrict__ y) {
  const int vecs = C / 8, Ho = H / 2, Wo = W / 2;
  const long long n = (long long)Ho * Wo * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        float t[8];
        ld8(x + ((size_t)(2 * oy + dy) * W + 2 * ox + dx) * ld_in + vc * 8, t);
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] += t[i];
      }
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] *= 0.25f;
    st8(y + (size_t)p * C + vc * 8, s);
  }
}
// adjoint: gx[2oy+dy, 2ox+dx] (+)= 0.25 gy[oy, ox]; an odd last row / column (floored away by the forward) gets 0
__global__ void avgpool2x_bwd_kernel(const act_t* __restrict__ gy, int H, int W, int C, int accumulate,
                                     act_t* __restrict__ gx) {
  const int vecs = C / 8, Ho = H / 2, Wo = W / 2;
  const long long n = (long long)H * W * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    const int ix = (int)(p % W), iy = (int)(p / W);
    float g[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a[8];
    if ((iy >> 1) < Ho && (ix >> 1) < Wo) ld8(gy + ((size_t)(iy >> 1) * Wo + (ix >> 1)) * C + vc * 8, g);
    if (accumulate) ld8(gx + (size_t)p * C + vc * 8, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = 0.25f * g[i] + (accumulate ? a[i] : 0.f);
    st8(gx + (size_t)p * C + vc * 8, g);
  }
}

// nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False) (cc12m_1.py:130): src = (dst + 0.5) / 2 - 0.5,
// clamped at 0; taps (i0, i0 + 1 clamped) with weights (1 - f, f)
__device__ __forceinline__ void up_taps(int o, int n_in, int& i0, int& i1, float& w1) {
  float src = (o + 0.5f) * 0.5f - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = (int)src;
  i1 = i0 + 1 < n_in ? i0 + 1 : n_in - 1;
  w1 = src - (float)i0;
}
__global__ void bilinear_up2x_kernel(const act_t* __restrict__ x, int H, int W, int C, act_t* __restrict__ y, int ld_out) {
  const int vecs = C / 8, Ho = 2 * H, Wo = 2 * W;
  const long long n = (long long)Ho * Wo * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    const int ox = (int)(p % Wo), oy = (int)(p / Wo);
    int y0, y1, x0, x1;
    float fy, fx;
    up_taps(oy, H, y0, y1, fy);
    up_taps(ox, W, x0, x1, fx);
    float a[8], b[8], c[8], d[8], r[8];
    ld8(x + ((size_t)y0 * W + x0) * C + vc * 8, a);
    ld8(x + ((size_t)y0 * W + x1) * C + vc * 8, b);
    ld8(x + ((size_t)y1 * W + x0) * C + vc * 8, c);
    ld8(x + ((size_t)y1 * W + x1) * C + vc * 8, d);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      r[i] = (1.f - fy) * ((1.f - fx) * a[i] + fx * b[i]) + fy * ((1.f - fx) * c[i] + fx * d[i]);
    st8(y + (size_t)p * ld_out + vc * 8, r);
  }
}
// adjoint in gather form: every input pixel collects from the (at most 4 x 4) outputs whose taps touch it
__global__ void bilinear_up2x_bwd_kernel(const act_t* __restrict__ gy, int H, int W, int C, int ld_gy,
                                         act_t* __restrict__ gx) {
  const int vecs = C / 8, Ho = 2 * H, Wo = 2 * W;
  const long long n = (long long)H * W * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    const int ix = (int)(p % W), iy = (int)(p / W);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int oy = max(0, 2 * iy - 2); oy <= min(Ho - 1, 2 * iy + 2); ++oy) {
      int y0, y1;
      float fy;
      up_taps(oy, H, y0, y1, fy);
      const float wy = (y0 == iy ? 1.f - fy : 0.f) + (y1 == iy ? fy : 0.f);
      if (wy == 0.f) continue;
      for (int ox = max(0, 2 * ix - 2); ox <= min(Wo - 1, 2 * ix + 2); ++ox) {
        int x0, x1;
        float fx;
        up_taps(ox, W, x0, x1, fx);
        const float wx = (x0 == ix ? 1.f - fx : 0.f) + (x1 == ix ? fx : 0.f);
        if (wx == 0.f) continue;
        float g[8];
        ld8(gy + ((size_t)oy * Wo + ox) * ld_gy + vc * 8, g);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += wy * wx * g[i];
      }
    }
    st8(gx + (size_t)p * C + vc * 8, acc);
  }
}

// dst[p, 0..C) (=|+=) src[p, 0..C) with independent pixel strides (SkipBlock's torch.cat and its split, cc12m_1.py:57-58)
__global__ void copy_channels_kernel(const act_t* __restrict__ src, int ld_src, act_t* __restrict__ dst, int ld_dst,
                                     int C, long long pixels, int accumulate) {
  const int vecs = C / 8;
  const long long n = pixels * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    if (accumulate) {
      float a[8], b[8];
      ld8(src + (size_t)p * ld_src + vc * 8, a);
      ld8(dst + (size_t)p * ld_dst + vc * 8, b);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] += b[i];
      st8(dst + (size_t)p * ld_dst + vc * 8, a);
    } else {
      *reinterpret_cast<uint4*>(dst + (size_t)p * ld_dst + vc * 8) =
          *reinterpret_cast<const uint4*>(src + (size_t)p * ld_src + vc * 8);
    }
  }
}

// explicit im2col of a 3x3 / pad 1 convolution for the tiny-spatial levels (W < 8: below the TMA tile of the
// implicit-GEMM path): A[p, tap * C + c] = x[p + off(tap), c] (zero outside)
__global__ void im2col3x3_kernel(const act_t* __restrict__ x, int H, int W, int C, act_t* __restrict__ A) {
  const int vecs = C / 8;
  const long long n = (long long)H * W * 9 * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long q = v / vecs;
    const int tap = (int)(q % 9);
    const long long p = q / 9;
    const int ix = (int)(p % W) + tap % 3 - 1, iy = (int)(p / W) + tap / 3 - 1;
    uint4 u = make_uint4(0, 0, 0, 0);
    if (ix >= 0 && ix < W && iy >= 0 && iy < H) u = *reinterpret_cast<const uint4*>(x + ((size_t)iy * W + ix) * C + vc * 8);
    *reinterpret_cast<uint4*>(A + ((size_t)p * 9 + tap) * C + vc * 8) = u;
  }
}

// y[r] = act(sum_k W[r, k] x[k] + b[r]) (+ res[r]); one warp per row, fp16 weights, fp32 everything else.
// The mapping network and every Modulation2d linear of the iteration (cc12m_1.py:30-38, 118-123, 244-246).
__global__ void __launch_bounds__(256) gemv_f16_kernel(const act_t* __restrict__ Wt, int K, int R,
                                                       const float* __restrict__ x, const float* __restrict__ bias,
                                                       int relu, const float* __restrict__ res, float* __restrict__ y) {
  const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= R) return;
  const act_t* w = Wt + (size_t)warp * K;
  float acc = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    float f[8];
    ld8(w + k, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += f[i] * x[k + i];
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    float v = acc + (bias ? bias[warp] : 0.f);
    if (relu) v = fmaxf(v, 0.f);
    if (res) v += res[warp];
    y[warp] = v;
  }
}

__global__ void vd_set_features_kernel(VdFeatures f, float* __restrict__ h0_tail, float* __restrict__ te) {
  const int i = threadIdx.x;
  if (i < 128) h0_tail[i] = f.v[i];
  else if (i < 144) te[i - 128] = f.v[i];
}

// canvas index of gen pixel p, or -1 outside the crop window
__device__ __forceinline__ int vd_crop_index(const VdCrop& c, int p) {
  const int y = p / c.gw - c.my, x = p % c.gw - c.mx;
  return (y >= 0 && y < c.h && x >= 0 && x < c.w) ? y * c.w + x : -1;
}
// pred = x alpha - v sigma; pixels = ClampWithGrad((pred + 1) / 2, 0, 1) (sampling.py:7-15, vdiff.py:159-163) on the
// window (vdiff.py:165-170)
__global__ void vd_finish_kernel(const float* __restrict__ vout, int ld, const float* __restrict__ x, float alpha,
                                 float sigma, VdCrop cr, float* __restrict__ v_planar, float* __restrict__ pred,
                                 float* __restrict__ pre, float* __restrict__ img) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, pixels = cr.gh * cr.gw;
  if (p >= pixels) return;
  const int q = vd_crop_index(cr, p), cpx = cr.h * cr.w;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t o = (size_t)c * pixels + p;
    const float v = vout[(size_t)p * ld + c];
    const float pr = x[o] * alpha - v * sigma;
    const float u = (pr + 1.f) * 0.5f;
    v_planar[o] = v;
    pred[o] = pr;
    if (q >= 0) {
      pre[(size_t)c * cpx + q] = u;
      img[(size_t)c * cpx + q] = fminf(fmaxf(u, 0.f), 1.f);
    }
  }
}
// g_pred = 0.5 g_img [g (pre - clamp pre) >= 0] inside the window, 0 outside; g_v = -sigma g_pred -> fp16 [pixels, ld]
// (scaled gradient stays scaled)
__global__ void vd_finish_bwd_kernel(const float* __restrict__ g_img, const float* __restrict__ pre, float sigma,
                                     VdCrop cr, int ld, float* __restrict__ g_pred, act_t* __restrict__ g_v) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, pixels = cr.gh * cr.gw;
  if (p >= pixels) return;
  const int q = vd_crop_index(cr, p), cpx = cr.h * cr.w;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t o = (size_t)c * pixels + p;
    float gp = 0.f;
    if (q >= 0) {
      const float g = g_img[(size_t)c * cpx + q], u = pre[(size_t)c * cpx + q];
      const float cl = fminf(fmaxf(u, 0.f), 1.f);
      gp = (g * (u - cl) >= 0.f) ? 0.5f * g : 0.f;
    }
    g_pred[o] = gp;
    g_v[(size_t)p * ld + c] = __float2half_rn(-sigma * gp);
  }
}
// z.grad = (alpha g_pred + g_in[:, 0..2]) / grad_scale
__global__ void vd_zgrad_kernel(const float* __restrict__ g_pred, const act_t* __restrict__ g_in, int ld, float alpha,
                                float inv_scale, int pixels, float* __restrict__ z_grad) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pixels) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t o = (size_t)c * pixels + p;
    z_grad[o] = (alpha * g_pred[o] + __half2float(g_in[(size_t)p * ld + c])) * inv_scale;
  }
}
// sampling.sample_step_noise (sampling.py:18-39): x <- pred a_next + (x sigma_i + v alpha_i) adj + noise ddim
__global__ void vd_renoise_kernel(float* __restrict__ x, const float* __restrict__ pred, const float* __restrict__ v,
                                  const float* __restrict__ noise, float alpha_i, float sigma_i, float alpha_next,
                                  float adjusted_sigma, float ddim_sigma, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float eps = x[i] * sigma_i + v[i] * alpha_i;
  x[i] = pred[i] * alpha_next + eps * adjusted_sigma + (noise ? noise[i] * ddim_sigma : 0.f);
}

}  // namespace

void vd_set_features(const VdFeatures& f, float* h0_tail, float* te, cudaStream_t st) {
  vd_set_features_kernel<<<1, 160, 0, st>>>(f, h0_tail, te);
}
void vd_input(const float* x, const float* te, int pixels, act_t* out, cudaStream_t st) {
  vd_input_kernel<<<(pixels + 255) / 256, 256, 0, st>>>(x, te, pixels, out);
}
void avgpool2x(const act_t* x, int H, int W, int C, int ld_in, act_t* y, cudaStream_t st) {
  avgpool2x_kernel<<<vgrid((long long)(H / 2) * (W / 2) * C / 8), 256, 0, st>>>(x, H, W, C, ld_in, y);
}
void avgpool2x_backward(const act_t* gy, int H, int W, int C, int accumulate, act_t* gx, cudaStream_t st) {
  avgpool2x_bwd_kernel<<<vgrid((long long)H * W * C / 8), 256, 0, st>>>(gy, H, W, C, accumulate, gx);
}
void bilinear_up2x(const act_t* x, int H, int W, int C, act_t* y, int ld_out, cudaStream_t st) {
  bilinear_up2x_kernel<<<vgrid((long long)4 * H * W * C / 8), 256, 0, st>>>(x, H, W, C, y, ld_out);
}
void bilinear_up2x_backward(const act_t* gy, int H, int W, int C, int ld_gy, act_t* gx, cudaStream_t st) {
  bilinear_up2x_bwd_kernel<<<vgrid((long long)H * W * C / 8), 256, 0, st>>>(gy, H, W, C, ld_gy, gx);
}
void copy_channels(const act_t* src, int ld_src, act_t* dst, int ld_dst, int C, long long pixels, int accumulate,
                   cudaStream_t st) {
  copy_channels_kernel<<<vgrid(pixels * C / 8), 256, 0, st>>>(src, ld_src, dst, ld_dst, C, pixels, accumulate);
}
void im2col3x3(const act_t* x, int H, int W, int C, act_t* A, cudaStream_t st) {
  im2col3x3_kernel<<<vgrid((long long)H * W * 9 * C / 8), 256, 0, st>>>(x, H, W, C, A);
}
void gemv_f16(const act_t* W, int K, int R, const float* x, const float* bias, int relu, const float* res, float* y,
              cudaStream_t st) {
  gemv_f16_kernel<<<(R * 32 + 255) / 256, 256, 0, st>>>(W, K, R, x, bias, relu, res, y);
}
void vd_finish(const float* vout, int ld, const float* x, float alpha, float sigma, VdCrop c, float* v_planar,
               float* pred, float* pre, float* img, cudaStream_t st) {
  const int pixels = c.gh * c.gw;
  vd_finish_kernel<<<(pixels + 255) / 256, 256, 0, st>>>(vout, ld, x, alpha, sigma, c, v_planar, pred, pre, img);
}
void vd_finish_backward(const float* g_img, const float* pre, float sigma, VdCrop c, int ld, float* g_pred, act_t* g_v,
                        cudaStream_t st) {
  const int pixels = c.gh * c.gw;
  vd_finish_bwd_kernel<<<(pixels + 255) / 256, 256, 0, st>>>(g_img, pre, sigma, c, ld, g_pred, g_v);
}
void vd_zgrad(const float* g_pred, const act_t* g_in, int ld, float alpha, float inv_scale, int pixels, float* z_grad,
              cudaStream_t st) {
  vd_zgrad_kernel<<<(pixels + 255) / 256, 256, 0, st>>>(g_pred, g_in, ld, alpha, inv_scale, pixels, z_grad);
}
void vd_renoise(float* x, const float* pred, const float* v, const float* noise, float alpha_i, float sigma_i,
                float alpha_next, float adjusted_sigma, float ddim_sigma, long long n, cudaStream_t st) {
  vd_renoise_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(x, pred, v, noise, alpha_i, sigma_i, alpha_next,
                                                            adjusted_sigma, ddim_sigma, n);
}

}  // namespace pxr
