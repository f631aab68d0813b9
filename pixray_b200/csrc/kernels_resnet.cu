// Row kernels of the CLIP ResNet image towers (engine_resnet.inc): the attention pool's token build, its single-query
// attention forward and backward, and the ReLU-masked adjoints of AvgPool2d(2) and of the token build.  The convolutions
// and projections run on the GEMM (gemm_tc.cu); the stem's input stage lives with the other preprocess kernels
// (kernels_cutouts.cu).
#include "kernels.cuh"
#include "launch.cuh"

namespace pxr {
namespace {

__device__ __forceinline__ void ld8h(const act_t* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = __half22float2(h[i]);
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}
__device__ __forceinline__ void st8h(act_t* p, const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
int grid_for(long long n) {
  long long g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  return (int)(g < 1 ? 1 : g);
}

__global__ void __launch_bounds__(256) pool_bwd_relu_kernel(const act_t* __restrict__ gy, const act_t* __restrict__ y,
                                                            int rows, int W, int C, act_t* __restrict__ gx) {
  pdl_prologue();
  const int vecs = C / 8, Wo = W / 2;
  const long long n = (long long)rows * W * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long p = v / vecs;
    const int ix = (int)(p % W);
    const long long iy = p / W;
    float g[8], a[8];
    ld8h(gy + ((size_t)(iy >> 1) * Wo + (ix >> 1)) * C + vc * 8, g);
    ld8h(y + (size_t)p * C + vc * 8, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = a[i] > 0.f ? 0.25f * g[i] : 0.f;
    st8h(gx + (size_t)p * C + vc * 8, g);
  }
}

// one thread per (image, 8 channels): the mean in fp32 over the image's pixels in pixel order
__global__ void __launch_bounds__(256) pool_tokens_kernel(const act_t* __restrict__ x, int B, int HW, int C,
                                                          const float* __restrict__ pos, act_t* __restrict__ tok) {
  pdl_prologue();
  const int vecs = C / 8;
  const long long n = (long long)B * vecs;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs), b = (int)(v / vecs);
    const int c0 = vc * 8;
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int p = 0; p < HW; ++p) {
      float a[8];
      ld8h(x + ((size_t)b * HW + p) * C + c0, a);
      const float* ps = pos + (size_t)(1 + p) * C + c0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] += a[i];
        a[i] += ps[i];
      }
      st8h(tok + ((size_t)b * (HW + 1) + 1 + p) * C + c0, a);
    }
    const float inv = 1.f / (float)HW;
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] = s[i] * inv + pos[c0 + i];
    st8h(tok + (size_t)b * (HW + 1) * C + c0, s);
  }
}

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
  return r;
}

constexpr int POOL_THREADS = 128;

// one CTA per (image, head): scores by warps over tokens (a lane holds 2 of the 64 dimensions), fp32 softmax, then
// o[d] summed over the tokens in two halves
__global__ void __launch_bounds__(POOL_THREADS) attnpool_fwd_kernel(const float* __restrict__ q, const act_t* __restrict__ kv,
                                                                    int T, int C, float scale, act_t* __restrict__ o,
                                                                    float* __restrict__ p_out) {
  pdl_prologue();
  __shared__ float qs[64], s[RN_POOL_MAX_T], part[POOL_THREADS], red[POOL_THREADS / 32];
  const int H = C / 64, b = blockIdx.x / H, h = blockIdx.x % H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 64) qs[tid] = q[(size_t)b * C + h * 64 + tid] * scale;
  __syncthreads();
  const act_t* kb = kv + (size_t)b * T * 2 * C + h * 64;
  for (int t = warp; t < T; t += POOL_THREADS / 32) {
    const float2 k2 = __half22float2(reinterpret_cast<const __half2*>(kb + (size_t)t * 2 * C)[lane]);
    float d = qs[2 * lane] * k2.x + qs[2 * lane + 1] * k2.y;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if (lane == 0) s[t] = d;
  }
  __syncthreads();
  float m = -INFINITY;
  for (int t = tid; t < T; t += POOL_THREADS) m = fmaxf(m, s[t]);
  m = block_reduce(m, red, true);
  float z = 0.f;
  for (int t = tid; t < T; t += POOL_THREADS) {
    const float e = __expf(s[t] - m);
    s[t] = e;
    z += e;
  }
  z = block_reduce(z, red, false);
  const float inv = 1.f / z;
  float* pb = p_out + ((size_t)b * H + h) * T;
  for (int t = tid; t < T; t += POOL_THREADS) {
    s[t] *= inv;
    pb[t] = s[t];
  }
  __syncthreads();
  const int d = tid & 63, half = tid >> 6;
  const act_t* vb = kb + C;
  float acc = 0.f;
  for (int t = half; t < T; t += 2) acc += s[t] * __half2float(vb[(size_t)t * 2 * C + d]);
  part[tid] = acc;
  __syncthreads();
  if (tid < 64) o[(size_t)b * C + h * 64 + d] = __float2half_rn(part[tid] + part[tid + 64]);
}

// dv_t = p_t g_o; dp_t = g_o . v_t; ds_t = p_t (dp_t - sum_t' p_t' dp_t'); dk_t = scale ds_t q; dq = scale sum_t ds_t k_t
__global__ void __launch_bounds__(POOL_THREADS) attnpool_bwd_kernel(const float* __restrict__ q, const act_t* __restrict__ kv,
                                                                    const float* __restrict__ p, const act_t* __restrict__ g_o,
                                                                    int T, int C, float scale, act_t* __restrict__ g_q,
                                                                    act_t* __restrict__ g_kv) {
  pdl_prologue();
  __shared__ float qs[64], go[64], ps[RN_POOL_MAX_T], ds[RN_POOL_MAX_T], part[POOL_THREADS], red[POOL_THREADS / 32];
  const int H = C / 64, b = blockIdx.x / H, h = blockIdx.x % H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 64) {
    qs[tid] = q[(size_t)b * C + h * 64 + tid] * scale;
    go[tid] = __half2float(g_o[(size_t)b * C + h * 64 + tid]);
  }
  const float* pb = p + ((size_t)b * H + h) * T;
  for (int t = tid; t < T; t += POOL_THREADS) ps[t] = pb[t];
  __syncthreads();
  const act_t* kb = kv + (size_t)b * T * 2 * C + h * 64;
  const act_t* vb = kb + C;
  for (int t = warp; t < T; t += POOL_THREADS / 32) {
    const float2 v2 = __half22float2(reinterpret_cast<const __half2*>(vb + (size_t)t * 2 * C)[lane]);
    float d = go[2 * lane] * v2.x + go[2 * lane + 1] * v2.y;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if (lane == 0) ds[t] = d;
  }
  __syncthreads();
  float dsum = 0.f;
  for (int t = tid; t < T; t += POOL_THREADS) dsum += ps[t] * ds[t];
  dsum = block_reduce(dsum, red, false);
  for (int t = tid; t < T; t += POOL_THREADS) ds[t] = ps[t] * (ds[t] - dsum);
  __syncthreads();
  act_t* gkb = g_kv + (size_t)b * T * 2 * C + h * 64;
  for (int i = tid; i < T * 64; i += POOL_THREADS) {
    const int t = i >> 6, d = i & 63;
    gkb[(size_t)t * 2 * C + d] = __float2half_rn(ds[t] * qs[d]);        // scale is inside qs
    gkb[(size_t)t * 2 * C + C + d] = __float2half_rn(ps[t] * go[d]);
  }
  const int d = tid & 63, half = tid >> 6;
  float acc = 0.f;
  for (int t = half; t < T; t += 2) acc += ds[t] * __half2float(kb[(size_t)t * 2 * C + d]);
  part[tid] = acc;
  __syncthreads();
  if (tid < 64) g_q[(size_t)b * C + h * 64 + d] = __float2half_rn(scale * (part[tid] + part[tid + 64]));
}

__global__ void __launch_bounds__(256) pool_tokens_bwd_kernel(const act_t* __restrict__ g_tok, const act_t* __restrict__ g_tok0,
                                                              const act_t* __restrict__ y, int B, int HW, int C,
                                                              act_t* __restrict__ gx) {
  pdl_prologue();
  const int vecs = C / 8;
  const long long n = (long long)B * HW * vecs;
  const float inv = 1.f / (float)HW;
  for (long long v = blockIdx.x * 256LL + threadIdx.x; v < n; v += (long long)gridDim.x * 256) {
    const int vc = (int)(v % vecs);
    const long long bp = v / vecs;
    const int b = (int)(bp / HW), pix = (int)(bp % HW);
    float g[8], g0[8], g1[8], a[8];
    ld8h(g_tok + ((size_t)b * (HW + 1) + 1 + pix) * C + vc * 8, g);
    ld8h(g_tok + (size_t)b * (HW + 1) * C + vc * 8, g0);
    ld8h(g_tok0 + (size_t)b * C + vc * 8, g1);
    ld8h(y + (size_t)bp * C + vc * 8, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = a[i] > 0.f ? g[i] + (g0[i] + g1[i]) * inv : 0.f;
    st8h(gx + (size_t)bp * C + vc * 8, g);
  }
}

}  // namespace

void rn_pool_bwd_relu(const act_t* gy, const act_t* y, int rows, int W, int C, act_t* gx, cudaStream_t st) {
  launch_pdl(pool_bwd_relu_kernel, dim3(grid_for((long long)rows * W * C / 8)), dim3(256), 0, st, gy, y, rows, W, C, gx);
}
void rn_pool_tokens(const act_t* x, int B, int HW, int C, const float* pos, act_t* tok, cudaStream_t st) {
  launch_pdl(pool_tokens_kernel, dim3(grid_for((long long)B * C / 8)), dim3(256), 0, st, x, B, HW, C, pos, tok);
}
void rn_attnpool_forward(const float* q, const act_t* kv, int B, int T, int C, float scale, act_t* o, float* p,
                         cudaStream_t st) {
  launch_pdl(attnpool_fwd_kernel, dim3(B * (C / 64)), dim3(POOL_THREADS), 0, st, q, kv, T, C, scale, o, p);
}
void rn_attnpool_backward(const float* q, const act_t* kv, const float* p, const act_t* g_o, int B, int T, int C,
                          float scale, act_t* g_q, act_t* g_kv, cudaStream_t st) {
  launch_pdl(attnpool_bwd_kernel, dim3(B * (C / 64)), dim3(POOL_THREADS), 0, st, q, kv, p, g_o, T, C, scale, g_q, g_kv);
}
void rn_pool_tokens_backward(const act_t* g_tok, const act_t* g_tok0, const act_t* y, int B, int HW, int C, act_t* gx,
                             cudaStream_t st) {
  launch_pdl(pool_tokens_bwd_kernel, dim3(grid_for((long long)B * HW * C / 8)), dim3(256), 0, st, g_tok, g_tok0, y, B, HW, C,
             gx);
}

}  // namespace pxr
