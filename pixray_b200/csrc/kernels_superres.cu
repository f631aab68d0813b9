// Pointwise passes of the super-resolution drawer (RRDBNet, engine_superres.inc): the RRDB's outer residual and the
// latent's gradient.  Every convolution of the net runs on the implicit-GEMM wgmma path (gemm_tc.cu).
#include "kernels.cuh"
#include "launch.cuh"

namespace pxr {
namespace {

__global__ void __launch_bounds__(256) sr_axpy_kernel(const act_t* __restrict__ a, int lda, float alpha,
                                                      const act_t* b, int ldb, act_t* y, int ldy, int vecs,
                                                      long long n) {
  pdl_prologue();
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const long long p = i / vecs;
    const int c0 = (int)(i % vecs) * 8;
    const uint4 ua = *reinterpret_cast<const uint4*>(a + p * lda + c0);
    uint4 ub = make_uint4(0, 0, 0, 0);
    if (b) ub = *reinterpret_cast<const uint4*>(b + p * ldb + c0);
    const __half2* ha = reinterpret_cast<const __half2*>(&ua);
    const __half2* hb = reinterpret_cast<const __half2*>(&ub);
    uint4 out;
    __half2* ho = reinterpret_cast<__half2*>(&out);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
      ho[j] = __floats2half2_rn(fmaf(alpha, fa.x, fb.x), fmaf(alpha, fa.y, fb.y));
    }
    *reinterpret_cast<uint4*>(y + p * ldy + c0) = out;
  }
}

__global__ void __launch_bounds__(256) sr_zgrad_kernel(const act_t* __restrict__ g, int ld, long long pixels,
                                                       float inv_scale, float* __restrict__ z_grad) {
  pdl_prologue();
  const long long i = blockIdx.x * 256LL + threadIdx.x;  // over [3, pixels]
  if (i >= 3 * pixels) return;
  const long long c = i / pixels, p = i % pixels;
  z_grad[i] = __half2float(g[p * ld + c]) * inv_scale;
}

int sr_grid(long long n) {
  const long long g = (n + 255) / 256;
  return (int)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}

}  // namespace

void sr_axpy(const act_t* a, int lda, float alpha, const act_t* b, int ldb, act_t* y, int ldy, int C, long long pixels,
             cudaStream_t st) {
  const long long n = pixels * (C / 8);
  launch_pdl(sr_axpy_kernel, dim3(sr_grid(n)), dim3(256), 0, st, a, lda, alpha, b, ldb, y, ldy, C / 8, n);
}

void sr_zgrad(const act_t* g, int ld, long long pixels, float inv_scale, float* z_grad, cudaStream_t st) {
  launch_pdl(sr_zgrad_kernel, dim3(sr_grid(3 * pixels)), dim3(256), 0, st, g, ld, pixels, inv_scale, z_grad);
}

}  // namespace pxr
