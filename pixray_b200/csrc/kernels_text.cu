// Text-tower row kernels (engine_text.inc): the token-embedding gather with the positional add into the residual
// stream, and the gather of each sequence's EOT row before ln_final / text_projection.
#include "kernels.cuh"
#include "launch.cuh"

namespace pxr {
namespace {

// y[r, :] = tok_emb[ids[r], :] + pos[r % T, :], four columns per thread, summed in fp32
template <typename YT>
__global__ void text_embed_kernel(const int* __restrict__ ids, const act_t* __restrict__ tok_emb,
                                  const float* __restrict__ pos, int T, long long n4, int W4, YT* __restrict__ y) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / W4;
    const int c4 = (int)(i % W4);
    const uint2 u = reinterpret_cast<const uint2*>(tok_emb + (size_t)ids[r] * W4 * 4)[c4];
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    const float4 p = reinterpret_cast<const float4*>(pos)[(r % T) * W4 + c4];
    const float4 s = make_float4(a.x + p.x, a.y + p.y, b.x + p.z, b.y + p.w);
    if constexpr (sizeof(YT) == 4) {
      reinterpret_cast<float4*>(y)[i] = s;
    } else {
      const __half2 lo = __floats2half2_rn(s.x, s.y), hi = __floats2half2_rn(s.z, s.w);
      uint2 o;
      o.x = *reinterpret_cast<const uint32_t*>(&lo);
      o.y = *reinterpret_cast<const uint32_t*>(&hi);
      reinterpret_cast<uint2*>(y)[i] = o;
    }
  }
}

// one block per gathered row, 16-byte vectors
__global__ void gather_rows_kernel(const uint4* __restrict__ x, const int* __restrict__ src, int v_per_row,
                                   uint4* __restrict__ y) {
  pdl_prologue();
  const int b = blockIdx.x;
  const uint4* s = x + (size_t)src[b] * v_per_row;
  for (int v = threadIdx.x; v < v_per_row; v += blockDim.x) y[(size_t)b * v_per_row + v] = s[v];
}

}  // namespace

void text_embed(const int* ids, const act_t* tok_emb, const float* pos, int T, int rows, int W, act_t* y16, float* y32,
                cudaStream_t st) {
  const long long n4 = (long long)rows * W / 4;
  const long long blocks = (n4 + 255) / 256;
  const int grid = (int)(blocks < 148 * 8 ? blocks : 148 * 8);
  if (y16) launch_pdl(text_embed_kernel<act_t>, dim3(grid), dim3(256), 0, st, ids, tok_emb, pos, T, n4, W / 4, y16);
  else launch_pdl(text_embed_kernel<float>, dim3(grid), dim3(256), 0, st, ids, tok_emb, pos, T, n4, W / 4, y32);
}

void gather_rows(const void* x, const int* src, int n, int W, int elem_bytes, void* y, cudaStream_t st) {
  const int v_per_row = W * elem_bytes / 16;
  launch_pdl(gather_rows_kernel, dim3(n), dim3(128), 0, st, static_cast<const uint4*>(x), src, v_per_row,
             static_cast<uint4*>(y));
}

}  // namespace pxr
