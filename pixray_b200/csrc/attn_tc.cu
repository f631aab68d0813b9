// See attn_tc.cuh.  sm_90a: tensor-core mma.sync m16n8k16 (fp16 x fp16 -> fp32), operands staged in shared memory.
#include "attn_tc.cuh"
#include "launch.cuh"
#include <cmath>
#include <cstdio>
#include <mutex>

namespace pxr {
namespace {

constexpr int AT_THREADS = 128;  // four warps, 16 rows each: one 64-row block per CTA
constexpr int LDS = 72;          // row pitch (halves) of [rows][64] tiles: 144 B, conflict-free fragment loads
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t ld32(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t pack(float x, float y) {
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}
// A fragment (16 x 16) of a row-major tile X[row][k] with pitch ld: rows r0.., k k0..
__device__ __forceinline__ void load_a(uint32_t (&a)[4], const __half* X, int ld, int r0, int k0, int g, int t) {
  a[0] = ld32(X + (r0 + g) * ld + k0 + 2 * t);
  a[1] = ld32(X + (r0 + g + 8) * ld + k0 + 2 * t);
  a[2] = ld32(X + (r0 + g) * ld + k0 + 2 * t + 8);
  a[3] = ld32(X + (r0 + g + 8) * ld + k0 + 2 * t + 8);
}
// A fragment of a 16-column slice (columns 2c, 2c+1 of the 8-column accumulator tiles) of accumulator rows
__device__ __forceinline__ void acc_to_a(uint32_t (&a)[4], const float (&x0)[4], const float (&x1)[4]) {
  a[0] = pack(x0[0], x0[1]);
  a[1] = pack(x0[2], x0[3]);
  a[2] = pack(x1[0], x1[1]);
  a[3] = pack(x1[2], x1[3]);
}
// Y[rows][64] <- rows [r0, r0 + n) of the [B*T, ld] tensor at column c0 (one image), zero past T
__device__ __forceinline__ void load_rows(__half* Y, const __half* src, int ld, int c0, int r0, int n, int T) {
  for (int i = threadIdx.x; i < n * 8; i += AT_THREADS) {
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < T) v = *reinterpret_cast<const uint4*>(src + (size_t)(r0 + r) * ld + c0 + c);
    *reinterpret_cast<uint4*>(Y + r * LDS + c) = v;
  }
}
// Yt[64][ldt] (transposed: Yt[d][row]) <- the same rows
__device__ __forceinline__ void load_rows_t(__half* Yt, int ldt, const __half* src, int ld, int c0, int r0, int n, int T) {
  for (int i = threadIdx.x; i < n * 8; i += AT_THREADS) {
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < T) v = *reinterpret_cast<const uint4*>(src + (size_t)(r0 + r) * ld + c0 + c);
    const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) Yt[(c + j) * ldt + r] = h[j];
  }
}
// dO rows [r0, r0 + 64) into Y (and Yt when non-null), D[r] = dO_r . O_r, lse[r] * log2(e) (zeros past T)
__device__ __forceinline__ void load_do_block(const AttnParams& p, int b, int h, int r0, __half* Y, __half* Yt, float* D,
                                              float* L) {
  const int T = p.T, W = p.W;
  for (int i = threadIdx.x; i < 64 * 8; i += AT_THREADS) {  // the 8 lanes of a row are adjacent: shuffle-reduce
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0), o = make_uint4(0, 0, 0, 0);
    if (r0 + r < T) {
      const size_t off = (size_t)(b * T + r0 + r) * W + h * 64 + c;
      v = *reinterpret_cast<const uint4*>(p.d_o + off);
      o = *reinterpret_cast<const uint4*>(p.o + off);
    }
    *reinterpret_cast<uint4*>(Y + r * LDS + c) = v;
    const __half* hv = reinterpret_cast<const __half*>(&v);
    const __half* ho = reinterpret_cast<const __half*>(&o);
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      d += __half2float(hv[j]) * __half2float(ho[j]);
      if (Yt) Yt[(c + j) * LDS + r] = hv[j];
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    if ((i & 7) == 0) {
      D[r] = d;
      L[r] = (r0 + r < T) ? p.lse[(size_t)(b * p.H + h) * T + r0 + r] * LOG2E : 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ forward
// CTA = (64-query block, head, image).  Warp w: query rows 16 w.. of the block; online softmax over 64-key blocks.
__global__ void __launch_bounds__(AT_THREADS) attn_fwd_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_at[];
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, TP = (T + 63) / 64 * 64, ld3 = 3 * p.W, ldv = TP + 8;
  __half* Qs = reinterpret_cast<__half*>(smem_at);
  __half* Ks = Qs + 64 * LDS;
  __half* Vt = Ks + TP * LDS;  // [64][TP + 8]: V transposed (the PV product's B operand is key-contiguous)
  const __half* base = p.qkv + (size_t)b * T * ld3;
  load_rows(Qs, base, ld3, h * 64, qb * 64, 64, T);
  load_rows(Ks, base, ld3, p.W + h * 64, 0, TP, T);
  load_rows_t(Vt, ldv, base, ld3, 2 * p.W + h * 64, 0, TP, T);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, r0 = warp * 16;
  uint32_t qa[4][4];
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) load_a(qa[kc], Qs, LDS, r0, kc * 16, g, t);
  float o[8][4] = {};
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float c = p.scale * LOG2E;
  for (int kb = 0; kb * 64 < T; ++kb) {
    float s[8][4] = {};
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half* kr = Ks + (kb * 64 + j * 8 + g) * LDS + kc * 16 + 2 * t;
        mma16816(s[j], qa[kc], ld32(kr), ld32(kr + 8));
      }
    float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kb * 64 + j * 8 + 2 * t + (e & 1);
        s[j][e] = key < T ? s[j][e] * c : -INFINITY;
        if (e < 2) x0 = fmaxf(x0, s[j][e]);
        else x1 = fmaxf(x1, s[j][e]);
      }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, off));
      x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, off));
    }
    const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);  // every key block holds a key < T: finite
    const float a0 = exp2f(m0 - n0), a1 = exp2f(m1 - n1);
    m0 = n0;
    m1 = n1;
    l0 *= a0;
    l1 *= a1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = exp2f(s[j][0] - n0);
      s[j][1] = exp2f(s[j][1] - n0);
      s[j][2] = exp2f(s[j][2] - n1);
      s[j][3] = exp2f(s[j][3] - n1);
      l0 += s[j][0] + s[j][1];
      l1 += s[j][2] + s[j][3];
      o[j][0] *= a0;
      o[j][1] *= a0;
      o[j][2] *= a1;
      o[j][3] *= a1;
    }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {  // 16 keys of the block
      uint32_t pa[4];
      acc_to_a(pa, s[2 * kc], s[2 * kc + 1]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half* vr = Vt + (j * 8 + g) * ldv + kb * 64 + kc * 16 + 2 * t;
        mma16816(o[j], pa, ld32(vr), ld32(vr + 8));
      }
    }
  }
#pragma unroll
  for (int off = 1; off < 4; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
  const int q0 = qb * 64 + r0 + g, q1 = q0 + 8;
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = h * 64 + j * 8 + 2 * t;
    if (q0 < T) *reinterpret_cast<uint32_t*>(p.o + (size_t)(b * T + q0) * p.W + col) = pack(o[j][0] * i0, o[j][1] * i0);
    if (q1 < T) *reinterpret_cast<uint32_t*>(p.o + (size_t)(b * T + q1) * p.W + col) = pack(o[j][2] * i1, o[j][3] * i1);
  }
  if (t == 0) {
    float* lse = p.lse + (size_t)(b * p.H + h) * T;
    if (q0 < T) lse[q0] = (m0 + log2f(l0)) * LN2;
    if (q1 < T) lse[q1] = (m1 + log2f(l1)) * LN2;
  }
}

// ------------------------------------------------------------------------------------------------------------ dQ
// CTA = (64-query block, head, image).  dQ_i = scale * sum_j P_ij (dP_ij - D_i) K_j with dP = dO V^T.
__global__ void __launch_bounds__(AT_THREADS) attn_bwd_dq_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_at[];
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, TP = (T + 63) / 64 * 64, ld3 = 3 * p.W, ldk = TP + 8;
  __half* Qs = reinterpret_cast<__half*>(smem_at);
  __half* dOs = Qs + 64 * LDS;
  __half* Ks = dOs + 64 * LDS;
  __half* Vs = Ks + TP * LDS;
  __half* Kt = Vs + TP * LDS;  // [64][TP + 8]
  float* Ds = reinterpret_cast<float*>(Kt + 64 * ldk);
  float* Ls = Ds + 64;
  const __half* base = p.qkv + (size_t)b * T * ld3;
  load_rows(Qs, base, ld3, h * 64, qb * 64, 64, T);
  load_rows(Ks, base, ld3, p.W + h * 64, 0, TP, T);
  load_rows(Vs, base, ld3, 2 * p.W + h * 64, 0, TP, T);
  load_rows_t(Kt, ldk, base, ld3, p.W + h * 64, 0, TP, T);
  load_do_block(p, b, h, qb * 64, dOs, nullptr, Ds, Ls);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, r0 = warp * 16;
  uint32_t qa[4][4], da[4][4];
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    load_a(qa[kc], Qs, LDS, r0, kc * 16, g, t);
    load_a(da[kc], dOs, LDS, r0, kc * 16, g, t);
  }
  const float L0 = Ls[r0 + g], L1 = Ls[r0 + g + 8], D0 = Ds[r0 + g], D1 = Ds[r0 + g + 8];
  const float c = p.scale * LOG2E;
  float dq[8][4] = {};
  for (int kb = 0; kb * 64 < T; ++kb) {
    float s[8][4] = {}, dp[8][4] = {};
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row = (kb * 64 + j * 8 + g) * LDS + kc * 16 + 2 * t;
        mma16816(s[j], qa[kc], ld32(Ks + row), ld32(Ks + row + 8));
        mma16816(dp[j], da[kc], ld32(Vs + row), ld32(Vs + row + 8));
      }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kb * 64 + j * 8 + 2 * t + (e & 1);
        const float pv = key < T ? exp2f(s[j][e] * c - (e < 2 ? L0 : L1)) : 0.f;
        s[j][e] = pv * (dp[j][e] - (e < 2 ? D0 : D1));
      }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      uint32_t a[4];
      acc_to_a(a, s[2 * kc], s[2 * kc + 1]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half* kr = Kt + (j * 8 + g) * ldk + kb * 64 + kc * 16 + 2 * t;
        mma16816(dq[j], a, ld32(kr), ld32(kr + 8));
      }
    }
  }
  const int q0 = qb * 64 + r0 + g, q1 = q0 + 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = h * 64 + j * 8 + 2 * t;
    if (q0 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + q0) * ld3 + col) = pack(dq[j][0] * p.scale, dq[j][1] * p.scale);
    if (q1 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + q1) * ld3 + col) = pack(dq[j][2] * p.scale, dq[j][3] * p.scale);
  }
}

// ------------------------------------------------------------------------------------------------------------ dK, dV
// CTA = (64-key block, head, image), loop over 64-query blocks.  Transposed scores: S^T = K Q^T, dP^T = V dO^T;
// dV_j = sum_i P_ij dO_i, dK_j = scale * sum_i P_ij (dP_ij - D_i) Q_i.
__global__ void __launch_bounds__(AT_THREADS) attn_bwd_dkv_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_at[];
  const int kb0 = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, ld3 = 3 * p.W;
  __half* Ks = reinterpret_cast<__half*>(smem_at);
  __half* Vs = Ks + 64 * LDS;
  __half* Qs = Vs + 64 * LDS;
  __half* dOs = Qs + 64 * LDS;
  __half* Qt = dOs + 64 * LDS;  // [64][LDS]: Q^T of the query block
  __half* dOt = Qt + 64 * LDS;
  float* Ds = reinterpret_cast<float*>(dOt + 64 * LDS);
  float* Ls = Ds + 64;
  const __half* base = p.qkv + (size_t)b * T * ld3;
  load_rows(Ks, base, ld3, p.W + h * 64, kb0 * 64, 64, T);
  load_rows(Vs, base, ld3, 2 * p.W + h * 64, kb0 * 64, 64, T);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, r0 = warp * 16;
  uint32_t ka[4][4], va[4][4];
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    load_a(ka[kc], Ks, LDS, r0, kc * 16, g, t);
    load_a(va[kc], Vs, LDS, r0, kc * 16, g, t);
  }
  const float c = p.scale * LOG2E;
  float dk[8][4] = {}, dv[8][4] = {};
  for (int qb = 0; qb * 64 < T; ++qb) {
    __syncthreads();  // the previous query block's tiles are consumed
    load_rows(Qs, base, ld3, h * 64, qb * 64, 64, T);
    load_rows_t(Qt, LDS, base, ld3, h * 64, qb * 64, 64, T);
    load_do_block(p, b, h, qb * 64, dOs, dOt, Ds, Ls);
    __syncthreads();
    float s[8][4] = {}, dp[8][4] = {};
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row = (j * 8 + g) * LDS + kc * 16 + 2 * t;
        mma16816(s[j], ka[kc], ld32(Qs + row), ld32(Qs + row + 8));
        mma16816(dp[j], va[kc], ld32(dOs + row), ld32(dOs + row + 8));
      }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int ql = j * 8 + 2 * t + (e & 1);
        const float pv = qb * 64 + ql < T ? exp2f(s[j][e] * c - Ls[ql]) : 0.f;
        s[j][e] = pv;
        dp[j][e] = pv * (dp[j][e] - Ds[ql]);
      }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {  // 16 queries
      uint32_t pa[4], sa[4];
      acc_to_a(pa, s[2 * kc], s[2 * kc + 1]);
      acc_to_a(sa, dp[2 * kc], dp[2 * kc + 1]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row = (j * 8 + g) * LDS + kc * 16 + 2 * t;
        mma16816(dv[j], pa, ld32(dOt + row), ld32(dOt + row + 8));
        mma16816(dk[j], sa, ld32(Qt + row), ld32(Qt + row + 8));
      }
    }
  }
  const int k0 = kb0 * 64 + r0 + g, k1 = k0 + 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = h * 64 + j * 8 + 2 * t;
    if (k0 < T) {
      __half* row = p.gqkv + (size_t)(b * T + k0) * ld3 + col;
      *reinterpret_cast<uint32_t*>(row + p.W) = pack(dk[j][0] * p.scale, dk[j][1] * p.scale);
      *reinterpret_cast<uint32_t*>(row + 2 * p.W) = pack(dv[j][0], dv[j][1]);
    }
    if (k1 < T) {
      __half* row = p.gqkv + (size_t)(b * T + k1) * ld3 + col;
      *reinterpret_cast<uint32_t*>(row + p.W) = pack(dk[j][2] * p.scale, dk[j][3] * p.scale);
      *reinterpret_cast<uint32_t*>(row + 2 * p.W) = pack(dv[j][2], dv[j][3]);
    }
  }
}

int fwd_smem(int TP) { return (64 * LDS + TP * LDS + 64 * (TP + 8)) * 2; }
int dq_smem(int TP) { return (2 * 64 * LDS + 2 * TP * LDS + 64 * (TP + 8)) * 2 + 2 * 64 * 4; }
int dkv_smem() { return 6 * 64 * LDS * 2 + 2 * 64 * 4; }

}  // namespace

bool attn_supported(int T, int head_dim, int W) { return head_dim == 64 && T >= 1 && T <= 240 && W % 64 == 0; }

int attn_plan_make(AttnPlan* plan, const __half* qkv, __half* o, const __half* d_o, __half* gqkv, float* lse, int B,
                   int T, int H, int W, float scale, int num_sms, char* err, int errlen) {
  (void)num_sms;
  *plan = AttnPlan{};
  if (!attn_supported(T, W / H, W) || W != 64 * H) {
    if (err && errlen > 0) snprintf(err, errlen, "fused attention needs 64-wide heads and T <= 240");
    return -1;
  }
  AttnParams& p = plan->p;
  p.qkv = qkv;
  p.o = o;
  p.lse = lse;
  p.d_o = d_o;
  p.gqkv = gqkv;
  p.T = T;
  p.H = H;
  p.B = B;
  p.W = W;
  p.scale = scale;
  const int TP = (T + 63) / 64 * 64;
  plan->smem_fwd = fwd_smem(TP);
  plan->smem_dq = dq_smem(TP);
  plan->smem_dkv = dkv_smem();
  const double tt = (double)T * T * 64 * 2 * B * H;
  plan->flops_fwd = 2 * tt;  // QK^T, PV
  plan->flops_bwd = 4 * tt;  // dP, dQ, dK, dV (the recomputed S is not algorithmic work)
  const double mw = (double)B * T * W * 2.0;  // one [B*T, W] fp16 tensor
  plan->bytes_fwd = 3 * mw + mw + 4.0 * B * H * T;
  plan->bytes_bwd = 3 * mw + mw + mw + 3 * mw + 4.0 * B * H * T;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, fwd_smem(256));
    cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dq_smem(256));
    cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dkv_smem());
  });
  return 0;
}

void attn_forward_launch(const AttnPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  launch_pdl(attn_fwd_kernel, dim3((p.T + 63) / 64, p.H, p.B), dim3(AT_THREADS), plan.smem_fwd, st, p);
}

void attn_backward_launch(const AttnPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  launch_pdl(attn_bwd_dq_kernel, dim3((p.T + 63) / 64, p.H, p.B), dim3(AT_THREADS), plan.smem_dq, st, p);
  launch_pdl(attn_bwd_dkv_kernel, dim3((p.T + 63) / 64, p.H, p.B), dim3(AT_THREADS), plan.smem_dkv, st, p);
}

}  // namespace pxr
