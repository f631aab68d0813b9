// See attn_tc.cuh.  sm_90a: tensor-core mma.sync m16n8k16 (fp16 x fp16 -> fp32), operands staged in shared memory by
// cp.async and fed to the MMAs by ldmatrix.
#include "attn_tc.cuh"
#include "launch.cuh"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <mutex>

namespace pxr {
namespace {

constexpr int AT_WARPS = 8;
constexpr int AT_THREADS = 32 * AT_WARPS;
constexpr int ROW_BYTES = 128;  // one 64-wide fp16 row of a staged tile
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ uint32_t pack(float x, float y) {
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}
// A fragment of a 16-column slice (columns 2c, 2c+1 of the 8-column accumulator tiles) of accumulator rows
__device__ __forceinline__ void acc_to_a(uint32_t (&a)[4], const float (&x0)[4], const float (&x1)[4]) {
  a[0] = pack(x0[0], x0[1]);
  a[1] = pack(x0[2], x0[3]);
  a[2] = pack(x1[0], x1[1]);
  a[3] = pack(x1[2], x1[3]);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// Staged tiles are [rows][64] fp16, 128-byte rows, the 16-byte chunk c of row r stored at chunk c ^ (r & 7): the eight
// row addresses of every ldmatrix 8x8 matrix fall in eight different bank groups.
__device__ __forceinline__ uint32_t swz(int r, int c) { return r * ROW_BYTES + ((c ^ (r & 7)) << 4); }

// Lane addresses of one ldmatrix.x4 (tile byte address, first row r0, first 8-column chunk c0 of the 16 columns):
//  frag_a: the A fragment of rows r0..r0+15, columns 8 c0..8 c0+15 (also the .trans B fragment of two 8-wide n-tiles
//          of a [k][n] tile: rows = k, columns = n);
//  frag_b: the B fragments of two 8-wide n-tiles (rows r0.., r0+8..) of a [n][k] tile, k = columns 8 c0..8 c0+15.
__device__ __forceinline__ uint32_t frag_a(uint32_t tile, int r0, int c0, int lane) {
  return tile + swz(r0 + (lane & 15), c0 + (lane >> 4));
}
__device__ __forceinline__ uint32_t frag_b(uint32_t tile, int r0, int c0, int lane) {
  return tile + swz(r0 + (lane & 7) + ((lane >> 4) << 3), c0 + ((lane >> 3) & 1));
}

// tile rows [0, r1 - r0) <- 64 columns of rows [r0, r1) of one image's [T, ld] slice at src; zeros past T
__device__ __forceinline__ void stage(uint32_t tile, const __half* src, int ld, int r0, int r1, int T) {
  for (int i = threadIdx.x; i < (r1 - r0) * 8; i += AT_THREADS) {
    const int r = i >> 3, c = i & 7, row = r0 + r;
    const __half* g = src + (size_t)(row < T ? row : 0) * ld + c * 8;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(tile + swz(r, c)), "l"(g), "r"(row < T ? 16 : 0)
                 : "memory");
  }
}
__device__ __forceinline__ void stage_wait() {
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
}

// The 16-row tiles [lo, hi) of the pair that CTA blockIdx.x of gridDim.x owns (query tiles, and key tiles in backward)
__device__ __forceinline__ void tile_range(int NT, int& lo, int& hi) {
  const int per = (NT + gridDim.x - 1) / gridDim.x;
  lo = min(NT, (int)blockIdx.x * per);
  hi = min(NT, lo + per);
}

// ------------------------------------------------------------------------------------------------------------ forward
// CTA = (split, head, image): K and V of the pair and the CTA's query tiles are staged once.  Warp w owns the 16-row
// query tiles lo + w, lo + w + 8, ...: online softmax over 64-key blocks, whose 16-key chunks past T are skipped.
__global__ void __launch_bounds__(AT_THREADS, 2) attn_fwd_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_at[];
  const int h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, TP = (T + 15) & ~15, ld3 = 3 * p.W;
  int lo, hi;
  tile_range(TP / 16, lo, hi);
  const uint32_t Ks = smem_u32(smem_at), Vs = Ks + TP * ROW_BYTES, Qs = Vs + TP * ROW_BYTES;
  const __half* base = p.qkv + (size_t)b * T * ld3 + h * 64;
  stage(Ks, base + p.W, ld3, 0, TP, T);
  stage(Vs, base + 2 * p.W, ld3, 0, TP, T);
  stage(Qs, base, ld3, lo * 16, hi * 16, T);
  stage_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float c = p.scale * LOG2E;
  for (int qt = lo + warp; qt < hi; qt += AT_WARPS) {
    uint32_t qa[4][4];
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) ldsm4(qa[kc], frag_a(Qs, (qt - lo) * 16, 2 * kc, lane));
    float o[8][4] = {};
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int kb = 0; kb * 64 < T; ++kb) {
      float s[8][4] = {};
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 keys
        if (kb * 64 + j2 * 16 >= T) break;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          uint32_t kf[4];
          ldsm4(kf, frag_b(Ks, kb * 64 + j2 * 16, 2 * kc, lane));
          mma16816(s[2 * j2], qa[kc], kf[0], kf[1]);
          mma16816(s[2 * j2 + 1], qa[kc], kf[2], kf[3]);
        }
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
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 keys: O += P V, V read transposed by ldmatrix.trans
        if (kb * 64 + j2 * 16 >= T) break;
        uint32_t pa[4];
        acc_to_a(pa, s[2 * j2], s[2 * j2 + 1]);
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t vf[4];
          ldsm4t(vf, frag_a(Vs, kb * 64 + j2 * 16, 2 * n2, lane));
          mma16816(o[2 * n2], pa, vf[0], vf[1]);
          mma16816(o[2 * n2 + 1], pa, vf[2], vf[3]);
        }
      }
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, off);
      l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    const int q0 = qt * 16 + g, q1 = q0 + 8;
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
}

// ------------------------------------------------------------------------------------------------------------ backward
// CTA = (split, head, image): Q, K, V and dO of the pair are staged once, D_i = dO_i . O_i and lse_i log2(e) go to
// shared memory for every row.  P = exp(S - lse) is recomputed in both phases; dS = P o (dP - D) with dP = dO V^T.
//   phase 1: warp w owns the key tiles lo + w, lo + w + 8, ... and runs over 16-query chunks of the transposed scores
//            S^T = K Q^T, dP^T = V dO^T: dV_j = sum_i P_ij dO_i, dK_j = scale sum_i dS_ij Q_i;
//   phase 2: warp w owns the query tiles lo + w, ... and runs over 16-key chunks: dQ_i = scale sum_j dS_ij K_j.
// Each output row is written by the one warp that owns its tile.
__global__ void __launch_bounds__(AT_THREADS, 2) attn_bwd_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_at[];
  const int h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, TP = (T + 15) & ~15, NT = TP / 16, W = p.W, ld3 = 3 * W;
  int lo, hi;
  tile_range(NT, lo, hi);
  const uint32_t Qs = smem_u32(smem_at), Ks = Qs + TP * ROW_BYTES, Vs = Ks + TP * ROW_BYTES, dOs = Vs + TP * ROW_BYTES;
  float* Ds = reinterpret_cast<float*>(reinterpret_cast<char*>(smem_at) + 4 * TP * ROW_BYTES);
  float* Ls = Ds + TP;
  const __half* base = p.qkv + (size_t)b * T * ld3 + h * 64;
  stage(Qs, base, ld3, 0, TP, T);
  stage(Ks, base + W, ld3, 0, TP, T);
  stage(Vs, base + 2 * W, ld3, 0, TP, T);
  stage(dOs, p.d_o + (size_t)b * T * W + h * 64, W, 0, TP, T);
  for (int i = threadIdx.x; i < TP * 8; i += AT_THREADS) {  // the 8 lanes of a row are adjacent: shuffle-reduce
    const int r = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0), o = make_uint4(0, 0, 0, 0);
    if (r < T) {
      const size_t off = (size_t)(b * T + r) * W + h * 64 + c;
      v = *reinterpret_cast<const uint4*>(p.d_o + off);
      o = *reinterpret_cast<const uint4*>(p.o + off);
    }
    const __half* hv = reinterpret_cast<const __half*>(&v);
    const __half* ho = reinterpret_cast<const __half*>(&o);
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) d += __half2float(hv[j]) * __half2float(ho[j]);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    if ((i & 7) == 0) {
      Ds[r] = d;
      Ls[r] = r < T ? p.lse[(size_t)(b * p.H + h) * T + r] * LOG2E : 0.f;
    }
  }
  stage_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float c = p.scale * LOG2E;

  for (int kt = lo + warp; kt < hi; kt += AT_WARPS) {  // phase 1: dK, dV of 16 keys
    uint32_t ka[4][4], va[4][4];
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      ldsm4(ka[kc], frag_a(Ks, kt * 16, 2 * kc, lane));
      ldsm4(va[kc], frag_a(Vs, kt * 16, 2 * kc, lane));
    }
    float dk[8][4] = {}, dv[8][4] = {};
    for (int q16 = 0; q16 < TP; q16 += 16) {
      float s[2][4] = {}, dp[2][4] = {};
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        uint32_t f[4];
        ldsm4(f, frag_b(Qs, q16, 2 * kc, lane));
        mma16816(s[0], ka[kc], f[0], f[1]);
        mma16816(s[1], ka[kc], f[2], f[3]);
        ldsm4(f, frag_b(dOs, q16, 2 * kc, lane));
        mma16816(dp[0], va[kc], f[0], f[1]);
        mma16816(dp[1], va[kc], f[2], f[3]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int q = q16 + j * 8 + 2 * t;
        const float2 L = *reinterpret_cast<const float2*>(Ls + q), D = *reinterpret_cast<const float2*>(Ds + q);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qe = q + (e & 1);
          const float pv = qe < T ? exp2f(s[j][e] * c - ((e & 1) ? L.y : L.x)) : 0.f;
          s[j][e] = pv;
          dp[j][e] = pv * (dp[j][e] - ((e & 1) ? D.y : D.x));
        }
      }
      uint32_t pa[4], sa[4];
      acc_to_a(pa, s[0], s[1]);
      acc_to_a(sa, dp[0], dp[1]);
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {  // dO and Q read transposed by ldmatrix.trans
        uint32_t f[4];
        ldsm4t(f, frag_a(dOs, q16, 2 * n2, lane));
        mma16816(dv[2 * n2], pa, f[0], f[1]);
        mma16816(dv[2 * n2 + 1], pa, f[2], f[3]);
        ldsm4t(f, frag_a(Qs, q16, 2 * n2, lane));
        mma16816(dk[2 * n2], sa, f[0], f[1]);
        mma16816(dk[2 * n2 + 1], sa, f[2], f[3]);
      }
    }
    const int k0 = kt * 16 + g, k1 = k0 + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = h * 64 + j * 8 + 2 * t;
      if (k0 < T) {
        __half* row = p.gqkv + (size_t)(b * T + k0) * ld3 + col;
        *reinterpret_cast<uint32_t*>(row + W) = pack(dk[j][0] * p.scale, dk[j][1] * p.scale);
        *reinterpret_cast<uint32_t*>(row + 2 * W) = pack(dv[j][0], dv[j][1]);
      }
      if (k1 < T) {
        __half* row = p.gqkv + (size_t)(b * T + k1) * ld3 + col;
        *reinterpret_cast<uint32_t*>(row + W) = pack(dk[j][2] * p.scale, dk[j][3] * p.scale);
        *reinterpret_cast<uint32_t*>(row + 2 * W) = pack(dv[j][2], dv[j][3]);
      }
    }
  }

  for (int qt = lo + warp; qt < hi; qt += AT_WARPS) {  // phase 2: dQ of 16 queries
    uint32_t qa[4][4], da[4][4];
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      ldsm4(qa[kc], frag_a(Qs, qt * 16, 2 * kc, lane));
      ldsm4(da[kc], frag_a(dOs, qt * 16, 2 * kc, lane));
    }
    const int r0 = qt * 16 + g;
    const float L0 = Ls[r0], L1 = Ls[r0 + 8], D0 = Ds[r0], D1 = Ds[r0 + 8];
    float dq[8][4] = {};
    for (int k16 = 0; k16 < TP; k16 += 16) {
      float s[2][4] = {}, dp[2][4] = {};
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        uint32_t f[4];
        ldsm4(f, frag_b(Ks, k16, 2 * kc, lane));
        mma16816(s[0], qa[kc], f[0], f[1]);
        mma16816(s[1], qa[kc], f[2], f[3]);
        ldsm4(f, frag_b(Vs, k16, 2 * kc, lane));
        mma16816(dp[0], da[kc], f[0], f[1]);
        mma16816(dp[1], da[kc], f[2], f[3]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = k16 + j * 8 + 2 * t + (e & 1);
          const float pv = key < T ? exp2f(s[j][e] * c - (e < 2 ? L0 : L1)) : 0.f;
          s[j][e] = pv * (dp[j][e] - (e < 2 ? D0 : D1));
        }
      uint32_t a[4];
      acc_to_a(a, s[0], s[1]);
#pragma unroll
      for (int n2 = 0; n2 < 4; ++n2) {  // K read transposed by ldmatrix.trans
        uint32_t f[4];
        ldsm4t(f, frag_a(Ks, k16, 2 * n2, lane));
        mma16816(dq[2 * n2], a, f[0], f[1]);
        mma16816(dq[2 * n2 + 1], a, f[2], f[3]);
      }
    }
    const int q0 = r0, q1 = r0 + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = h * 64 + j * 8 + 2 * t;
      if (q0 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + q0) * ld3 + col) = pack(dq[j][0] * p.scale, dq[j][1] * p.scale);
      if (q1 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + q1) * ld3 + col) = pack(dq[j][2] * p.scale, dq[j][3] * p.scale);
    }
  }
}

int round16(int T) { return (T + 15) & ~15; }
int tiles_per_split(int T, int splits) { return (round16(T) / 16 + splits - 1) / splits; }
int fwd_smem(int T, int splits) { return (2 * round16(T) + 16 * tiles_per_split(T, splits)) * ROW_BYTES; }
int bwd_smem(int T) { return 4 * round16(T) * ROW_BYTES + 2 * round16(T) * 4; }

}  // namespace

bool attn_supported(int T, int head_dim, int W) { return head_dim == 64 && T >= 1 && T <= 240 && W % 64 == 0; }

int attn_plan_make(AttnPlan* plan, const __half* qkv, __half* o, const __half* d_o, __half* gqkv, float* lse, int B,
                   int T, int H, int W, float scale, int num_sms, char* err, int errlen) {
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
  // One CTA per (image, head) pair stages the pair once.  With fewer pairs than SMs, the pair's 16-row tiles are split
  // over up to num_sms / pairs CTAs (each stages the pair again) so that every SM gets work.
  const long pairs = (long)B * H;
  const int sms = num_sms > 0 ? num_sms : 1, NT = round16(T) / 16;
  const int want = (int)std::min<long>(NT, std::max<long>(1, (sms + pairs - 1) / pairs));
  plan->splits = (NT + tiles_per_split(T, want) - 1) / tiles_per_split(T, want);  // no CTA without a tile
  plan->smem_fwd = fwd_smem(T, plan->splits);
  plan->smem_bwd = bwd_smem(T);
  const double tt = (double)T * T * 64 * 2 * B * H;
  plan->flops_fwd = 2 * tt;  // QK^T, PV
  plan->flops_bwd = 4 * tt;  // dP, dQ, dK, dV (the recomputed S is not algorithmic work)
  const double mw = (double)B * T * W * 2.0;  // one [B*T, W] fp16 tensor
  plan->bytes_fwd = 3 * mw + mw + 4.0 * B * H * T;
  plan->bytes_bwd = 3 * mw + mw + mw + 3 * mw + 4.0 * B * H * T;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, fwd_smem(240, 1));
    cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bwd_smem(240));
  });
  return 0;
}

void attn_forward_launch(const AttnPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  launch_pdl(attn_fwd_kernel, dim3(plan.splits, p.H, p.B), dim3(AT_THREADS), plan.smem_fwd, st, p);
}

void attn_backward_launch(const AttnPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  launch_pdl(attn_bwd_kernel, dim3(plan.splits, p.H, p.B), dim3(AT_THREADS), plan.smem_bwd, st, p);
}

}  // namespace pxr
