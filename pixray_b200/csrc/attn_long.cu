// See attn_long.cuh.  sm_90a: tensor-core mma.sync m16n8k16 (fp16 x fp16 -> fp32); 64-row tiles streamed into shared
// memory by cp.async (two buffers: tile k + 1 loads while tile k is multiplied) and fed to the MMAs by ldmatrix.
#include "attn_long.cuh"
#include "attn_frag.cuh"
#include "launch.cuh"
#include <cmath>
#include <cstdio>
#include <mutex>

namespace pxr {
namespace {

using namespace attn_frag;

constexpr int TILE = 64;                      // rows of a streamed tile
constexpr int TILE_BYTES = TILE * ROW_BYTES;  // 8 KiB
constexpr int FWD_WARPS = 4;                  // forward: 32 query rows per warp
constexpr int FWD_ROWS = 32 * FWD_WARPS;
constexpr int BWD_WARPS = 8;                  // backward: 16 rows (queries / keys) per warp
constexpr int BWD_ROWS = 16 * BWD_WARPS;

// tile rows [0, n) <- 64 columns of rows [r0, r0 + n) of one image's [T, ld] slice at src; zeros past T
template <int NT>
__device__ __forceinline__ void stage_rows(uint32_t tile, const __half* src, int ld, int r0, int n, int T) {
  for (int i = threadIdx.x; i < n * 8; i += NT) {
    const int r = i >> 3, c = i & 7, row = r0 + r;
    const __half* g = src + (size_t)(row < T ? row : 0) * ld + c * 8;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(tile + swz(r, c)), "l"(g), "r"(row < T ? 16 : 0)
                 : "memory");
  }
}
// n floats src[r0 .. r0 + n) -> dst (shared byte address); zeros past T
template <int NT>
__device__ __forceinline__ void stage_f32(uint32_t dst, const float* src, int r0, int n, int T) {
  for (int i = threadIdx.x; i < n; i += NT) {
    const int row = r0 + i;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + 4 * i), "l"(src + (row < T ? row : 0)),
                 "r"(row < T ? 4 : 0)
                 : "memory");
  }
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------------------------ forward
// CTA = (128 query rows, head, image).  Shared memory: Q [128][64], then two buffers of K [64][64] | V [64][64].
// Warp w owns query rows 32 w .. 32 w + 31 of the block as two 16-row MMA tiles; every K / V fragment it loads feeds
// both.  Key chunks of 16 past T do no MMA work; keys past T inside a chunk are masked to -inf.
__global__ void __launch_bounds__(32 * FWD_WARPS, 2) attn_long_fwd_kernel(const __grid_constant__ AttnParams p) {
  pdl_prologue();
  extern __shared__ uint4 smem_al[];
  const int h = blockIdx.y, b = blockIdx.z, q0 = blockIdx.x * FWD_ROWS;
  const int T = p.T, ld3 = 3 * p.W, nkb = (T + TILE - 1) / TILE;
  const uint32_t Qs = smem_u32(smem_al), KV = Qs + FWD_ROWS * ROW_BYTES;
  const __half* base = p.qkv + (size_t)b * T * ld3 + h * 64;
  stage_rows<32 * FWD_WARPS>(Qs, base, ld3, q0, FWD_ROWS, T);
  stage_rows<32 * FWD_WARPS>(KV, base + p.W, ld3, 0, TILE, T);
  stage_rows<32 * FWD_WARPS>(KV + TILE_BYTES, base + 2 * p.W, ld3, 0, TILE, T);
  cp_commit();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bool active = q0 + warp * 32 < T;
  const float c = p.scale * LOG2E;
  uint32_t qa[2][4][4];
  float o[2][8][4] = {};
  float m[2][2] = {{-INFINITY, -INFINITY}, {-INFINITY, -INFINITY}}, l[2][2] = {};
  for (int kb = 0; kb < nkb; ++kb) {
    if (kb + 1 < nkb) {
      const uint32_t nxt = KV + ((kb + 1) & 1) * 2 * TILE_BYTES;
      stage_rows<32 * FWD_WARPS>(nxt, base + p.W, ld3, (kb + 1) * TILE, TILE, T);
      stage_rows<32 * FWD_WARPS>(nxt + TILE_BYTES, base + 2 * p.W, ld3, (kb + 1) * TILE, TILE, T);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (kb == 0) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) ldsm4(qa[mt][kc], frag_a(Qs, warp * 32 + mt * 16, 2 * kc, lane));
      }
      const uint32_t Ks = KV + (kb & 1) * 2 * TILE_BYTES, Vs = Ks + TILE_BYTES;
      const int k0 = kb * TILE;
      float s[2][8][4] = {};
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 keys
        if (k0 + j2 * 16 >= T) break;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          uint32_t kf[4];
          ldsm4(kf, frag_b(Ks, j2 * 16, 2 * kc, lane));
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma16816(s[mt][2 * j2], qa[mt][kc], kf[0], kf[1]);
            mma16816(s[mt][2 * j2 + 1], qa[mt][kc], kf[2], kf[3]);
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int key = k0 + j * 8 + 2 * t + (e & 1);
            s[mt][j][e] = key < T ? s[mt][j][e] * c : -INFINITY;
            if (e < 2) x0 = fmaxf(x0, s[mt][j][e]);
            else x1 = fmaxf(x1, s[mt][j][e]);
          }
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
          x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, off));
          x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, off));
        }
        const float n0 = fmaxf(m[mt][0], x0), n1 = fmaxf(m[mt][1], x1);  // every key tile holds a key < T: finite
        const float a0 = exp2f(m[mt][0] - n0), a1 = exp2f(m[mt][1] - n1);
        m[mt][0] = n0;
        m[mt][1] = n1;
        l[mt][0] *= a0;
        l[mt][1] *= a1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s[mt][j][0] = exp2f(s[mt][j][0] - n0);
          s[mt][j][1] = exp2f(s[mt][j][1] - n0);
          s[mt][j][2] = exp2f(s[mt][j][2] - n1);
          s[mt][j][3] = exp2f(s[mt][j][3] - n1);
          l[mt][0] += s[mt][j][0] + s[mt][j][1];
          l[mt][1] += s[mt][j][2] + s[mt][j][3];
          o[mt][j][0] *= a0;
          o[mt][j][1] *= a0;
          o[mt][j][2] *= a1;
          o[mt][j][3] *= a1;
        }
      }
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 keys: O += P V, V read transposed by ldmatrix.trans
        if (k0 + j2 * 16 >= T) break;
        uint32_t pa[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) acc_to_a(pa[mt], s[mt][2 * j2], s[mt][2 * j2 + 1]);
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t vf[4];
          ldsm4t(vf, frag_a(Vs, j2 * 16, 2 * n2, lane));
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma16816(o[mt][2 * n2], pa[mt], vf[0], vf[1]);
            mma16816(o[mt][2 * n2 + 1], pa[mt], vf[2], vf[3]);
          }
        }
      }
    }
    __syncthreads();  // the buffer just read is the one the next iteration refills
  }
  if (!active) return;
  float* lse = p.lse + (size_t)(b * p.H + h) * T;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    float l0 = l[mt][0], l1 = l[mt][1];
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, off);
      l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    const int r0 = q0 + warp * 32 + mt * 16 + g, r1 = r0 + 8;
    const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = h * 64 + j * 8 + 2 * t;
      if (r0 < T) *reinterpret_cast<uint32_t*>(p.o + (size_t)(b * T + r0) * p.W + col) = pack(o[mt][j][0] * i0, o[mt][j][1] * i0);
      if (r1 < T) *reinterpret_cast<uint32_t*>(p.o + (size_t)(b * T + r1) * p.W + col) = pack(o[mt][j][2] * i1, o[mt][j][3] * i1);
    }
    if (t == 0) {
      if (r0 < T) lse[r0] = (m[mt][0] + log2f(l0)) * LN2;
      if (r1 < T) lse[r1] = (m[mt][1] + log2f(l1)) * LN2;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ backward
// dQ: CTA = (128 query rows, head, image).  Shared memory: Q [128][64], dO [128][64], lse log2(e) and D of the 128
// rows, then two buffers of K | V.  D_i = dO_i . O_i is formed here (8 adjacent lanes per row, shuffle-reduced) and
// also stored to `delta` for the dK / dV kernel.  Warp w owns query rows 16 w .. 16 w + 15 and runs over 16-key chunks:
// S = Q K^T, dP = dO V^T, dS = P o (dP - D), dQ += dS K (K read transposed by ldmatrix.trans).
__global__ void __launch_bounds__(32 * BWD_WARPS, 2) attn_long_dq_kernel(const __grid_constant__ AttnParams p,
                                                                         float* delta) {
  pdl_prologue();
  extern __shared__ uint4 smem_al[];
  const int h = blockIdx.y, b = blockIdx.z, q0 = blockIdx.x * BWD_ROWS;
  const int T = p.T, W = p.W, ld3 = 3 * W, nkb = (T + TILE - 1) / TILE;
  const uint32_t Qs = smem_u32(smem_al), dOs = Qs + BWD_ROWS * ROW_BYTES, KV = dOs + BWD_ROWS * ROW_BYTES;
  float* Ls = reinterpret_cast<float*>(reinterpret_cast<char*>(smem_al) + 2 * BWD_ROWS * ROW_BYTES + 4 * TILE_BYTES);
  float* Ds = Ls + BWD_ROWS;
  const __half* base = p.qkv + (size_t)b * T * ld3 + h * 64;
  const __half* dob = p.d_o + (size_t)b * T * W + h * 64;
  constexpr int NT = 32 * BWD_WARPS;
  stage_rows<NT>(Qs, base, ld3, q0, BWD_ROWS, T);
  stage_rows<NT>(dOs, dob, W, q0, BWD_ROWS, T);
  stage_rows<NT>(KV, base + W, ld3, 0, TILE, T);
  stage_rows<NT>(KV + TILE_BYTES, base + 2 * W, ld3, 0, TILE, T);
  cp_commit();
  const size_t pair = (size_t)(b * p.H + h) * T;
  for (int i = threadIdx.x; i < BWD_ROWS * 8; i += NT) {  // the 8 lanes of a row are adjacent: shuffle-reduce
    const int r = i >> 3, row = q0 + r, cc = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0), ov = make_uint4(0, 0, 0, 0);
    if (row < T) {
      const size_t off = (size_t)(b * T + row) * W + h * 64 + cc;
      v = *reinterpret_cast<const uint4*>(p.d_o + off);
      ov = *reinterpret_cast<const uint4*>(p.o + off);
    }
    const __half* hv = reinterpret_cast<const __half*>(&v);
    const __half* ho = reinterpret_cast<const __half*>(&ov);
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) d += __half2float(hv[j]) * __half2float(ho[j]);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 4);
    if ((i & 7) == 0) {
      Ds[r] = d;
      Ls[r] = row < T ? p.lse[pair + row] * LOG2E : 0.f;
      if (row < T) delta[pair + row] = d;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bool active = q0 + warp * 16 < T;
  const float c = p.scale * LOG2E;
  uint32_t qa[4][4], da[4][4];
  float L0 = 0.f, L1 = 0.f, D0 = 0.f, D1 = 0.f;
  float dq[8][4] = {};
  for (int kb = 0; kb < nkb; ++kb) {
    if (kb + 1 < nkb) {
      const uint32_t nxt = KV + ((kb + 1) & 1) * 2 * TILE_BYTES;
      stage_rows<NT>(nxt, base + W, ld3, (kb + 1) * TILE, TILE, T);
      stage_rows<NT>(nxt + TILE_BYTES, base + 2 * W, ld3, (kb + 1) * TILE, TILE, T);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (kb == 0) {
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          ldsm4(qa[kc], frag_a(Qs, warp * 16, 2 * kc, lane));
          ldsm4(da[kc], frag_a(dOs, warp * 16, 2 * kc, lane));
        }
        const int r = warp * 16 + g;
        L0 = Ls[r];
        L1 = Ls[r + 8];
        D0 = Ds[r];
        D1 = Ds[r + 8];
      }
      const uint32_t Ks = KV + (kb & 1) * 2 * TILE_BYTES, Vs = Ks + TILE_BYTES;
      const int k0 = kb * TILE;
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 keys
        if (k0 + j2 * 16 >= T) break;
        float s[2][4] = {}, dp[2][4] = {};
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          uint32_t f[4];
          ldsm4(f, frag_b(Ks, j2 * 16, 2 * kc, lane));
          mma16816(s[0], qa[kc], f[0], f[1]);
          mma16816(s[1], qa[kc], f[2], f[3]);
          ldsm4(f, frag_b(Vs, j2 * 16, 2 * kc, lane));
          mma16816(dp[0], da[kc], f[0], f[1]);
          mma16816(dp[1], da[kc], f[2], f[3]);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int key = k0 + j2 * 16 + j * 8 + 2 * t + (e & 1);
            const float pv = key < T ? exp2f(s[j][e] * c - (e < 2 ? L0 : L1)) : 0.f;
            s[j][e] = pv * (dp[j][e] - (e < 2 ? D0 : D1));
          }
        uint32_t a[4];
        acc_to_a(a, s[0], s[1]);
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t f[4];
          ldsm4t(f, frag_a(Ks, j2 * 16, 2 * n2, lane));
          mma16816(dq[2 * n2], a, f[0], f[1]);
          mma16816(dq[2 * n2 + 1], a, f[2], f[3]);
        }
      }
    }
    __syncthreads();
  }
  if (!active) return;
  const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = h * 64 + j * 8 + 2 * t;
    if (r0 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + r0) * ld3 + col) = pack(dq[j][0] * p.scale, dq[j][1] * p.scale);
    if (r1 < T) *reinterpret_cast<uint32_t*>(p.gqkv + (size_t)(b * T + r1) * ld3 + col) = pack(dq[j][2] * p.scale, dq[j][3] * p.scale);
  }
}

// dK / dV: CTA = (128 key rows, head, image).  Shared memory: K [128][64], V [128][64], then two buffers of
// Q [64][64] | dO [64][64] | lse [64] | D [64] of a 64-query chunk.  Warp w owns key rows 16 w .. 16 w + 15 and runs
// over 16-query chunks of the transposed scores S^T = K Q^T, dP^T = V dO^T: dV += P^T dO, dK += dS^T Q (dO and Q read
// transposed by ldmatrix.trans).
constexpr int CHUNK_BYTES = 2 * TILE_BYTES + 2 * TILE * 4;  // Q | dO | lse | D

__global__ void __launch_bounds__(32 * BWD_WARPS, 2) attn_long_dkv_kernel(const __grid_constant__ AttnParams p,
                                                                          const float* delta) {
  pdl_prologue();
  extern __shared__ uint4 smem_al[];
  const int h = blockIdx.y, b = blockIdx.z, k0 = blockIdx.x * BWD_ROWS;
  const int T = p.T, W = p.W, ld3 = 3 * W, nqb = (T + TILE - 1) / TILE;
  const uint32_t Ks = smem_u32(smem_al), Vs = Ks + BWD_ROWS * ROW_BYTES, CH = Vs + BWD_ROWS * ROW_BYTES;
  const float* chunk_f = reinterpret_cast<const float*>(reinterpret_cast<const char*>(smem_al) + 2 * BWD_ROWS * ROW_BYTES +
                                                        2 * TILE_BYTES);
  const __half* base = p.qkv + (size_t)b * T * ld3 + h * 64;
  const __half* dob = p.d_o + (size_t)b * T * W + h * 64;
  const size_t pair = (size_t)(b * p.H + h) * T;
  constexpr int NT = 32 * BWD_WARPS;
  auto stage_chunk = [&](int buf, int r0) {
    const uint32_t ch = CH + buf * CHUNK_BYTES;
    stage_rows<NT>(ch, base, ld3, r0, TILE, T);
    stage_rows<NT>(ch + TILE_BYTES, dob, W, r0, TILE, T);
    stage_f32<NT>(ch + 2 * TILE_BYTES, p.lse + pair, r0, TILE, T);
    stage_f32<NT>(ch + 2 * TILE_BYTES + TILE * 4, delta + pair, r0, TILE, T);
  };
  stage_rows<NT>(Ks, base + W, ld3, k0, BWD_ROWS, T);
  stage_rows<NT>(Vs, base + 2 * W, ld3, k0, BWD_ROWS, T);
  stage_chunk(0, 0);
  cp_commit();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bool active = k0 + warp * 16 < T;
  const float c = p.scale * LOG2E;
  uint32_t ka[4][4], va[4][4];
  float dk[8][4] = {}, dv[8][4] = {};
  for (int qb = 0; qb < nqb; ++qb) {
    if (qb + 1 < nqb) {
      stage_chunk((qb + 1) & 1, (qb + 1) * TILE);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (qb == 0) {
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          ldsm4(ka[kc], frag_a(Ks, warp * 16, 2 * kc, lane));
          ldsm4(va[kc], frag_a(Vs, warp * 16, 2 * kc, lane));
        }
      }
      const uint32_t Qc = CH + (qb & 1) * CHUNK_BYTES, dOc = Qc + TILE_BYTES;
      const float* Lc = chunk_f + (qb & 1) * (CHUNK_BYTES / 4);
      const float* Dc = Lc + TILE;
      const int qbase = qb * TILE;
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {  // 16 queries
        if (qbase + j2 * 16 >= T) break;
        float s[2][4] = {}, dp[2][4] = {};
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          uint32_t f[4];
          ldsm4(f, frag_b(Qc, j2 * 16, 2 * kc, lane));
          mma16816(s[0], ka[kc], f[0], f[1]);
          mma16816(s[1], ka[kc], f[2], f[3]);
          ldsm4(f, frag_b(dOc, j2 * 16, 2 * kc, lane));
          mma16816(dp[0], va[kc], f[0], f[1]);
          mma16816(dp[1], va[kc], f[2], f[3]);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int ql = j2 * 16 + j * 8 + 2 * t;  // query of column e & 1 = 0, local to the chunk
          const float2 L = *reinterpret_cast<const float2*>(Lc + ql), D = *reinterpret_cast<const float2*>(Dc + ql);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int qe = qbase + ql + (e & 1);
            const float pv = qe < T ? exp2f(s[j][e] * c - ((e & 1) ? L.y : L.x) * LOG2E) : 0.f;
            s[j][e] = pv;
            dp[j][e] = pv * (dp[j][e] - ((e & 1) ? D.y : D.x));
          }
        }
        uint32_t pa[4], sa[4];
        acc_to_a(pa, s[0], s[1]);
        acc_to_a(sa, dp[0], dp[1]);
#pragma unroll
        for (int n2 = 0; n2 < 4; ++n2) {
          uint32_t f[4];
          ldsm4t(f, frag_a(dOc, j2 * 16, 2 * n2, lane));
          mma16816(dv[2 * n2], pa, f[0], f[1]);
          mma16816(dv[2 * n2 + 1], pa, f[2], f[3]);
          ldsm4t(f, frag_a(Qc, j2 * 16, 2 * n2, lane));
          mma16816(dk[2 * n2], sa, f[0], f[1]);
          mma16816(dk[2 * n2 + 1], sa, f[2], f[3]);
        }
      }
    }
    __syncthreads();
  }
  if (!active) return;
  const int r0 = k0 + warp * 16 + g, r1 = r0 + 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = h * 64 + j * 8 + 2 * t;
    if (r0 < T) {
      __half* row = p.gqkv + (size_t)(b * T + r0) * ld3 + col;
      *reinterpret_cast<uint32_t*>(row + W) = pack(dk[j][0] * p.scale, dk[j][1] * p.scale);
      *reinterpret_cast<uint32_t*>(row + 2 * W) = pack(dv[j][0], dv[j][1]);
    }
    if (r1 < T) {
      __half* row = p.gqkv + (size_t)(b * T + r1) * ld3 + col;
      *reinterpret_cast<uint32_t*>(row + W) = pack(dk[j][2] * p.scale, dk[j][3] * p.scale);
      *reinterpret_cast<uint32_t*>(row + 2 * W) = pack(dv[j][2], dv[j][3]);
    }
  }
}

constexpr int FWD_SMEM = FWD_ROWS * ROW_BYTES + 4 * TILE_BYTES;
constexpr int DQ_SMEM = 2 * BWD_ROWS * ROW_BYTES + 4 * TILE_BYTES + 2 * BWD_ROWS * 4;
constexpr int DKV_SMEM = 2 * BWD_ROWS * ROW_BYTES + 2 * CHUNK_BYTES;

}  // namespace

bool attn_long_supported(int T, int head_dim, int W) { return head_dim == 64 && T >= 1 && W % 64 == 0; }

int attn_long_plan_make(AttnLongPlan* plan, const __half* qkv, __half* o, const __half* d_o, __half* gqkv, float* lse,
                        float* delta, int B, int T, int H, int W, float scale, char* err, int errlen) {
  *plan = AttnLongPlan{};
  if (H < 1 || W % H || !attn_long_supported(T, W / H, W) || W != 64 * H || B < 1 || B > 65535 || H > 65535) {
    if (err && errlen > 0) snprintf(err, errlen, "streaming attention needs 64-wide heads (got W=%d over H=%d), T >= 1", W, H);
    return -1;
  }
  if (d_o && !delta) {
    if (err && errlen > 0) snprintf(err, errlen, "streaming attention backward needs a [B*H*T] delta workspace");
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
  plan->delta = delta;
  const double tt = (double)T * T * 64 * 2 * B * H;
  plan->flops_fwd = 2 * tt;  // QK^T, PV
  plan->flops_bwd = 4 * tt;  // dP, dQ, dK, dV (the recomputed S, and the second dP, are not algorithmic work)
  const double mw = (double)B * T * W * 2.0;  // one [B*T, W] fp16 tensor
  plan->bytes_fwd = 3 * mw + mw + 4.0 * B * H * T;
  plan->bytes_bwd = 3 * mw + mw + mw + 3 * mw + 4.0 * B * H * T;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncSetAttribute(attn_long_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM);
    cudaFuncSetAttribute(attn_long_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM);
    cudaFuncSetAttribute(attn_long_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DKV_SMEM);
  });
  return 0;
}

void attn_long_forward_launch(const AttnLongPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  launch_pdl(attn_long_fwd_kernel, dim3((p.T + FWD_ROWS - 1) / FWD_ROWS, p.H, p.B), dim3(32 * FWD_WARPS), FWD_SMEM, st, p);
}

// dQ first: it forms D for the dK / dV kernel
void attn_long_backward_launch(const AttnLongPlan& plan, cudaStream_t st) {
  const AttnParams& p = plan.p;
  const dim3 grid((p.T + BWD_ROWS - 1) / BWD_ROWS, p.H, p.B);
  launch_pdl(attn_long_dq_kernel, grid, dim3(32 * BWD_WARPS), DQ_SMEM, st, p, plan.delta);
  launch_pdl(attn_long_dkv_kernel, grid, dim3(32 * BWD_WARPS), DKV_SMEM, st, p, static_cast<const float*>(plan.delta));
}

}  // namespace pxr
