// See gemm_tc.cuh for the contract.  sm_90a only (wgmma + TMA + mbarrier).
#include "gemm_tc.cuh"
#include "launch.cuh"
#include "ptx.cuh"
#include <cstdio>
#include <cstring>
#include <mutex>

namespace pxr {
using namespace ptx;

namespace {

constexpr uint32_t A_TILE_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;  // 16 KiB
constexpr uint32_t MN_ATOM_BYTES = 64 * GEMM_BLOCK_K * 2;           // one 64(MN) x 64(K) MN-major TMA box

struct TileCoord {
  int tn, tm, z, b0, b1, n0, m0, h0, w0;
};

__device__ __forceinline__ TileCoord make_coord(const GemmParams& p, int tn, int tm, int z) {
  TileCoord t;
  t.tn = tn;
  t.tm = tm;
  t.z = z;
  t.b0 = z % p.nb0;
  t.b1 = z / p.nb0;
  t.n0 = tn * p.block_n;
  t.m0 = tm * GEMM_BLOCK_M;
  t.h0 = 0;
  t.w0 = 0;
  if (p.a_mode == OP_CONV) {
    t.h0 = (tm / p.tiles_w) * p.tile_h;
    t.w0 = (tm % p.tiles_w) * p.tile_w;
  }
  return t;
}

__device__ __forceinline__ TileCoord decode_tile(const GemmParams& p, int tile) {
  TileCoord t;
  t.tn = tile % p.tiles_n;
  int r = tile / p.tiles_n;
  t.tm = r % p.tiles_m;
  t.z = r / p.tiles_m;
  t.b0 = t.z % p.nb0;
  t.b1 = t.z / p.nb0;
  t.n0 = t.tn * p.block_n;
  t.m0 = t.tm * GEMM_BLOCK_M;
  t.h0 = 0;
  t.w0 = 0;
  if (p.a_mode == OP_CONV) {
    t.h0 = (t.tm / p.tiles_w) * p.tile_h;
    t.w0 = (t.tm % p.tiles_w) * p.tile_w;
  }
  return t;
}

__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float quickgelu(float x) { return x * fast_sigmoid(1.702f * x); }
__device__ __forceinline__ float quickgelu_grad(float u) {
  float s = fast_sigmoid(1.702f * u);
  return s * (1.f + 1.702f * u * (1.f - s));
}
// exact GELU (nn.GELU(): u Phi(u) = 0.5 u (1 + erf(u / sqrt 2))) and its derivative Phi(u) + u phi(u), in fp32 -- no
// tanh form.  Phi(u) = 0.5 erfc(-u / sqrt 2): 1 + erff cancels for u < -4 (erf -> -1), where gelu(u) is an fp16 subnormal
// and the fp32 cancellation error exceeds its ulp; erfcf keeps the relative accuracy there.
__device__ __forceinline__ float gelu_phi(float u) { return 0.5f * erfcf(u * -0.70710678118654752f); }
__device__ __forceinline__ float gelu_erf(float u) { return u * gelu_phi(u); }
__device__ __forceinline__ float gelu_erf_grad(float u) {
  return gelu_phi(u) + u * 0.39894228040143268f * expf(-0.5f * u * u);
}

constexpr int TB_LD = 33;                       // transposer row pitch (floats): conflict-free both ways
constexpr int TB_FLOATS = 32 * TB_LD;           // one 32 x 32 block per epilogue warp
constexpr int TB_WARP_BYTES = TB_FLOATS * 4 + 32 * 8 + 32 * 4;  // + per-row offset / row-index tables
constexpr int GEMM_EPI_WARPS = 8;

// Row <-> column layout exchange through the warp-private smem block.
//   row layout   : thread = accumulator row, registers = columns                 (one row of the staged tile)
//   store layout : lane = (row_sub, 16-byte chunk of the row)                    (what coalesced global access wants)
struct RowInfo {
  long long off;  // element offset of this thread's row in the output tensors, -1 if the row is out of range
  int row;        // logical row index (bias_per_row)
};

__device__ __forceinline__ RowInfo row_info(const GemmParams& p, const TileCoord& t, int r_tile) {
  RowInfo ri;
  bool valid;
  if (p.a_mode == OP_CONV) {
    const int h = t.h0 + r_tile / p.tile_w, w = t.w0 + r_tile % p.tile_w;
    valid = (h < p.conv_H) && (w < p.conv_W);
    ri.row = h * p.conv_W + w;
    ri.off = (static_cast<long long>(t.z) * p.conv_H * p.conv_W + ri.row) * p.ldc;
  } else {
    ri.row = t.m0 + r_tile;
    valid = ri.row < p.M;
    ri.off = t.b0 * p.out_bs0 + t.b1 * p.out_bs1 + static_cast<long long>(ri.row) * p.ldc;
  }
  if (!valid) ri.off = -1;
  return ri;
}

// Load `width` (16 or 32) accumulator columns of this thread's row of the staged tile (shared memory, 16-byte aligned).
__device__ __forceinline__ void load_acc(const float* src, int width, float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 f = (j < 4 || width > 16) ? reinterpret_cast<const float4*>(src)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    v[4 * j] = f.x;
    v[4 * j + 1] = f.y;
    v[4 * j + 2] = f.z;
    v[4 * j + 3] = f.w;
  }
}

template <int E>
__device__ __forceinline__ void ld_f16(const __half* p, bool vec, int nv, float (&x)[E]) {
  if (vec) {
    if (E == 8) {
      uint4 u = *reinterpret_cast<const uint4*>(p);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __half22float2(h[j]);
        x[2 * j] = f.x;
        x[2 * j + 1] = f.y;
      }
    } else {
      uint2 u = *reinterpret_cast<const uint2*>(p);
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float2 f = __half22float2(h[j]);
        x[2 * j] = f.x;
        x[2 * j + 1] = f.y;
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < E; ++j) x[j] = (j < nv) ? __half2float(p[j]) : 0.f;
  }
}
template <int E>
__device__ __forceinline__ void st_f16(__half* p, bool vec, int nv, const float (&x)[E]) {
  if (vec) {
    if (E == 8) {
      uint4 u;
      __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
      *reinterpret_cast<uint4*>(p) = u;
    } else {
      uint2 u;
      __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
      for (int j = 0; j < 2; ++j) h[j] = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
      *reinterpret_cast<uint2*>(p) = u;
    }
  } else {
#pragma unroll
    for (int j = 0; j < E; ++j)
      if (j < nv) p[j] = __float2half_rn(x[j]);
  }
}
template <int E>
__device__ __forceinline__ void ld_f32(const float* p, bool vec, int nv, float (&x)[E]) {
  if (vec) {
#pragma unroll
    for (int j = 0; j < E / 4; ++j) {
      float4 f = reinterpret_cast<const float4*>(p)[j];
      x[4 * j] = f.x;
      x[4 * j + 1] = f.y;
      x[4 * j + 2] = f.z;
      x[4 * j + 3] = f.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < E; ++j) x[j] = (j < nv) ? p[j] : 0.f;
  }
}
template <int E>
__device__ __forceinline__ void st_f32(float* p, bool vec, int nv, const float (&x)[E]) {
  if (vec) {
#pragma unroll
    for (int j = 0; j < E / 4; ++j)
      reinterpret_cast<float4*>(p)[j] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
  } else {
#pragma unroll
    for (int j = 0; j < E; ++j)
      if (j < nv) p[j] = x[j];
  }
}

// Geometry of the store layout for E elements per lane (8: all-fp16 tensors, 4: an fp32 tensor takes part).
template <int E>
struct BlockMap {
  static constexpr int CH = 32 / E;    // 16-byte chunks per 32-column row
  static constexpr int RPI = 32 / CH;  // rows covered by one warp instruction
  static constexpr int NIT = 32 / RPI; // iterations per block
};

// Which input tensor (if any) is prefetched for the block: residual fp32, residual fp16 or the saved pre-activation.
__device__ __forceinline__ int prefetch_kind(const GemmParams& p) {
  return p.res_f32 ? 1
                   : (p.res_f16 ? 2
                                : ((p.act == ACT_QUICKGELU_BWD || p.act == ACT_GELU_BWD || p.act == ACT_LRELU_BWD ||
                                    p.act == ACT_RELU_BWD) ? 3 : 0));
}

// Issue the global loads of the block's input tensor BEFORE the accumulator block is read, so their DRAM latency
// overlaps it (a load-use chain per row made the fp32-residual GEMMs latency-bound).
template <int E>
__device__ __forceinline__ void prefetch_block(const GemmParams& p, const long long* s_off, int lane, int col_base,
                                               int col_limit, int kind, uint4 (&pf)[BlockMap<E>::NIT]) {
  using M = BlockMap<E>;
  const int chunk = lane % M::CH, rsub = lane / M::CH;
  const int col = col_base + chunk * E;
  const bool vec = p.vec_ok && (col_limit - col >= E);
  if (!vec || kind == 0) return;
#pragma unroll
  for (int it = 0; it < M::NIT; ++it) {
    const long long off_r = s_off[it * M::RPI + rsub];
    if (off_r < 0) continue;
    const long long o = off_r + col;
    if (kind == 1) {
      if (E == 4) pf[it] = *reinterpret_cast<const uint4*>(p.res_f32 + o);
    } else {
      const __half* src = (kind == 2) ? p.res_f16 : p.aux_in;
      if (E == 8) pf[it] = *reinterpret_cast<const uint4*>(src + o);
      else {
        uint2 u = *reinterpret_cast<const uint2*>(src + o);
        pf[it].x = u.x;
        pf[it].y = u.y;
      }
    }
  }
}

template <int E>
__device__ __forceinline__ void unpack_pf(const uint4& u, int kind, float (&x)[E]) {
  if (kind == 1) {
    x[0] = __uint_as_float(u.x);
    x[1] = __uint_as_float(u.y);
    x[2] = __uint_as_float(u.z);
    x[3] = __uint_as_float(u.w);
  } else {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < E / 2; ++j) {
      float2 f = __half22float2(h[j]);
      x[2 * j] = f.x;
      x[2 * j + 1] = f.y;
    }
  }
}

// Generic epilogue of one staged 32 x 32 block.  E elements per lane: 8 when every tensor is fp16 (16-byte accesses,
// 8 rows per warp instruction), 4 when an fp32 tensor takes part (16-byte accesses on the fp32 side, 4 rows).
// ERF: the kernels that take the exact-GELU codes; the others compile without them (erfcf costs registers and stack).
template <int E, bool ERF>
__device__ __forceinline__ void epilogue_block(const GemmParams& p, const float* tb, int ld, const long long* s_off,
                                               const int* s_row, int lane, int col_base, int col_limit, int kind,
                                               const uint4 (&pf)[BlockMap<E>::NIT]) {
  using M = BlockMap<E>;
  const int chunk = lane % M::CH, rsub = lane / M::CH;
  const int c0 = chunk * E;
  const int col = col_base + c0;
  int nv = col_limit - col;  // col_limit = min(N, end of this tile)
  nv = nv < 0 ? 0 : (nv > E ? E : nv);
  const bool vec = p.vec_ok && nv == E;
  float bias[E];
#pragma unroll
  for (int j = 0; j < E; ++j) bias[j] = (p.bias && !p.bias_per_row && j < nv) ? p.bias[col + j] : 0.f;
  if (nv == 0) return;
#pragma unroll
  for (int it = 0; it < M::NIT; ++it) {
    const int r = it * M::RPI + rsub;
    const long long off_r = s_off[r];
    if (off_r < 0) continue;
    const long long o = off_r + col;
    float x[E];
#pragma unroll
    for (int j = 0; j < E; ++j) x[j] = tb[r * ld + c0 + j] * p.alpha + bias[j];
    if (p.bias && p.bias_per_row) {
      const float b = p.bias[s_row[r]];
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] += b;
    }
    unsigned neg = 0;  // ACT_LRELU_BWD: the masked columns whose saved activation is <= 0 (applied after the residual)
    if (p.act == ACT_LRELU) {
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] = fmaxf(x[j], 0.2f * x[j]);
    } else if (p.act == ACT_LRELU_BWD && col + E > p.act_col0) {
      float u[E];
      if (vec && kind == 3) unpack_pf<E>(pf[it], 3, u);
      else ld_f16<E>(p.aux_in + o, vec, nv, u);
#pragma unroll
      for (int j = 0; j < E; ++j) neg |= (col + j >= p.act_col0 && !(u[j] > 0.f)) ? 1u << j : 0u;
    } else if (p.act == ACT_RELU_BWD) {
      float u[E];
      if (vec && kind == 3) unpack_pf<E>(pf[it], 3, u);
      else ld_f16<E>(p.aux_in + o, vec, nv, u);
#pragma unroll
      for (int j = 0; j < E; ++j) neg |= !(u[j] > 0.f) ? 1u << j : 0u;
    } else if (p.act == ACT_QUICKGELU) {
      if (p.aux_out) st_f16<E>(p.aux_out + o, vec, nv, x);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] = quickgelu(x[j]);
    } else if (p.act == ACT_QUICKGELU_BWD) {
      float u[E];
      if (vec && kind == 3) unpack_pf<E>(pf[it], 3, u);
      else ld_f16<E>(p.aux_in + o, vec, nv, u);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] *= quickgelu_grad(u[j]);
    } else if (ERF && p.act == ACT_GELU) {
      if (p.aux_out) st_f16<E>(p.aux_out + o, vec, nv, x);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] = gelu_erf(__half2float(__float2half_rn(x[j])));  // of the saved fp16 u
    } else if (ERF && p.act == ACT_GELU_BWD) {
      float u[E];
      if (vec && kind == 3) unpack_pf<E>(pf[it], 3, u);
      else ld_f16<E>(p.aux_in + o, vec, nv, u);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] *= gelu_erf_grad(u[j]);
    }
    if (p.res_f32) {
      float t[E];
      if (vec && kind == 1 && E == 4) unpack_pf<E>(pf[it], 1, t);
      else ld_f32<E>(p.res_f32 + o, vec, nv, t);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] += t[j];
    }
    if (p.res_f16) {
      float t[E];
      if (vec && kind == 2) unpack_pf<E>(pf[it], 2, t);
      else ld_f16<E>(p.res_f16 + o, vec, nv, t);
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] += t[j];
    }
    if (neg) {
#pragma unroll
      for (int j = 0; j < E; ++j)
        if (neg & (1u << j)) x[j] = p.act == ACT_RELU_BWD ? 0.f : x[j] * 0.2f;
    }
    if (p.act == ACT_RELU) {
#pragma unroll
      for (int j = 0; j < E; ++j) x[j] = fmaxf(x[j], 0.f);
    }
    if (p.out_f32) st_f32<E>(p.out_f32 + o, vec, nv, x);
    if (p.out_f16) st_f16<E>(p.out_f16 + o, vec, nv, x);
  }
}

// TMA producer (one lane): walks this CTA's tiles and fills the stage ring.
// This single thread paces the whole kernel, so its loop body is kept short: specialised on the operand modes (no runtime
// divisions for the tap / k offset, no mode branches), (tap, kk) carried as running counters, 32-bit shared addresses.
template <int AM, int BM>
__device__ __forceinline__ void producer_tiles(const GemmParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                               uint32_t stage_bytes) {
  const uint32_t smem0 = smem_u32(smem), full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
  const int k_per_tap = p.k_blocks_per_tap * GEMM_BLOCK_K;
  const int n_atoms = p.block_n / 64;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int bb0 = p.b_batched ? t.b0 : 0, bb1 = p.b_batched ? t.b1 : 0;
    const int kb_begin = p.k_splits > 1 ? t.z * p.kb_per_split : 0;
    const int kb_end = p.k_splits > 1 ? min(p.num_k_blocks, kb_begin + p.kb_per_split) : p.num_k_blocks;
    const int img = p.k_splits > 1 ? 0 : t.z;  // split-K: z is the split, there is one image
    const int ab0 = p.k_splits > 1 ? 0 : t.b0, ab1 = p.k_splits > 1 ? 0 : t.b1;  // ... and one (unbatched) A
    int tap = 0, kk = 0, ty = -1, tx = -1;     // running tap index, k offset inside the tap, tap offset (dy, dx)
    if (AM == OP_CONV) {
      tap = kb_begin / p.k_blocks_per_tap;
      kk = (kb_begin - tap * p.k_blocks_per_tap) * GEMM_BLOCK_K;
      if (p.num_taps == 9) {
        ty = tap / 3 - 1;
        tx = tap % 3 - 1;
      } else {
        ty = tx = 0;
      }
    } else {
      kk = kb_begin * GEMM_BLOCK_K;
    }
    int b_row = t.n0 + tap * p.b_tap_rows;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      const uint32_t fb = full0 + stage * 8, sa = smem0 + stage * stage_bytes, sb = sa + A_TILE_BYTES;
      mbar_wait_s(empty0 + stage * 8, phase ^ 1);
      mbar_arrive_expect_tx_s(fb, stage_bytes);
      if (AM == OP_KMAJOR) {
        tma_load_4d_s(&p.tma_a, fb, sa, kk, t.m0, ab0, ab1);
      } else if (AM == OP_MNMAJOR) {
        tma_load_4d_s(&p.tma_a, fb, sa, t.m0, kk, ab0, ab1);
        tma_load_4d_s(&p.tma_a, fb, sa + MN_ATOM_BYTES, t.m0 + 64, kk, ab0, ab1);
      } else {
        tma_load_4d_s(&p.tma_a, fb, sa, kk, t.w0 + tx, t.h0 + ty, img);
      }
      if (BM == OP_KMAJOR) {
        tma_load_4d_s(&p.tma_b, fb, sb, kk, b_row, bb0, bb1);
      } else {
        for (int j = 0; j < n_atoms; ++j)
          tma_load_4d_s(&p.tma_b, fb, sb + j * MN_ATOM_BYTES, t.n0 + 64 * j, kk, bb0, bb1);
      }
      kk += GEMM_BLOCK_K;
      if (AM == OP_CONV && kk == k_per_tap) {  // next filter tap
        kk = 0;
        b_row += p.b_tap_rows;
        if (++tx == 2) {
          tx = -1;
          ++ty;
        }
      }
      if (++stage == p.stages) {
        stage = 0;
        phase ^= 1;
      }
    }
  }
}

__device__ __forceinline__ void producer_loop(const GemmParams& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                              uint32_t stage_bytes) {
  if (p.a_mode == OP_CONV) {
    producer_tiles<OP_CONV, OP_KMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
  } else if (p.a_mode == OP_KMAJOR) {
    if (p.b_mode == OP_KMAJOR) producer_tiles<OP_KMAJOR, OP_KMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
    else producer_tiles<OP_KMAJOR, OP_MNMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
  } else {
    if (p.b_mode == OP_KMAJOR) producer_tiles<OP_MNMAJOR, OP_KMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
    else producer_tiles<OP_MNMAJOR, OP_MNMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
  }
}

// Accumulator of one warpgroup: 64 rows x NCH 64-column wgmma fragments, sized per kernel: NF for the 64- / 128-wide
// fp16 kernels, two for the generic-width kernel (this kernel's tiles are at most 128 wide, so a 16-column tail always lands in the
// first two fragments).
template <int NCH>
struct WgAcc {
  float d[NCH][32];
};
template <int NF>
using AccFor = WgAcc<NF ? NF : 2>;

// MMA warpgroup `wg` (0 or 1: tile rows [64 wg, 64 wg + 64)): wgmma over the k-blocks of one tile.  A k-block is four
// k16 steps; each step issues block_n / 64 m64n64 instructions and, for block_n % 64, up to three m64n16 ones.  The
// shared-memory descriptors are built once; a stage / k-step advance is an add on their address field (bits [0,14) =
// address >> 4, and the whole ring sits below 256 KiB, so the add never carries out of the field).  The stage read by
// k-block kb is released once kb's wgmma group has completed (checked after k-block kb + 1 has been issued).
// NF > 0: fp16 operands and block_n == 64 NF, so every instruction of a k-step is known at compile time and the fragments
// take 32 NF registers (runtime-guarded wgmma or a larger live fragment make ptxas serialise the chain); NF == 0 covers
// every other width and bf16.
template <int TA, int TB, int NF>
__device__ __forceinline__ void mma_tile(const GemmParams& p, AccFor<NF>& acc, int wg, int n_kb, uint32_t smem0, uint32_t full0,
                                         uint64_t* empty_bar, uint32_t stage_bytes, int& stage, uint32_t& phase) {
  // K-major: 8-row groups 1024 B apart, a 64-row slab is 8 KiB; K advance = 32 B inside the swizzled row.
  // MN-major: 64-wide MN atoms 8192 B apart (LBO), 8-deep K groups 1024 B apart (SBO); K advance = 2048 B.
  const uint64_t a_kstep = (TA ? 2048 : 32) >> 4, b_kstep = (TB ? 2048 : 32) >> 4;
  const uint64_t a_desc0 = make_smem_desc_sw128(smem0 + wg * 8192, TA ? MN_ATOM_BYTES : 0, 1024);
  const uint64_t b_desc0 = make_smem_desc_sw128(smem0 + A_TILE_BYTES, TB ? MN_ATOM_BYTES : 0, 1024);
  const uint64_t stage_step = stage_bytes >> 4;
  const int nfull = NF ? NF : p.block_n / 64, ntail = NF ? 0 : (p.block_n % 64) / 16;
  const int bf16 = NF ? 0 : p.fmt;
  constexpr int NCH = NF ? NF : 2;
  const bool elected = (threadIdx.x & 127) == 0;
  int prev = -1;
  for (int kb = 0; kb < n_kb; ++kb) {
    mbar_wait_s(full0 + stage * 8, phase);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = a_desc0 + stage * stage_step + k * a_kstep, bd = b_desc0 + stage * stage_step + k * b_kstep;
      const uint32_t scale_d = (kb | k) ? 1u : 0u;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        if (j < nfull) wgmma_m64n64<TA, TB>(acc.d[j], ad, bd + j * (8192 >> 4), scale_d, bf16);
        if (!NF && j == nfull) {  // 16-column tail (K-major B only: MN-major B tiles are multiples of 64 wide)
#pragma unroll
          for (int t = 0; t < 3; ++t)
            if (t < ntail) wgmma_m64n16<TA, TB>(acc.d[j] + 8 * t, ad, bd + (j * 8192 + t * 2048) / 16, scale_d, bf16);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && elected) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == p.stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  if (prev >= 0 && elected) mbar_arrive(&empty_bar[prev]);
}

// Write this warpgroup's fragments into the staged tile: row-major fp32, row pitch ld floats.
template <int NCH>
__device__ __forceinline__ void dump_acc(const WgAcc<NCH>& acc, float* tile, int ld, int block_n) {
  const int t = threadIdx.x & 127;
  const int r0 = (threadIdx.x >> 7) * 64 + (t >> 5) * 16 + ((t & 31) >> 2), c0 = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = 64 * j + 8 * i + c0;
      if (64 * j + 8 * i < block_n) {
        *reinterpret_cast<float2*>(tile + r0 * ld + c) = make_float2(acc.d[j][4 * i], acc.d[j][4 * i + 1]);
        *reinterpret_cast<float2*>(tile + (r0 + 8) * ld + c) = make_float2(acc.d[j][4 * i + 2], acc.d[j][4 * i + 3]);
      }
    }
  }
}

__device__ __forceinline__ int tile_k_blocks(const GemmParams& p, int tile) {
  if (p.k_splits <= 1) return p.num_k_blocks;
  const int kb_begin = (tile / (p.tiles_m * p.tiles_n)) * p.kb_per_split;
  return min(p.num_k_blocks, kb_begin + p.kb_per_split) - kb_begin;
}

// ------------------------------------------------------------------------------------------------ tensor-map epilogue
// The generic epilogue above is instruction- and latency-bound: every element goes through a row-to-column exchange and
// every input tensor is a dependent global load.
// Here each lane keeps its accumulator ROW: it writes 64 contiguous bytes (32 fp16 / 16 fp32 columns) of that row into a
// 32-row x 64-byte box in shared memory (64B-swizzled, conflict-free), and one lane hands the box to a TMA store.
// Input tensors (residual, saved pre-activation) come in through TMA loads into the same box, two blocks ahead, and the
// result overwrites them in place.  ~2 instructions per element, no dependent global loads, clipping by the tensor map.
constexpr int TE_BUF_BYTES = 2048;  // 32 rows x 64 bytes
constexpr int TE_BUFS = 4;          // boxes per epilogue warp
constexpr int TE_WARP_BYTES = TE_BUFS * TE_BUF_BYTES;
constexpr int TE_BAR_BYTES = 1024;  // barrier block (stage ring, per-warp input barriers)

// byte offset of 16-byte chunk c (0..3) of row r (0..31) in a CU_TENSOR_MAP_SWIZZLE_64B box (chunk ^= address bits 7..8)
__device__ __forceinline__ uint32_t te_off(int r, int c) {
  return static_cast<uint32_t>(r * 64 + ((c ^ ((r >> 1) & 3)) << 4));
}
__device__ __forceinline__ uint4 pack8(const float* x) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
  return u;
}
__device__ __forceinline__ void unpack8(const uint4& u, float* x) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __half22float2(h[j]);
    x[2 * j] = f.x;
    x[2 * j + 1] = f.y;
  }
}

// QuickGELU and its derivative on packed fp16 pairs for the tensor-map epilogue (the fp32 form costs ~8 instructions per
// element with two MUFU ops and makes the fc1 / fc2-dgrad epilogues ALU-bound).  sigmoid(z) = 0.5 tanh(z / 2) + 0.5 with tanh.approx.f16x2: one MUFU per pair.
// The operands are already fp16 here (u is stored as fp16; the reference runs its CLIP in fp16 on CUDA, slip.py:176).
__device__ __forceinline__ __half2 tanh_h2(__half2 x) {
  uint32_t r, a = *reinterpret_cast<uint32_t*>(&x);
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(r) : "r"(a));
  return *reinterpret_cast<__half2*>(&r);
}
__device__ __forceinline__ __half2 sigmoid1702_h2(__half2 u) {
  const __half2 t = tanh_h2(__hmul2(u, __float2half2_rn(0.851f)));
  return __hfma2(t, __float2half2_rn(0.5f), __float2half2_rn(0.5f));
}
__device__ __forceinline__ __half2 quickgelu_h2(__half2 u) { return __hmul2(u, sigmoid1702_h2(u)); }
__device__ __forceinline__ __half2 quickgelu_grad_h2(__half2 u) {
  const __half2 s = sigmoid1702_h2(u);
  const __half2 a = __hmul2(u, __float2half2_rn(1.702f));
  const __half2 b = __hfma2(__hneg2(s), a, a);  // 1.702 u (1 - s)
  return __hfma2(s, b, s);                       // s (1 + 1.702 u (1 - s))
}

// Per-element arithmetic of both tensor-map epilogues (this kernel's and gemm_wide_kernel's), so the two compute the
// same bits: x = acc * alpha, then + bias, each rounded on its own (__fmul_rn / __fadd_rn: FMUL then FADD, never a
// contracted FFMA), then the mode's tail on one column pair.  `in` is the pair of the input tensor (residual or saved
// pre-activation); the forward activations also return the saved fp16 pre-activation in `aux`.
__device__ __forceinline__ float te_scale(float acc, float alpha) { return __fmul_rn(acc, alpha); }
__device__ __forceinline__ float te_add(float x, float b) { return __fadd_rn(x, b); }
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 bits_h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
template <int MODE>
__device__ __forceinline__ uint32_t te_pair(float x0, float x1, uint32_t in, uint32_t& aux) {
  if (MODE == TE_F16) return h2_bits(__floats2half2_rn(x0, x1));
  if (MODE == TE_RES16) {
    const float2 u = __half22float2(bits_h2(in));
    return h2_bits(__floats2half2_rn(te_add(x0, u.x), te_add(x1, u.y)));
  }
  if (MODE == TE_GELU || MODE == TE_ERF_GELU) {  // the saved pre-activation (fp16), and the activation of exactly that value
    const __half2 u = __floats2half2_rn(x0, x1);
    aux = h2_bits(u);
    if (MODE == TE_GELU) return h2_bits(quickgelu_h2(u));
    const float2 v = __half22float2(u);
    return h2_bits(__floats2half2_rn(gelu_erf(v.x), gelu_erf(v.y)));
  }
  if (MODE == TE_GELU_BWD) return h2_bits(__hmul2(__floats2half2_rn(x0, x1), quickgelu_grad_h2(bits_h2(in))));
  // TE_ERF_GELU_BWD: fp32 product, as the generic epilogue forms it
  const float2 v = __half22float2(bits_h2(in));
  return h2_bits(__floats2half2_rn(__fmul_rn(x0, gelu_erf_grad(v.x)), __fmul_rn(x1, gelu_erf_grad(v.y))));
}

// One tile of the tensor-map epilogue for warp `warp` (rows [32 q, 32 q + 32) of the tile, column blocks half, half + 2,
// ...).  `cnt` counts the blocks this warp has processed: box rotation and input-barrier parity.
template <int MODE>
__device__ __forceinline__ void tma_epilogue_tile(const GemmParams& p, const TileCoord& t, uint8_t* wbuf,
                                                  uint64_t* in_bar, const float* arow, int warp, int lane,
                                                  uint32_t& cnt) {
  constexpr bool F32 = (MODE == TE_RES32);
  constexpr bool ACT_FWD = (MODE == TE_GELU || MODE == TE_ERF_GELU);
  constexpr bool ACT_BWD = (MODE == TE_GELU_BWD || MODE == TE_ERF_GELU_BWD);
  constexpr bool IN = (ACT_BWD || MODE == TE_RES32 || MODE == TE_RES16);
  constexpr int BW = F32 ? 16 : 32;  // columns per 64-byte box row
  const int q = warp & 3;            // row quarter of the tile
  const int half = warp >> 2;        // the two warps of a quarter alternate over the column blocks
  {
    // tensor-map coordinates of this warp's 32 rows: (col, row, b0, b1) or, for conv, (col, w, h, image)
    int c1, c2, c3;
    if (p.a_mode == OP_CONV) {
      c1 = t.w0;
      c2 = t.h0 + (q * 32) / p.tile_w;
      c3 = t.z;
    } else {
      c1 = t.m0 + q * 32;
      c2 = t.b0;
      c3 = t.b1;
    }
    // blocks with at least one column inside N; this warp takes s = half, half + 2, ...
    const int ncols = min(p.N - t.n0, p.block_n);
    const int nblk = (ncols + BW - 1) / BW;
    const int my = (nblk - half + 1) / 2;
    if (IN && lane == 0) {
      bulk_wait_group_read<1>();
      for (int j = 0; j < 2 && j < my; ++j) {
        const uint32_t b = (cnt + j) & 3;
        mbar_arrive_expect_tx(&in_bar[b], TE_BUF_BYTES);
        tma_load_4d(&p.tma_d, &in_bar[b], wbuf + b * TE_BUF_BYTES, t.n0 + (half + 2 * j) * BW, c1, c2, c3);
      }
    }
    for (int j = 0; j < my; ++j) {
      const int s = half + 2 * j;
      const int col = t.n0 + s * BW;
      const uint32_t k = cnt + j;
      uint8_t* buf = wbuf + (ACT_FWD ? (k & 1) * 2 : (k & 3)) * TE_BUF_BYTES;
      if (lane == 0) {
        if (IN) {
          if (j + 2 < my) {
            const uint32_t b = (k + 2) & 3;
            bulk_wait_group_read<1>();  // the box's previous store (two blocks back) has drained
            mbar_arrive_expect_tx(&in_bar[b], TE_BUF_BYTES);
            tma_load_4d(&p.tma_d, &in_bar[b], wbuf + b * TE_BUF_BYTES, t.n0 + (s + 4) * BW, c1, c2, c3);
          }
        } else if (ACT_FWD) {
          bulk_wait_group_read<1>();
        } else {
          bulk_wait_group_read<3>();
        }
      }
      __syncwarp();
      // accumulator columns of this row
      float x[BW];
      {
        float a[32];
        load_acc(arow + s * BW, (!F32 && p.block_n - s * BW > 16) ? 32 : 16, a);  // block_n % 32 == 16: last block half wide
#pragma unroll
        for (int i = 0; i < BW; ++i) x[i] = te_scale(a[i], p.alpha);
      }
      if (p.bias) {
        const float4* bp = reinterpret_cast<const float4*>(p.bias + col);
#pragma unroll
        for (int i = 0; i < BW / 4; ++i) {
          const float4 b = __ldg(bp + i);
          x[4 * i] = te_add(x[4 * i], b.x);
          x[4 * i + 1] = te_add(x[4 * i + 1], b.y);
          x[4 * i + 2] = te_add(x[4 * i + 2], b.z);
          x[4 * i + 3] = te_add(x[4 * i + 3], b.w);
        }
      }
      if (IN) mbar_wait(&in_bar[k & 3], (k >> 2) & 1);
      if constexpr (MODE == TE_RES32) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float4* ptr = reinterpret_cast<float4*>(buf + te_off(lane, c));
          const float4 r = *ptr;
          *ptr = make_float4(te_add(x[4 * c], r.x), te_add(x[4 * c + 1], r.y), te_add(x[4 * c + 2], r.z),
                             te_add(x[4 * c + 3], r.w));
        }
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint4* ptr = reinterpret_cast<uint4*>(buf + te_off(lane, c));
          const uint4 in = IN ? *ptr : make_uint4(0, 0, 0, 0);
          uint4 o, aux = make_uint4(0, 0, 0, 0);
          const float* xc = x + 8 * c;
          o.x = te_pair<MODE>(xc[0], xc[1], in.x, aux.x);
          o.y = te_pair<MODE>(xc[2], xc[3], in.y, aux.y);
          o.z = te_pair<MODE>(xc[4], xc[5], in.z, aux.z);
          o.w = te_pair<MODE>(xc[6], xc[7], in.w, aux.w);
          if (ACT_FWD) {  // box: the pre-activation (tma_d); box + 1: the activation (tma_c)
            *ptr = aux;
            *reinterpret_cast<uint4*>(buf + TE_BUF_BYTES + te_off(lane, c)) = o;
          } else {
            *ptr = o;
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        if (ACT_FWD) {
          tma_store_4d(&p.tma_d, buf, col, c1, c2, c3);
          tma_store_4d(&p.tma_c, buf + TE_BUF_BYTES, col, c1, c2, c3);
        } else {
          tma_store_4d(&p.tma_c, buf, col, c1, c2, c3);
        }
        bulk_commit_group();
      }
    }
    cnt += my;
  }
}

constexpr int GEMM_BAR_BYTES = 1024;  // stage-ring barriers, per-warp input barriers (tensor-map epilogue)

// Row pitch (floats) of the staged accumulator tile: a multiple of 4 (16-byte row reads) that is 4 mod 32, so the
// epilogue's thread-per-row 16-byte reads hit distinct banks within each quarter warp.
__host__ __device__ __forceinline__ int acc_ld(int block_n) { return (block_n + 31) / 32 * 32 + 4; }

// Warps 0..7 = two MMA warpgroups (tile rows 0..63, 64..127) that afterwards run the epilogue, warp 8 = TMA producer.
// Per tile: wgmma into registers, fragments -> staged fp32 tile in shared memory, epilogue from there.  The producer runs
// ahead through the stage ring, so the next tile's operands stream in while the epilogue of this one runs.
// TE: the tensor-map epilogue's mode, or TE_NONE for the generic epilogue.  HAS_IN: the generic epilogue reads an input
// tensor (residual / saved pre-activation) that is prefetched; kept out of the input-free kernel so that one stays lean.
template <bool HAS_IN, int TE, int NF, bool ERF = false>
__device__ __forceinline__ void gemm_body(const GemmParams& p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  // keep the pointer derived from the __shared__ symbol (offset arithmetic only) so smem accesses compile to LDS/STS
  const uint32_t smem_base_u32 = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((smem_base_u32 + 1023u) & ~1023u) - smem_base_u32);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t stage_bytes = A_TILE_BYTES + static_cast<uint32_t>(p.block_n) * GEMM_BLOCK_K * 2;

  uint8_t* bar_block = smem + static_cast<size_t>(p.stages) * stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bar_block);
  uint64_t* empty_bar = full_bar + GEMM_MAX_STAGES;
  uint64_t* in_bars = reinterpret_cast<uint64_t*>(bar_block + 256);  // [GEMM_EPI_WARPS][TE_BUFS]
  const int ald = acc_ld(p.block_n);
  float* acc_tile = reinterpret_cast<float*>(bar_block + GEMM_BAR_BYTES);
  uint8_t* epi_base = reinterpret_cast<uint8_t*>(acc_tile + GEMM_BLOCK_M * ald);  // 1024-byte aligned

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tma_a);
    prefetch_tmap(&p.tma_b);
    if (TE != TE_NONE) prefetch_tmap(&p.tma_c);
    if (TE != TE_NONE && TE != TE_F16) prefetch_tmap(&p.tma_d);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrive per MMA warpgroup
    }
    if (TE != TE_NONE)
      for (int i = 0; i < GEMM_EPI_WARPS * TE_BUFS; ++i) mbar_init(&in_bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touched only parameters and shared memory

  if (warp == GEMM_EPI_WARPS) {
    if (lane == 0) producer_loop(p, smem, full_bar, empty_bar, stage_bytes);
    return;
  }
  const int wg = warp >> 2;
  const int q = warp & 3, half = warp >> 2;  // epilogue: row quarter, and which column slabs of it
  const float* arow = acc_tile + (q * 32 + lane) * ald;
  uint8_t* wbase = epi_base + static_cast<size_t>(warp) * (TE != TE_NONE ? TE_WARP_BYTES : TB_WARP_BYTES);
  long long* s_off = reinterpret_cast<long long*>(wbase + TB_FLOATS * 4);
  int* s_row = reinterpret_cast<int*>(wbase + TB_FLOATS * 4 + 32 * 8);
  const bool wide = (p.out_f32 != nullptr) || (p.res_f32 != nullptr);
  const uint32_t smem0 = smem_u32(smem), full0 = smem_u32(full_bar);
  int stage = 0;
  uint32_t phase = 0, cnt = 0;
  AccFor<NF> acc;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int n_kb = tile_k_blocks(p, tile);
    if (p.a_mode == OP_MNMAJOR) {
      if (p.b_mode == OP_MNMAJOR) mma_tile<1, 1, NF>(p, acc, wg, n_kb, smem0, full0, empty_bar, stage_bytes, stage, phase);
      else mma_tile<1, 0, NF>(p, acc, wg, n_kb, smem0, full0, empty_bar, stage_bytes, stage, phase);
    } else {
      if (p.b_mode == OP_MNMAJOR) mma_tile<0, 1, NF>(p, acc, wg, n_kb, smem0, full0, empty_bar, stage_bytes, stage, phase);
      else mma_tile<0, 0, NF>(p, acc, wg, n_kb, smem0, full0, empty_bar, stage_bytes, stage, phase);
    }
    dump_acc(acc, acc_tile, ald, p.block_n);
    named_bar_sync(1, GEMM_EPI_WARPS * 32);
    if (TE != TE_NONE) {
      tma_epilogue_tile<TE>(p, t, wbase, in_bars + warp * TE_BUFS, arow, warp, lane, cnt);
    } else {
      const RowInfo ri = row_info(p, t, q * 32 + lane);
      s_off[lane] = ri.off;
      s_row[lane] = ri.row;
      __syncwarp();
      const int nslab = (p.block_n + 31) / 32;
      const int col_limit = min(p.N, t.n0 + p.block_n);
      const int kind = HAS_IN ? prefetch_kind(p) : 0;
      const float* blk = acc_tile + q * 32 * ald;
      for (int s = half; s < nslab; s += 2) {
        if (wide) {
          uint4 pf[BlockMap<4>::NIT];
          if (HAS_IN) prefetch_block<4>(p, s_off, lane, t.n0 + s * 32, col_limit, kind, pf);
          epilogue_block<4, ERF>(p, blk + s * 32, ald, s_off, s_row, lane, t.n0 + s * 32, col_limit, kind, pf);
        } else {
          uint4 pf[BlockMap<8>::NIT];
          if (HAS_IN) prefetch_block<8>(p, s_off, lane, t.n0 + s * 32, col_limit, kind, pf);
          epilogue_block<8, ERF>(p, blk + s * 32, ald, s_off, s_row, lane, t.n0 + s * 32, col_limit, kind, pf);
        }
      }
    }
    named_bar_sync(1, GEMM_EPI_WARPS * 32);  // the staged tile is free for the next tile's fragments
  }
  if (TE != TE_NONE && lane == 0) bulk_wait_group<0>();
}

template <int NF, bool ERF = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<false, TE_NONE, NF, ERF>(p);
}
template <int NF, bool ERF = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_in_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<true, TE_NONE, NF, ERF>(p);
}
template <int MODE, int NF>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tce_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<false, MODE, NF>(p);
}

// -------------------------------------------------------------------------------- wide kernel: 128 x 192 / 128 x 256
// For fp16 GEMMs with a K-major, unbatched A, no split-K and a tensor-map epilogue other than TE_RES32 (the ViT linear
// layers and their dgrads), a requested block_n of 192 or 256 runs here instead of in gemm_body.
//   * 384 threads.  Warpgroup 0 is the producer: one lane walks producer_tiles, the warpgroup drops to 40 registers.
//     Warpgroups 1 and 2 own tile rows [0, 64) and [64, 128) and rise to 232 registers: 40 * 128 + 232 * 256 = 64,512
//     = 168 * 384, what one CTA holds at __launch_bounds__(384, 1).  A 64 x 256 fp32 accumulator is 128 of them.
//   * One m64nBNk16 wgmma per consumer warpgroup and k16 step (a single static instruction, no runtime-guarded chain),
//     each stage released as soon as its wgmma group has retired, as in mma_tile.
//   * Epilogue straight from the accumulator registers, 64 columns at a time: each warp converts its 16 rows to fp16
//     (te_pair, the arithmetic of tma_epilogue_tile), writes them with stmatrix into a 16 x 128-byte box (128-byte
//     swizzle) and hands the box to a TMA store, which clips ragged M and N.  TE_ERF_GELU_BWD stays on gemm_body: its
//     32 erfc / exp evaluations per chunk beside the 128-register accumulator spill at 232 registers.  An input tensor (fp16 residual, saved
//     pre-activation) arrives by TMA in the same box up to two chunks ahead and is read into the fragment layout with
//     ldmatrix.  No staged fp32 tile and no barrier between the consumer warpgroups; the producer refills the ring for
//     the next tile while they run it.
// Shared memory (227 KiB = 232,448 bytes): 1 KiB alignment slack, the stage ring, GEMM_BAR_BYTES of barriers and two
// 2 KiB boxes per consumer warp (32 KiB); the ring gets the remaining 197,632 bytes: 4 stages of 48 KiB at BN = 256,
// 4 of 40 KiB at BN = 192.
constexpr int WB_BYTES = 2048;  // one box: 16 rows x 64 fp16 columns
constexpr int WB_BOXES = 2;     // per consumer warp
constexpr int WIDE_CONSUMER_WARPS = 8;
constexpr int WIDE_EPI_BYTES = WIDE_CONSUMER_WARPS * WB_BOXES * WB_BYTES;

// byte offset of 16-byte chunk c (0..7) of row r (0..15) in a CU_TENSOR_MAP_SWIZZLE_128B box (chunk ^= address bits 7..9)
__device__ __forceinline__ uint32_t wb_off(int r, int c) {
  return static_cast<uint32_t>(r * 128 + ((c ^ (r & 7)) << 4));
}

// Consumer warpgroup `wg` (0 or 1): wgmma over the n_kb k-blocks of one tile, as mma_tile with one instruction per k16
// step.  `first` runs once the first k-block has been issued (the epilogue's input prefetch).
template <int BN, int TB, typename First>
__device__ __forceinline__ void mma_tile_wide(float (&acc)[BN / 2], int wg, int n_kb, int stages, uint32_t smem0,
                                              uint32_t full0, uint64_t* empty_bar, int& stage, uint32_t& phase,
                                              First&& first) {
  constexpr uint32_t stage_bytes = A_TILE_BYTES + BN * GEMM_BLOCK_K * 2;
  const uint64_t b_kstep = (TB ? 2048 : 32) >> 4;
  const uint64_t a_desc0 = make_smem_desc_sw128(smem0 + wg * 8192, 0, 1024);
  const uint64_t b_desc0 = make_smem_desc_sw128(smem0 + A_TILE_BYTES, TB ? MN_ATOM_BYTES : 0, 1024);
  const bool elected = (threadIdx.x & 127) == 0;
  int prev = -1;
  for (int kb = 0; kb < n_kb; ++kb) {
    mbar_wait_s(full0 + stage * 8, phase);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = a_desc0 + stage * (stage_bytes >> 4) + k * (32 >> 4);
      const uint64_t bd = b_desc0 + stage * (stage_bytes >> 4) + k * b_kstep;
      const uint32_t scale_d = (kb | k) ? 1u : 0u;
      if constexpr (BN == 256) wgmma_m64n256<0, TB>(acc, ad, bd, scale_d);
      else wgmma_m64n192<0, TB>(acc, ad, bd, scale_d);
    }
    wgmma_commit();
    if (kb == 0) first();
    wgmma_wait<1>();
    if (prev >= 0 && elected) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  if (prev >= 0 && elected) mbar_arrive(&empty_bar[prev]);
}

// TMA load of the input tensor's 64-column chunk at `col` into one box of this warp (lane 0)
__device__ __forceinline__ void wide_in_load(const GemmParams& p, uint64_t* bar, uint8_t* box, int col, int row0,
                                             const TileCoord& t) {
  mbar_arrive_expect_tx(bar, WB_BYTES);
  tma_load_4d(&p.tma_d, bar, box, col, row0, t.b0, t.b1);
}

// One tile's epilogue for one consumer warp: rows [row0, row0 + 16) of the output, the 64-column chunks with at least one
// column inside N.  `cnt` counts the chunks this warp has processed: chunk j of the tile goes to box (cnt + j) % 2 (the
// forward activations use both boxes for every chunk).  in_ph: the parity of each box's input barrier.
template <int MODE, int BN>
__device__ __forceinline__ void wide_epilogue_tile(const GemmParams& p, const TileCoord& t, const float (&acc)[BN / 2],
                                                   uint8_t* wbuf, uint64_t* in_bar, int row0, int lane, uint32_t& cnt,
                                                   uint32_t& in_ph) {
  constexpr bool ACT_FWD = (MODE == TE_GELU || MODE == TE_ERF_GELU);
  constexpr bool IN = (MODE == TE_RES16 || MODE == TE_GELU_BWD || MODE == TE_ERF_GELU_BWD);
  const int nch = (min(p.N - t.n0, BN) + 63) / 64;
  const uint32_t wb0 = smem_u32(wbuf);
  // stmatrix / ldmatrix x4 over column groups (2 q, 2 q + 1): matrix m = lane / 8 is rows 8 (m % 2) .. + 7 of group
  // 2 q + m / 2, and its register is the fragment's pair 4 q + m, i.e. accumulator registers 8 q + 2 m, + 1 of the chunk
  const int mrow = (lane & 7) + 8 * ((lane >> 3) & 1), mgrp = lane >> 4;
#pragma unroll
  for (int j = 0; j < BN / 64; ++j) {
    if (j < nch) {
      const int col = t.n0 + 64 * j;
      const int b = ACT_FWD ? 0 : ((cnt + j) & 1);
      const uint32_t box = wb0 + b * WB_BYTES;
      if (lane == 0) {
        if (ACT_FWD) bulk_wait_group_read<0>();  // both boxes' stores of the previous chunk have read them
        else if (!IN) bulk_wait_group_read<1>();  // this box's store, two chunks back (possibly in the previous tile)
      }
      __syncwarp();
      uint32_t in[16];
      if (IN) {
        mbar_wait(&in_bar[b], (in_ph >> b) & 1);
        in_ph ^= 1u << b;
#pragma unroll
        for (int q = 0; q < 4; ++q) ldmatrix_x4(box + wb_off(mrow, 2 * q + mgrp), in[4 * q], in[4 * q + 1], in[4 * q + 2], in[4 * q + 3]);
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) in[i] = 0;
      }
      uint32_t out[16], aux[16];
#pragma unroll
      for (int g = 0; g < 8; ++g) {  // column group g: columns col + 8 g + 2 (lane % 4), + 1; rows lo / hi
        const int c = col + 8 * g + 2 * (lane & 3);
        float2 bb = make_float2(0.f, 0.f);
        if (p.bias && c < p.N) bb = __ldg(reinterpret_cast<const float2*>(p.bias + c));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 32 * j + 4 * g + 2 * h;
          float x0 = te_scale(acc[r], p.alpha), x1 = te_scale(acc[r + 1], p.alpha);
          if (p.bias) {
            x0 = te_add(x0, bb.x);
            x1 = te_add(x1, bb.y);
          }
          aux[2 * g + h] = 0;
          out[2 * g + h] = te_pair<MODE>(x0, x1, in[2 * g + h], aux[2 * g + h]);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t o = wb_off(mrow, 2 * q + mgrp);
        if (ACT_FWD) {  // box 0: the pre-activation (tma_d), box 1: the activation (tma_c)
          stmatrix_x4(wb0 + o, aux[4 * q], aux[4 * q + 1], aux[4 * q + 2], aux[4 * q + 3]);
          stmatrix_x4(wb0 + WB_BYTES + o, out[4 * q], out[4 * q + 1], out[4 * q + 2], out[4 * q + 3]);
        } else {
          stmatrix_x4(box + o, out[4 * q], out[4 * q + 1], out[4 * q + 2], out[4 * q + 3]);
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        if (ACT_FWD) {
          tma_store_4d(&p.tma_d, wbuf, col, row0, t.b0, t.b1);
          tma_store_4d(&p.tma_c, wbuf + WB_BYTES, col, row0, t.b0, t.b1);
        } else {
          tma_store_4d(&p.tma_c, wbuf + b * WB_BYTES, col, row0, t.b0, t.b1);
        }
        bulk_commit_group();
        if (IN && j + 2 < nch) {
          bulk_wait_group_read<0>();  // the store just issued has read the box
          wide_in_load(p, &in_bar[b], wbuf + b * WB_BYTES, col + 128, row0, t);
        }
      }
    }
  }
  cnt += nch;
}

template <int MODE, int BN, int TB>
__global__ void __launch_bounds__(GEMM_WIDE_THREADS, 1) gemm_wide_kernel(const __grid_constant__ GemmParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base_u32 = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((smem_base_u32 + 1023u) & ~1023u) - smem_base_u32);
  constexpr uint32_t stage_bytes = A_TILE_BYTES + BN * GEMM_BLOCK_K * 2;
  constexpr bool IN = (MODE == TE_RES16 || MODE == TE_GELU_BWD || MODE == TE_ERF_GELU_BWD);
  uint8_t* bar_block = smem + static_cast<size_t>(p.stages) * stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bar_block);
  uint64_t* empty_bar = full_bar + GEMM_MAX_STAGES;
  uint64_t* in_bars = reinterpret_cast<uint64_t*>(bar_block + 256);  // [WIDE_CONSUMER_WARPS][WB_BOXES]
  uint8_t* boxes = bar_block + GEMM_BAR_BYTES;                        // 1024-byte aligned (128-byte swizzle)

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tma_a);
    prefetch_tmap(&p.tma_b);
    prefetch_tmap(&p.tma_c);
    if (MODE != TE_F16) prefetch_tmap(&p.tma_d);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    for (int i = 0; i < WIDE_CONSUMER_WARPS * WB_BOXES; ++i) mbar_init(&in_bars[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touched only parameters and shared memory

  if (threadIdx.x < 128) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) producer_tiles<OP_KMAJOR, TB ? OP_MNMAJOR : OP_KMAJOR>(p, smem, full_bar, empty_bar, stage_bytes);
    return;
  }
  setmaxnreg_inc<232>();
  const int wg = (threadIdx.x >> 7) - 1;  // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
  const int cw = (threadIdx.x >> 5) - 4;  // consumer warp 0..7
  const int lane = threadIdx.x & 31;
  uint8_t* wbuf = boxes + cw * (WB_BOXES * WB_BYTES);
  uint64_t* in_bar = in_bars + cw * WB_BOXES;
  const uint32_t smem0 = smem_u32(smem), full0 = smem_u32(full_bar);
  int stage = 0;
  uint32_t phase = 0, cnt = 0, in_ph = 0;
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(p, tile);
    const int row0 = t.m0 + 64 * wg + 16 * (cw & 3);
    mma_tile_wide<BN, TB>(acc, wg, p.num_k_blocks, p.stages, smem0, full0, empty_bar, stage, phase, [&] {
      if (IN && lane == 0) {  // the first two input chunks, while the rest of the tile's k-blocks run
        const int nch = (min(p.N - t.n0, BN) + 63) / 64;
        bulk_wait_group_read<0>();  // the previous tile's stores have read the boxes
        for (int j = 0; j < WB_BOXES && j < nch; ++j)
          wide_in_load(p, &in_bar[(cnt + j) & 1], wbuf + ((cnt + j) & 1) * WB_BYTES, t.n0 + 64 * j, row0, t);
      }
    });
    wide_epilogue_tile<MODE, BN>(p, t, acc, wbuf, in_bar, row0, lane, cnt, in_ph);
  }
  if (lane == 0) bulk_wait_group<0>();
}

template <int BN, int TB>
void (*wide_kernel(const GemmParams& p))(GemmParams) {
  switch (p.tma_epi) {
    case TE_F16: return gemm_wide_kernel<TE_F16, BN, TB>;
    case TE_RES16: return gemm_wide_kernel<TE_RES16, BN, TB>;
    case TE_GELU: return gemm_wide_kernel<TE_GELU, BN, TB>;
    case TE_GELU_BWD: return gemm_wide_kernel<TE_GELU_BWD, BN, TB>;
    case TE_ERF_GELU: return gemm_wide_kernel<TE_ERF_GELU, BN, TB>;
    default: return nullptr;
  }
}

// The kernel for a plan: fragment width NF (see mma_tile) and epilogue.
template <int NF>
void (*plain_kernel(const GemmParams& p))(GemmParams) {
  switch (p.tma_epi) {
    case TE_F16: return gemm_tce_kernel<TE_F16, NF>;
    case TE_GELU: return gemm_tce_kernel<TE_GELU, NF>;
    case TE_GELU_BWD: return gemm_tce_kernel<TE_GELU_BWD, NF>;
    case TE_RES32: return gemm_tce_kernel<TE_RES32, NF>;
    case TE_RES16: return gemm_tce_kernel<TE_RES16, NF>;
    case TE_ERF_GELU: return gemm_tce_kernel<TE_ERF_GELU, NF>;
    case TE_ERF_GELU_BWD: return gemm_tce_kernel<TE_ERF_GELU_BWD, NF>;
    default: break;
  }
  const bool erf = p.act == ACT_GELU || p.act == ACT_GELU_BWD;
  if (p.res_f32 || p.res_f16 || p.act == ACT_QUICKGELU_BWD || p.act == ACT_GELU_BWD || p.act == ACT_LRELU_BWD ||
      p.act == ACT_RELU_BWD)
    return erf ? gemm_tc_in_kernel<NF, true> : gemm_tc_in_kernel<NF>;
  return erf ? gemm_tc_kernel<NF, true> : gemm_tc_kernel<NF>;
}
void (*kernel_for(const GemmParams& p))(GemmParams) {
  if (p.block_n == 256) return p.b_mode == OP_MNMAJOR ? wide_kernel<256, 1>(p) : wide_kernel<256, 0>(p);
  if (p.block_n == 192) return p.b_mode == OP_MNMAJOR ? wide_kernel<192, 1>(p) : wide_kernel<192, 0>(p);
  if (p.fmt == 0 && p.block_n == 128) return plain_kernel<2>(p);
  if (p.fmt == 0 && p.block_n == 64) return plain_kernel<1>(p);
  return plain_kernel<0>(p);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

void set_err(char* err, int errlen, const char* msg) {
  if (err && errlen > 0) snprintf(err, errlen, "%s", msg);
}

// 4-D tensor map, zero fill out of bounds.  fmt 0 = fp16, 1 = bf16, 2 = fp32; operands use the 128-byte swizzle, the
// epilogue boxes (64-byte rows) the 64-byte swizzle.
int encode_tmap4(CUtensorMap* out, const void* ptr, int fmt, const uint64_t dims[4], const uint64_t strides_elems[3],
                 const uint32_t box[4], char* err, int errlen, bool swizzle64 = false) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_err(err, errlen, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return -1;
  }
  cuuint64_t gdims[4], gstrides[3];
  cuuint32_t gbox[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
  }
  for (int i = 0; i < 3; ++i) {
    gstrides[i] = strides_elems[i] * (fmt == 2 ? 4 : 2);
    if (gstrides[i] % 16 != 0 || gstrides[i] == 0) {
      set_err(err, errlen, "TMA global stride must be a non-zero multiple of 16 bytes");
      return -2;
    }
  }
  if (reinterpret_cast<uintptr_t>(ptr) % 16 != 0) {
    set_err(err, errlen, "TMA global address must be 16-byte aligned");
    return -3;
  }
  const CUtensorMapDataType dt = fmt == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                          : (fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  CUresult r = fn(out, dt, 4, const_cast<void*>(ptr), gdims, gstrides, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d): dims %llu,%llu,%llu,%llu box %u,%u,%u,%u", (int)r,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             (unsigned long long)dims[3], box[0], box[1], box[2], box[3]);
    set_err(err, errlen, buf);
    return -4;
  }
  return 0;
}

int encode_operand(CUtensorMap* out, const GemmOperand& op, int rows_box, int fmt, char* err, int errlen) {
  // batch strides for extent-1 dims still need to be valid multiples of 16 bytes
  long long bs0 = op.nb0 > 1 ? op.bs0 : 0, bs1 = op.nb1 > 1 ? op.bs1 : 0;
  uint64_t dims[4], strides[3];
  uint32_t box[4];
  if (op.mode == OP_KMAJOR) {
    dims[0] = op.k_extent;
    dims[1] = op.mn_extent;
    box[0] = GEMM_BLOCK_K;
    box[1] = rows_box;
  } else {
    dims[0] = op.mn_extent;
    dims[1] = op.k_extent;
    box[0] = 64;
    box[1] = GEMM_BLOCK_K;
  }
  dims[2] = op.nb0;
  dims[3] = op.nb1;
  box[2] = box[3] = 1;
  strides[0] = op.ld;
  strides[1] = bs0 ? bs0 : op.ld * dims[1];
  strides[2] = bs1 ? bs1 : strides[1] * dims[2];
  return encode_tmap4(out, op.ptr, fmt, dims, strides, box, err, errlen);
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

}  // namespace

int tmap_encode_4d(CUtensorMap* out, const void* ptr, int fmt, const uint64_t dims[4], const uint64_t strides_elems[3],
                   const uint32_t box[4], char* err, int errlen) {
  return encode_tmap4(out, ptr, fmt, dims, strides_elems, box, err, errlen);
}

namespace {
// Widest tile of gemm_body: the staged fp32 accumulator tile (128 x block_n) shares the 227 KiB of shared memory with the
// stage ring and the epilogue buffers; at 128 columns two stages still fit beside the tensor-map epilogue's boxes, three
// beside the generic epilogue's.  192 and 256 run in gemm_wide_kernel when the plan allows it (gemm_wide_ok); any other
// wider request runs as 128.
constexpr int GEMM_MAX_BN_PLAIN = 128;

int effective_block_n(int block_n) { return block_n > GEMM_MAX_BN_PLAIN ? GEMM_MAX_BN_PLAIN : block_n; }
bool wide_block_n(int block_n) { return block_n == 192 || block_n == 256; }

// Tensor-map epilogue (see tma_epilogue_tile) when the epilogue is one of its shapes and every tensor can be described
// by a tensor map; anything else keeps the generic epilogue.  PXR_GEMM_TMA_EPI=0 disables it globally.
int decide_tma_epi(const GemmParams& p, const GemmEpilogue& e, int block_n) {
  static const bool enabled = [] {
    const char* v = getenv("PXR_GEMM_TMA_EPI");
    return !(v && atoi(v) == 0);
  }();
  if (!enabled || e.tma_epi < 0 || e.bias_per_row || p.fmt != 0 || p.k_splits > 1) return TE_NONE;
  int mode = TE_NONE;
  const bool no_res = !e.res_f32 && !e.res_f16;
  if (e.act == ACT_NONE && e.out_f16 && !e.out_f32 && !e.res_f32 && !e.aux_out) mode = e.res_f16 ? TE_RES16 : TE_F16;
  else if ((e.act == ACT_QUICKGELU || e.act == ACT_GELU) && e.aux_out && e.out_f16 && !e.out_f32 && no_res)
    mode = e.act == ACT_GELU ? TE_ERF_GELU : TE_GELU;
  else if ((e.act == ACT_QUICKGELU_BWD || e.act == ACT_GELU_BWD) && e.aux_in && e.out_f16 && !e.out_f32 && no_res)
    mode = e.act == ACT_GELU_BWD ? TE_ERF_GELU_BWD : TE_GELU_BWD;
  else if (e.act == ACT_NONE && e.out_f32 && !e.out_f16 && e.res_f32 && !e.res_f16 && !e.aux_out) mode = TE_RES32;
  if (mode == TE_NONE) return TE_NONE;
  const int bw = mode == TE_RES32 ? 16 : 32;
  const int eb = mode == TE_RES32 ? 4 : 2;
  if (block_n % bw && p.tiles_n != 1) return TE_NONE;  // a partial last block would spill into the next tile's columns
  if (e.bias && (!aligned16(e.bias) || p.N % bw)) return TE_NONE;
  if ((e.ldc * eb) % 16 || (e.bs0 * eb) % 16 || (e.bs1 * eb) % 16) return TE_NONE;
  if (!aligned16(e.out_f16) || !aligned16(e.out_f32) || !aligned16(e.aux_in) || !aligned16(e.aux_out) ||
      !aligned16(e.res_f32) || !aligned16(e.res_f16))
    return TE_NONE;
  if (p.a_mode == OP_CONV && (32 % p.tile_w)) return TE_NONE;
  // TMA clips the innermost dimension at 16-byte granularity: a ragged N overwrites the columns up to the next 16-byte
  // boundary (with alpha * 0 when B's out-of-range rows are zero-filled), so they must be padding inside the row pitch
  const int gran = 16 / eb;
  if (p.N % gran && (e.ldc < (p.N + gran - 1) / gran * gran || e.bias)) return TE_NONE;
  return mode;
}

// Boxes of 32 rows x 64 bytes, 64-byte swizzle (tma_epilogue_tile) or, for the wide kernel, 16 rows x 64 fp16 columns,
// 128-byte swizzle (wide_epilogue_tile).
int encode_epilogue_map(CUtensorMap* out, const void* ptr, bool f32, const GemmParams& p, const GemmEpilogue& e,
                        char* err, int errlen) {
  const bool wide = p.block_n > GEMM_MAX_BN_PLAIN;
  uint64_t dims[4], strides[3];
  uint32_t box[4];
  const uint64_t ldc = static_cast<uint64_t>(e.ldc);
  dims[0] = p.N;
  box[0] = wide ? 64 : (f32 ? 16 : 32);
  if (p.a_mode == OP_CONV) {
    dims[1] = p.conv_W;
    dims[2] = p.conv_H;
    dims[3] = p.nb0;
    strides[0] = ldc;
    strides[1] = ldc * p.conv_W;
    strides[2] = ldc * p.conv_W * p.conv_H;
    box[1] = p.tile_w;
    box[2] = 32 / p.tile_w;
    box[3] = 1;
  } else {
    const int nb1 = p.total_tiles / (p.tiles_m * p.tiles_n * p.nb0);
    dims[1] = p.M;
    dims[2] = p.nb0;
    dims[3] = nb1;
    strides[0] = ldc;
    strides[1] = p.nb0 > 1 ? static_cast<uint64_t>(e.bs0) : ldc * p.M;
    strides[2] = nb1 > 1 ? static_cast<uint64_t>(e.bs1) : strides[1] * p.nb0;
    box[1] = wide ? 16 : 32;
    box[2] = box[3] = 1;
  }
  return encode_tmap4(out, ptr, f32 ? 2 : 0, dims, strides, box, err, errlen, !wide);
}

// bytes the epilogue must move for `mn` output elements: every output written once, every input tensor read once
double epilogue_bytes(const GemmEpilogue& e, double mn) {
  double b = 0;
  if (e.out_f16) b += 2 * mn;
  if (e.out_f32) b += 4 * mn;
  if (e.aux_out) b += 2 * mn;
  if (e.aux_in) b += 2 * mn;
  if (e.res_f16) b += 2 * mn;
  if (e.res_f32) b += 4 * mn;
  return b;
}

int finish_plan(GemmPlan* plan, const GemmEpilogue& epi, int block_n, int num_sms, char* err, int errlen) {
  GemmParams& p = plan->p;
  const bool wide = wide_block_n(block_n);  // gemm_plan_make keeps 192 / 256 only for plans gemm_wide_ok accepts
  if (!wide && (block_n < 16 || block_n > GEMM_MAX_BN_PLAIN || block_n % 16)) {
    set_err(err, errlen, "block_n must be a multiple of 16 in [16, 128], or 192 / 256");
    return -10;
  }
  if (epi.act != ACT_NONE && epi.act != ACT_QUICKGELU && epi.act != ACT_QUICKGELU_BWD && epi.act != ACT_LRELU &&
      epi.act != ACT_LRELU_BWD && epi.act != ACT_GELU && epi.act != ACT_GELU_BWD && epi.act != ACT_RELU &&
      epi.act != ACT_RELU_BWD) {
    set_err(err, errlen, "unknown epilogue activation (act must be 0 none, 1 QuickGELU, 2 QuickGELU backward, 4 LeakyReLU, "
                         "5 LeakyReLU backward, 6 GELU, 7 GELU backward, 8 ReLU or 9 ReLU backward)");
    return -12;
  }
  if ((epi.act == ACT_LRELU_BWD || epi.act == ACT_RELU_BWD) && !epi.aux_in) {
    set_err(err, errlen, "the (Leaky)ReLU backward needs the saved post-activation (aux_in)");
    return -14;
  }
  if (epi.act == ACT_GELU_BWD && !epi.aux_in) {
    set_err(err, errlen, "the GELU backward needs the saved pre-activation (aux_in)");
    return -14;
  }
  if (p.b_mode == OP_MNMAJOR && block_n % 64) {
    set_err(err, errlen, "MN-major B needs block_n % 64 == 0");
    return -11;
  }
  p.block_n = block_n;
  p.tma_epi = decide_tma_epi(p, epi, block_n);
  if (p.tma_epi != TE_NONE) {
    const bool f32 = p.tma_epi == TE_RES32;
    int rc = encode_epilogue_map(&p.tma_c, f32 ? static_cast<const void*>(epi.out_f32) : epi.out_f16, f32, p, epi, err,
                                 errlen);
    const void* second = (p.tma_epi == TE_GELU || p.tma_epi == TE_ERF_GELU)  ? static_cast<const void*>(epi.aux_out)
                         : (p.tma_epi == TE_GELU_BWD || p.tma_epi == TE_ERF_GELU_BWD) ? static_cast<const void*>(epi.aux_in)
                         : p.tma_epi == TE_RES32                                 ? static_cast<const void*>(epi.res_f32)
                         : p.tma_epi == TE_RES16                                 ? static_cast<const void*>(epi.res_f16)
                                                                                 : nullptr;
    if (!rc && second) rc = encode_epilogue_map(&p.tma_d, second, f32, p, epi, err, errlen);
    if (rc) p.tma_epi = TE_NONE;  // a stride the tensor map cannot express: generic epilogue
  }
  if (wide && (p.tma_epi == TE_NONE || p.tma_epi == TE_RES32 || p.tma_epi == TE_ERF_GELU_BWD)) {
    set_err(err, errlen, "192- / 256-wide tiles need an fp16 tensor-map epilogue");
    return -15;
  }
  const int stage_bytes = A_TILE_BYTES + block_n * GEMM_BLOCK_K * 2;
  const int epi_smem = wide ? GEMM_BAR_BYTES + WIDE_EPI_BYTES
                            : GEMM_BAR_BYTES + GEMM_BLOCK_M * acc_ld(block_n) * 4 +
                                  GEMM_EPI_WARPS * (p.tma_epi != TE_NONE ? TE_WARP_BYTES : TB_WARP_BYTES);
  int stages = (227 * 1024 - 1024 - epi_smem) / stage_bytes;
  if (stages > GEMM_MAX_STAGES) stages = GEMM_MAX_STAGES;
  if (stages < 2) {  // mma_tile releases a stage only after the next one has been issued
    set_err(err, errlen, "block_n too wide for a two-stage ring in shared memory");
    return -13;
  }
  p.stages = stages;
  p.alpha = epi.alpha;
  p.bias = epi.bias;
  p.bias_per_row = epi.bias_per_row;
  p.act = epi.act;
  p.act_col0 = epi.act_col0;
  p.aux_in = epi.aux_in;
  p.aux_out = epi.aux_out;
  p.res_f32 = epi.res_f32;
  p.res_f16 = epi.res_f16;
  p.out_f32 = epi.out_f32;
  p.out_f16 = epi.out_f16;
  p.ldc = epi.ldc;
  p.out_bs0 = epi.bs0;
  p.out_bs1 = epi.bs1;
  p.vec_ok = (epi.ldc % 8 == 0) && (epi.bs0 % 8 == 0) && (epi.bs1 % 8 == 0) && aligned16(epi.aux_in) &&
             aligned16(epi.aux_out) && aligned16(epi.res_f32) && aligned16(epi.res_f16) && aligned16(epi.out_f32) &&
             aligned16(epi.out_f16);
  plan->grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  plan->smem_bytes = stages * stage_bytes + 1024 + epi_smem;
  static std::once_flag once;
  std::call_once(once, [] {
    for (int nf = 0; nf < 3; ++nf)
      for (int te = TE_NONE; te <= TE_ERF_GELU_BWD; ++te)
        for (int act : {ACT_NONE, ACT_QUICKGELU_BWD, ACT_GELU, ACT_GELU_BWD}) {  // every generic kernel
          GemmParams q{};
          q.fmt = 0;
          q.block_n = nf == 2 ? 128 : (nf == 1 ? 64 : 16);
          q.tma_epi = te;
          q.act = act;
          cudaFuncSetAttribute(kernel_for(q), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        }
    for (int bn : {192, 256})
      for (int bm : {OP_KMAJOR, OP_MNMAJOR})
        for (int te : {TE_F16, TE_RES16, TE_GELU, TE_GELU_BWD, TE_ERF_GELU}) {  // every wide kernel
          GemmParams q{};
          q.block_n = bn;
          q.b_mode = bm;
          q.tma_epi = te;
          cudaFuncSetAttribute(kernel_for(q), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        }
  });
  return 0;
}

}  // namespace

bool gemm_wide_ok(const GemmOperand& A, int N, const GemmEpilogue& epi, int fmt) {
  if (fmt != 0 || A.mode != OP_KMAJOR || A.nb0 != 1 || A.nb1 != 1 || epi.k_splits > 1) return false;
  GemmParams q{};  // what decide_tma_epi reads of a plan; at 192 / 256 columns every 32-column block is whole
  q.fmt = fmt;
  q.N = N;
  q.a_mode = A.mode;
  q.k_splits = 1;
  q.tiles_n = 1;
  const int te = decide_tma_epi(q, epi, 256);
  return te != TE_NONE && te != TE_RES32 && te != TE_ERF_GELU_BWD;
}

int gemm_plan_make(GemmPlan* plan, const GemmOperand& A, const GemmOperand& B, int M, int N, int K,
                   const GemmEpilogue& epi, int block_n, int fmt, int num_sms, char* err, int errlen) {
  *plan = GemmPlan{};
  GemmParams& p = plan->p;
  if (A.mode == OP_CONV || B.mode == OP_CONV) {
    set_err(err, errlen, "use conv_plan_make for conv operands");
    return -20;
  }
  if (!(wide_block_n(block_n) && gemm_wide_ok(A, N, epi, fmt))) block_n = effective_block_n(block_n);
  p.M = M;
  p.N = N;
  p.fmt = fmt;
  p.a_mode = A.mode;
  p.b_mode = B.mode;
  p.num_taps = 1;
  p.k_blocks_per_tap = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  p.num_k_blocks = p.k_blocks_per_tap;
  p.tiles_m = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  p.tiles_n = (N + block_n - 1) / block_n;
  const int nb0 = A.nb0, nb1 = A.nb1;
  p.nb0 = nb0;
  p.b_batched = (B.nb0 > 1 || B.nb1 > 1) ? 1 : 0;
  if (p.b_batched && (B.nb0 != nb0 || B.nb1 != nb1)) {
    set_err(err, errlen, "batched B must have the same batch extents as A");
    return -21;
  }
  p.total_tiles = p.tiles_m * p.tiles_n * nb0 * nb1;
  p.k_splits = 1;
  p.kb_per_split = p.num_k_blocks;
  GemmEpilogue epi_s = epi;
  if (epi.k_splits > 1) {  // split-K: the batch index of a tile becomes the split (fp32 partial sums, slab z of out_f32)
    if (nb0 != 1 || nb1 != 1 || !epi.out_f32 || epi.out_f16 || epi.bias || epi.res_f16 || epi.res_f32 || epi.act != ACT_NONE) {
      set_err(err, errlen, "split-K GEMM: unbatched operands, plain fp32 partial sums only");
      return -22;
    }
    p.kb_per_split = (p.num_k_blocks + epi.k_splits - 1) / epi.k_splits;
    p.k_splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;
    p.nb0 = p.k_splits;
    p.total_tiles = p.tiles_m * p.tiles_n * p.k_splits;
    epi_s.bs0 = (long long)M * epi.ldc;
  }
  int rc = encode_operand(&p.tma_a, A, GEMM_BLOCK_M, fmt, err, errlen);
  if (rc) return rc;
  rc = encode_operand(&p.tma_b, B, block_n, fmt, err, errlen);
  if (rc) return rc;
  plan->flops = 2.0 * M * N * K * nb0 * nb1;
  {
    const double nb = (double)nb0 * nb1, mn = (double)M * N * nb;
    plan->bytes = 2.0 * M * K * nb + 2.0 * N * K * (p.b_batched ? nb : 1.0) + epilogue_bytes(epi, mn);
  }
  return finish_plan(plan, epi_s, block_n, num_sms, err, errlen);
}

int conv_plan_make(GemmPlan* plan, const void* in, long long in_ld, int batch, int H, int W, int c_in, const void* wt,
                   int cout_pad, int n_out, int ksize, const GemmEpilogue& epi, int block_n, int fmt, int num_sms,
                   char* err, int errlen) {
  *plan = GemmPlan{};
  GemmParams& p = plan->p;
  if (c_in % 64 || (ksize != 1 && ksize != 3)) {
    set_err(err, errlen, "conv: c_in must be a multiple of 64 and ksize 1 or 3");
    return -30;
  }
  if (W < 1 || H < 1) {
    set_err(err, errlen, "conv: empty image");
    return -31;
  }
  // M tile = tile_h x tile_w pixels (8 x 16 or 16 x 8).  Any W works: columns past the image are zero-filled by the
  // TMA loads and clipped by the stores (tensor-map epilogue) / predicated off (generic epilogue); pick the width that
  // wastes the fewest columns (pixray's presets give latents such as 9 x 9, 18 x 18, 12 x 6: pixray.py:1864-1878)
  block_n = effective_block_n(block_n);
  const int waste16 = (W + 15) / 16 * 16, waste8 = (W + 7) / 8 * 8;
  int tile_w = (waste16 <= waste8) ? 16 : 8;
  int tile_h = GEMM_BLOCK_M / tile_w;
  p.M = H * W;
  p.N = n_out;
  p.fmt = fmt;
  p.a_mode = OP_CONV;
  p.b_mode = OP_KMAJOR;
  p.num_taps = ksize * ksize;
  p.k_blocks_per_tap = c_in / 64;
  p.num_k_blocks = p.num_taps * p.k_blocks_per_tap;
  p.conv_H = H;
  p.conv_W = W;
  p.tile_h = tile_h;
  p.tile_w = tile_w;
  p.tiles_w = (W + tile_w - 1) / tile_w;
  p.tiles_m = p.tiles_w * ((H + tile_h - 1) / tile_h);
  p.tiles_n = (n_out + block_n - 1) / block_n;
  p.nb0 = batch;
  p.b_batched = 0;
  p.b_tap_rows = cout_pad;
  p.total_tiles = p.tiles_m * p.tiles_n * batch;
  p.k_splits = 1;
  p.kb_per_split = p.num_k_blocks;
  if (epi.k_splits > 1) {
    if (batch != 1 || !epi.out_f32 || epi.out_f16 || epi.bias || epi.res_f16 || epi.res_f32 || epi.act != ACT_NONE) {
      set_err(err, errlen, "split-K conv: one image, plain fp32 partial sums only");
      return -32;
    }
    p.kb_per_split = (p.num_k_blocks + epi.k_splits - 1) / epi.k_splits;
    p.k_splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;
    p.nb0 = p.k_splits;  // decode_tile: z = split
    p.total_tiles = p.tiles_m * p.tiles_n * p.k_splits;
  }
  {
    uint64_t dims[4] = {(uint64_t)c_in, (uint64_t)W, (uint64_t)H, (uint64_t)batch};
    uint64_t strides[3] = {(uint64_t)in_ld, (uint64_t)in_ld * W, (uint64_t)in_ld * W * H};
    uint32_t box[4] = {64, (uint32_t)tile_w, (uint32_t)tile_h, 1};
    int rc = encode_tmap4(&p.tma_a, in, fmt, dims, strides, box, err, errlen);
    if (rc) return rc;
  }
  {
    GemmOperand B;
    B.ptr = wt;
    B.mode = OP_KMAJOR;
    B.ld = c_in;
    B.mn_extent = (long long)p.num_taps * cout_pad;
    B.k_extent = c_in;
    int rc = encode_operand(&p.tma_b, B, block_n, fmt, err, errlen);
    if (rc) return rc;
  }
  plan->flops = 2.0 * H * W * (double)n_out * c_in * p.num_taps * batch;
  plan->bytes = 2.0 * H * W * (double)c_in * batch + 2.0 * (double)n_out * c_in * p.num_taps +
                epilogue_bytes(epi, (double)H * W * n_out * batch * (epi.k_splits > 1 ? epi.k_splits : 1));
  GemmEpilogue e = epi;
  return finish_plan(plan, e, block_n, num_sms, err, errlen);
}

namespace {
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, int splits, long long pixels,
                                                            int N, int ld_ws, const float* __restrict__ bias,
                                                            const __half* __restrict__ res, __half* __restrict__ out,
                                                            int ld_out) {
  pdl_prologue();
  const int vecs = N / 8;
  const long long n = pixels * vecs;
  const size_t slab = static_cast<size_t>(pixels) * ld_ws;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const long long px = i / vecs;
    const int c0 = static_cast<int>(i % vecs) * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bias ? bias[c0 + j] : 0.f;
    const float* src = ws + static_cast<size_t>(px) * ld_ws + c0;
    uint4 r16 = make_uint4(0, 0, 0, 0);
    if (res) r16 = *reinterpret_cast<const uint4*>(res + static_cast<size_t>(px) * ld_out + c0);
    // the partial sums are independent loads: issue four splits' worth before the (fixed-order) adds, so the loop pays
    // one L2 round trip per four splits instead of one per split
    int s0 = 0;
    for (; s0 + 4 <= splits; s0 += 4) {
      float4 a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * slab));
        b[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * slab + 4));
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {  // fixed order: deterministic
        acc[0] += a[u].x;
        acc[1] += a[u].y;
        acc[2] += a[u].z;
        acc[3] += a[u].w;
        acc[4] += b[u].x;
        acc[5] += b[u].y;
        acc[6] += b[u].z;
        acc[7] += b[u].w;
      }
    }
    for (; s0 < splits; ++s0) {
      const float4 a = __ldcg(reinterpret_cast<const float4*>(src + s0 * slab)), b = __ldcg(reinterpret_cast<const float4*>(src + s0 * slab + 4));
      acc[0] += a.x;
      acc[1] += a.y;
      acc[2] += a.z;
      acc[3] += a.w;
      acc[4] += b.x;
      acc[5] += b.y;
      acc[6] += b.z;
      acc[7] += b.w;
    }
    if (res) {
      float r[8];
      unpack8(r16, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += r[j];
    }
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(px) * ld_out + c0) = pack8(acc);
  }
}
}  // namespace

void splitk_reduce(const float* ws, int splits, long long pixels, int N, int ld_ws, const float* bias,
                   const __half* res, __half* out, int ld_out, cudaStream_t stream) {
  const long long n = pixels * (N / 8);
  long long g = (n + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  launch_pdl(splitk_reduce_kernel, dim3(static_cast<int>(g)), dim3(256), 0, stream, ws, splits, pixels, N, ld_ws, bias, res, out, ld_out);
}

void gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
  const int threads = plan.p.block_n > GEMM_MAX_BN_PLAIN ? GEMM_WIDE_THREADS : GEMM_THREADS;
  launch_pdl(kernel_for(plan.p), dim3(plan.grid), dim3(threads), plan.smem_bytes, stream, plan.p);
}

}  // namespace pxr
