// Fragment helpers shared by the fused attention kernels (attn_tc.cu, attn_long.cu): warp-level mma.sync m16n8k16
// (fp16 x fp16 -> fp32), ldmatrix loads from swizzled 64-wide fp16 tiles, and the accumulator -> A-fragment repack.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace pxr {
namespace attn_frag {

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

}  // namespace attn_frag
}  // namespace pxr
