// wgmma / TMA GEMM for sm_90a: the one dense-contraction kernel of the engine.
//
//   D[m, n] = epilogue( alpha * sum_k A[m, k] * B[n, k] )          fp16 (or bf16) operands, fp32 accumulate
//
// One persistent kernel covers every dense op on the pixray hot path (SURVEY.md §2.2 K1/K2/K9):
//   * linear layers and their dgrad (CLIP ViT: qkv / out_proj / c_fc / c_proj, patch embed),
//   * batched attention products (QK^T, PV and the four backward products) by selecting K-major or
//     MN-major operands per side -- no transposed copies are ever materialised,
//   * 3x3 / 1x1 convolutions of the VQGAN decoder as implicit GEMM: the A operand is fetched by a 4-D TMA
//     box (C, W, H, B) shifted per filter tap, out-of-image halo zero-filled by TMA.
//
// Structure (tiles up to 128 wide): warps 0..7 = two MMA warpgroups (64 tile rows each, fp32 accumulators in registers)
// that then run the epilogue, warp 8 = TMA producer.  smem ring of `stages` {A 128x64, B block_n x 64} tiles (128-byte
// swizzle); after the main loop the fragments are staged as a row-major fp32 tile in shared memory, from which the
// epilogue warps read whole rows and write coalesced, while the producer already streams the next tile's operands into
// the ring.  192- and 256-wide tiles (gemm_wide_ok) run in a second kernel: a producer warpgroup, two consumer
// warpgroups with one m64nNk16 wgmma per k-step, and an epilogue straight from the accumulator registers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace pxr {

enum OperandMode : int { OP_KMAJOR = 0, OP_MNMAJOR = 1, OP_CONV = 2 };
// Code 3 is unassigned (it named the removed softmax epilogue) and stays refused.
// ACT_LRELU: LeakyReLU(0.2) after the bias.  ACT_LRELU_BWD: the sum (accumulator + bias + residual) times 1 where the saved
// post-activation aux_in is > 0, else 0.2, in the columns >= act_col0 (the others pass unmasked): the dense blocks of the
// super-resolution net mask one channel slice of a wider gradient (engine_superres.inc).
// ACT_GELU / ACT_GELU_BWD: exact (erf) GELU of timm's ViT MLP (nn.GELU()), the counterparts of the QuickGELU pair:
// forward stores the pre-activation u to aux_out as fp16 and returns gelu of exactly that fp16 value; backward multiplies
// the sum by Phi(u) + u phi(u) of the saved fp16 u.  Both are evaluated in fp32 (erfcf / expf).
// ACT_RELU / ACT_RELU_BWD: the CLIP ResNet blocks.  Forward: max(0, accumulator + bias + residual), the ReLU after the
// residual add (relu(main + identity) of a bottleneck).  Backward: the same sum where the saved post-activation aux_in is
// > 0, else 0.  Both run on the generic epilogue.
enum EpiAct : int {
  ACT_NONE = 0, ACT_QUICKGELU = 1, ACT_QUICKGELU_BWD = 2, ACT_LRELU = 4, ACT_LRELU_BWD = 5, ACT_GELU = 6, ACT_GELU_BWD = 7,
  ACT_RELU = 8, ACT_RELU_BWD = 9
};

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;
constexpr int GEMM_MAX_STAGES = 8;
constexpr int GEMM_THREADS = 288;  // warps 0..7 MMA + epilogue, warp 8 TMA
constexpr int GEMM_WIDE_THREADS = 384;  // 192- / 256-wide tiles: warpgroup 0 TMA, warpgroups 1..2 MMA + epilogue

struct GemmParams {
  CUtensorMap tma_a;
  CUtensorMap tma_b;
  // tiling
  int M, N;            // logical output extent per batch (predication)
  int block_n;         // multiple of 16, <= 128 (multiple of 64 when B is MN-major); or 192 / 256 (gemm_wide_ok)
  int stages;
  int num_k_blocks;    // taps * k_blocks_per_tap
  int k_blocks_per_tap;
  int num_taps;        // 1 or 9
  int tiles_m, tiles_n, total_tiles;
  int nb0;             // batch z -> (z % nb0, z / nb0)
  int a_mode, b_mode, b_batched;
  int b_tap_rows;      // conv: B row offset per tap
  int fmt;             // 0 = f16, 1 = bf16 (operand element type)
  // conv geometry (a_mode == OP_CONV): M tile = tile_h x tile_w pixels
  int conv_H, conv_W, tile_h, tile_w, tiles_w;
  // epilogue
  float alpha;
  const float* bias;
  int bias_per_row;
  int act;
  int act_col0;        // ACT_LRELU_BWD: first masked column
  const __half* aux_in;
  __half* aux_out;
  const float* res_f32;
  const __half* res_f16;
  float* out_f32;
  __half* out_f16;
  long long ldc, out_bs0, out_bs1;
  int vec_ok;          // 16-byte vector epilogue accesses allowed (alignment checked on host)
  // split-K (conv only): the "batch" index of a tile selects the k-block range [z * kb_per_split, ...) and the fp32
  // partial-sum slab z of the output workspace; k_splits == 1 otherwise
  int k_splits, kb_per_split;
  // tensor-map epilogue (tma_epi != TE_NONE): outputs leave through TMA stores of 32-row x 64-byte boxes staged in
  // shared memory in the accumulator's own row-per-lane layout; input tensors arrive the same way (prefetched)
  int tma_epi;
  CUtensorMap tma_c;   // main output (out_f16 / out_f32)
  CUtensorMap tma_d;   // second tensor: aux_out (TE_GELU), aux_in (TE_GELU_BWD), res_f32 (TE_RES32), res_f16 (TE_RES16)
};

// TE_GELU / TE_GELU_BWD: the activation pair with the saved pre-activation; QuickGELU (ACT_QUICKGELU*) as TE_GELU /
// TE_GELU_BWD, exact GELU (ACT_GELU*) as TE_ERF_GELU / TE_ERF_GELU_BWD -- one code path, specialised on the activation.
enum TmaEpi : int {
  TE_NONE = 0, TE_F16 = 1, TE_GELU = 2, TE_GELU_BWD = 3, TE_RES32 = 4, TE_RES16 = 5, TE_ERF_GELU = 6, TE_ERF_GELU_BWD = 7
};

// Host-side description of one operand.
struct GemmOperand {
  const void* ptr = nullptr;
  int mode = OP_KMAJOR;
  long long ld = 0;        // elements between consecutive rows of the stored matrix (pixel stride for conv)
  long long mn_extent = 0; // rows (M or N) visible to TMA (out-of-bounds rows read as zero)
  long long k_extent = 0;  // reduction extent visible to TMA
  int nb0 = 1, nb1 = 1;    // batch extents
  long long bs0 = 0, bs1 = 0;  // batch strides (elements)
};

struct GemmEpilogue {
  float alpha = 1.f;
  const float* bias = nullptr;
  int bias_per_row = 0;
  int act = ACT_NONE;
  int act_col0 = 0;   // ACT_LRELU_BWD only: columns below it are stored unmasked
  const __half* aux_in = nullptr;
  __half* aux_out = nullptr;
  const float* res_f32 = nullptr;
  const __half* res_f16 = nullptr;
  float* out_f32 = nullptr;
  __half* out_f16 = nullptr;
  long long ldc = 0, bs0 = 0, bs1 = 0;
  int tma_epi = 0;    // 0 = auto (tensor-map epilogue when the tensors allow it), -1 = force the generic epilogue
  int k_splits = 1;   // conv_plan_make only: > 1 writes fp32 partial sums [k_splits][pixels][ldc] to out_f32
};

struct GemmPlan {
  GemmParams p;
  int grid = 0;
  int smem_bytes = 0;
  double flops = 0;   // 2*M*N*K*batches (algorithmic)
  double bytes = 0;   // compulsory traffic: each operand read once, each epilogue tensor read / written once
};

// Whether a plain GEMM may use 192- or 256-column tiles (the 384-thread kernel of gemm_tc.cu): fp16, A K-major and
// unbatched, no split-K, and an epilogue the tensor-map path takes with fp16 outputs (bias, fp16 residual, QuickGELU
// forward / backward, exact GELU forward).  gemm_plan_make runs any other request wider than 128 columns as 128.
bool gemm_wide_ok(const GemmOperand& A, int N, const GemmEpilogue& epi, int fmt);

// Plain (possibly batched) GEMM.  K is the reduction length; M, N output extents per batch.
// Returns 0 on success; on failure writes a message to err (if non-null).
int gemm_plan_make(GemmPlan* plan, const GemmOperand& A, const GemmOperand& B, int M, int N, int K,
                   const GemmEpilogue& epi, int block_n, int fmt, int num_sms, char* err, int errlen);

// Implicit-GEMM convolution (ksize 1 or 3, stride 1, "same" zero padding) over NHWC activations:
//   out[b, h, w, n] = sum_{tap, c} in[b, h+dy(tap), w+dx(tap), c] * Wt[tap * cout_pad + n, c]
// `in` has c_in (multiple of 64) channels at pixel stride in_ld; `wt` is [taps * cout_pad, c_in] K-major.
int conv_plan_make(GemmPlan* plan, const void* in, long long in_ld, int batch, int H, int W, int c_in,
                   const void* wt, int cout_pad, int n_out, int ksize, const GemmEpilogue& epi, int block_n, int fmt,
                   int num_sms, char* err, int errlen);

void gemm_launch(const GemmPlan& plan, cudaStream_t stream);

// out[p, n] = fp16( sum_s ws[s][p][n] + bias[n] + res[p][n] ), n < N: the epilogue of a split-K convolution.
// ws: [splits][pixels][ld_ws] fp32; res / out: [pixels][ld_out] fp16 (res may be null); N, ld_* multiples of 8.
void splitk_reduce(const float* ws, int splits, long long pixels, int N, int ld_ws, const float* bias,
                   const __half* res, __half* out, int ld_out, cudaStream_t stream);

// 4-D tiled tensor map, zero fill out of bounds, 128-byte swizzle (fmt 0 = fp16, 1 = bf16, 2 = fp32); strides in elements.
// Returns 0 on success, otherwise writes a message to err.
int tmap_encode_4d(CUtensorMap* out, const void* ptr, int fmt, const uint64_t dims[4], const uint64_t strides_elems[3],
                   const uint32_t box[4], char* err, int errlen);

}  // namespace pxr
