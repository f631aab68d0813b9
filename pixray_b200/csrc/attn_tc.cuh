// Fused multi-head self-attention of the CLIP ViT (nn.MultiheadAttention inside SLIP/models.py:18-64 residual blocks;
// openai-CLIP VisionTransformer) and of the v-diffusion U-Net for sm_90a: one kernel for the forward, one for the
// backward, both on the tensor cores (warp-level mma.sync m16n8k16, fp16 operands, fp32 accumulators in registers).
// Replaces, per layer, {QK^T GEMM, softmax, PV GEMM} and {dP GEMM, softmax backward, dQ / dK / dV GEMMs} of the unfused
// path.  Sequences longer than 257 tokens run on the streaming kernels of attn_long.cuh; 241..257 on the unfused path.
//
// Flash-attention style: a CTA owns one (image, head) pair -- or, with fewer pairs than SMs, a share of the pair's
// 16-row tiles -- and stages the pair's Q, K, V (backward: and dO) once in shared memory with cp.async; ldmatrix feeds
// the MMAs, .trans where an operand is needed transposed.  The scores of a warp's 16 rows live in registers and are never
// written to memory.  T is rounded up to 16, not further: key chunks and query tiles past T do no MMA work.  Forward
// keeps only the row log-sum-exp; backward recomputes P = exp(S - lse) from Q, K, takes D_i = dO_i . O_i once per row,
// and accumulates dK / dV over key tiles, then dQ over query tiles, in the same kernel.  Every output element is written
// by exactly one thread (no atomics), so results are deterministic.  With at least one pair per SM and T <= 208 the
// backward runs on attn_bwd_wg (attn_wg.cu), the wgmma kernel that forms every score product once.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pxr {

struct AttnParams {
  const __half* qkv;      // [B*T, 3W]: q | k | v, head h at columns h*64 of each third
  __half* o;              // forward out / backward in: [B*T, W]
  float* lse;             // [B*H, T] natural-log sum-exp of the scaled scores
  const __half* d_o;      // backward in [B*T, W]
  __half* gqkv;           // backward out [B*T, 3W]: dq | dk | dv
  int T, H, B, W;
  float scale;            // S = scale * q k^T
  int causal;             // forward only: row q attends to keys <= q (the text towers' mask); 0 in every ViT / U-Net block
};

// attn_bwd_wg's operands (attn_wg.cu): tensor maps over qkv viewed as (3W columns, T rows, B images) with 64- and
// 16-row boxes, and over dO viewed as (W, T, B) with 16-row boxes; 64 columns per box, 128-byte swizzle, rows >= T of an
// image read as zeros.
struct AttnWgArgs {
  CUtensorMap kv, q, d_o;
  AttnParams p;
};

enum { ATTN_BWD_AUTO = 0, ATTN_BWD_MMA = 1, ATTN_BWD_WG = 2 };

struct AttnPlan {
  AttnParams p;
  int splits = 1;  // CTAs per (image, head) pair
  int bwd = ATTN_BWD_MMA;  // the backward kernel: attn_bwd_kernel (ATTN_BWD_MMA) or attn_bwd_wg (ATTN_BWD_WG)
  AttnWgArgs wg;
  int smem_fwd = 0, smem_bwd = 0;
  double flops_fwd = 0, flops_bwd = 0;
  double bytes_fwd = 0, bytes_bwd = 0;  // compulsory traffic: qkv in, o out (+ lse) / qkv, o, dO in, dqkv out
};

// true when the fused kernels cover this shape (head width 64, T <= 240, 16-byte aligned rows)
bool attn_supported(int T, int head_dim, int W);
// qkv: [B*T, 3W]; o: [B*T, W]; d_o: [B*T, W]; gqkv: [B*T, 3W]; lse: [B*H*T].  causal: the forward masks keys after each
// row (the backward kernel has no mask: a causal plan is forward only).  bwd: ATTN_BWD_AUTO takes attn_bwd_wg for a
// non-causal backward with at least one (image, head) pair per SM and T <= 208 (attn_bwd_wg_fits), attn_bwd_kernel
// otherwise; ATTN_BWD_MMA / ATTN_BWD_WG force one (the latter fails where it cannot run; the engine forces the former
// with PXR_ATTN_BWD=mma).
int attn_plan_make(AttnPlan* plan, const __half* qkv, __half* o, const __half* d_o, __half* gqkv, float* lse, int B,
                   int T, int H, int W, float scale, int num_sms, char* err, int errlen, bool causal = false,
                   int bwd = ATTN_BWD_AUTO);
void attn_forward_launch(const AttnPlan& plan, cudaStream_t st);
void attn_backward_launch(const AttnPlan& plan, cudaStream_t st);

// attn_wg.cu: the wgmma backward for one (image, head) pair per CTA
bool attn_bwd_wg_fits(int T);  // its shared memory holds the pair (T <= 208)
int attn_bwd_wg_prepare(AttnPlan* plan, char* err, int errlen);  // encodes plan->wg from plan->p
void attn_bwd_wg_launch(const AttnPlan& plan, cudaStream_t st);

}  // namespace pxr
