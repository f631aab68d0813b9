// Streaming fused multi-head self-attention for sequences longer than attn_tc.cu stages (T > 240): the ViT-L/14@336px
// image tower (T = 577) and anything longer.  Same tensors and layouts as attn_tc.cuh (AttnParams), 64-wide heads, any
// B, H and T >= 1; sm_90a, warp-level mma.sync m16n8k16 (fp16 operands, fp32 accumulators), operands fed by ldmatrix.
//
// Flash-attention style, with K / V (backward: Q / dO) streamed through shared memory in 64-row tiles, double-buffered
// with cp.async, so shared memory no longer grows with T:
//   forward   CTA = 128 query rows of one (image, head) pair, each warp 32 of them (two 16-row MMA tiles share every K
//             and V fragment); online softmax in registers; writes O and the natural-log row log-sum-exp.
//   backward  two kernels, no atomics.  dQ: CTA = 128 query rows, streams K / V, forms D_i = dO_i . O_i for its rows
//             (stored to the plan's `delta` workspace) and accumulates dQ_i = scale sum_j dS_ij K_j.  dK / dV (launched
//             second): CTA = 128 key rows, streams Q / dO with their lse and D, accumulates dV_j = sum_i P_ij dO_i and
//             dK_j = scale sum_i dS_ij Q_i.  P = exp(S - lse) is recomputed in both from Q, K; dS = P o (dP - D).
// Rows and keys past T are zero-filled in shared memory and masked (T = 577 = 9 * 64 + 1).  Every output element is
// written by exactly one thread, so repeated runs are bit-identical.
#pragma once
#include "attn_tc.cuh"

namespace pxr {

struct AttnLongPlan {
  AttnParams p;
  float* delta = nullptr;  // backward workspace [B*H*T] (D_i = dO_i . O_i), owned by the caller
  double flops_fwd = 0, flops_bwd = 0;  // algorithmic: 2 / 4 T^2 d products per pair (recomputed S, dP not counted)
  double bytes_fwd = 0, bytes_bwd = 0;  // compulsory traffic, as AttnPlan
};

// true when the streaming kernels cover this shape (head width 64, T >= 1, 16-byte aligned rows)
bool attn_long_supported(int T, int head_dim, int W);
// qkv: [B*T, 3W]; o: [B*T, W]; d_o: [B*T, W]; gqkv: [B*T, 3W]; lse, delta: [B*H*T] (delta may be null without backward)
int attn_long_plan_make(AttnLongPlan* plan, const __half* qkv, __half* o, const __half* d_o, __half* gqkv, float* lse,
                        float* delta, int B, int T, int H, int W, float scale, char* err, int errlen);
void attn_long_forward_launch(const AttnLongPlan& plan, cudaStream_t st);
void attn_long_backward_launch(const AttnLongPlan& plan, cudaStream_t st);

}  // namespace pxr
