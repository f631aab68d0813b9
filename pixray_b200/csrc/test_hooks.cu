// C-ABI test hooks: expose single kernels of the engine so tests/ can check each against the oracle / torch.
// These are not part of the reference-facing surface (include/pixray_b200.h lists them under "test hooks").
#include "../../include/pixray_b200.h"
#include "gemm_tc.cuh"
#include "attn_tc.cuh"
#include "attn_long.cuh"
#include "color_jitter.cuh"
#include "pool_bounds.cuh"
#include "raster_samples.cuh"
#include "kernels.cuh"
#include <cstdio>
#include <cstring>

using namespace pxr;

static int g_num_sms = 0;
static int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

static void fill_epilogue(GemmEpilogue& e, const pxr_test_gemm_desc* d) {
  e.alpha = d->alpha;
  e.bias = d->bias;
  e.bias_per_row = d->bias_per_row;
  e.act = d->act;
  e.aux_in = static_cast<const __half*>(d->aux_in);
  e.aux_out = static_cast<__half*>(d->aux_out);
  e.res_f32 = d->res_f32;
  e.res_f16 = static_cast<const __half*>(d->res_f16);
  e.out_f32 = d->out_f32;
  e.out_f16 = static_cast<__half*>(d->out_f16);
  e.ldc = d->ldc;
  e.bs0 = d->c_bs0;
  e.bs1 = d->c_bs1;
  e.tma_epi = d->tma_epi;
  e.act_col0 = d->act_col0;
  e.k_splits = d->k_splits;
}

// the plan pxr_test_gemm runs for a descriptor (B takes A's batch extents when b_batched)
static int desc_plan(GemmPlan* plan, const pxr_test_gemm_desc* d, char* err, int errlen) {
  GemmOperand A, B;
  A.ptr = d->a;
  A.mode = d->a_mode;
  A.ld = d->lda;
  A.mn_extent = d->a_mn_extent;
  A.k_extent = d->a_k_extent;
  A.nb0 = d->nb0;
  A.nb1 = d->nb1;
  A.bs0 = d->a_bs0;
  A.bs1 = d->a_bs1;
  B.ptr = d->b;
  B.mode = d->b_mode;
  B.ld = d->ldb;
  B.mn_extent = d->b_mn_extent;
  B.k_extent = d->b_k_extent;
  B.nb0 = d->b_batched ? d->nb0 : 1;
  B.nb1 = d->b_batched ? d->nb1 : 1;
  B.bs0 = d->b_bs0;
  B.bs1 = d->b_bs1;
  GemmEpilogue e;
  fill_epilogue(e, d);
  return gemm_plan_make(plan, A, B, d->M, d->N, d->K, e, d->block_n, d->fmt, num_sms(), err, errlen);
}

extern "C" int pxr_test_gemm(const pxr_test_gemm_desc* d, char* err, int errlen) {
  GemmPlan plan;
  int rc = desc_plan(&plan, d, err, errlen);
  if (rc) return rc;
  for (int i = 0; i < (d->repeat > 0 ? d->repeat : 1); ++i) gemm_launch(plan, static_cast<cudaStream_t>(d->stream));
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) {
    if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
    return -100;
  }
  return 0;
}

extern "C" int pxr_test_gemm_plan_info(const pxr_test_gemm_desc* d, int out[6]) {
  GemmPlan plan;
  int rc = desc_plan(&plan, d, nullptr, 0);
  if (rc) return rc;
  const int info[6] = {plan.p.wide, plan.p.block_n, plan.p.stages, plan.p.tma_epi, plan.grid, plan.p.k_splits};
  for (int i = 0; i < 6; ++i) out[i] = info[i];
  return 0;
}

extern "C" int pxr_test_conv(const pxr_test_gemm_desc* d, int batch, int H, int W, int c_in, int cout_pad, int ksize,
                             char* err, int errlen) {
  GemmEpilogue e;
  fill_epilogue(e, d);
  GemmPlan plan;
  int rc = conv_plan_make(&plan, d->a, d->lda, batch, H, W, c_in, d->b, cout_pad, d->N, ksize, e, d->block_n, d->fmt,
                          num_sms(), err, errlen, !d->narrow_kernel);
  if (rc) return rc;
  for (int i = 0; i < (d->repeat > 0 ? d->repeat : 1); ++i) gemm_launch(plan, static_cast<cudaStream_t>(d->stream));
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) {
    if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
    return -100;
  }
  return 0;
}

extern "C" int pxr_test_conv_plan_info(const pxr_test_gemm_desc* d, int batch, int H, int W, int c_in, int cout_pad,
                                       int ksize, int out[6]) {
  GemmEpilogue e;
  fill_epilogue(e, d);
  GemmPlan plan;
  int rc = conv_plan_make(&plan, d->a, d->lda, batch, H, W, c_in, d->b, cout_pad, d->N, ksize, e, d->block_n, d->fmt,
                          num_sms(), nullptr, 0, !d->narrow_kernel);
  if (rc) return rc;
  const int info[6] = {plan.p.wide, plan.p.block_n, plan.p.stages, plan.p.tma_epi, plan.grid, plan.p.k_splits};
  for (int i = 0; i < 6; ++i) out[i] = info[i];
  return 0;
}

static int sync_status() {
  cudaError_t ce = cudaDeviceSynchronize();
  if (ce == cudaSuccess) ce = cudaGetLastError();
  return ce == cudaSuccess ? 0 : -100;
}

// splitk_reduce on caller DEVICE tensors: ws [splits][pixels][ld_ws] fp32 -> out [pixels][ld_out] fp16 (+ bias, + res)
extern "C" int pxr_test_splitk_reduce(const float* ws, int splits, long long pixels, int N, int ld_ws, const float* bias,
                                      const void* res, void* out, int ld_out) {
  if (!ws || !out || splits < 1 || pixels < 1 || N < 8 || N % 8 || ld_ws < N || ld_ws % 8 || ld_out < N || ld_out % 8)
    return -1;
  splitk_reduce(ws, splits, pixels, N, ld_ws, bias, static_cast<const __half*>(res), static_cast<__half*>(out), ld_out,
                nullptr);
  return sync_status();
}

// The Prompt loss kernel (prompt_loss, kernels_clip.cu) on caller DEVICE tensors: e [B, D] -> e_unit [B, D], losses
// [max slot + 1] (summed into: the caller zeroes them), de [B, D] fp32 and de16 [B, D] fp16 (nullable).
extern "C" int pxr_test_prompt_loss(const float* e, int B, int D, const float* prompts, const float* weights,
                                    const float* stops, const int* slots, const float* inv_rows, int n, int cutn_global,
                                    float grad_scale, float* e_unit, float* losses, float* de, void* de16) {
  if (!e || !de || B < 1 || D < 1 || n < 0 || cutn_global < 1 || (n > 0 && (!prompts || !weights || !stops || !losses)))
    return -1;
  float* part = nullptr;
  unsigned int* count = nullptr;
  if (n > 0 && (cudaMalloc(&part, sizeof(float) * B * n) != cudaSuccess || cudaMalloc(&count, sizeof(unsigned int)) != cudaSuccess ||
                cudaMemset(count, 0, sizeof(unsigned int)) != cudaSuccess)) {
    cudaFree(part);
    return -100;
  }
  prompt_loss(e, B, D, prompts, weights, stops, slots, inv_rows, n, cutn_global, grad_scale, e_unit, losses, de,
              static_cast<act_t*>(de16), part, count, nullptr);
  const int rc = sync_status();
  cudaFree(part);
  cudaFree(count);
  return rc;
}

// Fused attention forward (+ backward when d_o != NULL) on caller tensors: qkv [B*T, 3W] fp16, o [B*T, W] fp16,
// lse [B*H*T] fp32, d_o [B*T, W] fp16, gqkv [B*T, 3W] fp16.
extern "C" int pxr_test_attention(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B, int T, int H,
                                  int W, float scale, int repeat, char* err, int errlen) {
  AttnPlan plan;
  int rc = attn_plan_make(&plan, static_cast<const __half*>(qkv), static_cast<__half*>(o),
                          static_cast<const __half*>(d_o), static_cast<__half*>(gqkv), lse, B, T, H, W, scale,
                          num_sms(), err, errlen);
  if (rc) return rc;
  for (int i = 0; i < (repeat > 0 ? repeat : 1); ++i) {
    attn_forward_launch(plan, nullptr);
    if (d_o) attn_backward_launch(plan, nullptr);
  }
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) {
    if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
    return -100;
  }
  return 0;
}

// As pxr_test_attention, with the backward kernel chosen by bwd_kernel (0: as the engine chooses, 1: attn_bwd_kernel,
// 2: attn_bwd_wg): the forward once, then the backward `repeat` times (none for repeat 0).  *used (nullable) receives the
// backward kernel the plan took (1 or 2).
extern "C" int pxr_test_attention_bwd_select(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B,
                                             int T, int H, int W, float scale, int bwd_kernel, int repeat, int* used,
                                             char* err, int errlen) {
  if (!d_o || !gqkv || bwd_kernel < 0 || bwd_kernel > 2) {
    if (err && errlen > 0) snprintf(err, errlen, "needs d_o, gqkv and a backward kernel 0, 1 or 2");
    return -1;
  }
  AttnPlan plan;
  int rc = attn_plan_make(&plan, static_cast<const __half*>(qkv), static_cast<__half*>(o),
                          static_cast<const __half*>(d_o), static_cast<__half*>(gqkv), lse, B, T, H, W, scale,
                          num_sms(), err, errlen, false, bwd_kernel);
  if (rc) return rc;
  if (used) *used = plan.bwd;
  attn_forward_launch(plan, nullptr);
  for (int i = 0; i < repeat; ++i) attn_backward_launch(plan, nullptr);
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) {
    if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
    return -100;
  }
  return 0;
}

// Causal attention forward on caller tensors, on the path the engine's add_attention takes: the fused kernel, or with
// PXR_FUSED_ATTN=0 the batched-GEMM chain S = scale q k^T -> causal row softmax -> O = P v (P allocated here).
extern "C" int pxr_test_attention_causal(const void* qkv, void* o, int B, int T, int H, int W, float scale, char* err,
                                         int errlen) {
  if (!qkv || !o || B < 1 || H < 1 || !attn_supported(T, W / H, W) || W != 64 * H) {
    if (err && errlen > 0) snprintf(err, errlen, "causal attention needs 64-wide heads and 1 <= T <= 240");
    return -1;
  }
  const char* fa = getenv("PXR_FUSED_ATTN");
  const __half* q = static_cast<const __half*>(qkv);
  if (!(fa && atoi(fa) == 0)) {
    float* lse = nullptr;
    if (cudaMalloc(&lse, sizeof(float) * B * H * T) != cudaSuccess) return -100;
    AttnPlan plan;
    int rc = attn_plan_make(&plan, q, static_cast<__half*>(o), nullptr, nullptr, lse, B, T, H, W, scale, num_sms(), err,
                            errlen, true);
    if (!rc) {
      attn_forward_launch(plan, nullptr);
      rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : -100;
    }
    cudaFree(lse);
    return rc;
  }
  const int ldT = (T + 7) / 8 * 8, rows = B * H * T;
  // (head, sequence) batch strides of qkv, o and P, as add_attention lays them out
  const long long qs0 = 64, qs1 = (long long)T * 3 * W, os0 = 64, os1 = (long long)T * W;
  const long long ps0 = (long long)T * ldT, ps1 = (long long)H * T * ldT;
  auto op = [&](const void* p, int mode, long long ld, long long mn, long long k, long long bs0, long long bs1) {
    GemmOperand g;
    g.ptr = p;
    g.mode = mode;
    g.ld = ld;
    g.mn_extent = mn;
    g.k_extent = k;
    g.nb0 = H;
    g.nb1 = B;
    g.bs0 = bs0;
    g.bs1 = bs1;
    return g;
  };
  __half* P = nullptr;
  if (cudaMalloc(&P, sizeof(__half) * rows * ldT) != cudaSuccess) return -100;
  GemmPlan s_plan, o_plan;
  GemmEpilogue es, eo;
  es.alpha = scale;
  es.out_f16 = P;
  es.ldc = ldT;
  es.bs0 = ps0;
  es.bs1 = ps1;
  eo.out_f16 = static_cast<__half*>(o);
  eo.ldc = W;
  eo.bs0 = os0;
  eo.bs1 = os1;
  const int bn_s = T <= 32 ? (T + 15) / 16 * 16 : T <= 128 ? (T + 63) / 64 * 64 : 128;
  int rc = gemm_plan_make(&s_plan, op(q, OP_KMAJOR, 3 * W, T, 64, qs0, qs1), op(q + W, OP_KMAJOR, 3 * W, T, 64, qs0, qs1),
                          T, T, 64, es, bn_s, 0, num_sms(), err, errlen);
  if (!rc)
    rc = gemm_plan_make(&o_plan, op(P, OP_KMAJOR, ldT, T, ldT, ps0, ps1), op(q + 2 * W, OP_MNMAJOR, 3 * W, 64, T, qs0, qs1),
                        T, 64, T, eo, 64, 0, num_sms(), err, errlen);
  if (!rc) {
    gemm_launch(s_plan, nullptr);
    rc = softmax_forward_causal(P, rows, T, ldT, nullptr);
    if (!rc) gemm_launch(o_plan, nullptr);
    if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = -100;
  }
  cudaFree(P);
  return rc;
}

// A fused or streaming attention record's plan, rebuilt through attn_plan_make / attn_long_plan_make on caller tensors
// (the record's own pointers are not touched), run once.
extern "C" int pxr_test_attention_plan(const pxr_test_attn_rec* r, const void* qkv, void* o, const void* d_o, void* gqkv,
                                       float* lse, float* delta, int bwd_kernel, int out2[2], char* err, int errlen) {
  if (!r || !qkv || !o || !lse || !out2 || (r->path != PXR_ATTN_FUSED && r->path != PXR_ATTN_STREAMING)) {
    if (err && errlen > 0) snprintf(err, errlen, "needs a fused or streaming record, qkv, o, lse and out2");
    return -1;
  }
  const __half* q = static_cast<const __half*>(qkv);
  __half* oh = static_cast<__half*>(o);
  const __half* g = static_cast<const __half*>(d_o);
  __half* gq = static_cast<__half*>(gqkv);
  int rc;
  if (r->path == PXR_ATTN_FUSED) {
    AttnPlan plan;
    rc = attn_plan_make(&plan, q, oh, g, gq, lse, r->images, r->T, r->heads, r->W, r->scale, num_sms(), err, errlen,
                        r->causal != 0, bwd_kernel);
    if (rc) return rc;
    out2[0] = plan.splits;
    out2[1] = plan.bwd;
    attn_forward_launch(plan, nullptr);
    if (d_o && gqkv) attn_backward_launch(plan, nullptr);
  } else {
    AttnLongPlan plan;
    rc = attn_long_plan_make(&plan, q, oh, g, gq, lse, delta, r->images, r->T, r->heads, r->W, r->scale, err, errlen);
    if (rc) return rc;
    out2[0] = 1;
    out2[1] = 0;
    attn_long_forward_launch(plan, nullptr);
    if (d_o && gqkv) attn_long_backward_launch(plan, nullptr);
  }
  cudaError_t ce = cudaDeviceSynchronize();
  if (ce == cudaSuccess) ce = cudaGetLastError();
  if (ce != cudaSuccess) {
    if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
    return -100;
  }
  return 0;
}

// Streaming fused attention (attn_long.cu) on the same caller tensors as pxr_test_attention; the backward's D workspace
// [B*H*T] fp32 is allocated here.
extern "C" int pxr_test_attention_long(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B, int T,
                                       int H, int W, float scale, int repeat, char* err, int errlen) {
  float* delta = nullptr;
  if (d_o && B > 0 && T > 0 && H > 0 && cudaMalloc(&delta, sizeof(float) * B * H * T) != cudaSuccess) {
    if (err) snprintf(err, errlen, "cudaMalloc of the delta workspace failed");
    return -100;
  }
  AttnLongPlan plan;
  int rc = attn_long_plan_make(&plan, static_cast<const __half*>(qkv), static_cast<__half*>(o),
                               static_cast<const __half*>(d_o), static_cast<__half*>(gqkv), lse, delta, B, T, H, W, scale,
                               err, errlen);
  if (!rc) {
    for (int i = 0; i < (repeat > 0 ? repeat : 1); ++i) {
      attn_long_forward_launch(plan, nullptr);
      if (d_o) attn_long_backward_launch(plan, nullptr);
    }
    cudaError_t ce = cudaGetLastError();
    if (ce == cudaSuccess && delta) ce = cudaDeviceSynchronize();  // the workspace is freed below
    if (ce != cudaSuccess) {
      if (err) snprintf(err, errlen, "launch failed: %s", cudaGetErrorString(ce));
      rc = -100;
    }
  }
  cudaFree(delta);
  return rc;
}

// The engine's row softmax (softmax_forward / softmax_forward_causal / softmax_backward, unfused attention) on caller
// DEVICE fp16 [rows, ld]: op 0 / 2: p_or_s holds the scores and is overwritten with the probabilities (2: causal);
// op 1: p_or_s holds P and dp holds dP, overwritten with dS = P * (dP - <P, dP>).
extern "C" int pxr_test_softmax(int op, void* p_or_s, void* dp, int rows, int cols, int ld) {
  if (!p_or_s || rows < 1 || cols < 1 || ld < cols || ld % 8 || op < 0 || op > 2 || (op == 1 && !dp)) return -1;
  if (op == 1) softmax_backward(static_cast<const act_t*>(p_or_s), static_cast<act_t*>(dp), rows, cols, ld, nullptr);
  else if (op == 2) {
    if (softmax_forward_causal(static_cast<act_t*>(p_or_s), rows, cols, ld, nullptr)) return -1;
  } else softmax_forward(static_cast<act_t*>(p_or_s), rows, cols, ld, nullptr);
  cudaError_t ce = cudaDeviceSynchronize();
  if (ce == cudaSuccess) ce = cudaGetLastError();
  return ce == cudaSuccess ? 0 : -100;
}

// One LayerNorm kernel chosen by `variant` (0: fp32 stream, 1: fp16 stream 8-byte vectors, 2: fp16 stream 16-byte
// vectors) whatever PXR_LN16_WIDE says, forward (x, pos, gamma, beta -> y16 / y32, stats) or backward (dy, x, pos, stats,
// gamma -> gx / gx16, accumulate adds to what they hold).  All DEVICE; x is fp32 for variant 0 and fp16 otherwise.
// -1 when that variant has no kernel for the width or the arguments.
extern "C" int pxr_test_layernorm(int variant, int backward, const void* x, long long x_stride, const float* pos, int T,
                                  const float* gamma, const float* beta, int rows, int W, float eps, void* y16, float* y32,
                                  float* stats, const void* dy, int accumulate, float* gx, void* gx16) {
  if (!x || !gamma || !stats || rows < 1 || (pos && T < 1)) return -2;
  int rc;
  if (backward)
    rc = layernorm_backward_variant(variant, static_cast<const act_t*>(dy), x, x_stride, pos, T, stats, gamma, rows, W,
                                    accumulate, gx, static_cast<act_t*>(gx16), nullptr);
  else
    rc = layernorm_forward_variant(variant, x, x_stride, pos, T, gamma, beta, rows, W, eps, static_cast<act_t*>(y16), y32,
                                   stats, nullptr);
  if (rc) return rc;
  cudaError_t ce = cudaDeviceSynchronize();
  if (ce == cudaSuccess) ce = cudaGetLastError();
  return ce == cudaSuccess ? 0 : -100;
}

// Host evaluation of the per-pixel ColorJitter body the cutout kernels run (color_jitter.cuh is host+device code):
// lets the CPU suite compare the arithmetic and its Jacobian with the oracle without a GPU.  rgb / g_out / out / g_in
// are HOST [n, 3]; g_out and g_in may be NULL.
extern "C" int pxr_test_color_jitter_host(const float* rgb, int n, int code, float saturation, float hue,
                                          const float* g_out, float* out, float* g_in) {
  if (!rgb || !out || n < 0) return -1;
  for (int i = 0; i < n; ++i) {
    float c[3] = {rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]};
    pxr::cj_apply(c, code, saturation, hue);
    for (int k = 0; k < 3; ++k) out[3 * i + k] = c[k];
    if (g_out && g_in) pxr::cj_vjp(rgb + 3 * i, code, saturation, hue, g_out + 3 * i, g_in + 3 * i);
  }
  return 0;
}

// The same body on the device (what cutout_fwd / cutout_bwd execute per pixel), for a device-vs-host comparison of the
// forward and of the vector-Jacobian product.  rgb / g_out / out / g_in are DEVICE [n, 3].
namespace {
__global__ void color_jitter_device_kernel(const float* rgb, int n, int code, float saturation, float hue,
                                           const float* g_out, float* out, float* g_in) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float in[3] = {rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]};
  float c[3] = {in[0], in[1], in[2]};
  pxr::cj_apply(c, code, saturation, hue);
  for (int k = 0; k < 3; ++k) out[3 * i + k] = c[k];
  if (g_out && g_in) {
    const float go[3] = {g_out[3 * i], g_out[3 * i + 1], g_out[3 * i + 2]};
    float gi[3];
    pxr::cj_vjp(in, code, saturation, hue, go, gi);
    for (int k = 0; k < 3; ++k) g_in[3 * i + k] = gi[k];
  }
}
}  // namespace

extern "C" int pxr_test_color_jitter_device(const float* rgb, int n, int code, float saturation, float hue,
                                            const float* g_out, float* out, float* g_in) {
  if (!rgb || !out || n < 0) return -1;
  if (n == 0) return 0;
  color_jitter_device_kernel<<<(n + 255) / 256, 256>>>(rgb, n, code, saturation, hue, g_out, out, g_in);
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : -2;
}

// The adaptive-pool window bounds as the DEVICE computes them (pool_bounds.cuh, the functions pool_fwd / pool_bwd call):
// starts / ends are DEVICE int [out_size].  Integer bookkeeping: the test asserts equality with ATen's formula.
namespace {
__global__ void pool_bounds_kernel(int in_size, int out_size, int* starts, int* ends) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_size) return;
  starts[i] = pxr::pool_start(i, in_size, out_size);
  ends[i] = pxr::pool_end(i, in_size, out_size);
}
}  // namespace

extern "C" int pxr_test_pool_bounds(int in_size, int out_size, int* starts, int* ends) {
  if (in_size < 1 || out_size < 1 || !starts || !ends) return -1;
  pool_bounds_kernel<<<(out_size + 255) / 256, 256>>>(in_size, out_size, starts, ends);
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : -2;
}

// The polygon rasteriser's sample positions from the function its kernels call (raster_samples.cuh): DEVICE float
// [H, W, 4, 2].
namespace {
__global__ void raster_samples_kernel(uint64_t seed, int iter, int H, int W, float* out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  for (int s = 0; s < 4; ++s) pxr::raster_sample(seed, iter, p % W, p / W, W, s, out[(size_t)p * 8 + 2 * s], out[(size_t)p * 8 + 2 * s + 1]);
}
}  // namespace

extern "C" int pxr_test_raster_samples(uint64_t seed, int iter, int H, int W, float* out) {
  if (H < 1 || W < 1 || !out) return -1;
  raster_samples_kernel<<<(H * W + 255) / 256, 256>>>(seed, iter, H, W, out);
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : -2;
}

// GroupNorm(32, C, eps 1e-6)(+ swish) forward, and backward when dy (or ws_dy) is given, on caller DEVICE tensors
// (NHWC fp16 [pixels, C]).  variant 0: the single-kernel grid-barrier GroupNorm; 1: one cluster per group
// (kernels_gn_group.cu); 2: the three-kernel GroupNorm (gn_stats + gn_apply, gn_backward).  variant 1 only: ws != NULL
// makes the forward the epilogue of a split-K convolution (x_out = fp16(sum_s ws[s] + bias + res), then normalised);
// ws_dy != NULL feeds the backward from split-K partials.
// scratch: variants 0 / 1: >= 64 * (num_sms + 2) floats + one zero-initialised u64 at its END (variant 0's grid barrier);
// variant 2: 2 * 64 * gn_num_partials(pixels, C) partials, then the 64 floats of the backward's gstats (no barrier word).
extern "C" int pxr_test_groupnorm(int variant, const void* x, const float* ws, int splits, const float* bias, const void* res,
                                  void* x_out, const float* gamma, const float* beta, int pixels, int C, int swish, void* y,
                                  float* stats, const void* dy, const float* ws_dy, int splits_dy, const void* dres, void* dx,
                                  float* scratch, int repeat) {
  const act_t* xin = static_cast<const act_t*>(x);
  const int nsm = num_sms();
  GridBarrier gb;  // the caller hands in a zeroed counter with every call
  gb.counter = reinterpret_cast<unsigned long long*>(scratch + 64 * (nsm + 2));
  if (variant == 0) {
    if (ws || ws_dy || !gn_coop_supported(pixels, C, nsm)) return -1;
  } else if (variant == 2) {
    // gn_partial_kernel: 256 threads = whole pixel lanes x C/8 vectors; a group is 4 channels or whole vectors
    if (ws || ws_dy || !x || pixels < 1 || C < 32 || C % 32 || 256 % (C / 8) || (C / 32 != 4 && (C / 32) % 8)) return -1;
  } else {
    if (!gn_group_possible(pixels, C)) return -2;
  }
  for (int it = 0; it < (repeat > 0 ? repeat : 1); ++it) {
    if (variant == 2) {
      float* gstats = scratch + 2 * 64 * gn_num_partials(pixels, C);
      gn_stats(xin, pixels, C, 1e-6f, scratch, stats, nullptr);
      gn_apply(xin, stats, gamma, beta, pixels, C, swish, static_cast<act_t*>(y), nullptr);
      if (dy)
        gn_backward(static_cast<const act_t*>(dy), xin, stats, gamma, beta, pixels, C, swish, static_cast<const act_t*>(dres),
                    scratch, gstats, static_cast<act_t*>(dx), nullptr);
    } else if (variant == 0) {
      gn_forward_coop(xin, gamma, beta, pixels, C, swish, 1e-6f, scratch, stats, static_cast<act_t*>(y), nsm, &gb, nullptr);
      if (dy)
        gn_backward_coop(static_cast<const act_t*>(dy), xin, stats, gamma, beta, pixels, C, swish,
                         static_cast<const act_t*>(dres), scratch, static_cast<act_t*>(dx), nsm, &gb, nullptr);
    } else {
      GnSplitK sk, skd;
      sk.ws = ws;
      sk.splits = splits;
      sk.ld_ws = C;
      sk.bias = bias;
      sk.res = static_cast<const act_t*>(res);
      sk.out = static_cast<act_t*>(x_out);
      skd.ws = ws_dy;
      skd.splits = splits_dy;
      skd.ld_ws = C;
      gn_forward_group(xin, ws ? &sk : nullptr, gamma, beta, pixels, C, swish, 1e-6f, stats, static_cast<act_t*>(y), nullptr);
      const act_t* xs = ws ? static_cast<const act_t*>(x_out) : xin;
      if (dy || ws_dy)
        gn_backward_group(static_cast<const act_t*>(dy), ws_dy ? &skd : nullptr, xs, stats, gamma, beta, pixels, C, swish,
                          static_cast<const act_t*>(dres), static_cast<act_t*>(dx), nullptr);
    }
  }
  return sync_status();
}

// The U-Net's GroupNorm(1, C) + modulation (+ activation, + residual) exactly as Engine::vd_norm / vd_norm_bwd call the
// grid-barrier kernels; scratch as variant 0 above.
extern "C" int pxr_test_groupnorm_unet(const void* x, const float* gamma, const float* beta, float gamma_add, int act,
                                       const void* res, float eps, int pixels, int C, void* y, float* stats, const void* dy,
                                       const void* dres, void* dx, float* scratch) {
  const int nsm = num_sms();
  if (!x || !y || !stats || !scratch || act < 0 || act > 2 || (dy && !dx) || !gn_coop_supported(pixels, C, nsm)) return -1;
  GridBarrier gb;
  gb.counter = reinterpret_cast<unsigned long long*>(scratch + 64 * (nsm + 2));
  GnOpts o;
  o.one_group = 1;
  o.gamma_add = gamma_add;
  o.res = static_cast<const act_t*>(res);
  const act_t* xin = static_cast<const act_t*>(x);
  gn_forward_coop(xin, gamma, beta, pixels, C, act, eps, scratch, stats, static_cast<act_t*>(y), nsm, &gb, nullptr, o);
  if (dy) {
    o.res = nullptr;  // the residual is a forward-only term: its gradient is dy itself, added by the caller
    gn_backward_coop(static_cast<const act_t*>(dy), xin, stats, gamma, beta, pixels, C, act, static_cast<const act_t*>(dres),
                     scratch, static_cast<act_t*>(dx), nsm, &gb, nullptr, o);
  }
  return sync_status();
}

// The same on either path vd_norm / vd_norm_bwd choose from: 0 the grid-barrier kernel (as above), 1 the three kernels.
extern "C" int pxr_test_groupnorm_unet_path(int path, const void* x, const float* gamma, const float* beta, float gamma_add,
                                            int act, const void* res, float eps, int pixels, int C, void* y, float* stats,
                                            const void* dy, const void* dres, void* dx, float* scratch) {
  if (path == 0) return pxr_test_groupnorm_unet(x, gamma, beta, gamma_add, act, res, eps, pixels, C, y, stats, dy, dres, dx, scratch);
  if (path != 1 || !x || !y || !stats || !scratch || act < 0 || act > 2 || (dy && !dx) || pixels < 1 || C < 32 || C % 32 ||
      256 % (C / 8) || (C / 32 != 4 && (C / 32) % 8))
    return -1;
  GnOpts o;
  o.one_group = 1;
  o.gamma_add = gamma_add;
  o.res = static_cast<const act_t*>(res);
  const act_t* xin = static_cast<const act_t*>(x);
  gn_stats(xin, pixels, C, eps, scratch, stats, nullptr, o);
  gn_apply(xin, stats, gamma, beta, pixels, C, act, static_cast<act_t*>(y), nullptr, o);
  if (dy) {
    o.res = nullptr;
    float* gstats = scratch + 2 * 64 * gn_num_partials(pixels, C);
    gn_backward(static_cast<const act_t*>(dy), xin, stats, gamma, beta, pixels, C, act, static_cast<const act_t*>(dres),
                scratch, gstats, static_cast<act_t*>(dx), nullptr, o);
  }
  return sync_status();
}

extern "C" int pxr_test_groupnorm_partials(int pixels, int C) {
  return pixels < 1 ? -1 : gn_num_partials(pixels, C);
}

// One resampling / copy launcher chosen by `op` (include/pixray_b200.h lists the ops and their layouts).
extern "C" int pxr_test_resample(int op, const void* in, int ld_in, void* out, int ld_out, int H, int W, int C, int accumulate) {
  if (!in || !out || C < 8 || C % 8 || H < 1 || W < 1) return -1;
  if (ld_in == 0) ld_in = C;
  if (ld_out == 0) ld_out = C;
  if (ld_in < C || ld_in % 8 || ld_out < C || ld_out % 8) return -1;
  // which side of each op takes a pixel stride, and whether it accumulates
  static const struct { bool ld_in, ld_out, acc; } caps[8] = {
      {true, false, false}, {false, false, false}, {true, false, false}, {false, false, true},
      {false, true, false}, {true, false, false},  {false, false, false}, {true, true, true}};
  if (op < 0 || op > 7) return -2;
  if ((!caps[op].ld_in && ld_in != C) || (!caps[op].ld_out && ld_out != C) || (!caps[op].acc && accumulate)) return -3;
  const act_t* x = static_cast<const act_t*>(in);
  act_t* y = static_cast<act_t*>(out);
  switch (op) {
    case 0: upsample2x(x, H, W, C, y, nullptr, ld_in); break;
    case 1: downsum2x(x, H, W, C, y, nullptr); break;
    case 2: avgpool2x(x, H, W, C, ld_in, y, nullptr); break;
    case 3: avgpool2x_backward(x, H, W, C, accumulate, y, nullptr); break;
    case 4: bilinear_up2x(x, H, W, C, y, ld_out, nullptr); break;
    case 5: bilinear_up2x_backward(x, H, W, C, ld_in, y, nullptr); break;
    case 6: im2col3x3(x, H, W, C, y, nullptr); break;
    default: copy_channels(x, ld_in, y, ld_out, C, (long long)H * W, accumulate, nullptr); break;
  }
  return sync_status();
}

extern "C" int pxr_test_gemv(const void* w, int K, int R, const float* x, const float* bias, int relu, const float* res,
                             float* y) {
  if (!w || !x || !y || K < 8 || K % 8 || R < 1) return -1;
  gemv_f16(static_cast<const act_t*>(w), K, R, x, bias, relu, res, y, nullptr);
  return sync_status();
}
