// Launchers of the non-GEMM kernels of the hot path (gather / pointwise / reduction; HBM-bound).
// Every launcher enqueues on `st` and returns; none synchronises.  Layouts: decoder activations are NHWC fp16
// ([pixels, C], C a multiple of 64); the CLIP residual stream is fp32 [tokens, W]; images are planar fp32 [3,H,W].
// Gradient tensors in fp16 carry grad_scale * dL (see DESIGN.md "fp16 backward").
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pxr {

typedef __half act_t;

// ------------------------------------------------------------------ VQGAN drawer (vqgan.py:60-64, 190-195)
// Nearest codebook row per latent position (exact fp32), straight-through output as NHWC fp16.
//   z: [C, hw] fp32 (NCHW of the reference's z with N=1); cbT: [C, n_e] fp32; c2: [n_e] = sum_k cb^2
//   part_d/part_i: scratch [hw, n_chunks]; idx: [hw]; zq: [hw, C] fp16; cb: [n_e, C] fp32
void vq_nearest(const float* z, const float* cbT, const float* c2, const float* cb, int C, int hw, int n_e,
                float* part_d, int* part_i, int* idx, act_t* zq, cudaStream_t st);
// The same search with the hw x n_e dot products on the tensor cores (kernels_vq_tc.cu): vq_prep -> one gemm_tc GEMM
// (zh [hw, C] x cbh [n_e, C]^T -> scores [hw, ld] fp32) -> vq_select, which re-evaluates in exact fp32 every code whose
// approximate distance lies within the rounding bound of the minimum, so the index is the one vq_nearest picks.
// pinfo: [hw][4] = {|x|^2, power-of-two scale, |x|_2, |x|_1}; cb_scale: the power of two the fp16 codebook copy carries;
// cmax2 / cmax1: max_j |c_j|_2, |c_j|_1; stats (may be null): {candidates rechecked, positions that fell back}, cumulative.
bool vq_tc_supported(int C, int n_e);
void vq_prep(const float* z, int C, int hw, act_t* zh, float* pinfo, cudaStream_t st);
void vq_select(const float* scores, int ld, const float* z, const float* cb, const float* c2, const float* pinfo,
               float cb_scale, float cmax2, float cmax1, int C, int hw, int n_e, int* idx, act_t* zq, int* stats,
               cudaStream_t st);
// z_grad[C, hw] fp32 = dzq[hw, C] fp16 / grad_scale   (ReplaceGrad: gradient of z_q goes to z unchanged)
void vq_backward(const act_t* dzq, float inv_scale, int C, int hw, float* z_grad, cudaStream_t st);

// Variants for the vdiff U-Net (cc12m_1.py:41-50, 78-97): GroupNorm(1, C) (one_group), gamma = modulation scale + 1
// (gamma_add, gamma/beta may be null = 0), activation `swish` argument: 0 none, 1 swish, 2 ReLU, forward residual add.
struct GnOpts {
  int one_group = 0;
  float gamma_add = 0.f;
  const act_t* res = nullptr;  // forward only: y = act(norm(x)) + res
};
// GroupNorm(32, C, eps) [+ swish] over NHWC fp16 in three kernels (partial sums, a fixed-order fold, an elementwise pass),
// for every shape: no shared-memory limit.  stats: [32][2] (mean, rstd); part: scratch [2 nblk][32][2] with nblk =
// gn_num_partials.  `o` takes the U-Net's variants as the single-kernel path below does (swish 2 = ReLU).
int gn_num_partials(int pixels, int C);
void gn_stats(const act_t* x, int pixels, int C, float eps, float* part, float* stats, cudaStream_t st, GnOpts o = GnOpts());
void gn_apply(const act_t* x, const float* stats, const float* gamma, const float* beta, int pixels, int C, int swish,
              act_t* y, cudaStream_t st, GnOpts o = GnOpts());
// dx = GroupNorm'(x) applied to dy (through the activation) [+ dres]; part scratch like gn_stats, gstats [32][2].
void gn_backward(const act_t* dy, const act_t* x, const float* stats, const float* gamma, const float* beta,
                 int pixels, int C, int swish, const act_t* dres, float* part, float* gstats, act_t* dx,
                 cudaStream_t st, GnOpts o = GnOpts());

// The same two operations as ONE kernel each (grid <= one block per SM, grid-wide barrier between the statistics and the apply
// phase, the block's slab of x kept in shared memory): 1 launch and 1 HBM pass instead of 3 launches and 2 passes.
// `part` needs 64 floats per block (<= num_sms blocks).  gn_coop_supported: the slab of a block fits shared memory.
// The grid-wide barrier is a monotonically growing device counter; `issued` mirrors on the host what the launches so far
// will have added, so each launch knows the value it waits for (one GridBarrier per stream).
struct GridBarrier {
  unsigned long long* counter = nullptr;  // device, zero-initialised
  unsigned long long issued = 0;
};
#ifdef __CUDACC__
// The GroupNorm kernels take the variance as E[x^2] - mean^2 from fp32 partial sums, whose rounding error grows with
// mean^2 / var (the sums of x^2 carry mean^2 where the variance is var): at a mean of 64 standard deviations rstd is off by
// up to 6e-4 relative.  A group whose mean exceeds sqrt(32) standard deviations (error below 5e-6) gets its statistics
// again from sums of x - mean, a second pass; every other group keeps the one-pass result.
__device__ __forceinline__ bool gn_refine_variance(double mean, double var) { return mean * mean > 32.0 * var; }
#endif
bool gn_coop_supported(int pixels, int C, int num_sms);
void gn_forward_coop(const act_t* x, const float* gamma, const float* beta, int pixels, int C, int swish, float eps,
                     float* part, float* stats, act_t* y, int num_sms, GridBarrier* gb, cudaStream_t st,
                     GnOpts o = GnOpts());
void gn_backward_coop(const act_t* dy, const act_t* x, const float* stats, const float* gamma, const float* beta,
                      int pixels, int C, int swish, const act_t* dres, float* part, act_t* dx, int num_sms,
                      GridBarrier* gb, cudaStream_t st, GnOpts o = GnOpts());

// GroupNorm(32, C) with one thread-block cluster per GROUP (kernels_gn_group.cu): no grid-wide barrier, for the layers
// whose group fits the registers of <= 8 CTAs (C/32 in {8, 16, 32} channels per group, pixels * C/256 <= 16384 units).
// `sk` (optional) makes the kernel the epilogue of a split-K convolution as well: forward sums the fp32 partials
// [splits][pixels][ld_ws] (+ bias + res), writes the result to sk->out (pitch C) and normalises it in the same pass;
// backward takes dy from the partials (no bias / res) instead of from memory.
struct GnSplitK {
  const float* ws = nullptr;
  int splits = 0, ld_ws = 0;
  const float* bias = nullptr;
  const act_t* res = nullptr;
  act_t* out = nullptr;
};
bool gn_group_supported(int pixels, int C);  // covered AND inside the size range where it is the faster kernel
bool gn_group_possible(int pixels, int C);   // covered at all (the launchers accept these)
void gn_forward_group(const act_t* x, const GnSplitK* sk, const float* gamma, const float* beta, int pixels, int C,
                      int swish, float eps, float* stats, act_t* y, cudaStream_t st);
void gn_backward_group(const act_t* dy, const GnSplitK* sk, const act_t* x, const float* stats, const float* gamma,
                       const float* beta, int pixels, int C, int swish, const act_t* dres, act_t* dx, cudaStream_t st);

// ---- VQGAN encoder side (taming Encoder; VqganDrawer.init_from_tensor, vqgan.py:174-185): forward only, init time
// image [3, H, W] fp32 in [-1, 1] -> NHWC fp16 [pixels, 64] (channels 3..63 zero: conv_in's padded reduction)
void image_to_nhwc64(const float* img, int pixels, act_t* out, cudaStream_t st);
// taming Downsample: F.pad(x, (0,1,0,1)) + Conv2d(k=3, stride=2, padding=0) == the odd positions of the stride-1 "same"
// convolution: y[i, j] = full[2 i + 1, 2 j + 1], [H, W, C] -> [H/2, W/2, C]
void subsample_odd(const act_t* full, int H, int W, int C, act_t* y, cudaStream_t st);
// z[c, p] = codebook[idx[p], c] (fp32): the quantised latent model.encode returns
void gather_codes(const float* cb, const int* idx, int C, int hw, float* z, cudaStream_t st);
// GumbelQuantize's eval forward (taming GumbelVQ: F.gumbel_softmax(logits, hard=True), then the einsum with the codebook):
// idx[p] = the first j maximising logits[p * ld + j] + noise[j * hw + p] (the temperature does not move the arg-max);
// z[c, p] = cb[idx[p], c].  logits: quantize.proj's output [hw, ld] fp32; noise: the Gumbel draws [n_e, hw] fp32.
void gumbel_select(const float* logits, int ld, const float* noise, const float* cb, int C, int hw, int n_e, int* idx,
                   float* z, cudaStream_t st);

// nearest, [H,W,C]->[2H,2W,C]; the input's pixel stride is ld_in (0: C), the output is dense
void upsample2x(const act_t* x, int H, int W, int C, act_t* y, cudaStream_t st, int ld_in = 0);
void downsum2x(const act_t* gy, int H, int W, int C, act_t* gx, cudaStream_t st);       // adjoint: [2H,2W,C]->[H,W,C]

// conv_out result [pixels, ld] fp32 (3 valid channels) -> image [3, pixels] = clamp((x+1)/2, 0, 1); pre = unclamped.
// shift = 0: clamp(x, 0, 1) (the super-resolution net's output is already an image in [0, 1]).
void image_finish(const float* conv_out, int ld, int pixels, float* pre, float* img, cudaStream_t st, int shift = 1);
// ClampWithGrad backward (vqgan.py:76-79) + d/dx of (x+1)/2 (shift = 0: without it) -> fp16 [pixels, ld] (ld >= 3; other
// channels untouched)
void image_finish_backward(const float* g_img, const float* pre, int pixels, int ld, act_t* g_out, cudaStream_t st,
                           int shift = 1);

// ---- super-resolution drawer (kernels_superres.cu; RRDBNet, engine_superres.inc).  NHWC fp16 tensors with pixel strides.
// y[p, c] = fp16(alpha a[p, c] + b[p, c]) for c < C (C % 8 == 0; b may be null; y may alias b): the RRDB's outer
// residual x + 0.2 rdb3(...) and its adjoint
void sr_axpy(const act_t* a, int lda, float alpha, const act_t* b, int ldb, act_t* y, int ldy, int C, long long pixels,
             cudaStream_t st);
// z_grad[c, p] = g[p, c] * inv_scale for c < 3: the latent's gradient out of the padded NHWC input of conv_first
void sr_zgrad(const act_t* g, int ld, long long pixels, float inv_scale, float* z_grad, cudaStream_t st);

// FastPixelDrawer.synth (fast_pixeldrawer.py:89-91): nearest upsample [3,rows,cols] -> [3,H,W] + clamp; and adjoint.
void pixel_synth(const float* z, int rows, int cols, int H, int W, float* pre, float* img, cudaStream_t st);
void pixel_synth_backward(const float* g_img, const float* pre, int rows, int cols, int H, int W, float inv_scale,
                          float* z_grad, cudaStream_t st);

// ------------------------------------------------------------------ polygon drawer (kernels_raster.cu; PixelDrawer.synth,
// pixeldrawer.py:330-367).  Fixed polygons with one RGBA fill each, z = [n, 4]; 2 x 2 jittered samples per pixel
// (raster_samples.cuh), even-odd fill, the topmost polygon containing a sample wins, pixel = mean of its samples.
// The shapes are binned once into a uniform grid of RASTER_TILE-pixel tiles; each tile lists the polygons whose bounding
// box meets it (closed intervals), topmost first.
constexpr int RASTER_TILE = 16;
struct RasterScene {
  const float2* xy;       // [total_vertices] vertices, polygon k = xy[off[k] .. off[k+1])
  const int* off;         // [n + 1]
  const float4* bbox;     // [n] {xmin, ymin, xmax, ymax} of the vertices
  const int* tile_start;  // [tiles_x * tiles_y + 1]
  const int* tile_list;   // polygon indices per tile, topmost (highest index) first
  int n, tiles_x;
};
// winner [4, H, W] int32 (-1: no polygon covers the sample); img [3, H, W] = sum of the winners' RGB / 4
void raster_forward(const RasterScene& s, const float* z, int H, int W, uint64_t seed, int iter, int* winner, float* img,
                    cudaStream_t st);
// z_grad[k, c] = 0.25 * inv_scale * sum of g_img[c, p] over the samples k won (c < 3); z_grad[k, 3] = 0.  One warp per
// polygon over its bounding box: one writer per element, fixed order, no atomics.
void raster_backward(const RasterScene& s, const int* winner, const float* g_img, int H, int W, float inv_scale,
                     float* z_grad, cudaStream_t st);

// ------------------------------------------------------------------ line-sketch drawer (kernels_strokes.cu; LineDrawer,
// linedrawer.py:44-166).  n_paths open paths of n_segments cubic Béziers over an opaque paper rectangle; every stroke is
// opaque black.  z = [points n_paths * (3 n_segments + 1) * 2 | widths n_paths | paper RGBA 4].
//   Geometry: each cubic is flattened into STROKE_CHORDS chords at t = i / STROKE_CHORDS; a path covers the points within
//   its width w (the half width) of one of its chords, i.e. a union of round-capped capsules.
//   Forward: 2 x 2 jittered samples per pixel (raster_samples.cuh); a sample's winner is the topmost path covering it.
//   The pixel's RGBA is the mean of its samples' (black, or the paper's RGBA), composited as synth does:
//   out = rgb a + (1 - a).
//   Backward: the exact derivative of the box-filtered coverage with respect to the outline, integral over the visible
//   capsule boundary of G(pixel) v_n ds, where G = sum_ch g_ch d out_ch / d coverage at the forward's coverage.  Straight
//   sides are walked across the pixel grid and their visible parts (no other capsule strictly covers them) integrate
//   exactly; each vertex circle uses STROKE_ARC_NODES midpoint nodes.  The paper colour gets the interior term.
//   Capsules are re-binned into RASTER_TILE tiles every render (the geometry moves every step).
constexpr int STROKE_CHORDS = 16;
constexpr int STROKE_ARC_NODES = 64;
struct StrokeScene {
  int n_paths, n_segments, n_caps, W, H, tiles_x, tiles_y, width_offset, paper_trainable;
  float4* caps;      // [n_caps] chord endpoints (ax, ay, bx, by); capsule c = chord c % S of segment c / S (path-major)
  int4* cap_tiles;   // [n_caps] tile range (tx0, ty0, tx1, ty1) of the box grown by the width; empty when tx1 < tx0
  int* tile_start;   // [tiles + 1]
  int* tile_list;    // [n_caps * tiles] capsule indices per tile, highest index (topmost) first
  int* winner;       // [4, H, W] path index per sample, -1 = paper
  float* pix_g;      // [H, W] d loss / d coverage
  float* paper_part; // [stroke_paper_blocks(H, W), 4]
  float* cap_grad;   // [n_caps, 5] d loss / d (a, b, w) of each capsule
};
int stroke_paper_blocks(int H, int W);
void stroke_flatten(const StrokeScene& s, const float* z, cudaStream_t st);
void stroke_bin(const StrokeScene& s, cudaStream_t st);  // count, scan, fill
void stroke_raster_forward(const StrokeScene& s, const float* z, uint64_t seed, int iter, float* img, cudaStream_t st);
// z_grad = inv_scale * d loss / dz (overwritten; the paper part is 0 unless paper_trainable).  No atomics: bit-identical
// on repeats.
void stroke_raster_backward(const StrokeScene& s, const float* z, const float* g_img, float inv_scale, float* z_grad,
                            cudaStream_t st);

// ------------------------------------------------------------------ FFT drawer (fftdrawer.py:78-84)
struct FftPlans;  // cuFFT C2R / R2C plans (3 planes of H x W), resolved through dlopen
FftPlans* fft_plans_create(int H, int W, cudaStream_t st, const char** err);
void fft_plans_destroy(FftPlans* p);
// spectrum [3,H,W/2+1,2] -> img [3,H,W] = sigmoid(M (irfft2(scale*spectrum, ortho) * contrast / std)); x, stats kept
void fft_synth_forward(FftPlans* pl, const float* spectrum, const float* scale, const float* M, float contrast,
                       float* scaled, float* x, double* part, float* stats, float* img, cudaStream_t st);
void fft_synth_backward(FftPlans* pl, const float* g_img, const float* img, const float* x, const float* scale,
                        const float* M, float contrast, const float* stats, float* g1, float* G, double* part,
                        float inv_scale, float* z_grad, cudaStream_t st);

// ------------------------------------------------------------------ MakeCutouts (pixray.py:445-511)
// (AdaptiveAvgPool2d + AdaptiveMaxPool2d) / 2 of the whole image, once (pixray.py:463); argmax kept for backward.
void pool_forward(const float* img, int H, int W, int cs, float* pooled, int* argmax, cudaStream_t st);
void pool_backward(const float* g_pooled, const int* argmax, int H, int W, int cs, float* g_img, cudaStream_t st,
                   int accumulate = 0);
// Spot prompts (pixray.py:453-459): cutout[0][mask_indexes] = 0 on the pooled image -- y = keep ? x : 0 with
// keep = (mask[i] != 0) XOR zero_where_set; the same call masks the gradient on the way back (in place when y == x)
void spot_mask_apply(const float* x, const unsigned char* mask, int zero_where_set, int n, float* y, cudaStream_t st);

// kornia.geometry.transform.rescale of the pooled image for non-square canvases (pixray.py:468-472): bilinear,
// align_corners=False ([3, in_h, in_w] -> [3, out_h, out_w]), and its adjoint (g_in must be zeroed by the caller)
void rescale_bilinear(const float* x, int in_h, int in_w, int out_h, int out_w, float* y, cudaStream_t st);
// 64-bit fixed-point accumulation (order-independent sums).  A pass that meets a NaN / Inf / out-of-range contribution
// writes its id to *poison; the conversion to fp32 then yields NaN for the whole tensor (ids only ever grow: no reset).
struct FxPass {
  unsigned int* poison = nullptr;  // device word
  unsigned int pass = 0;           // > 0, unique per accumulate + convert pair on that word
};
// acc: zeroed 64-bit fixed-point accumulator of 3 * in_h * in_w entries (cleared again on return)
void rescale_bilinear_backward(const float* gy, int in_h, int in_w, int out_h, int out_w, long long* acc, FxPass fx, float* gx,
                               cudaStream_t st);

struct CutoutArgs {
  const float* pooled;     // [3, src_h, src_w]: the pooled image (cs x cs), stretched when the canvas is not square
  const float* minv;       // [n_local, 9] src_pix <- dst_pix homographies (device)
  const float* noise_facs; // [n_local]            (noise_mode 1)
  const float* noise;      // [n_local, 3, cs, cs] (noise_mode 1)
  const float* jitter;     // [n_local, 3] {code, saturation_factor, hue_factor} (color_jitter.cuh) or nullptr
  int noise_mode;          // 0 none, 1 explicit facs + noise, 2 engine Philox (seed, iter)
  float noise_fac;         // U(0, noise_fac) upper bound for mode 2 (pixray.py:439)
  int cs, n_local, first_global, cutn_zoom, zoom_padding;
  int src_h, src_w;        // size of `pooled` (== cs, cs on a square canvas)
  float fill;
  uint64_t seed;
  int iter;
  uint32_t rng_stream;     // Philox stream offset of the cutout set (transforms.h cut_rng_stream; 0 for set 0)
};
int cutout_num_blocks(int n_local, int cs);
// batch [n_local,3,cs,cs] fp32; block partial min/max (+ element index) for the global range normalise (slip.py:21-36)
void cutout_forward(const CutoutArgs& a, float* batch, float* part_min, float* part_max, int* part_imin,
                    int* part_imax, cudaStream_t st);
// multi-rank range exchange helpers: xbuf = {min, -max} for one allreduce(min)
void range_pack(const float* range, float* xbuf, cudaStream_t st);
void range_unpack(const float* xbuf, float* range, int* irange, cudaStream_t st);
// partials of an arbitrary buffer (same layout as cutout_forward's), nparts blocks
void minmax_partials(const float* x, long long n, int nparts, float* part_min, float* part_max, int* part_imin,
                     int* part_imax, cudaStream_t st);
// range[0]=min, range[1]=R (max of x-min, 1 if zero), range[2]=max, range[3]=R!=0; irange = argmin / argmax element
void minmax_reduce(const float* batch_or_null, const float* part_min, const float* part_max, const int* part_imin,
                   const int* part_imax, int nparts, float* range, int* irange, cudaStream_t st);
// The perceptor's input normalisation (transforms.Normalize of its preprocess)
struct ChannelNorm {
  float mean[3], std[3];
};
constexpr ChannelNorm kClipNorm = {{0.48145466f, 0.4578275f, 0.40821073f}, {0.26862954f, 0.26130258f, 0.27577711f}};  // slip.py:55
constexpr ChannelNorm kImageNetNorm = {{0.485f, 0.456f, 0.406f}, {0.229f, 0.224f, 0.225f}};  // SLIP_Base, slip.py:117-121
// patches[(n*gp + py)*gp + px, (c*P + iy)*P + ix] = ((x - min)/R - mean_c)/std_c   (slip.py:52-60 + conv1 im2col)
void patchify_forward(const float* batch, const float* range, int n, int cs, int P, int ld, act_t* patches,
                      const ChannelNorm& nrm, cudaStream_t st);
// g_batch (=|+=) d/d(batch) of the direct term; sums_fx[0] += sum g_a, sums_fx[1] += sum g_a * a / R in 64-bit fixed point
// (order-independent: identical bits on every run); range_sums_finish converts to fp32 and clears the accumulator
void patchify_backward(const act_t* g_patches, const float* batch, const float* range, int n, int cs, int P, int ld,
                       int accumulate, float* g_batch, long long* sums_fx, FxPass fx, const ChannelNorm& nrm,
                       cudaStream_t st);
void range_sums_finish(long long* sums_fx, FxPass fx, float* sums, cudaStream_t st);
// adds the argmin / argmax terms of the global range normalise, then scatters through the bilinear taps
// g_pooled: [3, src_h, src_w] (overwritten); acc: zeroed fixed-point accumulator of the same extent (cleared again on return)
void cutout_backward(const CutoutArgs& a, const float* g_batch, const float* range, const int* irange,
                     const float* sums, long long* acc, FxPass fx, float* g_pooled, cudaStream_t st);

// ------------------------------------------------------------------ CLIP ViT (slip.py:62-66; SLIP/models.py:18-64)
// y = LN(x [+ pos[row % T]]) * gamma + beta ; x fp32 [rows, W]; outputs optional fp16 / fp32; stats [rows][2]
// W = 128 * k, k in [1, 8]; row r of x starts at x + r * x_stride (class-token rows: stride T * W).
// All four return 0, or -1 without launching anything when W has no kernel.
int layernorm_forward(const float* x, long long x_stride, const float* pos, int T, const float* gamma,
                      const float* beta, int rows, int W, float eps, act_t* y16, float* y32, float* stats,
                      cudaStream_t st);
// the same on an fp16 residual stream (x fp16)
int layernorm_forward(const act_t* x, long long x_stride, const float* pos, int T, const float* gamma,
                      const float* beta, int rows, int W, float eps, act_t* y16, float* y32, float* stats,
                      cudaStream_t st);
// gx (+)= LN'(x) applied to dy (fp16, scaled); also writes gx16 = fp16(gx).  accumulate=0 overwrites gx.
// dy is compact [rows, W]; x, gx, gx16 rows are x_stride apart
int layernorm_backward(const act_t* dy, const float* x, long long x_stride, const float* pos, int T,
                       const float* stats, const float* gamma, int rows, int W, int accumulate, float* gx,
                       act_t* gx16, cudaStream_t st);
// fp16 residual stream: x fp16; with gx == nullptr the stream gradient lives in gx16 alone (accumulate reads it there)
int layernorm_backward(const act_t* dy, const act_t* x, long long x_stride, const float* pos, int T,
                       const float* stats, const float* gamma, int rows, int W, int accumulate, float* gx,
                       act_t* gx16, cudaStream_t st);
// One LayerNorm kernel family chosen explicitly (the functions above choose by stream type and PXR_LN16_WIDE):
//   LN_F32_STREAM: fp32 x; LN_F16_VEC4: fp16 x, 8-byte vectors; LN_F16_VEC8: fp16 x, 16-byte vectors (W % 256 == 0,
//   no pos, fp16 output / gradient only).  -1 when the variant has no kernel for these arguments.
enum { LN_F32_STREAM = 0, LN_F16_VEC4 = 1, LN_F16_VEC8 = 2 };
int layernorm_forward_variant(int variant, const void* x, long long x_stride, const float* pos, int T, const float* gamma,
                              const float* beta, int rows, int W, float eps, act_t* y16, float* y32, float* stats,
                              cudaStream_t st);
int layernorm_backward_variant(int variant, const act_t* dy, const void* x, long long x_stride, const float* pos, int T,
                               const float* stats, const float* gamma, int rows, int W, int accumulate, float* gx,
                               act_t* gx16, cudaStream_t st);
// timm ViT tokens (no LayerNorm before the blocks): y[r] = t[r] + pos[r % T] into the residual stream, y16 (fp16) when
// non-null, else y32; t [rows, W], pos [T, W] fp32, W % 4 == 0
void add_pos_embed(const float* t, const float* pos, int T, int rows, int W, act_t* y16, float* y32, cudaStream_t st);
// in-place row softmax over the first `cols` of each row of length ld (pad columns zeroed); rows total; any ld % 8 == 0
void softmax_forward(act_t* s, int rows, int cols, int ld, cudaStream_t st);
void softmax_backward(const act_t* p, act_t* dp_to_ds, int rows, int cols, int ld, cudaStream_t st);
// causal attention rows (blocks of `cols` rows, one per (head, sequence)): row r keeps columns [0, r % cols], the rest
// become exact zeros.  ld <= 1024; -1 without launching anything otherwise
int softmax_forward_causal(act_t* s, int rows, int cols, int ld, cudaStream_t st);
// Text towers (kernels_text.cu).  x[r] = tok_emb[ids[r]] + pos[r % T] into the residual stream: y16 (fp16) when non-null,
// else y32.  tok_emb [vocab, W] fp16, pos [T, W] fp32, ids [rows] already checked against the vocabulary; W % 4 == 0
void text_embed(const int* ids, const act_t* tok_emb, const float* pos, int T, int rows, int W, act_t* y16, float* y32,
                cudaStream_t st);
// y[b] = x[src[b]] for b < n: rows of W elements (elem_bytes 2 or 4, W * elem_bytes % 16 == 0) gathered into a compact buffer
void gather_rows(const void* x, const int* src, int n, int W, int elem_bytes, void* y, cudaStream_t st);
// Prompt.forward for all prompts of one perceptor + its gradient w.r.t. the un-normalised embeds.
//   e [B, D]; prompts [n, D] (unit rows), weights/stops [n]; de [B, D].  slots / inv_rows (nullable): row j adds into
//   losses[slots[j]] with 1 / (rows of its Prompt) -- multi-row embeds (image prompts).  losses += partial, caller zeroes;
//   the partials are summed in a fixed order (the same bits on every run) through part [B, n] floats of scratch and
//   `count`, one zero-initialised counter the call leaves at zero.  Both may be null when n == 0.
void prompt_loss(const float* e, int B, int D, const float* prompts, const float* weights, const float* stops,
                 const int* slots, const float* inv_rows, int n, int cutn_global, float grad_scale, float* e_unit,
                 float* losses, float* de, act_t* de16, float* part, unsigned int* count, cudaStream_t st);

// ------------------------------------------------------------------ optimiser (pixray.py:538-539, 1484-1487)
// Adam (bias-corrected, torch.optim.Adam semantics) on z with gradient g * inv_scale, then clip_z to per-channel
// [zmin, zmax] (vqgan.py:202-204) or, when zmin == nullptr, by clip_mode:
//   CLIP_NONE  no clamp
//   CLIP_01    [0, 1] (fast_pixeldrawer.py:98-100)
//   CLIP_RGBA  z is [n, 4] RGBA fill colours: RGB to [0, 1], alpha to [1, 1] (pixeldrawer.py:378-382)
//   CLIP_STROKES  the line drawer's z: range 1 (the widths) to [lo1, hi1] (linedrawer.py:179-184)
// ZRanges splits z into [0, end0) [end0, end1) [end1, n), each with its own multiple of the learning rate: the line
// drawer's three Adams (linedrawer.py:128-136).  Every other drawer uses one range at scale 1 (zranges_single).
enum { CLIP_NONE = 0, CLIP_01 = 1, CLIP_RGBA = 2, CLIP_STROKES = 3 };
struct ZRanges {
  int end0, end1;
  float scale[3];
  float lo1, hi1;
};
inline ZRanges zranges_single() { return ZRanges{0x7fffffff, 0x7fffffff, {1.f, 1.f, 1.f}, 0.f, 0.f}; }
#ifdef __CUDACC__
__device__ __forceinline__ int zrange_of(const ZRanges& r, int i) { return i < r.end0 ? 0 : i < r.end1 ? 1 : 2; }
__device__ __forceinline__ float clip_mode_apply(int clip_mode, int i, float zi, const ZRanges& r) {
  if (clip_mode == CLIP_01) return fminf(fmaxf(zi, 0.f), 1.f);
  if (clip_mode == CLIP_RGBA) return (i & 3) == 3 ? 1.f : fminf(fmaxf(zi, 0.f), 1.f);
  if (clip_mode == CLIP_STROKES && zrange_of(r, i) == 1) return fminf(fmaxf(zi, r.lo1), r.hi1);
  return zi;
}
#endif
// The update rule (PXR_OPT_* in include/pixray_b200.h, pixray.py:536-551), every one with pixray's constructor defaults
// and the engine's betas / eps:
//   ADAM      m, v            torch.optim.Adam
//   ADAMW     m, v            torch.optim.AdamW, weight decay kAdamWDecay applied to z before the Adam step
//   ADAGRAD   s (in v)        torch.optim.Adagrad, eps kAdagradEps, no lr decay, accumulator starts at 0
//   ADAMAX    m, u (in v)     torch.optim.Adamax
//   DIFFGRAD  m, v, p         torch_optimizer 0.1.0 DiffGrad: Adam moments times the friction 1 / (1 + exp(-|p - g|)),
//                             p = the previous gradient; eps outside the bias correction
// The step count t belongs to the current instance of the rule; a fresh instance has t = 0 and all state at 0.
enum { OPT_ADAM = 0, OPT_ADAMW = 1, OPT_ADAGRAD = 2, OPT_ADAMAX = 3, OPT_DIFFGRAD = 4, OPT_KINDS = 5 };
constexpr double kAdamWDecay = 0.01, kAdagradEps = 1e-10;
// the learning-rate multiplier of step t: 1 / bc1 (Adam, AdamW, Adamax), sqrt(bc2) / bc1 (DiffGrad), 1 (Adagrad), as
// step = lr * num / den in double
__host__ __device__ inline double opt_step_size(int kind, double lr, double bc1, double bc2) {
  if (kind == OPT_ADAGRAD) return lr;
  if (kind == OPT_DIFFGRAD) return lr * sqrt(bc2) / bc1;
  return lr / bc1;
}
inline int opt_state_arrays(int kind) { return kind == OPT_DIFFGRAD ? 3 : 2; }  // z-sized arrays besides z (Adagrad's m idle)
// p: DiffGrad's previous gradient (nullptr for the other kinds)
void adam_clip_step(int kind, float* z, float* m, float* v, float* p, const float* g, float inv_scale, int n,
                    int per_channel, const float* zmin, const float* zmax, int clip_mode, const ZRanges& zr, float lr,
                    float b1, float b2, float eps, int t, cudaStream_t st);

// ------------------------------------------------------------------ device-side checkdrop + Adam (pixray.py:1090-1109, 1464-1512)
// train()'s per-iteration control decisions without a host round trip.  The optimiser step of iteration `it` reads the
// iteration's loss vector, decides like checkdrop / the scheduled learning-rate drops / auto_stop do, applies the update
// rule + clip_z with the CURRENT learning rate and optimiser state, and -- when the decision is "rebuild the optimisers" --
// leaves a fresh instance of the rule (state 0, t = 0) at learning_rate / 10^num_loss_drop behind for the next iteration, or raises `stopped` when
// the drops are used up (after which further iterations leave z untouched).  State is double-buffered (read cur, write
// next) so every block of the kernel sees the same decision inputs.
struct DropState {
  float best_loss;     // 1e20 after a rebuild (pixray.py:1509)
  int best_iter;
  int num_loss_drop;
  int stopped;
  float lr;
  int adam_t;          // steps taken by the current optimiser instance, whichever rule it runs
  int pad[2];
};
struct DropConfig {
  float base_lr;       // args.learning_rate, or the drawer's own rate (fftdrawer.py:63-67)
  int iter_drop_delay; // 12 (pixray.py:1987)
  int max_loss_drops;  // len(args.learning_rate_drops)
  int auto_stop;
  int n_sched;
  int sched[16];       // args.learning_rate_drops: iterations at which the rate drops regardless of the losses
};
// What the host may poll without synchronising (pinned, mapped memory; seq_begin == seq_end == iteration + 1 when the
// record is consistent).
struct DropStatus {
  volatile int seq_begin;
  int iter;
  float loss_sum, best_loss;
  int best_iter, num_loss_drop, stopped, rebuilt;
  float lr;
  int n_losses;
  float losses[64];
  volatile int seq_end;
};
void adam_clip_managed(int kind, float* z, float* m, float* v, float* p, const float* g, float* best_z, float inv_scale, int n,
                       int per_channel, const float* zmin, const float* zmax, int clip_mode, const ZRanges& zr, float b1,
                       float b2, float eps, const float* losses, int n_losses, int iter, const DropConfig& cfg,
                       const DropState* cur, DropState* next, DropStatus* status_mapped, cudaStream_t st);
// acc (=|+=) g: gradient accumulation over the `batches` passes of one iteration (pixray.py:1464-1482)
void accumulate_f32(const float* g, float* acc, long long n, int accumulate, cudaStream_t st);

// ------------------------------------------------------------------ auxiliary losses (Losses/*.py), kernels_losses.cu
// Every launcher adds grad_scale * weight * dL/dx into the fp32 gradient buffer of the tensor the reference loss reads
// and writes (image losses) or accumulates (cutout / embedding losses: per-rank partial sums) the weighted loss value.
// `part`: scratch of max(4 * AUX_MAX_BLOCKS, n_local) doubles.  `weight` = the loss's own *_weight setting times the
// custom_loss spec weight (pixray.py:1388).
constexpr int AUX_MAX_BLOCKS = 1024;
// Anchors to a stored copy (pixray.py:1344-1375).  anchor_z: kind 0 spherical / 1 mse/2 / 2 cosine embedding between the
// latent and `ref` (n floats each), adds weight * dL/dz into z_grad (unscaled fp32) and writes the weighted value.
// anchor_pix: weight/2 * l1(img, ref) with its sign gradient (times grad_scale) into g_img.
void anchor_z(int kind, const float* z, const float* ref, int n, float weight, float* z_grad, float* loss_out, cudaStream_t st);
void anchor_pix(const float* img, const float* ref, long long n, float weight, float grad_scale, float* g_img, double* part,
                float* loss_out, cudaStream_t st);
void aux_symmetry(const float* img, int H, int W, float weight, float grad_scale, float* g_img, double* part,
                  float* loss_out, cudaStream_t st);
// margins = (left, right, upper, lower) in pixels (EdgeLoss.py:82-88), colour in [0,1]; target [3, H, W] replaces the
// colour and mask [H, W] (> 0: masked) replaces the margins when not null
void aux_edge(const float* img, int H, int W, const int margins[4], const float color[3], const float* target,
              const float* mask, float edge_color_weight, float global_color_weight, float weight, float grad_scale,
              float* g_img, double* part, float* loss_out, cudaStream_t st);
void aux_gaussian(const float* img, int H, int W, float stdy, float stdx, const float color255[3], float weight,
                  float grad_scale, float* g_img, double* part, float* loss_out, cudaStream_t st);
// best_out (optional): nearest-palette index per pixel [n_img * cs * cs] (the loss's integer bookkeeping)
void aux_palette(const float* batch, int n_img, int cs, int cutn_global, const float* palette_dev, int n_colors,
                 float weight, float grad_scale, float* g_batch, int* best_out, double* part, float* loss_out,
                 cudaStream_t st);
// saturation: local moment sums (4 doubles) -> [allreduce over ranks] -> gradient from the global moments
void aux_saturation_moments(const float* batch, int n_img, int cs, double* part, double* sums, cudaStream_t st);
void aux_saturation_grad(const float* batch, int n_img, int cs, int cutn_global, const double* sums, float weight,
                         float grad_scale, int write_loss, float* g_batch, float* loss_out, cudaStream_t st);
// A: scratch [(n_img * cs + 2) * cs] floats; halo: [2][2][3][cs] rows around this rank's slab (unused when world == 1).
// accumulate = 0 stores the gradient instead of adding it (the blurred path's scratch).
void aux_smoothness(const float* batch, int n_img, int cs, int first_global, int cutn_global, const float* halo,
                    float spacing, int kind, int edge_order, float weight, float grad_scale, float* A, float* g_batch,
                    int accumulate, double* part, float* loss_out, cudaStream_t st);
// smoothness_gaussian_kernel: the valid blur of [n_img, 3, cs, cs] by the separable taps u (x) u (n each) into
// out [n_img, 3, cs', cs'], cs' = cs - n + 1, and its adjoint added into g_batch.  tmp: [n_img, 3, cs, cs'] scratch.
void aux_smooth_blur(const float* batch, int n_img, int cs, const float* taps, int n, float* tmp, float* out,
                     cudaStream_t st);
void aux_smooth_blur_adjoint(const float* g_out, int n_img, int cs, const float* taps, int n, float* tmp, float* g_batch,
                             cudaStream_t st);
void aux_smooth_pack_halo(const float* batch, int n_img, int cs, int rank, float* xbuf, cudaStream_t st);
void aux_smooth_unpack_halo(const float* xbuf, int cs, int rank, int world, float* halo, cudaStream_t st);
void aux_aesthetic(const float* e, int n_local, int D, int cutn_global, const float* w_dev, float bias, float target,
                   float weight, float grad_scale, float* de, __half* de16, double* part, float* loss_out,
                   cudaStream_t st);

// ------------------------------------------------------------------ filters (kernels_filters.cu; filters/*.py, pixray.py:1203-1222)
// planar fp32 [3, H, W]; roll = torch.roll(x, (sh, sw), (2, 3)); *_backward: gx (=|+=) adjoint(gy)
void filter_roll(const float* x, int H, int W, int sh, int sw, float* y, cudaStream_t st);
void filter_roll_backward(const float* gy, int H, int W, int sh, int sw, int accumulate, float* gx, cudaStream_t st);
// wallpaper "shift": [3,H,W] -> [3,2H,W] (second row of tiles offset by W/2), rolled by (sh, sw)
void filter_wallpaper_shift(const float* x, int H, int W, int sh, int sw, float* y, cudaStream_t st);
void filter_wallpaper_shift_backward(const float* gy, int H, int W, int sh, int sw, int accumulate, float* gx, cudaStream_t st);
void filter_crop(const float* x, int H, int W, int top, int left, int Hc, int Wc, float* y, cudaStream_t st);
void filter_crop_backward(const float* gy, int H, int W, int top, int left, int Hc, int Wc, float* gx, cudaStream_t st);
// loss_out (nullable) (=|+=) weight * mse(first em, last em) / em along axis (0: columns, 1: rows);
// g (nullable) += grad_scale * weight * dloss/dx, one writer per element
void filter_edge_match(const float* x, int H, int W, int em, int axis, float weight, float grad_scale, int accumulate_loss,
                       float* g, float* loss_out, cudaStream_t st);
// nearest palette colour (first minimum), loss = weight * (beta + 1) * mean((z_q - z)^2); part: AUX_MAX_BLOCKS doubles
void filter_colorlookup(const float* x, int pixels, const float* pal, int n_col, float beta, float weight, float* y,
                        int* best_out, double* part, float* loss_out, cudaStream_t st);
void filter_colorlookup_backward(const float* gy, const float* x, const float* y, int pixels, float beta, float weight,
                                 float grad_scale, int accumulate, float* gx, cudaStream_t st);

// ------------------------------------------------------------------ vdiff drawer (kernels_vdiff.cu; cc12m_1.py, sampling.py)
struct VdFeatures {
  float v[144];  // [cos, sin] Fourier features of t: 128 for the mapping network, 16 timestep planes
};
void vd_set_features(const VdFeatures& f, float* h0_tail, float* te, cudaStream_t st);
void vd_input(const float* x, const float* te, int pixels, act_t* out, cudaStream_t st);  // [pixels, 64]: x | te | 0
void avgpool2x(const act_t* x, int H, int W, int C, int ld_in, act_t* y, cudaStream_t st);
void avgpool2x_backward(const act_t* gy, int H, int W, int C, int accumulate, act_t* gx, cudaStream_t st);
void bilinear_up2x(const act_t* x, int H, int W, int C, act_t* y, int ld_out, cudaStream_t st);   // align_corners=False
void bilinear_up2x_backward(const act_t* gy, int H, int W, int C, int ld_gy, act_t* gx, cudaStream_t st);
void copy_channels(const act_t* src, int ld_src, act_t* dst, int ld_dst, int C, long long pixels, int accumulate,
                   cudaStream_t st);
void im2col3x3(const act_t* x, int H, int W, int C, act_t* A, cudaStream_t st);  // A [pixels, 9 C], tap-major
void gemv_f16(const act_t* W, int K, int R, const float* x, const float* bias, int relu, const float* res, float* y,
              cudaStream_t st);
// The U-Net runs at the gen size (gh, gw); the canvas (h, w) is its window at rows my.., columns mx.. (VdiffDrawer.synth's
// centre crop, vdiff.py:165-170).  v / pred / g_pred / g_v are gen-size, pre / img / g_img canvas-size; g_pred and g_v are
// zero outside the window.
struct VdCrop {
  int gh, gw, h, w, my, mx;
};
void vd_finish(const float* vout, int ld, const float* x, float alpha, float sigma, VdCrop c, float* v_planar,
               float* pred, float* pre, float* img, cudaStream_t st);
void vd_finish_backward(const float* g_img, const float* pre, float sigma, VdCrop c, int ld, float* g_pred, act_t* g_v,
                        cudaStream_t st);
void vd_zgrad(const float* g_pred, const act_t* g_in, int ld, float alpha, float inv_scale, int pixels, float* z_grad,
              cudaStream_t st);
void vd_renoise(float* x, const float* pred, const float* v, const float* noise, float alpha_i, float sigma_i,
                float alpha_next, float adjusted_sigma, float ddim_sigma, long long n, cudaStream_t st);

// ------------------------------------------------------------------ CLIP ResNet image towers (kernels_resnet.cu; openai-CLIP
// ModifiedResNet).  Activations NHWC fp16 with C a multiple of 8; B images of HW pixels each.
// Stem input (kernels_cutouts.cu): cols [n (cs/2)^2, 64] = the stride-2, pad-1 3x3 im2col of the normalised cutouts
// (column (c * 3 + ky) * 3 + kx, columns >= 27 zero), and its adjoint gathered into g_batch (=|+=) with the range sums
// accumulated as patchify_backward does.
void rn_stem_forward(const float* batch, const float* range, int n, int cs, act_t* cols, const ChannelNorm& nrm,
                     cudaStream_t st);
void rn_stem_backward(const act_t* g_cols, const float* batch, const float* range, int n, int cs, int accumulate,
                      float* g_batch, long long* sums_fx, FxPass fx, const ChannelNorm& nrm, cudaStream_t st);
// gx = avgpool2x_backward(gy) * (y > 0): the adjoint of AvgPool2d(2) after a ReLU whose output is y.  rows = images * H.
void rn_pool_bwd_relu(const act_t* gy, const act_t* y, int rows, int W, int C, act_t* gx, cudaStream_t st);
// attnpool tokens: tok[b, 0] = mean_p x[b, p] + pos[0], tok[b, 1 + p] = x[b, p] + pos[1 + p]; tok fp16 [B, HW + 1, C]
void rn_pool_tokens(const act_t* x, int B, int HW, int C, const float* pos, act_t* tok, cudaStream_t st);
// single-query attention of the pool: q fp32 [B, C] (token 0's projection), kv fp16 [B T, 2C] (k | v), 64-wide heads,
// T <= RN_POOL_MAX_T.  o fp16 [B, C]; p fp32 [B, C / 64, T] the softmax, kept for the backward.
constexpr int RN_POOL_MAX_T = 256;
void rn_attnpool_forward(const float* q, const act_t* kv, int B, int T, int C, float scale, act_t* o, float* p,
                         cudaStream_t st);
// its backward from g_o fp16 [B, C]: g_q fp16 [B, C], g_kv fp16 [B T, 2C]
void rn_attnpool_backward(const float* q, const act_t* kv, const float* p, const act_t* g_o, int B, int T, int C,
                          float scale, act_t* g_q, act_t* g_kv, cudaStream_t st);
// adjoint of rn_pool_tokens times the block ReLU: gx[b, p] = (g_tok[b, 1 + p] + (g_tok[b, 0] + g_tok0[b]) / HW) * (y[b, p] > 0)
void rn_pool_tokens_backward(const act_t* g_tok, const act_t* g_tok0, const act_t* y, int B, int HW, int C, act_t* gx,
                             cudaStream_t st);

void fill_f32(float* p, float v, long long n, cudaStream_t st);
void cast_f32_to_f16(const float* x, act_t* y, long long n, float scale, cudaStream_t st);

}  // namespace pxr
