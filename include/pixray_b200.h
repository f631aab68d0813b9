/* pixray_b200 -- C ABI of the H100-native (sm_90a) engine for pixray's per-iteration hot path.
 *
 * Plain C: pointers and sizes only, no torch types.  Every entry point below replaces one method the reference's
 * Python loop calls each iteration (file:line are relative to the reference checkout, pixray/pixray @ 37b03cf):
 *
 *   pxr_synth          <- drawer.synth(cur_iteration)          pixray.py:1206, vqgan.py:190-195, fast_pixeldrawer.py:89-91,
 *                                                              fftdrawer.py:78-84, vdiff.py:159-172
 *   pxr_make_cutouts   <- MakeCutouts.forward(out)             pixray.py:445-511 (cached-transform semantics 480-486)
 *   pxr_encode_image   <- CLIP_Base.encode_image(cutouts)      slip.py:21-42, 52-66
 *   pxr_prompt_loss    <- Prompt.forward(embeds) per prompt    pixray.py:268-280 (spherical_dist_loss 262-265)
 *   pxr_backward       <- sum(lossAll).backward()              pixray.py:1481-1482
 *   pxr_step           <- opt.step(); drawer.clip_z()          pixray.py:1484-1487, 538-539, vqgan.py:202-204
 *   pxr_iterate        <- one pass of train()                  pixray.py:1436-1512 (ascend_txt 1243-1406)
 *
 * Conventions: functions return 0 on success and a negative code on failure; pxr_last_error() gives the message.
 * All work is enqueued on ONE engine-owned CUDA stream; only pxr_sync, pxr_read_* and the *_host variants block.
 * A handle is owned by one host thread (the reference keeps its session in module globals, pixray.py:1022-1063:
 * one session per process, not re-entrant).  Buffers passed in are device pointers unless the name says host;
 * layouts at the boundary are the reference's: NCHW fp32 images, [cutn, D] fp32 embeddings.
 * There is no CPU fallback: without a CUDA device pxr_create fails.
 */
#ifndef PIXRAY_B200_H
#define PIXRAY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pxr_engine* pxr_handle;

enum { PXR_DRAWER_VQGAN = 0, PXR_DRAWER_PIXEL = 1, PXR_DRAWER_FFT = 2, PXR_DRAWER_VDIFF = 3, PXR_DRAWER_POLYGON = 4,
       PXR_DRAWER_SUPERRES = 5, PXR_DRAWER_STROKES = 6 };
enum { PXR_PAD_REFLECTION = 0, PXR_PAD_BORDER = 1, PXR_PAD_ZEROS = 2 };
enum { PXR_DTYPE_F16 = 0, PXR_DTYPE_BF16 = 1 };
/* module ids for pxr_load_weight */
enum { PXR_MOD_VQGAN = 0, PXR_MOD_CLIP0 = 1, PXR_MOD_CLIP1 = 2, PXR_MOD_CLIP2 = 3, PXR_MOD_CLIP3 = 4 };

/* ViT towers: the fields as named.  CLIP ResNet towers (PXR_TOWER_CLIP_RESNET): width = the stem width w (64 for RN50),
 * layers = the number of bottleneck blocks over all four stages (16 for RN50), heads = the attention pool's heads
 * (64-wide), patch unused (0). */
typedef struct {
  int width;     /* transformer width (768 for ViT-B) */
  int layers;    /* 12 */
  int heads;     /* 12 */
  int patch;     /* 16 or 32 */
  int image_res; /* the cut_size of the perceptor's MakeCutouts (pixray.py:643-649); the first perceptor's == cut_size */
  int out_dim;   /* 512 */
} pxr_clip_cfg;

typedef struct {
  int device;            /* CUDA ordinal */
  int rank, world;       /* cutout-shard rank / number of ranks (1 = single GPU) */
  int drawer;            /* PXR_DRAWER_* */
  int image_h, image_w;  /* canvas (vqgan: multiple of 16) */
  /* taming Decoder hyper-parameters (vqgan.py:122-142: model.decoder / model.quantize) */
  /* super-resolution drawer: ch = num_feat (0 -> 64) */
  int z_channels, n_embed, ch, num_res_blocks, attn_resolution, n_levels, resolution;
  int ch_mult[8];
  /* pixel drawer grid (fast_pixeldrawer.py:37-63) */
  int grid_rows, grid_cols;
  /* MakeCutouts(cut_size, cutn) pixray.py:400-443; cutn is the GLOBAL count, this rank owns a slice */
  int cutn, cut_size;
  /* 1 to 4 perceptors.  One cutout set per distinct image_res, in order of first appearance (pixray.py:642-649): set 0 is
   * cut_size (the first perceptor's), and each perceptor scores only its own set's batch. */
  int n_clip;
  pxr_clip_cfg clip[4];
  float noise_fac;       /* pixray.py:439 (0.1) */
  uint64_t seed;
  int op_dtype;          /* PXR_DTYPE_*: tensor-core operand type (accumulation is always fp32) */
  float grad_scale;      /* backward runs on grad_scale * dL (fp16 range management); 0 = default */
  float beta1, beta2, adam_eps; /* optim.Adam defaults 0.9 / 0.999 / 1e-8 when 0 */
  /* fft drawer (fftdrawer.py:16-22, 57-61): fft_image(decay_power) / to_valid_rgb(colors) / image_f(contrast) */
  float fft_decay, fft_colors, fft_contrast; /* 0 -> 1.5 / 1.5 / 0.9 */
  /* global_aspect_width = args.size[0] / args.size[1] (pixray.py:1931): != 1 stretches the pooled cut_size x cut_size image
   * to [cut_size, int(cut_size * a)] (a > 1) or [int(cut_size / a), cut_size] (a < 1) before the warps (pixray.py:468-472)
   * and changes the wide stack's affine (pixray.py:420-432).  0 = 1 (square). */
  float cut_aspect;
  /* the stretched size itself, int(cut_size * a) resp. int(cut_size * (1 / a)) as the reference's Python floats give it
   * (kornia rescale truncates); 0 = derive from cut_aspect (which, being a C float, can round across an integer) */
  int cut_src_h, cut_src_w;
  /* super-resolution drawer (RRDBNet): RRDB blocks (0 -> 23) and dense-block growth channels (0 -> 32) */
  int num_block, num_grow_ch;
} pxr_config;

/* Per-iteration cutout parameters (SURVEY.md Appendix A): what kornia's augmentations sample per cutout, made explicit.
 * transforms[cutn*9]: row-major 3x3 "dst_pix <- src_pix" homographies exactly as MakeCutouts.transforms caches them
 * (pixray.py:498; src = the pooled image, stretched when cut_aspect != 1); indices [0, int(0.6*cutn)) form the zoom group, the rest the wide group (pixray.py:407, 493-494). */
typedef struct {
  const float* transforms; /* host, [cutn, 3, 3] */
  int zoom_padding;        /* PXR_PAD_REFLECTION on even iterations, PXR_PAD_BORDER on odd (pixray.py:1250-1253) */
  float fill;              /* wide-group fill grey = random.random() (pixray.py:1255-1258) */
  /* batch + facs * randn_like(batch) (pixray.py:508-510).  Given together: replayed as is.  Both NULL: with
   * transforms == NULL the engine draws them (Philox keyed by seed, iteration and GLOBAL element index), with explicit
   * transforms the call is a deterministic replay WITHOUT noise.  One without the other is an error (-61). */
  const float* noise_facs; /* host, [cutn] ~ U(0, noise_fac) (pixray.py:509) */
  const float* noise;      /* DEVICE, [cutn,3,cs,cs] standard normal (pixray.py:510) */
  /* K.ColorJitter(hue=0.1, saturation=0.1, p=0.8), the last stage of both stacks (pixray.py:416, 436): host
   * [cutn, 3] rows {code, saturation_factor, hue_factor}.  code 0 = this cutout missed the Bernoulli(p); else
   * 256 + o0 + 4*o1 + 16*o2 + 64*o3 with o_k the transform applied k-th (0 brightness, 1 contrast, 2 saturation,
   * 3 hue: kornia's params["order"]).  NULL with explicit transforms = no jitter (the cached-transform replay,
   * pixray.py:480-486); with transforms == NULL the engine draws these too (pxr_set_color_jitter). */
  const float* color_jitter;
} pxr_cut_params;

const char* pxr_last_error(pxr_handle h); /* h may be NULL for creation errors */
const char* pxr_version(void);

int pxr_create(const pxr_config* cfg, pxr_handle* out);
void pxr_destroy(pxr_handle h);

/* Weights by the reference's state_dict key (e.g. "decoder.conv_in.weight", "quantize.embedding.weight",
 * "visual.transformer.resblocks.0.attn.in_proj_weight").  data: fp32, host or device; copied and repacked. */
int pxr_load_weight(pxr_handle h, int module_id, const char* name, const float* data, const int64_t* dims, int ndim);
/* After all weights: builds every kernel plan / workspace.  Fails listing the first missing weight. */
int pxr_finalize(pxr_handle h);

/* Image tower of perceptor clip_idx, before pxr_finalize (default PXR_TOWER_OPENAI_CLIP):
 *   OPENAI_CLIP  openai-CLIP VisionTransformer (clip.load, slip.py:173-186): CLIP mean / std, conv1 without bias,
 *                class_embedding + positional_embedding, ln_pre, QuickGELU, LayerNorm eps 1e-5, ln_post, proj
 *   TIMM_VIT     timm VisionTransformer of SLIP_Base (slip.py:84-157, SLIP/models.py:130-134): ImageNet mean / std,
 *                patch_embed.proj with bias, cls_token + pos_embed without a LayerNorm before the blocks, exact GELU,
 *                LayerNorm eps 1e-6, final norm, image_projection; keys visual.* and image_projection after the
 *                checkpoint's `module.` prefix is stripped
 *   CLIP_RESNET  openai-CLIP ModifiedResNet (clip.load of RN50 / RN101 / RN50x4 / RN50x16 / RN50x64): CLIP mean / std,
 *                a three-conv stem (conv1 stride 2) with AvgPool2d(2), four stages of bottlenecks (AvgPool2d before the
 *                stride-2 convs), eval-mode BatchNorm (eps 1e-5, folded into the convs at pxr_finalize), ReLU, and the
 *                attention pool (mean token + positional_embedding, q / k / v / c_proj, token 0 as the only query).
 *                The block counts per stage are read from the visual.layerN.i.* keys; their sum must equal
 *                pxr_clip_cfg.layers, and the pool's positional_embedding must have (image_res / 32)^2 + 1 rows. */
enum { PXR_TOWER_OPENAI_CLIP = 0, PXR_TOWER_TIMM_VIT = 1, PXR_TOWER_CLIP_RESNET = 2 };
int pxr_set_clip_tower(pxr_handle h, int clip_idx, int kind);

/* Prompt(embed, weight, stop) list of one perceptor (pixray.py:859-915).  embeds host [n, D]. */
int pxr_set_prompts(pxr_handle h, int clip_idx, const float* embeds, int n, int D, const float* weights,
                    const float* stops);

/* Image prompts (pixray.py:1308-1336, pmsImageTable): imgs host or device fp32 [n, 3, H, W] in [0, 1] at the output
 * size (copied).  Every iteration -- inside pxr_iterate / pxr_make_cutouts, before the main pass -- each image is cut
 * with that iteration's cached transforms (no ColorJitter on the cached path, pixray.py:480-486; fresh noise, or the
 * explicit noise of pxr_cut_params replayed), encoded by every perceptor, and scored as a throwaway
 * Prompt(embed [cutn, D], weights[k]) (weights NULL = 1, args.image_prompt_weight otherwise) whose loss follows that
 * perceptor's text prompts in the loss vector.  Cutout-sharded ranks exchange the [cutn, D] rows (one allreduce).
 * n = 0 clears. */
int pxr_set_image_prompts(pxr_handle h, const float* imgs, int n, const float* weights);
/* the same with every target at its own size: imgs[k] fp32 [3, hs[k], ws[k]] (resize_image keeps the source aspect and never
 * upsamples, pixray.py:514-518; MakeCutouts pools any size to cut_size x cut_size, pixray.py:463) */
int pxr_set_image_prompts_sized(pxr_handle h, const float* const* imgs, const int* hs, const int* ws, int n,
                                const float* weights);

/* Spot prompts (args.spot_prompts / spot_prompts_off: pixray.py:917-931, 1262-1293; mask from fetch_spot_indexes 370-394,
 * applied to the pooled image at 453-459).  which = 1: `embeds` are scored on cutouts of the image with the SPOT zeroed
 * (make_cutouts(out, spot=1) zeroes mask >= 0.5), which = 0: with everything but the spot zeroed.  Every pxr_iterate then
 * runs one more cutout + encode + backward pass per kind (cached transforms of the iteration, no ColorJitter, fresh noise);
 * their losses come FIRST in the perceptor's part of the loss vector (spot, spot off, prompts, image prompts).
 * mask: host bytes [3, cut_size, cut_size], != 0 where the resized RGB mask image is >= 0.5.  Both fail (-69) in a session
 * with more than one cutout set (the reference cuts those with the last set's MakeCutouts, pixray.py:1270-1276). */
int pxr_set_spot_prompts(pxr_handle h, int clip_idx, int which, const float* embeds, int n, int D, const float* weights,
                         const float* stops);
int pxr_set_spot_mask(pxr_handle h, const unsigned char* mask);

/* Multi-GPU: 128-byte ncclUniqueId from rank 0; the engine owns the communicator. */
int pxr_set_comm(pxr_handle h, const void* nccl_unique_id, int rank, int world);
int pxr_get_unique_id(void* out128);

int pxr_synth(pxr_handle h, const float* z, float* out_img /* [3,H,W] */);
/* Polygon drawer (PXR_DRAWER_POLYGON; PixelDrawer with pixel_type hex / tri / diamond / knit / rectshift,
 * pixeldrawer.py:200-367): n fixed polygons, each filled with one RGBA colour; z = [n, 4] (the reference's get_z layout).
 * xy: host [total_vertices, 2] canvas coordinates, polygon k = vertices offsets[k] .. offsets[k+1]-1 (offsets host [n+1],
 * offsets[0] = 0), in draw order: later polygons cover earlier ones.  3 to 8 vertices each (8 = knit), finite
 * coordinates.  Before pxr_finalize.  The render takes 2 x 2 stratified jittered samples per pixel (Philox keyed by seed
 * and iteration), even-odd fill, topmost polygon wins, pixel = mean of its samples, no clamp; clip_z keeps RGB in [0, 1]
 * and alpha at 1. */
int pxr_set_polygons(pxr_handle h, const float* xy, const int* offsets, int n);
/* Line-sketch drawer (PXR_DRAWER_STROKES; LineDrawer, linedrawer.py): n_paths open paths of n_segments cubic Béziers,
 * stroked in opaque black over an opaque paper rectangle.  z = [points n_paths x (3 n_segments + 1) x 2 canvas
 * coordinates | stroke widths n_paths (half widths) | paper RGBA 4].  The fused Adam steps the three ranges at lr,
 * lr / 10 and lr / 100 (the paper only when paper_trainable, else it stays fixed) and clamps the widths to
 * [1, max_width]; the managed step keeps no best-z copy.  The render takes the polygon drawer's 2 x 2 jittered samples
 * (pxr_test_raster_samples); a sample is covered when it lies within a path's width of one of its chords (each cubic
 * flattened into 16 chords).  Before pxr_finalize; max_width finite and positive. */
int pxr_set_strokes(pxr_handle h, int n_paths, int n_segments, float max_width, int paper_trainable);
/* The iteration the per-op pxr_synth renders (drawer.synth(cur_iteration)): keys the polygon drawer's sample positions,
 * ignored by the other drawers.  pxr_iterate uses its own `iter` (and leaves it set). */
int pxr_set_synth_iteration(pxr_handle h, int iter);
/* z = model.encode(img)[0]: VqganDrawer.init_from_tensor / reapply_from_tensor / get_z_from_tensor (vqgan.py:174-185) --
 * taming Encoder + quant_conv + nearest codebook row.  img device [3,H,W] in [-1,1]; z_out device [z_channels,h,w].
 * Available when the weights loaded before pxr_finalize include the checkpoint's encoder.* and quant_conv.* tensors.
 * Refused on a GumbelVQ engine (codebook quantize.embed.weight): that one encodes with pxr_vqgan_encode_gumbel. */
int pxr_vqgan_encode(pxr_handle h, const float* img, float* z_out);
/* model.encode(img)[0] of a GumbelVQ (taming GumbelQuantize in eval mode, hard Gumbel-softmax): taming Encoder +
 * quant_conv, logits = quantize.proj(h) [n_embed, h, w], then per position the first code maximising logits + noise, and
 * z_out = that code's row of quantize.embed.weight, exactly (the reference's straight-through value differs from the row by
 * at most one fp32 rounding).  noise: device [n_embed, h, w] fp32, the Gumbel draws -log(Exp(1)) F.gumbel_softmax adds.
 * Needs the checkpoint's encoder.*, quant_conv.* and quantize.proj.* tensors; refused on a nearest-code engine. */
int pxr_vqgan_encode_gumbel(pxr_handle h, const float* img, const float* noise, float* z_out);
/* Distribution of the engine-drawn ColorJitter: Bernoulli(p) per cutout, saturation_factor ~ U(1-s, 1+s),
 * hue_factor ~ U(-hue, hue), one random order per group and iteration.  Defaults = the reference's call sites
 * (0.8, 0.1, 0.1); p = 0 turns the stage off. */
int pxr_set_color_jitter(pxr_handle h, float p, float saturation, float hue);
int pxr_make_cutouts(pxr_handle h, const float* img, const pxr_cut_params* p, int iter,
                     float* out_batch /* [cutn_local,3,cs,cs] */);
/* Cutout sets (after pxr_finalize): returns their number and writes each one's cut size to cut_sizes[0..3] (0 past the
 * last).  pxr_make_cutouts_set cuts set `set` (its own augmentations and noise, Philox streams of its own; the fill grey
 * and padding mode are shared) into out_batch [cutn_local, 3, cs, cs] of that set's cs; pxr_make_cutouts is set 0.
 * pxr_encode_image reads the batch of the perceptor's own set: a caller batch must have that set's size, and without
 * one the set must have been cut since the last pxr_backward.  pxr_backward takes back every set cut since the last
 * backward (set 0 when none was), adding their image gradients. */
int pxr_cutout_sets(pxr_handle h, int* cut_sizes /* [4] */);
int pxr_make_cutouts_set(pxr_handle h, int set, const float* img, const pxr_cut_params* p, int iter,
                         float* out_batch /* [cutn_local,3,cs,cs] */);
int pxr_encode_image(pxr_handle h, int clip_idx, const float* batch, float* out_embeds /* [cutn_local, D] */);

/* Text tower of perceptor clip_idx (CLIP.encode_text, SLIP/models.py:136-150): built at pxr_finalize when the weights
 * loaded for the perceptor include token_embedding.weight, positional_embedding, transformer.resblocks.*, ln_final.* and
 * text_projection.  pxr_text_tower returns 1 and its shape when it exists, 0 when not (the outputs are then 0), < 0 on
 * error.  pxr_encode_text: tokens_host [n, ctx] int32 host ids (ctx == the tower's context, every id inside the
 * vocabulary) -> out device fp32 [n, D], the un-normalised embeddings of encode_text(...).float(); any n. */
int pxr_text_tower(pxr_handle h, int clip_idx, int* width, int* layers, int* ctx, int* out_dim);
int pxr_encode_text(pxr_handle h, int clip_idx, const int32_t* tokens_host, int n, int ctx, float* out);
int pxr_prompt_loss(pxr_handle h, int clip_idx, const float* embeds, float* out_losses /* [n_prompts] */);
int pxr_backward(pxr_handle h, float* z_grad);
int pxr_step(pxr_handle h, float* z, float lr, int iter);
int pxr_iterate(pxr_handle h, float* z, float lr, int iter, const pxr_cut_params* p,
                float* out_losses_host /* pinned or pageable; may be NULL */);
/* pxr_iterate with one pxr_cut_params per cutout set, in set order (p NULL: the engine draws every set's).  A session
 * with more than one set takes explicit parameters only here: pxr_iterate with p != NULL fails (-69). */
int pxr_iterate_sets(pxr_handle h, float* z, float lr, int iter, const pxr_cut_params* p /* [n_sets] or NULL */,
                     float* out_losses_host);
/* Auxiliary losses: Losses/*.py behind LossInterface.get_loss, summed into the iteration's loss list by ascend_txt
 * (pixray.py:1384-1393, custom_loss spec "name:weight").  Each becomes one more entry of the loss vector (a cutout-space
 * one, marked (cutouts) below, one entry per cutout set in set order, pixray.py:1392-1398) (after the
 * prompts, in the order added) and one more term of the gradient.  params (host floats), by kind:
 *   SYMMETRY   {symmetry_weight}                                            Losses/SymmetryLoss.py:14-17   (image)
 *   SATURATION {saturation_weight}                                          Losses/SaturationLoss.py:15-30 (cutouts)
 *   PALETTE    {palette_weight, r0,g0,b0, r1,g1,b1, ...}  colours in [0,1]  Losses/PaletteLoss.py:25-35    (cutouts)
 *   SMOOTHNESS {smoothness_weight, type (0 default, 1 clipped, 2 log), spacing[, edge_order (1|2)[, n, taps[n*n]]]}
 *              Losses/SmoothnessLoss.py:9-108 (cutouts).  n > 0: GaussianSmoothing's normalised 2-D kernel (row-major,
 *              separable), a valid blur before torch.gradient; cut_size - n + 1 must be >= edge_order + 1.
 *   EDGE       {edge_color_weight, global_color_weight, left,right,upper,lower (pixels), r,g,b[, mode,
 *              target[3*H*W] if mode & 1, mask[H*W] if mode & 2]}  Losses/EdgeLoss.py:60-108 (image).  The target
 *              replaces the colour; the mask (> 0: masked) replaces the margins.  H, W: the canvas.
 *   GAUSSIAN   {gaussian_weight, std_y, std_x, R,G,B (0..255)}              Losses/GaussianLoss.py:31-44   (image)
 *   AESTHETIC  {aesthetic_target, bias, w[D]}  linear head on the last perceptor's embeddings  Losses/AestheticLoss.py:30-33 */
enum { PXR_LOSS_SYMMETRY = 0, PXR_LOSS_SATURATION = 1, PXR_LOSS_PALETTE = 2, PXR_LOSS_SMOOTHNESS = 3, PXR_LOSS_EDGE = 4,
       PXR_LOSS_GAUSSIAN = 5, PXR_LOSS_AESTHETIC = 6 };
int pxr_add_aux_loss(pxr_handle h, int kind, float weight, const float* params, int n_params);
int pxr_clear_aux_losses(pxr_handle h);

/* Anchors to a stored copy: the init_weight family and image_labels of ascend_txt (pixray.py:1344-1375).  Each is one entry
 * of the loss vector after the prompts and before the auxiliary losses, in the order added (the reference's order is
 * image_labels..., init_weight, init_weight_dist, init_weight_pix, init_weight_cos).
 *   SPHERICAL  spherical_dist_loss(z.reshape(1,-1), ref.reshape(1,-1)) * weight      init_weight, image_label_weight
 *   MSE        F.mse_loss(z, ref) * weight / 2                                        init_weight_dist
 *   COS        F.cosine_embedding_loss(z.reshape(1,-1), ref.reshape(1,-1), 1) * weight  init_weight_cos
 *   PIX        F.l1_loss(out, ref) * weight / 2, ref = init_image_tensor [3,H,W] in [0,1]   init_weight_pix
 * `ref` (host or device floats) is copied: the latent's element count for the first three (z_orig = drawer.get_z_copy(),
 * pixray.py:719, or an encoded label image), 3*H*W of the image MakeCutouts sees for PIX.  The latent terms add to z.grad
 * after the drawer backward; PIX adds to the image gradient before it.  Replicated on every rank when sharded. */
enum { PXR_ANCHOR_SPHERICAL = 0, PXR_ANCHOR_MSE = 1, PXR_ANCHOR_COS = 2, PXR_ANCHOR_PIX = 3 };
int pxr_add_anchor(pxr_handle h, int kind, float weight, const float* ref, long long n);
int pxr_clear_anchors(pxr_handle h);
int pxr_num_losses(pxr_handle h, int* out); /* filters + prompts of every perceptor + auxiliary losses */

/* Filters (args.filters "name:weight,..."; FilterInterface.forward(img) -> (img, loss), pixray.py:651-668, applied to the
 * drawer's output before MakeCutouts in do_synth_and_filter, pixray.py:1203-1222).  Inside pxr_iterate only.  params:
 *   TILER     {}                                               filters/tiler.py: torch.roll by random (h, w) shifts
 *   WALLPAPER {type (0 none, 1 shift, 2 horizontal, 3 vertical), wallpaper_edge_match}   filters/wallpaper.py
 *   LOOKUP    {lookup_beta, r0,g0,b0, ...} palette in [0,1]     filters/colorlookup.py (nearest colour, straight-through)
 * Each filter owns one entry at the FRONT of the loss vector (its weighted loss; 0 for the loss-free ones).  The random
 * shifts are engine-drawn per iteration (Philox by seed / iteration) or fixed through pxr_set_filter_shifts. */
enum { PXR_FILTER_TILER = 0, PXR_FILTER_WALLPAPER = 1, PXR_FILTER_LOOKUP = 2 };
int pxr_add_filter(pxr_handle h, int kind, float weight, const float* params, int n_params);
int pxr_clear_filters(pxr_handle h);
int pxr_set_filter_shifts(pxr_handle h, int filter_idx, int rand_h, int rand_w);
int pxr_read_losses(pxr_handle h, float* out_host); /* blocking: the loss vector of the last forward / backward */

/* Super-resolution drawer (PXR_DRAWER_SUPERRES; SuperResolutionDrawer, super_resolution.py, with RealESRGANer at tile 0 /
 * pre_pad 0 / scale 4): z = the low-resolution image [1, 3, H/4, W/4] in [0, 1] (image_h, image_w multiples of 4), synth =
 * clamp_with_grad(RRDBNet(z), 0, 1) with RRDBNet(3, 3, num_feat = ch, num_block, num_grow_ch, scale 4) (basicsr's
 * rrdbnet_arch).  Weights under the checkpoint's own keys (conv_first, body.{i}.rdb{1,2,3}.conv{1..5}, conv_body,
 * conv_up1, conv_up2, conv_hr, conv_last; .weight / .bias) through pxr_load_weight(PXR_MOD_VQGAN = the drawer slot).
 * clip_z clamps z to [0, 1]. */

/* vdiff drawer (PXR_DRAWER_VDIFF; VdiffDrawer, vdiff.py:58-190, over diffusion/models/cc12m_1.py).  z = x [1,3,H,W];
 * weights under the checkpoint's own keys through pxr_load_weight(module PXR_MOD_VQGAN = the drawer slot).
 *   set_schedule : sample_state's steps / alphas / sigmas (vdiff.py:113-126, sampling.py:41-51), n = iterations + 1
 *   set_clip_embed: extra_args["clip_embed"] (pixray.py:880-885), host [512]
 *   set_iteration: the schedule index the per-op pxr_synth uses (pxr_iterate uses its own `iter`)
 *   renoise      : drawer.makenoise(cur_it) (vdiff.py:156-157, sampling.sample_step_noise 18-39) on the pred / v the last
 *                  synth kept; noise: device [3,H,W] standard normal (torch.randn_like), or NULL for eta = 0 */
int pxr_vdiff_set_schedule(pxr_handle h, const float* steps, const float* alphas, const float* sigmas, int n);
int pxr_vdiff_set_clip_embed(pxr_handle h, const float* embed, int D);
int pxr_vdiff_set_iteration(pxr_handle h, int i);
int pxr_vdiff_renoise(pxr_handle h, float* z, int i, const float* noise);
/* the U-Net's size (VdiffDrawer's gen_height / gen_width, vdiff.py:55-58), before pxr_finalize: sides multiples of 64,
 * each at least the canvas's.  x (z), v, pred and the optimiser state are [1, 3, gen_h, gen_w]; the image is the canvas-size
 * window at rows (gen_h - H) / 2.., columns (gen_w - W) / 2.. of (pred + 1) / 2 clamped.  Not called: gen = the canvas. */
int pxr_vdiff_set_gen_size(pxr_handle h, int gen_h, int gen_w);

int pxr_reset_optimizer(pxr_handle h); /* rebuild_optimisers: a fresh instance of the current rule (pixray.py:520-555, 1511) */

/* args.optimiser (pixray.py:536-551): the update rule of pxr_step / pxr_iterate, each with the constructor defaults pixray
 * builds it with (only lr is passed).  AdamW, Adamax and DiffGrad take beta1 / beta2 / adam_eps from pxr_config; AdamW's
 * weight decay is 0.01 and Adagrad's eps 1e-10.  Valid after pxr_finalize; has pxr_reset_optimizer's effects (fresh state,
 * t = 0, and in managed mode fresh drop bookkeeping) and refuses an unknown kind.  The default is PXR_OPT_ADAM.
 * Checkpoints of an Adam session are version 1 {header, z, m, v}; the other rules write version 2 {header, kind, z,
 * state arrays} (Adagrad: m, unused, and s; Adamax: m, u; DiffGrad: m, v, previous gradient).  A blob loads only into a session of
 * its own rule. */
enum { PXR_OPT_ADAM = 0, PXR_OPT_ADAMW, PXR_OPT_ADAGRAD, PXR_OPT_ADAMAX, PXR_OPT_DIFFGRAD };
int pxr_set_optimizer(pxr_handle h, int kind);

/* train()'s control decisions on the device (checkdrop pixray.py:1090-1109; scheduled learning-rate drops, auto-stop and
 * rebuild_optimisers 1464-1512): the optimiser step of every pxr_iterate reads the iteration's loss vector, tracks the best
 * loss, drops the learning rate (fresh Adam at base_lr / 10^drops) at the iterations in `drops` or -- with auto_stop --
 * when the loss has not improved for iter_drop_delay iterations, and stops updating z once max_loss_drops is exceeded.
 * No host synchronisation: pxr_iterate's `lr` is ignored afterwards and pxr_poll_status reads the last completed
 * iteration's record from pinned memory. */
typedef struct {
  int iter;            /* the iteration this record describes */
  float loss_sum;      /* sum(lossAll) of that iteration */
  float best_loss;     /* after the iteration (1e20 right after a rebuild) */
  int best_iter, num_loss_drop;
  int stopped;         /* train() would have returned False: later iterations leave z untouched */
  int rebuilt;         /* the iteration ended with rebuild_optimisers */
  float lr;            /* learning rate the NEXT iteration uses */
  int n_losses;
  float losses[64];
} pxr_status;
int pxr_set_schedule(pxr_handle h, float base_lr, int iter_drop_delay, int max_loss_drops, int auto_stop, const int* drops,
                     int n_drops);
int pxr_poll_status(pxr_handle h, pxr_status* out); /* 0 ok, 1 no consistent record yet; never blocks */
/* args.batches (pixray.py:1464-1482): every pxr_iterate runs this many ascend_txt + backward passes with fresh
 * engine-drawn augmentations, accumulates z.grad over them and takes ONE optimiser step */
int pxr_set_batches(pxr_handle h, int batches);
/* hand pxr_step the gradient to apply (device [z_numel]); the per-op plugin loop accumulates several passes itself */
int pxr_set_z_grad(pxr_handle h, const float* z_grad);
int pxr_sync(pxr_handle h);

/* Checkpoint of the optimisation state for resume (SURVEY.md 8f-3): {z, Adam m, v, step count, learning-rate / best-loss /
 * drop bookkeeping} as one host blob of pxr_state_size bytes.  Load into an engine of the same configuration (after
 * pxr_set_schedule when the saved session was device-managed) and keep calling pxr_iterate with the next iteration number:
 * the engine-drawn augmentations are keyed by (seed, iteration), so the continuation follows the uninterrupted run. */
int pxr_state_size(pxr_handle h, int64_t* nbytes);
int pxr_save_state(pxr_handle h, void* host_buf);
int pxr_load_state(pxr_handle h, const void* host_buf);

/* Introspection used by tests and bench.py */
int pxr_num_kernel_launches(pxr_handle h, int64_t* out); /* launches issued since create */
/* one iteration with CUDA events around every launch: out6 = {gemm ms, gemm launches, gemm algorithmic FLOPs,
 * other ms, other launches, whole-iteration ms}; feeds bench.py's roofline object */
int pxr_profile_iteration(pxr_handle h, float* z, float lr, int iter, double* out6);
/* the same, plus the compulsory (algorithmic) bytes of the tensor-core launches: each operand read once, each epilogue
 * tensor read / written once -- the denominator against which measured DRAM traffic shows wasted re-reads */
int pxr_profile_iteration2(pxr_handle h, float* z, float lr, int iter, double* out6, double* tensor_bytes);
int pxr_get_stream(pxr_handle h, void** out);
int pxr_z_numel(pxr_handle h, int64_t* out);
int pxr_z_bounds(pxr_handle h, float* zmin, float* zmax); /* device [z_channels]: codebook per-channel min/max */

/* ---------------------------------------------------------------- test hooks (used only by tests/) */
/* copy a named internal buffer (e.g. "g_img", "batch", "clip0.gx") to `out` (host or device) */
int pxr_debug_read(pxr_handle h, const char* name, void* out, int64_t nbytes);

typedef struct {
  const void* a;
  int a_mode; /* 0 K-major, 1 MN-major */
  long long lda, a_mn_extent, a_k_extent, a_bs0, a_bs1;
  const void* b;
  int b_mode, b_batched;
  long long ldb, b_mn_extent, b_k_extent, b_bs0, b_bs1;
  int nb0, nb1;
  int M, N, K, block_n, fmt;
  float alpha;
  const float* bias;
  int bias_per_row, act; /* act: 0 none, 1 QuickGELU (+ pre-activation to aux_out), 2 QuickGELU backward, 4 LeakyReLU(0.2),
                          * 5 LeakyReLU backward (see act_col0), 6 exact GELU 0.5 u (1 + erf(u / sqrt 2)) of the fp16
                          * pre-activation u (+ u to aux_out), 7 GELU backward: times Phi(u) + u phi(u) of the saved fp16 u
                          * (aux_in); others are refused */
  const void* aux_in;
  void* aux_out;
  const float* res_f32;
  const void* res_f16;
  float* out_f32;
  void* out_f16;
  long long ldc, c_bs0, c_bs1;
  void* stream;
  int repeat;
  int cta_group; /* ignored: sm_90 has no CTA-pair MMA, every GEMM runs single-CTA tiles (kept for the struct layout) */
  int tma_epi;   /* 0 auto (tensor-map epilogue when the tensors allow it), -1 force the generic epilogue */
  /* act 5: out = (alpha acc + bias + residual) * (aux_in > 0 ? 1 : 0.2) in the columns >= act_col0, aux_in = the saved
   * post-activation (same layout as the output); the columns below act_col0 are stored unmasked */
  int act_col0;
  /* pxr_test_conv only: 1 runs the plan on the 288-thread kernel (tiles at most 128 wide) even when the 384-thread one
   * would take it, so that a test can compare the two on the same inputs.  0: the kernel the engine would use. */
  int narrow_kernel;
  /* > 1: split-K.  The plan runs ceil(nkb / ceil(nkb / k_splits)) splits of ceil(nkb / k_splits) 64-deep k-blocks each and
   * writes split s's fp32 partial sums to slab s of out_f32 (slab pitch M * ldc for a GEMM, H * W * ldc for a conv);
   * needs one unbatched image, out_f32 only, no bias, residual or activation.  0 or 1: one split. */
  int k_splits;
} pxr_test_gemm_desc;

int pxr_test_gemm(const pxr_test_gemm_desc* d, char* err, int errlen);
/* implicit-GEMM conv over NHWC fp16: d->a = input (pixel stride lda), d->b = weights [taps*cout_pad, c_in] */
int pxr_test_conv(const pxr_test_gemm_desc* d, int batch, int H, int W, int c_in, int cout_pad, int ksize, char* err,
                  int errlen);
/* the split-K reduce: out[p, c] = fp16(bias[c] + ws[0][p, c] + ... + ws[splits-1][p, c] + res[p, c]) for c < N, in that
 * order.  ws DEVICE fp32 [splits][pixels][ld_ws]; bias (nullable) fp32 [N]; res (nullable) / out fp16 [pixels][ld_out];
 * N, ld_ws, ld_out multiples of 8.  Synchronous; -1 on unsupported arguments. */
int pxr_test_splitk_reduce(const float* ws, int splits, long long pixels, int N, int ld_ws, const float* bias, const void* res,
                           void* out, int ld_out);

/* one conv weight operand the engine packed: the fp16 operand of n elements at ptr holds checkpoint weight w
 * [cout][cin][taps] element (co, ci, t) at t' s_tap + co s_co + (ci - ci0) s_ci, t' = taps - 1 - t when flip, else t,
 * for ci in [ci0, ci1); every other element is 0.  tag: the checkpoint prefix of the conv; src: an opaque id of the host
 * weights it was packed from (a forward operand and its dgrad operands share tag and src). */
typedef struct {
  char tag[128];
  const void* ptr;
  const void* src;
  long long n, s_tap, s_co, s_ci;
  int cout, cin, taps, flip, ci0, ci1;
} pxr_test_pack_rec;

/* one convolution plan the engine built (one per add_conv), with the plan's choices.  k_splits > 1: the plan writes fp32
 * partial sums and the split-K reduce applies bias, residual and the fp16 store; block_n .. grid are then the split
 * plan's.  has_* / in_place / out_f32 / ldc / act describe the convolution's own epilogue (in_place: the residual is the
 * output; out_f32: an fp32 output instead of fp16). */
typedef struct {
  char label[192];
  const void* wt;
  const float* bias;
  int batch, H, W, c_in;
  long long in_ld;
  int cout_pad, n_out, ks;
  int block_n, wide, k_splits, tma_epi, stages, grid;
  int act, act_col0;
  int has_bias, has_res, has_aux, in_place, out_f32;
  long long ldc;
} pxr_test_conv_rec;

/* the conv plans built so far, in build order: fills out[0 .. min(max, n) - 1], *count = n */
int pxr_test_conv_records(pxr_handle h, pxr_test_conv_rec* out, int max, int* count);
/* the packed conv operands so far, in packing order, as pxr_test_conv_records.  index >= 0 also copies operand `index`
 * (n fp16 elements) to the DEVICE buffer dst; with dst_bias, n_bias floats of `bias` too, which must be the bias of a
 * recorded plan on that operand with n_bias <= its n_out.  Synchronous. */
int pxr_test_packed_weights(pxr_handle h, pxr_test_pack_rec* out, int max, int* count, int index, void* dst,
                            const float* bias, float* dst_bias, int n_bias);
/* builds the plan pxr_test_conv would run, without launching it: out = {wide, block_n, stages, tma_epi, grid, k_splits} */
int pxr_test_conv_plan_info(const pxr_test_gemm_desc* d, int batch, int H, int W, int c_in, int cout_pad, int ksize,
                            int out[6]);

/* one plain GEMM plan the engine built (one per add_gemm / split add_gemm_splitk), with the plan's choices.  Operands as
 * GemmOperand (gemm_tc.cuh): mode 0 K-major (element (r, k) at r ld + k), 1 MN-major (at k ld + r), batch (b0, b1) at
 * b0 bs0 + b1 bs1; B's batch extents are 1 or A's.  The epilogue fields are the plan's own; in_place: the residual is the
 * output.  k_splits > 1: the plan writes fp32 partial sums [k_splits][M][ldc] to out_f32 (the split-K workspace) and the
 * reduce applies red_bias, red_res and the fp16 store to red_out at pitch ld_out; red_* are null otherwise.  k_blocks:
 * the 64-deep k-blocks the plan runs over (all splits together). */
typedef struct {
  char label[192];
  const void* a;
  int a_mode, a_nb0, a_nb1;
  long long lda, a_mn_extent, a_k_extent, a_bs0, a_bs1;
  const void* b;
  int b_mode, b_nb0, b_nb1;
  long long ldb, b_mn_extent, b_k_extent, b_bs0, b_bs1;
  int M, N, K;
  float alpha;
  const float* bias;
  int bias_per_row, act, act_col0, in_place;
  const void* aux_in;
  void* aux_out;
  const float* res_f32;
  const void* res_f16;
  float* out_f32;
  void* out_f16;
  long long ldc, c_bs0, c_bs1;
  int block_n, wide, stages, tma_epi, grid, k_splits, k_blocks;
  const float* red_bias;
  const void* red_res;
  void* red_out;
  long long ld_out;
} pxr_test_gemm_rec;

/* the GEMM plans built so far, in build order, as pxr_test_conv_records */
int pxr_test_gemm_records(pxr_handle h, pxr_test_gemm_rec* out, int max, int* count);
/* builds the plan pxr_test_gemm would run, without launching it: out = {wide, block_n, stages, tma_epi, grid, k_splits} */
int pxr_test_gemm_plan_info(const pxr_test_gemm_desc* d, int out[6]);
/* one attention the engine planned (one per add_attention call), in build order.  site: the caller (an image or text
 * tower's block, a U-Net attention's checkpoint key, a decoder AttnBlock's prefix).  path: PXR_ATTN_FUSED (attn_tc.cu),
 * PXR_ATTN_STREAMING (attn_long.cu) or PXR_ATTN_CHAIN (batched GEMMs around the row softmax).  backward: a backward was
 * planned.  Tensors in attn_tc.cuh's layout: qkv / gqkv [images T, 3 W] (q | k | v, head h at column h d of each
 * third), o / d_o [images T, W], W = heads d; d_o and gqkv may be set without a backward.  lse (fused, streaming) and
 * delta (streaming with a backward) fp32 [images heads T], else null.  Chain: P and dP fp16 [images heads T, ldT]
 * (dP null without a backward; dP_shared: the caller's scratch, shared with other calls), gemm[]: the indices in
 * pxr_test_gemm_records of its S = scale q k^T, O = P v, dP = dO v^T, dq = scale dS k, dk = scale dS^T q and
 * dv = P^T dO plans (-1: not planned).  Fused: splits (CTAs per (image, head) pair) and bwd (1 attn_bwd_kernel,
 * 2 attn_bwd_wg); 1 and 0 on the other paths. */
enum { PXR_ATTN_FUSED = 0, PXR_ATTN_STREAMING = 1, PXR_ATTN_CHAIN = 2 };
typedef struct {
  char site[96];
  int path, multihead, causal, backward;
  int images, heads, T, d, W;
  float scale;
  const void* qkv;
  void* o;
  const void* d_o;
  void* gqkv;
  float* lse;
  float* delta;
  void* P;
  void* dP;
  int ldT, dP_shared;
  int splits, bwd;
  int gemm[6];
} pxr_test_attn_rec;

/* the attentions planned so far, in build order, as pxr_test_conv_records */
int pxr_test_attention_records(pxr_handle h, pxr_test_attn_rec* out, int max, int* count);
/* rebuilds a fused or streaming record's plan from its shape, scale and causal flag on caller DEVICE tensors laid out as
 * the record's (d_o / gqkv null: forward only; delta: the streaming backward's workspace), runs its forward and, with
 * d_o and gqkv, its backward once, synchronously.  bwd_kernel as pxr_test_attention_bwd_select (0: the plan's own
 * choice).  out2 = {splits, bwd} of the plan, as the record holds them. */
int pxr_test_attention_plan(const pxr_test_attn_rec* r, const void* qkv, void* o, const void* d_o, void* gqkv, float* lse,
                            float* delta, int bwd_kernel, int out2[2], char* err, int errlen);
/* the engine's live device allocations (dalloc / upload), in allocation order: ptr[i], bytes[i] for i < min(max, n),
 * *count = n */
int pxr_test_allocations(pxr_handle h, const void** ptr, long long* bytes, int max, int* count);

/* host-side evaluation of the ColorJitter pixel body and its vector-Jacobian product (no GPU needed) */
int pxr_test_color_jitter_host(const float* rgb, int n, int code, float saturation, float hue, const float* g_out,
                               float* out, float* g_in);
/* the same body on the device; all pointers are DEVICE [n, 3] (default stream, synchronous) */
int pxr_test_color_jitter_device(const float* rgb, int n, int code, float saturation, float hue, const float* g_out,
                                 float* out, float* g_in);

/* adaptive-pool window bounds as the device computes them (pool_fwd / pool_bwd): DEVICE int [out_size] each */
int pxr_test_pool_bounds(int in_size, int out_size, int* starts, int* ends);

/* the polygon drawer's sample positions as the device computes them (raster_samples.cuh): out DEVICE float
 * [H, W, 4, 2], sample s = dx + 2 dy of pixel (x, y) as (x, y) canvas coordinates */
int pxr_test_raster_samples(uint64_t seed, int iter, int H, int W, float* out);

/* fused ViT attention (attn_tc.cu): forward, and backward when d_o != NULL.  qkv [B*T, 3W], o / d_o [B*T, W],
 * gqkv [B*T, 3W] fp16 device tensors, lse [B*H*T] fp32; heads are 64 wide (W = 64 H), T <= 240 */
int pxr_test_attention(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B, int T, int H, int W,
                       float scale, int repeat, char* err, int errlen);

/* pxr_test_attention's forward once, then its backward `repeat` times (none for 0) on the kernel bwd_kernel selects
 * (0: as the engine chooses, 1: attn_bwd_kernel, 2: attn_bwd_wg); *used (nullable) receives the kernel taken (1 or 2) */
int pxr_test_attention_bwd_select(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B, int T, int H,
                                  int W, float scale, int bwd_kernel, int repeat, int* used, char* err, int errlen);

/* causal attention forward (the text towers): o [B*T, W] from qkv [B*T, 3W] fp16 device tensors, row t attending to
 * keys <= t; 64-wide heads (W = 64 H), T <= 240.  The fused kernel, or with PXR_FUSED_ATTN=0 in the environment the
 * batched-GEMM chain with the causal row softmax, as the engine would choose */
int pxr_test_attention_causal(const void* qkv, void* o, int B, int T, int H, int W, float scale, char* err, int errlen);

/* streaming fused attention (attn_long.cu), same arguments: any T >= 1, 64-wide heads (W = 64 H).  The backward's
 * [B*H*T] fp32 workspace is allocated and freed inside the call */
int pxr_test_attention_long(const void* qkv, void* o, float* lse, const void* d_o, void* gqkv, int B, int T, int H,
                            int W, float scale, int repeat, char* err, int errlen);

/* GroupNorm(32, C, eps 1e-6)(+ swish) of the VQGAN decoder (taming Normalize + nonlinearity), forward and -- when dy or
 * ws_dy is given -- backward, on DEVICE NHWC fp16 tensors [pixels, C].  variant 0: single-kernel grid-barrier version,
 * 1: one thread-block cluster per group; with ws / ws_dy (variant 1) the kernel is also the epilogue of a split-K
 * convolution (fp32 partial sums [splits][pixels][C]); 2: the three-kernel version (statistics, final, apply), which the
 * engine takes when neither of the others fits.  scratch: variants 0 and 1: 64 * (num_sms + 2) floats + 8 zeroed bytes
 * (the grid barrier's counter, at float offset 64 * (num_sms + 2)); variant 2: 128 * gn_partials + 64 floats with
 * gn_partials = ceil(pixels / r), r = ceil(pixels / 592) rounded up to a multiple of 32 (at least 32). */
int pxr_test_groupnorm(int variant, const void* x, const float* ws, int splits, const float* bias, const void* res,
                       void* x_out, const float* gamma, const float* beta, int pixels, int C, int swish, void* y,
                       float* stats, const void* dy, const float* ws_dy, int splits_dy, const void* dres, void* dx,
                       float* scratch, int repeat);

/* the vdiff U-Net's norm (GroupNorm(1, C) + modulation, as vd_norm / vd_norm_bwd run it on the grid-barrier kernel):
 * y = act(norm(x) * (gamma + gamma_add) + beta) (+ res), act 0 none, 1 swish, 2 ReLU; gamma / beta / res nullable;
 * backward when dy is given: dx = norm'(x) applied to dy through the activation (+ dres).  DEVICE NHWC fp16 [pixels, C],
 * stats [32][2]; scratch as variant 0 of pxr_test_groupnorm (its counter zeroed before every call).  -1 when the
 * single-kernel path does not cover the shape. */
int pxr_test_groupnorm_unet(const void* x, const float* gamma, const float* beta, float gamma_add, int act, const void* res,
                            float eps, int pixels, int C, void* y, float* stats, const void* dy, const void* dres, void* dx,
                            float* scratch);
/* the same on the path `path` names: 0 the single-kernel GroupNorm (scratch as above; -1 where it does not cover the
 * shape), 1 the three-kernel GroupNorm the U-Net takes where the single kernel does not fit (any shape with C % 32 == 0,
 * 256 % (C / 8) == 0; scratch: 2 * 64 * partials floats (pxr_test_groupnorm_partials) then the backward's 64). */
int pxr_test_groupnorm_unet_path(int path, const void* x, const float* gamma, const float* beta, float gamma_add, int act,
                                 const void* res, float eps, int pixels, int C, void* y, float* stats, const void* dy,
                                 const void* dres, void* dx, float* scratch);
int pxr_test_groupnorm_partials(int pixels, int C); /* the three-kernel path's block partials at this shape */

/* one resampling / copy kernel on DEVICE NHWC fp16 tensors, by op:
 *   0 upsample2x              in [H, W] (pixel stride ld_in) -> out [2H, 2W]             nearest
 *   1 downsum2x               in [2H, 2W] -> out [H, W]                                  sum of each 2 x 2 block
 *   2 avgpool2x               in [H, W] (pixel stride ld_in) -> out [H/2, W/2]           mean of each 2 x 2 block
 *   3 avgpool2x_backward      in [H/2, W/2] -> out [H, W] (accumulate: adds to out)      its adjoint
 *   4 bilinear_up2x           in [H, W] -> out [2H, 2W] (pixel stride ld_out)            bilinear, align_corners=False
 *   5 bilinear_up2x_backward  in [2H, 2W] (pixel stride ld_in) -> out [H, W]             its adjoint
 *   6 im2col3x3               in [H, W] -> out [H W, 9 C], tap-major, zero outside
 *   7 copy_channels           in [H W] (pixel stride ld_in) -> out (pixel stride ld_out), C channels (accumulate: adds)
 * Sides without a stride above are dense (ld 0 or C); ld 0 means C.  Synchronous.  -1: C % 8 != 0, H or W < 1, or an
 * ld below C or not a multiple of 8; -2: unknown op; -3: a stride or accumulate the op does not take. */
int pxr_test_resample(int op, const void* in, int ld_in, void* out, int ld_out, int H, int W, int C, int accumulate);

/* the U-Net's fp16-weight GEMV: y[r] = act(sum_k w[r, k] x[k] + bias[r]) (+ res[r]), act = ReLU when relu != 0.
 * w DEVICE fp16 [R, K] (K % 8 == 0), x / bias / res / y DEVICE fp32; bias and res nullable.  Synchronous. */
int pxr_test_gemv(const void* w, int K, int R, const float* x, const float* bias, int relu, const float* res, float* y);

/* the row softmax of the unfused attention on DEVICE fp16 [rows, ld] (ld % 8 == 0, cols <= ld; pad columns come back
 * 0): op 0 turns the scores in p_or_s into probabilities in place; op 2 does the same with row r (of each block of cols
 * rows) attending to columns <= r (the text towers' causal softmax); op 1 overwrites dp (dP) with
 * dS = P * (dP - <P, dP>), P in p_or_s.  Synchronous on the default stream. */
int pxr_test_softmax(int op, void* p_or_s, void* dp, int rows, int cols, int ld);

/* the Prompt loss (pixray.py:275-280) of B embeddings against n prompt rows, as the engine runs it: e [B, D] ->
 * e_unit [B, D] (nullable) = e / max(|e|, 1e-12); losses[slots[j]] += |w_j| dist_bj inv_rows[j] / cutn_global summed over
 * the rows b (the caller zeroes losses; slots / inv_rows nullable: j / 1); de [B, D] = grad_scale * d(sum of losses) / de
 * with the gradient of row (b, j) kept only where dist_bj > stops[j] (replace_grad(dists, maximum(dists, stop))),
 * de16 (nullable) its fp16 copy.  dist_bj = 2 asin(min(|e_unit_b - p_j| / 2, 1))^2 sign(w_j).  All DEVICE; D * 8 bytes of
 * shared memory per block.  Synchronous on the default stream; -1 on bad arguments. */
int pxr_test_prompt_loss(const float* e, int B, int D, const float* prompts, const float* weights, const float* stops,
                         const int* slots, const float* inv_rows, int n, int cutn_global, float grad_scale, float* e_unit,
                         float* losses, float* de, void* de16);

/* one CLIP LayerNorm kernel chosen explicitly -- variant 0: fp32 residual stream, 1: fp16 stream with 8-byte vectors,
 * 2: fp16 stream with 16-byte vectors (W % 256 == 0, no pos, fp16 output only) -- forward, or backward (accumulate
 * adds into gx / gx16).  Arguments as the engine's layernorm_forward / layernorm_backward; x is fp32 for variant 0 and
 * fp16 otherwise; y16, dy, gx16 fp16; all DEVICE.  Returns -1 when the variant has no kernel for the width. */
int pxr_test_layernorm(int variant, int backward, const void* x, long long x_stride, const float* pos, int T,
                       const float* gamma, const float* beta, int rows, int W, float eps, void* y16, float* y32,
                       float* stats, const void* dy, int accumulate, float* gx, void* gx16);

#ifdef __cplusplus
}
#endif
#endif
