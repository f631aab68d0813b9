// The engine behind include/pixray_b200.h: owns weights (repacked to the kernels' layouts), every activation /
// gradient buffer, the pre-built kernel plans ("op lists") for forward and the hand-written backward chain, Adam state
// and the per-iteration cutout parameters.  One handle = one rank = one CUDA stream.
//
// Hot path order per iteration (pixray.py:1243-1406, 1436-1512):
//   drawer.synth -> pool -> cutouts -> [per perceptor: patchify -> ViT -> head (or stem -> ResNet -> attnpool) -> Prompt loss]
//   -> backward of all of the above by hand (dgrad only: every network is frozen, vqgan.py:125, slip.py:176)
//   -> [allreduce z.grad] -> Adam -> clip_z
#include "engine.cuh"
#include "comm.cuh"
#include "attn_tc.cuh"
#include "attn_long.cuh"
#include "transforms.h"
#include <algorithm>
#include <atomic>
#include <map>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>

namespace pxr {

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct VSpec;  // one element of the vdiff U-Net description (engine_vdiff.inc)

// ===================================================================================================== Engine
class Engine {
 public:
  pxr_config cfg;
  cudaStream_t st = nullptr;
  std::string err;
  int64_t launches = 0;
  int num_sms = 132;
  int fmt = 0;
  float S = 4096.f;  // grad scale
  bool gn_coop = true;        // PXR_GN_COOP=0: three-kernel GroupNorm instead of the cooperative single-kernel one
  bool stream16 = true;       // the ViT residual stream and its gradient in fp16, like the reference's CUDA path (clip.load gives a half model, slip.py:176); PXR_CLIP_STREAM=32 keeps them in fp32
  bool fused_attn = true;     // PXR_FUSED_ATTN=0: fall back to the batched-GEMM attention (attn_tc.cu covers T <= 240,
                              // attn_long.cu T > 257)
  bool attn_bwd_mma = false;  // PXR_ATTN_BWD=mma: the fused attention backward on attn_bwd_kernel where attn_bwd_wg would run
  std::map<std::string, HostWeight> weights[5];
  std::vector<void*> allocs;
  std::vector<size_t> alloc_bytes;  // bytes of allocs[i] (pxr_test_allocations)
  bool finalized = false;
  std::map<std::string, std::pair<void*, size_t>> dbg;  // named internal buffers (tests / debugging)
  void reg(const std::string& n, void* p, size_t bytes) { dbg[n] = {p, bytes}; }
  // what pack_conv packed and what add_conv planned, in order (pxr_test_packed_weights / pxr_test_conv_records)
  std::vector<pxr_test_pack_rec> pack_log;
  std::vector<pxr_test_conv_rec> conv_log;
  // what add_gemm / add_gemm_splitk planned, in order (pxr_test_gemm_records)
  std::vector<pxr_test_gemm_rec> gemm_log;
  // what add_attention planned, in order (pxr_test_attention_records)
  std::vector<pxr_test_attn_rec> attn_log;

  // sharding
  int n_local = 0, first_global = 0;

  // ---- drawer
  float* z_buf = nullptr;   // engine copy of z
  float* z_grad = nullptr;
  float *adam_m = nullptr, *adam_v = nullptr;
  int adam_t = 0;
  // the optimiser's update rule (PXR_OPT_*); Adagrad keeps its sum in adam_v, Adamax its norm; DiffGrad's previous
  // gradient lives in opt_p, allocated when DiffGrad is first chosen
  int opt_kind = PXR_OPT_ADAM;
  float* opt_p = nullptr;
  void reset_opt_state();
  // device-side checkdrop / learning-rate drops / auto-stop (kernels.cuh): off until pxr_set_schedule
  bool managed = false;
  DropConfig drop_cfg{};
  DropState* drop_state = nullptr;        // [2], double-buffered on the device
  DropStatus* drop_status = nullptr;      // pinned, mapped
  DropStatus* drop_status_dev = nullptr;  // its device address
  float* best_z = nullptr;
  int drop_parity = 0;
  // gradient accumulation over the `batches` passes of one iteration (pixray.py:1464-1482)
  int batches = 1;
  float* z_grad_acc = nullptr;
  int rng_iter = 0;  // key of the engine-drawn cutout parameters: iteration, and pass within the iteration
  int64_t z_numel = 0;
  float *zmin = nullptr, *zmax = nullptr;  // [z_channels]
  float *img = nullptr, *img_pre = nullptr, *g_img = nullptr;  // [3,H,W]
  OpList drawer_fwd, drawer_bwd;  // bwd stored in execution order

  // ---- filters between synth and cutouts (do_synth_and_filter, pixray.py:1203-1222; filters/*.py), fused path only.
  // A filter is a short chain of primitives; `cut_img` / `g_cut_img` [3, cut_h, cut_w] are what MakeCutouts and the image
  // losses see (== img / g_img without filters; wallpaper "shift" doubles the height, edge_match trims).
  enum { FP_ROLL = 0, FP_WSHIFT = 1, FP_CROP = 2, FP_EDGE = 3, FP_LOOKUP = 4 };
  struct FilterPrim {
    int kind, filter;       // primitive kind, index of the filter it belongs to (= its loss slot)
    int Hin, Win, Hout, Wout;
    int use_h = 0, use_w = 0;            // ROLL: which shifts apply
    int top = 0, left = 0;               // CROP
    int em = 0, axis = 0, accumulate = 0;  // EDGE
    float beta = 0.f;                    // LOOKUP
    const float* in = nullptr;           // input tensor (forward)
    float* g_in = nullptr;               // gradient buffer of the input tensor
    float *out = nullptr, *g_out = nullptr;
  };
  struct Filter {
    int kind;               // PXR_FILTER_*
    float weight;
    int wp_type = 0, em = 0;
    float beta = 10.f;
    float* pal = nullptr;
    int n_col = 0;
    int H = 0, W = 0;       // input size of the filter (the shifts are drawn in [0, H) x [0, W), like the reference)
    int sh = 0, sw = 0;     // this iteration's shifts
    int fixed_h = -1, fixed_w = -1;  // explicit shifts for replays (pxr_set_filter_shifts)
  };
  std::vector<Filter> filters;
  std::vector<FilterPrim> fprims;
  float *cut_img = nullptr, *g_cut_img = nullptr;
  int cut_h = 0, cut_w = 0;
  bool filtered_valid = false;  // cut_img holds the filtered image of the current z (fused path); else use img
  int* lookup_best = nullptr;  // nearest-colour index per pixel of a lookup's input (the largest of the program's lookups)
  size_t lookup_best_n = 0;
  void rebuild_filters();
  void filters_forward(int iter);
  void filters_backward();
  const float* cur_cut_img() const { return filtered_valid ? cut_img : img; }
  float* cur_g_cut_img() const { return filtered_valid ? g_cut_img : g_img; }
  int cur_cut_h() const { return filtered_valid ? cut_h : cfg.image_h; }
  int cur_cut_w() const { return filtered_valid ? cut_w : cfg.image_w; }

  // ---- cutouts: one cutout set per distinct perceptor input resolution, in order of first appearance (the reference's
  // cutoutsTable, pixray.py:642-649).  Set 0 has the first perceptor's resolution, cfg.cut_size.  Every set is cut from the
  // same image with its own augmentations and noise; its perceptors see only its batch.
  static constexpr int RING = 8;
  struct CutSet {
    int cs = 0;
    float *pooled = nullptr, *g_pooled = nullptr, *batch = nullptr, *g_batch = nullptr;
    int src_h = 0, src_w = 0;
    float *cut_src = nullptr, *g_cut_src = nullptr;  // [3, src_h, src_w]; == pooled / g_pooled when square
    int* pool_argmax = nullptr;
    float *part_min = nullptr, *part_max = nullptr, *range = nullptr, *sums = nullptr;
    int *part_imin = nullptr, *part_imax = nullptr, *irange = nullptr;
    int n_parts = 0;
    float* minv_host[RING] = {nullptr};   // pinned
    float* facs_host[RING] = {nullptr};
    cudaEvent_t ring_ev[RING] = {nullptr};
    int ring_pos = 0;
    float *minv_dev = nullptr, *facs_dev = nullptr;
    CutoutArgs cut_args;
    float* img_prompts = nullptr;  // [n_img, 3, src_h, src_w]: the pooled (and stretched) image prompt targets
    // cutout-space auxiliary losses' scratch
    float* aux_A = nullptr;       // smoothness per-pixel factor
    float* aux_halo = nullptr;    // smoothness rows of the neighbouring ranks
    float* aux_xbuf = nullptr;    // smoothness halo exchange buffer
    float* aux_blur = nullptr;    // smoothness_gaussian_kernel: blurred batch, its gradient, the one-axis scratch
    float* aux_g_blur = nullptr;  //   (allocated when the first blurred smoothness loss is added, [n_local, 3, cs, cs] each)
    float* aux_blur_tmp = nullptr;
    int* aux_best = nullptr;      // palette argmin per pixel (bookkeeping, also a debug buffer)
    bool cut = false;             // cut since the last backward (the per-op path's pxr_backward takes these back)
  };
  std::vector<CutSet> sets;
  int set_of[4] = {0, 0, 0, 0};  // cutout set of each perceptor
  int n_sets() const { return (int)sets.size(); }
  // non-square canvas (cfg.cut_aspect != 1): the warps sample from a stretch of the pooled image (pixray.py:468-472)
  double aspect = 1.0;
  long long *sums_fx = nullptr, *grad_fx = nullptr;  // 64-bit fixed-point accumulators (order-independent sums, kernels_cutouts.cu)
  unsigned int* fx_poison = nullptr;                   // [2]: pass id of the last non-finite contribution to {gradient images, range sums}
  unsigned int fx_pass = 0;
  FxPass next_fx(int word) {
    FxPass f;
    f.poison = fx_poison + word;
    f.pass = ++fx_pass;
    return f;
  }
  float cj_p = 0.8f, cj_sat = 0.1f, cj_hue = 0.1f;  // K.ColorJitter(hue=0.1, saturation=0.1, p=0.8), pixray.py:416, 436

  // ---- perceptors
  // the weights of one pre-norm transformer block (openai-CLIP ResidualAttentionBlock, timm Block), image or text tower
  struct BlockW {
    act_t *wqkv, *wo, *wfc, *wproj;
    float *bqkv, *bo, *bfc, *bproj;
    NormW ln1, ln2;
  };
  BlockW load_block(int mod, const std::string& prefix, int Wd, bool timm);
  // What add_block reads and writes.  The residual stream runs x_in -> x_mid (after the attention) -> x_out (after the
  // MLP); ln_1, qkv and the attention cover all images * T rows at pitch W, the row-wise tail from out_proj on covers
  // `rows` rows `ld` apart (the class rows only, pitch T W, in the ViT's last layer).  h16 / gact / u hold the tail's
  // rows compactly.  The g* buffers are read only when add_block builds a backward (gx == nullptr on an fp16 stream).
  struct BlockIO {
    const void* x_in;
    void *x_mid, *x_out;
    float *stats1, *stats2;
    act_t *h16, *qkv, *o, *u, *gact;
    int images, heads, T, rows;
    long long ld;
    int act;  // ACT_QUICKGELU or ACT_GELU
    float eps;
    bool causal;
    std::string site;  // the tower and layer, for the attention record
    act_t *go = nullptr, *gqkv = nullptr, *dP = nullptr, *g4 = nullptr, *gh = nullptr, *gx16 = nullptr;
    float* gx = nullptr;
  };
  act_t* add_block(OpList& fwd, OpList* bwd, const BlockW& w, const BlockIO& b);
  void add_head(OpList& l, const void* x, long long ld, int rows, const NormW& n, float eps, act_t* h16, float* stats,
                const act_t* proj16, int Wd, int D, float* out);
  // The residual stream's element type (fp16 with stream16, else fp32) is decided here: a LayerNorm of its rows (pitch
  // ld), its backward (gx, gx16 rows ld apart too), and a GEMM epilogue out = res + A B^T into the stream.
  Op stream_ln_fwd(const void* x, long long ld, const NormW& n, int rows, int Wd, float eps, act_t* y16, float* stats) const;
  Op stream_ln_bwd(const act_t* dy, const void* x, long long ld, const float* stats, const NormW& n, int rows, int Wd,
                   int accumulate, float* gx, act_t* gx16) const;
  void stream_residual(GemmEpilogue& e, const void* res, void* out) const;
  struct Clip {
    pxr_clip_cfg c;
    int tower = PXR_TOWER_OPENAI_CLIP;  // pxr_set_clip_tower
    ChannelNorm norm = kClipNorm;       // the tower's preprocess mean / std
    int T, np, Kp, ldT, M, B;
    // weights
    act_t* conv1 = nullptr;
    float *cls = nullptr, *pos = nullptr, *conv1_b = nullptr;
    NormW ln_pre, ln_post;
    struct Layer {
      BlockW w;
      // saved activations
      void *x_in, *x_mid;  // residual stream before / between the two sub-blocks: fp32, or fp16 with stream16
      float *stats1, *stats2;
      act_t *qkv, *P, *u;
      act_t* o = nullptr;     // fused attention: per-layer attention output (backward needs D = dO . O)
    };
    std::vector<Layer> layers;
    // buffers
    act_t *patches, *g_patches, *h16, *o16, *gact, *g4, *gh, *go, *gqkv, *dP, *gx16;
    float *t, *stats_pre, *stats_post, *e, *e_unit, *de, *gx;
    void* x_out;  // residual stream after the last block (fp32 / fp16)
    act_t *proj16, *hcls, *gcls, *de16;
    // prompts
    float *prompts = nullptr, *pweights = nullptr, *pstops = nullptr, *losses = nullptr;
    int n_prompts = 0, loss_offset = 0;  // n_prompts = loss slots of this perceptor (text + image prompts)
    // rows of `prompts`: n_text single-row Prompts, then cutn rows per image prompt (refreshed every iteration)
    std::vector<float> text_rows, text_w, text_stop;
    int n_text = 0, n_rows = 0;
    int* pslot = nullptr;
    float* pinv = nullptr;
    float* scratch = nullptr;  // pxr_prompt_loss on caller-provided embeddings
    float* ploss_part = nullptr;          // the prompt loss's per-row terms, [B, most rows of one call]
    unsigned int* ploss_count = nullptr;  // its last-block ticket
    // spot prompts (pixray.py:1283-1293): text Prompts scored on the embeddings of the masked cutouts.
    // [1] = args.spot_prompts (make_cutouts(out, spot=1)), [0] = args.spot_prompts_off (spot=0)
    struct Spot {
      std::vector<float> rows, w, stop;
      int n = 0, loss_offset = 0;
      float *d_rows = nullptr, *d_w = nullptr, *d_stop = nullptr, *d_inv = nullptr;
      int* d_slot = nullptr;
    } spot[2];
    OpList fwd, bwd;
  };
  Clip clip[4];
  // ---- text towers (engine_text.inc): encode_text of a perceptor whose weights carry token_embedding.weight.  Built at
  // finalize (host weights are dropped there), forward only, TEXT_CHUNK sequences per run of the op list.
  struct Text {
    int W = 0, L = 0, T = 0, D = 0, heads = 0, vocab = 0;
    act_t *tok = nullptr, *proj16 = nullptr;  // token_embedding [vocab, W], text_projection [W, D]
    float* pos = nullptr;                     // positional_embedding [T, W]
    NormW ln_final;
    std::vector<BlockW> layers;
    int *ids = nullptr, *eot = nullptr;  // [TEXT_CHUNK * T] token ids, [TEXT_CHUNK] row of each sequence's EOT
    void *x0 = nullptr, *x1 = nullptr, *xe = nullptr;  // residual stream ping-pong, gathered EOT rows
    act_t *h16 = nullptr, *qkv = nullptr, *o = nullptr, *u = nullptr, *gact = nullptr, *he = nullptr;
    float *stats = nullptr, *e = nullptr;  // e: [TEXT_CHUNK, D] embeddings
    OpList fwd;
  };
  static constexpr int TEXT_CHUNK = 32;
  std::unique_ptr<Text> text[4];
  void build_text(int i);
  void encode_text(int i, const int32_t* tokens, int n, int ctx, float* out);
  // ---- CLIP ResNet image towers (engine_resnet.inc): the perceptor's Clip keeps its prompts, embeddings and op lists;
  // this holds the tower's own weights and the stem's im2col rows the input stage reads and writes
  struct RnConv {  // a conv with its BatchNorm folded, channel counts padded to multiples of 64
    act_t *w = nullptr, *wd = nullptr;
    float* b = nullptr;
    int cin = 0, cout = 0, ks = 1;
  };
  struct Resnet {
    act_t *cols = nullptr, *g_cols = nullptr;  // [B (cs/2)^2, 64]
    act_t *wq = nullptr, *wkv = nullptr, *wc = nullptr;
    float *bq = nullptr, *bkv = nullptr, *bc = nullptr, *pos = nullptr;
  };
  std::unique_ptr<Resnet> rn[4];
  RnConv rn_conv(int mod, const std::string& conv, const std::string& bn, int cin, int cout, int ks, bool flat);
  void build_resnet(int i);
  // the tower's input stage: the cutouts (batch, range) -> its first GEMM operand, and back into g_batch
  void clip_input(int i);
  void clip_input_backward(int i, bool accumulate, FxPass fx);
  float* losses_dev = nullptr;   // [total prompts]
  float* losses_scratch = nullptr;  // loss vector of the passes b > 0 of an iteration (batches > 1)
  float* losses_host = nullptr;  // pinned
  int total_prompts = 0;
  // image prompts (pixray.py:1308-1336): target images, cut + encoded every iteration with the cached transforms
  // the targets are each set's img_prompts, POOLED ((avg + max) / 2 of each image at its own size, pixray.py:463):
  // constants, pooled once when they are set, not every iteration
  int n_img = 0;
  std::vector<float> img_w;
  void rebuild_prompt_rows();
  void encode_image_prompts(int s);
  // spot passes (one cutout set only): the mask (device [3, cs, cs], != 0 where the mask image is >= 0.5) and the masked pooled image
  unsigned char* spot_mask = nullptr;
  float* pooled_masked = nullptr;
  bool any_spot(int which) const {
    for (int i = 0; i < cfg.n_clip; ++i)
      if (clip[i].spot[which].n > 0) return true;
    return false;
  }
  static const char* spot_multiset_error() {
    return "spot prompts with perceptors of different input resolutions are not built: the reference cuts every "
           "resolution's spot batch with the last MakeCutouts (pixray.py:1270-1276 reuses the loop variable make_cutouts) "
           "and rescales it to each perceptor with torchvision's Resize (slip.py:53-57), whose antialiasing depends on "
           "the torchvision version";
  }
  bool spot_accumulated = false;  // a spot pass of this iteration already wrote d loss / d image: the main pass adds to it
  bool spot_pass(int which, bool accumulate_img);
  void backward_to_image(int s, const CutoutArgs& a, int mask_which, bool accumulate_img, bool main_pass);
  void backward_drawer();

  // ---- auxiliary losses (Losses/*.py; pixray.py:1384-1393): extra loss-vector entries after the prompts
  struct AuxLoss {
    int kind;
    float weight;
    std::vector<float> prm;
    float* dev = nullptr;  // palette colours / aesthetic head weights / smoothness blur taps / edge target, then mask
    int n_dev = 0;
  };
  std::vector<AuxLoss> aux;
  double* aux_part = nullptr;   // reduction scratch
  double* aux_sums = nullptr;   // saturation moments (4)
  // ---- anchors to a stored copy (pixray.py:1344-1375): loss-vector entries between the prompts and the auxiliary losses
  struct Anchor {
    int kind;      // PXR_ANCHOR_*
    float weight;
    float* ref = nullptr;
    size_t n = 0;
  };
  std::vector<Anchor> anchors;
  void anchors_on_image();  // init_weight_pix: into the (filtered) image gradient, before the drawer backward
  void anchors_on_z();      // z-space terms: into z.grad, after the drawer backward
  int aux_base() const { return total_prompts + (int)anchors.size(); }
  // a cutout-space loss (saturation, palette, smoothness) has one entry per cutout set, in set order (the list its
  // get_loss returns, spliced into the loss vector by pixray.py:1392-1398); every other loss has one
  static bool aux_per_set(int kind) {
    return kind == PXR_LOSS_SATURATION || kind == PXR_LOSS_PALETTE || kind == PXR_LOSS_SMOOTHNESS;
  }
  int aux_width(int kind) const { return aux_per_set(kind) ? n_sets() : 1; }
  int aux_slot(size_t k, int s = 0) const {
    int off = aux_base();
    for (size_t j = 0; j < k; ++j) off += aux_width(aux[j].kind);
    return off + s;
  }
  int num_losses() const { return aux_slot(aux.size()); }  // total_prompts includes the filter slots in front
  void aux_after_embed();   // aesthetic: needs de of the last perceptor (after its prompt_loss)
  void aux_on_cutouts(int s);  // saturation / palette / smoothness: add into the set's g_batch
  void aux_on_image();      // symmetry / edge / gaussian: add into g_img

  // ---- comm (multi-GPU, cutout sharding): one NCCL communicator owned by the engine (comm.cuh)
  void* comm = nullptr;
  float* xbuf = nullptr;  // {min, -max} exchange buffer
  void nccl_check(int rc, const char* what) {
    if (rc != 0) {
      const char* m = Comm::api().err_str ? Comm::api().err_str(rc) : "?";
      throw EngineError(-91, std::string(what) + ": NCCL error " + m);
    }
  }

  explicit Engine(const pxr_config& c) : cfg(c) {}
  ~Engine();

  template <class T>
  T* dalloc(size_t n, bool zero = true) {
    void* p = nullptr;
    size_t bytes = (n * sizeof(T) + 255) / 256 * 256;
    PXR_CUDA(cudaMalloc(&p, bytes));
    if (zero) PXR_CUDA(cudaMemsetAsync(p, 0, bytes, st));
    allocs.push_back(p);
    alloc_bytes.push_back(bytes);
    return static_cast<T*>(p);
  }
  // release one tracked allocation early (buffers that are rebuilt when prompts change); cudaFree waits for the device
  template <class T>
  void dfree(T*& p) {
    if (!p) return;
    auto it = std::find(allocs.begin(), allocs.end(), static_cast<void*>(p));
    if (it != allocs.end()) {
      cudaFree(*it);
      alloc_bytes.erase(alloc_bytes.begin() + (it - allocs.begin()));
      allocs.erase(it);
    }
    p = nullptr;
  }
  template <class T>
  T* upload(const std::vector<T>& v) {
    T* p = dalloc<T>(v.size(), false);
    PXR_CUDA(cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st));
    PXR_CUDA(cudaStreamSynchronize(st));  // v may be a temporary
    return p;
  }
  act_t* upload_f16(const std::vector<float>& v) {
    std::vector<act_t> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
    return upload(h);
  }
  const HostWeight& W(int mod, const std::string& name, std::initializer_list<int64_t> dims = {}) {
    auto it = weights[mod].find(name);
    if (it == weights[mod].end()) throw EngineError(-40, "missing weight '" + name + "' (module " + std::to_string(mod) + ")");
    if (dims.size()) {
      std::vector<int64_t> want(dims);
      if (it->second.dims != want) {
        std::string got;
        for (auto d : it->second.dims) got += std::to_string(d) + ",";
        throw EngineError(-41, "weight '" + name + "' has shape [" + got + "] which does not match the configured architecture");
      }
    }
    return it->second;
  }

  // profiling (pxr_profile_iteration): CUDA-event pair around every op, split gemm_tc_kernel vs everything else
  bool profiling = false;
  struct ProfRec {
    cudaEvent_t a, b;
    double flops;
    double bytes;
    int launches;
    std::string name;
  };
  std::vector<ProfRec> prof;
  void prof_begin(ProfRec& r) {
    PXR_CUDA(cudaEventCreate(&r.a));
    PXR_CUDA(cudaEventCreate(&r.b));
    PXR_CUDA(cudaEventRecord(r.a, st));
  }
  // a stage outside the op lists (the cutouts of one set) as one profile record; its launches are not counted again
  void prof_begin_stage(ProfRec& r, const std::string& name) {
    r.flops = r.bytes = 0.0;
    r.launches = 0;
    r.name = name;
    prof_begin(r);
  }
  void prof_end_stage(ProfRec& r) {
    PXR_CUDA(cudaEventRecord(r.b, st));
    prof.push_back(r);
  }
  bool trace = false;  // PXR_TRACE=1: print every op before it runs and synchronise after it (localises a hanging kernel)
  void run(OpList& l) {
    for (size_t i = 0; i < l.ops.size(); ++i) {
      if (trace) {
        fprintf(stderr, "[pxr op] %s\n", l.names[i].empty() ? "(unnamed)" : l.names[i].c_str());
        fflush(stderr);
        l.ops[i]();
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) throw EngineError(-202, std::string("op '") + l.names[i] + "' failed: " + cudaGetErrorString(e));
      } else if (profiling) {
        ProfRec r;
        r.flops = l.flops[i];
        r.bytes = l.bytes[i];
        r.launches = l.launches[i];
        r.name = l.names[i];
        prof_begin(r);
        l.ops[i]();
        PXR_CUDA(cudaEventRecord(r.b, st));
        prof.push_back(r);
      } else {
        l.ops[i]();
      }
      launches += l.launches[i];
    }
  }
  void check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw EngineError(-201, std::string(what) + ": " + cudaGetErrorString(e));
  }

  // ------------------------------------------------------------------ plan helpers
  static GemmOperand opK(const void* p, long long ld, long long mn, long long k, int nb0 = 1, long long bs0 = 0,
                         int nb1 = 1, long long bs1 = 0) {
    GemmOperand o;
    o.ptr = p;
    o.mode = OP_KMAJOR;
    o.ld = ld;
    o.mn_extent = mn;
    o.k_extent = k;
    o.nb0 = nb0;
    o.nb1 = nb1;
    o.bs0 = bs0;
    o.bs1 = bs1;
    return o;
  }
  static GemmOperand opMN(const void* p, long long ld, long long mn, long long k, int nb0 = 1, long long bs0 = 0,
                          int nb1 = 1, long long bs1 = 0) {
    GemmOperand o = opK(p, ld, mn, k, nb0, bs0, nb1, bs1);
    o.mode = OP_MNMAJOR;
    return o;
  }
  // Tile width by a wave-quantisation cost model: a persistent grid of num_sms CTAs runs ceil(tiles / num_sms) waves
  // of tiles whose cost grows with bn (plus a fixed per-tile overhead); e.g. M = 12608, N = 768 is 297 tiles of 256
  // (3 waves for 2.007 waves of work) but 396 tiles of 192 (3 cheaper waves).  wide: the GEMM or convolution may use
  // 192- and 256-wide tiles (gemm_wide_ok); every other one has tiles of at most 128 columns.
  int pick_bn(int N, bool b_mn, long long m_tiles, bool wide = false) const {
    const int step = b_mn ? 64 : 16;
    {  // PXR_GEMM_BN="3072:256,768:192": tile width by output width, for A/B measurements of the cost model's choices
      static const std::map<int, int> forced = [] {
        std::map<int, int> m;
        if (const char* e = getenv("PXR_GEMM_BN")) {
          int n = 0, bn = 0, used = 0;
          while (sscanf(e, "%d:%d%n", &n, &bn, &used) == 2) {
            m[n] = bn;
            e += used;
            if (*e == ',') ++e;
          }
        }
        return m;
      }();
      auto it = forced.find(N);
      if (it != forced.end() && it->second % step == 0 && m_tiles > 16) return it->second;
    }
    // N <= 128: one tile column.  Above 32 columns round up to 64 / 128, the widths with a compile-time wgmma chain
    // (gemm_tc.cu, mma_tile); the extra columns read zero-filled rows of B and are not stored.
    auto narrow = [step](int n) { const int b = round_up(n, step); return b <= 32 ? b : round_up(n, 64); };
    if (N <= 128 && m_tiles * 1 >= num_sms / 2) return narrow(N);
    int best = 0;
    double best_cost = 1e30;
    for (int bn : {256, 192, 128, 64}) {
      if (bn % step || (bn > 128 && !wide)) continue;
      const long long tiles = m_tiles * ((N + bn - 1) / bn);
      const long long waves = (tiles + num_sms - 1) / num_sms;
      // narrower tiles re-read A more often and sit closer to the smem-bandwidth limit: mild penalty
      const double cost = (double)waves * (bn + 40.0) * (bn >= 192 ? 1.0 : (bn == 128 ? 1.06 : 1.2));
      if (cost < best_cost - 1e-9) {
        best_cost = cost;
        best = bn;
      }
    }
    if (N < best) best = narrow(N);
    return best;
  }
  void add_gemm(OpList& l, const GemmOperand& A, const GemmOperand& B, int M, int N, int K, const GemmEpilogue& e,
                int bn = 0) {
    if (!bn) bn = pick_bn(N, B.mode == OP_MNMAJOR, (long long)((M + 127) / 128) * A.nb0 * A.nb1, gemm_wide_ok(A, N, e, fmt));
    auto plan = std::make_shared<GemmPlan>();
    char buf[256] = {0};
    int rc = gemm_plan_make(plan.get(), A, B, M, N, K, e, bn, fmt, num_sms, buf, sizeof buf);
    if (rc) throw EngineError(rc, std::string("gemm plan: ") + buf);
    cudaStream_t s = st;
    const std::string label = gemm_label("gemm", *plan, A.mode, B.mode, e);
    log_gemm(label, *plan, A, B, M, N, K, e, nullptr);
    l.add(1, [plan, s] { gemm_launch(*plan, s); }, plan->flops, label, plan->bytes);
  }
  // one gemm_log record: the operands and epilogue the plan was made from, its choices, and for a split-K plan (epilogue
  // e = the fp32 partial sums) the reduce's bias, residual and output from `red`
  void log_gemm(const std::string& label, const GemmPlan& plan, const GemmOperand& A, const GemmOperand& B, int M, int N,
                int K, const GemmEpilogue& e, const GemmEpilogue* red) {
    pxr_test_gemm_rec r{};
    snprintf(r.label, sizeof r.label, "%s", label.c_str());
    r.a = A.ptr;
    r.a_mode = A.mode;
    r.a_nb0 = A.nb0;
    r.a_nb1 = A.nb1;
    r.lda = A.ld;
    r.a_mn_extent = A.mn_extent;
    r.a_k_extent = A.k_extent;
    r.a_bs0 = A.bs0;
    r.a_bs1 = A.bs1;
    r.b = B.ptr;
    r.b_mode = B.mode;
    r.b_nb0 = B.nb0;
    r.b_nb1 = B.nb1;
    r.ldb = B.ld;
    r.b_mn_extent = B.mn_extent;
    r.b_k_extent = B.k_extent;
    r.b_bs0 = B.bs0;
    r.b_bs1 = B.bs1;
    r.M = M;
    r.N = N;
    r.K = K;
    r.alpha = e.alpha;
    r.bias = e.bias;
    r.bias_per_row = e.bias_per_row;
    r.act = e.act;
    r.act_col0 = e.act_col0;
    r.in_place = (e.res_f16 && e.res_f16 == e.out_f16) || (e.res_f32 && e.res_f32 == e.out_f32) ||
                 (red && red->res_f16 && red->res_f16 == red->out_f16);
    r.aux_in = e.aux_in;
    r.aux_out = e.aux_out;
    r.res_f32 = e.res_f32;
    r.res_f16 = e.res_f16;
    r.out_f32 = e.out_f32;
    r.out_f16 = e.out_f16;
    r.ldc = e.ldc;
    r.c_bs0 = e.bs0;
    r.c_bs1 = e.bs1;
    r.block_n = plan.p.block_n;
    r.wide = plan.p.wide;
    r.stages = plan.p.stages;
    r.tma_epi = plan.p.tma_epi;
    r.grid = plan.grid;
    r.k_splits = plan.p.k_splits;
    r.k_blocks = plan.p.num_k_blocks;
    if (red) {
      r.red_bias = red->bias;
      r.red_res = red->res_f16;
      r.red_out = red->out_f16;
      r.ld_out = red->ldc;
    }
    gemm_log.push_back(r);
  }
  static std::string gemm_label(const char* kind, const GemmPlan& p, int am, int bm, const GemmEpilogue& e) {
    char b[256];
    snprintf(b, sizeof b, "%s M=%d N=%d K=%d batch=%d bn=%d A%s B%s act=%d%s%s%s%s%s%s", kind, p.p.M, p.p.N,
             p.p.num_k_blocks * GEMM_BLOCK_K, p.p.total_tiles / (p.p.tiles_m * p.p.tiles_n), p.p.block_n, am == OP_MNMAJOR ? "mn" : "k", bm == OP_MNMAJOR ? "mn" : "k",
             e.act, e.bias ? " bias" : "", e.res_f32 ? " res32" : "", e.res_f16 ? " res16" : "", e.out_f32 ? " o32" : "",
             e.out_f16 ? " o16" : "", e.aux_out ? " aux" : "");
    return b;
  }
  // Small-spatial convolutions (16x16 / 32x32 latents: 2..64 output tiles, K up to 4608) leave most SMs idle and are
  // bound by the per-SM operand feed; split-K spreads the taps over the idle SMs (fp32 partial sums to a workspace, then
  // one fixed-order reduce + bias / residual / fp16 epilogue kernel: deterministic).
  bool conv_splitk = true;  // PXR_CONV_SPLITK=0 disables
  bool clip_last_cls = true;  // PXR_CLIP_LAST_CLS=0: the last ViT layer's row-wise tail on all rows instead of the class rows
  bool gn_group = true;     // PXR_GN_GROUP=0: never use the cluster-per-group GroupNorm (kernels_gn_group.cu)
  bool gn_fuse_sk = true;   // PXR_GN_FUSE_SPLITK=0: keep splitk_reduce and GroupNorm as two kernels
  bool gn_fuse_fwd = true, gn_fuse_bwd = true;  // PXR_GN_FUSE_FWD / PXR_GN_FUSE_BWD = 0: per direction (diagnostics)
  // the split-K reduce most recently appended by add_conv: a GroupNorm over exactly its output, appended next to the same
  // list, replaces that op by the fused reduce + GroupNorm kernel
  // (one slot per op list: forward and backward lists are built interleaved)
  struct PendingSplitK {
    size_t op_index = 0;
    const act_t* out = nullptr;
    int ld_out = 0, n_out = 0;
    long long px = 0;
    GnSplitK sk;
  };
  std::map<const OpList*, PendingSplitK> pend_sk;
  const GnSplitK* take_pending_splitk(OpList& l, const act_t* tensor, int px, int C, bool need_plain) {
    auto it = pend_sk.find(&l);
    if (!gn_fuse_sk || it == pend_sk.end()) return nullptr;
    const PendingSplitK& q = it->second;
    if (l.ops.empty() || q.op_index != l.ops.size() - 1 || q.out != tensor || q.px != px || q.n_out != C || q.ld_out != C)
      return nullptr;
    if (need_plain && (q.sk.bias || q.sk.res)) return nullptr;
    return &q.sk;
  }
  float* splitk_ws = nullptr;
  size_t splitk_ws_elems = 0;
  // Split count for an output of `rows` x N in `tiles` tiles over nkb k-blocks: enough splits to fill the idle SMs with at
  // least four k-blocks each; 1 (no split) unless the epilogue is an fp16 store the reduce can apply (bias, fp16 residual)
  // and the partial sums fit the workspace.
  int splitk_count(const GemmEpilogue& e, long long rows, int N, int nkb, long long tiles) const {
    if (!conv_splitk || !splitk_ws || !e.out_f16 || e.out_f32 || e.res_f32 || e.aux_out || e.act != ACT_NONE || N % 8 ||
        e.ldc % 8 || tiles * 2 > num_sms || nkb < 8)
      return 1;
    int splits = 1;
    const int want = (int)std::min<long long>(num_sms / tiles, nkb / 4);
    if (want >= 2) {
      const int kbps = (nkb + want - 1) / want;
      splits = (nkb + kbps - 1) / kbps;
    }
    return (size_t)splits * rows * N > splitk_ws_elems ? 1 : splits;
  }
  // in_ld: pixel stride of `in` (0: cin); the conv reads its first cin channels
  void add_conv(OpList& l, const act_t* in, int H, int Wd, int cin, const act_t* wt, int cout_pad, int n_out, int ks,
                const GemmEpilogue& e, long long in_ld = 0, int batch = 1) {
    if (in_ld <= 0) in_ld = cin;
    const long long m_tiles = (long long)(H * Wd + 127) / 128 * batch;
    int bn = pick_bn(cout_pad < 64 ? cout_pad : n_out, false, m_tiles);
    if (bn > cout_pad) bn = cout_pad;
    cudaStream_t s = st;
    char kind[32];
    snprintf(kind, sizeof kind, "conv%dx%d", ks, ks);
    const int nkb = ks * ks * cin / 64;
    const int splits = batch > 1 ? 1 : splitk_count(e, (long long)H * Wd, n_out, nkb, m_tiles * ((n_out + bn - 1) / bn));
    if (splits == 1 && cout_pad >= 64) {  // a conv the 384-thread kernel takes may also use 192- / 256-wide tiles
      GemmOperand A;
      A.mode = OP_CONV;
      if (gemm_wide_ok(A, n_out, e, fmt)) bn = std::min(pick_bn(n_out, false, m_tiles, true), cout_pad);
    }
    auto plan = std::make_shared<GemmPlan>();
    char buf[256] = {0};
    auto log = [&](const std::string& label) {
      const GemmParams& p = plan->p;
      pxr_test_conv_rec r{};
      snprintf(r.label, sizeof r.label, "%s", label.c_str());
      r.wt = wt;
      r.bias = e.bias;
      r.batch = batch;
      r.H = H;
      r.W = Wd;
      r.c_in = cin;
      r.in_ld = in_ld;
      r.cout_pad = cout_pad;
      r.n_out = n_out;
      r.ks = ks;
      r.block_n = p.block_n;
      r.wide = p.wide;
      r.k_splits = p.k_splits;
      r.tma_epi = p.tma_epi;
      r.stages = p.stages;
      r.grid = plan->grid;
      r.act = e.act;
      r.act_col0 = e.act_col0;
      r.has_bias = e.bias != nullptr;
      r.has_res = e.res_f16 != nullptr;
      r.has_aux = e.aux_in != nullptr;
      r.in_place = e.res_f16 && e.res_f16 == e.out_f16;
      r.out_f32 = e.out_f32 != nullptr;
      r.ldc = e.ldc;
      conv_log.push_back(r);
    };
    if (splits > 1) {
      GemmEpilogue pe;
      pe.out_f32 = splitk_ws;
      pe.ldc = n_out;
      pe.k_splits = splits;
      int rc = conv_plan_make(plan.get(), in, in_ld, 1, H, Wd, cin, wt, cout_pad, n_out, ks, pe, bn, fmt, num_sms, buf, sizeof buf);
      if (rc) throw EngineError(rc, std::string("conv plan (split-K): ") + buf);
      const float* ws = splitk_ws;
      const float* bias = e.bias;
      const act_t* res = e.res_f16;
      act_t* out = e.out_f16;
      const int ld_out = (int)e.ldc;
      const long long px = (long long)H * Wd;
      std::string label = gemm_label(kind, *plan, OP_KMAJOR, OP_KMAJOR, e) + " splitK=" + std::to_string(plan->p.k_splits);
      log(label);
      l.add(1, [=] { gemm_launch(*plan, s); }, plan->flops, label, plan->bytes);
      // the reduce is its own op so that a GroupNorm right behind it can absorb it (add_gn / add_gn_bwd)
      l.add(1, [=] { splitk_reduce(ws, plan->p.k_splits, px, n_out, n_out, bias, res, out, ld_out, s); }, 0.0,
            "splitk_reduce px=" + std::to_string(px) + " N=" + std::to_string(n_out) + " splits=" + std::to_string(plan->p.k_splits));
      PendingSplitK& q = pend_sk[&l];
      q.op_index = l.ops.size() - 1;
      q.out = out;
      q.ld_out = ld_out;
      q.px = px;
      q.n_out = n_out;
      q.sk.ws = ws;
      q.sk.splits = plan->p.k_splits;
      q.sk.ld_ws = n_out;
      q.sk.bias = bias;
      q.sk.res = res;
      q.sk.out = out;
      return;
    }
    int rc = conv_plan_make(plan.get(), in, in_ld, batch, H, Wd, cin, wt, cout_pad, n_out, ks, e, bn, fmt, num_sms, buf,
                            sizeof buf);
    if (rc) throw EngineError(rc, std::string("conv plan: ") + buf);
    const std::string label = gemm_label(kind, *plan, OP_KMAJOR, OP_KMAJOR, e);
    log(label);
    l.add(1, [plan, s] { gemm_launch(*plan, s); }, plan->flops, label, plan->bytes);
  }

  // Split-K for a plain K-major GEMM with few output tiles and a long reduction (the vdiff U-Net's 4x4 ... 1x1 levels:
  // M <= 16 pixels, K = 9 * cin up to 18432): partial sums to the shared workspace, then the same fixed-order reduce.
  void add_gemm_splitk(OpList& l, const GemmOperand& A, const GemmOperand& B, int M, int N, int K, const GemmEpilogue& e) {
    const int bn = pick_bn(N, false, (M + 127) / 128);
    const int nkb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
    const long long tiles = (long long)((M + 127) / 128) * ((N + bn - 1) / bn);
    const int splits = e.alpha == 1.f ? splitk_count(e, M, N, nkb, tiles) : 1;  // the reduce applies no alpha
    if (splits <= 1) {
      add_gemm(l, A, B, M, N, K, e);
      return;
    }
    auto plan = std::make_shared<GemmPlan>();
    char buf[256] = {0};
    GemmEpilogue pe;
    pe.out_f32 = splitk_ws;
    pe.ldc = N;
    pe.k_splits = splits;
    pe.tma_epi = -1;
    int rc = gemm_plan_make(plan.get(), A, B, M, N, K, pe, bn, fmt, num_sms, buf, sizeof buf);
    if (rc) throw EngineError(rc, std::string("gemm plan (split-K): ") + buf);
    cudaStream_t s = st;
    const float* ws = splitk_ws;
    const float* bias = e.bias;
    const act_t* res = e.res_f16;
    act_t* out = e.out_f16;
    const int ld_out = (int)e.ldc;
    std::string label = gemm_label("gemm", *plan, A.mode, B.mode, e) + " splitK=" + std::to_string(plan->p.k_splits);
    log_gemm(label, *plan, A, B, M, N, K, pe, &e);
    l.add(2, [=] {
      gemm_launch(*plan, s);
      splitk_reduce(ws, plan->p.k_splits, M, N, N, bias, res, out, ld_out, s);
    }, plan->flops, label, plan->bytes);
  }

  // ------------------------------------------------------------------ build steps
  void create();
  void finalize();
  void build_vqgan();
  void build_pixel();
  void build_polygon();
  // polygon drawer: host copies from pxr_set_polygons ([total_vertices, 2] and [n + 1] offsets), the binned scene, the
  // per-sample winners of the last render, and the iteration that keys the render's sample positions
  std::vector<float> poly_xy;
  std::vector<int> poly_off;
  RasterScene scene{};
  int* poly_winner = nullptr;
  int synth_iter = 0;
  void build_strokes();
  // line-sketch drawer: the shape from pxr_set_strokes and the per-render scene (kernels.cuh StrokeScene)
  int stroke_paths = 0, stroke_segments = 0, stroke_paper = 0;
  float stroke_max_width = 0.f;
  StrokeScene sscene{};
  ZRanges zr = zranges_single();  // per-range Adam rates and clamp (the line drawer's three optimisers)
  void build_fft();
  FftPlans* fft = nullptr;
  void build_cutouts();
  void build_clip(int i);
  ConvW load_conv(const std::string& prefix, int cin, int cout, int ks, int cin_real = 0, bool has_bias = true);
  act_t* pack_conv(const std::string& tag, const std::vector<float>& w, int cout, int cin, int taps, size_t n, size_t s_tap,
                   size_t s_co, size_t s_ci, bool flip, int ci0 = 0, int ci1 = INT_MAX);
  // VQGAN encoder (taming Encoder + quant_conv + nearest code): VqganDrawer.init_from_tensor / reapply_from_tensor /
  // get_z_from_tensor (vqgan.py:174-185).  Forward only; built at finalize when the checkpoint carries encoder.* tensors.
  OpList enc_fwd;
  bool have_encoder = false;
  float* enc_img = nullptr;   // [3, H, W] input in [-1, 1]
  float* enc_z = nullptr;     // [C, hw] result
  // a GumbelVQ checkpoint (codebook quantize.embed.weight): the encoder quantises with quantize.proj's logits plus the
  // caller's Gumbel noise [n_embed, hw] (pxr_vqgan_encode_gumbel) instead of the nearest code
  bool vq_gumbel = false;
  float* enc_noise = nullptr;
  void build_vqgan_encoder();
  NormW load_norm(int mod, const std::string& prefix, int c);
  Act new_act(int H, int Wd, int C, bool grad = true) {
    Act a;
    a.H = H;
    a.W = Wd;
    a.C = C;
    a.p = dalloc<act_t>((size_t)H * Wd * C);
    if (grad) a.g = dalloc<act_t>((size_t)H * Wd * C);
    return a;
  }
  // the codebook [n_embed, z_channels], its transpose and squared row norms, as the nearest-code search reads them
  // (build_vqgan; the encoder's quantiser reads the same copies)
  float *vq_cb = nullptr, *vq_cbT = nullptr, *vq_c2 = nullptr;
  // decoder blocks: append forward ops to drawer_fwd, push the backward closure list (reverse order) to bwd_stack
  std::vector<OpList> bwd_stack;
  float* gn_part = nullptr;  // scratch for GN partial sums (sized for the largest layer)
  GridBarrier gn_bar;        // grid barrier state of the single-kernel GroupNorm
  Act conv_fwd_bwd(const Act& x, const ConvW& w, OpList& bwd);
  Act upsample(const Act& x, const std::string& prefix);
  struct GNSaved {
    float* stats;
    float* gstats;
  };
  // taming ResnetBlock / AttnBlock, shared by the decoder and the encoder: the forward builder appends to `l` and returns
  // what the backward builder needs (grad = false allocates no gradient buffers: the encoder); the backward builder
  // pushes its op list onto bwd_stack
  struct ResBlock {
    NormW n1, n2;
    ConvW c1, c2, sc;
    Act x, a1, h1, a2, out;
    GNSaved s1, s2;
  };
  struct AttnBlock {
    NormW n;
    act_t* wqkv;
    ConvW po;
    Act x, a, O, out;
    act_t* gqkv;
    GNSaved s;
    OpList attn_bwd;  // dO -> gqkv, from add_attention
  };
  ResBlock resblock_fwd(OpList& l, const Act& x, const std::string& prefix, int cin, int cout, bool grad);
  void resblock_bwd(const ResBlock& r);
  AttnBlock attnblock_fwd(OpList& l, const Act& x, const std::string& prefix, int c, bool grad);
  void attnblock_bwd(const AttnBlock& a);
  // Self-attention O = softmax(scale q k^T) v of `images` x `heads` heads of width d over T tokens, in attn_tc.cuh's
  // layout: qkv and gqkv [images T, 3 heads d] (q | k | v, head h at column h d of each third), o and d_o
  // [images T, heads d].  Appends the forward to `fwd` and, when `bwd` is given, the backward (d_o -> gqkv) to *bwd.
  // multihead (the ViT, the U-Net): the fused kernels when attn_fused() holds (attn_tc.cu, T <= 240), the streaming
  // ones when attn_streamed() holds (attn_long.cu, T > 257), else the batched-GEMM chain with tile widths fixed for the
  // head-batched shapes; otherwise (taming's AttnBlock) always the chain, tile widths by add_gemm.
  // The chain's P is allocated here (and returned; nullptr on the fused paths), its dP too unless the caller passes a
  // scratch that several calls share.  causal (the text towers): row t attends to tokens <= t; forward only, multihead,
  // on the fused kernel or the chain with a causal row softmax (T <= 240 either way).  Each call appends one record to
  // attn_log; `site` names the caller there.
  act_t* add_attention(const std::string& site, OpList& fwd, OpList* bwd, const act_t* qkv, act_t* o, const act_t* d_o, act_t* gqkv, int images,
                       int heads, int T, int d, float scale, bool multihead, act_t* dP = nullptr, bool causal = false);
  bool attn_fused(int T, int d, int heads) const { return fused_attn && attn_supported(T, d, heads * d); }
  // T = 256 / 257 (the vdiff 16^2 level, ViT-L/14) stay on the chain: the streaming kernels start past them
  bool attn_streamed(int T, int d, int heads) const {
    return fused_attn && T > 257 && attn_long_supported(T, d, heads * d);
  }
  GNSaved add_gn(OpList& l, const Act& x, const NormW& n, int swish, act_t* y);
  void add_gn_bwd(OpList& l, const act_t* dy, const act_t* x, const GNSaved& s, const NormW& n, int px, int C, int swish,
                  const act_t* dres, act_t* dx);

  // ------------------------------------------------------------------ vdiff drawer (engine_vdiff.inc)
  struct VConv;
  void build_vdiff();
  VConv vd_load_conv(const std::string& prefix, int cin_real, int cin, int cout, int ks, bool has_bias, bool tiny);
  void vd_conv_fwd(OpList& l, const act_t* x, int H, int Wd, const VConv& v, GemmEpilogue e);
  void vd_conv_bwd(OpList& l, const act_t* dy, int H, int Wd, const VConv& v, GemmEpilogue e);
  void vd_check_col(size_t elems) const;
  GNSaved vd_norm(OpList& l, const Act& x, const float* gamma, const float* beta, float gamma_add, int act,
                  const act_t* res, act_t* y);
  void vd_norm_bwd(OpList& l, const act_t* dy, const Act& x, const GNSaved& s, const float* gamma, const float* beta,
                   float gamma_add, int act, const act_t* dres, act_t* dx);
  Act vd_block(const Act& x, const std::string& key, const VSpec& sp);
  Act vd_attn(const Act& x, const std::string& key, const VSpec& sp);
  Act vd_skip(const Act& x, const std::string& key, const VSpec& sp);
  Act vd_elem(const Act& x, const std::string& key, const VSpec& sp);
  int vd_add_modulation(const std::string& wkey, int c);
  void vdiff_prepare(int iter);
  void vdiff_forward();
  void vdiff_backward();
  std::vector<float> vd_steps, vd_alphas, vd_sigmas, vd_map_ff, vd_t_ff, vd_mod_host;
  bool vd_have_embed = false;
  int vd_iter = 0, vd_iter_request = 0, vd_mod_rows = 0;
  float *vd_pred = nullptr, *vd_v = nullptr, *vd_gpred = nullptr, *vd_vout = nullptr, *vd_mod_out = nullptr,
        *vd_h0 = nullptr, *vd_te = nullptr, *vd_tmp[5] = {nullptr}, *vd_b[5] = {nullptr};
  act_t *vd_gv = nullptr, *vd_col = nullptr, *vd_xin = nullptr, *vd_gin = nullptr, *vd_wmod = nullptr, *vd_w[5] = {nullptr};
  // the U-Net's size (pxr_vdiff_set_gen_size; 0: the canvas) and the canvas's window in it
  int vd_gen_h = 0, vd_gen_w = 0;
  VdCrop vd_crop{};
  size_t vd_col_elems = 0, gn_part_elems = 0;
  float* vd_gstats = nullptr;  // the three-kernel GroupNorm backward's [32][2] fold (one norm runs at a time)

  // ------------------------------------------------------------------ super-resolution drawer (engine_superres.inc)
  struct SrConv;
  void build_superres();
  SrConv sr_load_conv(const std::string& prefix, int cin, int cout, float scale);

  // ------------------------------------------------------------------ execution
  void prepare_cut_params(int s, const pxr_cut_params* p, int iter);
  void forward_drawer() {
    if (cfg.drawer == PXR_DRAWER_VDIFF) vdiff_forward();
    else run(drawer_fwd);
  }
  void forward_cutouts(int s);
  void forward_clip(int i);
  void loss_clip(int i);
  void backward_all();
  int clip_mode() const;
  void step(float lr);
  void step_managed(int iter);
  void write_initial_drop_state();
};

Engine::~Engine() {
  if (st) cudaStreamSynchronize(st);
  if (comm && Comm::api().destroy) Comm::api().destroy(comm);
  fft_plans_destroy(fft);
  for (void* p : allocs) cudaFree(p);
  for (CutSet& K : sets)
    for (int i = 0; i < RING; ++i) {
      if (K.minv_host[i]) cudaFreeHost(K.minv_host[i]);
      if (K.facs_host[i]) cudaFreeHost(K.facs_host[i]);
      if (K.ring_ev[i]) cudaEventDestroy(K.ring_ev[i]);
    }
  if (losses_host) cudaFreeHost(losses_host);
  if (drop_status) cudaFreeHost(const_cast<DropStatus*>(drop_status));
  if (st) cudaStreamDestroy(st);
}

void Engine::create() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    throw EngineError(-1, "no CUDA device: pixray_b200 has no CPU fallback");
  if (cfg.device < 0 || cfg.device >= ndev) throw EngineError(-2, "invalid CUDA device ordinal");
  PXR_CUDA(cudaSetDevice(cfg.device));
  cudaDeviceProp prop;
  PXR_CUDA(cudaGetDeviceProperties(&prop, cfg.device));
  if (prop.major != 9) throw EngineError(-3, std::string("pixray_b200 needs an sm_90 GPU (H100); found ") + prop.name);
  num_sms = prop.multiProcessorCount;
  PXR_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  if (cfg.world < 1) cfg.world = 1;
  if (cfg.cutn % cfg.world) throw EngineError(-4, "cutn must be divisible by world");
  n_local = cfg.cutn / cfg.world;
  first_global = cfg.rank * n_local;
  fmt = cfg.op_dtype;
  if (fmt != PXR_DTYPE_F16) throw EngineError(-5, "only PXR_DTYPE_F16 operands are wired through the pointwise kernels");
  if (cfg.grad_scale > 0) S = cfg.grad_scale;
  if (const char* fa = getenv("PXR_FUSED_ATTN")) fused_attn = atoi(fa) != 0;
  if (const char* ab = getenv("PXR_ATTN_BWD")) attn_bwd_mma = strcmp(ab, "mma") == 0;
  if (const char* cs16 = getenv("PXR_CLIP_STREAM")) stream16 = atoi(cs16) != 32;
  if (const char* gc = getenv("PXR_GN_COOP")) gn_coop = atoi(gc) != 0;
  if (const char* sk = getenv("PXR_CONV_SPLITK")) conv_splitk = atoi(sk) != 0;
  if (const char* lc = getenv("PXR_CLIP_LAST_CLS")) clip_last_cls = atoi(lc) != 0;
  if (const char* gg = getenv("PXR_GN_GROUP")) gn_group = atoi(gg) != 0;
  if (const char* gf = getenv("PXR_GN_FUSE_SPLITK")) gn_fuse_sk = atoi(gf) != 0;
  if (const char* gf = getenv("PXR_GN_FUSE_FWD")) gn_fuse_fwd = atoi(gf) != 0;
  if (const char* gf = getenv("PXR_GN_FUSE_BWD")) gn_fuse_bwd = atoi(gf) != 0;
  if (const char* tr = getenv("PXR_TRACE")) trace = atoi(tr) != 0;
  if (cfg.beta1 <= 0) cfg.beta1 = 0.9f;
  if (cfg.beta2 <= 0) cfg.beta2 = 0.999f;
  if (cfg.adam_eps <= 0) cfg.adam_eps = 1e-8f;
  if (cfg.cut_size % 4) throw EngineError(-6, "cut_size must be a multiple of 4");
}

// ===================================================================================================== weights
NormW Engine::load_norm(int mod, const std::string& prefix, int c) {
  NormW n;
  n.gamma = upload(W(mod, prefix + ".weight", {c}).data);
  n.beta = upload(W(mod, prefix + ".bias", {c}).data);
  return n;
}

// The one conv weight packer: scatters a PyTorch weight w [cout][cin][taps] into a zeroed fp16 operand of n elements,
// (co, ci, t) to t' s_tap + co s_co + (ci - ci0) s_ci, where t' = t, or taps - 1 - t with flip (a dgrad: dx[p] = sum_t
// dy[p + off(t)] W[.., flipped t]).  Only the input channels [ci0, ci1) are packed.  tag: the conv's checkpoint prefix,
// recorded with the layout for pxr_test_packed_weights.
act_t* Engine::pack_conv(const std::string& tag, const std::vector<float>& w, int cout, int cin, int taps, size_t n,
                         size_t s_tap, size_t s_co, size_t s_ci, bool flip, int ci0, int ci1) {
  std::vector<float> f(n, 0.f);
  for (int co = 0; co < cout; ++co)
    for (int ci = ci0; ci < std::min(ci1, cin); ++ci)
      for (int t = 0; t < taps; ++t)
        f[(flip ? taps - 1 - t : t) * s_tap + co * s_co + (ci - ci0) * s_ci] = w[((size_t)co * cin + ci) * taps + t];
  act_t* p = upload_f16(f);
  pxr_test_pack_rec r{};
  snprintf(r.tag, sizeof r.tag, "%s", tag.c_str());
  r.ptr = p;
  r.src = w.data();
  r.n = (long long)n;
  r.s_tap = (long long)s_tap;
  r.s_co = (long long)s_co;
  r.s_ci = (long long)s_ci;
  r.cout = cout;
  r.cin = cin;
  r.taps = taps;
  r.flip = flip;
  r.ci0 = ci0;
  r.ci1 = std::min(ci1, cin);
  pack_log.push_back(r);
  return p;
}

// cin_real < cin: the stored tensor has cin_real input channels and the activation is zero-padded to cin (conv_in: 3 -> 64)
ConvW Engine::load_conv(const std::string& prefix, int cin, int cout, int ks, int cin_real, bool has_bias) {
  if (cin_real <= 0) cin_real = cin;
  const HostWeight& w = W(PXR_MOD_VQGAN, prefix + ".weight", {cout, cin_real, ks, ks});
  ConvW c;
  c.cin = cin;
  c.cout = cout;
  c.ks = ks;
  c.cout_pad = round_up(cout, 16);
  c.cout_k = round_up(cout, 64);
  c.cin_rows = round_up(cin, 16);
  const int taps = ks * ks;
  if (cin % 64) throw EngineError(-42, "conv '" + prefix + "': input channels must be a multiple of 64");
  c.w = pack_conv(prefix, w.data, cout, cin_real, taps, (size_t)taps * c.cout_pad * cin, (size_t)c.cout_pad * cin, cin, 1, false);
  c.wd = pack_conv(prefix, w.data, cout, cin_real, taps, (size_t)taps * c.cin_rows * c.cout_k, (size_t)c.cin_rows * c.cout_k,
                   1, c.cout_k, true);
  if (has_bias) c.bias = upload(W(PXR_MOD_VQGAN, prefix + ".bias", {cout}).data);
  return c;
}

// ===================================================================================================== VQGAN drawer
Engine::GNSaved Engine::add_gn(OpList& l, const Act& x, const NormW& n, int swish, act_t* y) {
  GNSaved s;
  s.stats = dalloc<float>(64);
  s.gstats = dalloc<float>(64);
  const act_t* xp = x.p;
  int px = x.pixels(), C = x.C;
  float* part = gn_part;
  float* stats = s.stats;
  cudaStream_t cs = st;
  NormW nn = n;
  const int nsm = num_sms;
  if (gn_group && gn_group_supported(px, C)) {
    const std::string shape = " px=" + std::to_string(px) + " C=" + std::to_string(C);
    if (const GnSplitK* pk = gn_fuse_fwd ? take_pending_splitk(l, xp, px, C, false) : nullptr) {
      const GnSplitK sk = *pk;
      l.ops.back() = [=] { gn_forward_group(nullptr, &sk, nn.gamma, nn.beta, px, C, swish, 1e-6f, stats, y, cs); };
      l.names.back() = "splitk_reduce+gn_fwd_group" + shape + " splits=" + std::to_string(sk.splits);
      pend_sk.erase(&l);
    } else {
      l.add(1, [=] { gn_forward_group(xp, nullptr, nn.gamma, nn.beta, px, C, swish, 1e-6f, stats, y, cs); }, 0.0,
            "gn_fwd_group" + shape);
    }
  } else if (gn_coop && gn_coop_supported(px, C, nsm)) {
    GridBarrier* gb = &gn_bar;
    l.add(1, [=] { gn_forward_coop(xp, nn.gamma, nn.beta, px, C, swish, 1e-6f, part, stats, y, nsm, gb, cs); }, 0.0,
          "gn_fwd_coop px=" + std::to_string(px) + " C=" + std::to_string(C));
  } else {
    l.add(3, [=] {
      gn_stats(xp, px, C, 1e-6f, part, stats, cs);
      gn_apply(xp, stats, nn.gamma, nn.beta, px, C, swish, y, cs);
    }, 0.0, "gn_fwd_3k px=" + std::to_string(px) + " C=" + std::to_string(C));
  }
  return s;
}

void Engine::add_gn_bwd(OpList& l, const act_t* dy, const act_t* x, const GNSaved& s, const NormW& n, int px, int C,
                        int swish, const act_t* dres, act_t* dx) {
  float* part = gn_part;
  cudaStream_t cs = st;
  const int nsm = num_sms;
  GridBarrier* gb = &gn_bar;
  if (gn_group && gn_group_supported(px, C)) {
    const std::string shape = " px=" + std::to_string(px) + " C=" + std::to_string(C);
    if (const GnSplitK* pk = gn_fuse_bwd ? take_pending_splitk(l, dy, px, C, true) : nullptr) {
      const GnSplitK sk = *pk;  // dy itself is never written: the reduced gradient lives in registers only
      l.ops.back() = [=] { gn_backward_group(nullptr, &sk, x, s.stats, n.gamma, n.beta, px, C, swish, dres, dx, cs); };
      l.names.back() = "splitk_reduce+gn_bwd_group" + shape + " splits=" + std::to_string(sk.splits);
      pend_sk.erase(&l);
    } else {
      l.add(1, [=] { gn_backward_group(dy, nullptr, x, s.stats, n.gamma, n.beta, px, C, swish, dres, dx, cs); }, 0.0,
            "gn_bwd_group" + shape);
    }
  } else if (gn_coop && gn_coop_supported(px, C, nsm))
    l.add(1, [=] { gn_backward_coop(dy, x, s.stats, n.gamma, n.beta, px, C, swish, dres, part, dx, nsm, gb, cs); }, 0.0,
          "gn_bwd_coop px=" + std::to_string(px) + " C=" + std::to_string(C));
  else
    l.add(3, [=] { gn_backward(dy, x, s.stats, n.gamma, n.beta, px, C, swish, dres, part, s.gstats, dx, cs); }, 0.0,
          "gn_bwd_3k px=" + std::to_string(px) + " C=" + std::to_string(C));
}

// y = conv(x) (+bias), returns y; appends dgrad op (x.g = conv_dgrad(y.g)) to bwd (caller orders it)
Act Engine::conv_fwd_bwd(const Act& x, const ConvW& w, OpList& bwd) {
  Act y = new_act(x.H, x.W, w.cout);
  GemmEpilogue e;
  e.bias = w.bias;
  e.out_f16 = y.p;
  e.ldc = y.C;
  add_conv(drawer_fwd, x.p, x.H, x.W, x.C, w.w, w.cout_pad, w.cout, w.ks, e);
  GemmEpilogue d;
  d.out_f16 = x.g;
  d.ldc = x.C;
  add_conv(bwd, y.g, x.H, x.W, w.cout_k, w.wd, w.cin_rows, w.cin, w.ks, d);
  return y;
}

Engine::ResBlock Engine::resblock_fwd(OpList& l, const Act& x, const std::string& prefix, int cin, int cout, bool grad) {
  ResBlock r;
  r.x = x;
  r.n1 = load_norm(PXR_MOD_VQGAN, prefix + ".norm1", cin);
  r.n2 = load_norm(PXR_MOD_VQGAN, prefix + ".norm2", cout);
  r.c1 = load_conv(prefix + ".conv1", cin, cout, 3);
  r.c2 = load_conv(prefix + ".conv2", cout, cout, 3);
  const int H = x.H, Wd = x.W;
  r.a1 = new_act(H, Wd, cin, grad);
  r.h1 = new_act(H, Wd, cout, grad);
  r.a2 = new_act(H, Wd, cout, grad);
  r.out = new_act(H, Wd, cout, grad);
  r.s1 = add_gn(l, x, r.n1, 1, r.a1.p);
  {
    GemmEpilogue e;
    e.bias = r.c1.bias;
    e.out_f16 = r.h1.p;
    e.ldc = cout;
    add_conv(l, r.a1.p, H, Wd, cin, r.c1.w, r.c1.cout_pad, cout, 3, e);
  }
  r.s2 = add_gn(l, r.h1, r.n2, 1, r.a2.p);
  if (cin != cout) {
    r.sc = load_conv(prefix + ".nin_shortcut", cin, cout, 1);
    GemmEpilogue e;
    e.bias = r.sc.bias;
    e.out_f16 = r.out.p;
    e.ldc = cout;
    add_conv(l, x.p, H, Wd, cin, r.sc.w, r.sc.cout_pad, cout, 1, e);
  }
  {
    GemmEpilogue e;
    e.bias = r.c2.bias;
    e.res_f16 = (cin != cout) ? r.out.p : x.p;
    e.out_f16 = r.out.p;
    e.ldc = cout;
    add_conv(l, r.a2.p, H, Wd, cout, r.c2.w, r.c2.cout_pad, cout, 3, e);
  }
  return r;
}

void Engine::resblock_bwd(const ResBlock& r) {
  const Act& x = r.x;
  const int H = x.H, Wd = x.W, px = x.pixels(), cin = r.c1.cin, cout = r.c1.cout;
  OpList b;  // execution order
  {
    GemmEpilogue e;
    e.out_f16 = r.a2.g;
    e.ldc = cout;
    add_conv(b, r.out.g, H, Wd, r.c2.cout_k, r.c2.wd, r.c2.cin_rows, cout, 3, e);
  }
  add_gn_bwd(b, r.a2.g, r.h1.p, r.s2, r.n2, px, cout, 1, nullptr, r.h1.g);
  {
    GemmEpilogue e;
    e.out_f16 = r.a1.g;
    e.ldc = cin;
    add_conv(b, r.h1.g, H, Wd, r.c1.cout_k, r.c1.wd, r.c1.cin_rows, cin, 3, e);
  }
  if (cin != cout) {
    GemmEpilogue e;
    e.out_f16 = x.g;
    e.ldc = cin;
    add_conv(b, r.out.g, H, Wd, r.sc.cout_k, r.sc.wd, r.sc.cin_rows, cin, 1, e);
    add_gn_bwd(b, r.a1.g, x.p, r.s1, r.n1, px, cin, 1, x.g, x.g);
  } else {
    add_gn_bwd(b, r.a1.g, x.p, r.s1, r.n1, px, cin, 1, r.out.g, x.g);
  }
  bwd_stack.push_back(std::move(b));
}

Engine::AttnBlock Engine::attnblock_fwd(OpList& l, const Act& x, const std::string& prefix, int c, bool grad) {
  AttnBlock a;
  a.x = x;
  a.n = load_norm(PXR_MOD_VQGAN, prefix + ".norm", c);
  // fused q/k/v 1x1 convs: weight [3c, c]
  std::vector<float> wq, bq;
  for (const char* nm : {".q", ".k", ".v"}) {
    const HostWeight& w = W(PXR_MOD_VQGAN, prefix + nm + ".weight", {c, c, 1, 1});
    const HostWeight& b = W(PXR_MOD_VQGAN, prefix + nm + ".bias", {c});
    wq.insert(wq.end(), w.data.begin(), w.data.end());
    bq.insert(bq.end(), b.data.begin(), b.data.end());
  }
  a.wqkv = upload_f16(wq);
  float* bqkv = upload(bq);
  a.po = load_conv(prefix + ".proj_out", c, c, 1);
  const int T = x.pixels();
  a.a = new_act(x.H, x.W, c, grad);
  a.O = new_act(x.H, x.W, c, grad);
  a.out = new_act(x.H, x.W, c, grad);
  act_t* qkv = dalloc<act_t>((size_t)T * 3 * c);
  a.gqkv = grad ? dalloc<act_t>((size_t)T * 3 * c) : nullptr;
  a.s = add_gn(l, x, a.n, 0, a.a.p);
  {
    GemmEpilogue e;
    e.bias = bqkv;
    e.out_f16 = qkv;
    e.ldc = 3 * c;
    add_gemm(l, opK(a.a.p, c, T, c), opK(a.wqkv, c, 3 * c, c), T, 3 * c, c, e);
  }
  add_attention(prefix, l, grad ? &a.attn_bwd : nullptr, qkv, a.O.p, a.O.g, a.gqkv, 1, 1, T, c, 1.f / std::sqrt((float)c), false);
  {
    GemmEpilogue e;
    e.bias = a.po.bias;
    e.res_f16 = x.p;
    e.out_f16 = a.out.p;
    e.ldc = c;
    add_conv(l, a.O.p, x.H, x.W, c, a.po.w, a.po.cout_pad, c, 1, e);
  }
  return a;
}

void Engine::attnblock_bwd(const AttnBlock& a) {
  const Act& x = a.x;
  const int T = x.pixels(), c = x.C;
  OpList b;
  {
    GemmEpilogue e;
    e.out_f16 = a.O.g;
    e.ldc = c;
    add_conv(b, a.out.g, x.H, x.W, a.po.cout_k, a.po.wd, a.po.cin_rows, c, 1, e);
  }
  b.append(a.attn_bwd);
  {  // da = dqkv Wqkv   (B = Wqkv stored [3c (k), c (n)] -> MN-major)
    GemmEpilogue e;
    e.out_f16 = a.a.g;
    e.ldc = c;
    add_gemm(b, opK(a.gqkv, 3 * c, T, 3 * c), opMN(a.wqkv, c, c, 3 * c), T, c, 3 * c, e);
  }
  add_gn_bwd(b, a.a.g, x.p, a.s, a.n, T, c, 0, a.out.g, x.g);
  bwd_stack.push_back(std::move(b));
}

act_t* Engine::add_attention(const std::string& site, OpList& fwd, OpList* bwd, const act_t* qkv, act_t* o,
                             const act_t* d_o, act_t* gqkv, int images, int heads, int T, int d, float scale,
                             bool multihead, act_t* dP, bool causal) {
  const int W = heads * d, ldT = round_up(T, 8);
  cudaStream_t cs = st;
  if (causal && (bwd || !multihead || !attn_supported(T, d, W)))
    throw EngineError(-54, "causal attention is forward only, with 64-wide heads and T <= 240");
  attn_log.emplace_back();
  pxr_test_attn_rec& rec = attn_log.back();
  snprintf(rec.site, sizeof rec.site, "%s", site.c_str());
  rec.multihead = multihead;
  rec.causal = causal;
  rec.backward = bwd != nullptr;
  rec.images = images;
  rec.heads = heads;
  rec.T = T;
  rec.d = d;
  rec.W = W;
  rec.scale = scale;
  rec.qkv = qkv;
  rec.o = o;
  rec.d_o = d_o;
  rec.gqkv = gqkv;
  rec.splits = 1;
  for (int& g : rec.gemm) g = -1;
  if (multihead && attn_fused(T, d, heads)) {  // S, softmax and PV in one kernel; S / P never leave the SM
    float* lse = dalloc<float>((size_t)images * heads * T);
    auto ap = std::make_shared<AttnPlan>();
    char buf[256] = {0};
    int rc = attn_plan_make(ap.get(), qkv, o, d_o, gqkv, lse, images, T, heads, W, scale, num_sms, buf, sizeof buf, causal,
                            attn_bwd_mma ? ATTN_BWD_MMA : ATTN_BWD_AUTO);
    if (rc) throw EngineError(rc, std::string("attention plan: ") + buf);
    rec.path = PXR_ATTN_FUSED;
    rec.lse = lse;
    rec.splits = ap->splits;
    rec.bwd = ap->bwd;
    char lab[96];
    snprintf(lab, sizeof lab, "attn_fwd%s B=%d T=%d heads=%d", causal ? "_causal" : "", images, T, heads);
    fwd.add(1, [ap, cs] { attn_forward_launch(*ap, cs); }, ap->flops_fwd, lab, ap->bytes_fwd);
    if (bwd) {  // dQ, dK, dV in one kernel (recomputes P from Q, K and the saved log-sum-exp)
      snprintf(lab, sizeof lab, "attn_bwd B=%d T=%d heads=%d", images, T, heads);
      bwd->add(1, [ap, cs] { attn_backward_launch(*ap, cs); }, ap->flops_bwd, lab, ap->bytes_bwd);
    }
    return nullptr;
  }
  if (multihead && attn_streamed(T, d, heads)) {  // K / V streamed through shared memory; S / P never leave the SM
    float* lse = dalloc<float>((size_t)images * heads * T);
    float* delta = bwd ? dalloc<float>((size_t)images * heads * T) : nullptr;
    auto ap = std::make_shared<AttnLongPlan>();
    char buf[256] = {0};
    int rc = attn_long_plan_make(ap.get(), qkv, o, d_o, gqkv, lse, delta, images, T, heads, W, scale, buf, sizeof buf);
    if (rc) throw EngineError(rc, std::string("attention plan: ") + buf);
    rec.path = PXR_ATTN_STREAMING;
    rec.lse = lse;
    rec.delta = delta;
    char lab[96];
    snprintf(lab, sizeof lab, "attn_long_fwd B=%d T=%d heads=%d", images, T, heads);
    fwd.add(1, [ap, cs] { attn_long_forward_launch(*ap, cs); }, ap->flops_fwd, lab, ap->bytes_fwd);
    if (bwd) {  // dQ (and D = dO . O), then dK / dV: two launches
      snprintf(lab, sizeof lab, "attn_long_bwd B=%d T=%d heads=%d", images, T, heads);
      bwd->add(2, [ap, cs] { attn_long_backward_launch(*ap, cs); }, ap->flops_bwd, lab, ap->bytes_bwd);
    }
    return nullptr;
  }
  // batched GEMMs over (head, image) around the row softmax; P and dP have a padded row pitch
  const int bn_s = multihead ? pick_bn(T, false, 1000) : 0, bn_d = multihead ? 64 : 0;  // T- / d-wide outputs
  const long long qs0 = d, qs1 = (long long)T * 3 * W;                          // (head, image) strides in qkv / gqkv
  const long long os0 = d, os1 = (long long)T * W;                              // ... in o / d_o
  const long long ps0 = (long long)T * ldT, ps1 = (long long)heads * T * ldT;   // ... in P / dP
  const int rows = images * heads * T;
  act_t* P = dalloc<act_t>((size_t)rows * ldT);
  rec.path = PXR_ATTN_CHAIN;
  rec.P = P;
  rec.ldT = ldT;
  int* gi = rec.gemm;  // the index the next add_gemm's record takes, for each GEMM of the chain in turn
  *gi++ = (int)gemm_log.size();
  {  // S = scale q k^T
    GemmEpilogue e;
    e.alpha = scale;
    e.out_f16 = P;
    e.ldc = ldT;
    e.bs0 = ps0;
    e.bs1 = ps1;
    add_gemm(fwd, opK(qkv, 3 * W, T, d, heads, qs0, images, qs1), opK(qkv + W, 3 * W, T, d, heads, qs0, images, qs1), T,
             T, d, e, bn_s);
  }
  if (causal) fwd.add(1, [=] { softmax_forward_causal(P, rows, T, ldT, cs); }, 0.0, "softmax_forward_causal");
  else fwd.add(1, [=] { softmax_forward(P, rows, T, ldT, cs); }, 0.0, "softmax_forward");
  *gi++ = (int)gemm_log.size();
  {  // O = P v
    GemmEpilogue e;
    e.out_f16 = o;
    e.ldc = W;
    e.bs0 = os0;
    e.bs1 = os1;
    add_gemm(fwd, opK(P, ldT, T, ldT, heads, ps0, images, ps1), opMN(qkv + 2 * W, 3 * W, d, T, heads, qs0, images, qs1),
             T, d, T, e, bn_d);
  }
  if (!bwd) return P;
  rec.dP_shared = dP != nullptr;
  if (!dP) dP = dalloc<act_t>((size_t)rows * ldT);
  rec.dP = dP;
  *gi++ = (int)gemm_log.size();
  {  // dP = dO v^T
    GemmEpilogue e;
    e.out_f16 = dP;
    e.ldc = ldT;
    e.bs0 = ps0;
    e.bs1 = ps1;
    add_gemm(*bwd, opK(d_o, W, T, d, heads, os0, images, os1), opK(qkv + 2 * W, 3 * W, T, d, heads, qs0, images, qs1), T,
             T, d, e, bn_s);
  }
  bwd->add(1, [=] { softmax_backward(P, dP, rows, T, ldT, cs); }, 0.0, "softmax_backward");  // dS, in place of dP
  *gi++ = (int)gemm_log.size();
  {  // dq = scale dS k
    GemmEpilogue e;
    e.alpha = scale;
    e.out_f16 = gqkv;
    e.ldc = 3 * W;
    e.bs0 = qs0;
    e.bs1 = qs1;
    add_gemm(*bwd, opK(dP, ldT, T, ldT, heads, ps0, images, ps1), opMN(qkv + W, 3 * W, d, T, heads, qs0, images, qs1), T,
             d, T, e, bn_d);
  }
  *gi++ = (int)gemm_log.size();
  {  // dk = scale dS^T q
    GemmEpilogue e;
    e.alpha = scale;
    e.out_f16 = gqkv + W;
    e.ldc = 3 * W;
    e.bs0 = qs0;
    e.bs1 = qs1;
    add_gemm(*bwd, opMN(dP, ldT, T, T, heads, ps0, images, ps1), opMN(qkv, 3 * W, d, T, heads, qs0, images, qs1), T, d,
             T, e, bn_d);
  }
  *gi++ = (int)gemm_log.size();
  {  // dv = P^T dO
    GemmEpilogue e;
    e.out_f16 = gqkv + 2 * W;
    e.ldc = 3 * W;
    e.bs0 = qs0;
    e.bs1 = qs1;
    add_gemm(*bwd, opMN(P, ldT, T, T, heads, ps0, images, ps1), opMN(d_o, W, d, T, heads, os0, images, os1), T, d, T, e,
             bn_d);
  }
  return P;
}

Act Engine::upsample(const Act& x, const std::string& prefix) {
  ConvW cw = load_conv(prefix + ".conv", x.C, x.C, 3);
  Act u = new_act(2 * x.H, 2 * x.W, x.C);
  cudaStream_t cs = st;
  drawer_fwd.add(1, [=] { upsample2x(x.p, x.H, x.W, x.C, u.p, cs); }, 0.0, "upsample2x");
  OpList b;
  Act out = conv_fwd_bwd(u, cw, b);
  b.add(1, [=] { downsum2x(u.g, x.H, x.W, x.C, x.g, cs); }, 0.0, "downsum2x");
  bwd_stack.push_back(std::move(b));
  return out;
}

void Engine::build_vqgan() {
  const int zc = cfg.z_channels, ne = cfg.n_embed, L = cfg.n_levels;
  if (L < 1 || L > 8) throw EngineError(-43, "n_levels must be in [1, 8]");
  const int f = 1 << (L - 1);
  if (cfg.image_h % f || cfg.image_w % f)
    throw EngineError(-44, "image size must be a multiple of 2^(n_levels-1)");
  const int h = cfg.image_h / f, w = cfg.image_w / f, hw = h * w;
  z_numel = (int64_t)zc * hw;
  // GN scratch sized for the largest activation
  // (the cooperative kernels use up to one block per SM, the three-kernel path two sets of gn_num_partials blocks)
  gn_part = dalloc<float>((size_t)std::max(2 * gn_num_partials(cfg.image_h * cfg.image_w, 64), num_sms + 1) * 64 + 64);
  gn_bar.counter = dalloc<unsigned long long>(1);
  splitk_ws_elems = (size_t)8 << 20;  // 32 MiB of fp32 partial sums: covers every conv the split-K rule selects
  splitk_ws = dalloc<float>(splitk_ws_elems, false);
  // codebook: taming VectorQuantizer's quantize.embedding or GumbelQuantize's quantize.embed.  Everything below reads it
  // the same way for both kinds: synth's nearest code and its backward, the z bounds, the optimiser (vqgan.py:149-153,
  // 190-195); only the encoder's quantiser differs (build_vqgan_encoder)
  const bool has_vq = weights[PXR_MOD_VQGAN].count("quantize.embedding.weight") > 0;
  vq_gumbel = weights[PXR_MOD_VQGAN].count("quantize.embed.weight") > 0;
  if (has_vq && vq_gumbel)
    throw EngineError(-41, "the VQGAN weights carry both quantize.embedding.weight and quantize.embed.weight");
  const HostWeight& cb = W(PXR_MOD_VQGAN, vq_gumbel ? "quantize.embed.weight" : "quantize.embedding.weight", {ne, zc});
  std::vector<float> cbT((size_t)zc * ne), c2(ne), mn(zc, 1e30f), mx(zc, -1e30f);
  for (int j = 0; j < ne; ++j) {
    float s = 0.f;
    for (int k = 0; k < zc; ++k) {
      float v = cb.data[(size_t)j * zc + k];
      cbT[(size_t)k * ne + j] = v;
      s += v * v;  // codebook.pow(2).sum(dim=1), vqgan.py:61
      mn[k] = std::min(mn[k], v);
      mx[k] = std::max(mx[k], v);
    }
    c2[j] = s;
  }
  float* d_cb = vq_cb = upload(cb.data);
  float* d_cbT = vq_cbT = upload(cbT);
  float* d_c2 = vq_c2 = upload(c2);
  zmin = upload(mn);  // vqgan.py:141-142
  zmax = upload(mx);
  const int n_chunks = (ne + 1023) / 1024;
  float* part_d = dalloc<float>((size_t)hw * n_chunks);
  int* part_i = dalloc<int>((size_t)hw * n_chunks);
  int* idx = dalloc<int>(hw);
  Act zq = new_act(h, w, zc);
  cudaStream_t cs = st;
  float* zb = z_buf = dalloc<float>(z_numel);
  z_grad = dalloc<float>(z_numel);
  bool vq_tc = vq_tc_supported(zc, ne);
  if (const char* e = getenv("PXR_VQ_TC")) vq_tc = vq_tc && atoi(e) != 0;
  if (vq_tc) {
    // distance matrix on the tensor cores, decision in exact fp32 (kernels_vq_tc.cu)
    float amax = 0.f, cmax2 = 0.f, cmax1 = 0.f;
    for (int j = 0; j < ne; ++j) {
      double s2 = 0.0, s1 = 0.0;
      for (int k = 0; k < zc; ++k) {
        const float v = std::fabs(cb.data[(size_t)j * zc + k]);
        amax = std::max(amax, v);
        s2 += (double)v * v;
        s1 += v;
      }
      cmax2 = std::max(cmax2, (float)std::sqrt(s2) * 1.000001f);
      cmax1 = std::max(cmax1, (float)s1 * 1.000001f);
    }
    int ex = 0;
    if (amax > 0.f) std::frexp(amax, &ex);
    const float cb_scale = std::ldexp(1.f, -ex);  // power of two: max |c| lands in [0.5, 1)
    std::vector<float> cbs(cb.data.size());
    for (size_t i = 0; i < cbs.size(); ++i) cbs[i] = cb.data[i] * cb_scale;
    act_t* cbh = upload_f16(cbs);
    act_t* zh = dalloc<act_t>((size_t)hw * zc);
    float* pinfo = dalloc<float>((size_t)hw * 4);
    float* scores = dalloc<float>((size_t)hw * ne, false);
    int* vq_stats = dalloc<int>(2);
    drawer_fwd.add(1, [=] { vq_prep(zb, zc, hw, zh, pinfo, cs); }, 0.0, "vq_prep");
    {
      GemmEpilogue e;
      e.out_f32 = scores;
      e.ldc = ne;
      add_gemm(drawer_fwd, opK(zh, zc, hw, zc), opK(cbh, zc, ne, zc), hw, ne, zc, e);
    }
    drawer_fwd.add(1, [=] { vq_select(scores, ne, zb, d_cb, d_c2, pinfo, cb_scale, cmax2, cmax1, zc, hw, ne, idx, zq.p, vq_stats, cs); },
                   0.0, "vq_select");
    reg("vq_stats", vq_stats, sizeof(int) * 2);  // {candidates rechecked in fp32, positions that fell back to the full search}, cumulative
  } else {
    drawer_fwd.add(2, [=] { vq_nearest(zb, d_cbT, d_c2, d_cb, zc, hw, ne, part_d, part_i, idx, zq.p, cs); }, 0.0, "vq_nearest");
  }
  reg("vq_idx", idx, sizeof(int) * hw);  // argmin code per latent position (vqgan.py:62): integer bookkeeping

  // post_quant_conv + decoder
  ConvW pq = load_conv("post_quant_conv", zc, zc, 1);
  OpList b_in;
  Act hq = conv_fwd_bwd(zq, pq, b_in);
  int block_in = cfg.ch * cfg.ch_mult[L - 1];
  ConvW cin = load_conv("decoder.conv_in", zc, block_in, 3);
  OpList b_in2;
  Act hcur = conv_fwd_bwd(hq, cin, b_in2);
  {
    OpList b;  // execution order: conv_in dgrad, then post_quant dgrad, then vq backward
    b.append(b_in2);
    b.append(b_in);
    float* zg = z_grad;
    float inv = 1.f / S;
    b.add(1, [=] { vq_backward(zq.g, inv, zc, hw, zg, cs); }, 0.0, "vq_backward");
    bwd_stack.push_back(std::move(b));
  }
  auto resblock = [&](const Act& x, const std::string& prefix, int cin, int cout) {
    const ResBlock r = resblock_fwd(drawer_fwd, x, prefix, cin, cout, true);
    resblock_bwd(r);
    return r.out;
  };
  auto attnblock = [&](const Act& x, const std::string& prefix, int c) {
    const AttnBlock a = attnblock_fwd(drawer_fwd, x, prefix, c, true);
    attnblock_bwd(a);
    return a.out;
  };
  hcur = resblock(hcur, "decoder.mid.block_1", block_in, block_in);
  hcur = attnblock(hcur, "decoder.mid.attn_1", block_in);
  hcur = resblock(hcur, "decoder.mid.block_2", block_in, block_in);
  int curr_res = cfg.resolution / f;
  for (int lv = L - 1; lv >= 0; --lv) {
    int block_out = cfg.ch * cfg.ch_mult[lv];
    for (int ib = 0; ib < cfg.num_res_blocks + 1; ++ib) {
      std::string p = "decoder.up." + std::to_string(lv) + ".block." + std::to_string(ib);
      hcur = resblock(hcur, p, block_in, block_out);
      block_in = block_out;
      if (curr_res == cfg.attn_resolution)
        hcur = attnblock(hcur, "decoder.up." + std::to_string(lv) + ".attn." + std::to_string(ib), block_in);
    }
    if (lv != 0) {
      hcur = upsample(hcur, "decoder.up." + std::to_string(lv) + ".upsample");
      curr_res *= 2;
    }
  }
  // norm_out, swish, conv_out -> image
  NormW no = load_norm(PXR_MOD_VQGAN, "decoder.norm_out", block_in);
  ConvW co = load_conv("decoder.conv_out", block_in, 3, 3);
  Act a = new_act(hcur.H, hcur.W, block_in);
  GNSaved s = add_gn(drawer_fwd, hcur, no, 1, a.p);
  const int px = hcur.pixels();
  float* co_out = dalloc<float>((size_t)px * co.cout_pad);
  act_t* co_g = dalloc<act_t>((size_t)px * co.cout_k);
  {
    GemmEpilogue e;
    e.bias = co.bias;
    e.out_f32 = co_out;
    e.ldc = co.cout_pad;
    add_conv(drawer_fwd, a.p, hcur.H, hcur.W, block_in, co.w, co.cout_pad, 3, 3, e);
  }
  img = dalloc<float>((size_t)3 * px);
  img_pre = dalloc<float>((size_t)3 * px);
  g_img = dalloc<float>((size_t)3 * px);
  {
    float *ip = img_pre, *im = img;
    int ld = co.cout_pad;
    drawer_fwd.add(1, [=] { image_finish(co_out, ld, px, ip, im, cs); }, 0.0, "image_finish");
  }
  {
    OpList b;
    float *gi = g_img, *ip = img_pre;
    int ldk = co.cout_k;
    float* part = gn_part;
    b.add(1, [=] { image_finish_backward(gi, ip, px, ldk, co_g, cs); }, 0.0, "image_finish_backward");
    GemmEpilogue e;
    e.out_f16 = a.g;
    e.ldc = block_in;
    add_conv(b, co_g, hcur.H, hcur.W, co.cout_k, co.wd, co.cin_rows, block_in, 3, e);
    Act hc = hcur;
    add_gn_bwd(b, a.g, hc.p, s, no, px, hc.C, 1, nullptr, hc.g);
    bwd_stack.push_back(std::move(b));
  }
  // flatten backward stack in reverse block order
  for (int i = (int)bwd_stack.size() - 1; i >= 0; --i) drawer_bwd.append(bwd_stack[i]);
  bwd_stack.clear();
  if (weights[PXR_MOD_VQGAN].count("encoder.conv_in.weight")) build_vqgan_encoder();
}

// taming Encoder (un-vendored: taming/modules/diffusionmodules/model.py, restated in oracle/ref_path.py): conv_in, per level
// num_res_blocks x ResnetBlock (+ AttnBlock at attn_resolution) and a strided Downsample, mid block_1 / attn_1 / block_2,
// norm_out + swish + conv_out; then VQModel.encode's quant_conv and the quantiser's nearest code.  The blocks are the
// decoder's forward builders; no backward and no gradient buffers (the encoder only runs at init / overlay time, never
// inside the gradient path).
void Engine::build_vqgan_encoder() {
  const int zc = cfg.z_channels, ne = cfg.n_embed, L = cfg.n_levels, H = cfg.image_h, Wd = cfg.image_w;
  cudaStream_t cs = st;
  auto act = [&](int h, int w, int c) { return new_act(h, w, c, false); };
  auto conv = [&](const Act& x, const ConvW& w) {
    Act y = act(x.H, x.W, w.cout);
    GemmEpilogue e;
    e.bias = w.bias;
    e.out_f16 = y.p;
    e.ldc = y.C;
    add_conv(enc_fwd, x.p, x.H, x.W, x.C, w.w, w.cout_pad, w.cout, w.ks, e);
    return y;
  };
  auto resblock = [&](const Act& x, const std::string& prefix, int cin, int cout) {
    return resblock_fwd(enc_fwd, x, prefix, cin, cout, false).out;
  };
  auto attnblock = [&](const Act& x, const std::string& prefix, int c) {
    return attnblock_fwd(enc_fwd, x, prefix, c, false).out;
  };
  enc_img = dalloc<float>((size_t)3 * H * Wd);
  Act x0 = act(H, Wd, 64);
  {
    float* im = enc_img;
    const int px = H * Wd;
    enc_fwd.add(1, [=] { image_to_nhwc64(im, px, x0.p, cs); }, 0.0, "image_to_nhwc64");
  }
  ConvW cin_w = load_conv("encoder.conv_in", 64, cfg.ch, 3, 3);
  Act hcur = conv(x0, cin_w);
  int curr_res = cfg.resolution, block_in = cfg.ch;
  for (int lv = 0; lv < L; ++lv) {
    const int block_out = cfg.ch * cfg.ch_mult[lv];
    for (int ib = 0; ib < cfg.num_res_blocks; ++ib) {
      const std::string p = "encoder.down." + std::to_string(lv) + ".block." + std::to_string(ib);
      hcur = resblock(hcur, p, block_in, block_out);
      block_in = block_out;
      if (curr_res == cfg.attn_resolution)
        hcur = attnblock(hcur, "encoder.down." + std::to_string(lv) + ".attn." + std::to_string(ib), block_in);
    }
    if (lv != L - 1) {
      ConvW dw = load_conv("encoder.down." + std::to_string(lv) + ".downsample.conv", block_in, block_in, 3);
      Act full = conv(hcur, dw);
      Act half = act(hcur.H / 2, hcur.W / 2, block_in);
      const int fh = hcur.H, fw = hcur.W, fc = block_in;
      enc_fwd.add(1, [=] { subsample_odd(full.p, fh, fw, fc, half.p, cs); }, 0.0, "subsample_odd");
      hcur = half;
      curr_res /= 2;
    }
  }
  hcur = resblock(hcur, "encoder.mid.block_1", block_in, block_in);
  hcur = attnblock(hcur, "encoder.mid.attn_1", block_in);
  hcur = resblock(hcur, "encoder.mid.block_2", block_in, block_in);
  NormW no = load_norm(PXR_MOD_VQGAN, "encoder.norm_out", block_in);
  Act a = act(hcur.H, hcur.W, block_in);
  add_gn(enc_fwd, hcur, no, 1, a.p);
  ConvW co = load_conv("encoder.conv_out", block_in, zc, 3);  // double_z = False for the VQ models
  Act hz = conv(a, co);
  ConvW qc = load_conv("quant_conv", zc, zc, 1);
  Act hq = conv(hz, qc);
  const int hw = hq.pixels();
  if ((int64_t)zc * hw != z_numel) throw EngineError(-44, "encoder output does not match the latent size");
  float *d_cb = vq_cb, *d_cbT = vq_cbT, *d_c2 = vq_c2;
  int* idx = nullptr;
  float *z32 = nullptr, *ez = nullptr;
  if (vq_gumbel) {
    // GumbelQuantize, eval mode: logits = quantize.proj(h), a 1x1 convolution to n_embed channels, in fp32 from the conv
    // plan; then per position the arg-max of logits + noise selects the code row.  The reference's value,
    // (y_hard - y_soft + y_soft) @ embed.weight, is that row to within one fp32 rounding; this writes the row exactly.
    ConvW pw = load_conv("quantize.proj", zc, ne, 1);
    const int ld = pw.cout_pad;
    float* logits = dalloc<float>((size_t)hw * ld);
    GemmEpilogue e;
    e.bias = pw.bias;
    e.out_f32 = logits;
    e.ldc = ld;
    add_conv(enc_fwd, hq.p, hq.H, hq.W, hq.C, pw.w, pw.cout_pad, pw.cout, 1, e);
    float* noise = enc_noise = dalloc<float>((size_t)ne * hw);
    idx = dalloc<int>(hw);
    z32 = dalloc<float>((size_t)zc * hw);
    ez = enc_z = dalloc<float>((size_t)zc * hw);
    enc_fwd.add(2, [=] {
      vq_backward(hq.p, 1.f, zc, hw, z32, cs);  // enc_h, as below
      gumbel_select(logits, ld, noise, d_cb, zc, hw, ne, idx, ez, cs);
    }, 0.0, "encoder gumbel quantise");
  } else {
    // quantise: the same exact fp32 nearest-code search as synth, on the decoder's codebook copies
    const int n_chunks = (ne + 1023) / 1024;
    float* part_d = dalloc<float>((size_t)hw * n_chunks);
    int* part_i = dalloc<int>((size_t)hw * n_chunks);
    idx = dalloc<int>(hw);
    z32 = dalloc<float>((size_t)zc * hw);
    act_t* zq16 = dalloc<act_t>((size_t)hw * zc);
    ez = enc_z = dalloc<float>((size_t)zc * hw);
    enc_fwd.add(4, [=] {
      vq_backward(hq.p, 1.f, zc, hw, z32, cs);  // NHWC fp16 -> [C, hw] fp32 (the same transpose kernel the decoder's backward ends with)
      vq_nearest(z32, d_cbT, d_c2, d_cb, zc, hw, ne, part_d, part_i, idx, zq16, cs);
      gather_codes(d_cb, idx, zc, hw, ez, cs);
    }, 0.0, "encoder quantise");
  }
  reg("enc_idx", idx, sizeof(int) * hw);
  reg("enc_h", z32, sizeof(float) * zc * hw);
  have_encoder = true;
}

void Engine::build_pixel() {
  const int rows = cfg.grid_rows, cols = cfg.grid_cols, H = cfg.image_h, Wd = cfg.image_w;
  if (rows < 1 || cols < 1) throw EngineError(-46, "pixel drawer needs grid_rows / grid_cols");
  z_numel = (int64_t)3 * rows * cols;
  z_buf = dalloc<float>(z_numel);
  z_grad = dalloc<float>(z_numel);
  img = dalloc<float>((size_t)3 * H * Wd);
  img_pre = dalloc<float>((size_t)3 * H * Wd);
  g_img = dalloc<float>((size_t)3 * H * Wd);
  cudaStream_t cs = st;
  float *zb = z_buf, *ip = img_pre, *im = img, *gi = g_img, *zg = z_grad;
  float inv = 1.f / S;
  drawer_fwd.add(1, [=] { pixel_synth(zb, rows, cols, H, Wd, ip, im, cs); }, 0.0, "pixel_synth");
  drawer_bwd.add(1, [=] { pixel_synth_backward(gi, ip, rows, cols, H, Wd, inv, zg, cs); }, 0.0, "pixel_synth_backward");
}

// PixelDrawer with shaped cells (pixeldrawer.py:200-304, 330-367): fixed polygons from pxr_set_polygons, z = [n, 4] RGBA
// fill colours.  The tile grid is built here once, on the host (kernels.cuh RasterScene).
void Engine::build_polygon() {
  const int n = (int)poly_off.size() - 1, H = cfg.image_h, Wd = cfg.image_w;
  if (n < 1) throw EngineError(-75, "polygon drawer: call pxr_set_polygons before pxr_finalize");
  z_numel = (int64_t)4 * n;
  z_buf = dalloc<float>(z_numel);
  z_grad = dalloc<float>(z_numel);
  img = dalloc<float>((size_t)3 * H * Wd);
  img_pre = img;  // no clamp in the render (pixeldrawer.py:342-355): the image is its own pre-activation
  g_img = dalloc<float>((size_t)3 * H * Wd);
  poly_winner = dalloc<int>((size_t)4 * H * Wd);
  const int T = RASTER_TILE, tx = (Wd + T - 1) / T, ty = (H + T - 1) / T;
  std::vector<float4> bbox(n);
  std::vector<int> tx0(n), tx1(n), ty0(n), ty1(n), count((size_t)tx * ty + 1, 0);
  for (int k = 0; k < n; ++k) {
    float4 b = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
    for (int i = poly_off[k]; i < poly_off[k + 1]; ++i) {
      const float x = poly_xy[2 * i], y = poly_xy[2 * i + 1];
      b.x = std::min(b.x, x);
      b.y = std::min(b.y, y);
      b.z = std::max(b.z, x);
      b.w = std::max(b.w, y);
    }
    bbox[k] = b;
    // tile j covers the closed interval [j T, (j + 1) T]: it meets [lo, hi] for ceil(lo / T) - 1 <= j <= floor(hi / T).
    // The box is clamped to one tile around the canvas first, so far-away (finite) coordinates convert to int safely;
    // a polygon entirely off the canvas gets an empty tile range.
    auto tile_lo = [T](double v, int n) { return (int)std::ceil(std::min(std::max(v, -(double)T), (double)n * T + T) / T) - 1; };
    auto tile_hi = [T](double v, int n) { return (int)std::floor(std::min(std::max(v, -(double)T), (double)n * T + T) / T); };
    tx0[k] = std::max(0, tile_lo(b.x, tx));
    tx1[k] = std::min(tx - 1, tile_hi(b.z, tx));
    ty0[k] = std::max(0, tile_lo(b.y, ty));
    ty1[k] = std::min(ty - 1, tile_hi(b.w, ty));
    for (int j = ty0[k]; j <= ty1[k]; ++j)
      for (int i = tx0[k]; i <= tx1[k]; ++i) ++count[(size_t)j * tx + i + 1];
  }
  for (size_t t = 1; t < count.size(); ++t) count[t] += count[t - 1];
  std::vector<int> fill(count.begin(), count.end() - 1), list(count.back() > 0 ? count.back() : 1, 0);
  for (int k = n - 1; k >= 0; --k)  // topmost first: shapes are drawn in index order, later over earlier
    for (int j = ty0[k]; j <= ty1[k]; ++j)
      for (int i = tx0[k]; i <= tx1[k]; ++i) list[fill[(size_t)j * tx + i]++] = k;
  std::vector<float2> xy(poly_xy.size() / 2);
  for (size_t i = 0; i < xy.size(); ++i) xy[i] = make_float2(poly_xy[2 * i], poly_xy[2 * i + 1]);
  scene.xy = upload(xy);
  scene.off = upload(poly_off);
  scene.bbox = upload(bbox);
  scene.tile_start = upload(count);
  scene.tile_list = upload(list);
  scene.n = n;
  scene.tiles_x = tx;
  cudaStream_t cs = st;
  float *zb = z_buf, *im = img, *gi = g_img, *zg = z_grad;
  int* win = poly_winner;
  const RasterScene sc = scene;
  const uint64_t seed = cfg.seed;
  const float inv = 1.f / S;
  const int* iter = &synth_iter;  // read when the op runs: pxr_iterate's iteration, or pxr_set_synth_iteration's
  drawer_fwd.add(1, [=] { raster_forward(sc, zb, H, Wd, seed, *iter, win, im, cs); }, 0.0, "raster_forward");
  drawer_bwd.add(1, [=] { raster_backward(sc, win, gi, H, Wd, inv, zg, cs); }, 0.0, "raster_backward");
}

// LineDrawer (linedrawer.py:44-166): z = [points | widths | paper RGBA]; the capsules are flattened and binned afresh on
// every render because the geometry is what the optimiser moves.  The three Adams of get_opts (linedrawer.py:128-136)
// become one fused Adam with rates x1 / x0.1 / x0.01 over the three ranges; the paper range has rate 0 unless it is
// trainable.  clip_z clamps the widths to [1, max_width].
void Engine::build_strokes() {
  const int N = stroke_paths, L = stroke_segments, H = cfg.image_h, Wd = cfg.image_w;
  if (N < 1) throw EngineError(-78, "line drawer: call pxr_set_strokes before pxr_finalize");
  const int n_pts = N * (3 * L + 1) * 2;
  z_numel = (int64_t)n_pts + N + 4;
  z_buf = dalloc<float>(z_numel);
  z_grad = dalloc<float>(z_numel);
  img = dalloc<float>((size_t)3 * H * Wd);
  img_pre = img;  // synth has no clamp (linedrawer.py:156-166)
  g_img = dalloc<float>((size_t)3 * H * Wd);
  StrokeScene& s = sscene;
  s.n_paths = N;
  s.n_segments = L;
  s.n_caps = N * L * STROKE_CHORDS;
  s.W = Wd;
  s.H = H;
  s.tiles_x = (Wd + RASTER_TILE - 1) / RASTER_TILE;
  s.tiles_y = (H + RASTER_TILE - 1) / RASTER_TILE;
  s.width_offset = n_pts;
  s.paper_trainable = stroke_paper;
  const size_t tiles = (size_t)s.tiles_x * s.tiles_y;
  s.caps = dalloc<float4>(s.n_caps);
  s.cap_tiles = dalloc<int4>(s.n_caps);
  s.tile_start = dalloc<int>(tiles + 1);
  s.tile_list = dalloc<int>((size_t)s.n_caps * tiles);  // every capsule in every tile: the geometry is unbounded
  s.winner = dalloc<int>((size_t)4 * H * Wd);
  s.pix_g = dalloc<float>((size_t)H * Wd);
  s.paper_part = dalloc<float>((size_t)stroke_paper_blocks(H, Wd) * 4);
  s.cap_grad = dalloc<float>((size_t)s.n_caps * 5);
  zr.end0 = n_pts;
  zr.end1 = n_pts + N;
  zr.scale[0] = 1.f;
  zr.scale[1] = 0.1f;
  zr.scale[2] = stroke_paper ? 0.01f : 0.f;
  zr.lo1 = 1.f;
  zr.hi1 = stroke_max_width;
  cudaStream_t cs = st;
  float *zb = z_buf, *im = img, *gi = g_img, *zg = z_grad;
  const StrokeScene sc = s;
  const uint64_t seed = cfg.seed;
  const float inv = 1.f / S;
  const int* iter = &synth_iter;
  drawer_fwd.add(1, [=] { stroke_flatten(sc, zb, cs); }, 0.0, "stroke_flatten");
  drawer_fwd.add(3, [=] { stroke_bin(sc, cs); }, 0.0, "stroke_bin");
  drawer_fwd.add(1, [=] { stroke_raster_forward(sc, zb, seed, *iter, im, cs); }, 0.0, "stroke_raster_fwd");
  drawer_bwd.add(3, [=] { stroke_raster_backward(sc, zb, gi, inv, zg, cs); }, 0.0, "stroke_raster_bwd");
}

// FftDrawer.synth (fftdrawer.py:78-84): params = rfft2 spectrum [1,3,H,W/2+1,2]; see kernels_fft.cu
void Engine::build_fft() {
  const int H = cfg.image_h, Wd = cfg.image_w, W2 = Wd / 2 + 1;
  if (Wd % 2) throw EngineError(-48, "fft drawer needs an even canvas width");
  const float decay = cfg.fft_decay > 0 ? cfg.fft_decay : 1.5f, colors = cfg.fft_colors > 0 ? cfg.fft_colors : 1.5f;
  const float contrast = cfg.fft_contrast > 0 ? cfg.fft_contrast : 0.9f;
  const char* msg = nullptr;
  fft = fft_plans_create(H, Wd, st, &msg);
  if (!fft) throw EngineError(-49, msg ? msg : "cuFFT unavailable");
  z_numel = (int64_t)3 * H * W2 * 2;
  // aphantasia fft_image: scale = 1 / max(|f|, 4 / max(h, w)) ** decay * sqrt(w * h) on the rfft2 frequency grid
  std::vector<float> sc((size_t)H * W2);
  for (int y = 0; y < H; ++y) {
    const double fy = (y < (H + 1) / 2 ? y : y - H) / (double)H;  // np.fft.fftfreq
    for (int x = 0; x < W2; ++x) {
      const double fx = (x < (Wd + 1) / 2 ? x : x - Wd) / (double)Wd;
      const double f = std::sqrt(fx * fx + fy * fy);
      sc[(size_t)y * W2 + x] = (float)(1.0 / std::pow(std::max(f, 4.0 / std::max(H, Wd)), (double)decay) * std::sqrt((double)Wd * H));
    }
  }
  // to_valid_rgb: colour-correlation matrix, first column / colors, normalised by the largest column norm
  const double base[3][3] = {{0.26, 0.09, 0.02}, {0.27, 0.00, -0.05}, {0.27, -0.09, 0.03}};
  double m[3][3], maxn = 0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m[r][c] = base[r][c] / (c == 0 ? colors : 1.0);
  for (int c = 0; c < 3; ++c) maxn = std::max(maxn, std::sqrt(m[0][c] * m[0][c] + m[1][c] * m[1][c] + m[2][c] * m[2][c]));
  std::vector<float> M(9);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) M[r * 3 + c] = (float)(m[r][c] / maxn);
  float* d_scale = upload(sc);
  float* d_M = upload(M);
  const size_t px = (size_t)H * Wd;
  z_buf = dalloc<float>(z_numel);
  z_grad = dalloc<float>(z_numel);
  img = dalloc<float>(3 * px);
  img_pre = dalloc<float>(3 * px);  // irfft output x (unnormalised)
  g_img = dalloc<float>(3 * px);
  float* scaled = dalloc<float>(z_numel);
  float* g1 = dalloc<float>(3 * px);
  float* G = dalloc<float>(z_numel);
  double* part = dalloc<double>(2 * 296 + 8);
  float* stats = dalloc<float>(4);
  cudaStream_t cs = st;
  FftPlans* pl = fft;
  float *zb = z_buf, *x = img_pre, *im = img, *gi = g_img, *zg = z_grad;
  const float inv = 1.f / S;
  drawer_fwd.add(5, [=] { fft_synth_forward(pl, zb, d_scale, d_M, contrast, scaled, x, part, stats, im, cs); }, 0.0, "fft_synth_forward");
  drawer_bwd.add(4, [=] { fft_synth_backward(pl, gi, im, x, d_scale, d_M, contrast, stats, g1, G, part, inv, zg, cs); }, 0.0, "fft_synth_backward");
}

// ===================================================================================================== cutouts
void Engine::build_cutouts() {
  if (cfg.n_clip < 1 || cfg.n_clip > 4) throw EngineError(-53, "n_clip must be 1, 2, 3 or 4");
  sets.clear();
  for (int i = 0; i < cfg.n_clip; ++i) {
    const int res = i == 0 ? cfg.cut_size : cfg.clip[i].image_res;
    int s = 0;
    while (s < n_sets() && sets[s].cs != res) ++s;
    if (s == n_sets()) {
      if (res < 4 || res % 4) throw EngineError(-6, "perceptor " + std::to_string(i) + ": image_res must be a multiple of 4");
      sets.emplace_back();
      sets.back().cs = res;
    }
    set_of[i] = s;
  }
  aspect = (cfg.cut_aspect > 0.f && cfg.cut_aspect != 1.f) ? (double)cfg.cut_aspect : 1.0;
  if (aspect > 8.0 || aspect < 0.125) throw EngineError(-66, "cut_aspect (canvas width / height) must be within [1/8, 8]");
  size_t fx_n = 0;
  for (int s = 0; s < n_sets(); ++s) {
    CutSet& K = sets[s];
    const int cs_ = K.cs;
    K.pooled = dalloc<float>((size_t)3 * cs_ * cs_);
    K.g_pooled = dalloc<float>((size_t)3 * cs_ * cs_);
    source_size(cs_, aspect, K.src_h, K.src_w);
    if (s == 0 && aspect != 1.0 && cfg.cut_src_h > 0 && cfg.cut_src_w > 0) {  // the caller's (double-precision) truncation wins
      if (std::abs(cfg.cut_src_h - K.src_h) > 1 || std::abs(cfg.cut_src_w - K.src_w) > 1)
        throw EngineError(-66, "cut_src_h / cut_src_w do not match cut_aspect");
      K.src_h = cfg.cut_src_h;
      K.src_w = cfg.cut_src_w;
    }
    if (aspect != 1.0) {
      K.cut_src = dalloc<float>((size_t)3 * K.src_h * K.src_w);
      K.g_cut_src = dalloc<float>((size_t)3 * K.src_h * K.src_w);
    } else {
      K.cut_src = K.pooled;
      K.g_cut_src = K.g_pooled;
    }
    fx_n = std::max(fx_n, (size_t)3 * std::max(K.src_h * K.src_w, cs_ * cs_));
    K.pool_argmax = dalloc<int>((size_t)3 * cs_ * cs_);
    K.batch = dalloc<float>((size_t)n_local * 3 * cs_ * cs_);
    K.g_batch = dalloc<float>((size_t)n_local * 3 * cs_ * cs_);
    K.n_parts = cutout_num_blocks(n_local, cs_);
    K.part_min = dalloc<float>(K.n_parts);
    K.part_max = dalloc<float>(K.n_parts);
    K.part_imin = dalloc<int>(K.n_parts);
    K.part_imax = dalloc<int>(K.n_parts);
    K.range = dalloc<float>(4);
    K.irange = dalloc<int>(4);
    K.sums = dalloc<float>(4);
    K.minv_dev = dalloc<float>((size_t)n_local * 12);  // 9 homography + 3 ColorJitter floats per cutout, one H2D copy
    K.facs_dev = dalloc<float>(n_local);
    for (int i = 0; i < RING; ++i) {
      PXR_CUDA(cudaMallocHost((void**)&K.minv_host[i], sizeof(float) * n_local * 12));
      PXR_CUDA(cudaMallocHost((void**)&K.facs_host[i], sizeof(float) * n_local));
      PXR_CUDA(cudaEventCreateWithFlags(&K.ring_ev[i], cudaEventDisableTiming));
    }
    CutoutArgs& ca = K.cut_args;
    memset(&ca, 0, sizeof ca);
    ca.pooled = K.cut_src;
    ca.src_h = K.src_h;
    ca.src_w = K.src_w;
    ca.minv = K.minv_dev;
    ca.cs = cs_;
    ca.n_local = n_local;
    ca.first_global = first_global;
    ca.cutn_zoom = (int)(0.6 * cfg.cutn);  // pixray.py:407
    ca.seed = cfg.seed;
    ca.noise_fac = cfg.noise_fac;
    ca.rng_stream = cut_rng_stream(s);
    K.aux_A = dalloc<float>(((size_t)n_local * cs_ + 2) * cs_);
    K.aux_halo = dalloc<float>((size_t)12 * cs_);
    K.aux_xbuf = dalloc<float>((size_t)12 * cs_ * cfg.world);
    K.aux_best = dalloc<int>((size_t)n_local * cs_ * cs_);
  }
  pooled_masked = dalloc<float>((size_t)3 * cfg.cut_size * cfg.cut_size);
  grad_fx = dalloc<long long>(fx_n);  // zeroed; each use clears it again
  sums_fx = dalloc<long long>(2);  // zero-initialised; every pass leaves it zeroed again
  fx_poison = dalloc<unsigned int>(2);
  xbuf = dalloc<float>(4);
}

// Host side of MakeCutouts: invert the cached "dst <- src" transforms (pixray.py:498) to the sampling maps the
// kernel uses (kornia warp_perspective inverts the normalised homography; with align_corners=True the
// normalisations cancel and src_pix = M^-1 dst_pix), stage them through pinned memory.
void Engine::prepare_cut_params(int s, const pxr_cut_params* p, int iter) {
  CutSet& K = sets[s];
  CutoutArgs& cut_args = K.cut_args;
  // engine-drawn parameters are keyed by (seed, rng_iter): pass b > 0 of an iteration (batches > 1) draws a fresh set,
  // like a second ascend_txt call does, while the padding mode still follows the iteration's parity (pixray.py:1250)
  const int key = rng_iter ? rng_iter : iter;
  const int slot = K.ring_pos;
  K.ring_pos = (K.ring_pos + 1) % RING;
  PXR_CUDA(cudaEventSynchronize(K.ring_ev[slot]));
  std::vector<float> gen;
  const float* T = p ? p->transforms : nullptr;
  int zoom_padding = p ? p->zoom_padding : ((iter % 2 == 0) ? PXR_PAD_REFLECTION : PXR_PAD_BORDER);  // pixray.py:1250
  float fill = p ? p->fill : 0.f;
  if (!T) {  // engine RNG (SURVEY.md Appendix A), keyed by (seed, iter, global cutout index) and the set's streams
    gen.resize((size_t)cfg.cutn * 9);
    sample_cutout_transforms(cfg.seed, key, cfg.cutn, K.cs, gen.data(), aspect, K.src_h, K.src_w, cut_args.rng_stream);
    T = gen.data();
    if (!p) fill = sample_fill(cfg.seed, key);  // shared by every set (pixray.py:1255-1258)
  }
  for (int n = 0; n < n_local; ++n) {
    double m[9], inv[9];
    for (int i = 0; i < 9; ++i) m[i] = T[(size_t)(first_global + n) * 9 + i];
    if (!invert3x3(m, inv)) throw EngineError(-60, "singular cutout transform");
    for (int i = 0; i < 9; ++i) K.minv_host[slot][n * 9 + i] = (float)inv[i];
  }
  // ColorJitter rows: explicit, or drawn like the transforms when those are the engine's own
  const float* J = p ? p->color_jitter : nullptr;
  std::vector<float> genj;
  if (!J && !(p && p->transforms) && cj_p > 0.f) {
    genj.resize((size_t)cfg.cutn * 3);
    sample_color_jitter(cfg.seed, key, cfg.cutn, cj_p, cj_sat, cj_hue, genj.data(), cut_args.rng_stream);
    J = genj.data();
  }
  float* jh = K.minv_host[slot] + (size_t)n_local * 9;
  if (J)
    for (int i = 0; i < n_local * 3; ++i) jh[i] = J[(size_t)first_global * 3 + i];
  cut_args.jitter = J ? K.minv_dev + (size_t)n_local * 9 : nullptr;
  PXR_CUDA(cudaMemcpyAsync(K.minv_dev, K.minv_host[slot], sizeof(float) * n_local * (J ? 12 : 9), cudaMemcpyHostToDevice, st));
  cut_args.zoom_padding = zoom_padding;
  cut_args.fill = fill;
  cut_args.iter = key;
  cut_args.noise = nullptr;
  cut_args.noise_facs = nullptr;
  if (cfg.noise_fac <= 0.f) {
    cut_args.noise_mode = 0;
  } else if (p && p->noise && p->noise_facs) {
    for (int n = 0; n < n_local; ++n) K.facs_host[slot][n] = p->noise_facs[first_global + n];
    PXR_CUDA(cudaMemcpyAsync(K.facs_dev, K.facs_host[slot], sizeof(float) * n_local, cudaMemcpyHostToDevice, st));
    cut_args.noise_mode = 1;
    cut_args.noise = p->noise + (size_t)first_global * 3 * K.cs * K.cs;
    cut_args.noise_facs = K.facs_dev;
  } else if (p && (p->noise || p->noise_facs)) {
    throw EngineError(-61, "pxr_cut_params: noise and noise_facs must be given together");
  } else if (p && p->transforms) {
    cut_args.noise_mode = 0;  // explicit transforms without noise: deterministic replay
  } else {
    cut_args.noise_mode = 2;
  }
  PXR_CUDA(cudaEventRecord(K.ring_ev[slot], st));
}

void Engine::forward_cutouts(int s) {
  CutSet& K = sets[s];
  ProfRec prof_rec;
  if (profiling) prof_begin_stage(prof_rec, "cutouts_fwd set " + std::to_string(s));
  // the cutout / embedding losses accumulate per-rank partial sums into their slots: set 0 clears every auxiliary slot
  // (one set: the launch as before), another set its own cutout-space entries
  if (s == 0 && !aux.empty()) {
    PXR_CUDA(cudaMemsetAsync(losses_dev + aux_base(), 0, sizeof(float) * (num_losses() - aux_base()), st));
  } else if (s > 0) {
    for (size_t k = 0; k < aux.size(); ++k)
      if (aux_per_set(aux[k].kind)) PXR_CUDA(cudaMemsetAsync(losses_dev + aux_slot(k, s), 0, sizeof(float), st));
  }
  pool_forward(cur_cut_img(), cur_cut_h(), cur_cut_w(), K.cs, K.pooled, K.pool_argmax, st);
  if (aspect != 1.0) {
    rescale_bilinear(K.pooled, K.cs, K.cs, K.src_h, K.src_w, K.cut_src, st);
    launches += 1;
  }
  cutout_forward(K.cut_args, K.batch, K.part_min, K.part_max, K.part_imin, K.part_imax, st);
  minmax_reduce(nullptr, K.part_min, K.part_max, K.part_imin, K.part_imax, K.n_parts, K.range, K.irange, st);
  launches += 3;
  if (comm) {  // global min / max over all ranks' cutouts of the set (slip.py:21-36 reduces over the whole batch)
    range_pack(K.range, xbuf, st);
    nccl_check(Comm::api().all_reduce(xbuf, xbuf, 2, Comm::kFloat32, Comm::kMin, comm, st), "allreduce(min,max)");
    range_unpack(xbuf, K.range, K.irange, st);
    launches += 3;
  }
  K.cut = true;
  if (profiling) prof_end_stage(prof_rec);
  check_launch("cutouts forward");
}

// ===================================================================================================== CLIP ViT
// The same tensors under two naming schemes: openai-CLIP's (the CLIP image tower under visual.transformer.resblocks.N,
// every text tower under transformer.resblocks.N) and timm's (SLIP's image tower): in_proj = attn.qkv (q | k | v, heads
// contiguous), out_proj = attn.proj, c_fc / c_proj = mlp.fc1 / mlp.fc2, ln_1 / ln_2 = norm1 / norm2.
Engine::BlockW Engine::load_block(int mod, const std::string& p, int Wd, bool timm) {
  static const char* const keys[2][10] = {
      {".attn.in_proj_weight", ".attn.in_proj_bias", ".attn.out_proj.weight", ".attn.out_proj.bias", ".mlp.c_fc.weight",
       ".mlp.c_fc.bias", ".mlp.c_proj.weight", ".mlp.c_proj.bias", ".ln_1", ".ln_2"},
      {".attn.qkv.weight", ".attn.qkv.bias", ".attn.proj.weight", ".attn.proj.bias", ".mlp.fc1.weight", ".mlp.fc1.bias",
       ".mlp.fc2.weight", ".mlp.fc2.bias", ".norm1", ".norm2"}};
  const char* const* k = keys[timm];
  BlockW b;
  b.wqkv = upload_f16(W(mod, p + k[0], {3 * Wd, Wd}).data);
  b.bqkv = upload(W(mod, p + k[1], {3 * Wd}).data);
  b.wo = upload_f16(W(mod, p + k[2], {Wd, Wd}).data);
  b.bo = upload(W(mod, p + k[3], {Wd}).data);
  b.wfc = upload_f16(W(mod, p + k[4], {4 * Wd, Wd}).data);
  b.bfc = upload(W(mod, p + k[5], {4 * Wd}).data);
  b.wproj = upload_f16(W(mod, p + k[6], {Wd, 4 * Wd}).data);
  b.bproj = upload(W(mod, p + k[7], {Wd}).data);
  b.ln1 = load_norm(mod, p + k[8], Wd);
  b.ln2 = load_norm(mod, p + k[9], Wd);
  return b;
}

Op Engine::stream_ln_fwd(const void* x, long long ld, const NormW& n, int rows, int Wd, float eps, act_t* y16,
                         float* stats) const {
  cudaStream_t cs = st;
  if (stream16) {
    const act_t* x16 = static_cast<const act_t*>(x);
    return [=] { layernorm_forward(x16, ld, nullptr, 1, n.gamma, n.beta, rows, Wd, eps, y16, nullptr, stats, cs); };
  }
  const float* x32 = static_cast<const float*>(x);
  return [=] { layernorm_forward(x32, ld, nullptr, 1, n.gamma, n.beta, rows, Wd, eps, y16, nullptr, stats, cs); };
}

Op Engine::stream_ln_bwd(const act_t* dy, const void* x, long long ld, const float* stats, const NormW& n, int rows,
                         int Wd, int accumulate, float* gx, act_t* gx16) const {
  cudaStream_t cs = st;
  if (stream16) {
    const act_t* x16 = static_cast<const act_t*>(x);
    return [=] { layernorm_backward(dy, x16, ld, nullptr, 1, stats, n.gamma, rows, Wd, accumulate, gx, gx16, cs); };
  }
  const float* x32 = static_cast<const float*>(x);
  return [=] { layernorm_backward(dy, x32, ld, nullptr, 1, stats, n.gamma, rows, Wd, accumulate, gx, gx16, cs); };
}

void Engine::stream_residual(GemmEpilogue& e, const void* res, void* out) const {
  if (stream16) {
    e.res_f16 = static_cast<const act_t*>(res);
    e.out_f16 = static_cast<act_t*>(out);
  } else {
    e.res_f32 = static_cast<const float*>(res);
    e.out_f32 = static_cast<float*>(out);
  }
}

// One pre-norm block, 64-wide heads:  x_mid = x_in + attn(ln_1(x_in)) Wo^T + bo,
// x_out = x_mid + act(ln_2(x_mid) Wfc^T + bfc) Wproj^T + bproj.  Appends the forward to `fwd` and, when `bwd` is given,
// the backward (gx16 / gx of x_out -> of x_in, accumulated in place) to *bwd in execution order; returns the attention
// chain's P (nullptr on the fused paths).
act_t* Engine::add_block(OpList& fwd, OpList* bwd, const BlockW& w, const BlockIO& b) {
  const int Wd = 64 * b.heads, M = b.images * b.T, Mr = b.rows;
  const long long xld = b.ld;
  fwd.add(1, stream_ln_fwd(b.x_in, Wd, w.ln1, M, Wd, b.eps, b.h16, b.stats1), 0.0, "layernorm_forward");
  {
    GemmEpilogue e;
    e.bias = w.bqkv;
    e.out_f16 = b.qkv;
    e.ldc = 3 * Wd;
    add_gemm(fwd, opK(b.h16, Wd, M, Wd), opK(w.wqkv, Wd, 3 * Wd, Wd), M, 3 * Wd, Wd, e);
  }
  OpList attn_bwd;
  act_t* P = add_attention(b.site, fwd, bwd ? &attn_bwd : nullptr, b.qkv, b.o, b.go, b.gqkv, b.images, b.heads, b.T, 64,
                           1.f / std::sqrt(64.f), true, b.dP, b.causal);
  {  // x_mid = x_in + O Wo^T + bo
    GemmEpilogue e;
    e.bias = w.bo;
    stream_residual(e, b.x_in, b.x_mid);
    e.ldc = xld;
    add_gemm(fwd, opK(b.o, xld, Mr, Wd), opK(w.wo, Wd, Wd, Wd), Mr, Wd, Wd, e);
  }
  fwd.add(1, stream_ln_fwd(b.x_mid, xld, w.ln2, Mr, Wd, b.eps, b.h16, b.stats2), 0.0, "layernorm_forward");
  {  // gact = act(h Wfc^T + bfc), keep the pre-activation u
    GemmEpilogue e;
    e.bias = w.bfc;
    e.act = b.act;
    e.aux_out = b.u;
    e.out_f16 = b.gact;
    e.ldc = 4 * Wd;
    add_gemm(fwd, opK(b.h16, Wd, Mr, Wd), opK(w.wfc, Wd, 4 * Wd, Wd), Mr, 4 * Wd, Wd, e);
  }
  {  // x_out = x_mid + gact Wproj^T + bproj
    GemmEpilogue e;
    e.bias = w.bproj;
    stream_residual(e, b.x_mid, b.x_out);
    e.ldc = xld;
    add_gemm(fwd, opK(b.gact, 4 * Wd, Mr, 4 * Wd), opK(w.wproj, 4 * Wd, Wd, 4 * Wd), Mr, Wd, 4 * Wd, e);
  }
  if (!bwd) return P;
  {  // g4 = (gx Wproj) * act'(u)
    GemmEpilogue e;
    e.act = b.act == ACT_GELU ? ACT_GELU_BWD : ACT_QUICKGELU_BWD;
    e.aux_in = b.u;
    e.out_f16 = b.g4;
    e.ldc = 4 * Wd;
    add_gemm(*bwd, opK(b.gx16, xld, Mr, Wd), opMN(w.wproj, 4 * Wd, 4 * Wd, Wd), Mr, 4 * Wd, Wd, e);
  }
  {  // gh = g4 Wfc
    GemmEpilogue e;
    e.out_f16 = b.gh;
    e.ldc = Wd;
    add_gemm(*bwd, opK(b.g4, 4 * Wd, Mr, 4 * Wd), opMN(w.wfc, Wd, Wd, 4 * Wd), Mr, Wd, 4 * Wd, e);
  }
  bwd->add(1, stream_ln_bwd(b.gh, b.x_mid, xld, b.stats2, w.ln2, Mr, Wd, 1, b.gx, b.gx16), 0.0, "layernorm_backward");
  if (Mr < M) {  // the attention backward reads dO = go for every token: zero outside the tail's rows
    const size_t go_bytes = (size_t)M * Wd * sizeof(act_t);
    act_t* go = b.go;
    cudaStream_t cs = st;
    bwd->add(1, [=] { cudaMemsetAsync(go, 0, go_bytes, cs); }, 0.0, "memset go");
  }
  {  // go = gx Wo
    GemmEpilogue e;
    e.out_f16 = b.go;
    e.ldc = xld;
    add_gemm(*bwd, opK(b.gx16, xld, Mr, Wd), opMN(w.wo, Wd, Wd, Wd), Mr, Wd, Wd, e);
  }
  bwd->append(attn_bwd);
  {  // gh = gqkv Wqkv
    GemmEpilogue e;
    e.out_f16 = b.gh;
    e.ldc = Wd;
    add_gemm(*bwd, opK(b.gqkv, 3 * Wd, M, 3 * Wd), opMN(w.wqkv, Wd, Wd, 3 * Wd), M, Wd, 3 * Wd, e);
  }
  bwd->add(1, stream_ln_bwd(b.gh, b.x_in, Wd, b.stats1, w.ln1, M, Wd, 1, b.gx, b.gx16), 0.0, "layernorm_backward");
  return P;
}

// A tower's head: LayerNorm of one row per sequence (`rows` rows ld apart in the stream x), then e = ln @ proj against
// the fp16 projection [W, D] read MN-major, fp32 embeddings [rows, D]
void Engine::add_head(OpList& l, const void* x, long long ld, int rows, const NormW& n, float eps, act_t* h16,
                      float* stats, const act_t* proj16, int Wd, int D, float* out) {
  l.add(1, stream_ln_fwd(x, ld, n, rows, Wd, eps, h16, stats), 0.0, "layernorm_forward");
  GemmEpilogue e;
  e.out_f32 = out;
  e.ldc = D;
  add_gemm(l, opK(h16, Wd, rows, Wd), opMN(proj16, D, D, Wd), rows, D, Wd, e);
}

void Engine::build_clip(int i) {
  Clip& C = clip[i];
  if (C.tower == PXR_TOWER_CLIP_RESNET) return build_resnet(i);
  C.c = cfg.clip[i];
  const int mod = PXR_MOD_CLIP0 + i;
  const int Wd = C.c.width, L = C.c.layers, Hh = C.c.heads, P = C.c.patch, D = C.c.out_dim;
  if (i == 0 && C.c.image_res != cfg.cut_size) throw EngineError(-50, "clip image_res must equal cut_size");
  const int res = sets[set_of[i]].cs;
  // a LayerNorm warp gives each lane whole 4-element vectors of every 128-column slice of the row
  if (Wd % 128 || Wd > 1024 || Wd != 64 * Hh)
    throw EngineError(-51, "ViT width " + std::to_string(Wd) + " with " + std::to_string(Hh) +
                               " heads: the width must be a multiple of 128 (the LayerNorm granularity), <= 1024, "
                               "with 64-wide heads");
  if (P < 2 || res % P) throw EngineError(-52, "patch size must divide the perceptor's input resolution");
  const int gp = res / P, np = gp * gp, T = np + 1, B = n_local, M = B * T, d = 64;
  const int Kp = round_up(3 * P * P, 64), ldT = round_up(T, 8);
  C.T = T;
  C.np = np;
  C.Kp = Kp;
  C.ldT = ldT;
  C.M = M;
  C.B = B;
  cudaStream_t cs = st;
  // The two towers differ only at the edges of the same pre-norm ViT (pxr_set_clip_tower): the timm one has a patch-embed
  // bias, no ln_pre (tokens + pos_embed enter the blocks directly), exact GELU, LayerNorm eps 1e-6, and its own key names.
  const bool timm = C.tower == PXR_TOWER_TIMM_VIT;
  const float eps = timm ? 1e-6f : 1e-5f;
  C.norm = timm ? kImageNetNorm : kClipNorm;
  const std::string k_patch = timm ? "visual.patch_embed.proj.weight" : "visual.conv1.weight";
  const std::string k_proj = timm ? "image_projection" : "visual.proj";
  const HostWeight& w_cls = timm ? W(mod, "visual.cls_token", {1, 1, Wd}) : W(mod, "visual.class_embedding", {Wd});
  const HostWeight& w_pos = timm ? W(mod, "visual.pos_embed", {1, T, Wd}) : W(mod, "visual.positional_embedding", {T, Wd});
  // ---- weights
  {
    const HostWeight& w = W(mod, k_patch, {Wd, 3, P, P});
    std::vector<float> f((size_t)Wd * Kp, 0.f);
    for (int o = 0; o < Wd; ++o)
      for (int k = 0; k < 3 * P * P; ++k) f[(size_t)o * Kp + k] = w.data[(size_t)o * 3 * P * P + k];
    C.conv1 = upload_f16(f);
  }
  if (timm) C.conv1_b = upload(W(mod, "visual.patch_embed.proj.bias", {Wd}).data);
  C.cls = upload(w_cls.data);
  C.pos = upload(w_pos.data);
  C.proj16 = upload_f16(W(mod, k_proj, {Wd, D}).data);
  if (!timm) C.ln_pre = load_norm(mod, "visual.ln_pre", Wd);
  C.ln_post = load_norm(mod, timm ? "visual.norm" : "visual.ln_post", Wd);
  // ---- buffers
  C.patches = dalloc<act_t>((size_t)B * np * Kp);
  C.g_patches = dalloc<act_t>((size_t)B * np * Kp);
  C.t = dalloc<float>((size_t)M * Wd);
  {  // class-token rows are constant: t[b*T + 0] = class_embedding (cls_token)
    std::vector<float> t0((size_t)M * Wd, 0.f);
    const auto& cls = w_cls.data;
    for (int b = 0; b < B; ++b)
      for (int k = 0; k < Wd; ++k) t0[(size_t)b * T * Wd + k] = cls[k];
    PXR_CUDA(cudaMemcpyAsync(C.t, t0.data(), t0.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    PXR_CUDA(cudaStreamSynchronize(st));
  }
  C.h16 = dalloc<act_t>((size_t)M * Wd);
  C.o16 = dalloc<act_t>((size_t)M * Wd);
  C.gact = dalloc<act_t>((size_t)M * 4 * Wd);
  C.g4 = dalloc<act_t>((size_t)M * 4 * Wd);
  C.gh = dalloc<act_t>((size_t)M * Wd);
  C.go = dalloc<act_t>((size_t)M * Wd);
  C.gqkv = dalloc<act_t>((size_t)M * 3 * Wd);
  const bool fuse_attn = attn_fused(T, d, Hh) || attn_streamed(T, d, Hh);  // attn_tc.cu T <= 240, attn_long.cu T > 257
  C.dP = fuse_attn ? nullptr : dalloc<act_t>((size_t)B * Hh * T * ldT);
  const bool s16 = stream16;
  const size_t xbytes = (size_t)M * Wd * (s16 ? sizeof(act_t) : sizeof(float));
  auto xalloc = [&]() -> void* { return dalloc<unsigned char>(xbytes); };
  // fp16 stream: its gradient lives in gx16 alone; fp32 stream: fp32 master gx + the fp16 copy the dgrad GEMMs read
  C.gx = s16 ? nullptr : dalloc<float>((size_t)M * Wd);
  C.gx16 = dalloc<act_t>((size_t)M * Wd);
  C.stats_pre = dalloc<float>((size_t)M * 2);
  C.stats_post = dalloc<float>((size_t)B * 2);
  C.e = dalloc<float>((size_t)B * D);
  C.e_unit = dalloc<float>((size_t)B * D);
  C.de = dalloc<float>((size_t)B * D);
  C.de16 = dalloc<act_t>((size_t)B * D);
  C.hcls = dalloc<act_t>((size_t)B * Wd);
  C.gcls = dalloc<act_t>((size_t)B * Wd);
  void* x_cur = xalloc();
  void* x0 = x_cur;
  C.layers.resize(L);
  std::vector<OpList> block_bwd(L);  // per layer, built with the forward, spliced into the backward in reverse

  // ---- forward: patch embed (conv1 as GEMM over im2col'd patches, written straight into the token rows 1..np)
  {
    GemmEpilogue e;
    e.bias = C.conv1_b;
    e.out_f32 = C.t + Wd;
    e.ldc = Wd;
    e.bs0 = (long long)T * Wd;
    add_gemm(C.fwd, opK(C.patches, Kp, np, Kp, B, (long long)np * Kp), opK(C.conv1, Kp, Wd, Kp), np, Wd, Kp, e);
  }
  {  // x0 = ln_pre(t + pos) (openai-CLIP), or t + pos_embed (timm)
    Clip* c = &C;
    void* xo = x0;
    act_t* xo16 = s16 ? static_cast<act_t*>(xo) : nullptr;
    float* xo32 = s16 ? nullptr : static_cast<float*>(xo);
    if (timm)
      C.fwd.add(1, [=] { add_pos_embed(c->t, c->pos, T, M, Wd, xo16, xo32, cs); }, 0.0, "add_pos_embed");
    else
      C.fwd.add(1, [=] {
        layernorm_forward(c->t, Wd, c->pos, T, c->ln_pre.gamma, c->ln_pre.beta, M, Wd, eps, xo16, xo32, c->stats_pre, cs);
      }, 0.0, "layernorm_forward");
  }
  BlockIO b;  // what every layer shares; the loop sets the rest
  b.h16 = C.h16;
  b.gact = C.gact;
  b.images = B;
  b.heads = Hh;
  b.T = T;
  b.act = timm ? ACT_GELU : ACT_QUICKGELU;
  b.eps = eps;
  b.causal = false;
  b.go = C.go;
  b.gqkv = C.gqkv;
  b.dP = C.dP;
  b.g4 = C.g4;
  b.gh = C.gh;
  b.gx16 = C.gx16;
  b.gx = C.gx;
  for (int l = 0; l < L; ++l) {
    Clip::Layer& Ly = C.layers[l];
    Ly.w = load_block(mod, (timm ? "visual.blocks." : "visual.transformer.resblocks.") + std::to_string(l), Wd, timm);
    b.x_in = Ly.x_in = x_cur;
    b.x_mid = Ly.x_mid = xalloc();
    b.x_out = x_cur = xalloc();
    b.stats1 = Ly.stats1 = dalloc<float>((size_t)M * 2);
    b.stats2 = Ly.stats2 = dalloc<float>((size_t)M * 2);
    b.qkv = Ly.qkv = dalloc<act_t>((size_t)M * 3 * Wd);
    b.u = Ly.u = dalloc<act_t>((size_t)M * 4 * Wd);
    if (fuse_attn) Ly.o = dalloc<act_t>((size_t)M * Wd);
    b.o = fuse_attn ? Ly.o : C.o16;
    // Last layer: only the class token's row of every image reaches ln_post / proj (slip.py:62-66 ->
    // VisionTransformer.forward takes x[:, 0, :]), and everything after the attention is row-wise -- out_proj, ln_2, the MLP
    // and their backward run on those B rows (row pitch T * W inside the [M, W] buffers) instead of on all M = B T rows.
    // Exact: the other rows' outputs are never read and their gradients are zero.  PXR_CLIP_LAST_CLS=0 computes all rows.
    const bool cls_only = clip_last_cls && l == L - 1;
    b.rows = cls_only ? B : M;
    b.ld = cls_only ? (long long)T * Wd : (long long)Wd;
    b.site = "clip" + std::to_string(i) + " block " + std::to_string(l);
    Ly.P = add_block(C.fwd, &block_bwd[l], Ly.w, b);
  }
  C.x_out = x_cur;
  // head: ln_post on the class-token rows (row stride T*W), then e = ln @ proj
  add_head(C.fwd, C.x_out, (long long)T * Wd, B, C.ln_post, eps, C.hcls, C.stats_post, C.proj16, Wd, D, C.e);

  // ---- backward (execution order).  Weight operands of the dgrad GEMMs are MN-major views of the forward weights.
  {  // head backward: gcls = de proj^T (proj [W, D] read K-major: n = W rows, k = D), then LN backward on class rows
    Clip* c = &C;
    GemmEpilogue e;
    e.out_f16 = C.gcls;
    e.ldc = Wd;
    add_gemm(C.bwd, opK(C.de16, D, B, D), opK(C.proj16, D, Wd, D), B, Wd, D, e);
    const size_t nbytes32 = (size_t)M * Wd * sizeof(float), nbytes16 = (size_t)M * Wd * sizeof(act_t);
    const Op ln_bwd = stream_ln_bwd(C.gcls, C.x_out, (long long)T * Wd, C.stats_post, C.ln_post, B, Wd, 0, C.gx, C.gx16);
    C.bwd.add(1, [=] {
      if (c->gx) cudaMemsetAsync(c->gx, 0, nbytes32, cs);
      cudaMemsetAsync(c->gx16, 0, nbytes16, cs);
      ln_bwd();
    });
  }
  for (int l = L - 1; l >= 0; --l) C.bwd.append(block_bwd[l]);
  {  // ln_pre backward (x = t + pos), then patch-embed dgrad on token rows 1..np of every image.  timm: x0 = t + pos_embed,
     // so the stream gradient in gx16 already is d/dt
    Clip* c = &C;
    if (!timm)
      C.bwd.add(1, [=] { layernorm_backward(c->gx16, c->t, Wd, c->pos, T, c->stats_pre, c->ln_pre.gamma, M, Wd, 0, c->gx, c->gx16, cs); }, 0.0, "layernorm_backward");
    GemmEpilogue e;
    e.out_f16 = C.g_patches;
    e.ldc = Kp;
    e.bs0 = (long long)np * Kp;
    add_gemm(C.bwd, opK(C.gx16 + Wd, Wd, np, Wd, B, (long long)T * Wd), opMN(C.conv1, Kp, Kp, Wd), np, Kp, Wd, e);
  }
}

void Engine::clip_input(int i) {
  Clip& C = clip[i];
  const CutSet& K = sets[set_of[i]];
  if (C.tower == PXR_TOWER_CLIP_RESNET) rn_stem_forward(K.batch, K.range, n_local, K.cs, rn[i]->cols, C.norm, st);
  else patchify_forward(K.batch, K.range, n_local, K.cs, C.c.patch, C.Kp, C.patches, C.norm, st);
  launches += 1;
}

void Engine::clip_input_backward(int i, bool accumulate, FxPass fx) {
  Clip& C = clip[i];
  const CutSet& K = sets[set_of[i]];
  if (C.tower == PXR_TOWER_CLIP_RESNET)
    rn_stem_backward(rn[i]->g_cols, K.batch, K.range, n_local, K.cs, accumulate, K.g_batch, sums_fx, fx, C.norm, st);
  else
    patchify_backward(C.g_patches, K.batch, K.range, n_local, K.cs, C.c.patch, C.Kp, accumulate, K.g_batch, sums_fx, fx,
                      C.norm, st);
  launches += 1;
}

void Engine::forward_clip(int i) {
  clip_input(i);
  run(clip[i].fwd);
  check_launch("clip forward");
}

// Prompt rows of every perceptor: its text prompts (one row each), then cutn rows per image prompt.  Row j carries its
// Prompt's weight / stop, the loss slot it sums into and 1 / (rows of that Prompt).
void Engine::rebuild_prompt_rows() {
  int off = (int)filters.size();  // filter losses come first in the reference's result list (pixray.py:1203-1222)
  for (int i = 0; i < cfg.n_clip; ++i) {
    Clip& C = clip[i];
    // the reference's result order per perceptor: spot prompts, spot-off prompts, prompts, image prompts (pixray.py:1283-1336)
    for (int which : {1, 0}) {
      Clip::Spot& sp = C.spot[which];
      dfree(sp.d_rows);
      dfree(sp.d_w);
      dfree(sp.d_stop);
      dfree(sp.d_inv);
      dfree(sp.d_slot);
      sp.loss_offset = off;
      if (sp.n > 0) {
        sp.d_rows = upload(sp.rows);
        sp.d_w = upload(sp.w);
        sp.d_stop = upload(sp.stop);
        sp.d_inv = upload(std::vector<float>(sp.n, 1.f));
        std::vector<int> slot(sp.n);
        for (int j = 0; j < sp.n; ++j) slot[j] = j;
        sp.d_slot = upload(slot);
        off += sp.n;
      }
    }
    const int D = C.c.out_dim, rows = C.n_text + n_img * cfg.cutn;
    const int most = std::max(rows, std::max(C.spot[0].n, C.spot[1].n));
    dfree(C.ploss_part);
    if (most > 0) C.ploss_part = dalloc<float>((size_t)C.B * most, false);
    if (!C.ploss_count) C.ploss_count = dalloc<unsigned int>(1);
    std::vector<float> pr((size_t)rows * D, 0.f), w(rows), stp(rows), inv(rows);
    std::vector<int> slot(rows);
    std::copy(C.text_rows.begin(), C.text_rows.end(), pr.begin());
    for (int j = 0; j < C.n_text; ++j) {
      w[j] = C.text_w[j];
      stp[j] = C.text_stop[j];
      slot[j] = j;
      inv[j] = 1.f;
    }
    for (int k = 0; k < n_img; ++k)
      for (int r = 0; r < cfg.cutn; ++r) {
        const int j = C.n_text + k * cfg.cutn + r;
        w[j] = img_w[k];
        stp[j] = -INFINITY;  // Prompt(embed, weight) with the default stop (pixray.py:1331-1333)
        slot[j] = C.n_text + k;
        inv[j] = 1.f / cfg.cutn;
      }
    dfree(C.prompts);
    dfree(C.pweights);
    dfree(C.pstops);
    dfree(C.pinv);
    dfree(C.pslot);
    if (rows > 0) {
      C.prompts = upload(pr);
      C.pweights = upload(w);
      C.pstops = upload(stp);
      C.pinv = upload(inv);
      C.pslot = dalloc<int>(rows);
      PXR_CUDA(cudaMemcpyAsync(C.pslot, slot.data(), sizeof(int) * rows, cudaMemcpyHostToDevice, st));
      PXR_CUDA(cudaStreamSynchronize(st));
    }
    C.n_rows = rows;
    C.n_prompts = C.n_text + n_img;
    C.loss_offset = off;
    off += C.n_prompts;
  }
  if (off + (int)anchors.size() + (num_losses() - aux_base()) > 64) throw EngineError(-16, "at most 64 losses (prompts + anchors + auxiliary) in total");
  total_prompts = off;
}

// The throwaway image Prompts of this iteration (pixray.py:1308-1336): make_cutouts(timg) replays the iteration's cached
// transforms (no ColorJitter on that path, pixray.py:480-486; fresh noise), perceptor.encode_image, and the [cutn, D]
// unit embeddings become the rows of Prompt(embed, weight).  Forward only: the targets are constants.  Runs before
// the main pass, which then overwrites every buffer used here.
void Engine::encode_image_prompts(int s) {
  if (n_img == 0) return;
  CutSet& K = sets[s];
  const size_t ncs = (size_t)3 * K.src_h * K.src_w;
  for (int k = 0; k < n_img; ++k) {
    CutoutArgs a = K.cut_args;
    a.jitter = nullptr;
    a.iter = K.cut_args.iter + (k + 1) * (1 << 24);  // engine-drawn noise: an independent Philox stream per call
    a.pooled = K.img_prompts + k * ncs;
    cutout_forward(a, K.batch, K.part_min, K.part_max, K.part_imin, K.part_imax, st);
    minmax_reduce(nullptr, K.part_min, K.part_max, K.part_imin, K.part_imax, K.n_parts, K.range, K.irange, st);
    launches += 2;
    if (comm) {
      range_pack(K.range, xbuf, st);
      nccl_check(Comm::api().all_reduce(xbuf, xbuf, 2, Comm::kFloat32, Comm::kMin, comm, st), "allreduce(min,max)");
      range_unpack(xbuf, K.range, K.irange, st);
      launches += 3;
    }
    for (int i = 0; i < cfg.n_clip; ++i) {  // each target is cut with its perceptor's own set (pixray.py:1308-1336)
      if (set_of[i] != s) continue;
      Clip& C = clip[i];
      const int D = C.c.out_dim;
      clip_input(i);
      run(C.fwd);
      float* rows = C.prompts + (size_t)(C.n_text + k * cfg.cutn) * D;
      if (comm) PXR_CUDA(cudaMemsetAsync(rows, 0, sizeof(float) * cfg.cutn * D, st));
      // zero prompt rows: the kernel only normalises (slip.py:66) into `rows`; de is overwritten by the main pass
      prompt_loss(C.e, C.B, D, C.prompts, C.pweights, C.pstops, C.pslot, C.pinv, 0, cfg.cutn, S,
                  rows + (size_t)first_global * D, losses_dev + C.loss_offset, C.de, C.de16, nullptr, nullptr, st);
      launches += 1;
      if (comm)  // every rank needs all cutn rows; each rank filled its own, the others are zero: the sum is exact
        nccl_check(Comm::api().all_reduce(rows, rows, (size_t)cfg.cutn * D, Comm::kFloat32, Comm::kSum, comm, st),
                   "allreduce(image prompt rows)");
    }
  }
  check_launch("image prompts");
}

void Engine::loss_clip(int i) {
  Clip& C = clip[i];
  if (C.n_prompts == 0) throw EngineError(-70, "no prompts set for perceptor " + std::to_string(i));
  prompt_loss(C.e, C.B, C.c.out_dim, C.prompts, C.pweights, C.pstops, C.pslot, C.pinv, C.n_rows, cfg.cutn, S, C.e_unit,
              losses_dev + C.loss_offset, C.de, C.de16, C.ploss_part, C.ploss_count, st);
  launches += 1;
  if (i == cfg.n_clip - 1 && !aux.empty()) aux_after_embed();
}

// ---- auxiliary losses.  Where each one enters the hand-written backward chain mirrors which tensor the reference
// loss reads: `globals["embeds"]` (pixray.py:1372-1376, the LAST perceptor's embeddings), `cur_cutouts`, or `out`.
void Engine::aux_after_embed() {
  for (size_t k = 0; k < aux.size(); ++k) {
    AuxLoss& a = aux[k];
    if (a.kind != PXR_LOSS_AESTHETIC) continue;
    Clip& C = clip[cfg.n_clip - 1];
    if (a.n_dev != C.c.out_dim) throw EngineError(-81, "aesthetic head width does not match the last perceptor's embedding");
    aux_aesthetic(C.e, C.B, C.c.out_dim, cfg.cutn, a.dev, a.prm[1], a.prm[0], a.weight, S, C.de, C.de16, aux_part,
                  losses_dev + aux_slot(k), st);
    launches += 2;
  }
}

void Engine::aux_on_cutouts(int s) {
  CutSet& K = sets[s];
  const int cs_ = K.cs;
  float* const batch = K.batch;
  float* const g_batch = K.g_batch;
  for (size_t k = 0; k < aux.size(); ++k) {
    AuxLoss& a = aux[k];
    if (!aux_per_set(a.kind)) continue;
    float* slot = losses_dev + aux_slot(k, s);
    if (a.kind == PXR_LOSS_SATURATION) {
      aux_saturation_moments(batch, n_local, cs_, aux_part, aux_sums, st);
      if (comm) nccl_check(Comm::api().all_reduce(aux_sums, aux_sums, 4, Comm::kFloat64, Comm::kSum, comm, st), "allreduce(saturation moments)");
      // the value is a function of the GLOBAL moments: one rank contributes it to the (summed) loss vector
      aux_saturation_grad(batch, n_local, cs_, cfg.cutn, aux_sums, a.weight * a.prm[0], S, cfg.rank == 0, g_batch, slot, st);
      launches += 3;
    } else if (a.kind == PXR_LOSS_PALETTE) {
      aux_palette(batch, n_local, cs_, cfg.cutn, a.dev, a.n_dev / 3, a.weight * a.prm[0], S, g_batch, K.aux_best, aux_part, slot, st);
      launches += 2;
    } else if (a.kind == PXR_LOSS_SMOOTHNESS) {
      // {w, type, spacing[, edge_order[, n, taps]]}: a.dev holds the n 1-D taps of the blur when n > 0
      const int order = a.prm.size() > 3 ? (int)a.prm[3] : 1, nt = a.dev ? a.n_dev : 0;
      const float* src = batch;
      int cs2 = cs_;
      if (nt) {  // the gradient runs on the blurred cutouts (SmoothnessLoss.py:92-94)
        cs2 = cs_ - nt + 1;
        aux_smooth_blur(batch, n_local, cs_, a.dev, nt, K.aux_blur_tmp, K.aux_blur, st);
        src = K.aux_blur;
        launches += 2;
      }
      if (comm) {  // torch.gradient runs over the stacked rows of ALL cutouts: two halo rows from each neighbour
        PXR_CUDA(cudaMemsetAsync(K.aux_xbuf, 0, sizeof(float) * 12 * cs2 * cfg.world, st));
        aux_smooth_pack_halo(src, n_local, cs2, cfg.rank, K.aux_xbuf, st);
        nccl_check(Comm::api().all_reduce(K.aux_xbuf, K.aux_xbuf, (size_t)12 * cs2 * cfg.world, Comm::kFloat32, Comm::kSum, comm, st), "allreduce(smoothness halo)");
        aux_smooth_unpack_halo(K.aux_xbuf, cs2, cfg.rank, cfg.world, K.aux_halo, st);
        launches += 3;
      }
      aux_smoothness(src, n_local, cs2, first_global, cfg.cutn, K.aux_halo, a.prm[2], (int)a.prm[1], order,
                     a.weight * a.prm[0], S, K.aux_A, nt ? K.aux_g_blur : g_batch, nt ? 0 : 1, aux_part, slot, st);
      launches += 3;
      if (nt) {
        aux_smooth_blur_adjoint(K.aux_g_blur, n_local, cs_, a.dev, nt, K.aux_blur_tmp, g_batch, st);
        launches += 2;
      }
    }
  }
}

void Engine::aux_on_image() {
  const int H = cur_cut_h(), Wd = cur_cut_w();
  const float* img = cur_cut_img();   // `out` of do_synth_and_filter: the FILTERED image (pixray.py:1384-1393)
  float* g_img = cur_g_cut_img();
  for (size_t k = 0; k < aux.size(); ++k) {
    AuxLoss& a = aux[k];
    float* slot = losses_dev + aux_slot(k);
    if (a.kind == PXR_LOSS_SYMMETRY) {
      aux_symmetry(img, H, Wd, a.weight * a.prm[0], S, g_img, aux_part, slot, st);
      launches += 2;
    } else if (a.kind == PXR_LOSS_EDGE) {
      const int m[4] = {(int)a.prm[2], (int)a.prm[3], (int)a.prm[4], (int)a.prm[5]};
      const int mode = a.prm.size() > 9 ? (int)a.prm[9] : 0;
      if (mode && (H != cfg.image_h || Wd != cfg.image_w))
        throw EngineError(-81, "edge loss target / mask were sized for the canvas, the image the loss reads differs");
      const float* target = (mode & 1) ? a.dev : nullptr;
      const float* mask = (mode & 2) ? a.dev + ((mode & 1) ? 3 * (size_t)H * Wd : 0) : nullptr;
      aux_edge(img, H, Wd, m, &a.prm[6], target, mask, a.prm[0], a.prm[1], a.weight, S, g_img, aux_part, slot, st);
      launches += 2;
    } else if (a.kind == PXR_LOSS_GAUSSIAN) {
      aux_gaussian(img, H, Wd, a.prm[1], a.prm[2], &a.prm[3], a.weight * a.prm[0], S, g_img, aux_part, slot, st);
      launches += 2;
    }
  }
}

// CLIP backward of every participating perceptor -> d loss / d cutouts -> (range terms, ColorJitter, warp adjoint) ->
// d loss / d pooled [-> un-stretch] [-> spot mask] -> d loss / d image (= or +=).  `a` = the cutout parameters of the pass
// whose activations are live; mask_which >= 0: a spot pass (only the perceptors with spot prompts of that kind ran).
void Engine::backward_to_image(int s, const CutoutArgs& a, int mask_which, bool accumulate_img, bool main_pass) {
  CutSet& K = sets[s];
  bool first = true;
  const FxPass fx_sums = next_fx(1);
  for (int i = 0; i < cfg.n_clip; ++i) {
    Clip& C = clip[i];
    if (set_of[i] != s || (mask_which >= 0 && C.spot[mask_which].n == 0)) continue;
    run(C.bwd);
    clip_input_backward(i, !first, fx_sums);
    first = false;
  }
  if (main_pass && !aux.empty()) aux_on_cutouts(s);
  ProfRec prof_rec;
  if (profiling) prof_begin_stage(prof_rec, "cutouts_bwd set " + std::to_string(s));
  range_sums_finish(sums_fx, fx_sums, K.sums, st);  // fixed point -> fp32 (and the accumulator is clean for the next pass)
  if (comm)  // d/dmin, d/dmax terms need the sums over ALL cutouts
    nccl_check(Comm::api().all_reduce(K.sums, K.sums, 2, Comm::kFloat32, Comm::kSum, comm, st), "allreduce(sums)");
  cutout_backward(a, K.g_batch, K.range, K.irange, K.sums, grad_fx, next_fx(0), K.g_cut_src, st);
  launches += 2;
  const int ncs = 3 * K.cs * K.cs;
  if (aspect != 1.0) {
    rescale_bilinear_backward(K.g_cut_src, K.cs, K.cs, K.src_h, K.src_w, grad_fx, next_fx(0), K.g_pooled, st);
    launches += 2;
  }
  if (mask_which >= 0) {  // cutout[0][mask_indexes] = 0 (pixray.py:466): no gradient through the zeroed pixels
    spot_mask_apply(K.g_pooled, spot_mask, mask_which == 1, ncs, K.g_pooled, st);
    launches += 1;
  }
  // the sets meet here: the first writes d loss / d image, every later one adds to it
  pool_backward(K.g_pooled, K.pool_argmax, cur_cut_h(), cur_cut_w(), K.cs, cur_g_cut_img(), st, accumulate_img ? 1 : 0);
  launches += 2;
  K.cut = false;
  if (profiling) prof_end_stage(prof_rec);
}

void Engine::backward_drawer() {
  if (comm) {
    // The path's one exchange step.  It sits on the IMAGE gradient, not on z.grad: ClampWithGrad's backward
    // (vqgan.py:76-79) masks by the sign of the incoming gradient, so the drawer backward is not linear in it and
    // must see the gradient of ALL cutouts.  Every rank then runs the (replicated) drawer backward on identical bits.
    Comm& c = Comm::api();
    nccl_check(c.group_start(), "group start");
    nccl_check(c.all_reduce(cur_g_cut_img(), cur_g_cut_img(), (size_t)3 * cur_cut_h() * cur_cut_w(), Comm::kFloat32, Comm::kSum,
                            comm, st),
               "allreduce(d loss / d image)");
    nccl_check(c.all_reduce(losses_dev, losses_dev, 64, Comm::kFloat32, Comm::kSum, comm, st), "allreduce(losses)");
    nccl_check(c.group_end(), "group end");
    launches += 2;
  }
  // image losses are replicated (every rank holds the same `out`): added after the exchange, values written, not summed
  if (!aux.empty()) aux_on_image();
  if (!anchors.empty()) anchors_on_image();
  if (filtered_valid) filters_backward();  // d loss / d filtered image -> d loss / d image (+ the filters' own loss gradients)
  if (cfg.drawer == PXR_DRAWER_VDIFF) vdiff_backward();
  else run(drawer_bwd);
  if (!anchors.empty()) anchors_on_z();
  check_launch("backward");
}

// init_weight_pix (pixray.py:1363-1368): l1 between `out` (the filtered image) and the init image, replicated on every rank
void Engine::anchors_on_image() {
  const long long n = 3LL * cur_cut_h() * cur_cut_w();
  for (size_t k = 0; k < anchors.size(); ++k) {
    Anchor& a = anchors[k];
    if (a.kind != PXR_ANCHOR_PIX) continue;
    if ((long long)a.n != n) throw EngineError(-82, "init_weight_pix: the init image must have the size of the (filtered) image");
    anchor_pix(cur_cut_img(), a.ref, n, a.weight, S, cur_g_cut_img(), aux_part, losses_dev + total_prompts + k, st);
    launches += 2;
  }
}

// init_weight / init_weight_dist / init_weight_cos / image_labels (pixray.py:1344-1375): terms between drawer.get_z() and
// a stored latent; their gradient never passes the drawer, so it is added to z.grad after the drawer backward
void Engine::anchors_on_z() {
  for (size_t k = 0; k < anchors.size(); ++k) {
    Anchor& a = anchors[k];
    if (a.kind == PXR_ANCHOR_PIX) continue;
    anchor_z(a.kind, z_buf, a.ref, (int)z_numel, a.weight, z_grad, losses_dev + total_prompts + k, st);
    launches += 1;
  }
}

// Every set cut since the last backward, in set order (set 0 alone when none was: a batch handed to pxr_encode_image)
void Engine::backward_all() {
  bool any = false;
  for (const CutSet& K : sets) any |= K.cut;
  bool acc = spot_accumulated;
  for (int s = 0; s < n_sets(); ++s) {
    if (!(sets[s].cut || (s == 0 && !any))) continue;
    backward_to_image(s, sets[s].cut_args, -1, acc, true);
    acc = true;
  }
  spot_accumulated = false;
  backward_drawer();
}

// One spot pass (pixray.py:1262-1293): the pooled image with the spot (which = 1) or everything but the spot (which = 0)
// zeroed, cut with THIS iteration's cached transforms (the cached path: no ColorJitter, fresh noise, pixray.py:480-486),
// encoded by every perceptor that has spot prompts of this kind, scored, and taken back to the image gradient right away
// (the activations are single-buffered; the drawer backward runs once, on the sum, in backward_drawer).
// `pooled` must hold the current image's pooling.  Returns false when no perceptor has such prompts.
bool Engine::spot_pass(int which, bool accumulate_img) {
  if (!any_spot(which)) return false;
  if (!spot_mask) throw EngineError(-71, "spot prompts need a spot mask (pxr_set_spot_mask)");
  CutSet& K = sets[0];  // spot prompts run in single-set sessions only (pxr_set_spot_prompts)
  const int ncs = 3 * K.cs * K.cs;
  spot_mask_apply(K.pooled, spot_mask, which == 1, ncs, pooled_masked, st);
  CutoutArgs a = K.cut_args;
  a.jitter = nullptr;
  a.iter = K.cut_args.iter + (9 + which) * (1 << 24);  // engine-drawn noise: its own Philox stream
  if (aspect != 1.0) {
    rescale_bilinear(pooled_masked, K.cs, K.cs, K.src_h, K.src_w, K.cut_src, st);
    a.pooled = K.cut_src;
    launches += 1;
  } else {
    a.pooled = pooled_masked;
  }
  cutout_forward(a, K.batch, K.part_min, K.part_max, K.part_imin, K.part_imax, st);
  minmax_reduce(nullptr, K.part_min, K.part_max, K.part_imin, K.part_imax, K.n_parts, K.range, K.irange, st);
  launches += 3;
  if (comm) {
    range_pack(K.range, xbuf, st);
    nccl_check(Comm::api().all_reduce(xbuf, xbuf, 2, Comm::kFloat32, Comm::kMin, comm, st), "allreduce(min,max)");
    range_unpack(xbuf, K.range, K.irange, st);
    launches += 3;
  }
  for (int i = 0; i < cfg.n_clip; ++i) {
    Clip& C = clip[i];
    Clip::Spot& sp = C.spot[which];
    if (sp.n == 0) continue;
    forward_clip(i);
    prompt_loss(C.e, C.B, C.c.out_dim, sp.d_rows, sp.d_w, sp.d_stop, sp.d_slot, sp.d_inv, sp.n, cfg.cutn, S, C.e_unit,
                losses_dev + sp.loss_offset, C.de, C.de16, C.ploss_part, C.ploss_count, st);
    launches += 1;
  }
  backward_to_image(0, a, which, accumulate_img, false);
  return true;
}

// clip_z without per-channel bounds: the fast pixel grid and the super-resolution latent clamp to [0, 1], the polygon fills
// RGB to [0, 1] and alpha to 1
int Engine::clip_mode() const {
  if (cfg.drawer == PXR_DRAWER_PIXEL || cfg.drawer == PXR_DRAWER_SUPERRES) return CLIP_01;
  if (cfg.drawer == PXR_DRAWER_POLYGON) return CLIP_RGBA;
  if (cfg.drawer == PXR_DRAWER_STROKES) return CLIP_STROKES;
  return CLIP_NONE;
}

void Engine::step(float lr) {
  ++adam_t;
  const int per_channel = (cfg.drawer == PXR_DRAWER_VQGAN) ? (int)(z_numel / cfg.z_channels) : 1;
  adam_clip_step(opt_kind, z_buf, adam_m, adam_v, opt_p, batches > 1 ? z_grad_acc : z_grad, 1.f, (int)z_numel, per_channel,
                 zmin, zmax, clip_mode(), zr, lr, cfg.beta1, cfg.beta2, cfg.adam_eps, adam_t, st);
  launches += 1;
}

// ---- filters (kernels_filters.cu).  Every filter becomes primitives over planar [3, H, W] buffers; EDGE primitives are taps
// (loss + gradient on the tensor they look at), the others produce a new tensor.
void Engine::rebuild_filters() {
  fprims.clear();
  int H = cfg.image_h, Wd = cfg.image_w;
  const float* cur = img;
  float* cur_g = g_img;
  auto produce = [&](FilterPrim pr, int Ho, int Wo) {
    pr.Hin = H;
    pr.Win = Wd;
    pr.Hout = Ho;
    pr.Wout = Wo;
    pr.in = cur;
    pr.g_in = cur_g;
    pr.out = dalloc<float>((size_t)3 * Ho * Wo);
    pr.g_out = dalloc<float>((size_t)3 * Ho * Wo);
    fprims.push_back(pr);
    cur = pr.out;
    cur_g = pr.g_out;
    H = Ho;
    Wd = Wo;
  };
  auto tap = [&](FilterPrim pr) {
    pr.Hin = pr.Hout = H;
    pr.Win = pr.Wout = Wd;
    pr.in = cur;
    pr.g_in = cur_g;
    fprims.push_back(pr);
  };
  for (size_t f = 0; f < filters.size(); ++f) {
    Filter& F = filters[f];
    F.H = H;
    F.W = Wd;
    FilterPrim pr{};
    pr.filter = (int)f;
    if (F.kind == PXR_FILTER_TILER) {
      pr.kind = FP_ROLL;
      pr.use_h = pr.use_w = 1;
      produce(pr, H, Wd);
    } else if (F.kind == PXR_FILTER_LOOKUP) {
      pr.kind = FP_LOOKUP;
      pr.beta = F.beta;
      produce(pr, H, Wd);
    } else {  // wallpaper.py:27-93
      const int em = F.em, em2 = em / 2;
      if (F.wp_type == 1) {  // "shift"
        pr.kind = FP_WSHIFT;
        produce(pr, 2 * H, Wd);
        continue;
      }
      const bool horiz = F.wp_type == 2 || F.wp_type == 0, vert = F.wp_type == 3 || F.wp_type == 0;
      int n_edge = 0;
      if (horiz && em != 0) {
        if (em > Wd || Wd - 2 * em2 < 1 || em2 < 1) throw EngineError(-73, "wallpaper_edge_match does not fit the image width");
        FilterPrim e = pr;
        e.kind = FP_EDGE;
        e.em = em;
        e.axis = 0;
        e.accumulate = n_edge++;
        tap(e);
        FilterPrim c = pr;
        c.kind = FP_CROP;
        c.left = em2;
        produce(c, H, Wd - 2 * em2);
      }
      if (vert && em != 0) {
        if (em > H || H - 2 * em2 < 1 || em2 < 1) throw EngineError(-73, "wallpaper_edge_match does not fit the image height");
        FilterPrim e = pr;
        e.kind = FP_EDGE;
        e.em = em;
        e.axis = 1;
        e.accumulate = n_edge++;
        tap(e);
        FilterPrim c = pr;
        c.kind = FP_CROP;
        c.top = em2;
        produce(c, H - 2 * em2, Wd);
      }
      pr.kind = FP_ROLL;
      pr.use_h = vert ? 1 : 0;
      pr.use_w = horiz ? 1 : 0;
      produce(pr, H, Wd);
    }
  }
  cut_img = const_cast<float*>(cur);
  g_cut_img = cur_g;
  cut_h = H;
  cut_w = Wd;
  // every "shift" wallpaper doubles the height, so a lookup late in the chain can see many times the canvas
  size_t lookup_px = 0;
  for (const FilterPrim& pr : fprims)
    if (pr.kind == FP_LOOKUP) lookup_px = std::max(lookup_px, (size_t)pr.Hin * pr.Win);
  if (lookup_px > lookup_best_n) {
    lookup_best = dalloc<int>(lookup_px);
    lookup_best_n = lookup_px;
  }
  reg("filtered", cut_img, (size_t)3 * cut_h * cut_w * 4);
  reg("g_filtered", g_cut_img, (size_t)3 * cut_h * cut_w * 4);
  rebuild_prompt_rows();
}

void Engine::filters_forward(int iter) {
  for (size_t f = 0; f < filters.size(); ++f) {
    Filter& F = filters[f];  // rand_w = torch.randint(0, W), rand_h = torch.randint(0, H), drawn by every filter call
    F.sh = F.fixed_h >= 0 ? F.fixed_h % F.H : (int)(philox_uniform(cfg.seed, (uint32_t)iter, 6u, 2 * f) * 0.999999f * F.H);
    F.sw = F.fixed_w >= 0 ? F.fixed_w % F.W : (int)(philox_uniform(cfg.seed, (uint32_t)iter, 6u, 2 * f + 1) * 0.999999f * F.W);
  }
  const float value_w = cfg.rank == 0 ? 1.f : 0.f;  // the loss vector is summed over ranks: one rank reports the replicated value
  for (FilterPrim& pr : fprims) {
    Filter& F = filters[pr.filter];
    float* slot = losses_dev + pr.filter;
    switch (pr.kind) {
      case FP_ROLL:
        filter_roll(pr.in, pr.Hin, pr.Win, pr.use_h ? F.sh % pr.Hin : 0, pr.use_w ? F.sw % pr.Win : 0, pr.out, st);
        break;
      case FP_WSHIFT: filter_wallpaper_shift(pr.in, pr.Hin, pr.Win, F.sh, F.sw, pr.out, st); break;
      case FP_CROP: filter_crop(pr.in, pr.Hin, pr.Win, pr.top, pr.left, pr.Hout, pr.Wout, pr.out, st); break;
      case FP_EDGE:
        filter_edge_match(pr.in, pr.Hin, pr.Win, pr.em, pr.axis, F.weight * value_w, 0.f, pr.accumulate, nullptr, slot, st);
        break;
      case FP_LOOKUP:
        filter_colorlookup(pr.in, pr.Hin * pr.Win, F.pal, F.n_col, pr.beta, F.weight * value_w, pr.out, lookup_best, aux_part, slot, st);
        launches += 1;
        break;
    }
    launches += 1;
  }
  filtered_valid = true;
  check_launch("filters forward");
}

void Engine::filters_backward() {
  for (int i = (int)fprims.size() - 1; i >= 0; --i) {
    FilterPrim& pr = fprims[i];
    Filter& F = filters[pr.filter];
    switch (pr.kind) {
      case FP_ROLL:
        filter_roll_backward(pr.g_out, pr.Hin, pr.Win, pr.use_h ? F.sh % pr.Hin : 0, pr.use_w ? F.sw % pr.Win : 0, 0, pr.g_in, st);
        break;
      case FP_WSHIFT: filter_wallpaper_shift_backward(pr.g_out, pr.Hin, pr.Win, F.sh, F.sw, 0, pr.g_in, st); break;
      case FP_CROP: filter_crop_backward(pr.g_out, pr.Hin, pr.Win, pr.top, pr.left, pr.Hout, pr.Wout, pr.g_in, st); break;
      case FP_EDGE:  // a tap: adds its loss gradient to the gradient of the tensor it looks at
        filter_edge_match(pr.in, pr.Hin, pr.Win, pr.em, pr.axis, F.weight, S, 0, pr.g_in, nullptr, st);
        break;
      case FP_LOOKUP:
        filter_colorlookup_backward(pr.g_out, pr.in, pr.out, pr.Hin * pr.Win, pr.beta, F.weight, S, 0, pr.g_in, st);
        break;
    }
    launches += 1;
  }
}

void Engine::write_initial_drop_state() {
  DropState s0{};
  s0.best_loss = 1e20f;
  s0.lr = drop_cfg.base_lr;
  PXR_CUDA(cudaMemcpyAsync(drop_state, &s0, sizeof s0, cudaMemcpyHostToDevice, st));
  PXR_CUDA(cudaMemcpyAsync(drop_state + 1, &s0, sizeof s0, cudaMemcpyHostToDevice, st));
  PXR_CUDA(cudaStreamSynchronize(st));  // s0 is a stack object
  drop_parity = 0;
  memset(const_cast<DropStatus*>(drop_status), 0, sizeof(DropStatus));
}

// opt.step() + clip_z + checkdrop + (scheduled | auto-stop) optimiser rebuild, all decided on the device
void Engine::step_managed(int iter) {
  const int per_channel = (cfg.drawer == PXR_DRAWER_VQGAN) ? (int)(z_numel / cfg.z_channels) : 1;
  const float* g = batches > 1 ? z_grad_acc : z_grad;
  // the line drawer's get_z_copy is None (linedrawer.py:189-190): no best-z snapshot for it
  float* best = cfg.drawer == PXR_DRAWER_STROKES ? nullptr : best_z;
  adam_clip_managed(opt_kind, z_buf, adam_m, adam_v, opt_p, g, best, 1.f, (int)z_numel, per_channel, zmin, zmax,
                    clip_mode(), zr, cfg.beta1, cfg.beta2, cfg.adam_eps, losses_dev, num_losses(), iter,
                    drop_cfg, drop_state + drop_parity, drop_state + (drop_parity ^ 1), drop_status_dev, st);
  drop_parity ^= 1;
  launches += 1;
}

void Engine::finalize() {
  if (finalized) return;
  if (cfg.drawer == PXR_DRAWER_VQGAN) build_vqgan();
  else if (cfg.drawer == PXR_DRAWER_PIXEL) build_pixel();
  else if (cfg.drawer == PXR_DRAWER_FFT) build_fft();
  else if (cfg.drawer == PXR_DRAWER_VDIFF) build_vdiff();
  else if (cfg.drawer == PXR_DRAWER_POLYGON) build_polygon();
  else if (cfg.drawer == PXR_DRAWER_SUPERRES) build_superres();
  else if (cfg.drawer == PXR_DRAWER_STROKES) build_strokes();
  else throw EngineError(-47, "unknown drawer kind");
  adam_m = dalloc<float>(z_numel);
  adam_v = dalloc<float>(z_numel);
  z_grad_acc = dalloc<float>(z_numel);
  best_z = dalloc<float>(z_numel);
  drop_state = dalloc<DropState>(2);
  {
    void* hp = nullptr;
    PXR_CUDA(cudaHostAlloc(&hp, sizeof(DropStatus), cudaHostAllocMapped));
    memset(hp, 0, sizeof(DropStatus));
    drop_status = static_cast<DropStatus*>(hp);
    void* dp = nullptr;
    PXR_CUDA(cudaHostGetDevicePointer(&dp, hp, 0));
    drop_status_dev = static_cast<DropStatus*>(dp);
  }
  build_cutouts();
  for (int i = 0; i < cfg.n_clip; ++i) build_clip(i);
  for (int i = 0; i < cfg.n_clip; ++i) build_text(i);
  losses_dev = dalloc<float>(64);
  losses_scratch = dalloc<float>(64);
  aux_part = dalloc<double>(std::max(4 * AUX_MAX_BLOCKS, n_local) + 8);
  aux_sums = dalloc<double>(4);
  PXR_CUDA(cudaMallocHost((void**)&losses_host, 64 * sizeof(float)));
  PXR_CUDA(cudaStreamSynchronize(st));
  {
    const size_t npx = (size_t)3 * cfg.image_h * cfg.image_w;
    reg("img", img, npx * 4);
    reg("img_pre", img_pre, npx * 4);
    reg("g_img", g_img, npx * 4);
    reg("filtered", img, npx * 4);  // the filter chain's output and its gradient; rebuild_filters moves them
    reg("g_filtered", g_img, npx * 4);
    // set 0's buffers under their plain names, every set's as setN.<name>
    for (int s = 0; s < n_sets(); ++s) {
      const CutSet& K = sets[s];
      const size_t kcs = (size_t)3 * K.cs * K.cs;
      for (const std::string& p : s == 0 ? std::vector<std::string>{"", "set0."} : std::vector<std::string>{"set" + std::to_string(s) + "."}) {
        reg(p + "pooled", K.pooled, kcs * 4);
        reg(p + "cut_src", K.cut_src, (size_t)3 * K.src_h * K.src_w * 4);
        reg(p + "pool_argmax", K.pool_argmax, kcs * 4);
        reg(p + "g_pooled", K.g_pooled, kcs * 4);
        reg(p + "batch", K.batch, kcs * n_local * 4);
        reg(p + "g_batch", K.g_batch, kcs * n_local * 4);
        reg(p + "range", K.range, 16);
        reg(p + "irange", K.irange, 16);
        reg(p + "sums", K.sums, 16);
        reg(p + "palette_best", K.aux_best, kcs / 3 * n_local * 4);
        reg(p + "minv", K.minv_dev, (size_t)n_local * 36);
      }
    }
    reg("z_grad", z_grad, z_numel * 4);
    reg("z_grad_acc", z_grad_acc, z_numel * 4);
    reg("best_z", best_z, z_numel * 4);
    reg("z", z_buf, z_numel * 4);
    reg("losses", losses_dev, 64 * 4);
    if (poly_winner) reg("poly_winner", poly_winner, npx / 3 * 4 * sizeof(int));
    if (sscene.winner) {
      reg("stroke_winner", sscene.winner, npx / 3 * 4 * sizeof(int));
      reg("stroke_caps", sscene.caps, (size_t)sscene.n_caps * sizeof(float4));
    }
    if (vd_pred) {  // gen-size
      reg("vd_pred", vd_pred, z_numel * 4);
      reg("vd_v", vd_v, z_numel * 4);
      reg("vd_gpred", vd_gpred, z_numel * 4);
    }
    for (int i = 0; i < cfg.n_clip; ++i) {
      Clip& C = clip[i];
      std::string p = "clip" + std::to_string(i) + ".";
      if (C.tower == PXR_TOWER_CLIP_RESNET) {  // the tower's own taps (clipN.rn.*) are registered by build_resnet
        reg(p + "e", C.e, (size_t)C.B * C.c.out_dim * 4);
        reg(p + "de", C.de, (size_t)C.B * C.c.out_dim * 4);
        reg(p + "de16", C.de16, (size_t)C.B * C.c.out_dim * 2);
        continue;
      }
      const size_t mw = (size_t)C.M * C.c.width;
      reg(p + "patches", C.patches, (size_t)C.B * C.np * C.Kp * 2);
      reg(p + "g_patches", C.g_patches, (size_t)C.B * C.np * C.Kp * 2);
      reg(p + "t", C.t, mw * 4);
      const size_t xb = stream16 ? 2 : 4;  // bytes per residual-stream element
      // every layer's saved activations: x{l} its input (x{L} is x_out), x_mid{l}, qkv{l}, u{l} the MLP pre-activation
      // (B rows, compact, in a class-rows-only last layer), and o{l} (fused attention) or P{l} (row softmax, pitch ldT)
      const int L = (int)C.layers.size();
      for (int l = 0; l < L; ++l) {
        const Clip::Layer& Ly = C.layers[l];
        const std::string s = std::to_string(l);
        reg(p + "x" + s, Ly.x_in, mw * xb);
        reg(p + "x_mid" + s, Ly.x_mid, mw * xb);
        reg(p + "qkv" + s, Ly.qkv, mw * 3 * 2);
        reg(p + "u" + s, Ly.u, mw * 4 * 2);
        if (Ly.o) reg(p + "o" + s, Ly.o, mw * 2);
        if (Ly.P) reg(p + "P" + s, Ly.P, (size_t)C.B * C.c.heads * C.T * C.ldT * 2);
      }
      reg(p + "x" + std::to_string(L), C.x_out, mw * xb);
      reg(p + "x_out", C.x_out, mw * xb);
      reg(p + "hcls", C.hcls, (size_t)C.B * C.c.width * 2);
      reg(p + "e", C.e, (size_t)C.B * C.c.out_dim * 4);
      reg(p + "de", C.de, (size_t)C.B * C.c.out_dim * 4);
      reg(p + "de16", C.de16, (size_t)C.B * C.c.out_dim * 2);
      if (C.gx) reg(p + "gx", C.gx, mw * 4);
      reg(p + "gx16", C.gx16, mw * 2);
    }
  }
  for (auto& m : weights) m.clear();  // host copies no longer needed
  finalized = true;
}

#include "engine_vdiff.inc"
#include "engine_superres.inc"
#include "engine_text.inc"
#include "engine_resnet.inc"

}  // namespace pxr

// ===================================================================================================== C ABI
using pxr::Engine;
using pxr::EngineError;

struct pxr_engine {
  Engine* e;
};
static thread_local std::string g_create_err;

#define PXR_TRY(h, ...)                                   \
  try {                                                   \
    __VA_ARGS__;                                          \
    return 0;                                             \
  } catch (const EngineError& ex) {                       \
    (h)->e->err = ex.what();                              \
    return ex.code;                                       \
  } catch (const std::exception& ex) {                    \
    (h)->e->err = ex.what();                              \
    return -999;                                          \
  }

extern "C" {

const char* pxr_version(void) { return "pixray_b200 0.1 (sm_90a)"; }
const char* pxr_last_error(pxr_handle h) { return h ? h->e->err.c_str() : g_create_err.c_str(); }

int pxr_create(const pxr_config* cfg, pxr_handle* out) {
  if (!cfg || !out) return -10;
  Engine* e = nullptr;
  try {
    e = new Engine(*cfg);
    e->create();
  } catch (const EngineError& ex) {
    g_create_err = ex.what();
    delete e;
    return ex.code;
  } catch (const std::exception& ex) {
    g_create_err = ex.what();
    delete e;
    return -999;
  }
  *out = new pxr_engine{e};
  return 0;
}

void pxr_destroy(pxr_handle h) {
  if (!h) return;
  delete h->e;
  delete h;
}

int pxr_load_weight(pxr_handle h, int module_id, const char* name, const float* data, const int64_t* dims, int ndim) {
  PXR_TRY(h, {
    if (module_id < 0 || module_id > PXR_MOD_CLIP3) throw EngineError(-11, "bad module id");
    if (h->e->finalized) throw EngineError(-12, "weights cannot change after pxr_finalize");
    pxr::HostWeight w;
    w.dims.assign(dims, dims + ndim);
    w.data.resize((size_t)w.numel());
    PXR_CUDA(cudaMemcpy(w.data.data(), data, w.data.size() * sizeof(float), cudaMemcpyDefault));
    h->e->weights[module_id][name] = std::move(w);
  });
}

int pxr_finalize(pxr_handle h) { PXR_TRY(h, h->e->finalize()); }

int pxr_set_clip_tower(pxr_handle h, int clip_idx, int kind) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->finalized) throw EngineError(-12, "pxr_set_clip_tower: the tower cannot change after pxr_finalize");
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    if (kind != PXR_TOWER_OPENAI_CLIP && kind != PXR_TOWER_TIMM_VIT && kind != PXR_TOWER_CLIP_RESNET)
      throw EngineError(-10, "unknown tower kind (0 openai-CLIP, 1 timm ViT, 2 CLIP ResNet)");
    e->clip[clip_idx].tower = kind;
  });
}

int pxr_text_tower(pxr_handle h, int clip_idx, int* width, int* layers, int* ctx, int* out_dim) {
  int has = 0;
  const int rc = [&]() -> int {
    PXR_TRY(h, {
      Engine* e = h->e;
      if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
      if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
      const Engine::Text* t = e->text[clip_idx].get();
      has = t ? 1 : 0;
      if (width) *width = t ? t->W : 0;
      if (layers) *layers = t ? t->L : 0;
      if (ctx) *ctx = t ? t->T : 0;
      if (out_dim) *out_dim = t ? t->D : 0;
    });
  }();
  return rc ? rc : has;
}

int pxr_encode_text(pxr_handle h, int clip_idx, const int32_t* tokens_host, int n, int ctx, float* out) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    e->encode_text(clip_idx, tokens_host, n, ctx, out);
  });
}

int pxr_set_prompts(pxr_handle h, int clip_idx, const float* embeds, int n, int D, const float* weights,
                    const float* stops) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    auto& C = e->clip[clip_idx];
    if (D != C.c.out_dim) throw EngineError(-15, "prompt embedding width does not match the perceptor");
    std::vector<float> pe((size_t)n * D);
    for (int j = 0; j < n; ++j) {  // F.normalize(self.embed), pixray.py:277
      double s = 0;
      for (int k = 0; k < D; ++k) s += (double)embeds[(size_t)j * D + k] * embeds[(size_t)j * D + k];
      double nrm = std::max(std::sqrt(s), 1e-12);
      for (int k = 0; k < D; ++k) pe[(size_t)j * D + k] = (float)(embeds[(size_t)j * D + k] / nrm);
    }
    C.text_rows = pe;
    C.text_w.assign(weights, weights + n);
    C.text_stop.assign(stops, stops + n);
    C.n_text = n;
    e->rebuild_prompt_rows();
  });
}

// Image prompts at their own sizes (the reference keeps each target at its aspect-preserving size, resize_image
// pixray.py:514-518, and MakeCutouts pools whatever it is given to cut_size x cut_size, pixray.py:463): imgs[k] is host or
// device fp32 [3, hs[k], ws[k]] in [0, 1].  Pooled here, once.
int pxr_set_image_prompts_sized(pxr_handle h, const float* const* imgs, const int* hs, const int* ws, int n,
                                const float* weights) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (n < 0 || (n > 0 && (!imgs || !hs || !ws))) throw EngineError(-17, "pxr_set_image_prompts: bad arguments");
    e->n_img = n;
    e->img_w.assign(n, 1.f);
    if (weights)
      for (int k = 0; k < n; ++k) e->img_w[k] = weights[k];
    for (Engine::CutSet& K : e->sets) e->dfree(K.img_prompts);
    for (Engine::CutSet& K : e->sets) {
      if (n == 0) break;
      const size_t ncs = (size_t)3 * K.src_h * K.src_w;
      K.img_prompts = e->dalloc<float>(ncs * n);
      for (int k = 0; k < n; ++k) {
        if (hs[k] < 1 || ws[k] < 1 || !imgs[k]) throw EngineError(-17, "pxr_set_image_prompts: empty image");
        float* tmp = nullptr;
        const size_t bytes = sizeof(float) * 3 * hs[k] * ws[k];
        PXR_CUDA(cudaMalloc(&tmp, bytes));
        cudaError_t ce = cudaMemcpyAsync(tmp, imgs[k], bytes, cudaMemcpyDefault, e->st);
        if (ce == cudaSuccess) {
          if (e->aspect != 1.0) {  // pooled like the canvas, then stretched like the canvas (pixray.py:463-472)
            pxr::pool_forward(tmp, hs[k], ws[k], K.cs, K.pooled, K.pool_argmax, e->st);
            pxr::rescale_bilinear(K.pooled, K.cs, K.cs, K.src_h, K.src_w, K.img_prompts + k * ncs, e->st);
          } else {
            pxr::pool_forward(tmp, hs[k], ws[k], K.cs, K.img_prompts + k * ncs, K.pool_argmax, e->st);
          }
          ce = cudaStreamSynchronize(e->st);
        }
        cudaFree(tmp);
        if (ce != cudaSuccess) throw EngineError(-200, std::string("image prompt upload failed: ") + cudaGetErrorString(ce));
      }
    }
    e->rebuild_prompt_rows();
  });
}

// Spot prompts (args.spot_prompts / args.spot_prompts_off, pixray.py:917-931, 1262-1293): which = 1 scores `embeds` on the
// cutouts of the image with the spot region zeroed (make_cutouts(out, spot=1)), which = 0 on the cutouts with everything
// BUT the spot zeroed.  n = 0 clears.  Needs pxr_set_spot_mask.  Fused path (pxr_iterate) only.
int pxr_set_spot_prompts(pxr_handle h, int clip_idx, int which, const float* embeds, int n, int D, const float* weights,
                         const float* stops) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    if (which != 0 && which != 1) throw EngineError(-72, "pxr_set_spot_prompts: which = 1 (spot) or 0 (spot off)");
    if (e->n_sets() > 1 && n > 0) throw EngineError(-69, e->spot_multiset_error());
    auto& C = e->clip[clip_idx];
    if (n > 0 && D != C.c.out_dim) throw EngineError(-15, "prompt embedding width does not match the perceptor");
    auto& sp = C.spot[which];
    sp.rows.assign((size_t)n * (n > 0 ? D : 0), 0.f);
    for (int j = 0; j < n; ++j) {  // F.normalize(self.embed), pixray.py:277
      double s2 = 0;
      for (int k = 0; k < D; ++k) s2 += (double)embeds[(size_t)j * D + k] * embeds[(size_t)j * D + k];
      const double nrm = std::max(std::sqrt(s2), 1e-12);
      for (int k = 0; k < D; ++k) sp.rows[(size_t)j * D + k] = (float)(embeds[(size_t)j * D + k] / nrm);
    }
    sp.w.assign(weights, weights + (n > 0 ? n : 0));
    sp.stop.assign(stops, stops + (n > 0 ? n : 0));
    sp.n = n > 0 ? n : 0;
    e->rebuild_prompt_rows();
  });
}

// mask: host bytes [3, cut_size, cut_size], != 0 where the (resized, RGB) mask image is >= 0.5 (fetch_spot_indexes,
// pixray.py:370-394)
int pxr_set_spot_mask(pxr_handle h, const unsigned char* mask) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (!mask) throw EngineError(-10, "pxr_set_spot_mask: null mask");
    if (e->n_sets() > 1) throw EngineError(-69, e->spot_multiset_error());
    const size_t n = (size_t)3 * e->cfg.cut_size * e->cfg.cut_size;
    if (!e->spot_mask) e->spot_mask = e->dalloc<unsigned char>(n);
    PXR_CUDA(cudaMemcpyAsync(e->spot_mask, mask, n, cudaMemcpyHostToDevice, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
  });
}

int pxr_set_image_prompts(pxr_handle h, const float* imgs, int n, const float* weights) {
  if (!h) return -10;
  const int H = h->e->cfg.image_h, W = h->e->cfg.image_w;
  std::vector<const float*> ptrs(n > 0 ? n : 0);
  std::vector<int> hs(ptrs.size(), H), ws(ptrs.size(), W);
  for (size_t k = 0; k < ptrs.size(); ++k) ptrs[k] = imgs ? imgs + k * (size_t)3 * H * W : nullptr;
  return pxr_set_image_prompts_sized(h, ptrs.data(), hs.data(), ws.data(), n, weights);
}

// The polygon drawer's shapes (PixelDrawer.encode_image, pixeldrawer.py:200-304): polygon k has the vertices
// xy[offsets[k] .. offsets[k + 1]) (host [total_vertices, 2]), in draw order.  Copied; before pxr_finalize.
int pxr_set_polygons(pxr_handle h, const float* xy, const int* offsets, int n) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_POLYGON) throw EngineError(-76, "pxr_set_polygons: not a polygon-drawer engine");
    if (e->finalized) throw EngineError(-12, "pxr_set_polygons: the polygons cannot change after pxr_finalize");
    if (n < 1) throw EngineError(-77, "pxr_set_polygons: n = " + std::to_string(n) + ", at least one polygon is needed");
    if (!xy || !offsets) throw EngineError(-10, "pxr_set_polygons: null pointer");
    if (offsets[0] != 0) throw EngineError(-77, "pxr_set_polygons: offsets[0] must be 0");
    for (int k = 0; k < n; ++k) {
      const int nv = offsets[k + 1] - offsets[k];
      if (nv < 3 || nv > 8)
        throw EngineError(-77, "pxr_set_polygons: polygon " + std::to_string(k) + " has " + std::to_string(nv) +
                                   " vertices; 3 to 8 are supported");
    }
    const int nv = offsets[n];
    for (int i = 0; i < 2 * nv; ++i)
      if (!std::isfinite(xy[i]))
        throw EngineError(-77, "pxr_set_polygons: vertex " + std::to_string(i / 2) + " has a non-finite coordinate");
    e->poly_xy.assign(xy, xy + 2 * nv);
    e->poly_off.assign(offsets, offsets + n + 1);
  });
}

// The line drawer's shape (LineDrawer.load_model, linedrawer.py:44-126): n_paths open paths of n_segments cubics, widths
// clamped to [1, max_width] by clip_z, the paper colour optimised only when paper_trainable.  Before pxr_finalize.
int pxr_set_strokes(pxr_handle h, int n_paths, int n_segments, float max_width, int paper_trainable) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_STROKES) throw EngineError(-79, "pxr_set_strokes: not a line-drawer engine");
    if (e->finalized) throw EngineError(-12, "pxr_set_strokes: the strokes cannot change after pxr_finalize");
    if (n_paths < 1 || n_segments < 1)
      throw EngineError(-80, "pxr_set_strokes: n_paths = " + std::to_string(n_paths) + ", n_segments = " +
                                 std::to_string(n_segments) + "; at least one of each is needed");
    if (!std::isfinite(max_width) || !(max_width > 0.f))
      throw EngineError(-80, "pxr_set_strokes: max_width must be finite and positive");
    e->stroke_paths = n_paths;
    e->stroke_segments = n_segments;
    e->stroke_max_width = max_width;
    e->stroke_paper = paper_trainable ? 1 : 0;
  });
}

// The vdiff U-Net's size (VdiffDrawer's gen_width / gen_height, vdiff.py:55-58): x, v and the optimiser state are
// [1, 3, gen_h, gen_w]; the image is the canvas-size window centred in it.  Before pxr_finalize; without it gen = canvas.
int pxr_vdiff_set_gen_size(pxr_handle h, int gen_h, int gen_w) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_VDIFF) throw EngineError(-59, "pxr_vdiff_set_gen_size: not a vdiff engine");
    if (e->finalized) throw EngineError(-12, "pxr_vdiff_set_gen_size: the U-Net size cannot change after pxr_finalize");
    if (gen_h < 64 || gen_w < 64 || gen_h % 64 || gen_w % 64)
      throw EngineError(-55, "pxr_vdiff_set_gen_size: " + std::to_string(gen_h) + " x " + std::to_string(gen_w) +
                                 "; the U-Net's sides must be multiples of 64 (six 2x down-samplings)");
    if (gen_h < e->cfg.image_h || gen_w < e->cfg.image_w)
      throw EngineError(-55, "pxr_vdiff_set_gen_size: " + std::to_string(gen_h) + " x " + std::to_string(gen_w) +
                                 " is smaller than the canvas " + std::to_string(e->cfg.image_h) + " x " +
                                 std::to_string(e->cfg.image_w));
    e->vd_gen_h = gen_h;
    e->vd_gen_w = gen_w;
  });
}

int pxr_set_synth_iteration(pxr_handle h, int iter) {
  PXR_TRY(h, h->e->synth_iter = iter);
}

int pxr_synth(pxr_handle h, const float* z, float* out_img) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (z) PXR_CUDA(cudaMemcpyAsync(e->z_buf, z, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    e->filtered_valid = false;  // the per-op path sees the drawer's image; filters live in the fused iteration
    e->forward_drawer();
    e->check_launch("synth");
    if (out_img)
      PXR_CUDA(cudaMemcpyAsync(out_img, e->img, sizeof(float) * 3 * e->cfg.image_h * e->cfg.image_w,
                               cudaMemcpyDeviceToDevice, e->st));
  });
}

// model.encode(init_tensor)[0] (VqganDrawer.init_from_tensor / reapply_from_tensor / get_z_from_tensor, vqgan.py:174-185):
// img device fp32 [3, H, W] in [-1, 1] -> z_out device fp32 [z_channels, h, w] = the codebook rows nearest to
// quant_conv(encoder(img)).  Needs the checkpoint's encoder.* / quant_conv.* tensors (loaded before pxr_finalize).
namespace {
void vqgan_encode(Engine* e, const char* what, const float* img, const float* noise, float* z_out) {
  if (e->cfg.drawer != PXR_DRAWER_VQGAN) throw EngineError(-67, std::string(what) + ": not a VQGAN engine");
  if (!e->have_encoder) throw EngineError(-67, std::string(what) + ": the loaded VQGAN weights carry no encoder.* tensors");
  if (e->vq_gumbel && !noise)
    throw EngineError(-67, std::string(what) + ": the loaded VQGAN is a GumbelVQ (codebook quantize.embed.weight); its "
                                               "encoder needs Gumbel noise: call pxr_vqgan_encode_gumbel");
  if (!e->vq_gumbel && noise)
    throw EngineError(-67, std::string(what) + ": the loaded VQGAN quantises by nearest code (codebook "
                                               "quantize.embedding.weight), not by Gumbel noise: call pxr_vqgan_encode");
  if (!img || !z_out) throw EngineError(-10, std::string(what) + ": null pointer");
  PXR_CUDA(cudaMemcpyAsync(e->enc_img, img, sizeof(float) * 3 * e->cfg.image_h * e->cfg.image_w, cudaMemcpyDeviceToDevice, e->st));
  if (noise)
    PXR_CUDA(cudaMemcpyAsync(e->enc_noise, noise, sizeof(float) * e->cfg.n_embed * (e->z_numel / e->cfg.z_channels),
                             cudaMemcpyDeviceToDevice, e->st));
  e->run(e->enc_fwd);
  e->check_launch("vqgan encode");
  PXR_CUDA(cudaMemcpyAsync(z_out, e->enc_z, sizeof(float) * e->z_numel, cudaMemcpyDeviceToDevice, e->st));
}
}  // namespace

int pxr_vqgan_encode(pxr_handle h, const float* img, float* z_out) {
  PXR_TRY(h, { vqgan_encode(h->e, "pxr_vqgan_encode", img, nullptr, z_out); });
}

int pxr_vqgan_encode_gumbel(pxr_handle h, const float* img, const float* noise, float* z_out) {
  PXR_TRY(h, {
    if (!noise) throw EngineError(-10, "pxr_vqgan_encode_gumbel: null noise pointer");
    vqgan_encode(h->e, "pxr_vqgan_encode_gumbel", img, noise, z_out);
  });
}

int pxr_set_color_jitter(pxr_handle h, float p, float saturation, float hue) {
  PXR_TRY(h, {
    if (!(p >= 0.f && p <= 1.f) || saturation < 0.f || saturation > 1.f || hue < 0.f || hue > 0.5f)
      throw EngineError(-62, "pxr_set_color_jitter: p in [0,1], saturation in [0,1], hue in [0,0.5]");
    h->e->cj_p = p;
    h->e->cj_sat = saturation;
    h->e->cj_hue = hue;
  });
}

int pxr_make_cutouts(pxr_handle h, const float* img, const pxr_cut_params* p, int iter, float* out_batch) {
  return pxr_make_cutouts_set(h, 0, img, p, iter, out_batch);
}

int pxr_cutout_sets(pxr_handle h, int* cut_sizes) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (!cut_sizes) throw EngineError(-10, "pxr_cutout_sets: null cut_sizes");
    for (int s = 0; s < 4; ++s) cut_sizes[s] = s < e->n_sets() ? e->sets[s].cs : 0;
    return e->n_sets();
  });
}

int pxr_make_cutouts_set(pxr_handle h, int set, const float* img, const pxr_cut_params* p, int iter, float* out_batch) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (set < 0 || set >= e->n_sets()) throw EngineError(-83, "bad cutout set index");
    if (img) {
      PXR_CUDA(cudaMemcpyAsync(e->img, img, sizeof(float) * 3 * e->cfg.image_h * e->cfg.image_w,
                               cudaMemcpyDeviceToDevice, e->st));
      e->filtered_valid = false;
    }
    const Engine::CutSet& K = e->sets[set];
    e->prepare_cut_params(set, p, iter);
    e->encode_image_prompts(set);
    e->forward_cutouts(set);
    if (out_batch)
      PXR_CUDA(cudaMemcpyAsync(out_batch, K.batch, sizeof(float) * e->n_local * 3 * K.cs * K.cs, cudaMemcpyDeviceToDevice,
                               e->st));
  });
}

int pxr_encode_image(pxr_handle h, int clip_idx, const float* batch, float* out_embeds) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    Engine::CutSet& K = e->sets[e->set_of[clip_idx]];
    if (batch) {
      // a caller-provided batch at the perceptor's resolution: recompute its global range exactly like
      // CLIP_Base.preprocess does
      const long long n = (long long)e->n_local * 3 * K.cs * K.cs;
      PXR_CUDA(cudaMemcpyAsync(K.batch, batch, sizeof(float) * n, cudaMemcpyDeviceToDevice, e->st));
      const int np_ = K.n_parts < 1024 ? K.n_parts : 1024;
      pxr::minmax_partials(K.batch, n, np_, K.part_min, K.part_max, K.part_imin, K.part_imax, e->st);
      pxr::minmax_reduce(nullptr, K.part_min, K.part_max, K.part_imin, K.part_imax, np_, K.range, K.irange, e->st);
      e->launches += 2;
      K.cut = true;
    } else if (e->n_sets() > 1 && !K.cut) {
      throw EngineError(-83, "perceptor " + std::to_string(clip_idx) + " reads cutout set " +
                                 std::to_string(e->set_of[clip_idx]) + " (" + std::to_string(K.cs) +
                                 " px), which has not been cut since the last backward: pxr_make_cutouts_set first");
    }
    e->forward_clip(clip_idx);
    auto& C = e->clip[clip_idx];
    // unit-norm embeddings (slip.py:66) are produced by the loss kernel; run it when prompts exist
    if (C.n_prompts > 0) {
      PXR_CUDA(cudaMemsetAsync(e->losses_dev + C.loss_offset, 0, sizeof(float) * C.n_prompts, e->st));
      e->loss_clip(clip_idx);
    }
    if (out_embeds)
      PXR_CUDA(cudaMemcpyAsync(out_embeds, C.n_prompts > 0 ? C.e_unit : C.e, sizeof(float) * C.B * C.c.out_dim,
                               cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_prompt_loss(pxr_handle h, int clip_idx, const float* embeds, float* out_losses) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (clip_idx < 0 || clip_idx >= e->cfg.n_clip) throw EngineError(-14, "bad clip index");
    auto& C = e->clip[clip_idx];
    if (embeds) {
      // Foreign embeddings (not the ones this engine's encode_image produced): scored as given into SCRATCH buffers --
      // the perceptor's own un-normalised embeddings and their gradient (C.e / C.de, which pxr_backward consumes together
      // with the saved ViT activations) stay what the last encode_image / prompt_loss pair left there.
      if (C.n_prompts == 0) throw EngineError(-70, "no prompts set for perceptor " + std::to_string(clip_idx));
      const size_t n = (size_t)C.B * C.c.out_dim;
      if (!C.scratch) C.scratch = e->dalloc<float>(3 * n + n);  // e | e_unit | de | de16 (fp16 in the last n floats' space)
      float *se = C.scratch, *su = C.scratch + n, *sd = C.scratch + 2 * n;
      pxr::act_t* sd16 = reinterpret_cast<pxr::act_t*>(C.scratch + 3 * n);
      float* sl = e->losses_scratch;
      PXR_CUDA(cudaMemcpyAsync(se, embeds, sizeof(float) * n, cudaMemcpyDeviceToDevice, e->st));
      PXR_CUDA(cudaMemsetAsync(sl, 0, 64 * sizeof(float), e->st));
      pxr::prompt_loss(se, C.B, C.c.out_dim, C.prompts, C.pweights, C.pstops, C.pslot, C.pinv, C.n_rows, e->cfg.cutn, e->S, su,
                       sl, sd, sd16, C.ploss_part, C.ploss_count, e->st);
      e->launches += 1;
      if (out_losses)
        PXR_CUDA(cudaMemcpyAsync(out_losses, sl, sizeof(float) * C.n_prompts, cudaMemcpyDeviceToDevice, e->st));
      return 0;
    }
    PXR_CUDA(cudaMemsetAsync(e->losses_dev + C.loss_offset, 0, sizeof(float) * C.n_prompts, e->st));
    e->loss_clip(clip_idx);
    if (out_losses)
      PXR_CUDA(cudaMemcpyAsync(out_losses, e->losses_dev + C.loss_offset, sizeof(float) * C.n_prompts,
                               cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_backward(pxr_handle h, float* z_grad) {
  PXR_TRY(h, {
    Engine* e = h->e;
    e->backward_all();
    if (z_grad)
      PXR_CUDA(cudaMemcpyAsync(z_grad, e->z_grad, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_step(pxr_handle h, float* z, float lr, int iter) {
  PXR_TRY(h, {
    Engine* e = h->e;
    (void)iter;
    e->step(lr);
    if (z) PXR_CUDA(cudaMemcpyAsync(z, e->z_buf, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_iterate(pxr_handle h, float* z, float lr, int iter, const pxr_cut_params* p, float* out_losses_host) {
  if (h && p && h->e->n_sets() > 1) {
    h->e->err = "pxr_iterate: this session has " + std::to_string(h->e->n_sets()) +
                " cutout sets; pass their cutout parameters to pxr_iterate_sets (one pxr_cut_params per set)";
    return -69;
  }
  return pxr_iterate_sets(h, z, lr, iter, p, out_losses_host);
}

int pxr_iterate_sets(pxr_handle h, float* z, float lr, int iter, const pxr_cut_params* p, float* out_losses_host) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (z) PXR_CUDA(cudaMemcpyAsync(e->z_buf, z, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    if (e->batches > 1 && p) throw EngineError(-63, "batches > 1 draws its cutout parameters in the engine: pass p = NULL");
    e->vd_iter_request = iter;
    e->synth_iter = iter;
    for (int b = 0; b < e->batches; ++b) {
      // every pass is one ascend_txt + backward (pixray.py:1464-1482): fresh augmentations, gradients accumulate in z.grad;
      // checkdrop and the reported loss vector use the FIRST pass (`if i == 0`, pixray.py:1466)
      e->rng_iter = b == 0 ? 0 : iter + b * (1 << 20);
      for (int s = 0; s < e->n_sets(); ++s) e->prepare_cut_params(s, p ? p + s : nullptr, iter);
      if (b == 0) PXR_CUDA(cudaMemsetAsync(e->losses_dev, 0, 64 * sizeof(float), e->st));
      else PXR_CUDA(cudaMemsetAsync(e->losses_scratch, 0, 64 * sizeof(float), e->st));
      float* keep = e->losses_dev;
      if (b > 0) e->losses_dev = e->losses_scratch;  // later passes must not disturb the first pass's loss vector
      try {
        for (int s = 0; s < e->n_sets(); ++s) e->encode_image_prompts(s);
        if (b == 0) {
          e->forward_drawer();  // same z: the image of the later passes is the same image
          if (!e->filters.empty()) e->filters_forward(iter);
        }
        if (e->any_spot(1) || e->any_spot(0)) {  // spot / spot-off prompts: their own masked cutout batches (pixray.py:1262-1293)
          Engine::CutSet& K = e->sets[0];
          pxr::pool_forward(e->cur_cut_img(), e->cur_cut_h(), e->cur_cut_w(), K.cs, K.pooled, K.pool_argmax, e->st);
          e->launches += 1;
          bool acc = false;
          acc |= e->spot_pass(1, acc);
          acc |= e->spot_pass(0, acc);
          e->spot_accumulated = acc;
        }
        for (int s = 0; s < e->n_sets(); ++s) {  // each set is cut from the same image (pixray.py:1266-1268)
          e->forward_cutouts(s);
          for (int i = 0; i < e->cfg.n_clip; ++i) {
            if (e->set_of[i] != s) continue;
            e->forward_clip(i);
            e->loss_clip(i);
          }
        }
        e->backward_all();
      } catch (...) {
        e->losses_dev = keep;
        e->rng_iter = 0;
        throw;
      }
      e->losses_dev = keep;
      if (e->batches > 1) {
        pxr::accumulate_f32(e->z_grad, e->z_grad_acc, e->z_numel, b > 0, e->st);
        e->launches += 1;
      }
    }
    e->rng_iter = 0;
    if (e->managed) e->step_managed(iter);
    else e->step(lr);
    if (z) PXR_CUDA(cudaMemcpyAsync(z, e->z_buf, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    if (out_losses_host) {
      PXR_CUDA(cudaMemcpyAsync(e->losses_host, e->losses_dev, 64 * sizeof(float), cudaMemcpyDeviceToHost, e->st));
      PXR_CUDA(cudaStreamSynchronize(e->st));
      memcpy(out_losses_host, e->losses_host, sizeof(float) * e->num_losses());
    }
  });
}

// train()'s control decisions on the device (checkdrop, scheduled learning-rate drops, auto-stop; pixray.py:1090-1109,
// 1464-1512).  After this call pxr_iterate ignores its `lr` argument: the engine owns the learning rate, the Adam step
// counter and the drop bookkeeping, and pxr_poll_status reports them without synchronising.  n_drops <= 16.
int pxr_set_schedule(pxr_handle h, float base_lr, int iter_drop_delay, int max_loss_drops, int auto_stop, const int* drops,
                     int n_drops) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (n_drops < 0 || n_drops > 16 || (n_drops > 0 && !drops)) throw EngineError(-64, "pxr_set_schedule: at most 16 scheduled drops");
    if (!(base_lr > 0.f) || iter_drop_delay < 0 || max_loss_drops < 0) throw EngineError(-64, "pxr_set_schedule: bad arguments");
    e->drop_cfg.base_lr = base_lr;
    e->drop_cfg.iter_drop_delay = iter_drop_delay;
    e->drop_cfg.max_loss_drops = max_loss_drops;
    e->drop_cfg.auto_stop = auto_stop ? 1 : 0;
    e->drop_cfg.n_sched = n_drops;
    for (int i = 0; i < n_drops; ++i) e->drop_cfg.sched[i] = drops[i];
    e->managed = true;
    PXR_CUDA(cudaMemsetAsync(e->adam_m, 0, e->z_numel * sizeof(float), e->st));
    PXR_CUDA(cudaMemsetAsync(e->adam_v, 0, e->z_numel * sizeof(float), e->st));
    if (e->opt_p) PXR_CUDA(cudaMemsetAsync(e->opt_p, 0, e->z_numel * sizeof(float), e->st));
    e->write_initial_drop_state();
  });
}

// Non-blocking: the record the last COMPLETED iteration left in pinned memory.  Returns 1 when there is no consistent
// record yet (no managed iteration has finished, or the kernel is mid-write: poll again), 0 on success.
int pxr_poll_status(pxr_handle h, pxr_status* out) {
  pxr::DropStatus* s = h->e->drop_status;
  if (!s || !out) return -10;
  const int e1 = s->seq_end;
  std::atomic_thread_fence(std::memory_order_acquire);
  pxr_status r;
  r.iter = s->iter;
  r.loss_sum = s->loss_sum;
  r.best_loss = s->best_loss;
  r.best_iter = s->best_iter;
  r.num_loss_drop = s->num_loss_drop;
  r.stopped = s->stopped;
  r.rebuilt = s->rebuilt;
  r.lr = s->lr;
  r.n_losses = s->n_losses;
  for (int k = 0; k < 64; ++k) r.losses[k] = s->losses[k];
  std::atomic_thread_fence(std::memory_order_acquire);
  const int e0 = s->seq_begin;
  if (e1 == 0 || e0 != e1) return 1;
  *out = r;
  return 0;
}

int pxr_set_batches(pxr_handle h, int batches) {
  PXR_TRY(h, {
    if (batches < 1 || batches > 64) throw EngineError(-65, "batches must be in [1, 64]");
    h->e->batches = batches;
  });
}

// z.grad for the next pxr_step from the caller (the plugin loop accumulates the gradients of several passes itself)
int pxr_set_z_grad(pxr_handle h, const float* z_grad) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!z_grad) throw EngineError(-10, "pxr_set_z_grad: null gradient");
    PXR_CUDA(cudaMemcpyAsync(e->z_grad, z_grad, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  });
}

// One full iteration with a CUDA-event pair around every op (engine stream).  out[0] = ms in gemm_tc_kernel launches,
// out[1] = number of those launches, out[2] = their algorithmic FLOPs, out[3] = ms in all other kernels,
// out[4] = number of other launches, out[5] = ms of the whole iteration (first event -> last event).
int pxr_profile_iteration(pxr_handle h, float* z, float lr, int iter, double* out6) {
  return pxr_profile_iteration2(h, z, lr, iter, out6, nullptr);
}

int pxr_profile_iteration2(pxr_handle h, float* z, float lr, int iter, double* out6, double* tensor_bytes) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (z) PXR_CUDA(cudaMemcpyAsync(e->z_buf, z, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    for (int s = 0; s < e->n_sets(); ++s) e->prepare_cut_params(s, nullptr, iter);
    PXR_CUDA(cudaMemsetAsync(e->losses_dev, 0, 64 * sizeof(float), e->st));
    e->prof.clear();
    e->profiling = true;
    cudaEvent_t t0;
    cudaEvent_t t1;
    PXR_CUDA(cudaEventCreate(&t0));
    PXR_CUDA(cudaEventCreate(&t1));
    PXR_CUDA(cudaEventRecord(t0, e->st));
    e->forward_drawer();
    for (int s = 0; s < e->n_sets(); ++s) {
      e->forward_cutouts(s);
      for (int i = 0; i < e->cfg.n_clip; ++i) {
        if (e->set_of[i] != s) continue;
        e->forward_clip(i);
        e->loss_clip(i);
      }
    }
    e->backward_all();
    e->step(lr);
    PXR_CUDA(cudaEventRecord(t1, e->st));
    e->profiling = false;
    PXR_CUDA(cudaStreamSynchronize(e->st));
    for (int i = 0; i < 6; ++i) out6[i] = 0;
    double tb = 0;
    FILE* dump = nullptr;
    if (const char* path = getenv("PXR_PROFILE_DUMP")) dump = fopen(path, "w");
    if (dump) fprintf(dump, "op,ms,gflop,launches\n");
    for (auto& r : e->prof) {
      float ms = 0;
      PXR_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
      if (dump) fprintf(dump, "%s,%.4f,%.3f,%d\n", r.name.empty() ? "op" : r.name.c_str(), ms, r.flops * 1e-9, r.launches);
      if (r.flops > 0) {
        out6[0] += ms;
        out6[1] += r.launches;
        out6[2] += r.flops;
        tb += r.bytes;
      } else {
        out6[3] += ms;
        out6[4] += r.launches;
      }
      cudaEventDestroy(r.a);
      cudaEventDestroy(r.b);
    }
    e->prof.clear();
    if (dump) fclose(dump);
    float tot = 0;
    PXR_CUDA(cudaEventElapsedTime(&tot, t0, t1));
    out6[5] = tot;
    if (tensor_bytes) *tensor_bytes = tb;
    cudaEventDestroy(t0);
    cudaEventDestroy(t1);
    if (z) PXR_CUDA(cudaMemcpyAsync(z, e->z_buf, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_vdiff_set_schedule(pxr_handle h, const float* steps, const float* alphas, const float* sigmas, int n) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_VDIFF) throw EngineError(-59, "not a vdiff engine");
    if (n < 1 || !steps || !alphas || !sigmas) throw EngineError(-59, "pxr_vdiff_set_schedule: empty schedule");
    e->vd_steps.assign(steps, steps + n);
    e->vd_alphas.assign(alphas, alphas + n);
    e->vd_sigmas.assign(sigmas, sigmas + n);
  });
}

int pxr_vdiff_set_clip_embed(pxr_handle h, const float* embed, int D) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_VDIFF || !e->finalized) throw EngineError(-59, "not a finalized vdiff engine");
    if (D != 512) throw EngineError(-59, "cc12m_1 is conditioned on a 512-wide CLIP embedding");
    // cc12m_1.py:244: F.normalize(clip_embed) * sqrt(D)
    std::vector<float> ce(embed, embed + D);
    double s = 0;
    for (float v : ce) s += (double)v * v;
    const double k = std::sqrt((double)D) / std::max(std::sqrt(s), 1e-12);
    for (float& v : ce) v = (float)(v * k);
    PXR_CUDA(cudaMemcpyAsync(e->vd_h0, ce.data(), sizeof(float) * D, cudaMemcpyHostToDevice, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
    e->vd_have_embed = true;
  });
}

int pxr_vdiff_set_iteration(pxr_handle h, int i) {
  h->e->vd_iter_request = i;
  return 0;
}

int pxr_vdiff_renoise(pxr_handle h, float* z, int i, const float* noise) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (e->cfg.drawer != PXR_DRAWER_VDIFF) throw EngineError(-59, "not a vdiff engine");
    const int n = (int)e->vd_steps.size();
    if (i < 0 || i >= n) throw EngineError(-59, "pxr_vdiff_renoise: iteration outside the schedule");
    if (z) PXR_CUDA(cudaMemcpyAsync(e->z_buf, z, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    if (i < n - 1) {  // sampling.py:24-37 with eta = 1
      const double a = e->vd_alphas[i], s = e->vd_sigmas[i], a1 = e->vd_alphas[i + 1], s1 = e->vd_sigmas[i + 1];
      const double ddim = std::sqrt(s1 * s1 / (s * s)) * std::sqrt(std::max(0.0, 1.0 - a * a / (a1 * a1)));
      const double adj = std::sqrt(std::max(0.0, s1 * s1 - ddim * ddim));
      pxr::vd_renoise(e->z_buf, e->vd_pred, e->vd_v, noise, (float)a, (float)s, (float)a1, (float)adj, (float)ddim,
                      e->z_numel, e->st);
      e->launches += 1;
    }
    if (z) PXR_CUDA(cudaMemcpyAsync(z, e->z_buf, e->z_numel * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_add_aux_loss(pxr_handle h, int kind, float weight, const float* params, int n_params) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (e->num_losses() + e->aux_width(kind) > 64)
      throw EngineError(-16, "at most 64 losses (prompts + auxiliary, a cutout-space loss once per cutout set) in total");
    auto need = [&](int n, const char* what) {
      if (n_params < n || !params) throw EngineError(-80, std::string("pxr_add_aux_loss: ") + what);
    };
    Engine::AuxLoss a;
    a.kind = kind;
    a.weight = weight;
    a.prm.assign(params, params + (n_params > 0 ? n_params : 0));
    switch (kind) {
      case PXR_LOSS_SYMMETRY: need(1, "symmetry needs {symmetry_weight}"); break;
      case PXR_LOSS_SATURATION: need(1, "saturation needs {saturation_weight}"); break;
      case PXR_LOSS_PALETTE:
        need(4, "palette needs {palette_weight, r,g,b, ...}");
        if ((n_params - 1) % 3) throw EngineError(-80, "pxr_add_aux_loss: palette colours come as r,g,b triples");
        a.dev = e->upload(std::vector<float>(params + 1, params + n_params));
        a.n_dev = n_params - 1;
        break;
      case PXR_LOSS_SMOOTHNESS: {
        need(3, "smoothness needs {smoothness_weight, type, spacing[, edge_order[, n, taps[n * n]]]}");
        if (params[1] < 0 || params[1] > 2 || params[2] <= 0) throw EngineError(-80, "pxr_add_aux_loss: smoothness type in {0,1,2}, spacing > 0");
        const int order = n_params > 3 ? (int)params[3] : 1;
        if (n_params > 3 && params[3] != 1.f && params[3] != 2.f)
          throw EngineError(-80, "pxr_add_aux_loss: smoothness edge_order must be 1 or 2 (torch.gradient)");
        const float nf = n_params > 4 ? params[4] : 0.f;
        if (nf < 0 || nf != std::floor(nf) || nf > 1024)
          throw EngineError(-80, "pxr_add_aux_loss: smoothness blur tap count must be an integer in [0, 1024] (kernel size >= 0)");
        const int n = (int)nf;
        if (n_params != (n_params > 4 ? 5 + n * n : n_params))
          throw EngineError(-80, "pxr_add_aux_loss: smoothness blur needs n * n taps after n");
        int min_cs = e->cfg.cut_size;
        for (const Engine::CutSet& K : e->sets) min_cs = std::min(min_cs, K.cs);
        const int cs2 = min_cs - (n ? n - 1 : 0);
        if (cs2 < order + 1)
          throw EngineError(-80, "pxr_add_aux_loss: smoothness blur leaves " + std::to_string(cs2) + " pixels per cutout side; "
                                 "torch.gradient with edge_order " + std::to_string(order) + " needs at least " +
                                 std::to_string(order + 1));
        if (n) {
          // GaussianSmoothing's kernel is u (x) u with sum(u) = 1: apply it as two 1-D passes of the row sums
          const float* K = params + 5;
          std::vector<double> u(n, 0.0);
          double kmax = 0.0, total = 0.0;
          for (int i = 0; i < n * n; ++i) {
            if (!std::isfinite(K[i]) || K[i] < 0.f)
              throw EngineError(-80, "pxr_add_aux_loss: smoothness blur taps must be finite and >= 0 (std > 0)");
            u[i / n] += K[i];
            kmax = std::max(kmax, (double)K[i]);
            total += K[i];
          }
          if (!(std::fabs(total - 1.0) <= 1e-4))
            throw EngineError(-80, "pxr_add_aux_loss: smoothness blur taps must sum to 1");
          for (int i = 0; i < n * n; ++i)
            if (std::fabs(K[i] - u[i / n] * u[i % n]) > 1e-5 * kmax)
              throw EngineError(-80, "pxr_add_aux_loss: smoothness blur taps must be separable (an outer product u u^T)");
          a.dev = e->upload(std::vector<float>(u.begin(), u.end()));
          a.n_dev = n;
          for (Engine::CutSet& K : e->sets) {
            if (K.aux_blur) continue;
            const size_t sz = (size_t)e->n_local * 3 * K.cs * K.cs;
            K.aux_blur = e->dalloc<float>(sz);
            K.aux_g_blur = e->dalloc<float>(sz);
            K.aux_blur_tmp = e->dalloc<float>(sz);
          }
        }
        break;
      }
      case PXR_LOSS_EDGE: {
        need(9, "edge needs {edge_color_weight, global_color_weight, left,right,upper,lower, r,g,b[, mode, target, mask]}");
        const int mode = n_params > 9 ? (int)params[9] : 0;
        if (n_params > 9 && (params[9] != (float)mode || mode < 0 || mode > 3))
          throw EngineError(-80, "pxr_add_aux_loss: edge mode is 0 (colour), 1 (target image), 2 (mask) or 3 (both)");
        const size_t hw = (size_t)e->cfg.image_h * e->cfg.image_w;
        const size_t extra = ((mode & 1) ? 3 * hw : 0) + ((mode & 2) ? hw : 0);
        if (n_params > 9 && (size_t)n_params != 10 + extra)
          throw EngineError(-80, "pxr_add_aux_loss: edge target must be [3, " + std::to_string(e->cfg.image_h) + ", " +
                                 std::to_string(e->cfg.image_w) + "] and mask [" + std::to_string(e->cfg.image_h) + ", " +
                                 std::to_string(e->cfg.image_w) + "] floats (the image the loss reads)");
        if (extra) {
          a.dev = e->upload(std::vector<float>(params + 10, params + n_params));
          a.n_dev = (int)extra;
          a.prm.resize(10);  // the arrays live on the device
        }
        break;
      }
      case PXR_LOSS_GAUSSIAN:
        need(6, "gaussian needs {gaussian_weight, std_y, std_x, R,G,B}");
        if (params[1] <= 0 || params[2] <= 0) throw EngineError(-80, "pxr_add_aux_loss: gaussian std must be positive");
        break;
      case PXR_LOSS_AESTHETIC:
        need(3, "aesthetic needs {target, bias, w[D]}");
        a.dev = e->upload(std::vector<float>(params + 2, params + n_params));
        a.n_dev = n_params - 2;
        break;
      default: throw EngineError(-80, "pxr_add_aux_loss: unknown loss kind");
    }
    e->aux.push_back(std::move(a));
  });
}

// Filters (args.filters = "name:weight,...", pixray.py:651-668; applied to drawer.synth's output before MakeCutouts,
// pixray.py:1203-1222).  params (host floats) by kind:
//   TILER     {}                                                       filters/tiler.py: torch.roll by random (h, w) shifts
//   WALLPAPER {type (0 none, 1 shift, 2 horizontal, 3 vertical), edge_match}   filters/wallpaper.py
//   LOOKUP    {lookup_beta, r0,g0,b0, r1,g1,b1, ...} palette in [0,1]   filters/colorlookup.py
// Each filter owns one entry at the FRONT of the loss vector (0 for the loss-free ones), in the order added.
int pxr_add_filter(pxr_handle h, int kind, float weight, const float* params, int n_params) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (e->num_losses() >= 64) throw EngineError(-16, "at most 64 losses (filters + prompts + auxiliary) in total");
    Engine::Filter F{};
    F.kind = kind;
    F.weight = weight;
    if (kind == PXR_FILTER_TILER) {
    } else if (kind == PXR_FILTER_WALLPAPER) {
      if (n_params < 2 || !params) throw EngineError(-74, "wallpaper needs {type, edge_match}");
      F.wp_type = (int)params[0];
      F.em = (int)params[1];
      if (F.wp_type < 0 || F.wp_type > 3 || F.em < 0) throw EngineError(-74, "wallpaper: type in 0..3, edge_match >= 0");
    } else if (kind == PXR_FILTER_LOOKUP) {
      if (n_params < 4 || !params || (n_params - 1) % 3) throw EngineError(-74, "lookup needs {lookup_beta, r,g,b, ...}");
      F.beta = params[0];
      F.pal = e->upload(std::vector<float>(params + 1, params + n_params));
      F.n_col = (n_params - 1) / 3;
    } else {
      throw EngineError(-74, "pxr_add_filter: unknown filter kind");
    }
    e->filters.push_back(F);
    try {
      e->rebuild_filters();
    } catch (...) {
      e->filters.pop_back();
      e->rebuild_filters();
      throw;
    }
  });
}

int pxr_clear_filters(pxr_handle h) {
  PXR_TRY(h, {
    h->e->filters.clear();
    h->e->filtered_valid = false;
    h->e->rebuild_filters();
  });
}

// Explicit (rand_h, rand_w) of one filter for replays / parity tests; negative = engine-drawn again.
int pxr_set_filter_shifts(pxr_handle h, int filter_idx, int rand_h, int rand_w) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (filter_idx < 0 || filter_idx >= (int)e->filters.size()) throw EngineError(-74, "pxr_set_filter_shifts: bad filter index");
    e->filters[filter_idx].fixed_h = rand_h;
    e->filters[filter_idx].fixed_w = rand_w;
  });
}

int pxr_add_anchor(pxr_handle h, int kind, float weight, const float* ref, long long n) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (kind < PXR_ANCHOR_SPHERICAL || kind > PXR_ANCHOR_PIX) throw EngineError(-82, "pxr_add_anchor: unknown kind");
    if (!ref) throw EngineError(-82, "pxr_add_anchor: null reference");
    const long long want = kind == PXR_ANCHOR_PIX ? n : (long long)e->z_numel;
    if (n != want || n <= 0) throw EngineError(-82, "pxr_add_anchor: a latent anchor has the latent's element count");
    if (e->num_losses() + 1 > 64) throw EngineError(-16, "at most 64 losses (prompts + anchors + auxiliary) in total");
    Engine::Anchor a;
    a.kind = kind;
    a.weight = weight;
    a.n = (size_t)n;
    a.ref = e->dalloc<float>(a.n);
    PXR_CUDA(cudaMemcpyAsync(a.ref, ref, sizeof(float) * a.n, cudaMemcpyDefault, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
    e->anchors.push_back(a);
  });
}

int pxr_clear_anchors(pxr_handle h) {
  PXR_TRY(h, {
    for (auto& a : h->e->anchors) h->e->dfree(a.ref);
    h->e->anchors.clear();
  });
}

int pxr_clear_aux_losses(pxr_handle h) {
  PXR_TRY(h, h->e->aux.clear());
}

int pxr_num_losses(pxr_handle h, int* out) {
  *out = h->e->num_losses();
  return 0;
}

int pxr_read_losses(pxr_handle h, float* out_host) {
  PXR_TRY(h, {
    Engine* e = h->e;
    PXR_CUDA(cudaMemcpyAsync(e->losses_host, e->losses_dev, 64 * sizeof(float), cudaMemcpyDeviceToHost, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
    memcpy(out_host, e->losses_host, sizeof(float) * e->num_losses());
  });
}

// a fresh instance of the current rule: state 0, t = 0; in managed mode the drop bookkeeping restarts too
void Engine::reset_opt_state() {
  PXR_CUDA(cudaMemsetAsync(adam_m, 0, z_numel * sizeof(float), st));
  PXR_CUDA(cudaMemsetAsync(adam_v, 0, z_numel * sizeof(float), st));
  if (opt_p) PXR_CUDA(cudaMemsetAsync(opt_p, 0, z_numel * sizeof(float), st));
  adam_t = 0;
  if (managed) write_initial_drop_state();  // a fresh session: best-loss tracking and the drop count restart too
}

int pxr_reset_optimizer(pxr_handle h) { PXR_TRY(h, h->e->reset_opt_state()); }

namespace {
const char* opt_name(int kind) {
  static const char* names[] = {"Adam", "AdamW", "Adagrad", "Adamax", "DiffGrad"};
  return kind >= 0 && kind < pxr::OPT_KINDS ? names[kind] : "unknown";
}
}  // namespace

static_assert(PXR_OPT_ADAM == pxr::OPT_ADAM && PXR_OPT_ADAMW == pxr::OPT_ADAMW && PXR_OPT_ADAGRAD == pxr::OPT_ADAGRAD &&
                  PXR_OPT_ADAMAX == pxr::OPT_ADAMAX && PXR_OPT_DIFFGRAD == pxr::OPT_DIFFGRAD,
              "the kernels' rule codes are the ABI's");

int pxr_set_optimizer(pxr_handle h, int kind) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->finalized) throw EngineError(-13, "call pxr_finalize first");
    if (kind < 0 || kind >= pxr::OPT_KINDS)
      throw EngineError(-93, "pxr_set_optimizer: unknown optimiser kind " + std::to_string(kind) +
                                 " (PXR_OPT_ADAM .. PXR_OPT_DIFFGRAD)");
    if (kind == PXR_OPT_DIFFGRAD && !e->opt_p) e->opt_p = e->dalloc<float>(e->z_numel);
    e->opt_kind = kind;
    e->reset_opt_state();
  });
}

// ---- checkpoint of the optimisation state (z, Adam m / v / step, the drop bookkeeping): resume = load + keep iterating
namespace {
struct StateHeader {
  uint32_t magic, version;
  int64_t z_numel;
  int32_t adam_t, managed, drop_parity, pad;
  pxr::DropState drop;
};
constexpr uint32_t kStateMagic = 0x50585253u;  // "PXRS"
// Version 1 (Adam): {header, z, m, v}.  Version 2 (every other rule): {header, kind, z, its two or three state arrays}.
struct StateKind {
  int32_t kind, pad;
};
int64_t state_payload_offset(int kind) { return (int64_t)sizeof(StateHeader) + (kind == PXR_OPT_ADAM ? 0 : (int64_t)sizeof(StateKind)); }
std::vector<float*> state_arrays(Engine* e, int kind) {
  std::vector<float*> a{e->z_buf, e->adam_m, e->adam_v};
  if (kind == PXR_OPT_DIFFGRAD) a.push_back(e->opt_p);
  return a;
}
}  // namespace

int pxr_state_size(pxr_handle h, int64_t* nbytes) {
  const int kind = h->e->opt_kind;
  *nbytes = state_payload_offset(kind) + (1 + pxr::opt_state_arrays(kind)) * h->e->z_numel * (int64_t)sizeof(float);
  return 0;
}

// host buffer of pxr_state_size bytes <- {header, [kind,] z, state arrays}.  Blocking.
int pxr_save_state(pxr_handle h, void* host_buf) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!host_buf) throw EngineError(-10, "pxr_save_state: null buffer");
    StateHeader hd{};
    hd.magic = kStateMagic;
    hd.version = e->opt_kind == PXR_OPT_ADAM ? 1 : 2;
    hd.z_numel = e->z_numel;
    hd.adam_t = e->adam_t;
    hd.managed = e->managed ? 1 : 0;
    hd.drop_parity = e->drop_parity;
    if (e->managed)
      PXR_CUDA(cudaMemcpyAsync(&hd.drop, e->drop_state + e->drop_parity, sizeof(pxr::DropState), cudaMemcpyDeviceToHost, e->st));
    char* out = static_cast<char*>(host_buf);
    const size_t zb = (size_t)e->z_numel * sizeof(float);
    char* payload = out + state_payload_offset(e->opt_kind);
    const std::vector<float*> arrays = state_arrays(e, e->opt_kind);
    for (size_t k = 0; k < arrays.size(); ++k)
      PXR_CUDA(cudaMemcpyAsync(payload + k * zb, arrays[k], zb, cudaMemcpyDeviceToHost, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
    memcpy(out, &hd, sizeof hd);
    if (hd.version == 2) {
      const StateKind sk{e->opt_kind, 0};
      memcpy(out + sizeof hd, &sk, sizeof sk);
    }
  });
}

// The inverse: the engine's z, Adam state and (when it was saved in managed mode and pxr_set_schedule was called here
// too) the learning-rate / best-loss / drop-count bookkeeping.  Blocking.
int pxr_load_state(pxr_handle h, const void* host_buf) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!host_buf) throw EngineError(-10, "pxr_load_state: null buffer");
    StateHeader hd;
    memcpy(&hd, host_buf, sizeof hd);
    if (hd.magic != kStateMagic || (hd.version != 1 && hd.version != 2))
      throw EngineError(-68, "pxr_load_state: not a pixray_b200 state blob");
    if (hd.z_numel != e->z_numel) throw EngineError(-68, "pxr_load_state: the blob belongs to a different latent shape");
    const char* in = static_cast<const char*>(host_buf);
    StateKind sk{PXR_OPT_ADAM, 0};
    if (hd.version == 2) memcpy(&sk, in + sizeof hd, sizeof sk);
    if (sk.kind == PXR_OPT_ADAM && hd.version == 2) throw EngineError(-68, "pxr_load_state: not a pixray_b200 state blob");
    if (sk.kind != e->opt_kind)
      throw EngineError(-68, std::string("pxr_load_state: the blob holds ") + opt_name(sk.kind) + " state, this session runs " +
                                 opt_name(e->opt_kind) + " (pxr_set_optimizer)");
    const size_t zb = (size_t)e->z_numel * sizeof(float);
    const char* payload = in + state_payload_offset(sk.kind);
    const std::vector<float*> arrays = state_arrays(e, sk.kind);
    for (size_t k = 0; k < arrays.size(); ++k)
      PXR_CUDA(cudaMemcpyAsync(arrays[k], payload + k * zb, zb, cudaMemcpyHostToDevice, e->st));
    e->adam_t = hd.adam_t;
    if (hd.managed && e->managed) {
      PXR_CUDA(cudaMemcpyAsync(e->drop_state + e->drop_parity, &hd.drop, sizeof(pxr::DropState), cudaMemcpyHostToDevice, e->st));
    }
    PXR_CUDA(cudaStreamSynchronize(e->st));
  });
}

int pxr_sync(pxr_handle h) { PXR_TRY(h, PXR_CUDA(cudaStreamSynchronize(h->e->st))); }

int pxr_num_kernel_launches(pxr_handle h, int64_t* out) {
  *out = h->e->launches;
  return 0;
}
int pxr_get_stream(pxr_handle h, void** out) {
  *out = h->e->st;
  return 0;
}
int pxr_z_numel(pxr_handle h, int64_t* out) {
  *out = h->e->z_numel;
  return 0;
}
int pxr_z_bounds(pxr_handle h, float* zmin, float* zmax) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (!e->zmin) throw EngineError(-18, "this drawer has no per-channel z bounds");
    PXR_CUDA(cudaMemcpyAsync(zmin, e->zmin, sizeof(float) * e->cfg.z_channels, cudaMemcpyDeviceToDevice, e->st));
    PXR_CUDA(cudaMemcpyAsync(zmax, e->zmax, sizeof(float) * e->cfg.z_channels, cudaMemcpyDeviceToDevice, e->st));
  });
}

int pxr_debug_read(pxr_handle h, const char* name, void* out, int64_t nbytes) {
  PXR_TRY(h, {
    Engine* e = h->e;
    auto it = e->dbg.find(name);
    if (it == e->dbg.end()) throw EngineError(-19, std::string("unknown debug buffer ") + name);
    if ((size_t)nbytes > it->second.second) throw EngineError(-19, "debug read larger than the buffer");
    PXR_CUDA(cudaMemcpyAsync(out, it->second.first, nbytes, cudaMemcpyDefault, e->st));
    PXR_CUDA(cudaStreamSynchronize(e->st));
  });
}

int pxr_test_conv_records(pxr_handle h, pxr_test_conv_rec* out, int max, int* count) {
  PXR_TRY(h, {
    const auto& log = h->e->conv_log;
    for (int i = 0; out && i < max && i < (int)log.size(); ++i) out[i] = log[i];
    if (count) *count = (int)log.size();
  });
}

int pxr_test_gemm_records(pxr_handle h, pxr_test_gemm_rec* out, int max, int* count) {
  PXR_TRY(h, {
    const auto& log = h->e->gemm_log;
    for (int i = 0; out && i < max && i < (int)log.size(); ++i) out[i] = log[i];
    if (count) *count = (int)log.size();
  });
}

int pxr_test_attention_records(pxr_handle h, pxr_test_attn_rec* out, int max, int* count) {
  PXR_TRY(h, {
    const auto& log = h->e->attn_log;
    for (int i = 0; out && i < max && i < (int)log.size(); ++i) out[i] = log[i];
    if (count) *count = (int)log.size();
  });
}

int pxr_test_allocations(pxr_handle h, const void** ptr, long long* bytes, int max, int* count) {
  PXR_TRY(h, {
    const Engine* e = h->e;
    for (int i = 0; i < max && i < (int)e->allocs.size(); ++i) {
      if (ptr) ptr[i] = e->allocs[i];
      if (bytes) bytes[i] = (long long)e->alloc_bytes[i];
    }
    if (count) *count = (int)e->allocs.size();
  });
}

int pxr_test_packed_weights(pxr_handle h, pxr_test_pack_rec* out, int max, int* count, int index, void* dst,
                            const float* bias, float* dst_bias, int n_bias) {
  PXR_TRY(h, {
    Engine* e = h->e;
    const auto& log = e->pack_log;
    for (int i = 0; out && i < max && i < (int)log.size(); ++i) out[i] = log[i];
    if (count) *count = (int)log.size();
    if (index < 0) return 0;
    if (index >= (int)log.size() || !dst) throw EngineError(-19, "pxr_test_packed_weights: no such operand");
    const pxr_test_pack_rec& r = log[index];
    PXR_CUDA(cudaMemcpyAsync(dst, r.ptr, (size_t)r.n * sizeof(pxr::act_t), cudaMemcpyDeviceToDevice, e->st));
    if (dst_bias) {
      bool known = false;
      for (const pxr_test_conv_rec& c : e->conv_log) known |= c.wt == r.ptr && c.bias == bias && bias && n_bias <= c.n_out;
      if (!known) throw EngineError(-19, "pxr_test_packed_weights: not the bias of a plan on that operand");
      PXR_CUDA(cudaMemcpyAsync(dst_bias, bias, (size_t)n_bias * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
    }
    PXR_CUDA(cudaStreamSynchronize(e->st));
  });
}

int pxr_set_comm(pxr_handle h, const void* nccl_unique_id, int rank, int world) {
  PXR_TRY(h, {
    Engine* e = h->e;
    if (world != e->cfg.world || rank != e->cfg.rank)
      throw EngineError(-92, "pxr_set_comm: rank/world differ from the pxr_config the engine was created with");
    if (world == 1) return 0;
    std::string msg;
    if (!pxr::Comm::api().load(&msg)) throw EngineError(-90, msg);
    pxr::NcclUniqueId id;
    memcpy(&id, nccl_unique_id, sizeof id);
    e->nccl_check(pxr::Comm::api().init_rank(&e->comm, world, id, rank), "ncclCommInitRank");
  });
}
int pxr_get_unique_id(void* out128) {
  std::string msg;
  if (!pxr::Comm::api().load(&msg)) {
    g_create_err = msg;
    return -90;
  }
  pxr::NcclUniqueId id;
  if (pxr::Comm::api().get_unique_id(&id) != 0) {
    g_create_err = "ncclGetUniqueId failed";
    return -91;
  }
  memcpy(out128, &id, sizeof id);
  return 0;
}

}  // extern "C"
