// libvitb200 engine: weight registry, workspace arena, forward orchestration of ViT / DeepViT / CaiT / CrossViT
// and the extern "C" boundary declared in include/vitb200.h.
//
// The op sequences restate the reference's call graphs (SURVEY.md section 3):
//   ViT / DeepViT  vit.py:159-177, deepvit.py:139-157      CaiT  cait.py:180-194      CrossViT  cross_vit.py:290-303
// with inference semantics (dropout = identity).  T = float runs the exact-fp32 SIMT kernels (numerics gate),
// T = __nv_bfloat16 runs the wgmma GEMM / tensor-core attention kernels with fp32 accumulation and statistics.
#include "../../include/vitb200.h"
#include "attention.cuh"
#include "common.h"
#include "kernels.cuh"

#include <dlfcn.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#ifndef VB_FWD_STREAMS
#define VB_FWD_STREAMS 1                 // 2 = split a large ViT batch into two half-batches on two streams (forward_impl); measured no gain
#endif
#ifndef VB_FWD_SPLIT_MIN_HALF
#define VB_FWD_SPLIT_MIN_HALF 64         // smallest half-batch worth a stream of its own
#endif
namespace vb {
namespace {

thread_local std::string g_last_error;

// ------------------------------------------------------------------------------------------ memory
struct DevMem {
  void* p = nullptr;
  size_t bytes = 0;
  DevMem() = default;
  DevMem(const DevMem&) = delete;
  DevMem& operator=(const DevMem&) = delete;
  ~DevMem() { if (p) cudaFree(p); }
  void ensure(size_t n) {
    if (n <= bytes) return;
    if (p) { cudaFree(p); p = nullptr; bytes = 0; }
    VB_CUDA(cudaMalloc(&p, n));
    bytes = n;
  }
};

// Bump allocator over a few large device blocks; reset() per forward keeps pointers stable across calls with
// the same shapes (so cached TMA descriptors stay valid).
class Arena {
 public:
  void reset() { for (auto& b : blocks_) b.off = 0; cur_ = 0; }
  void* alloc(size_t bytes) {
    bytes = (bytes + 1023) & ~static_cast<size_t>(1023);
    for (; cur_ < blocks_.size(); ++cur_) {
      Block& b = blocks_[cur_];
      if (b.off + bytes <= b.mem->bytes) { void* p = static_cast<char*>(b.mem->p) + b.off; b.off += bytes; return p; }
    }
    Block nb;
    nb.mem.reset(new DevMem());
    nb.mem->ensure(bytes > kBlock ? bytes : kBlock);
    nb.off = bytes;
    blocks_.push_back(std::move(nb));
    cur_ = blocks_.size() - 1;
    return blocks_.back().mem->p;
  }
  template <typename T> T* get(size_t count) { return static_cast<T*>(alloc(count * sizeof(T))); }

 private:
  static constexpr size_t kBlock = static_cast<size_t>(256) << 20;
  struct Block { std::unique_ptr<DevMem> mem; size_t off = 0; };
  std::vector<Block> blocks_;
  size_t cur_ = 0;
};

// ------------------------------------------------------------------------------------------ weights
struct Weight {
  std::string name;
  std::vector<int64_t> shape;
  size_t count = 0;
  float* dev = nullptr;   // fp32 copy in the Keras layout
  bool set = false;
};

struct Linear {
  const float* W = nullptr;      // [K, N] fp32
  const float* bias = nullptr;   // [N] or null
  __nv_bfloat16* Wt = nullptr;   // [N, ldw] bf16, K-major, zero padded
  int K = 0, N = 0, ldw = 0;
  // LayerNorm folded into this Dense (bf16 engine): Wt holds gamma-scaled weights, ln_c2 replaces the bias
  const float* ln_c1 = nullptr;
  const float* ln_c2 = nullptr;
  int ln_d = 0;                  // the LayerNorm's true width when K is zero-padded beyond it (0: K)
  float ln_eps = 1e-3f;          // Keras LayerNormalization; CvT's own LayerNorm: 1e-5 (cvt.py:31)
};
struct Norm { const float* gamma = nullptr; const float* beta = nullptr; int D = 0; };

struct Epi {
  const float* bias = nullptr;
  const float* scale = nullptr;
  const void* res = nullptr;
  int ldr = 0;
  bool gelu = false;
  bool hswish = false;               // hard-swish instead (LeViT MLP, levit.py:37)
  int act() const { return gelu ? ACT_GELU : hswish ? ACT_HSWISH : ACT_NONE; }
  const float* ln_stats = nullptr;   // (sum, sumsq) partials per 64-column chunk of the A operand's rows for a LayerNorm-folded Dense, [M, K/64, 2]
  float* stats_out = nullptr;        // emit (sum, sumsq) partials of every 64-column chunk of the output rows, [M, N/64, 2]
};

struct LayerW {                    // one pre-norm transformer layer in any of the four dialects
  Norm attn_norm, ff_norm;
  Linear to_qkv, to_q, to_kv, to_out, fc1, fc2;
  bool fused_qkv = false, project_out = true;
  const float* mix_a = nullptr;    // DeepViT reattn_weights / CaiT mix_pre
  const float* mix_b = nullptr;    // CaiT mix_post
  Norm reattn_norm;                // DeepViT
  const float* attn_scale = nullptr;  // CaiT LayerScale
  const float* ff_scale = nullptr;
  int heads = 0, dim_head = 0, variant = 0;   // dim_head: head width of the q/k/v ACTIVATIONS (the padded width when dh_model < it)
  int dh_model = 0;                  // the model's dim_head: softmax scale dh_model^-0.5 (vit.py:57)
  int t2t_D = 0, t2t_Dp = 0;         // tensor-core T2T soft-split layer: true width D (LayerNorm, softmax scale), padded width Dp
  bool folded = false;               // attn_norm / ff_norm folded into to_qkv (to_q, to_kv) / fc1
};

// One LeViT Transformer layer (levit.py:141-162): attention (queries on every step-th pixel of the fmap x fmap map) + MLP.
// The BatchNormalizations are folded into the convolutions; q, k and v heads are zero-padded to the activation head width dh.
struct LevitBlockW {
  int dim = 0, dim_out = 0, heads = 0, fmap = 0, step = 1, dh = 0;
  int dp = 0, dp_out = 0;            // row pitches of the input / output token rows: dim / dim_out (bf16: padded, zero columns)
  bool residual = false;             // attn_residual (levit.py:146): not downsampling and dim == dim_out
  Linear qkv;                        // [q | k | v] (step 1) or [k | v] (step 2), each heads * dh wide
  Linear q;                          // step 2: the queries of the even pixels
  Linear to_out, fc1, fc2;
  const float* pos = nullptr;        // [heads][fmap^2] relative-position bias / scale
  float scale = 0.f;                 // dim_key^-0.5
};

// One CvT Transformer layer (cvt.py:142-147) on channel rows zero-padded to dp (bf16) / dim (fp32).  The depthwise convolutions
// carry their BatchNormalization folded (taps [k*k][dp] scaled, plus a per-channel shift); the MLP's PreNorm is folded into fc1
// in the bf16 engine.
struct CvtBlockW {
  int dim = 0, dp = 0, heads = 0, k = 0, kv_stride = 1;
  Norm attn_norm, ff_norm;           // gamma / beta [dp], zero on pad channels
  const float *wq = nullptr, *bq = nullptr, *wkv = nullptr, *bkv = nullptr;
  Linear pw_q, pw_kv, to_out, fc1, fc2;
};
struct CvtStageW {                   // cvt.py:186-192: Conv2D (SAME, bias) + LayerNorm + Transformer
  int dim = 0, dp = 0, k = 0, stride = 1;
  Linear conv;
  Norm norm;
  std::vector<CvtBlockW> blocks;
};

// CvT: BN(dw(y)) = dw_{s * taps}(y) + (beta - mean * s) with s = gamma / sqrt(var + 1e-5) (inference statistics, cvt.py:85).
// Exact under SAME zero padding, which adds nothing to either form.  taps: the Keras depthwise kernel [k, k, 1, C]; w: taps
// [k*k][Cp] and shift [Cp], zero on channels >= C.
inline void cvt_fold_dw(const std::vector<double>& taps, const std::vector<double>& gamma, const std::vector<double>& beta,
                        const std::vector<double>& mean, const std::vector<double>& var, int k, int C, int Cp, std::vector<double>& w,
                        std::vector<double>& shift) {
  w.assign(static_cast<size_t>(k) * k * Cp, 0.0);
  shift.assign(Cp, 0.0);
  for (int c = 0; c < C; ++c) {
    const double sc = gamma[c] / std::sqrt(var[c] + 1e-5);
    for (int t = 0; t < k * k; ++t) w[static_cast<size_t>(t) * Cp + c] = taps[static_cast<size_t>(t) * C + c] * sc;
    shift[c] = beta[c] - mean[c] * sc;
  }
}

// One Twins-SVT Transformer layer (twins_svt.py:192-213) on channel rows zero-padded to dp (bf16) / dim (fp32): x = x + f(LN(x))
// for local attention, MLP, global attention, MLP; stage 4 has no local attention and no first MLP (has_local=False, :255).  The
// bf16 engine folds the PreNorm LayerNorms of the fused local q|k|v, the global to_q and the fc1s into those GEMMs.
struct MlpW { Norm norm; Linear fc1, fc2; };   // PreNorm MLP (Twins-SVT, CrossFormer): LayerNorm eps 1e-5, fc1, GELU, fc2
struct TwinsLayerW {
  bool local = false;
  Norm local_norm, global_norm;      // gamma / beta [dp], zero on pad channels
  Linear qkv, local_out;             // local: to_q | to_kv as one [dp, 1536] GEMM, to_out
  Linear to_q, to_kv, global_out;    // global: to_q [dp, 512], to_kv [k * k * dim, 1024] over the VALID k x k patch rows
  MlpW ff1, ff2;
};
struct TwinsStageW {                 // twins_svt.py:252-259: PatchEmbedding, Transformer(depth 1), PEG, Transformer(depth)
  int dim = 0, dp = 0, patch = 1, local = 0, global_k = 1, peg_k = 3;
  Linear proj;                       // rows in unfold_same's (p1, p2, c) order
  const float *peg_w = nullptr, *peg_b = nullptr;   // PEG taps [k*k][dp] with the residual on the centre tap, bias [dp]
  std::vector<TwinsLayerW> pre, post;
};

// One CrossFormer Transformer layer (crossformer.py:196-203) on channel rows zero-padded to dp (bf16) / dim (fp32): short attention,
// MLP, long attention, MLP, each x = f(x) + x with f's own LayerNorm first (eps 1e-5); the bf16 engine folds those LayerNorms into
// the q|k|v and fc1 GEMMs.  Attention has heads = dim / 32 of width 32, inner width I = 32 * heads.
struct CrossformerAttnW {
  int wsz = 1;
  bool dilated = false;              // the long attention's windows (crossformer.py:146)
  Norm norm;
  Linear qkv;                        // [q | k | v], 3 I columns (bf16: padded to a multiple of 64); wsz == 1: v alone, I columns
  Linear to_out;                     // [I, dp]
  const float* table = nullptr;      // the DynamicPositionBias window table, (2 wsz - 1)^2 (wsz > 1)
};
struct CrossformerLayerW { CrossformerAttnW short_attn, long_attn; MlpW ff1, ff2; };
struct CrossformerStageW {           // crossformer.py:248-255: CrossEmbedLayer, Transformer
  int dim = 0, dp = 0, heads = 0, kmax = 1, stride = 1;
  Linear embed;                      // every kernel nested in the kmax x kmax one, rows in unfold_same's (row, column, channel) order
  std::vector<CrossformerLayerW> layers;
};

struct EmbedW { Linear patch; const float* pos = nullptr; const float* cls = nullptr; int dim = 0, n_pos = 0; };
struct CrossW { bool proj = false; Linear project_in, project_out, to_q, to_kv, to_out; Norm norm; };

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace
}  // namespace vb

using namespace vb;

static_assert(offsetof(vb_config, cct_conv_layers) == VB_CONFIG_SIZE_ABI7, "VB_CONFIG_SIZE_ABI7 is the struct before the CCT fields");

// ------------------------------------------------------------------------------------------ NCCL (loaded on demand)
// The five entry points of the NCCL 2.x C API the data-parallel path needs, declared here so that neither nccl.h nor a
// link-time libnccl is required: ncclUniqueId is 128 opaque bytes passed by value, ncclComm_t an opaque pointer,
// ncclFloat32 == 7, ncclSuccess == 0.
namespace vb {
namespace {
struct NcclId { char internal[128]; };
struct NcclApi {
  int (*GetUniqueId)(NcclId*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  if (api.ok) return api;
  void* lib = nullptr;
  if (const char* p = getenv("VB_NCCL_LIB")) lib = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  VB_CHECK(lib != nullptr, std::string("NCCL not found (set VB_NCCL_LIB to libnccl.so.2): ") + (dlerror() ? dlerror() : ""));
  api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
  api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(lib, "ncclAllGather"));
  api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
  api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
  VB_CHECK(api.GetUniqueId && api.CommInitRank && api.AllGather && api.CommDestroy && api.GetErrorString,
           "the NCCL library lacks one of ncclGetUniqueId / ncclCommInitRank / ncclAllGather / ncclCommDestroy / ncclGetErrorString");
  api.ok = true;
  return api;
}
void nccl_check(int rc, const char* what) {
  if (rc != 0) throw vb::Error(5, std::string(what) + " failed: " + nccl().GetErrorString(rc));
}
}  // namespace
}  // namespace vb

struct vb_handle {
  vb_config cfg;
  int device = 0;
  void* dp_comm = nullptr;          // ncclComm_t of the data-parallel group (vb_dp_init)
  int dp_rank = 0, dp_world = 1;
  bool finalized = false;
  std::string error;
  std::vector<Weight> weights;
  std::map<std::string, int> windex;
  std::vector<std::unique_ptr<DevMem>> owned;
  Arena arena;
  DevMem img_dev, logits_dev, tok_dev, tokens_in, tokens_out;
  long long last_launches = 0;

  // optional per-kernel-class timing: CUDA events recorded on the launch stream around each call
  enum { PROF_GEMM = 0, PROF_ATTN = 1, PROF_LN = 2, PROF_EMBED = 3, PROF_OTHER = 4, PROF_GEMM_GELU = 5, PROF_GEMM_RES = 6, PROF_NUM = 7 };
  struct ProfRec { int cls; cudaEvent_t a, b; double flops; double bytes; };
  bool profiling = false;
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> event_pool;
  double prof_ms[PROF_NUM] = {0}, prof_flops[PROF_NUM] = {0}, prof_bytes[PROF_NUM] = {0};
  long long prof_calls[PROF_NUM] = {0};
  // side streams of the per-image T2T soft-split attention (layer_t2t): forked from / joined into the forward's stream with
  // timing-less events, so that the branch is part of a captured graph like everything else
  static constexpr int T2T_MAX_STREAMS = 4;
  cudaStream_t side_streams[T2T_MAX_STREAMS - 1] = {nullptr, nullptr, nullptr};
  cudaEvent_t fork_event = nullptr, join_events[T2T_MAX_STREAMS - 1] = {nullptr, nullptr, nullptr};
  cudaStream_t half_stream = nullptr;                    // second half-batch of a split forward (forward_impl)
  cudaEvent_t fwd_fork_event = nullptr, fwd_join_event = nullptr;
  void ensure_side_streams() {
    if (fork_event != nullptr) return;
    VB_CUDA(cudaStreamCreateWithFlags(&half_stream, cudaStreamNonBlocking));
    VB_CUDA(cudaEventCreateWithFlags(&fwd_fork_event, cudaEventDisableTiming));
    VB_CUDA(cudaEventCreateWithFlags(&fwd_join_event, cudaEventDisableTiming));
    VB_CUDA(cudaEventCreateWithFlags(&fork_event, cudaEventDisableTiming));
    for (int i = 0; i < T2T_MAX_STREAMS - 1; ++i) {
      VB_CUDA(cudaStreamCreateWithFlags(&side_streams[i], cudaStreamNonBlocking));
      VB_CUDA(cudaEventCreateWithFlags(&join_events[i], cudaEventDisableTiming));
    }
  }
  void destroy_side_streams() {
    if (fork_event == nullptr) return;
    cudaEventDestroy(fork_event);
    cudaEventDestroy(fwd_fork_event); cudaEventDestroy(fwd_join_event); cudaStreamDestroy(half_stream);
    for (int i = 0; i < T2T_MAX_STREAMS - 1; ++i) { cudaEventDestroy(join_events[i]); cudaStreamDestroy(side_streams[i]); }
    fork_event = nullptr;
  }
  cudaEvent_t get_event() {
    if (!event_pool.empty()) { cudaEvent_t e = event_pool.back(); event_pool.pop_back(); return e; }
    cudaEvent_t e;
    VB_CUDA(cudaEventCreate(&e));
    return e;
  }
  struct ProfScope {
    vb_handle* h; cudaStream_t s; int idx = -1;
    ProfScope(vb_handle* h_, int cls, double flops, double bytes, cudaStream_t s_) : h(h_), s(s_) {
      if (!h->profiling) return;
      ProfRec r{cls, h->get_event(), h->get_event(), flops, bytes};
      cudaEventRecord(r.a, s);
      h->prof_recs.push_back(r);
      idx = static_cast<int>(h->prof_recs.size()) - 1;
    }
    ~ProfScope() { if (idx >= 0) cudaEventRecord(h->prof_recs[idx].b, s); }
  };
  void prof_collect() {
    if (prof_recs.empty()) return;
    cudaDeviceSynchronize();
    for (auto& r : prof_recs) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
        prof_ms[r.cls] += ms; prof_flops[r.cls] += r.flops; prof_bytes[r.cls] += r.bytes; prof_calls[r.cls] += 1;
      }
      event_pool.push_back(r.a); event_pool.push_back(r.b);
    }
    prof_recs.clear();
  }

  // model structure (filled by finalize)
  EmbedW embed, sm_embed, lg_embed;
  std::vector<LayerW> layers, cls_layers, t2t_layers;   // t2t_layers: the one-layer transformers between the soft splits (t2t.py:35)
  Norm merger_norm;                                     // PatchMerger (vit_with_patch_merger.py:46-47)
  const float* merger_queries = nullptr;
  struct T2TStage { int k, stride, dim; };              // dim = channels * prod(k^2) up to and including this stage (t2t.py:63)
  std::vector<T2TStage> t2t_stages() const {
    const int ks[4] = {cfg.t2t_k0, cfg.t2t_k1, cfg.t2t_k2, cfg.t2t_k3}, ss[4] = {cfg.t2t_s0, cfg.t2t_s1, cfg.t2t_s2, cfg.t2t_s3};
    std::vector<T2TStage> st;
    int d = cfg.channels;
    for (int i = 0; i < cfg.t2t_num_layers; ++i) { d *= ks[i] * ks[i]; st.push_back(T2TStage{ks[i], ss[i], d}); }
    return st;
  }
  static int conv_output_size(int size, int k, int stride) {   // t2t.py:14-15 with padding = stride // 2
    return static_cast<int>((static_cast<double>(size - k + 2 * (stride / 2)) / stride) + 1);
  }
  // CCT tokenizer (cct.py:188-200): conv layer i maps cin -> cout channels, 64 (Tokenizer in_planes) between layers, dim after the last
  std::vector<Linear> cct_convs;
  Norm cct_norm;
  const float* cct_pool_w = nullptr;                      // attention_pool Dense(1): kernel [dim, 1], bias [1]
  const float* cct_pool_b = nullptr;
  int cct_conv_cin(int i) const { return i == 0 ? cfg.channels : 64; }
  int cct_conv_cout(int i) const { return i == cfg.cct_conv_layers - 1 ? cfg.dim : 64; }
  // token grid of an h x w image after the tokenizer: SAME convolution and max-pool, ceil(size / stride) each
  void cct_grid(int* h, int* w) const {
    for (int i = 0; i < cfg.cct_conv_layers; ++i) {
      *h = (*h + cfg.cct_stride - 1) / cfg.cct_stride; *w = (*w + cfg.cct_stride - 1) / cfg.cct_stride;
      *h = (*h + cfg.cct_pool_stride - 1) / cfg.cct_pool_stride; *w = (*w + cfg.cct_pool_stride - 1) / cfg.cct_pool_stride;
    }
  }
  int cct_sequence_length() const { int h = cfg.image_h, w = cfg.image_w; cct_grid(&h, &w); return h * w; }   // cct.py:331-333
  // LeViT (levit.py:164-226): the stem convolutions, the blocks of every Transformer in backbone order, the heads
  vb_levit_config lv{};
  std::vector<Linear> lv_stem;
  std::vector<LevitBlockW> lv_blocks;
  Linear lv_distill;
  struct LevitPlan { std::string pre; int dim, dim_out, heads, fmap, mult; bool down; };
  // levit.py:194-204: stage s = depths[s] blocks on the fmap map; between stages one shrink block (2 * heads, mlp_mult 2, the
  // queries on the even pixels) after which fmap = ceil(fmap / 2).  pre: the attribute path of the block's [attn, mlp] pair.
  std::vector<LevitPlan> levit_plan() const {
    std::vector<LevitPlan> v;
    int fmap = cfg.image_h / 16, t = 0;
    for (int st = 0; st < lv.stages; ++st, ++t) {
      for (int L = 0; L < lv.depths[st]; ++L)
        v.push_back({"backbone." + std::to_string(t) + ".layers." + std::to_string(L) + ".", lv.dims[st], lv.dims[st], lv.heads[st], fmap,
                     lv.mlp_mult, false});
      if (st + 1 < lv.stages) {
        ++t;
        v.push_back({"backbone." + std::to_string(t) + ".layers.0.", lv.dims[st], lv.dims[st + 1], 2 * lv.heads[st], fmap, 2, true});
        fmap = (fmap + 1) / 2;
      }
    }
    return v;
  }
  int levit_stem_cout(int i) const { return i == 0 ? 32 : i == 1 ? 64 : i == 2 ? 128 : lv.dims[0]; }   // levit.py:187-192
  // activation head width of q, k and v: the bf16 engine pads to the flash kernel's 64 (wider heads: a multiple of 64)
  int levit_dh() const {
    const int m = lv.dim_key > lv.dim_value ? lv.dim_key : lv.dim_value;
    return bf16() ? round_up(m, 64) : m;
  }
  // Width the bf16 engine carries a channel dimension of LeViT / CvT at: a multiple of 64, so that every GEMM of a block (N = a
  // channel width) runs on the wgmma kernel.  Pad columns are zero and stay zero: zero weights and biases, hard-swish(0) = GELU(0) =
  // 0, and LayerNorm gammas and betas padded with zeros.
  int channel_width(int d) const { return bf16() ? round_up(d, 64) : d; }
  // CvT (cvt.py:149-202): the three stages, then the average pool and the Dense head (`head`)
  vb_cvt_config cv{};
  std::vector<CvtStageW> cvt_stages;
  static std::string cvt_pre(int st) { return "cvt_layers." + std::to_string(st) + "."; }
  int cvt_cin(int st) const { return st == 0 ? cfg.channels : cv.emb_dim[st - 1]; }
  // Twins-SVT (twins_svt.py:215-268): the four stages, then the average pool and the Dense head (`head`)
  vb_twins_svt_config tw{};
  std::vector<TwinsStageW> twins_stages;
  static std::string twins_pre(int st) { return "svt_layers." + std::to_string(st) + "."; }
  int twins_cin(int st) const { return st == 0 ? cfg.channels : tw.emb_dim[st - 1]; }
  static constexpr int kTwinsInner = 512;        // 8 heads of 64: Transformer is never passed heads / dim_head (twins_svt.py:254-258)
  // CrossFormer (crossformer.py:205-269): the four stages, then the average pool and the Dense head (`head`)
  vb_crossformer_config cf{};
  std::vector<CrossformerStageW> cf_stages;
  static std::string cf_pre(int st) { return "crossformer_layers." + std::to_string(st) + "."; }
  int cf_cin(int st) const { return st == 0 ? cfg.channels : cf.dim[st - 1]; }
  std::vector<int> cf_kernels(int st) const {                // CrossEmbedLayer sorts them (crossformer.py:34)
    std::vector<int> k(cf.kernels[st], cf.kernels[st] + cf.n_kernels[st]);
    std::sort(k.begin(), k.end());
    return k;
  }
  std::vector<int> cf_dim_scales(int st) const {             // crossformer.py:38-39
    const int d = cf.dim[st], n = cf.n_kernels[st];
    std::vector<int> v;
    int sum = 0;
    for (int i = 1; i < n; ++i) { v.push_back(d >> i); sum += d >> i; }
    v.push_back(d - sum);
    return v;
  }
  struct XBlock { std::vector<LayerW> sm_layers, lg_layers; Norm sm_final, lg_final; std::vector<CrossW> sm_attend_lg, lg_attend_sm; };
  std::vector<XBlock> xblocks;
  Norm head_norm, sm_head_norm, lg_head_norm;
  Linear head, sm_head, lg_head;

  // cached patch-embedding residual terms, keyed by (embed ptr, batch, rows)
  struct ResKey { const void* e; int B, rows; bool operator<(const ResKey& o) const { return std::tie(e, B, rows) < std::tie(o.e, o.B, o.rows); } };
  std::map<ResKey, std::unique_ptr<DevMem>> embed_res;

  // cached wgmma GEMM plans (TMA descriptors)
  using PlanKey = std::array<uintptr_t, 16>;
  std::map<PlanKey, GemmBf16> plans;

  // Whole-forward CUDA graphs (vb_forward): the launch sequence of one (image pointer, logits pointer, batch, h, w, stream)
  // combination is captured on its SECOND call (the first runs eagerly and does every lazy host-side step: arena growth,
  // kernel attributes, descriptor / residual caches) and replayed from the third on.  Workspace pointers are stable (the
  // arena is reset, never freed, per forward), so a replay touches exactly the memory the eager run would.  Programmatic
  // dependent launches are captured as programmatic edges.  VB_NO_GRAPH=1 disables it; profiling and the legacy default
  // stream (which cannot be captured) always run eagerly.
  struct GraphKey {
    const void* img; void* out; int B, H, W; cudaStream_t s;
    bool operator<(const GraphKey& o) const { return std::tie(img, out, B, H, W, s) < std::tie(o.img, o.out, o.B, o.H, o.W, o.s); }
  };
  struct GraphEntry { cudaGraphExec_t exec = nullptr; int calls = 0; long long launches = 0; bool failed = false; };
  std::map<GraphKey, GraphEntry> graphs;
  // cumulative over the handle's life (vb_graph_stats): a key whose capture failed runs eagerly until its graph is dropped
  long long graph_captures = 0, graph_replays = 0, graph_failures = 0;
  std::string graph_last_failure;
  void drop_graphs() {
    for (auto& g : graphs) if (g.second.exec) cudaGraphExecDestroy(g.second.exec);
    graphs.clear();
  }

  bool bf16() const { return cfg.precision == VB_PRECISION_BF16; }
  // the device copies of the registered weights: what this handle's head-mix cache entries are keyed by
  std::vector<const void*> weight_pointers() const {
    std::vector<const void*> p;
    for (const auto& w : weights) p.push_back(w.dev);
    return p;
  }

  // ---------------------------------------------------------------- weight registry
  void expect(const std::string& name, std::vector<int64_t> shape) {
    Weight w;
    w.name = name;
    w.shape = std::move(shape);
    w.count = 1;
    for (auto d : w.shape) w.count *= static_cast<size_t>(d);
    windex[name] = static_cast<int>(weights.size());
    weights.push_back(std::move(w));
  }
  void expect_dense(const std::string& n, int din, int dout, bool bias = true) {
    expect(n + ".kernel", {din, dout});
    if (bias) expect(n + ".bias", {dout});
  }
  void expect_ln(const std::string& n, int d) { expect(n + ".gamma", {d}); expect(n + ".beta", {d}); }
  void expect_layer(const std::string& pre, int dim, int heads, int dh, int mlp, int kind) {
    const int inner = heads * dh;
    expect_ln(pre + "attn_norm", dim);
    if (kind == VB_KIND_VIT || kind == VB_KIND_DEEPVIT) expect_dense(pre + "to_qkv", dim, 3 * inner, false);
    else { expect_dense(pre + "to_q", dim, inner, false); expect_dense(pre + "to_kv", dim, 2 * inner, false); }
    if (kind == VB_KIND_DEEPVIT) { expect(pre + "reattn_weights", {heads, heads}); expect_ln(pre + "reattn_norm", heads); }
    if (kind == VB_KIND_CAIT) { expect(pre + "mix_pre", {heads, heads}); expect(pre + "mix_post", {heads, heads}); }
    const bool po = !(kind == VB_KIND_VIT && heads == 1 && dh == dim);   // vit.py:53
    if (po) expect_dense(pre + "to_out", inner, dim);
    expect_ln(pre + "ff_norm", dim);
    expect_dense(pre + "fc1", dim, mlp);
    expect_dense(pre + "fc2", mlp, dim);
  }
  void build_expected() {
    const vb_config& c = cfg;
    const int C = c.channels;
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_PARALLEL_VIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      expect("pos_embedding", {1, np + 1, c.dim});
      expect("cls_token", {1, 1, c.dim});
      expect_dense("patch", c.patch_h * c.patch_w * C, c.dim);
      for (int L = 0; L < c.depth; ++L) {
        if (c.kind == VB_KIND_PARALLEL_VIT) {   // branch i = (attention fn i, feed-forward fn i) of layer L (parallel_vit.py:109-112)
          for (int i = 0; i < c.parallel_branches; ++i)
            expect_layer("layers." + std::to_string(L) + ".branch" + std::to_string(i) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
        } else {
          expect_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, c.kind);
        }
      }
      expect_ln("head_norm", c.dim);
      expect_dense("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_PATCH_MERGER_VIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      expect("pos_embedding", {1, np + 1, c.dim});                       // vit_with_patch_merger.py:163
      expect_dense("patch", c.patch_h * c.patch_w * C, c.dim);
      for (int L = 0; L < c.depth; ++L) expect_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
      expect_ln("patch_merger.norm", c.dim);
      expect("patch_merger.queries", {c.patch_merge_num_tokens, c.dim});
      expect_ln("head_norm", c.dim);
      expect_dense("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_T2T_VIT) {
      const auto st = t2t_stages();
      int out = c.image_h;
      for (size_t i = 0; i < st.size(); ++i) {
        out = conv_output_size(out, st[i].k, st[i].stride);             // t2t.py:66
        if (i + 1 < st.size())                                           // Transformer(dim=d, heads=1, depth=1, dim_head=d, mlp_dim=d) t2t.py:69-70
          expect_layer("t2t." + std::to_string(i) + ".layers.0.", st[i].dim, 1, st[i].dim, st[i].dim, VB_KIND_VIT);
      }
      expect_dense("patch", st.back().dim, c.dim);                        // t2t.py:73
      expect("pos_embedding", {1, out * out + 1, c.dim});                 // :76
      expect("cls_token", {1, 1, c.dim});
      for (int L = 0; L < c.depth; ++L) expect_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
      expect_ln("head_norm", c.dim);
      expect_dense("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_CCT) {
      for (int i = 0; i < c.cct_conv_layers; ++i)                         // Conv2D(use_bias=False) kernel [k, k, cin, cout]
        expect("tokenizer.conv." + std::to_string(i) + ".kernel", {c.cct_kernel, c.cct_kernel, cct_conv_cin(i), cct_conv_cout(i)});
      if (c.cct_pos_emb != VB_CCT_POS_NONE) expect("positional_emb", {1, cct_sequence_length(), c.dim});   // cct.py:250-256
      for (int L = 0; L < c.depth; ++L) {                                 // TransformerEncoderLayer cct.py:139-157
        const std::string pre = "layers." + std::to_string(L) + ".";
        expect_ln(pre + "attn_norm", c.dim);                              // pre_norm
        expect_dense(pre + "to_qkv", c.dim, 3 * c.dim, false);
        expect_dense(pre + "to_out", c.dim, c.dim);                       // self_attn.proj
        expect_ln(pre + "norm1", c.dim);
        expect_dense(pre + "fc1", c.dim, c.mlp_dim);                      // linear1
        expect_dense(pre + "fc2", c.mlp_dim, c.dim);                      // linear2
      }
      expect_ln("norm", c.dim);                                           // cct.py:266
      expect_dense("attention_pool", c.dim, 1);                           // :248
      expect_dense("head", c.dim, c.num_classes);                         // fc :267
    } else if (c.kind == VB_KIND_LEVIT) {
      auto expect_bn = [&](const std::string& n, int d) {
        for (const char* leaf : {"gamma", "beta", "moving_mean", "moving_variance"}) expect(n + "." + leaf, {d});
      };
      for (int i = 0; i < 4; ++i) {
        expect("conv_embedding." + std::to_string(i) + ".kernel", {3, 3, i == 0 ? C : levit_stem_cout(i - 1), levit_stem_cout(i)});
        expect("conv_embedding." + std::to_string(i) + ".bias", {levit_stem_cout(i)});
      }
      for (const auto& b : levit_plan()) {
        const std::string a = b.pre + "0.";                              // Attention levit.py:64-117
        const int hk = b.heads * lv.dim_key, hv = b.heads * lv.dim_value, hidden = b.dim_out * b.mult;
        for (const char* n : {"to_q", "to_k", "to_v"}) {
          const int w = n[3] == 'v' ? hv : hk;
          expect(a + n + ".0.kernel", {1, 1, b.dim, w});
          expect_bn(a + n + ".1", w);
        }
        expect(a + "pos_bias.embeddings", {b.fmap * b.fmap, b.heads});
        expect(a + "to_out.1.kernel", {1, 1, hv, b.dim_out});
        expect(a + "to_out.1.bias", {b.dim_out});
        expect_bn(a + "to_out.2", b.dim_out);
        expect(b.pre + "1.net.0.kernel", {1, 1, b.dim_out, hidden});      // MLP levit.py:48-62
        expect(b.pre + "1.net.0.bias", {hidden});
        expect(b.pre + "1.net.3.kernel", {1, 1, hidden, b.dim_out});
        expect(b.pre + "1.net.3.bias", {b.dim_out});
      }
      const int dl = lv.dims[lv.stages - 1];
      expect_dense("mlp_head", dl, c.num_classes);
      if (lv.num_distill_classes > 0) expect_dense("distill_head", dl, lv.num_distill_classes);
    } else if (c.kind == VB_KIND_CVT) {
      auto expect_ln4 = [&](const std::string& n, int d) { expect(n + ".g", {1, 1, 1, d}); expect(n + ".b", {1, 1, 1, d}); };   // cvt.py:35-36
      for (int st = 0; st < VB_CVT_STAGES; ++st) {
        const std::string p = cvt_pre(st);
        const int d = cv.emb_dim[st], k = cv.proj_kernel[st], inner = 64 * cv.heads[st], hidden = d * cv.mlp_mult[st];
        expect(p + "0.kernel", {cv.emb_kernel[st], cv.emb_kernel[st], cvt_cin(st), d});          // cvt.py:187
        expect(p + "0.bias", {d});
        expect_ln4(p + "1", d);
        for (int L = 0; L < cv.depth[st]; ++L) {
          const std::string b = p + "2.layers." + std::to_string(L) + ".";
          expect_ln4(b + "0.norm", d);
          for (int kv = 0; kv < 2; ++kv) {                                // DepthWiseConv2d cvt.py:79-92, bias=False (:103-104)
            const std::string n = b + (kv ? "0.fn.to_kv.net." : "0.fn.to_q.net.");
            expect(n + "0.kernel", {k, k, 1, d});
            for (const char* leaf : {"gamma", "beta", "moving_mean", "moving_variance"}) expect(n + "1." + leaf, {d});
            expect(n + "2.kernel", {1, 1, d, (kv ? 2 : 1) * inner});
          }
          expect(b + "0.fn.to_out.0.kernel", {1, 1, inner, d});            // cvt.py:106-109
          expect(b + "0.fn.to_out.0.bias", {d});
          expect_ln4(b + "1.norm", d);
          expect(b + "1.fn.net.0.kernel", {1, 1, d, hidden});              // MLP cvt.py:63-77
          expect(b + "1.fn.net.0.bias", {hidden});
          expect(b + "1.fn.net.3.kernel", {1, 1, hidden, d});
          expect(b + "1.fn.net.3.bias", {d});
        }
      }
      expect_dense("cvt_layers.3.1", cv.emb_dim[VB_CVT_STAGES - 1], c.num_classes);   // cvt.py:195-198
    } else if (c.kind == VB_KIND_TWINS_SVT) {
      auto expect_ln4 = [&](const std::string& n, int d) { expect(n + ".g", {1, 1, 1, d}); expect(n + ".b", {1, 1, 1, d}); };   // :50-51
      const int I = kTwinsInner;
      for (int st = 0; st < VB_TWINS_STAGES; ++st) {
        const std::string p = twins_pre(st);
        const int d = tw.emb_dim[st], ps = tw.patch_size[st], kg = tw.global_k[st], k = tw.peg_kernel_size;
        auto expect_mlp = [&](const std::string& m) {                      // Residual(PreNorm(MLP)) :78-92,201,203
          expect_ln4(m + ".fn.norm", d);
          expect(m + ".fn.fn.net.0.kernel", {1, 1, d, 4 * d});
          expect(m + ".fn.fn.net.0.bias", {4 * d});
          expect(m + ".fn.fn.net.3.kernel", {1, 1, 4 * d, d});
          expect(m + ".fn.fn.net.3.bias", {d});
        };
        expect(p + "0.proj.kernel", {1, 1, twins_cin(st) * ps * ps, d});   // PatchEmbedding :99
        expect(p + "0.proj.bias", {d});
        for (int t : {1, 3}) {
          for (int L = 0; L < (t == 1 ? 1 : tw.depth[st]); ++L) {
            const std::string b = p + std::to_string(t) + ".layers." + std::to_string(L) + ".";
            if (st < VB_TWINS_STAGES - 1) {                                  // LocalAttention :127-133
              expect_ln4(b + "0.fn.norm", d);
              expect(b + "0.fn.fn.to_q.kernel", {1, 1, d, I});
              expect(b + "0.fn.fn.to_kv.kernel", {1, 1, d, 2 * I});
              expect(b + "0.fn.fn.to_out.0.kernel", {1, 1, I, d});
              expect(b + "0.fn.fn.to_out.0.bias", {d});
              expect_mlp(b + "1");
            }
            expect_ln4(b + "2.fn.norm", d);                                  // GlobalAttention :167-173
            expect(b + "2.fn.fn.to_q.kernel", {1, 1, d, I});
            expect(b + "2.fn.fn.to_kv.kernel", {kg, kg, d, 2 * I});
            expect(b + "2.fn.fn.to_out.0.kernel", {1, 1, I, d});
            expect(b + "2.fn.fn.to_out.0.bias", {d});
            expect_mlp(b + "3");
          }
          if (t == 1) {
            expect(p + "2.proj.fn.kernel", {k, k, 1, d});                    // PEG :111
            expect(p + "2.proj.fn.bias", {d});
          }
        }
      }
      expect_dense("svt_layers.4.1", tw.emb_dim[VB_TWINS_STAGES - 1], c.num_classes);   // :261-264
    } else if (c.kind == VB_KIND_CROSSFORMER) {
      auto expect_ln4 = [&](const std::string& n, int d) { expect(n + ".g", {1, 1, 1, d}); expect(n + ".b", {1, 1, 1, d}); };   // :77-78
      for (int st = 0; st < VB_CROSSFORMER_STAGES; ++st) {
        const std::string p = cf_pre(st);
        const int d = cf.dim[st], I = 32 * (d / 32), d4 = d / 4;
        const auto ks = cf_kernels(st), ds = cf_dim_scales(st);
        for (size_t i = 0; i < ks.size(); ++i) {                          // CrossEmbedLayer :41-43
          expect(p + "0.convs." + std::to_string(i) + ".kernel", {ks[i], ks[i], cf_cin(st), ds[i]});
          expect(p + "0.convs." + std::to_string(i) + ".bias", {ds[i]});
        }
        for (int L = 0; L < cf.depth[st]; ++L) {
          const std::string b = p + "1.layers." + std::to_string(L) + ".";
          for (const char* a : {"0.", "2."}) {                            // Attention :104-131
            expect_ln4(b + a + "norm", d);
            expect(b + a + "to_qkv.kernel", {1, 1, d, 3 * I});
            expect(b + a + "to_out.kernel", {1, 1, I, d});
            expect(b + a + "to_out.bias", {d});
            const std::string dpb = b + a + "dpb.dpb_layers.";             // DynamicPositionBias :51-71
            for (int li : {0, 3, 6, 9}) {
              expect(dpb + std::to_string(li) + ".kernel", {li == 0 ? 2 : d4, li == 9 ? 1 : d4});
              expect(dpb + std::to_string(li) + ".bias", {li == 9 ? 1 : d4});
            }
            for (int li : {1, 4, 7}) expect_ln(dpb + std::to_string(li), d4);
          }
          for (const char* m : {"1.", "3."}) {                            // MLP :89-102
            expect_ln4(b + m + "net.0", d);
            expect(b + m + "net.1.kernel", {1, 1, d, 4 * d});
            expect(b + m + "net.1.bias", {4 * d});
            expect(b + m + "net.4.kernel", {1, 1, 4 * d, d});
            expect(b + m + "net.4.bias", {d});
          }
        }
      }
      expect_dense("to_logits.1", cf.dim[VB_CROSSFORMER_STAGES - 1], c.num_classes);   // :258-261
    } else if (c.kind == VB_KIND_CAIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      expect("pos_embedding", {1, np, c.dim});
      expect("cls_token", {1, 1, c.dim});
      expect_dense("patch", c.patch_h * c.patch_w * C, c.dim);
      for (int st = 0; st < 2; ++st) {
        const std::string stack = st == 0 ? "patch_transformer" : "cls_transformer";
        const int depth = st == 0 ? c.depth : c.cls_depth;
        for (int L = 0; L < depth; ++L) {
          const std::string pre = stack + ".layers." + std::to_string(L) + ".";
          expect(pre + "attn_scale", {1, 1, c.dim});
          expect(pre + "ff_scale", {1, 1, c.dim});
          expect_layer(pre, c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_CAIT);
        }
      }
      expect_ln("head_norm", c.dim);
      expect_dense("head", c.dim, c.num_classes);
    } else {
      for (int b = 0; b < 2; ++b) {
        const std::string br = b == 0 ? "sm" : "lg";
        const int dim = b == 0 ? c.sm_dim : c.lg_dim, p = b == 0 ? c.sm_patch_size : c.lg_patch_size;
        const int np = (c.image_h / p) * (c.image_w / p);
        expect_dense(br + "_embed.patch", p * p * C, dim);
        expect(br + "_embed.pos_embedding", {1, np + 1, dim});
        expect(br + "_embed.cls_token", {1, 1, dim});
      }
      const int xinner = c.cross_attn_heads * c.cross_attn_dim_head;
      for (int D = 0; D < c.cross_depth; ++D) {
        const std::string bp = "blocks." + std::to_string(D) + ".";
        for (int b = 0; b < 2; ++b) {
          const std::string br = b == 0 ? "sm" : "lg";
          const int dim = b == 0 ? c.sm_dim : c.lg_dim;
          const int depth = b == 0 ? c.sm_enc_depth : c.lg_enc_depth, heads = b == 0 ? c.sm_enc_heads : c.lg_enc_heads;
          const int dh = b == 0 ? c.sm_enc_dim_head : c.lg_enc_dim_head, mlp = b == 0 ? c.sm_enc_mlp_dim : c.lg_enc_mlp_dim;
          for (int L = 0; L < depth; ++L) expect_layer(bp + br + "_enc.layers." + std::to_string(L) + ".", dim, heads, dh, mlp, VB_KIND_CROSSVIT);
          expect_ln(bp + br + "_enc.final_norm", dim);
        }
        for (int R = 0; R < c.cross_attn_depth; ++R) {
          for (int b = 0; b < 2; ++b) {
            const std::string n = bp + "cross." + std::to_string(R) + (b == 0 ? ".sm_attend_lg." : ".lg_attend_sm.");
            const int din = b == 0 ? c.sm_dim : c.lg_dim, dout = b == 0 ? c.lg_dim : c.sm_dim;
            if (din != dout) { expect_dense(n + "project_in", din, dout); expect_dense(n + "project_out", dout, din); }
            expect_ln(n + "norm", dout);
            expect_dense(n + "to_q", dout, xinner, false);
            expect_dense(n + "to_kv", dout, 2 * xinner, false);
            expect_dense(n + "to_out", xinner, dout);
          }
        }
      }
      expect_ln("sm_head_norm", c.sm_dim); expect_dense("sm_head", c.sm_dim, c.num_classes);
      expect_ln("lg_head_norm", c.lg_dim); expect_dense("lg_head", c.lg_dim, c.num_classes);
    }
  }

  // finalize-time replacements of registered weights by derived device copies (head-padded kernels)
  std::map<std::string, const float*> woverride;
  const float* W(const std::string& name) const {
    auto ov = woverride.find(name);
    if (ov != woverride.end()) return ov->second;
    auto it = windex.find(name);
    VB_CHECK(it != windex.end(), "internal: unknown weight " + name);
    return weights[it->second].dev;
  }
  bool has(const std::string& name) const { return windex.count(name) != 0; }

  Linear make_linear(const std::string& n, int K, int N, bool bias = true, const Norm* fold = nullptr, int ldw_min = 0) {
    Linear L;
    L.W = W(n + ".kernel");
    L.bias = bias ? W(n + ".bias") : nullptr;
    L.K = K; L.N = N; L.ldw = round_up(K, 8) > ldw_min ? round_up(K, 8) : ldw_min;
    if (bf16()) {
      owned.emplace_back(new DevMem());
      owned.back()->ensure(static_cast<size_t>(N) * L.ldw * sizeof(__nv_bfloat16));
      L.Wt = static_cast<__nv_bfloat16*>(owned.back()->p);
      pack_weight_bf16(L.W, L.Wt, K, N, L.ldw, 0, fold ? fold->gamma : nullptr);
      if (fold) {
        owned.emplace_back(new DevMem());
        owned.back()->ensure(static_cast<size_t>(N) * 2 * sizeof(float));
        float* c = static_cast<float*>(owned.back()->p);
        ln_fold_consts(L.W, L.Wt, L.ldw, fold->beta, L.bias, c, c + N, K, N, 0);
        L.ln_c1 = c; L.ln_c2 = c + N;
      }
    }
    return L;
  }
  // Two bias-free Dense layers applied to the same input (CaiT to_q / to_kv on x, cait.py:114-119) as ONE wgmma GEMM:
  // the packed K-major weights and the LayerNorm-fold constants of `a` and `b` are laid out back to back, so the output
  // columns are [a | b] = [q | k | v], the layout the fused to_qkv of vit.py produces.  bf16 engine only.
  Linear make_linear_pair(const std::string& na, int NA, const std::string& nb, int NB, int K, const Norm* fold) {
    Linear L;
    L.W = nullptr; L.bias = nullptr;
    L.K = K; L.N = NA + NB; L.ldw = round_up(K, 8);
    owned.emplace_back(new DevMem());
    owned.back()->ensure(static_cast<size_t>(L.N) * L.ldw * sizeof(__nv_bfloat16));
    L.Wt = static_cast<__nv_bfloat16*>(owned.back()->p);
    float* c = nullptr;
    if (fold) {
      owned.emplace_back(new DevMem());
      owned.back()->ensure(static_cast<size_t>(L.N) * 2 * sizeof(float));
      c = static_cast<float*>(owned.back()->p);
      L.ln_c1 = c; L.ln_c2 = c + L.N;
    }
    const std::string names[2] = {na, nb};
    const int widths[2] = {NA, NB};
    int n0 = 0;
    for (int i = 0; i < 2; ++i) {
      const float* Wi = W(names[i] + ".kernel");
      __nv_bfloat16* Wti = L.Wt + static_cast<size_t>(n0) * L.ldw;
      pack_weight_bf16(Wi, Wti, K, widths[i], L.ldw, 0, fold ? fold->gamma : nullptr);
      if (fold) ln_fold_consts(Wi, Wti, L.ldw, fold->beta, nullptr, c + n0, c + L.N + n0, K, widths[i], 0);
      n0 += widths[i];
    }
    return L;
  }
  Norm make_norm(const std::string& n, int D) { return Norm{W(n + ".gamma"), W(n + ".beta"), D}; }
  // fold_ok: the layer is only ever used as a self-attention layer (its LayerNorms feed nothing but GEMMs)
  LayerW make_layer(const std::string& pre, int dim, int heads, int dh, int mlp, int kind, bool fold_ok = true) {
    LayerW l;
    l.dh_model = dh;
    // Plain softmax attention with dim_head < 64 (bf16 engine): widen every head to the fused attention kernel's 64 columns
    // with zero weights -- extra to_qkv / to_q / to_kv output columns (q, k, v pad columns are exactly 0, so QK^T and the
    // real PV columns are unchanged) and zero to_out input rows.  Costs (64 / dh - 1) more flops in those two GEMMs and buys
    // the tensor-core attention path for e.g. dim_head 48 / 32 (the head-mixing variants have their own kernel, attn_mix).
    const bool to_out_present = has(pre + "to_out.kernel");
    if (bf16() && dh < 64 && dh % 8 == 0 && to_out_present && dim % 8 == 0 && getenv("VB_NO_HEAD_PAD") == nullptr &&
        (kind == VB_KIND_VIT || kind == VB_KIND_CROSSVIT)) {
      const int dhp = 64;
      auto padded = [&](const std::string& n, int other, int groups, int pad_rows) {
        owned.emplace_back(new DevMem());
        owned.back()->ensure(static_cast<size_t>(other) * groups * heads * dhp * sizeof(float));
        float* wp = static_cast<float*>(owned.back()->p);
        pad_heads_f32(W(n), wp, other, groups, heads, dh, dhp, pad_rows, 0);
        woverride[n] = wp;
      };
      if (kind == VB_KIND_VIT) padded(pre + "to_qkv.kernel", dim, 3, 0);
      else { padded(pre + "to_q.kernel", dim, 1, 0); padded(pre + "to_kv.kernel", dim, 2, 0); }
      padded(pre + "to_out.kernel", dim, 1, 1);
      dh = dhp;
    }
    const int inner = heads * dh;
    l.heads = heads; l.dim_head = dh;
    l.attn_norm = make_norm(pre + "attn_norm", dim);
    l.ff_norm = make_norm(pre + "ff_norm", dim);
    // LayerNorm folding needs every GEMM of the layer on the wgmma path (all widths multiples of 64)
    l.folded = bf16() && fold_ok && dim % 64 == 0 && inner % 64 == 0 && mlp % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr;
    const Norm* fa = l.folded ? &l.attn_norm : nullptr;
    const Norm* ff = l.folded ? &l.ff_norm : nullptr;
    if (kind == VB_KIND_VIT || kind == VB_KIND_DEEPVIT) { l.fused_qkv = true; l.to_qkv = make_linear(pre + "to_qkv", dim, 3 * inner, false, fa); }
    else if (bf16() && fold_ok && dim % 8 == 0) {   // self-attention only: q and kv read the same rows -> one GEMM
      l.fused_qkv = true;
      l.to_qkv = make_linear_pair(pre + "to_q", inner, pre + "to_kv", 2 * inner, dim, fa);
    } else { l.to_q = make_linear(pre + "to_q", dim, inner, false, fa); l.to_kv = make_linear(pre + "to_kv", dim, 2 * inner, false, fa); }
    if (kind == VB_KIND_DEEPVIT) { l.variant = 1; l.mix_a = W(pre + "reattn_weights"); l.reattn_norm = make_norm(pre + "reattn_norm", heads); }
    if (kind == VB_KIND_CAIT) {
      l.variant = 2; l.mix_a = W(pre + "mix_pre"); l.mix_b = W(pre + "mix_post");
      l.attn_scale = W(pre + "attn_scale"); l.ff_scale = W(pre + "ff_scale");
    }
    l.project_out = has(pre + "to_out.kernel");
    if (l.project_out) l.to_out = make_linear(pre + "to_out", inner, dim);
    l.fc1 = make_linear(pre + "fc1", dim, mlp, true, ff);
    l.fc2 = make_linear(pre + "fc2", mlp, dim);
    return l;
  }
  // One-layer transformer between two T2T soft splits (t2t.py:35,45-46: heads = 1, dim_head = mlp_dim = dim = D = channels * prod(k^2),
  // 147 and 1323 at the default t2t_layers; no out-projection, vit.py:53) on the tensor cores: every width is zero-padded to
  // Dp = round_up(D, 64) -- token rows [n, Dp] with zero pad columns, to_qkv columns [q | k | v] each Dp wide, fc1 / fc2 Dp x Dp --
  // so that all four GEMMs and the per-image QK^T / PV products run on the wgmma GEMM kernel; LayerNorm and the softmax scale keep
  // the true D.  Zero weights and biases keep the pad columns exactly zero through the layer (GELU(0) = 0).
  static bool t2t_tensor_path_enabled() { static const bool off = getenv("VB_NO_T2T_TC") != nullptr; return !off; }
  LayerW make_t2t_layer(const std::string& pre, int D) {
    const int Dp = round_up(D, 64);
    auto padded = [&](const std::string& n, int other, int groups, int pad_rows, const float* src, int dh_src) {
      owned.emplace_back(new DevMem());
      owned.back()->ensure(static_cast<size_t>(other) * groups * Dp * sizeof(float));
      float* wp = static_cast<float*>(owned.back()->p);
      pad_heads_f32(src, wp, other, groups, 1, dh_src, Dp, pad_rows, 0);
      woverride[n] = wp;
      return wp;
    };
    padded(pre + "to_qkv.kernel", D, 3, 0, W(pre + "to_qkv.kernel"), D);                    // [D, 3 D] -> [D, 3 Dp]
    padded(pre + "fc1.kernel", D, 1, 0, W(pre + "fc1.kernel"), D);                          // [D, D] -> [D, Dp]
    padded(pre + "fc1.bias", 1, 1, 0, W(pre + "fc1.bias"), D);
    const float* rows_padded = padded(pre + "fc2.kernel", D, 1, 1, W(pre + "fc2.kernel"), D);   // [D, D] -> [Dp, D] (zero input rows)
    padded(pre + "fc2.kernel", Dp, 1, 0, rows_padded, D);                                   // -> [Dp, Dp]
    padded(pre + "fc2.bias", 1, 1, 0, W(pre + "fc2.bias"), D);
    LayerW l;
    l.heads = 1; l.dim_head = Dp; l.dh_model = D; l.t2t_D = D; l.t2t_Dp = Dp;
    l.attn_norm = make_norm(pre + "attn_norm", D);
    l.ff_norm = make_norm(pre + "ff_norm", D);
    l.fused_qkv = true; l.project_out = false;
    l.to_qkv = make_linear(pre + "to_qkv", D, 3 * Dp, false, nullptr, Dp);
    l.fc1 = make_linear(pre + "fc1", D, Dp, true, nullptr, Dp);
    l.fc2 = make_linear(pre + "fc2", Dp, Dp, true, nullptr, Dp);
    l.to_qkv.K = Dp; l.fc1.K = Dp;                                                        // the A operands are Dp wide (zero pad columns)
    return l;
  }
  // CCT TransformerEncoderLayer (cct.py:159-174): pre_norm folds into to_qkv as in make_layer; norm1 replaces the stream itself
  // (the fc2 residual is the normalised row), so it runs as a LayerNorm in place and fc1 reads the normalised rows unfolded.
  LayerW make_cct_layer(const std::string& pre, int dim, int heads, int mlp) {
    LayerW l;
    l.heads = heads; l.dim_head = dim / heads; l.dh_model = l.dim_head;
    l.attn_norm = make_norm(pre + "attn_norm", dim);
    l.ff_norm = make_norm(pre + "norm1", dim);
    l.folded = bf16() && dim % 64 == 0 && mlp % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr;   // every GEMM on the wgmma path
    l.fused_qkv = true;
    l.to_qkv = make_linear(pre + "to_qkv", dim, 3 * dim, false, l.folded ? &l.attn_norm : nullptr);
    l.to_out = make_linear(pre + "to_out", dim, dim);
    l.fc1 = make_linear(pre + "fc1", dim, mlp);
    l.fc2 = make_linear(pre + "fc2", mlp, dim);
    return l;
  }
  EmbedW make_embed(const std::string& pre, int p_h, int p_w, int dim, int n_pos, bool with_cls = true, int K = 0) {
    EmbedW e;
    e.patch = make_linear(pre + "patch", K > 0 ? K : p_h * p_w * cfg.channels, dim);
    e.pos = W(pre + "pos_embedding");
    e.cls = with_cls ? W(pre + "cls_token") : nullptr;   // CaiT adds its cls token after the patch stage (cait.py:189)
    e.dim = dim; e.n_pos = n_pos;
    return e;
  }

  void finalize() {
    for (auto& w : weights) VB_CHECK(w.set, "vb_finalize: weight '" + w.name + "' was never set");
    VB_CUDA(cudaSetDevice(device));
    owned.clear(); layers.clear(); cls_layers.clear(); t2t_layers.clear(); xblocks.clear(); plans.clear(); embed_res.clear(); cct_convs.clear();
    lv_stem.clear(); lv_blocks.clear(); cvt_stages.clear(); twins_stages.clear(); cf_stages.clear();
    woverride.clear();
    drop_graphs();
    const vb_config& c = cfg;
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_PARALLEL_VIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np + 1);
      for (int L = 0; L < c.depth; ++L) {
        if (c.kind == VB_KIND_PARALLEL_VIT) {   // `layers` holds depth x parallel_branches entries, branches of a layer adjacent
          for (int i = 0; i < c.parallel_branches; ++i)
            layers.push_back(make_layer("layers." + std::to_string(L) + ".branch" + std::to_string(i) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
        } else {
          layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, c.kind));
        }
      }
      head_norm = make_norm("head_norm", c.dim);
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_PATCH_MERGER_VIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np + 1, false);
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
      merger_norm = make_norm("patch_merger.norm", c.dim);
      merger_queries = W("patch_merger.queries");
      head_norm = make_norm("head_norm", c.dim);
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_T2T_VIT) {
      const auto st = t2t_stages();
      int out = c.image_h;
      for (size_t i = 0; i < st.size(); ++i) {
        out = conv_output_size(out, st[i].k, st[i].stride);
        if (i + 1 < st.size()) {
          const std::string pre = "t2t." + std::to_string(i) + ".layers.0.";
          if (bf16() && t2t_tensor_path_enabled()) t2t_layers.push_back(make_t2t_layer(pre, st[i].dim));
          else t2t_layers.push_back(make_layer(pre, st[i].dim, 1, st[i].dim, st[i].dim, VB_KIND_VIT, false));
        }
      }
      embed = make_embed("", 0, 0, c.dim, out * out + 1, true, st.back().dim);
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
      head_norm = make_norm("head_norm", c.dim);
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_CCT) {
      // the 4-D kernel [k, k, cin, cout] is the Dense [k*k*cin, cout] over unfold_same's (row, column, channel) vectors
      for (int i = 0; i < c.cct_conv_layers; ++i)
        cct_convs.push_back(make_linear("tokenizer.conv." + std::to_string(i), c.cct_kernel * c.cct_kernel * cct_conv_cin(i), cct_conv_cout(i), false));
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_cct_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.mlp_dim));
      cct_norm = make_norm("norm", c.dim);
      cct_pool_w = W("attention_pool.kernel");
      cct_pool_b = W("attention_pool.bias");
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_LEVIT) {
      finalize_levit();
    } else if (c.kind == VB_KIND_CVT) {
      finalize_cvt();
    } else if (c.kind == VB_KIND_TWINS_SVT) {
      finalize_twins();
    } else if (c.kind == VB_KIND_CROSSFORMER) {
      finalize_crossformer();
    } else if (c.kind == VB_KIND_CAIT) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np, false);
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_layer("patch_transformer.layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_CAIT));
      for (int L = 0; L < c.cls_depth; ++L) cls_layers.push_back(make_layer("cls_transformer.layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_CAIT, false));
      head_norm = make_norm("head_norm", c.dim);
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else {
      const int nps = (c.image_h / c.sm_patch_size) * (c.image_w / c.sm_patch_size);
      const int npl = (c.image_h / c.lg_patch_size) * (c.image_w / c.lg_patch_size);
      sm_embed = make_embed("sm_embed.", c.sm_patch_size, c.sm_patch_size, c.sm_dim, nps + 1);
      lg_embed = make_embed("lg_embed.", c.lg_patch_size, c.lg_patch_size, c.lg_dim, npl + 1);
      const int xinner = c.cross_attn_heads * c.cross_attn_dim_head;
      for (int D = 0; D < c.cross_depth; ++D) {
        XBlock xb;
        const std::string bp = "blocks." + std::to_string(D) + ".";
        for (int L = 0; L < c.sm_enc_depth; ++L) xb.sm_layers.push_back(make_layer(bp + "sm_enc.layers." + std::to_string(L) + ".", c.sm_dim, c.sm_enc_heads, c.sm_enc_dim_head, c.sm_enc_mlp_dim, VB_KIND_CROSSVIT));
        for (int L = 0; L < c.lg_enc_depth; ++L) xb.lg_layers.push_back(make_layer(bp + "lg_enc.layers." + std::to_string(L) + ".", c.lg_dim, c.lg_enc_heads, c.lg_enc_dim_head, c.lg_enc_mlp_dim, VB_KIND_CROSSVIT));
        xb.sm_final = make_norm(bp + "sm_enc.final_norm", c.sm_dim);
        xb.lg_final = make_norm(bp + "lg_enc.final_norm", c.lg_dim);
        for (int R = 0; R < c.cross_attn_depth; ++R) {
          for (int b = 0; b < 2; ++b) {
            const std::string n = bp + "cross." + std::to_string(R) + (b == 0 ? ".sm_attend_lg." : ".lg_attend_sm.");
            const int din = b == 0 ? c.sm_dim : c.lg_dim, dout = b == 0 ? c.lg_dim : c.sm_dim;
            CrossW x;
            x.proj = din != dout;
            if (x.proj) { x.project_in = make_linear(n + "project_in", din, dout); x.project_out = make_linear(n + "project_out", dout, din); }
            x.norm = make_norm(n + "norm", dout);
            x.to_q = make_linear(n + "to_q", dout, xinner, false);
            x.to_kv = make_linear(n + "to_kv", dout, 2 * xinner, false);
            x.to_out = make_linear(n + "to_out", xinner, dout);
            (b == 0 ? xb.sm_attend_lg : xb.lg_attend_sm).push_back(x);
          }
        }
        xblocks.push_back(std::move(xb));
      }
      sm_head_norm = make_norm("sm_head_norm", c.sm_dim); sm_head = make_linear_f32("sm_head", c.sm_dim, c.num_classes);
      lg_head_norm = make_norm("lg_head_norm", c.lg_dim); lg_head = make_linear_f32("lg_head", c.lg_dim, c.num_classes);
    }
    VB_CUDA(cudaDeviceSynchronize());
    finalized = true;
  }
  // ---- LeViT weight packing: BatchNormalization folded into the convolutions on the host in double, heads zero-padded
  std::vector<double> host_weight(const std::string& name) const {
    const Weight& w = weights[windex.at(name)];
    std::vector<float> f(w.count);
    VB_CUDA(cudaMemcpy(f.data(), w.dev, w.count * sizeof(float), cudaMemcpyDeviceToHost));
    return std::vector<double>(f.begin(), f.end());
  }
  // y = BN(x W + b) = x (W s) + ((b - mean) s + beta),  s = gamma / sqrt(var + 1e-5)  (levit.py:76, inference statistics)
  void fold_bn(std::vector<double>& Wkn, std::vector<double>& bias, int K, int N, const std::string& bn) const {
    const auto g = host_weight(bn + ".gamma"), be = host_weight(bn + ".beta"), mu = host_weight(bn + ".moving_mean"),
               var = host_weight(bn + ".moving_variance");
    for (int n = 0; n < N; ++n) {
      const double sc = g[n] / std::sqrt(var[n] + 1e-5);
      for (int k = 0; k < K; ++k) Wkn[static_cast<size_t>(k) * N + n] *= sc;
      bias[n] = (bias[n] - mu[n]) * sc + be[n];
    }
  }
  const float* upload_owned(const std::vector<double>& v) {
    std::vector<float> f(v.begin(), v.end());
    owned.emplace_back(new DevMem());
    owned.back()->ensure(f.size() * sizeof(float));
    VB_CUDA(cudaMemcpy(owned.back()->p, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice));
    return static_cast<const float*>(owned.back()->p);
  }
  // W [K, N] (Keras layout) as the top-left block of a zero [Kp, Np]
  static std::vector<double> pad_kn(const std::vector<double>& W, int K, int N, int Kp, int Np) {
    std::vector<double> out(static_cast<size_t>(Kp) * Np, 0.0);
    for (int k = 0; k < K; ++k)
      for (int n = 0; n < N; ++n) out[static_cast<size_t>(k) * Np + n] = W[static_cast<size_t>(k) * N + n];
    return out;
  }
  static std::vector<double> pad_n(const std::vector<double>& b, int Np) {
    std::vector<double> out(b);
    out.resize(Np, 0.0);
    return out;
  }
  // a Dense [K, N] + bias (none when `bias` is empty) made on the host, packed like a registered one (under a name of its own in
  // woverride), with the LayerNorm `fold` folded in when given
  Linear linear_from_host(const std::string& key, const std::vector<double>& Wkn, const std::vector<double>& bias, int K, int N,
                          const Norm* fold = nullptr) {
    woverride[key + ".kernel"] = upload_owned(Wkn);
    if (!bias.empty()) woverride[key + ".bias"] = upload_owned(bias);
    return make_linear(key, K, N, !bias.empty(), fold);
  }
  // ---- CvT weight packing: channel widths zero-padded (bf16), BatchNormalizations folded into the depthwise taps and a shift
  Norm padded_norm(const std::string& n, int d, int dp) {        // CvT's LayerNorm g / b [1, 1, 1, d] -> [dp]
    return Norm{upload_owned(pad_n(host_weight(n + ".g"), dp)), upload_owned(pad_n(host_weight(n + ".b"), dp)), d};
  }
  void finalize_cvt() {
    for (int st = 0; st < VB_CVT_STAGES; ++st) {
      CvtStageW S;
      const std::string p = cvt_pre(st);
      const int d = cv.emb_dim[st], dp = channel_width(d), ke = cv.emb_kernel[st], K = ke * ke * cvt_cin(st);
      S.dim = d; S.dp = dp; S.k = ke; S.stride = cv.emb_stride[st];
      S.conv = linear_from_host("cvt." + p + "0", pad_kn(host_weight(p + "0.kernel"), K, d, K, dp), pad_n(host_weight(p + "0.bias"), dp), K, dp);
      S.norm = padded_norm(p + "1", d, dp);
      const int inner = 64 * cv.heads[st], hidden = d * cv.mlp_mult[st], hp = channel_width(hidden), k = cv.proj_kernel[st];
      for (int L = 0; L < cv.depth[st]; ++L) {
        const std::string b = p + "2.layers." + std::to_string(L) + ".", key = "cvt." + b;
        CvtBlockW w;
        w.dim = d; w.dp = dp; w.heads = cv.heads[st]; w.k = k; w.kv_stride = cv.kv_proj_stride[st];
        w.attn_norm = padded_norm(b + "0.norm", d, dp);
        w.ff_norm = padded_norm(b + "1.norm", d, dp);
        for (int kv = 0; kv < 2; ++kv) {
          const std::string n = b + (kv ? "0.fn.to_kv.net." : "0.fn.to_q.net.");
          std::vector<double> taps, shift;
          cvt_fold_dw(host_weight(n + "0.kernel"), host_weight(n + "1.gamma"), host_weight(n + "1.beta"), host_weight(n + "1.moving_mean"),
                      host_weight(n + "1.moving_variance"), k, d, dp, taps, shift);
          const int N = (kv ? 2 : 1) * inner;
          Linear pw = linear_from_host(key + (kv ? "pw_kv" : "pw_q"), pad_kn(host_weight(n + "2.kernel"), d, N, dp, N), {}, dp, N);
          if (kv) { w.wkv = upload_owned(taps); w.bkv = upload_owned(shift); w.pw_kv = pw; }
          else { w.wq = upload_owned(taps); w.bq = upload_owned(shift); w.pw_q = pw; }
        }
        const std::string o = b + "0.fn.to_out.0", m0 = b + "1.fn.net.0", m3 = b + "1.fn.net.3";
        w.to_out = linear_from_host(key + "to_out", pad_kn(host_weight(o + ".kernel"), inner, d, inner, dp), pad_n(host_weight(o + ".bias"), dp),
                                    inner, dp);
        w.fc1 = linear_from_host(key + "fc1", pad_kn(host_weight(m0 + ".kernel"), d, hidden, dp, hp), pad_n(host_weight(m0 + ".bias"), hp), dp, hp,
                                 bf16() ? &w.ff_norm : nullptr);
        w.fc1.ln_d = d;
        w.fc1.ln_eps = 1e-5f;
        w.fc2 = linear_from_host(key + "fc2", pad_kn(host_weight(m3 + ".kernel"), hidden, d, hp, dp), pad_n(host_weight(m3 + ".bias"), dp), hp, dp);
        S.blocks.push_back(std::move(w));
      }
      cvt_stages.push_back(std::move(S));
    }
    head = make_linear_f32("cvt_layers.3.1", cv.emb_dim[VB_CVT_STAGES - 1], cfg.num_classes);
  }
  // ---- Twins-SVT weight packing: channel widths zero-padded (bf16), the patch kernel's rows permuted, the PEG residual folded
  // A PreNorm MLP of width 4 d: the LayerNorm `norm` (g / b), the Dense layers n0 (d -> 4 d) and n3 (4 d -> d) as 1x1 Conv2D
  // kernels, widths padded, the LayerNorm folded into fc1 in the bf16 engine.  key: the packed copies' own names.
  MlpW prenorm_mlp(const std::string& key, const std::string& norm, const std::string& n0, const std::string& n3, int d, int dp) {
    MlpW w;
    const int hidden = 4 * d, hp = channel_width(hidden);
    w.norm = padded_norm(norm, d, dp);
    w.fc1 = linear_from_host(key + n0, pad_kn(host_weight(n0 + ".kernel"), d, hidden, dp, hp), pad_n(host_weight(n0 + ".bias"), hp), dp,
                             hp, bf16() ? &w.norm : nullptr);
    w.fc1.ln_d = d;
    w.fc1.ln_eps = 1e-5f;
    w.fc2 = linear_from_host(key + n3, pad_kn(host_weight(n3 + ".kernel"), hidden, d, hp, dp), pad_n(host_weight(n3 + ".bias"), dp), hp, dp);
    return w;
  }
  MlpW twins_mlp(const std::string& m, int d, int dp) {
    return prenorm_mlp("twins.", m + ".fn.norm", m + ".fn.fn.net.0", m + ".fn.fn.net.3", d, dp);
  }
  TwinsLayerW twins_layer_weights(const std::string& b, int st, int d, int dp) {
    TwinsLayerW w;
    const int I = kTwinsInner, kg = tw.global_k[st];
    auto folded = [&](Linear L) { L.ln_d = d; L.ln_eps = 1e-5f; return L; };   // twins_svt.py:46: eps 1e-5
    auto to_out = [&](const std::string& n) {
      return linear_from_host("twins." + n, pad_kn(host_weight(n + ".kernel"), I, d, I, dp), pad_n(host_weight(n + ".bias"), dp), I, dp);
    };
    w.local = st < VB_TWINS_STAGES - 1;
    if (w.local) {
      w.local_norm = padded_norm(b + "0.fn.norm", d, dp);
      const auto q = host_weight(b + "0.fn.fn.to_q.kernel"), kv = host_weight(b + "0.fn.fn.to_kv.kernel");
      std::vector<double> qkv(static_cast<size_t>(d) * 3 * I);           // [d, q | k | v]
      for (int r = 0; r < d; ++r) {
        std::copy(q.begin() + static_cast<size_t>(r) * I, q.begin() + static_cast<size_t>(r + 1) * I, qkv.begin() + static_cast<size_t>(r) * 3 * I);
        std::copy(kv.begin() + static_cast<size_t>(r) * 2 * I, kv.begin() + static_cast<size_t>(r + 1) * 2 * I,
                  qkv.begin() + static_cast<size_t>(r) * 3 * I + I);
      }
      w.qkv = folded(linear_from_host("twins." + b + "0.qkv", pad_kn(qkv, d, 3 * I, dp, 3 * I), {}, dp, 3 * I, bf16() ? &w.local_norm : nullptr));
      w.local_out = to_out(b + "0.fn.fn.to_out.0");
      w.ff1 = twins_mlp(b + "1", d, dp);
    }
    w.global_norm = padded_norm(b + "2.fn.norm", d, dp);
    w.to_q = folded(linear_from_host("twins." + b + "2.to_q", pad_kn(host_weight(b + "2.fn.fn.to_q.kernel"), d, I, dp, I), {}, dp, I,
                                     bf16() ? &w.global_norm : nullptr));
    // [kg, kg, d, 2I] is the Dense [kg*kg*d, 2I] over unfold_same's (row, column, channel) vectors of the true d channels
    w.to_kv = linear_from_host("twins." + b + "2.to_kv", host_weight(b + "2.fn.fn.to_kv.kernel"), {}, kg * kg * d, 2 * I);
    w.global_out = to_out(b + "2.fn.fn.to_out.0");
    w.ff2 = twins_mlp(b + "3", d, dp);
    return w;
  }
  void finalize_twins() {
    for (int st = 0; st < VB_TWINS_STAGES; ++st) {
      TwinsStageW S;
      const std::string p = twins_pre(st);
      const int d = tw.emb_dim[st], dp = channel_width(d), ps = tw.patch_size[st], cin = twins_cin(st), K = ps * ps * cin, k = tw.peg_kernel_size;
      S.dim = d; S.dp = dp; S.patch = ps; S.local = tw.local_patch_size[st]; S.global_k = tw.global_k[st]; S.peg_k = k;
      // 'b (h p1) (w p2) c -> b h w (c p1 p2)' (twins_svt.py:103): the reference's row c * p^2 + p1 * p + p2 is unfold_same's
      // row (p1 * p + p2) * cin + c
      const auto wr = host_weight(p + "0.proj.kernel");
      std::vector<double> wp(static_cast<size_t>(K) * d);
      for (int c = 0; c < cin; ++c)
        for (int t = 0; t < ps * ps; ++t)
          std::copy(wr.begin() + static_cast<size_t>(c * ps * ps + t) * d, wr.begin() + static_cast<size_t>(c * ps * ps + t + 1) * d,
                    wp.begin() + static_cast<size_t>(t * cin + c) * d);
      S.proj = linear_from_host("twins." + p + "0.proj", pad_kn(wp, K, d, K, dp), pad_n(host_weight(p + "0.proj.bias"), dp), K, dp);
      // PEG (:108-115): x + dw(x) + b is one depthwise convolution whose centre tap ((k-1)/2, (k-1)/2) has 1 added (TF SAME at
      // stride 1 pads (k-1)/2 on the top / left, so that tap reads the pixel itself)
      const auto taps = host_weight(p + "2.proj.fn.kernel");
      std::vector<double> pw(static_cast<size_t>(k) * k * dp, 0.0);
      const int centre = ((k - 1) / 2) * k + (k - 1) / 2;
      for (int t = 0; t < k * k; ++t)
        for (int c = 0; c < d; ++c) pw[static_cast<size_t>(t) * dp + c] = taps[static_cast<size_t>(t) * d + c] + (t == centre ? 1.0 : 0.0);
      S.peg_w = upload_owned(pw);
      S.peg_b = upload_owned(pad_n(host_weight(p + "2.proj.fn.bias"), dp));
      for (int t : {1, 3})
        for (int L = 0; L < (t == 1 ? 1 : tw.depth[st]); ++L)
          (t == 1 ? S.pre : S.post).push_back(twins_layer_weights(p + std::to_string(t) + ".layers." + std::to_string(L) + ".", st, d, dp));
      twins_stages.push_back(std::move(S));
    }
    head = make_linear_f32("svt_layers.4.1", tw.emb_dim[VB_TWINS_STAGES - 1], cfg.num_classes);
  }
  // ---- CrossFormer weight packing: the nested cross-scale kernel, the DynamicPositionBias tables, channel widths zero-padded (bf16)
  // DynamicPositionBias (crossformer.py:51-71,158-165) on the offsets range(-w, w + 1)^2 in (row, column) order: 3 x [Dense ->
  // LayerNormalization (eps 1e-3) -> ReLU], Dense(1).  The reference indexes the result with rel_pos_indices (:126-131), whose
  // offset w - 1 and row pitch 2 w - 1 read only its first (2 w - 1)^2 entries: those are the table (PosBias::wsz).
  std::vector<double> cf_window_table(const std::string& n, int w, int d4) const {
    const int side = 2 * w + 1, t = (2 * w - 1) * (2 * w - 1);
    std::vector<double> Wl[4], bl[4], g[3], be[3];
    for (int i = 0; i < 4; ++i) { Wl[i] = host_weight(n + std::to_string(3 * i) + ".kernel"); bl[i] = host_weight(n + std::to_string(3 * i) + ".bias"); }
    for (int i = 0; i < 3; ++i) { g[i] = host_weight(n + std::to_string(3 * i + 1) + ".gamma"); be[i] = host_weight(n + std::to_string(3 * i + 1) + ".beta"); }
    std::vector<double> table(t);
    for (int e = 0; e < t; ++e) {
      std::vector<double> x = {static_cast<double>(e / side - w), static_cast<double>(e % side - w)};
      for (int i = 0; i < 4; ++i) {
        const int din = static_cast<int>(x.size()), dout = i == 3 ? 1 : d4;
        std::vector<double> y(bl[i].begin(), bl[i].end());
        for (int k = 0; k < din; ++k)
          for (int o = 0; o < dout; ++o) y[o] += x[k] * Wl[i][static_cast<size_t>(k) * dout + o];
        if (i < 3) {
          double mean = 0.0, var = 0.0;
          for (double v : y) mean += v;
          mean /= dout;
          for (double v : y) var += (v - mean) * (v - mean);
          const double rstd = 1.0 / std::sqrt(var / dout + 1e-3);
          for (int o = 0; o < dout; ++o) y[o] = std::max(0.0, (y[o] - mean) * rstd * g[i][o] + be[i][o]);
        }
        x.swap(y);
      }
      table[e] = x[0];
    }
    return table;
  }
  CrossformerAttnW cf_attention(const std::string& a, int d, int dp, int wsz, bool dilated) {
    CrossformerAttnW w;
    const int I = 32 * (d / 32), key_n = wsz == 1 ? I : 3 * I, N = bf16() ? round_up(key_n, 64) : key_n;
    w.wsz = wsz;
    w.dilated = dilated;
    w.norm = padded_norm(a + "norm", d, dp);
    auto qkv = host_weight(a + "to_qkv.kernel");                   // [d, q | k | v]
    if (wsz == 1) {                                                // softmax over one score is 1: only v is needed (its third)
      std::vector<double> v(static_cast<size_t>(d) * I);
      for (int r = 0; r < d; ++r)
        std::copy(qkv.begin() + static_cast<size_t>(r) * 3 * I + 2 * I, qkv.begin() + static_cast<size_t>(r + 1) * 3 * I, v.begin() + static_cast<size_t>(r) * I);
      qkv.swap(v);
    } else {
      w.table = upload_owned(cf_window_table(a + "dpb.dpb_layers.", wsz, d / 4));
    }
    w.qkv = linear_from_host("cf." + a + "qkv", pad_kn(qkv, d, key_n, dp, N), {}, dp, N, bf16() ? &w.norm : nullptr);
    w.qkv.ln_d = d;
    w.qkv.ln_eps = 1e-5f;                                          // crossformer.py:74
    w.to_out = linear_from_host("cf." + a + "to_out", pad_kn(host_weight(a + "to_out.kernel"), I, d, I, dp), pad_n(host_weight(a + "to_out.bias"), dp),
                                I, dp);
    return w;
  }
  void finalize_crossformer() {
    for (int st = 0; st < VB_CROSSFORMER_STAGES; ++st) {
      CrossformerStageW S;
      const std::string p = cf_pre(st);
      const int d = cf.dim[st], dp = channel_width(d), cin = cf_cin(st);
      const auto ks = cf_kernels(st), ds = cf_dim_scales(st);
      const int K = ks.back();
      S.dim = d; S.dp = dp; S.heads = d / 32; S.kmax = K; S.stride = cf.stride[st];
      // CrossEmbedLayer (:45-48) as one K x K convolution: kernel i sits at offset (K - k_i) / 2 of the K x K grid (TF SAME pads the
      // smaller half first; with equal parities and every k_i >= stride the offset is exact for any map), its outputs at columns
      // [sum of the earlier dim_scales, + ds[i]) -- the concat order
      std::vector<double> Wn(static_cast<size_t>(K) * K * cin * dp, 0.0), bn(dp, 0.0);
      int col0 = 0;
      for (size_t i = 0; i < ks.size(); ++i) {
        const std::string n = p + "0.convs." + std::to_string(i);
        const int k = ks[i], o = (K - k) / 2, dsi = ds[i];
        const auto wk = host_weight(n + ".kernel"), bk = host_weight(n + ".bias");
        for (int ky = 0; ky < k; ++ky)
          for (int kx = 0; kx < k; ++kx)
            for (int c = 0; c < cin; ++c)
              for (int oc = 0; oc < dsi; ++oc)
                Wn[((static_cast<size_t>(ky + o) * K + kx + o) * cin + c) * dp + col0 + oc] = wk[((static_cast<size_t>(ky) * k + kx) * cin + c) * dsi + oc];
        for (int oc = 0; oc < dsi; ++oc) bn[col0 + oc] = bk[oc];
        col0 += dsi;
      }
      S.embed = linear_from_host("cf." + p + "0", Wn, bn, K * K * cin, dp);
      for (int L = 0; L < cf.depth[st]; ++L) {
        const std::string b = p + "1.layers." + std::to_string(L) + ".";
        CrossformerLayerW l;
        l.short_attn = cf_attention(b + "0.", d, dp, cf.local_wsz[st], false);
        l.ff1 = prenorm_mlp("cf.", b + "1.net.0", b + "1.net.1", b + "1.net.4", d, dp);
        l.long_attn = cf_attention(b + "2.", d, dp, cf.global_wsz[st], true);
        l.ff2 = prenorm_mlp("cf.", b + "3.net.0", b + "3.net.1", b + "3.net.4", d, dp);
        S.layers.push_back(std::move(l));
      }
      cf_stages.push_back(std::move(S));
    }
    head = make_linear_f32("to_logits.1", cf.dim[VB_CROSSFORMER_STAGES - 1], cfg.num_classes);
  }
  void finalize_levit() {
    const int dh = levit_dh();
    int cin = cfg.channels;
    for (int i = 0; i < 4; ++i) {                                       // stem; the 32-channel map is written 64 wide (zero columns)
      const std::string n = "conv_embedding." + std::to_string(i);
      const int cout = levit_stem_cout(i), np = i == 0 ? 64 : channel_width(cout), K = 9 * cin;
      lv_stem.push_back(linear_from_host("levit." + n, pad_kn(host_weight(n + ".kernel"), K, cout, K, np),
                                         pad_n(host_weight(n + ".bias"), np), K, np));
      cin = cout;
    }
    for (const auto& p : levit_plan()) {
      LevitBlockW b;
      b.dim = p.dim; b.dim_out = p.dim_out; b.heads = p.heads; b.fmap = p.fmap; b.step = p.down ? 2 : 1; b.dh = dh;
      b.dp = channel_width(p.dim); b.dp_out = channel_width(p.dim_out);
      b.residual = !p.down && p.dim == p.dim_out;
      const std::string a = p.pre + "0.", key = "levit." + a;
      const int H = p.heads, dk = lv.dim_key, dv = lv.dim_value, HD = H * dh, dp = b.dp, dpo = b.dp_out;
      // one projection folded and head-padded: head h's real columns [h*dh, h*dh + w) of a [dp, H*dh] block (rows >= dim zero)
      auto proj = [&](const char* n, int w, std::vector<double>& Wcat, std::vector<double>& bcat, int off, int ncat) {
        auto Wn = host_weight(a + n + ".0.kernel");
        std::vector<double> bn(H * w, 0.0);
        fold_bn(Wn, bn, p.dim, H * w, a + n + ".1");
        for (int h = 0; h < H; ++h)
          for (int d = 0; d < w; ++d) {
            const int src = h * w + d, dst = off + h * dh + d;
            for (int k = 0; k < p.dim; ++k) Wcat[static_cast<size_t>(k) * ncat + dst] = Wn[static_cast<size_t>(k) * H * w + src];
            bcat[dst] = bn[src];
          }
      };
      const int nkv = p.down ? 2 * HD : 3 * HD, koff = p.down ? 0 : HD;
      std::vector<double> Wkv(static_cast<size_t>(dp) * nkv, 0.0), bkv(nkv, 0.0);
      if (!p.down) proj("to_q", dk, Wkv, bkv, 0, nkv);
      proj("to_k", dk, Wkv, bkv, koff, nkv);
      proj("to_v", dv, Wkv, bkv, koff + HD, nkv);
      b.qkv = linear_from_host(key + "qkv", Wkv, bkv, dp, nkv);
      if (p.down) {
        std::vector<double> Wq(static_cast<size_t>(dp) * HD, 0.0), bq(HD, 0.0);
        proj("to_q", dk, Wq, bq, 0, HD);
        b.q = linear_from_host(key + "q", Wq, bq, dp, HD);
      }
      {                                                                 // to_out: GELU -> Conv2D(1x1, bias) -> BN (levit.py:93-98)
        auto Wo = host_weight(a + "to_out.1.kernel"), bo = host_weight(a + "to_out.1.bias");
        fold_bn(Wo, bo, H * dv, p.dim_out, a + "to_out.2");
        std::vector<double> Wp(static_cast<size_t>(HD) * dpo, 0.0);
        for (int h = 0; h < H; ++h)
          for (int d = 0; d < dv; ++d)
            for (int o = 0; o < p.dim_out; ++o)
              Wp[(static_cast<size_t>(h) * dh + d) * dpo + o] = Wo[(static_cast<size_t>(h) * dv + d) * p.dim_out + o];
        b.to_out = linear_from_host(key + "to_out", Wp, pad_n(bo, dpo), HD, dpo);
      }
      b.scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(dk)));
      b.pos = upload_owned(levit_pos_table(host_weight(a + "pos_bias.embeddings"), p.fmap * p.fmap, H, dk));
      const int hidden = p.dim_out * p.mult, hp = channel_width(hidden);
      const std::string m0 = p.pre + "1.net.0", m3 = p.pre + "1.net.3";
      b.fc1 = linear_from_host(key + "fc1", pad_kn(host_weight(m0 + ".kernel"), p.dim_out, hidden, dpo, hp), pad_n(host_weight(m0 + ".bias"), hp),
                               dpo, hp);
      b.fc2 = linear_from_host(key + "fc2", pad_kn(host_weight(m3 + ".kernel"), hidden, p.dim_out, hp, dpo), pad_n(host_weight(m3 + ".bias"), dpo),
                               hp, dpo);
      lv_blocks.push_back(std::move(b));
    }
    const int dl = lv.dims[lv.stages - 1];
    head = make_linear_f32("mlp_head", dl, cfg.num_classes);
    if (lv.num_distill_classes > 0) lv_distill = make_linear_f32("distill_head", dl, lv.num_distill_classes);
  }
  // [heads][fmap^2] = embeddings[e, h] / scale with scale = dim_key^-0.5 (levit.py:117): the table the attention kernels add
  static std::vector<double> levit_pos_table(const std::vector<double>& emb, int f2, int heads, int dim_key) {
    std::vector<double> t(static_cast<size_t>(heads) * f2);
    const double inv_scale = std::sqrt(static_cast<double>(dim_key));
    for (int h = 0; h < heads; ++h)
      for (int e = 0; e < f2; ++e) t[static_cast<size_t>(h) * f2 + e] = emb[static_cast<size_t>(e) * heads + h] * inv_scale;
    return t;
  }

  Linear make_linear_f32(const std::string& n, int K, int N) {  // classifier head always runs in fp32
    Linear L;
    L.W = W(n + ".kernel"); L.bias = W(n + ".bias"); L.K = K; L.N = N; L.ldw = K;
    return L;
  }

  // ---------------------------------------------------------------- ops
  template <typename T>
  void linear(const T* A, int lda, int M, const Linear& L, T* out, int ldc, const Epi& e, cudaStream_t s);

  template <typename T>
  void attention(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq, int nk,
                 const LayerW& l, cudaStream_t s) {
    const float scale = l.dh_model != l.dim_head ? 1.0f / sqrtf(static_cast<float>(l.dh_model)) : 0.f;
    attention_dispatch<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, l.heads, l.dim_head, l.variant, l.mix_a, l.mix_b,
                          l.reattn_norm.gamma, l.reattn_norm.beta, s, scale);
  }
  template <typename T>
  void attention_dispatch(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq, int nk,
                          int heads, int dh, int variant, const float* mix_a, const float* mix_b, const float* g, const float* b,
                          cudaStream_t s, float scale = 0.f, const Window* win = nullptr, const PosBias* pb = nullptr);

  template <typename T>
  const T* embed_residual(const EmbedW& e, int B, int rows, cudaStream_t s) {
    ResKey key{&e, B, rows};
    auto it = embed_res.find(key);
    if (it == embed_res.end()) {
      // one entry per (embedding, batch, rows) actually in use; a server that sweeps batch / image sizes must not grow
      // without bound (77 MB per ViT-B/16 B=256 entry): beyond a handful of shapes start over
      if (embed_res.size() >= 6) { VB_CUDA(cudaStreamSynchronize(s)); embed_res.clear(); drop_graphs(); }
      std::unique_ptr<DevMem> m(new DevMem());
      m->ensure(static_cast<size_t>(B) * rows * e.dim * sizeof(T));
      build_embed_residual<T>(static_cast<T*>(m->p), e.pos, e.cls, e.patch.bias, B, rows, e.dim, e.cls != nullptr, s);
      it = embed_res.emplace(key, std::move(m)).first;
    }
    return static_cast<const T*>(it->second->p);
  }

  // patch embedding + cls token + pos embedding -> X [B*rows, dim]   (vit.py:160-165 / cait.py:181-184)
  template <typename T>
  T* embed_tokens(const EmbedW& e, const float* img, int B, int H, int Wd, int ph, int pw, int* rows_out, cudaStream_t s,
                  float** stats_out = nullptr) {
    VB_CHECK(H % ph == 0 && Wd % pw == 0, "Image dimensions must be divisible by the patch size.");
    const int np = (H / ph) * (Wd / pw);
    const int has_cls = e.cls != nullptr ? 1 : 0;
    const int rows = np + has_cls;
    VB_CHECK(rows <= e.n_pos, "image has more patches than pos_embedding rows");
    const int Kp = bf16() ? e.patch.ldw : e.patch.K;
    const int M = B * rows;
    T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, 4.0 * B * H * Wd * cfg.channels + static_cast<double>(sizeof(T)) * M * Kp, s);
      im2col<T>(img, col, B, H, Wd, cfg.channels, ph, pw, has_cls, Kp, s);
    }
    *rows_out = rows;
    return embed_from_cols<T>(e, col, Kp, B, rows, s, stats_out);
  }
  // X = cols . W + bias + (pos (+ cls on row 0)): the Dense of the patch embedding with cls concat and positions folded
  // into its residual operand.  cols [B*rows, Kp]: patch vectors, zero in the cls rows and in the pad columns.
  template <typename T>
  T* embed_from_cols(const EmbedW& e, const T* col, int Kp, int B, int rows, cudaStream_t s, float** stats_out) {
    const int M = B * rows;
    const T* R = embed_residual<T>(e, B, rows, s);
    T* X = arena.get<T>(static_cast<size_t>(M) * e.dim);
    Epi ep; ep.bias = e.patch.bias; ep.res = R; ep.ldr = e.dim;
    if (stats_out != nullptr && bf16() && e.dim % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr) {
      *stats_out = arena.get<float>(static_cast<size_t>(M) * (e.dim / 64) * 2);
      ep.stats_out = *stats_out;
    }
    Linear L = e.patch;
    L.K = Kp;  // im2col zero-pads the patch vector to the packed weight pitch
    linear<T>(col, Kp, M, L, X, e.dim, ep, s);
    return X;
  }

  // T2TViT.patch_embedding + cls + positions (t2t.py:58-74,97-103): soft split i = unfold_same over the previous token map
  // (the image for i = 0), every split but the last followed by a one-layer transformer of width channels * prod(k^2);
  // the last split writes the im2col operand of the Dense(dim) directly (cls rows / pad columns zero).
  template <typename T>
  T* embed_t2t(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s, float** stats_out) {
    const auto st = t2t_stages();
    const T* map = nullptr;
    int mh = H, mw = Wd, mc = cfg.channels, map_ld = 0;
    for (size_t i = 0; i < st.size(); ++i) {
      const int oh = (mh + st[i].stride - 1) / st[i].stride, ow = (mw + st[i].stride - 1) / st[i].stride;
      const int D = st[i].dim, n = oh * ow;
      VB_CHECK(i == 0 || mh == mw, "T2TViT: token maps after the first soft split must be square (t2t.py:41)");
      const bool last = i + 1 == st.size();
      const bool tc = !last && t2t_layers[i].t2t_Dp > 0;               // tensor-core layer: token rows padded to Dp columns
      const int ld = last ? (bf16() ? embed.patch.ldw : embed.patch.K) : (tc ? t2t_layers[i].t2t_Dp : D);
      const int cls_row = last ? 1 : 0;
      T* out = arena.get<T>(static_cast<size_t>(B) * (n + cls_row) * ld);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(i == 0 ? 4 : sizeof(T)) * B * mh * mw * mc + static_cast<double>(sizeof(T)) * B * (n + cls_row) * ld, s);
        if (i == 0) unfold_same<float, T>(img, out, B, mh, mw, mc, st[i].k, st[i].stride, cls_row, ld, s);
        else unfold_same<T, T>(map, out, B, mh, mw, mc, st[i].k, st[i].stride, cls_row, ld, s, map_ld);
      }
      if (last) {
        VB_CHECK(n + 1 <= embed.n_pos, "image has more patches than pos_embedding rows");
        *rows_out = n + 1;
        return embed_from_cols<T>(embed, out, ld, B, n + 1, s, stats_out);
      }
      if (tc) layer_t2t<T>(out, B, n, t2t_layers[i], s);
      else layer_self<T>(out, B, n, D, t2t_layers[i], s);
      map = out; mh = oh; mw = ow; mc = D; map_ld = ld;
    }
    VB_CHECK(false, "T2TViT needs at least one t2t layer");
    return nullptr;
  }

  // CCT Tokenizer + positional embedding (cct.py:211-215,278-286): per conv layer, unfold_same of the previous map (the fp32
  // image first) into the Dense operand (zero-padded to the packed weight pitch), the GEMM, then ReLU + SAME max-pool.  The last
  // pool adds the positions ('sine' / 'learnable') or writes zero rows up to sequence_length ('none').  -> X [B*rows, dim]
  template <typename T>
  T* tokenize_cct(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s) {
    const vb_config& c = cfg;
    const T* map = nullptr;
    T* out = nullptr;
    int mh = H, mw = Wd, mc = c.channels;
    for (int i = 0; i < c.cct_conv_layers; ++i) {
      const Linear& conv = cct_convs[i];
      const int oh = (mh + c.cct_stride - 1) / c.cct_stride, ow = (mw + c.cct_stride - 1) / c.cct_stride;
      const int M = B * oh * ow, Kp = bf16() ? conv.ldw : conv.K;
      T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(i == 0 ? 4 : sizeof(T)) * B * mh * mw * mc + static_cast<double>(sizeof(T)) * M * Kp, s);
        if (i == 0) unfold_same<float, T>(img, col, B, mh, mw, mc, c.cct_kernel, c.cct_stride, 0, Kp, s);
        else unfold_same<T, T>(map, col, B, mh, mw, mc, c.cct_kernel, c.cct_stride, 0, Kp, s);
      }
      T* conv_out = arena.get<T>(static_cast<size_t>(M) * conv.N);
      Linear L = conv;
      L.K = Kp;
      linear<T>(col, Kp, M, L, conv_out, conv.N, Epi(), s);
      const int ph = (oh + c.cct_pool_stride - 1) / c.cct_pool_stride, pw = (ow + c.cct_pool_stride - 1) / c.cct_pool_stride;
      int rows = ph * pw;
      const float* pos = nullptr;
      if (i + 1 == c.cct_conv_layers) {
        const int n_seq = cct_sequence_length();
        if (c.cct_pos_emb != VB_CCT_POS_NONE) {                          // cct.py:286: x += positional_emb must broadcast
          VB_CHECK(rows == n_seq, "CCT: the image gives " + std::to_string(rows) + " tokens but the positional embedding has " +
                                  std::to_string(n_seq) + " rows (with 'sine' / 'learnable' the image must give img_size's token count)");
          pos = W("positional_emb");
        } else if (rows < n_seq) {
          rows = n_seq;                                                  // cct.py:278-280: zero rows up to sequence_length
        }
      }
      out = arena.get<T>(static_cast<size_t>(B) * rows * conv.N);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, static_cast<double>(sizeof(T)) * (static_cast<double>(M) + static_cast<double>(B) * rows) * conv.N, s);
        maxpool_relu_same<T>(conv_out, out, B, oh, ow, conv.N, c.cct_pool_kernel, c.cct_pool_stride, pos, rows, s);
      }
      map = out; mh = ph; mw = pw; mc = conv.N;
      *rows_out = rows;
    }
    return out;
  }

  // `call` up to the transformer for every kind with one token stream
  template <typename T>
  T* embed_any(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s, float** stats_out) {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT has two token streams: no single embedding stage");
    if (cfg.kind == VB_KIND_T2T_VIT) return embed_t2t<T>(img, B, H, Wd, rows_out, s, stats_out);
    return embed_tokens<T>(embed, img, B, H, Wd, cfg.patch_h, cfg.patch_w, rows_out, s, stats_out);
  }

  // PatchMerger.call (vit_with_patch_merger.py:49-55) = single-head attention of nt learned queries over LN(x) with
  // keys = values = LN(x) and scale dim^-0.5 (:45) -- exactly attention with heads = 1, dim_head = dim.
  template <typename T>
  T* patch_merge(const T* X, int B, int rows, int dim, const Norm& norm, const float* queries, int nt, cudaStream_t s) {
    T* Y = arena.get<T>(static_cast<size_t>(B) * rows * dim);
    ln<T>(X, norm, Y, B * rows, dim, s);
    T* Q = arena.get<T>(static_cast<size_t>(B) * nt * dim);
    broadcast_rows<T>(queries, Q, B, nt, dim, s);
    T* O = arena.get<T>(static_cast<size_t>(B) * nt * dim);
    attention_dispatch<T>(Q, dim, Y, dim, Y, dim, O, dim, B, nt, rows, 1, dim, 0, nullptr, nullptr, nullptr, nullptr, s);
    return O;
  }

  // wgmma GEMM on raw operands through the plan cache (the T2T soft-split attention products)
  void gemm_cached(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, int b_rows, void* out, int ldc, int M, int N, int K,
                   const __nv_bfloat16* res, int ldr, bool out_f32, int cls, cudaStream_t s) {
    ProfScope ps(this, cls, 2.0 * M * N * K, 2.0 * (static_cast<double>(M) * K + static_cast<double>(N) * K) + (out_f32 ? 4.0 : 2.0) * M * N, s);
    PlanKey key{};
    const uintptr_t parts[16] = {reinterpret_cast<uintptr_t>(A), static_cast<uintptr_t>(lda), reinterpret_cast<uintptr_t>(Wt),
                                 reinterpret_cast<uintptr_t>(out), static_cast<uintptr_t>(ldc), static_cast<uintptr_t>(M),
                                 static_cast<uintptr_t>(N), static_cast<uintptr_t>(K), static_cast<uintptr_t>(ldw),
                                 static_cast<uintptr_t>(b_rows), reinterpret_cast<uintptr_t>(res), static_cast<uintptr_t>(ldr),
                                 static_cast<uintptr_t>(out_f32), 0x7247u, 0, 0};
    for (int i = 0; i < 16; ++i) key[i] = parts[i];
    auto it = plans.find(key);
    if (it == plans.end()) {
      if (plans.size() > 8192) plans.clear();
      it = plans.emplace(key, gemm_bf16_plan(A, lda, Wt, ldw, static_cast<__nv_bfloat16*>(out), ldc, M, N, K, nullptr, nullptr, res, ldr,
                                             false, out_f32, b_rows)).first;
    }
    gemm_bf16_run(it->second, s);
  }

  // One T2T soft-split transformer layer on the tensor cores (see make_t2t_layer).  X [B*n, Dp] bf16, zero pad columns, updated
  // in place.  Attention with ONE head of width D = 147 / 1323 over n = 3136 / 784 tokens (t2t.py:35) does not fit the fused
  // attention kernels' head widths: per image, S = Q K^T (wgmma GEMM, fp32 out), softmax rows -> bf16 P, O = P V (wgmma GEMM
  // against V^T, residual X added in its epilogue).  The score / probability buffers of ONE image (39 + 20 MB at n = 3136) are
  // reused for every image, so at n = 784 (4 MB) they stay in the 50 MB L2 instead of streaming B x n x n floats through HBM.
  template <typename T>
  void layer_t2t(T* X, int B, int n, const LayerW& l, cudaStream_t s);

  // one pre-norm layer, self-attention over all rows (vit.py:101-102, cait.py:150-151, cross_vit.py:109-111).
  // `stats` (bf16 engine, folded layers): per-row (sum, sumsq) partials of X, valid on entry iff *stats_valid; the
  // residual GEMMs keep them up to date, so no LayerNorm kernel runs at all.
  template <typename T>
  void layer_self(T* X, int B, int rows, int dim, const LayerW& l, cudaStream_t s, float* stats = nullptr,
                  bool* stats_valid = nullptr) {
    const int M = B * rows, inner = l.heads * l.dim_head;
    const bool fold = l.folded && stats != nullptr;
    if (fold && !*stats_valid) { ensure_stats(X, dim, stats, M, s); *stats_valid = true; }
    T* Y = arena.get<T>(static_cast<size_t>(M) * dim);
    T* O = arena.get<T>(static_cast<size_t>(M) * inner);
    const T* A = X;
    Epi eq;
    if (fold) eq.ln_stats = stats;
    else { VB_CHECK(!l.folded, "internal: folded layer without statistics"); ln<T>(X, l.attn_norm, Y, M, dim, s); A = Y; }
    if (l.fused_qkv) {
      T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * inner);
      Epi e = eq; e.bias = l.to_qkv.ln_c2;
      linear<T>(A, dim, M, l.to_qkv, QKV, 3 * inner, e, s);
      attention<T>(QKV, 3 * inner, QKV + inner, 3 * inner, QKV + 2 * inner, 3 * inner, O, inner, B, rows, rows, l, s);
    } else {
      T* Q = arena.get<T>(static_cast<size_t>(M) * inner);
      T* KV = arena.get<T>(static_cast<size_t>(M) * 2 * inner);
      Epi e1 = eq; e1.bias = l.to_q.ln_c2;
      Epi e2 = eq; e2.bias = l.to_kv.ln_c2;
      linear<T>(A, dim, M, l.to_q, Q, inner, e1, s);
      linear<T>(A, dim, M, l.to_kv, KV, 2 * inner, e2, s);
      attention<T>(Q, inner, KV, 2 * inner, KV + inner, 2 * inner, O, inner, B, rows, rows, l, s);
    }
    if (l.project_out) {
      Epi e; e.bias = l.to_out.bias; e.scale = l.attn_scale; e.res = X; e.ldr = dim;
      if (fold) e.stats_out = stats;
      linear<T>(O, inner, M, l.to_out, X, dim, e, s);
    } else {
      add_tokens<T>(X, O, static_cast<long long>(M) * dim, s);   // vit.py:53: identity out-projection
      if (fold) ensure_stats(X, dim, stats, M, s);
    }
    feed_forward<T>(X, M, dim, l, Y, s, fold ? stats : nullptr);
  }
  // One CCT TransformerEncoderLayer (cct.py:159-174, dropout / drop-path the identity):
  //   x = x + proj(MHA(pre_norm(x)));  x = norm1(x);  x = x + linear2(GELU(linear1(x)))
  // pre_norm is folded into to_qkv through the row statistics (bf16 engine); norm1 rewrites the rows in place, and fc2, whose
  // residual is those normalised rows, emits the statistics the next layer's fold reads.
  template <typename T>
  void layer_cct(T* X, int B, int rows, int dim, const LayerW& l, cudaStream_t s, float* stats, bool* stats_valid) {
    const int M = B * rows, inner = l.heads * l.dim_head;
    const bool fold = l.folded && stats != nullptr;
    if (fold && !*stats_valid) { ensure_stats(X, dim, stats, M, s); *stats_valid = true; }
    T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * inner);
    T* O = arena.get<T>(static_cast<size_t>(M) * inner);
    const T* A = X;
    Epi eq;
    if (fold) { eq.ln_stats = stats; eq.bias = l.to_qkv.ln_c2; }
    else {
      VB_CHECK(!l.folded, "internal: folded layer without statistics");
      T* Y = arena.get<T>(static_cast<size_t>(M) * dim);
      ln<T>(X, l.attn_norm, Y, M, dim, s);
      A = Y;
    }
    linear<T>(A, dim, M, l.to_qkv, QKV, 3 * inner, eq, s);
    attention<T>(QKV, 3 * inner, QKV + inner, 3 * inner, QKV + 2 * inner, 3 * inner, O, inner, B, rows, rows, l, s);
    Epi e; e.bias = l.to_out.bias; e.res = X; e.ldr = dim;
    linear<T>(O, inner, M, l.to_out, X, dim, e, s);
    ln<T>(X, l.ff_norm, X, M, dim, s);                                  // cct.py:165: the stream is replaced by norm1(x)
    T* Hb = arena.get<T>(static_cast<size_t>(M) * l.fc1.N);
    Epi e1; e1.gelu = true; e1.bias = l.fc1.bias;
    linear<T>(X, dim, M, l.fc1, Hb, l.fc1.N, e1, s);
    Epi e2; e2.bias = l.fc2.bias; e2.res = X; e2.ldr = dim;
    if (fold) e2.stats_out = stats;
    linear<T>(Hb, l.fc1.N, M, l.fc2, X, dim, e2, s);
  }
  // One parallel_vit layer (parallel_vit.py:114-117): x = sum_i attn_i(LN_i(x)) + x ; x = sum_i ff_i(LN'_i(x)) + x.
  // Every branch reads the SAME x, so the sums accumulate in a second buffer through the residual epilogue of the
  // branch's last GEMM (branch 0: res = x, out = acc; branch i > 0: res = out = acc); the attention half goes X -> Acc, the
  // feed-forward half Acc -> X.  The branches' LayerNorms share the row statistics of x, so folding still applies.
  template <typename T>
  void layer_parallel(T* X, T* Acc, int B, int rows, int dim, const LayerW* br, int nbr, cudaStream_t s, float* stats, bool* stats_valid) {
    const int M = B * rows, inner = br[0].heads * br[0].dim_head;
    const bool fold = br[0].folded && stats != nullptr;
    if (fold && !*stats_valid) { ensure_stats(X, dim, stats, M, s); *stats_valid = true; }
    T* Y = arena.get<T>(static_cast<size_t>(M) * dim);
    T* O = arena.get<T>(static_cast<size_t>(M) * inner);
    T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * inner);
    T* Hb = arena.get<T>(static_cast<size_t>(M) * br[0].fc1.N);
    // ---- attention branches: X -> Acc
    for (int i = 0; i < nbr; ++i) {
      const LayerW& l = br[i];
      const T* A = X;
      Epi eq;
      if (fold) { eq.ln_stats = stats; eq.bias = l.to_qkv.ln_c2; }
      else { VB_CHECK(!l.folded, "internal: folded layer without statistics"); ln<T>(X, l.attn_norm, Y, M, dim, s); A = Y; }
      linear<T>(A, dim, M, l.to_qkv, QKV, 3 * inner, eq, s);
      attention<T>(QKV, 3 * inner, QKV + inner, 3 * inner, QKV + 2 * inner, 3 * inner, O, inner, B, rows, rows, l, s);
      const bool last = i == nbr - 1;
      if (l.project_out) {
        Epi e; e.bias = l.to_out.bias; e.res = i == 0 ? X : Acc; e.ldr = dim;
        if (fold && last) e.stats_out = stats;
        linear<T>(O, inner, M, l.to_out, Acc, dim, e, s);
      } else {                                               // parallel_vit.py:74: Identity out-projection (inner == dim)
        if (i == 0) VB_CUDA(cudaMemcpyAsync(Acc, X, static_cast<size_t>(M) * dim * sizeof(T), cudaMemcpyDeviceToDevice, s));
        add_tokens<T>(Acc, O, static_cast<long long>(M) * dim, s);
        if (fold && last) ensure_stats(Acc, dim, stats, M, s);
      }
    }
    // ---- feed-forward branches: Acc -> X
    for (int i = 0; i < nbr; ++i) {
      const LayerW& l = br[i];
      const T* A = Acc;
      Epi e1; e1.gelu = true;
      if (fold) { e1.ln_stats = stats; e1.bias = l.fc1.ln_c2; }
      else { ln<T>(Acc, l.ff_norm, Y, M, dim, s); A = Y; e1.bias = l.fc1.bias; }
      linear<T>(A, dim, M, l.fc1, Hb, l.fc1.N, e1, s);
      Epi e2; e2.bias = l.fc2.bias; e2.res = i == 0 ? Acc : X; e2.ldr = dim;
      if (fold && i == nbr - 1) e2.stats_out = stats;
      linear<T>(Hb, l.fc1.N, M, l.fc2, X, dim, e2, s);
    }
  }
  template <typename T>
  void ensure_stats(const T* X, int dim, float* stats, int M, cudaStream_t s);
  template <typename T>
  void ln(const T* x, const Norm& n, T* y, int M, int dim, cudaStream_t s) {
    ProfScope ps(this, PROF_LN, 0.0, 2.0 * sizeof(T) * M * dim, s);
    layernorm<T>(x, dim, n.gamma, n.beta, y, dim, M, dim, s);
  }
  template <typename T>
  void feed_forward(T* X, int M, int dim, const LayerW& l, T* Y, cudaStream_t s, float* stats = nullptr) {
    T* Hb = arena.get<T>(static_cast<size_t>(M) * l.fc1.N);
    Epi e1; e1.gelu = true;
    const T* A = X;
    if (stats != nullptr) { e1.ln_stats = stats; e1.bias = l.fc1.ln_c2; }
    else { VB_CHECK(!l.folded, "internal: folded layer without statistics"); ln<T>(X, l.ff_norm, Y, M, dim, s); A = Y; e1.bias = l.fc1.bias; }
    linear<T>(A, dim, M, l.fc1, Hb, l.fc1.N, e1, s);
    Epi e2; e2.bias = l.fc2.bias; e2.scale = l.ff_scale; e2.res = X; e2.ldr = dim;
    e2.stats_out = stats;
    linear<T>(Hb, l.fc1.N, M, l.fc2, X, dim, e2, s);
  }
  template <typename T>
  void add_tokens(T* X, const T* O, long long count, cudaStream_t s);

  // CaiT class-attention layer: x [B,1,dim] attends over [LN(x) ; patches] (cait.py:57-58,109-112,150-151)
  template <typename T>
  void layer_cls(T* Cx, T* ctx, int B, int nctx, int dim, const LayerW& l, cudaStream_t s) {
    const int inner = l.heads * l.dim_head;
    T* Yc = arena.get<T>(static_cast<size_t>(B) * dim);
    layernorm<T>(Cx, dim, l.attn_norm.gamma, l.attn_norm.beta, Yc, dim, B, dim, s);
    copy_tokens<T>(Yc, 1, 0, ctx, nctx, 0, 1, B, dim, s);
    T* Q = arena.get<T>(static_cast<size_t>(B) * inner);
    T* KV = arena.get<T>(static_cast<size_t>(B) * nctx * 2 * inner);
    T* O = arena.get<T>(static_cast<size_t>(B) * inner);
    linear<T>(Yc, dim, B, l.to_q, Q, inner, Epi(), s);
    linear<T>(ctx, dim, B * nctx, l.to_kv, KV, 2 * inner, Epi(), s);
    attention<T>(Q, inner, KV, 2 * inner, KV + inner, 2 * inner, O, inner, B, 1, nctx, l, s);
    Epi e; e.bias = l.to_out.bias; e.scale = l.attn_scale; e.res = Cx; e.ldr = dim;
    linear<T>(O, inner, B, l.to_out, Cx, dim, e, s);
    feed_forward<T>(Cx, B, dim, l, Yc, s);
  }

  // CrossViT: cls [B,dcls] attends over [LN(Pin(cls)) ; other-branch patches]  (cross_vit.py:128-138,69-93,159-160)
  template <typename T>
  void cross_attend(T* cls, int dcls, T* ctx, int nctx, int dctx, const CrossW& x, int B, cudaStream_t s) {
    const int heads = cfg.cross_attn_heads, dh = cfg.cross_attn_dim_head, inner = heads * dh;
    T* xp = cls;
    if (x.proj) {
      xp = arena.get<T>(static_cast<size_t>(B) * dctx);
      Epi e; e.bias = x.project_in.bias;
      linear<T>(cls, dcls, B, x.project_in, xp, dctx, e, s);
    }
    T* y = arena.get<T>(static_cast<size_t>(B) * dctx);
    layernorm<T>(xp, dctx, x.norm.gamma, x.norm.beta, y, dctx, B, dctx, s);
    copy_tokens<T>(y, 1, 0, ctx, nctx, 0, 1, B, dctx, s);
    T* Q = arena.get<T>(static_cast<size_t>(B) * inner);
    T* KV = arena.get<T>(static_cast<size_t>(B) * nctx * 2 * inner);
    T* O = arena.get<T>(static_cast<size_t>(B) * inner);
    linear<T>(y, dctx, B, x.to_q, Q, inner, Epi(), s);
    linear<T>(ctx, dctx, B * nctx, x.to_kv, KV, 2 * inner, Epi(), s);
    attention_dispatch<T>(Q, inner, KV, 2 * inner, KV + inner, 2 * inner, O, inner, B, 1, nctx, heads, dh, 0, nullptr, nullptr,
                          nullptr, nullptr, s);
    if (x.proj) {
      T* a = arena.get<T>(static_cast<size_t>(B) * dctx);
      Epi e1; e1.bias = x.to_out.bias;
      linear<T>(O, inner, B, x.to_out, a, dctx, e1, s);
      Epi e2; e2.bias = x.project_out.bias; e2.res = cls; e2.ldr = dcls;
      linear<T>(a, dctx, B, x.project_out, cls, dcls, e2, s);
    } else {
      Epi e; e.bias = x.to_out.bias; e.res = cls; e.ldr = dcls;
      linear<T>(O, inner, B, x.to_out, cls, dcls, e, s);
    }
  }

  template <typename T>
  void classify(const T* X, int rows, int dim, const Norm& hn, const Linear& hd, int B, int mean_pool, float* logits,
                bool accumulate, cudaStream_t s) {
    float* z = arena.get<float>(static_cast<size_t>(B) * dim);
    pool_layernorm<T>(X, rows, dim, hn.gamma, hn.beta, z, B, dim, mean_pool, s);
    gemm_simt<float, float, float>(z, dim, hd.W, hd.N, 1, logits, hd.N, B, hd.N, dim, hd.bias, nullptr,
                                   accumulate ? logits : nullptr, hd.N, 0, s);
  }

  // Images are independent, so a large batch can run as two half-batches on two streams (the forward's own and `half_stream`,
  // forked / joined with timing-less events and therefore part of a captured graph): while one half's kernel drains -- last
  // epilogues, CTAs finishing at different times, the dependent launch waiting for the whole grid -- the other half's next
  // kernel already has CTAs on the freed SMs.  Results are bit-identical to the unsplit forward (every kernel's tile
  // arithmetic is independent of the batch, tests: test_batch_independence_and_determinism).  ViT, DeepViT and CaiT only (T2T
  // and CrossViT fork streams of their own).
  // The split doubles the number of launches (half the tiles per kernel); its speed on the H100 is not measured.  Off by
  // default (VB_FWD_STREAMS=2 enables it).
  template <typename T>
  void forward_impl(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    arena.reset();
    static const char* fs_env = getenv("VB_FWD_STREAMS");
    const int want = fs_env != nullptr ? atoi(fs_env) : VB_FWD_STREAMS;
    const bool split = want >= 2 && !profiling && bf16() && B >= 2 * VB_FWD_SPLIT_MIN_HALF &&
                       (cfg.kind == VB_KIND_VIT || cfg.kind == VB_KIND_DEEPVIT || cfg.kind == VB_KIND_CAIT);
    if (!split) { forward_body<T>(img, B, H, Wd, logits, s); return; }
    ensure_side_streams();
    const int B0 = (B + 1) / 2;
    VB_CUDA(cudaEventRecord(fwd_fork_event, s));
    VB_CUDA(cudaStreamWaitEvent(half_stream, fwd_fork_event, 0));
    forward_body<T>(img, B0, H, Wd, logits, s);
    forward_body<T>(img + static_cast<size_t>(B0) * H * Wd * cfg.channels, B - B0, H, Wd, logits + static_cast<size_t>(B0) * cfg.num_classes, half_stream);
    VB_CUDA(cudaEventRecord(fwd_join_event, half_stream));
    VB_CUDA(cudaStreamWaitEvent(s, fwd_join_event, 0));
  }

  template <typename T>
  void forward_body(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    const vb_config& c = cfg;
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_T2T_VIT) {
      int rows = 0;
      float* stats = nullptr;
      T* X = embed_any<T>(img, B, H, Wd, &rows, s, &stats);
      bool sv = stats != nullptr;
      for (const auto& l : layers) layer_self<T>(X, B, rows, c.dim, l, s, stats, &sv);
      classify<T>(X, rows, c.dim, head_norm, head, B, c.pool == VB_POOL_MEAN, logits, false, s);
    } else if (c.kind == VB_KIND_PATCH_MERGER_VIT) {   // vit_with_patch_merger.py:174-185, Transformer.call :118-126
      int rows = 0;
      float* stats = nullptr;
      T* X = embed_tokens<T>(embed, img, B, H, Wd, c.patch_h, c.patch_w, &rows, s, &stats);
      bool sv = stats != nullptr;
      for (int L = 0; L < c.depth; ++L) {
        layer_self<T>(X, B, rows, c.dim, layers[L], s, stats, &sv);
        if (L == c.patch_merge_layer_index) {
          X = patch_merge<T>(X, B, rows, c.dim, merger_norm, merger_queries, c.patch_merge_num_tokens, s);
          rows = c.patch_merge_num_tokens;
          sv = false;                                    // new token rows: the row statistics are recomputed by the next layer
        }
      }
      classify<T>(X, rows, c.dim, head_norm, head, B, 1, logits, false, s);   // Reduce('b n d -> b d', 'mean') :169
    } else if (c.kind == VB_KIND_PARALLEL_VIT) {
      int rows = 0;
      float* stats = nullptr;
      T* X = embed_tokens<T>(embed, img, B, H, Wd, c.patch_h, c.patch_w, &rows, s, &stats);
      bool sv = stats != nullptr;
      T* Acc = arena.get<T>(static_cast<size_t>(B) * rows * c.dim);
      for (int L = 0; L < c.depth; ++L)
        layer_parallel<T>(X, Acc, B, rows, c.dim, &layers[static_cast<size_t>(L) * c.parallel_branches], c.parallel_branches, s, stats, &sv);
      classify<T>(X, rows, c.dim, head_norm, head, B, c.pool == VB_POOL_MEAN, logits, false, s);
    } else if (c.kind == VB_KIND_CAIT) {
      int rows = 0;
      float* stats = nullptr;
      T* X = embed_tokens<T>(embed, img, B, H, Wd, c.patch_h, c.patch_w, &rows, s, &stats);
      bool sv = stats != nullptr;
      for (const auto& l : layers) layer_self<T>(X, B, rows, c.dim, l, s, stats, &sv);
      T* Cx = arena.get<T>(static_cast<size_t>(B) * c.dim);
      broadcast_row<T>(W("cls_token"), Cx, 1, B, c.dim, s);
      T* ctx = arena.get<T>(static_cast<size_t>(B) * (rows + 1) * c.dim);
      copy_tokens<T>(X, rows, 0, ctx, rows + 1, 1, rows, B, c.dim, s);
      for (const auto& l : cls_layers) layer_cls<T>(Cx, ctx, B, rows + 1, c.dim, l, s);
      classify<T>(Cx, 1, c.dim, head_norm, head, B, 0, logits, false, s);
    } else if (c.kind == VB_KIND_LEVIT) {
      levit_forward<T>(img, B, H, Wd, logits, nullptr, s);
    } else if (c.kind == VB_KIND_CVT) {
      cvt_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_TWINS_SVT) {
      twins_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_CROSSFORMER) {
      crossformer_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_CCT) {                   // CCT.call cct.py:342-345, TransformerClassifier.call :277-305
      int rows = 0;
      T* X = tokenize_cct<T>(img, B, H, Wd, &rows, s);
      float* stats = (bf16() && c.dim % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr)
                         ? arena.get<float>(static_cast<size_t>(B) * rows * (c.dim / 64) * 2) : nullptr;
      bool sv = false;
      for (const auto& l : layers) layer_cct<T>(X, B, rows, c.dim, l, s, stats, &sv);
      float* z = arena.get<float>(static_cast<size_t>(B) * c.dim);
      {
        ProfScope ps(this, PROF_LN, 4.0 * B * rows * c.dim, static_cast<double>(sizeof(T)) * B * rows * c.dim, s);
        seq_pool<T>(X, rows, c.dim, cct_norm.gamma, cct_norm.beta, cct_pool_w, cct_pool_b, z, B, s);   // :291-299
      }
      gemm_simt<float, float, float>(z, c.dim, head.W, head.N, 1, logits, head.N, B, head.N, c.dim, head.bias, nullptr, nullptr,
                                     head.N, 0, s);                                                   // fc :303
    } else {
      int ns = 0, nl = 0;
      float *st_s = nullptr, *st_g = nullptr;
      T* S = embed_tokens<T>(sm_embed, img, B, H, Wd, c.sm_patch_size, c.sm_patch_size, &ns, s, &st_s);
      T* G = embed_tokens<T>(lg_embed, img, B, H, Wd, c.lg_patch_size, c.lg_patch_size, &nl, s, &st_g);
      bool sv_s = st_s != nullptr, sv_g = st_g != nullptr;
      T* sm_cls = arena.get<T>(static_cast<size_t>(B) * c.sm_dim);
      T* lg_cls = arena.get<T>(static_cast<size_t>(B) * c.lg_dim);
      T* ctx_lg = arena.get<T>(static_cast<size_t>(B) * nl * c.lg_dim);   // [LN(Pin(sm_cls)) ; lg patches]
      T* ctx_sm = arena.get<T>(static_cast<size_t>(B) * ns * c.sm_dim);   // [LN(Pin(lg_cls)) ; sm patches]
      // The two towers of a multi-scale block are independent until the cross-attention (cross_vit.py:185-190): the large-patch
      // tower (n = 17 at the README configuration: GEMMs of a few tiles) runs on a side stream beside the small-patch one, forked
      // and joined with timing-less events (part of the captured graph).  VB_CROSSVIT_STREAMS=1 keeps one stream.
      static const char* xs_env = getenv("VB_CROSSVIT_STREAMS");
      const bool two = (xs_env != nullptr ? atoi(xs_env) : 2) >= 2 && !profiling && bf16();
      cudaStream_t sg = s;
      if (two) { ensure_side_streams(); sg = side_streams[0]; }
      for (const auto& xb : xblocks) {
        if (two) { VB_CUDA(cudaEventRecord(fork_event, s)); VB_CUDA(cudaStreamWaitEvent(sg, fork_event, 0)); }
        for (const auto& l : xb.sm_layers) layer_self<T>(S, B, ns, c.sm_dim, l, s, st_s, &sv_s);
        layernorm<T>(S, c.sm_dim, xb.sm_final.gamma, xb.sm_final.beta, S, c.sm_dim, B * ns, c.sm_dim, s);
        for (const auto& l : xb.lg_layers) layer_self<T>(G, B, nl, c.lg_dim, l, sg, st_g, &sv_g);
        layernorm<T>(G, c.lg_dim, xb.lg_final.gamma, xb.lg_final.beta, G, c.lg_dim, B * nl, c.lg_dim, sg);
        sv_s = sv_g = false;   // the trailing LayerNorm and the cls write-back below change the token rows
        copy_tokens<T>(G, nl, 0, lg_cls, 1, 0, 1, B, c.lg_dim, sg);
        copy_tokens<T>(G, nl, 1, ctx_lg, nl, 1, nl - 1, B, c.lg_dim, sg);
        if (two) { VB_CUDA(cudaEventRecord(join_events[0], sg)); VB_CUDA(cudaStreamWaitEvent(s, join_events[0], 0)); }
        copy_tokens<T>(S, ns, 0, sm_cls, 1, 0, 1, B, c.sm_dim, s);
        copy_tokens<T>(S, ns, 1, ctx_sm, ns, 1, ns - 1, B, c.sm_dim, s);
        for (size_t R = 0; R < xb.sm_attend_lg.size(); ++R) {
          cross_attend<T>(sm_cls, c.sm_dim, ctx_lg, nl, c.lg_dim, xb.sm_attend_lg[R], B, s);
          cross_attend<T>(lg_cls, c.lg_dim, ctx_sm, ns, c.sm_dim, xb.lg_attend_sm[R], B, s);
        }
        copy_tokens<T>(sm_cls, 1, 0, S, ns, 0, 1, B, c.sm_dim, s);
        copy_tokens<T>(lg_cls, 1, 0, G, nl, 0, 1, B, c.lg_dim, s);
      }
      classify<T>(S, ns, c.sm_dim, sm_head_norm, sm_head, B, 0, logits, false, s);
      classify<T>(G, nl, c.lg_dim, lg_head_norm, lg_head, B, 0, logits, true, s);
    }
  }

  // LeViT.call (levit.py:214-226): stem -> backbone -> GlobalAvgPool2D -> mlp_head (and distill_head when distill != null).
  // The token rows of every block are the NHWC map, pixel-major: row b * fmap^2 + r * fmap + c.
  static constexpr const char* kLevitNoStages = "LeViT runs as a whole forward only: its stem / backbone / head stages have no entry of their own";
  template <typename T>
  void levit_forward(const float* img, int B, int H, int Wd, float* logits, float* distill, cudaStream_t s) {
    const int fmap = cfg.image_h / 16;
    int mh = H, mw = Wd, mc = cfg.channels, ld_in = 0;
    for (int i = 0; i < 4; ++i) { mh = (mh + 1) / 2; mw = (mw + 1) / 2; }
    VB_CHECK(mh == fmap && mw == fmap, "LeViT: an " + std::to_string(H) + " x " + std::to_string(Wd) + " image gives a " + std::to_string(mh) +
                                       " x " + std::to_string(mw) + " feature map after the four stride-2 stem convolutions, but the "
                                       "position biases are built for " + std::to_string(fmap) + " x " + std::to_string(fmap) +
                                       " (image_size // 16, levit.py:194)");
    mh = H; mw = Wd;
    const T* map = nullptr;
    T* X = nullptr;
    for (int i = 0; i < 4; ++i) {                                       // conv_embedding levit.py:187-192
      const Linear& conv = lv_stem[i];
      const int oh = (mh + 1) / 2, ow = (mw + 1) / 2, M = B * oh * ow, Kp = bf16() ? conv.ldw : conv.K;
      T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(i == 0 ? 4 : sizeof(T)) * B * mh * mw * mc + static_cast<double>(sizeof(T)) * M * Kp, s);
        if (i == 0) unfold_same<float, T>(img, col, B, mh, mw, mc, 3, 2, 0, Kp, s);
        else unfold_same<T, T>(map, col, B, mh, mw, mc, 3, 2, 0, Kp, s, ld_in);
      }
      X = arena.get<T>(static_cast<size_t>(M) * conv.N);
      Linear L = conv;
      L.K = Kp;
      Epi e; e.bias = conv.bias;
      linear<T>(col, Kp, M, L, X, conv.N, e, s);
      map = X; mh = oh; mw = ow; mc = levit_stem_cout(i); ld_in = conv.N;
    }
    int f = fmap;
    for (const auto& b : lv_blocks) {
      X = levit_block<T>(X, B, b, s);
      f = (b.fmap + b.step - 1) / b.step;
    }
    const int dl = lv.dims[lv.stages - 1], ldl = channel_width(dl);
    float* z = arena.get<float>(static_cast<size_t>(B) * dl);
    {
      ProfScope ps(this, PROF_LN, 1.0 * B * f * f * dl, static_cast<double>(sizeof(T)) * B * f * f * dl, s);
      pool_layernorm<T>(X, f * f, ldl, nullptr, nullptr, z, B, dl, 1, s);  // GlobalAvgPool2D (levit.py:206-208)
    }
    gemm_simt<float, float, float>(z, dl, head.W, head.N, 1, logits, head.N, B, head.N, dl, head.bias, nullptr, nullptr, head.N, 0, s);
    if (distill != nullptr)
      gemm_simt<float, float, float>(z, dl, lv_distill.W, lv_distill.N, 1, distill, lv_distill.N, B, lv_distill.N, dl, lv_distill.bias,
                                     nullptr, nullptr, lv_distill.N, 0, s);
  }
  // One LeViT block (levit.py:156-162): x = attn(x) + (x if attn_residual else 0); x = mlp(x) + x.  X [B * fmap^2, dp] ->
  // [B * nq, dp_out] (a new buffer when the block shrinks the map, X updated in place otherwise); pad columns stay zero.
  template <typename T>
  T* levit_block(T* X, int B, const LevitBlockW& b, cudaStream_t s) {
    const int f2 = b.fmap * b.fmap, nqs = (b.fmap + b.step - 1) / b.step, nq = nqs * nqs, HD = b.heads * b.dh;
    const int Mk = B * f2, Mq = B * nq;
    T* O = arena.get<T>(static_cast<size_t>(Mq) * HD);
    PosBias pb;
    pb.table = b.pos; pb.fmap = b.fmap; pb.step = b.step; pb.gelu_out = true;
    if (b.step == 1) {
      T* QKV = arena.get<T>(static_cast<size_t>(Mk) * 3 * HD);
      Epi e; e.bias = b.qkv.bias;
      linear<T>(X, b.dp, Mk, b.qkv, QKV, 3 * HD, e, s);
      attention_bias<T>(QKV, 3 * HD, QKV + HD, 3 * HD, QKV + 2 * HD, 3 * HD, O, HD, B, nq, f2, b, pb, s);
    } else {                                                            // queries of the even pixels (1x1 conv, stride 2, VALID)
      T* Xq = arena.get<T>(static_cast<size_t>(Mq) * b.dp);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * Mq * b.dp, s);
        gather_grid<T>(X, b.dp, Xq, b.dp, B, b.fmap, b.fmap, b.dp, b.step, s);
      }
      T* Q = arena.get<T>(static_cast<size_t>(Mq) * HD);
      T* KV = arena.get<T>(static_cast<size_t>(Mk) * 2 * HD);
      Epi eq; eq.bias = b.q.bias;
      linear<T>(Xq, b.dp, Mq, b.q, Q, HD, eq, s);
      Epi ek; ek.bias = b.qkv.bias;
      linear<T>(X, b.dp, Mk, b.qkv, KV, 2 * HD, ek, s);
      attention_bias<T>(Q, HD, KV, 2 * HD, KV + HD, 2 * HD, O, HD, B, nq, f2, b, pb, s);
    }
    T* Y = b.residual ? X : arena.get<T>(static_cast<size_t>(Mq) * b.dp_out);
    Epi eo; eo.bias = b.to_out.bias;
    if (b.residual) { eo.res = X; eo.ldr = b.dp; }
    linear<T>(O, HD, Mq, b.to_out, Y, b.dp_out, eo, s);
    T* Hb = arena.get<T>(static_cast<size_t>(Mq) * b.fc1.N);
    Epi e1; e1.hswish = true; e1.bias = b.fc1.bias;
    linear<T>(Y, b.dp_out, Mq, b.fc1, Hb, b.fc1.N, e1, s);
    Epi e2; e2.bias = b.fc2.bias; e2.res = Y; e2.ldr = b.dp_out;
    linear<T>(Hb, b.fc1.N, Mq, b.fc2, Y, b.dp_out, e2, s);
    return Y;
  }
  template <typename T>
  void attention_bias(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq, int nk,
                      const LevitBlockW& b, const PosBias& pb, cudaStream_t s) {
    ProfScope ps(this, PROF_ATTN, 4.0 * B * b.heads * nq * nk * b.dh, static_cast<double>(sizeof(T)) * B * b.heads * b.dh * (2.0 * nq + 2.0 * nk), s);
    if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, b.heads, b.dh, 0, nullptr, nullptr, nullptr, nullptr, s, b.scale, &pb))
      return;
    float* S = arena.get<float>(static_cast<size_t>(B) * b.heads * nq * ((nk + 15) & ~15));
    attention_generic<T>(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, b.heads, b.dh, 0, nullptr, nullptr, nullptr, nullptr, s, b.scale, &pb);
  }

  // CvT.call (cvt.py:182-202): per stage, Conv2D (SAME, bias) -> LayerNorm -> blocks; then GlobalAvgPool2D -> Dense.  Token rows
  // are the NHWC map, pixel-major, channel widths zero-padded to channel_width.  Any h x w: each SAME stride gives ceil.
  static constexpr const char* kCvtNoStages = "CvT runs as a whole forward only: its stem / stage / head steps have no entry of their own";
  template <typename T>
  void cvt_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    int mh = H, mw = Wd, mc = cfg.channels, ld_in = 0;
    const T* map = nullptr;
    T* X = nullptr;
    for (const CvtStageW& S : cvt_stages) {
      const int oh = (mh + S.stride - 1) / S.stride, ow = (mw + S.stride - 1) / S.stride, M = B * oh * ow;
      const int Kp = bf16() ? S.conv.ldw : S.conv.K;
      T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(map == nullptr ? 4 : sizeof(T)) * B * mh * mw * mc +
                                                 static_cast<double>(sizeof(T)) * M * Kp, s);
        if (map == nullptr) unfold_same<float, T>(img, col, B, mh, mw, mc, S.k, S.stride, 0, Kp, s);
        else unfold_same<T, T>(map, col, B, mh, mw, mc, S.k, S.stride, 0, Kp, s, ld_in);
      }
      T* Y = arena.get<T>(static_cast<size_t>(M) * S.dp);
      Linear L = S.conv;
      L.K = Kp;
      Epi e; e.bias = S.conv.bias;
      linear<T>(col, Kp, M, L, Y, S.dp, e, s);
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = bf16() ? arena.get<float>(static_cast<size_t>(M) * (S.dp / 64) * 2) : nullptr;
      {
        ProfScope ps(this, PROF_LN, 8.0 * M * S.dim, 2.0 * sizeof(T) * M * S.dp, s);
        layernorm<T>(Y, S.dp, S.norm.gamma, S.norm.beta, X, S.dp, M, S.dim, s, S.dp, 1e-5f);   // cvt.py:188
      }
      if (bf16()) ensure_stats<T>(X, S.dp, stats, M, s);               // the first block's PreNorm statistics
      for (const CvtBlockW& b : S.blocks) cvt_block<T>(X, B, oh, ow, b, stats, s);
      map = X; mh = oh; mw = ow; mc = S.dim; ld_in = S.dp;
    }
    const int dl = cv.emb_dim[VB_CVT_STAGES - 1];
    float* z = arena.get<float>(static_cast<size_t>(B) * dl);
    {
      ProfScope ps(this, PROF_LN, 1.0 * B * mh * mw * dl, static_cast<double>(sizeof(T)) * B * mh * mw * dl, s);
      pool_layernorm<T>(X, mh * mw, ld_in, nullptr, nullptr, z, B, dl, 1, s);   // GlobalAvgPool2D cvt.py:196
    }
    gemm_simt<float, float, float>(z, dl, head.W, head.N, 1, logits, head.N, B, head.N, dl, head.bias, nullptr, nullptr, head.N, 0, s);
  }
  // One CvT layer (cvt.py:144-145): x = attn(LN(x)) + x; x = mlp(LN(x)) + x, in place on X [B*H*W, dp].  bf16: `stats` holds the
  // (sum, sumsq) partials of X's rows on entry and on exit (emitted by the residual epilogues), and the depthwise kernel and fc1
  // apply the LayerNorms from them; fp32: separate LayerNorms.
  template <typename T>
  void cvt_block(T* X, int B, int H, int Wd, const CvtBlockW& b, float* stats, cudaStream_t s) {
    const int dp = b.dp, HD = 64 * b.heads, st = b.kv_stride;
    const int Ho = (H + st - 1) / st, Wo = (Wd + st - 1) / st, M = B * H * Wd, Mk = B * Ho * Wo;
    T* Qd = arena.get<T>(static_cast<size_t>(M) * dp);
    T* KVd = arena.get<T>(static_cast<size_t>(Mk) * dp);
    T* Y = bf16() ? nullptr : arena.get<T>(static_cast<size_t>(M) * dp);
    if (Y != nullptr) {                                                 // fp32: PreNorm LayerNorm of the attention (cvt.py:53)
      ProfScope ps(this, PROF_LN, 8.0 * M * b.dim, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(X, dp, b.attn_norm.gamma, b.attn_norm.beta, Y, dp, M, b.dim, s, dp, 1e-5f);
    }
    {
      ProfScope ps(this, PROF_OTHER, 2.0 * b.k * b.k * b.dim * (static_cast<double>(M) + Mk),
                   static_cast<double>(sizeof(T)) * dp * (2.0 * M + Mk) + (stats ? 8.0 * M * (dp / 64) : 0.0), s);
      dwconv_qkv<T>(Y ? Y : X, dp, Y ? nullptr : stats, b.attn_norm.gamma, b.attn_norm.beta, b.dim, 1e-5f, b.wq, b.bq, Qd, dp, b.wkv, b.bkv,
                    KVd, dp, B, H, Wd, dp, b.k, st, s);
    }
    T* Q = arena.get<T>(static_cast<size_t>(M) * HD);
    T* KV = arena.get<T>(static_cast<size_t>(Mk) * 2 * HD);
    linear<T>(Qd, dp, M, b.pw_q, Q, HD, Epi(), s);                      // cvt.py:86 (no bias)
    linear<T>(KVd, dp, Mk, b.pw_kv, KV, 2 * HD, Epi(), s);
    T* O = arena.get<T>(static_cast<size_t>(M) * HD);
    attention_dispatch<T>(Q, HD, KV, 2 * HD, KV + HD, 2 * HD, O, HD, B, H * Wd, Ho * Wo, b.heads, 64, 0, nullptr, nullptr, nullptr, nullptr, s);
    Epi eo; eo.bias = b.to_out.bias; eo.res = X; eo.ldr = dp; eo.stats_out = stats;
    linear<T>(O, HD, M, b.to_out, X, dp, eo, s);
    const T* fin = X;
    if (Y != nullptr) {
      ProfScope ps(this, PROF_LN, 8.0 * M * b.dim, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(X, dp, b.ff_norm.gamma, b.ff_norm.beta, Y, dp, M, b.dim, s, dp, 1e-5f);
      fin = Y;
    }
    T* Hb = arena.get<T>(static_cast<size_t>(M) * b.fc1.N);
    Epi e1; e1.gelu = true;
    if (Y == nullptr) { e1.bias = b.fc1.ln_c2; e1.ln_stats = stats; } else { e1.bias = b.fc1.bias; }
    linear<T>(fin, dp, M, b.fc1, Hb, b.fc1.N, e1, s);
    Epi e2; e2.bias = b.fc2.bias; e2.res = X; e2.ldr = dp; e2.stats_out = stats;
    linear<T>(Hb, b.fc1.N, M, b.fc2, X, dp, e2, s);
  }

  // TwinsSVT.call (twins_svt.py:266-268): per stage, PatchEmbedding -> Transformer(1) -> PEG -> Transformer(depth); then
  // GlobalAvgPool2D -> Dense.  Token rows are the NHWC map, pixel-major, channel widths zero-padded to channel_width; no stage
  // permutes its map.  bf16: `stats` holds the (sum, sumsq) partials of X's rows between sub-blocks (emitted by the patch
  // embedding's and the residual GEMMs' epilogues, and after the PEG by a row-statistics pass).
  static constexpr const char* kTwinsNoStages =
      "Twins-SVT runs as a whole forward only: its patch-embedding / stage / head steps have no entry of their own";
  // The reference's shape rules (twins_svt.py:103,141,168 through einops and Keras), checked before anything runs.
  void twins_check_size(int H, int Wd) const {
    int h = H, w = Wd;
    for (int st = 0; st < VB_TWINS_STAGES; ++st) {
      const std::string where = "Twins-SVT stage " + std::to_string(st + 1) + ": the " + std::to_string(h) + " x " + std::to_string(w) + " map ";
      const int ps = tw.patch_size[st], pl = tw.local_patch_size[st], kg = tw.global_k[st];
      VB_CHECK(h % ps == 0 && w % ps == 0, where + "is not divisible by patch_size " + std::to_string(ps));
      h /= ps; w /= ps;
      const std::string after = "Twins-SVT stage " + std::to_string(st + 1) + ": the " + std::to_string(h) + " x " + std::to_string(w) + " map ";
      VB_CHECK(st == VB_TWINS_STAGES - 1 || (h % pl == 0 && w % pl == 0),
               after + "is not divisible by local_patch_size " + std::to_string(pl));
      VB_CHECK(h >= kg && w >= kg, after + "is smaller than global_k " + std::to_string(kg) + " (a VALID convolution)");
    }
  }
  template <typename T>
  void twins_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    twins_check_size(H, Wd);
    int mh = H, mw = Wd, mc = cfg.channels, ld_in = 0;
    const T* map = nullptr;
    T* X = nullptr;
    for (const TwinsStageW& S : twins_stages) {
      const int oh = mh / S.patch, ow = mw / S.patch, M = B * oh * ow;
      const int Kp = bf16() ? S.proj.ldw : S.proj.K;
      T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(map == nullptr ? 4 : sizeof(T)) * B * mh * mw * mc +
                                                 static_cast<double>(sizeof(T)) * M * Kp, s);
        if (map == nullptr) unfold_same<float, T>(img, col, B, mh, mw, mc, S.patch, S.patch, 0, Kp, s);
        else unfold_same<T, T>(map, col, B, mh, mw, mc, S.patch, S.patch, 0, Kp, s, ld_in);
      }
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = bf16() ? arena.get<float>(static_cast<size_t>(M) * (S.dp / 64) * 2) : nullptr;
      Linear L = S.proj;
      L.K = Kp;
      Epi e; e.bias = S.proj.bias; e.stats_out = stats;
      linear<T>(col, Kp, M, L, X, S.dp, e, s);
      for (const TwinsLayerW& l : S.pre) twins_layer<T>(X, B, oh, ow, S, l, stats, s);
      T* Y = arena.get<T>(static_cast<size_t>(M) * S.dp);             // the PEG's halo reads the unmodified map
      {
        ProfScope ps(this, PROF_OTHER, 2.0 * S.peg_k * S.peg_k * M * S.dim, 2.0 * sizeof(T) * M * S.dp, s);
        dwconv_qkv<T>(X, S.dp, nullptr, nullptr, nullptr, S.dim, 1e-5f, S.peg_w, S.peg_b, Y, S.dp, nullptr, nullptr, nullptr, S.dp, B, oh, ow,
                      S.dp, S.peg_k, 1, s);
      }
      X = Y;
      if (bf16()) ensure_stats<T>(X, S.dp, stats, M, s);
      for (const TwinsLayerW& l : S.post) twins_layer<T>(X, B, oh, ow, S, l, stats, s);
      map = X; mh = oh; mw = ow; mc = S.dim; ld_in = S.dp;
    }
    const int dl = tw.emb_dim[VB_TWINS_STAGES - 1];
    float* z = arena.get<float>(static_cast<size_t>(B) * dl);
    {
      ProfScope ps(this, PROF_LN, 1.0 * B * mh * mw * dl, static_cast<double>(sizeof(T)) * B * mh * mw * dl, s);
      pool_layernorm<T>(X, mh * mw, ld_in, nullptr, nullptr, z, B, dl, 1, s);   // GlobalAvgPool2D twins_svt.py:262
    }
    gemm_simt<float, float, float>(z, dl, head.W, head.N, 1, logits, head.N, B, head.N, dl, head.bias, nullptr, nullptr, head.N, 0, s);
  }
  // One Transformer layer (twins_svt.py:206-211) in place on X [B*H*W, dp].  bf16: the PreNorm LayerNorms are folded into the
  // fused local q|k|v, the global to_q and the fc1s (from `stats`), and applied on load by the global to_kv's patch gather; fp32:
  // separate LayerNorms.
  template <typename T>
  void twins_layer(T* X, int B, int H, int Wd, const TwinsStageW& S, const TwinsLayerW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, M = B * H * Wd, I = kTwinsInner;
    T* Y = bf16() ? nullptr : arena.get<T>(static_cast<size_t>(M) * dp);
    auto prenorm = [&](const Norm& n) -> const T* {
      if (Y == nullptr) return X;
      ProfScope ps(this, PROF_LN, 8.0 * M * d, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(X, dp, n.gamma, n.beta, Y, dp, M, d, s, dp, 1e-5f);
      return Y;
    };
    auto folded = [&](const Linear& L) {
      Epi e;
      if (Y == nullptr) { e.bias = L.ln_c2; e.ln_stats = stats; } else { e.bias = L.bias; }
      return e;
    };
    auto residual = [&](const T* A, int lda, const Linear& L) {     // X = A W + b + X, and X's new row statistics
      Epi e; e.bias = L.bias; e.res = X; e.ldr = dp; e.stats_out = stats;
      linear<T>(A, lda, M, L, X, dp, e, s);
    };
    auto mlp = [&](const MlpW& m) {                              // twins_svt.py:78-92
      const T* a = prenorm(m.norm);
      T* Hb = arena.get<T>(static_cast<size_t>(M) * m.fc1.N);
      Epi e1 = folded(m.fc1);
      e1.gelu = true;
      linear<T>(a, dp, M, m.fc1, Hb, m.fc1.N, e1, s);
      residual(Hb, m.fc1.N, m.fc2);
    };
    T* O = arena.get<T>(static_cast<size_t>(M) * I);
    if (l.local) {                                                    // LocalAttention twins_svt.py:135-156
      const T* a = prenorm(l.local_norm);
      T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * I);
      linear<T>(a, dp, M, l.qkv, QKV, 3 * I, folded(l.qkv), s);
      Window win;
      win.p = S.local; win.nx = Wd / S.local; win.ny = H / S.local;
      const int n = S.local * S.local;
      attention_dispatch<T>(QKV, 3 * I, QKV + I, 3 * I, QKV + 2 * I, 3 * I, O, I, B * win.nx * win.ny, n, n, I / 64, 64, 0, nullptr, nullptr,
                            nullptr, nullptr, s, 0.f, &win);
      residual(O, I, l.local_out);
      mlp(l.ff1);
    }
    // GlobalAttention twins_svt.py:175-190: q from every pixel, k|v from the VALID k x k stride-k convolution of LN(x)
    const T* a = prenorm(l.global_norm);
    T* Q = arena.get<T>(static_cast<size_t>(M) * I);
    linear<T>(a, dp, M, l.to_q, Q, I, folded(l.to_q), s);
    const int k = S.global_k, kh = (H - k) / k + 1, kw = (Wd - k) / k + 1, Mk = B * kh * kw;
    const int Kp = bf16() ? l.to_kv.ldw : l.to_kv.K;
    T* col = arena.get<T>(static_cast<size_t>(Mk) * Kp);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(sizeof(T)) * Mk * Kp * 2.0, s);
      UnfoldMode um;
      um.valid = true;
      if (Y == nullptr) { um.stats = stats; um.parts = dp / 64; um.d = d; um.eps = 1e-5f; um.gamma = l.global_norm.gamma; um.beta = l.global_norm.beta; }
      unfold_same<T, T>(a, col, B, H, Wd, d, k, k, 0, Kp, s, dp, &um);
    }
    T* KV = arena.get<T>(static_cast<size_t>(Mk) * 2 * I);
    Linear Lk = l.to_kv;
    Lk.K = Kp;
    linear<T>(col, Kp, Mk, Lk, KV, 2 * I, Epi(), s);
    attention_dispatch<T>(Q, I, KV, 2 * I, KV + I, 2 * I, O, I, B, H * Wd, kh * kw, I / 64, 64, 0, nullptr, nullptr, nullptr, nullptr, s);
    residual(O, I, l.global_out);
    mlp(l.ff2);
  }

  // CrossFormer.call (crossformer.py:263-269): per stage, CrossEmbedLayer -> Transformer; then the mean over the map -> Dense.
  // Token rows are the NHWC map, pixel-major, channel widths zero-padded to channel_width; no stage permutes its map (the windowed
  // attention reads and writes the map's own rows).  bf16: `stats` holds the (sum, sumsq) partials of X's rows between sub-blocks
  // (emitted by the embedding's and the residual GEMMs' epilogues).
  static constexpr const char* kCrossformerNoStages =
      "CrossFormer runs as a whole forward only: its embedding / stage / head steps have no entry of their own";
  // The reference's shape rule (crossformer.py:144,146 through einops), checked before anything runs.
  void cf_check_size(int H, int Wd) const {
    int h = H, w = Wd;
    for (int st = 0; st < VB_CROSSFORMER_STAGES; ++st) {
      h = (h + cf.stride[st] - 1) / cf.stride[st];
      w = (w + cf.stride[st] - 1) / cf.stride[st];
      const std::string where = "CrossFormer stage " + std::to_string(st + 1) + ": the " + std::to_string(h) + " x " + std::to_string(w) + " map ";
      VB_CHECK(h % cf.local_wsz[st] == 0 && w % cf.local_wsz[st] == 0, where + "is not divisible by local_window_size " + std::to_string(cf.local_wsz[st]));
      VB_CHECK(h % cf.global_wsz[st] == 0 && w % cf.global_wsz[st] == 0, where + "is not divisible by global_window_size " + std::to_string(cf.global_wsz[st]));
    }
  }
  template <typename T>
  void crossformer_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    cf_check_size(H, Wd);
    int mh = H, mw = Wd, mc = cfg.channels, ld_in = 0;
    const T* map = nullptr;
    T* X = nullptr;
    for (const CrossformerStageW& S : cf_stages) {
      const int oh = (mh + S.stride - 1) / S.stride, ow = (mw + S.stride - 1) / S.stride, M = B * oh * ow;
      const int Kp = bf16() ? S.embed.ldw : S.embed.K;
      T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
      {
        ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(map == nullptr ? 4 : sizeof(T)) * B * mh * mw * mc +
                                                 static_cast<double>(sizeof(T)) * M * Kp, s);
        if (map == nullptr) unfold_same<float, T>(img, col, B, mh, mw, mc, S.kmax, S.stride, 0, Kp, s);
        else unfold_same<T, T>(map, col, B, mh, mw, mc, S.kmax, S.stride, 0, Kp, s, ld_in);
      }
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = bf16() ? arena.get<float>(static_cast<size_t>(M) * (S.dp / 64) * 2) : nullptr;
      Linear L = S.embed;
      L.K = Kp;
      Epi e; e.bias = S.embed.bias; e.stats_out = stats;
      linear<T>(col, Kp, M, L, X, S.dp, e, s);
      for (const CrossformerLayerW& l : S.layers) crossformer_layer<T>(X, B, oh, ow, S, l, stats, s);
      map = X; mh = oh; mw = ow; mc = S.dim; ld_in = S.dp;
    }
    const int dl = cf.dim[VB_CROSSFORMER_STAGES - 1];
    float* z = arena.get<float>(static_cast<size_t>(B) * dl);
    {
      ProfScope ps(this, PROF_LN, 1.0 * B * mh * mw * dl, static_cast<double>(sizeof(T)) * B * mh * mw * dl, s);
      pool_layernorm<T>(X, mh * mw, ld_in, nullptr, nullptr, z, B, dl, 1, s);   // Reduce('b h w c -> b c', 'mean') crossformer.py:259
    }
    gemm_simt<float, float, float>(z, dl, head.W, head.N, 1, logits, head.N, B, head.N, dl, head.bias, nullptr, nullptr, head.N, 0, s);
  }
  // One Transformer layer (crossformer.py:198-202) in place on X [B*H*W, dp].  bf16: the LayerNorms folded into q|k|v and fc1 (from
  // `stats`); fp32: separate LayerNorms.
  template <typename T>
  void crossformer_layer(T* X, int B, int H, int Wd, const CrossformerStageW& S, const CrossformerLayerW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, M = B * H * Wd, I = 32 * S.heads;
    T* Y = bf16() ? nullptr : arena.get<T>(static_cast<size_t>(M) * dp);
    auto prenorm = [&](const Norm& n) -> const T* {
      if (Y == nullptr) return X;
      ProfScope ps(this, PROF_LN, 8.0 * M * d, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(X, dp, n.gamma, n.beta, Y, dp, M, d, s, dp, 1e-5f);
      return Y;
    };
    auto folded = [&](const Linear& L) {
      Epi e;
      if (Y == nullptr) { e.bias = L.ln_c2; e.ln_stats = stats; } else { e.bias = L.bias; }
      return e;
    };
    auto residual = [&](const T* A, int lda, const Linear& L) {     // X = A W + b + X, and X's new row statistics
      Epi e; e.bias = L.bias; e.res = X; e.ldr = dp; e.stats_out = stats;
      linear<T>(A, lda, M, L, X, dp, e, s);
    };
    auto mlp = [&](const MlpW& m) {                                   // crossformer.py:89-102
      const T* a = prenorm(m.norm);
      T* Hb = arena.get<T>(static_cast<size_t>(M) * m.fc1.N);
      Epi e1 = folded(m.fc1);
      e1.gelu = true;
      linear<T>(a, dp, M, m.fc1, Hb, m.fc1.N, e1, s);
      residual(Hb, m.fc1.N, m.fc2);
    };
    auto attend = [&](const CrossformerAttnW& at) {                   // crossformer.py:133-180
      const T* a = prenorm(at.norm);
      const int ld = at.qkv.N;
      T* QKV = arena.get<T>(static_cast<size_t>(M) * ld);
      linear<T>(a, dp, M, at.qkv, QKV, ld, folded(at.qkv), s);
      if (at.wsz > 1) {                                               // wsz == 1: the output is v itself, which QKV holds
        Window win;
        win.p = at.wsz; win.nx = Wd / at.wsz; win.ny = H / at.wsz; win.dilated = at.dilated;
        PosBias pb;
        pb.table = at.table; pb.wsz = at.wsz;
        const int n = at.wsz * at.wsz;
        attention_dispatch<T>(QKV, ld, QKV + I, ld, QKV + 2 * I, ld, QKV, ld, B * win.nx * win.ny, n, n, S.heads, 32, 0, nullptr, nullptr,
                              nullptr, nullptr, s, 0.f, &win, &pb);
      }
      residual(QKV, ld, at.to_out);                                   // to_out reads the I output (or v) columns
    };
    attend(l.short_attn);
    mlp(l.ff1);
    attend(l.long_attn);
    mlp(l.ff2);
  }

  // DistillMixin.call (distill.py:16-45) on top of a ViT: embed -> append the distillation token as the LAST row ->
  // transformer over n + 2 rows -> head on the first n + 1 rows, and the last row returned as is.
  template <typename T>
  void distill_impl(const float* img, int B, int H, int Wd, const float* distill_token, float* logits, float* distill_out, cudaStream_t s) {
    const vb_config& c = cfg;
    VB_CHECK(c.kind == VB_KIND_VIT, "vb_forward_distill supports ViT (distill.py:47 DistillableViT)");
    arena.reset();
    int rows = 0;
    T* E = embed_tokens<T>(embed, img, B, H, Wd, c.patch_h, c.patch_w, &rows, s, nullptr);
    const int rd = rows + 1;
    T* X = arena.get<T>(static_cast<size_t>(B) * rd * c.dim);
    copy_tokens<T>(E, rows, 0, X, rd, 0, rows, B, c.dim, s);
    T* last = X + static_cast<size_t>(rows) * c.dim;                 // row `rows` of image 0; image pitch rd rows
    broadcast_row<T>(distill_token, last, rd, B, c.dim, s);
    float* stats = (bf16() && c.dim % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr) ? arena.get<float>(static_cast<size_t>(B) * rd * (c.dim / 64) * 2) : nullptr;
    bool sv = false;
    for (const auto& l : layers) layer_self<T>(X, B, rd, c.dim, l, s, stats, &sv);
    T* Xh = arena.get<T>(static_cast<size_t>(B) * rows * c.dim);     // x[:, :-1]
    copy_tokens<T>(X, rd, 0, Xh, rows, 0, rows, B, c.dim, s);
    classify<T>(Xh, rows, c.dim, head_norm, head, B, c.pool == VB_POOL_MEAN, logits, false, s);
    T* D = arena.get<T>(static_cast<size_t>(B) * c.dim);             // x[:, -1]
    copy_tokens<T>(X, rd, rows, D, 1, 0, 1, B, c.dim, s);
    const long long count = static_cast<long long>(B) * c.dim;
    if (sizeof(T) == 4) VB_CUDA(cudaMemcpyAsync(distill_out, D, count * 4, cudaMemcpyDeviceToDevice, s));
    else convert<__nv_bfloat16, float>(reinterpret_cast<const __nv_bfloat16*>(D), distill_out, count, s);
  }

  template <typename T>
  void tokens_impl(const float* tok, int B, int n, float* out, cudaStream_t s) {
    VB_CHECK(cfg.kind == VB_KIND_VIT || cfg.kind == VB_KIND_DEEPVIT || cfg.kind == VB_KIND_T2T_VIT,
             "vb_forward_tokens supports ViT / DeepViT / T2TViT");
    arena.reset();
    const long long count = static_cast<long long>(B) * n * cfg.dim;
    T* X;
    if (sizeof(T) == 4) {
      X = reinterpret_cast<T*>(arena.get<float>(count));
      VB_CUDA(cudaMemcpyAsync(X, tok, count * 4, cudaMemcpyDeviceToDevice, s));
    } else {
      X = arena.get<T>(count);
      convert<float, __nv_bfloat16>(tok, reinterpret_cast<__nv_bfloat16*>(X), count, s);
    }
    float* stats = (bf16() && cfg.dim % 64 == 0 && getenv("VB_NO_LN_FOLD") == nullptr) ? arena.get<float>(static_cast<size_t>(B) * n * (cfg.dim / 64) * 2) : nullptr;
    bool sv = false;
    for (const auto& l : layers) layer_self<T>(X, B, n, cfg.dim, l, s, stats, &sv);
    if (sizeof(T) == 4) VB_CUDA(cudaMemcpyAsync(out, X, count * 4, cudaMemcpyDeviceToDevice, s));
    else convert<__nv_bfloat16, float>(reinterpret_cast<const __nv_bfloat16*>(X), out, count, s);
  }

  // ---------------------------------------------------------------- stage entries (vb_forward_embed / _head / vb_patch_to_emb)
  static constexpr const char* kCctNoStages = "CCT runs as a whole forward only: its tokenizer / classifier stages have no entry of their own";
  int embed_rows(int H, int Wd) const {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT has two token streams: no single embedding stage");
    VB_CHECK(cfg.kind != VB_KIND_CCT, kCctNoStages);
    VB_CHECK(cfg.kind != VB_KIND_LEVIT, kLevitNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CVT, kCvtNoStages);
    VB_CHECK(cfg.kind != VB_KIND_TWINS_SVT, kTwinsNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CROSSFORMER, kCrossformerNoStages);
    if (cfg.kind == VB_KIND_T2T_VIT) {
      int h = H, w = Wd;
      for (const auto& st : t2t_stages()) { h = (h + st.stride - 1) / st.stride; w = (w + st.stride - 1) / st.stride; }
      return h * w + 1;
    }
    VB_CHECK(H % cfg.patch_h == 0 && Wd % cfg.patch_w == 0, "Image dimensions must be divisible by the patch size.");
    const bool has_cls = cfg.kind != VB_KIND_CAIT && cfg.kind != VB_KIND_PATCH_MERGER_VIT;
    return (H / cfg.patch_h) * (Wd / cfg.patch_w) + (has_cls ? 1 : 0);
  }
  template <typename T>
  void to_f32(const T* X, float* out, long long count, cudaStream_t s) {
    if (sizeof(T) == 4) VB_CUDA(cudaMemcpyAsync(out, X, count * 4, cudaMemcpyDeviceToDevice, s));
    else convert<__nv_bfloat16, float>(reinterpret_cast<const __nv_bfloat16*>(X), out, count, s);
  }
  template <typename T>
  void embed_impl(const float* img, int B, int H, int Wd, float* tokens, cudaStream_t s) {
    arena.reset();
    int rows = 0;
    T* X = embed_any<T>(img, B, H, Wd, &rows, s, nullptr);
    to_f32<T>(X, tokens, static_cast<long long>(B) * rows * cfg.dim, s);
  }
  template <typename T>
  void head_impl(const float* tok, int B, int n, float* logits, cudaStream_t s) {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT sums two heads: no single mlp_head stage");
    VB_CHECK(cfg.kind != VB_KIND_CCT, kCctNoStages);
    VB_CHECK(cfg.kind != VB_KIND_LEVIT, kLevitNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CVT, kCvtNoStages);
    VB_CHECK(cfg.kind != VB_KIND_TWINS_SVT, kTwinsNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CROSSFORMER, kCrossformerNoStages);
    arena.reset();
    const long long count = static_cast<long long>(B) * n * cfg.dim;
    T* X = arena.get<T>(count);
    convert_rows<float, T>(tok, cfg.dim, X, cfg.dim, static_cast<long long>(B) * n, cfg.dim, s);
    const bool mean = cfg.kind == VB_KIND_PATCH_MERGER_VIT || (cfg.kind != VB_KIND_CAIT && cfg.pool == VB_POOL_MEAN);
    classify<T>(X, n, cfg.dim, head_norm, head, B, mean ? 1 : 0, logits, false, s);
  }
  template <typename T>
  void patch_to_emb_impl(const float* patches, int rows, float* out, cudaStream_t s) {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT has two patch embeddings");
    VB_CHECK(cfg.kind != VB_KIND_CCT, kCctNoStages);
    VB_CHECK(cfg.kind != VB_KIND_LEVIT, kLevitNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CVT, kCvtNoStages);
    VB_CHECK(cfg.kind != VB_KIND_TWINS_SVT, kTwinsNoStages);
    VB_CHECK(cfg.kind != VB_KIND_CROSSFORMER, kCrossformerNoStages);
    arena.reset();
    const int K = embed.patch.K, Kp = bf16() ? embed.patch.ldw : K;
    T* col = arena.get<T>(static_cast<size_t>(rows) * Kp);
    convert_rows<float, T>(patches, K, col, Kp, rows, K, s);
    T* Y = arena.get<T>(static_cast<size_t>(rows) * cfg.dim);
    Epi ep; ep.bias = embed.patch.bias;
    Linear L = embed.patch;
    L.K = Kp;
    linear<T>(col, Kp, rows, L, Y, cfg.dim, ep, s);
    to_f32<T>(Y, out, static_cast<long long>(rows) * cfg.dim, s);
  }
};

// ------------------------------------------------------------------------------------------ op dispatch
template <>
void vb_handle::linear<float>(const float* A, int lda, int M, const Linear& L, float* out, int ldc, const Epi& e, cudaStream_t s) {
  gemm_simt<float, float, float>(A, lda, L.W, L.N, 1, out, ldc, M, L.N, L.K, e.bias, e.scale,
                                 static_cast<const float*>(e.res), e.ldr, e.act(), s);
}
template <>
void vb_handle::linear<__nv_bfloat16>(const __nv_bfloat16* A, int lda, int M, const Linear& L, __nv_bfloat16* out, int ldc,
                                      const Epi& e, cudaStream_t s) {
  const int K = L.K;
  const __nv_bfloat16* res = static_cast<const __nv_bfloat16*>(e.res);
  const bool fast = gemm_bf16_supported(M, L.N, K, lda, L.ldw, ldc) && (res == nullptr || e.ldr % 8 == 0);
  const bool folded = L.ln_c1 != nullptr;
  VB_CHECK(!folded || (fast && e.ln_stats != nullptr && K % 64 == 0), "internal: LayerNorm-folded Dense needs the wgmma path and row statistics");
  VB_CHECK(e.stats_out == nullptr || fast, "internal: row statistics requested from a non-wgmma GEMM");
  ProfScope ps(this, !fast ? PROF_OTHER : e.act() != ACT_NONE ? PROF_GEMM_GELU : res ? PROF_GEMM_RES : PROF_GEMM, 2.0 * M * L.N * K,
               2.0 * (static_cast<double>(M) * K + static_cast<double>(L.N) * K + static_cast<double>(M) * L.N * (res ? 2 : 1)), s);
  if (fast) {
    PlanKey key{};
    const uintptr_t parts[16] = {reinterpret_cast<uintptr_t>(A), static_cast<uintptr_t>(lda), reinterpret_cast<uintptr_t>(L.Wt),
                                 reinterpret_cast<uintptr_t>(out), static_cast<uintptr_t>(ldc), static_cast<uintptr_t>(M),
                                 static_cast<uintptr_t>(L.N), static_cast<uintptr_t>(K), reinterpret_cast<uintptr_t>(e.bias),
                                 reinterpret_cast<uintptr_t>(e.scale), reinterpret_cast<uintptr_t>(res),
                                 static_cast<uintptr_t>(e.ldr), static_cast<uintptr_t>(e.act()),
                                 reinterpret_cast<uintptr_t>(e.ln_stats), reinterpret_cast<uintptr_t>(L.ln_c1),
                                 reinterpret_cast<uintptr_t>(e.stats_out)};
    for (int i = 0; i < 16; ++i) key[i] = parts[i];
    auto it = plans.find(key);
    if (it == plans.end()) {
      if (plans.size() > 8192) plans.clear();      // shape sweeps: bounded host memory (a plan is four 128-byte tensor maps)
      GemmBf16 g = gemm_bf16_plan(A, lda, L.Wt, L.ldw, out, ldc, M, L.N, K, e.bias, e.scale, res, e.ldr, e.act());
      if (folded) { g.ln_c1 = L.ln_c1; g.ln_stats = e.ln_stats; g.ln_parts = K / 64; g.ln_inv_d = 1.0f / static_cast<float>(L.ln_d > 0 ? L.ln_d : K);
                    g.ln_eps = L.ln_eps; }
      if (e.stats_out) { g.stats_out = e.stats_out; }
      it = plans.emplace(key, g).first;
    }
    gemm_bf16_run(it->second, s);
  } else {
    gemm_simt<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(A, lda, L.Wt, 1, L.ldw, out, ldc, M, L.N, K, e.bias, e.scale, res,
                                                           e.ldr, e.act(), s);
  }
}

template <>
void vb_handle::ensure_stats<float>(const float*, int, float*, int, cudaStream_t) {}
template <>
void vb_handle::ensure_stats<__nv_bfloat16>(const __nv_bfloat16* X, int dim, float* stats, int M, cudaStream_t s) {
  ProfScope ps(this, PROF_LN, 0.0, 2.0 * M * dim, s);
  row_stats_bf16(X, dim, stats, M, dim, s);
}

template <>
void vb_handle::layer_t2t<float>(float*, int, int, const LayerW&, cudaStream_t) { VB_CHECK(false, "internal: tensor-core T2T layer in the fp32 engine"); }
template <>
void vb_handle::layer_t2t<__nv_bfloat16>(__nv_bfloat16* X, int B, int n, const LayerW& l, cudaStream_t s) {
  using bf = __nv_bfloat16;
  const int D = l.t2t_D, Dp = l.t2t_Dp, M = B * n, npad = round_up(n, 64);
  bf* Y = arena.get<bf>(static_cast<size_t>(M) * Dp);
  bf* QKV = arena.get<bf>(static_cast<size_t>(M) * 3 * Dp);
  bf* Vt = arena.get<bf>(static_cast<size_t>(B) * Dp * npad);
  // Images are independent: ns of them are in flight on ns streams (the forward's own + side streams), each with its own score /
  // probability buffers.  The per-image kernels are small (16 pair tiles for Q K^T at n = 784) and strictly dependent, so one
  // stream leaves most SMs idle and pays every launch gap (389 launches per T2T step at batch 64).  Two streams
  // when one image's buffers are large (n = 3136: 59 MB each, more than the 50 MB L2 already), four otherwise.
  const size_t s_elems = static_cast<size_t>(n) * npad;
  static const char* ns_env = getenv("VB_T2T_STREAMS");
  int ns = ns_env != nullptr ? atoi(ns_env) : (s_elems * 6 > (48u << 20) ? 2 : 4);
  ns = std::max(1, std::min(ns, std::min(B, static_cast<int>(T2T_MAX_STREAMS))));
  if (profiling) ns = 1;                                         // per-class event timing wants one stream
  float* S[T2T_MAX_STREAMS];
  bf* P[T2T_MAX_STREAMS];
  cudaStream_t st[T2T_MAX_STREAMS];
  for (int i = 0; i < ns; ++i) { S[i] = arena.get<float>(s_elems); P[i] = arena.get<bf>(s_elems); }
  st[0] = s;
  if (ns > 1) {
    ensure_side_streams();
    for (int i = 1; i < ns; ++i) st[i] = side_streams[i - 1];
  }
  { ProfScope ps(this, PROF_LN, 0.0, 4.0 * M * D, s); layernorm<bf>(X, Dp, l.attn_norm.gamma, l.attn_norm.beta, Y, Dp, M, D, s, Dp); }
  linear<bf>(Y, Dp, M, l.to_qkv, QKV, 3 * Dp, Epi(), s);
  {
    ProfScope ps(this, PROF_OTHER, 0.0, 4.0 * M * Dp, s);
    transpose_rows_bf16(QKV + 2 * Dp, 3 * Dp, static_cast<long long>(n) * 3 * Dp, Vt, npad, static_cast<long long>(Dp) * npad, B, n, npad, Dp, s);
  }
  const float scale_log2 = (1.0f / sqrtf(static_cast<float>(D))) * 1.4426950408889634f;
  if (ns > 1) {
    VB_CUDA(cudaEventRecord(fork_event, s));
    for (int i = 1; i < ns; ++i) VB_CUDA(cudaStreamWaitEvent(st[i], fork_event, 0));
  }
  for (int b = 0; b < B; ++b) {
    const int i = b % ns;
    const bf* Qb = QKV + static_cast<size_t>(b) * n * 3 * Dp;
    bf* Xb = X + static_cast<size_t>(b) * n * Dp;
    gemm_cached(Qb, 3 * Dp, Qb + Dp, 3 * Dp, n, S[i], npad, n, npad, Dp, nullptr, 0, true, PROF_ATTN, st[i]);       // S = Q K^T
    { ProfScope ps(this, PROF_ATTN, 0.0, 6.0 * n * npad, st[i]); softmax_rows_bf16(S[i], npad, P[i], npad, n, n, npad, scale_log2, st[i]); }
    gemm_cached(P[i], npad, Vt + static_cast<size_t>(b) * Dp * npad, npad, 0, Xb, Dp, n, Dp, npad, Xb, Dp, false, PROF_ATTN, st[i]);   // X += P V
  }
  for (int i = 1; i < ns; ++i) {
    VB_CUDA(cudaEventRecord(join_events[i - 1], st[i]));
    VB_CUDA(cudaStreamWaitEvent(s, join_events[i - 1], 0));
  }
  { ProfScope ps(this, PROF_LN, 0.0, 4.0 * M * D, s); layernorm<bf>(X, Dp, l.ff_norm.gamma, l.ff_norm.beta, Y, Dp, M, D, s, Dp); }
  bf* Hb = arena.get<bf>(static_cast<size_t>(M) * Dp);
  Epi e1; e1.gelu = true; e1.bias = l.fc1.bias;
  linear<bf>(Y, Dp, M, l.fc1, Hb, Dp, e1, s);
  Epi e2; e2.bias = l.fc2.bias; e2.res = X; e2.ldr = Dp;
  linear<bf>(Hb, Dp, M, l.fc2, X, Dp, e2, s);
}

template <typename T>
void vb_handle::attention_dispatch(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq,
                                   int nk, int heads, int dh, int variant, const float* mix_a, const float* mix_b, const float* g,
                                   const float* b, cudaStream_t s, float scale, const Window* win, const PosBias* pb) {
  // windowed attention (Twins-SVT's local, CrossFormer's short / long with pb, its window table): B windows of nq = nk = p^2
  // tokens in the map's own rows
  if (win != nullptr) {
    const int HD = heads * dh;
    VB_CHECK(k == q + HD && v == q + 2 * HD && ldk == ldq && ldv == ldq && variant == 0, "internal: windowed attention reads fused q|k|v rows");
    const double fl = 4.0 * B * heads * nq * nk * dh, by = static_cast<double>(sizeof(T)) * B * heads * dh * (2.0 * nq + 2.0 * nk);
    {
      ProfScope ps(this, PROF_ATTN, fl, by, s);
      if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, s, 0.f, pb, win))
        return;
    }
    // off the flash kernel: the rows permuted to window-major order, the materialised-scores path, the output rows permuted back
    const long long rows = static_cast<long long>(B) * nq;
    T* qkvw = arena.get<T>(static_cast<size_t>(rows) * 3 * HD);
    T* ow = arena.get<T>(static_cast<size_t>(rows) * HD);
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * 3 * HD, s); window_rows<T>(q, ldq, qkvw, 3 * HD, 3 * HD, *win, rows, true, s); }
    {
      ProfScope ps(this, PROF_ATTN, fl, by, s);
      float* S = arena.get<float>(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15));
      attention_generic<T>(qkvw, 3 * HD, qkvw + HD, 3 * HD, qkvw + 2 * HD, 3 * HD, ow, HD, S, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr,
                           nullptr, s, 0.f, pb);
    }
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * HD, s); window_rows<T>(ow, HD, out, ldo, HD, *win, rows, false, s); }
    return;
  }
  ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * nq * nk * dh + (variant == 1 ? 2.0 : variant == 2 ? 4.0 : 0.0) * B * nq * nk * heads * heads,
               static_cast<double>(sizeof(T)) * B * heads * dh * (2.0 * nq + 2.0 * nk), s);
  if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, variant, mix_a, mix_b, g, b, s, scale)) return;
  VB_CHECK(scale <= 0.f, "internal: a head-padded layer must run on the fused attention kernel");
  float* S = arena.get<float>(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15));   // row pitch padded for the bf16-P path
  attention_generic<T>(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, heads, dh, variant, mix_a, mix_b, g, b, s);
}

template <>
void vb_handle::add_tokens<float>(float* X, const float* O, long long count, cudaStream_t s) { add_inplace_f32(X, O, count, s); }
template <>
void vb_handle::add_tokens<__nv_bfloat16>(__nv_bfloat16* X, const __nv_bfloat16* O, long long count, cudaStream_t s) {
  // rare path (heads == 1 and dim_head == dim): go through fp32 scratch
  float* a = arena.get<float>(count);
  float* b = arena.get<float>(count);
  convert<__nv_bfloat16, float>(X, a, count, s);
  convert<__nv_bfloat16, float>(O, b, count, s);
  add_inplace_f32(a, b, count, s);
  convert<float, __nv_bfloat16>(a, X, count, s);
}

// ------------------------------------------------------------------------------------------ C ABI
namespace {

template <typename F>
int guarded(vb_handle* h, F&& f) {
  try {
    f();
    return 0;
  } catch (const vb::Error& e) {
    (h ? h->error : g_last_error) = e.what();
    return e.code;
  } catch (const std::exception& e) {
    (h ? h->error : g_last_error) = e.what();
    return 3;
  } catch (...) {
    (h ? h->error : g_last_error) = "unknown error";
    return 4;
  }
}

void validate(const vb_config& c) {
  VB_CHECK(c.struct_size == static_cast<int32_t>(sizeof(vb_config)) || c.struct_size == VB_CONFIG_SIZE_ABI7,
           "vb_config.struct_size mismatch (ABI)");
  VB_CHECK(c.kind != VB_KIND_LEVIT, "LeViT: create the handle with vb_create_levit (its stages are a vb_levit_config)");
  VB_CHECK(c.kind != VB_KIND_CVT, "CvT: create the handle with vb_create_cvt (its stages are a vb_cvt_config)");
  VB_CHECK(c.kind != VB_KIND_TWINS_SVT, "Twins-SVT: create the handle with vb_create_twins_svt (its stages are a vb_twins_svt_config)");
  VB_CHECK(c.kind != VB_KIND_CROSSFORMER, "CrossFormer: create the handle with vb_create_crossformer (its stages are a vb_crossformer_config)");
  VB_CHECK(c.kind >= VB_KIND_VIT && c.kind <= VB_KIND_CCT, "unknown model kind");
  if (c.kind == VB_KIND_CCT) {
    VB_CHECK(c.channels == 3 && c.num_classes > 0 && c.image_h > 0 && c.image_w > 0, "bad image / class configuration");
    VB_CHECK(c.cct_conv_layers >= 1 && c.cct_conv_layers <= 8, "CCT: n_conv_layers must be in [1, 8]");
    VB_CHECK(c.cct_kernel > 0 && c.cct_stride > 0 && c.cct_pool_kernel > 0 && c.cct_pool_stride > 0,
             "CCT: kernel / stride / pooling sizes must be positive");
    VB_CHECK(c.cct_pos_emb >= VB_CCT_POS_SINE && c.cct_pos_emb <= VB_CCT_POS_NONE, "CCT: unknown positional embedding kind");
    VB_CHECK(c.dim > 0 && c.dim <= 1024 && c.depth >= 0 && c.heads > 0 && c.heads <= 32 && c.mlp_dim > 0, "bad transformer dimensions");
    VB_CHECK(c.dim % c.heads == 0 && c.dim_head == c.dim / c.heads, "CCT: embedding_dim must be divisible by num_heads");
    VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
    return;
  }
  VB_CHECK(c.kind != VB_KIND_PARALLEL_VIT || (c.parallel_branches >= 1 && c.parallel_branches <= 8), "num_parallel_branches must be in [1, 8]");
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0 && c.image_h > 0 && c.image_w > 0, "bad image / class configuration");
  if (c.kind == VB_KIND_CROSSVIT) {
    VB_CHECK(c.image_h == c.image_w, "CrossViT takes a square integer image_size");
    VB_CHECK(c.sm_patch_size > 0 && c.lg_patch_size > 0 && c.image_h % c.sm_patch_size == 0 && c.image_h % c.lg_patch_size == 0,
             "Image dimensions must be divisible by the patch size.");
    VB_CHECK(c.sm_dim > 0 && c.lg_dim > 0 && c.cross_depth > 0 && c.cross_attn_depth >= 0, "bad CrossViT dimensions");
    VB_CHECK(c.sm_enc_heads <= 32 && c.lg_enc_heads <= 32 && c.cross_attn_heads <= 32, "at most 32 heads");
  } else {
    if (c.kind == VB_KIND_T2T_VIT) {
      VB_CHECK(c.image_h == c.image_w, "T2TViT takes a square integer image_size");
      VB_CHECK(c.t2t_num_layers >= 1 && c.t2t_num_layers <= 4, "t2t_layers: between 1 and 4 (kernel_size, stride) pairs");
      const int ks[4] = {c.t2t_k0, c.t2t_k1, c.t2t_k2, c.t2t_k3}, ss[4] = {c.t2t_s0, c.t2t_s1, c.t2t_s2, c.t2t_s3};
      long long d = c.channels;
      for (int i = 0; i < c.t2t_num_layers; ++i) {
        VB_CHECK(ks[i] > 0 && ss[i] > 0, "t2t_layers: kernel sizes and strides must be positive");
        d *= static_cast<long long>(ks[i]) * ks[i];
        VB_CHECK(d <= (1 << 20), "t2t_layers: token width channels * prod(kernel_size^2) is too large");
      }
    } else {
      VB_CHECK(c.patch_h > 0 && c.patch_w > 0 && c.image_h % c.patch_h == 0 && c.image_w % c.patch_w == 0,
               "Image dimensions must be divisible by the patch size.");
    }
    VB_CHECK(c.kind != VB_KIND_PATCH_MERGER_VIT || c.patch_merge_num_tokens > 0, "patch_merge_num_tokens must be positive");
    VB_CHECK(c.dim > 0 && c.depth >= 0 && c.heads > 0 && c.dim_head > 0 && c.mlp_dim > 0, "bad transformer dimensions");
    VB_CHECK(c.heads <= 32, "at most 32 heads");
    VB_CHECK(c.pool == VB_POOL_CLS || c.pool == VB_POOL_MEAN, "pool type must be either cls (cls token) or mean (mean pooling)");
  }
}

void validate_levit(const vb_config& c, const vb_levit_config& lv) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0 && c.image_h > 0 && c.image_h == c.image_w, "LeViT: bad image / class configuration");
  VB_CHECK(lv.stages >= 1 && lv.stages <= VB_LEVIT_MAX_STAGES, "LeViT: stages must be in [1, 8]");
  VB_CHECK(lv.dim_key > 0 && lv.dim_value > 0 && lv.mlp_mult > 0 && lv.num_distill_classes >= 0, "LeViT: bad dim_key / dim_value / mlp_mult");
  for (int s = 0; s < lv.stages; ++s)
    VB_CHECK(lv.dims[s] > 0 && lv.depths[s] >= 0 && lv.heads[s] > 0, "LeViT: bad stage dimensions");
  // levit.py:194 vs the stem: image_size // 16 must be the size four ceil-halvings give, or the bias cannot broadcast
  int f = c.image_h;
  for (int i = 0; i < 4; ++i) f = (f + 1) / 2;
  VB_CHECK(c.image_h >= 16 && f == c.image_h / 16,
           "LeViT: image_size " + std::to_string(c.image_h) + " gives a " + std::to_string(f) + " x " + std::to_string(f) +
           " map after the stem but position biases for image_size // 16 = " + std::to_string(c.image_h / 16));
}

void validate_cvt(const vb_config& c, const vb_cvt_config& cv) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0, "CvT: bad channel / class configuration");
  for (int st = 0; st < VB_CVT_STAGES; ++st) {
    VB_CHECK(cv.emb_dim[st] > 0 && cv.emb_kernel[st] > 0 && cv.emb_stride[st] > 0 && cv.heads[st] > 0 && cv.depth[st] >= 0 &&
             cv.mlp_mult[st] > 0, "CvT: bad stage configuration");
    VB_CHECK(cv.proj_kernel[st] >= 1 && cv.proj_kernel[st] <= 7, "CvT: proj_kernel must be in [1, 7] (the depthwise kernel's halo tile)");
    VB_CHECK(cv.kv_proj_stride[st] == 1 || cv.kv_proj_stride[st] == 2, "CvT: kv_proj_stride must be 1 or 2");
  }
}

void validate_twins(const vb_config& c, const vb_twins_svt_config& tw) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0, "Twins-SVT: bad channel / class configuration");
  for (int st = 0; st < VB_TWINS_STAGES; ++st)
    VB_CHECK(tw.emb_dim[st] > 0 && tw.patch_size[st] > 0 && tw.local_patch_size[st] > 0 && tw.global_k[st] > 0 && tw.depth[st] >= 0,
             "Twins-SVT: bad stage configuration");
  VB_CHECK(tw.peg_kernel_size >= 1 && tw.peg_kernel_size <= 7, "Twins-SVT: peg_kernel_size must be in [1, 7] (the depthwise kernel's halo tile)");
}

void validate_crossformer(const vb_config& c, const vb_crossformer_config& cf) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0, "CrossFormer: bad channel / class configuration");
  for (int st = 0; st < VB_CROSSFORMER_STAGES; ++st) {
    const std::string stage = "CrossFormer stage " + std::to_string(st + 1) + ": ";
    VB_CHECK(cf.dim[st] >= 32, stage + "dim must be at least 32 (heads = dim // 32 of width 32)");
    VB_CHECK(cf.depth[st] >= 0 && cf.global_wsz[st] > 0 && cf.local_wsz[st] > 0 && cf.stride[st] > 0, stage + "bad depth / window / stride");
    VB_CHECK(cf.n_kernels[st] >= 1 && cf.n_kernels[st] <= VB_CROSSFORMER_MAX_KERNELS,
             stage + "between 1 and " + std::to_string(VB_CROSSFORMER_MAX_KERNELS) + " cross-embedding kernel sizes are supported");
    std::string ks;
    bool pos = true, parity = true, above = true;
    for (int i = 0; i < cf.n_kernels[st]; ++i) {
      const int k = cf.kernels[st][i];
      ks += (i ? ", " : "") + std::to_string(k);
      pos = pos && k > 0;
      parity = parity && (k - cf.kernels[st][0]) % 2 == 0;
      above = above && k >= cf.stride[st];
    }
    VB_CHECK(pos, stage + "kernel sizes must be positive");
    VB_CHECK(parity && above, stage + "kernel sizes (" + ks + ") at stride " + std::to_string(cf.stride[st]) +
                                  ": the nested cross-scale embedding needs kernels of one parity, each at least the stride");
  }
}

}  // namespace

// ---------------------------------------------------------------- single-operator entry points
namespace {
struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  ~Timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
};
template <typename F>
void timed(int iters, float* elapsed_ms, F&& f) {
  f();  // first run produces the result (and warms up)
  VB_CUDA(cudaDeviceSynchronize());
  if (elapsed_ms && iters > 0) {
    Timer t;
    VB_CUDA(cudaEventRecord(t.a, 0));
    for (int i = 0; i < iters; ++i) f();
    VB_CUDA(cudaEventRecord(t.b, 0));
    VB_CUDA(cudaEventSynchronize(t.b));
    float ms = 0.f;
    VB_CUDA(cudaEventElapsedTime(&ms, t.a, t.b));
    *elapsed_ms = ms / iters;
  }
}
void require_gpu() {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  VB_CHECK(e == cudaSuccess && ndev > 0, "no CUDA device available -- libvitb200 has no CPU fallback");
}
template <typename T>
T* upload(DevMem& m, const float* host, size_t count) {
  m.ensure(count * sizeof(T) + 16);
  if (sizeof(T) == 4) {
    VB_CUDA(cudaMemcpy(m.p, host, count * 4, cudaMemcpyHostToDevice));
  } else {
    DevMem tmp;
    tmp.ensure(count * 4);
    VB_CUDA(cudaMemcpy(tmp.p, host, count * 4, cudaMemcpyHostToDevice));
    convert<float, __nv_bfloat16>(static_cast<const float*>(tmp.p), static_cast<__nv_bfloat16*>(m.p), static_cast<long long>(count), 0);
    VB_CUDA(cudaDeviceSynchronize());
  }
  return static_cast<T*>(m.p);
}
// Erases the head-mix cache entries of an op entry's temporary weight copies when the entry returns: the copies are freed then,
// and a later allocation at the same address must not find their values.  No other handle's entry is touched.
struct MixCacheScope {
  std::vector<const void*> p;
  ~MixCacheScope() { attention_mix_cache_erase(p); }
};
template <typename T>
void download(const T* dev, float* host, size_t count) {
  if (sizeof(T) == 4) {
    VB_CUDA(cudaMemcpy(host, dev, count * 4, cudaMemcpyDeviceToHost));
  } else {
    DevMem tmp;
    tmp.ensure(count * 4);
    convert<__nv_bfloat16, float>(reinterpret_cast<const __nv_bfloat16*>(dev), static_cast<float*>(tmp.p), static_cast<long long>(count), 0);
    VB_CUDA(cudaMemcpy(host, tmp.p, count * 4, cudaMemcpyDeviceToHost));
  }
}
}  // namespace

namespace {
// Shared plumbing of the stage entries: optional host->device staging of the input, device staging of a host output,
// launch accounting, and the final copy + synchronise when the output is a host buffer.
template <typename F>
void staged_call(vb_handle* h, const float* in, int32_t in_mem, size_t in_bytes, float* out, int32_t out_mem, size_t out_bytes,
                 cudaStream_t s, F&& body) {
  VB_CUDA(cudaSetDevice(h->device));
  const long long before = launch_counter();
  const float* in_d = in;
  if (in_mem == VB_MEM_HOST) {
    h->tokens_in.ensure(in_bytes);
    VB_CUDA(cudaMemcpyAsync(h->tokens_in.p, in, in_bytes, cudaMemcpyHostToDevice, s));
    in_d = static_cast<const float*>(h->tokens_in.p);
  }
  float* out_d = out;
  if (out_mem == VB_MEM_HOST) {
    h->tokens_out.ensure(out_bytes);
    out_d = static_cast<float*>(h->tokens_out.p);
  }
  body(in_d, out_d);
  h->last_launches = launch_counter() - before;
  if (out_mem == VB_MEM_HOST) {
    VB_CUDA(cudaMemcpyAsync(out, out_d, out_bytes, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
  }
}
}  // namespace

extern "C" {

int vb_abi_version(void) { return VB_ABI_VERSION; }

int vb_create(const vb_config* cfg, int device, vb_handle** out) {
  return guarded(nullptr, [&] {
    VB_CHECK(cfg != nullptr && out != nullptr, "vb_create: null argument");
    // a client of the ABI-7 struct without the CCT fields passes the shorter size: read only its bytes, zero the rest
    const int32_t size = cfg->struct_size;
    VB_CHECK(size == static_cast<int32_t>(sizeof(vb_config)) || size == VB_CONFIG_SIZE_ABI7, "vb_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, cfg, static_cast<size_t>(size));
    validate(c);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, "vb_create: no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, "vb_create: bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, "vb_create: libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}

int vb_create_levit(const vb_config* base, const vb_levit_config* lv, int device, vb_handle** out) {
  return guarded(nullptr, [&] {
    VB_CHECK(base != nullptr && lv != nullptr && out != nullptr, "vb_create_levit: null argument");
    VB_CHECK(base->struct_size == static_cast<int32_t>(sizeof(vb_config)) || base->struct_size == VB_CONFIG_SIZE_ABI7,
             "vb_config.struct_size mismatch (ABI)");
    VB_CHECK(lv->struct_size == static_cast<int32_t>(sizeof(vb_levit_config)), "vb_levit_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, base, static_cast<size_t>(base->struct_size));
    VB_CHECK(c.kind == VB_KIND_LEVIT, "vb_create_levit: base.kind must be VB_KIND_LEVIT");
    validate_levit(c, *lv);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, "vb_create_levit: no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, "vb_create_levit: bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, "vb_create_levit: libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->cfg.dim = lv->dims[lv->stages - 1];
    h->lv = *lv;
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}

int vb_create_cvt(const vb_config* base, const vb_cvt_config* cvt, int device, vb_handle** out) {
  return guarded(nullptr, [&] {
    VB_CHECK(base != nullptr && cvt != nullptr && out != nullptr, "vb_create_cvt: null argument");
    VB_CHECK(base->struct_size == static_cast<int32_t>(sizeof(vb_config)) || base->struct_size == VB_CONFIG_SIZE_ABI7,
             "vb_config.struct_size mismatch (ABI)");
    VB_CHECK(cvt->struct_size == static_cast<int32_t>(sizeof(vb_cvt_config)), "vb_cvt_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, base, static_cast<size_t>(base->struct_size));
    VB_CHECK(c.kind == VB_KIND_CVT, "vb_create_cvt: base.kind must be VB_KIND_CVT");
    validate_cvt(c, *cvt);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, "vb_create_cvt: no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, "vb_create_cvt: bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, "vb_create_cvt: libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->cfg.dim = cvt->emb_dim[VB_CVT_STAGES - 1];
    h->cv = *cvt;
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}

int vb_create_twins_svt(const vb_config* base, const vb_twins_svt_config* tw, int device, vb_handle** out) {
  return guarded(nullptr, [&] {
    VB_CHECK(base != nullptr && tw != nullptr && out != nullptr, "vb_create_twins_svt: null argument");
    VB_CHECK(base->struct_size == static_cast<int32_t>(sizeof(vb_config)) || base->struct_size == VB_CONFIG_SIZE_ABI7,
             "vb_config.struct_size mismatch (ABI)");
    VB_CHECK(tw->struct_size == static_cast<int32_t>(sizeof(vb_twins_svt_config)), "vb_twins_svt_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, base, static_cast<size_t>(base->struct_size));
    VB_CHECK(c.kind == VB_KIND_TWINS_SVT, "vb_create_twins_svt: base.kind must be VB_KIND_TWINS_SVT");
    validate_twins(c, *tw);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, "vb_create_twins_svt: no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, "vb_create_twins_svt: bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, "vb_create_twins_svt: libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->cfg.dim = tw->emb_dim[VB_TWINS_STAGES - 1];
    h->tw = *tw;
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}

int vb_create_crossformer(const vb_config* base, const vb_crossformer_config* cfc, int device, vb_handle** out) {
  return guarded(nullptr, [&] {
    VB_CHECK(base != nullptr && cfc != nullptr && out != nullptr, "vb_create_crossformer: null argument");
    VB_CHECK(base->struct_size == static_cast<int32_t>(sizeof(vb_config)) || base->struct_size == VB_CONFIG_SIZE_ABI7,
             "vb_config.struct_size mismatch (ABI)");
    VB_CHECK(cfc->struct_size == static_cast<int32_t>(sizeof(vb_crossformer_config)), "vb_crossformer_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, base, static_cast<size_t>(base->struct_size));
    VB_CHECK(c.kind == VB_KIND_CROSSFORMER, "vb_create_crossformer: base.kind must be VB_KIND_CROSSFORMER");
    validate_crossformer(c, *cfc);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, "vb_create_crossformer: no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, "vb_create_crossformer: bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, "vb_create_crossformer: libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->cfg.dim = cfc->dim[VB_CROSSFORMER_STAGES - 1];
    h->cf = *cfc;
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}

int vb_num_weights(vb_handle* h) { return h ? static_cast<int>(h->weights.size()) : -1; }

int vb_weight_info(vb_handle* h, int32_t index, const char** name, int64_t* shape4, int32_t* ndim) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CHECK(index >= 0 && index < static_cast<int>(h->weights.size()), "weight index out of range");
    const Weight& w = h->weights[index];
    if (name) *name = w.name.c_str();
    if (ndim) *ndim = static_cast<int32_t>(w.shape.size());
    if (shape4) for (size_t i = 0; i < w.shape.size() && i < 4; ++i) shape4[i] = w.shape[i];
  });
}

int vb_set_weight(vb_handle* h, const char* name, const float* host_data, const int64_t* shape, int32_t ndim) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && name != nullptr && host_data != nullptr && shape != nullptr, "vb_set_weight: null argument");
    auto it = h->windex.find(name);
    VB_CHECK(it != h->windex.end(), std::string("vb_set_weight: this model has no weight named '") + name + "'");
    Weight& w = h->weights[it->second];
    bool ok = static_cast<size_t>(ndim) == w.shape.size();
    for (int i = 0; ok && i < ndim; ++i) ok = shape[i] == w.shape[i];
    VB_CHECK(ok, std::string("vb_set_weight: shape mismatch for '") + name + "'");
    VB_CUDA(cudaSetDevice(h->device));
    if (w.dev == nullptr) VB_CUDA(cudaMalloc(reinterpret_cast<void**>(&w.dev), w.count * sizeof(float)));
    VB_CUDA(cudaMemcpy(w.dev, host_data, w.count * sizeof(float), cudaMemcpyHostToDevice));
    w.set = true;
    h->finalized = false;
  });
}

int vb_finalize(vb_handle* h) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    attention_mix_cache_erase(h->weight_pointers());        // new values behind the same pointers; other handles keep theirs
    h->finalize();
  });
}

int vb_forward(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
               int32_t logits_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && logits != nullptr, "vb_forward: null argument");
    VB_CHECK(h->finalized, "vb_forward: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward: bad batch / image size");
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const size_t img_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const size_t out_bytes = static_cast<size_t>(batch) * h->cfg.num_classes * sizeof(float);
    const float* img_d = img;
    if (img_mem == VB_MEM_HOST) {
      h->img_dev.ensure(img_bytes);
      VB_CUDA(cudaMemcpyAsync(h->img_dev.p, img, img_bytes, cudaMemcpyHostToDevice, s));
      img_d = static_cast<const float*>(h->img_dev.p);
    }
    float* out_d = logits;
    if (logits_mem == VB_MEM_HOST) {
      h->logits_dev.ensure(out_bytes);
      out_d = static_cast<float*>(h->logits_dev.p);
    }
    auto run_eager = [&] {
      if (h->bf16()) h->forward_impl<__nv_bfloat16>(img_d, batch, img_h, img_w, out_d, s);
      else h->forward_impl<float>(img_d, batch, img_h, img_w, out_d, s);
    };
    static const bool graphs_off = getenv("VB_NO_GRAPH") != nullptr;
    const bool graphable = !graphs_off && !h->profiling && s != nullptr && s != cudaStreamLegacy;
    bool done = false;
    if (graphable) {
      if (h->graphs.size() > 64) h->drop_graphs();                         // shape / pointer sweeps: bounded
      vb_handle::GraphEntry& ge = h->graphs[vb_handle::GraphKey{img_d, out_d, batch, img_h, img_w, s}];
      ++ge.calls;
      if (ge.exec != nullptr) {
        VB_CUDA(cudaGraphLaunch(ge.exec, s));
        count_launch(static_cast<int>(ge.launches));
        ++h->graph_replays;
        done = true;
      } else if (ge.calls == 2 && !ge.failed) {
        cudaGraph_t graph = nullptr;
        const long long l0 = launch_counter();
        std::string why;
        const cudaError_t eb = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        if (eb == cudaSuccess) {
          bool ok = true;
          try { run_eager(); } catch (const std::exception& e) { ok = false; why = e.what(); }
          const cudaError_t ec = cudaStreamEndCapture(s, &graph);
          cudaError_t ei = cudaSuccess;
          if (ok && ec == cudaSuccess && graph != nullptr && (ei = cudaGraphInstantiate(&ge.exec, graph, 0)) == cudaSuccess) {
            ge.launches = launch_counter() - l0;
            VB_CUDA(cudaGraphLaunch(ge.exec, s));
            ++h->graph_captures;
            done = true;
          } else {
            if (ok) why = std::string(ec != cudaSuccess ? "cudaStreamEndCapture: " : "cudaGraphInstantiate: ") +
                          cudaGetErrorString(ec != cudaSuccess ? ec : ei);
            ge.exec = nullptr;
          }
          if (graph != nullptr) cudaGraphDestroy(graph);
        } else {
          why = std::string("cudaStreamBeginCapture: ") + cudaGetErrorString(eb);
        }
        if (!done) {                                                        // stay eager for this key
          ge.failed = true;
          ++h->graph_failures;
          h->graph_last_failure = why;
          cudaGetLastError();
        }
      }
    }
    if (!done) run_eager();
    h->last_launches = launch_counter() - before;
    if (logits_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(logits, out_d, out_bytes, cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_forward_distill(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                       const float* distill_token, float* logits, float* distill_out, int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && logits != nullptr && distill_out != nullptr, "vb_forward_distill: null argument");
    VB_CHECK(h->finalized, "vb_forward_distill: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward_distill: bad batch / image size");
    VB_CHECK(h->cfg.kind != VB_KIND_CVT, "vb_forward_distill: CvT has no distillation head");
    VB_CHECK(h->cfg.kind != VB_KIND_TWINS_SVT, "vb_forward_distill: Twins-SVT has no distillation head");
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSFORMER, "vb_forward_distill: CrossFormer has no distillation head");
    const bool levit = h->cfg.kind == VB_KIND_LEVIT;
    VB_CHECK(levit || distill_token != nullptr, "vb_forward_distill: null argument");
    VB_CHECK(!levit || (distill_token == nullptr && h->lv.num_distill_classes > 0),
             "vb_forward_distill: a LeViT takes no distillation token (pass NULL) and needs num_distill_classes > 0");
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const int dim = levit ? h->lv.num_distill_classes : h->cfg.dim;
    const size_t img_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const size_t log_bytes = static_cast<size_t>(batch) * h->cfg.num_classes * sizeof(float);
    const size_t dis_bytes = static_cast<size_t>(batch) * dim * sizeof(float);
    const float* img_d = img;
    if (img_mem == VB_MEM_HOST) {
      h->img_dev.ensure(img_bytes);
      VB_CUDA(cudaMemcpyAsync(h->img_dev.p, img, img_bytes, cudaMemcpyHostToDevice, s));
      img_d = static_cast<const float*>(h->img_dev.p);
    }
    // the distillation token is always a host vector of `dim` floats (a trainable variable of the caller, distill.py:133)
    if (!levit) {
      h->tokens_in.ensure(static_cast<size_t>(dim) * sizeof(float));
      VB_CUDA(cudaMemcpyAsync(h->tokens_in.p, distill_token, static_cast<size_t>(dim) * sizeof(float), cudaMemcpyHostToDevice, s));
    }
    float* log_d = logits;
    float* dis_d = distill_out;
    if (out_mem == VB_MEM_HOST) {
      h->logits_dev.ensure(log_bytes);
      h->tokens_out.ensure(dis_bytes);
      log_d = static_cast<float*>(h->logits_dev.p);
      dis_d = static_cast<float*>(h->tokens_out.p);
    }
    const float* tok_d = static_cast<const float*>(h->tokens_in.p);
    if (levit) {
      h->arena.reset();
      if (h->bf16()) h->levit_forward<__nv_bfloat16>(img_d, batch, img_h, img_w, log_d, dis_d, s);
      else h->levit_forward<float>(img_d, batch, img_h, img_w, log_d, dis_d, s);
    } else if (h->bf16()) {
      h->distill_impl<__nv_bfloat16>(img_d, batch, img_h, img_w, tok_d, log_d, dis_d, s);
    } else {
      h->distill_impl<float>(img_d, batch, img_h, img_w, tok_d, log_d, dis_d, s);
    }
    h->last_launches = launch_counter() - before;
    if (out_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(logits, log_d, log_bytes, cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaMemcpyAsync(distill_out, dis_d, dis_bytes, cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_forward_tokens(vb_handle* h, const float* tokens, int32_t tokens_mem, int32_t batch, int32_t n, float* out,
                      int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && tokens != nullptr && out != nullptr, "vb_forward_tokens: null argument");
    VB_CHECK(h->finalized, "vb_forward_tokens: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && n > 0, "vb_forward_tokens: bad shape");
    VB_CHECK(h->cfg.kind != VB_KIND_CVT, vb_handle::kCvtNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_TWINS_SVT, vb_handle::kTwinsNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSFORMER, vb_handle::kCrossformerNoStages);
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const size_t bytes = static_cast<size_t>(batch) * n * h->cfg.dim * sizeof(float);
    const float* in_d = tokens;
    float* out_d = out;
    if (tokens_mem == VB_MEM_HOST || out_mem == VB_MEM_HOST) h->tok_dev.ensure(2 * bytes);
    if (tokens_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(h->tok_dev.p, tokens, bytes, cudaMemcpyHostToDevice, s));
      in_d = static_cast<const float*>(h->tok_dev.p);
    }
    if (out_mem == VB_MEM_HOST) out_d = reinterpret_cast<float*>(static_cast<char*>(h->tok_dev.p) + bytes);
    if (h->bf16()) h->tokens_impl<__nv_bfloat16>(in_d, batch, n, out_d, s);
    else h->tokens_impl<float>(in_d, batch, n, out_d, s);
    h->last_launches = launch_counter() - before;
    if (out_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(out, out_d, bytes, cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_embed_rows(vb_handle* h, int32_t img_h, int32_t img_w) {
  int rows = -1;
  const int rc = guarded(h, [&] {
    VB_CHECK(h != nullptr && img_h > 0 && img_w > 0, "vb_embed_rows: bad arguments");
    rows = h->embed_rows(img_h, img_w);
  });
  return rc == 0 ? rows : -rc;
}

int vb_forward_embed(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* tokens,
                     int32_t tokens_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && tokens != nullptr, "vb_forward_embed: null argument");
    VB_CHECK(h->finalized, "vb_forward_embed: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward_embed: bad batch / image size");
    const int rows = h->embed_rows(img_h, img_w);
    const size_t in_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const size_t out_bytes = static_cast<size_t>(batch) * rows * h->cfg.dim * sizeof(float);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    staged_call(h, img, img_mem, in_bytes, tokens, tokens_mem, out_bytes, s, [&](const float* in_d, float* out_d) {
      if (h->bf16()) h->embed_impl<__nv_bfloat16>(in_d, batch, img_h, img_w, out_d, s);
      else h->embed_impl<float>(in_d, batch, img_h, img_w, out_d, s);
    });
  });
}

int vb_forward_head(vb_handle* h, const float* tokens, int32_t tokens_mem, int32_t batch, int32_t n, float* logits,
                    int32_t logits_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && tokens != nullptr && logits != nullptr, "vb_forward_head: null argument");
    VB_CHECK(h->finalized, "vb_forward_head: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && n > 0, "vb_forward_head: bad shape");
    const size_t in_bytes = static_cast<size_t>(batch) * n * h->cfg.dim * sizeof(float);
    const size_t out_bytes = static_cast<size_t>(batch) * h->cfg.num_classes * sizeof(float);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    staged_call(h, tokens, tokens_mem, in_bytes, logits, logits_mem, out_bytes, s, [&](const float* in_d, float* out_d) {
      if (h->bf16()) h->head_impl<__nv_bfloat16>(in_d, batch, n, out_d, s);
      else h->head_impl<float>(in_d, batch, n, out_d, s);
    });
  });
}

int vb_to_patch(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* patches,
                int32_t patches_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && patches != nullptr, "vb_to_patch: null argument");
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSVIT && h->cfg.kind != VB_KIND_T2T_VIT && h->cfg.kind != VB_KIND_CCT &&
             h->cfg.kind != VB_KIND_LEVIT && h->cfg.kind != VB_KIND_CVT && h->cfg.kind != VB_KIND_TWINS_SVT &&
             h->cfg.kind != VB_KIND_CROSSFORMER,
             "vb_to_patch: the model has no single Rearrange patch layer");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_to_patch: bad batch / image size");
    const vb_config& c = h->cfg;
    VB_CHECK(img_h % c.patch_h == 0 && img_w % c.patch_w == 0, "Image dimensions must be divisible by the patch size.");
    const int np = (img_h / c.patch_h) * (img_w / c.patch_w), pd = c.patch_h * c.patch_w * c.channels;
    const size_t in_bytes = static_cast<size_t>(batch) * img_h * img_w * c.channels * sizeof(float);
    const size_t out_bytes = static_cast<size_t>(batch) * np * pd * sizeof(float);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    staged_call(h, img, img_mem, in_bytes, patches, patches_mem, out_bytes, s, [&](const float* in_d, float* out_d) {
      im2col<float>(in_d, out_d, batch, img_h, img_w, c.channels, c.patch_h, c.patch_w, 0, pd, s);
    });
  });
}

int vb_patch_to_emb(vb_handle* h, const float* patches, int32_t patches_mem, int32_t rows, float* out, int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && patches != nullptr && out != nullptr, "vb_patch_to_emb: null argument");
    VB_CHECK(h->finalized, "vb_patch_to_emb: call vb_finalize after setting the weights");
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSVIT, "vb_patch_to_emb: CrossViT has two patch embeddings");
    VB_CHECK(h->cfg.kind != VB_KIND_CCT, vb_handle::kCctNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_LEVIT, vb_handle::kLevitNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_CVT, vb_handle::kCvtNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_TWINS_SVT, vb_handle::kTwinsNoStages);
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSFORMER, vb_handle::kCrossformerNoStages);
    VB_CHECK(rows > 0, "vb_patch_to_emb: bad shape");
    const size_t in_bytes = static_cast<size_t>(rows) * h->embed.patch.K * sizeof(float);
    const size_t out_bytes = static_cast<size_t>(rows) * h->cfg.dim * sizeof(float);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    staged_call(h, patches, patches_mem, in_bytes, out, out_mem, out_bytes, s, [&](const float* in_d, float* out_d) {
      if (h->bf16()) h->patch_to_emb_impl<__nv_bfloat16>(in_d, rows, out_d, s);
      else h->patch_to_emb_impl<float>(in_d, rows, out_d, s);
    });
  });
}

int vb_dp_unique_id(void* id128) {
  return guarded(nullptr, [&] {
    VB_CHECK(id128 != nullptr, "vb_dp_unique_id: null argument");
    NcclId id;
    nccl_check(nccl().GetUniqueId(&id), "ncclGetUniqueId");
    memcpy(id128, id.internal, sizeof id.internal);
  });
}

int vb_dp_init(vb_handle* h, const void* id128, int32_t rank, int32_t world) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && id128 != nullptr, "vb_dp_init: null argument");
    VB_CHECK(world >= 1 && rank >= 0 && rank < world, "vb_dp_init: need 0 <= rank < world");
    VB_CHECK(h->dp_comm == nullptr, "vb_dp_init: the handle already belongs to a data-parallel group");
    VB_CUDA(cudaSetDevice(h->device));
    NcclId id;
    memcpy(id.internal, id128, sizeof id.internal);
    void* comm = nullptr;
    nccl_check(nccl().CommInitRank(&comm, world, id, rank), "ncclCommInitRank");
    h->dp_comm = comm; h->dp_rank = rank; h->dp_world = world;
  });
}

int vb_forward_allgather(vb_handle* h, const float* img, int32_t img_mem, int32_t local_batch, int32_t img_h, int32_t img_w,
                         float* gathered, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && gathered != nullptr, "vb_forward_allgather: null argument");
    VB_CHECK(h->dp_comm != nullptr, "vb_forward_allgather: call vb_dp_init first");
    const size_t count = static_cast<size_t>(local_batch) * h->cfg.num_classes;
    float* mine = gathered + static_cast<size_t>(h->dp_rank) * count;        // this rank's slice of the gather buffer
    const int rc = vb_forward(h, img, img_mem, local_batch, img_h, img_w, mine, VB_MEM_DEVICE, stream);
    if (rc != 0) throw vb::Error(rc, h->error);
    // in place (sendbuff = recvbuff + rank * count), same stream: the head kernel's logits feed the collective directly
    nccl_check(nccl().AllGather(mine, gathered, count, /*ncclFloat32*/ 7, h->dp_comm, static_cast<cudaStream_t>(stream)),
               "ncclAllGather");
  });
}

int64_t vb_last_launch_count(vb_handle* h) { return h ? h->last_launches : -1; }

int vb_graph_stats(vb_handle* h, int64_t* captures, int64_t* replays, int64_t* failures, const char** last_failure) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    if (captures) *captures = h->graph_captures;
    if (replays) *replays = h->graph_replays;
    if (failures) *failures = h->graph_failures;
    if (last_failure) *last_failure = h->graph_last_failure.c_str();
  });
}

int32_t vb_last_attention_path(void) { return take_last_attention_path(); }

int vb_profile_enable(vb_handle* h, int32_t on) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CUDA(cudaSetDevice(h->device));
    h->prof_collect();
    h->profiling = on != 0;
  });
}

int vb_profile_read(vb_handle* h, double* ms, double* flops, double* bytes, int64_t* calls, int32_t reset) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CUDA(cudaSetDevice(h->device));
    h->prof_collect();
    for (int i = 0; i < vb_handle::PROF_NUM; ++i) {
      if (ms) ms[i] = h->prof_ms[i];
      if (flops) flops[i] = h->prof_flops[i];
      if (bytes) bytes[i] = h->prof_bytes[i];
      if (calls) calls[i] = h->prof_calls[i];
      if (reset) { h->prof_ms[i] = h->prof_flops[i] = h->prof_bytes[i] = 0; h->prof_calls[i] = 0; }
    }
  });
}

const char* vb_last_error(vb_handle* h) { return h ? h->error.c_str() : g_last_error.c_str(); }

void vb_destroy(vb_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->dp_comm != nullptr) { nccl().CommDestroy(h->dp_comm); h->dp_comm = nullptr; }
  attention_mix_cache_erase(h->weight_pointers());
  h->drop_graphs();
  for (auto& w : h->weights) if (w.dev) cudaFree(w.dev);
  h->prof_collect();
  for (auto e : h->event_pool) cudaEventDestroy(e);
  h->destroy_side_streams();
  delete h;
}


int vb_op_linear(int32_t precision, const float* a, const float* w, const float* bias, const float* scale, const float* res,
                 int32_t gelu, float* out, int32_t M, int32_t N, int32_t K, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(a && w && out && M > 0 && N > 0 && K > 0, "vb_op_linear: bad arguments");
    DevMem dA, dW, dWt, dB, dS, dR, dO;
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    const float* ds = scale ? upload<float>(dS, scale, N) : nullptr;
    const float* dw = upload<float>(dW, w, static_cast<size_t>(K) * N);
    if (precision == VB_PRECISION_FP32) {
      const float* da = upload<float>(dA, a, static_cast<size_t>(M) * K);
      const float* dr = res ? upload<float>(dR, res, static_cast<size_t>(M) * N) : nullptr;
      dO.ensure(static_cast<size_t>(M) * N * 4);
      float* dout = static_cast<float*>(dO.p);
      timed(iters, elapsed_ms, [&] { gemm_simt<float, float, float>(da, K, dw, N, 1, dout, N, M, N, K, db, ds, dr, N, gelu, 0); });
      download<float>(dout, out, static_cast<size_t>(M) * N);
    } else {
      VB_CHECK(gemm_bf16_supported(M, N, K, K, K, N), "vb_op_linear(bf16): need N % 64 == 0 and K % 8 == 0");
      const __nv_bfloat16* da = upload<__nv_bfloat16>(dA, a, static_cast<size_t>(M) * K);
      const __nv_bfloat16* dr = res ? upload<__nv_bfloat16>(dR, res, static_cast<size_t>(M) * N) : nullptr;
      dWt.ensure(static_cast<size_t>(N) * K * 2);
      pack_weight_bf16(dw, static_cast<__nv_bfloat16*>(dWt.p), K, N, K, 0);
      dO.ensure(static_cast<size_t>(M) * N * 2);
      __nv_bfloat16* dout = static_cast<__nv_bfloat16*>(dO.p);
      GemmBf16 g = gemm_bf16_plan(da, K, static_cast<const __nv_bfloat16*>(dWt.p), K, dout, N, M, N, K, db, ds, dr, N, gelu != 0);
      timed(iters, elapsed_ms, [&] { gemm_bf16_run(g, 0); });
      download<__nv_bfloat16>(dout, out, static_cast<size_t>(M) * N);
    }
  });
}

int vb_op_attention(int32_t precision, int32_t variant, const float* q, const float* k, const float* v, const float* mix_a,
                    const float* mix_b, const float* ln_gamma, const float* ln_beta, float* out, int32_t B, int32_t nq, int32_t nk,
                    int32_t heads, int32_t dim_head, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(q && k && v && out && B > 0 && nq > 0 && nk > 0 && heads > 0 && dim_head > 0, "vb_op_attention: bad arguments");
    VB_CHECK(variant >= 0 && variant <= 2, "vb_op_attention: variant must be 0, 1 or 2");
    const int inner = heads * dim_head;
    DevMem dQ, dK, dV, dO, dS, dMa, dMb, dG, dBt;
    const float* ma = mix_a ? upload<float>(dMa, mix_a, heads * heads) : nullptr;
    const float* mb = mix_b ? upload<float>(dMb, mix_b, heads * heads) : nullptr;
    const float* g = ln_gamma ? upload<float>(dG, ln_gamma, heads) : nullptr;
    const float* bt = ln_beta ? upload<float>(dBt, ln_beta, heads) : nullptr;
    const MixCacheScope mix_scope{{ma, mb, g, bt}};
    const size_t cq = static_cast<size_t>(B) * nq * inner, ck = static_cast<size_t>(B) * nk * inner;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* q_d = upload<T>(dQ, q, cq);
      const T* k_d = upload<T>(dK, k, ck);
      const T* v_d = upload<T>(dV, v, ck);
      dO.ensure(cq * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      dS.ensure(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15) * 4);
      timed(iters, elapsed_ms, [&] {
        if (!attention_fast<T>(q_d, inner, k_d, inner, v_d, inner, o_d, inner, B, nq, nk, heads, dim_head, variant, ma, mb, g, bt, 0))
          attention_generic<T>(q_d, inner, k_d, inner, v_d, inner, o_d, inner, static_cast<float*>(dS.p), B, nq, nk, heads,
                               dim_head, variant, ma, mb, g, bt, 0);
      });
      download<T>(o_d, out, cq);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_patch_merger(int32_t precision, const float* x, const float* gamma, const float* beta, const float* queries, float* out,
                       int32_t B, int32_t n, int32_t D, int32_t nt, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && queries && out && B > 0 && n > 0 && D > 0 && nt > 0, "vb_op_patch_merger: bad arguments");
    DevMem dX, dG, dB, dQf, dY, dQ, dO, dS;
    const float* g = upload<float>(dG, gamma, D);
    const float* b = upload<float>(dB, beta, D);
    const float* qf = upload<float>(dQf, queries, static_cast<size_t>(nt) * D);
    const size_t cx = static_cast<size_t>(B) * n * D, co = static_cast<size_t>(B) * nt * D;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, cx);
      dY.ensure(cx * sizeof(T) + 16); dQ.ensure(co * sizeof(T) + 16); dO.ensure(co * sizeof(T) + 16);
      dS.ensure(static_cast<size_t>(B) * nt * ((n + 15) & ~15) * 4);
      T* y_d = static_cast<T*>(dY.p);
      T* q_d = static_cast<T*>(dQ.p);
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] {
        layernorm<T>(x_d, D, g, b, y_d, D, B * n, D, 0);
        broadcast_rows<T>(qf, q_d, B, nt, D, 0);
        if (!attention_fast<T>(q_d, D, y_d, D, y_d, D, o_d, D, B, nt, n, 1, D, 0, nullptr, nullptr, nullptr, nullptr, 0))
          attention_generic<T>(q_d, D, y_d, D, y_d, D, o_d, D, static_cast<float*>(dS.p), B, nt, n, 1, D, 0, nullptr, nullptr, nullptr,
                               nullptr, 0);
      });
      download<T>(o_d, out, co);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_layernorm(int32_t precision, const float* x, const float* gamma, const float* beta, float* out, int32_t M, int32_t D,
                    int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && out && M > 0 && D > 0, "vb_op_layernorm: bad arguments");
    DevMem dX, dG, dB, dO;
    const float* g = upload<float>(dG, gamma, D);
    const float* b = upload<float>(dB, beta, D);
    const size_t cnt = static_cast<size_t>(M) * D;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, cnt);
      dO.ensure(cnt * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] { layernorm<T>(x_d, D, g, b, o_d, D, M, D, 0); });
      download<T>(o_d, out, cnt);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_ln_linear(const float* x, const float* gamma, const float* beta, const float* w, const float* bias, int32_t gelu,
                    float* out, int32_t M, int32_t N, int32_t K, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && w && out && M > 0 && N > 0 && K > 0, "vb_op_ln_linear: bad arguments");
    VB_CHECK(N % 64 == 0 && K % 64 == 0, "vb_op_ln_linear: the folded form needs N % 64 == 0 and K % 64 == 0");
    DevMem dX, dG, dBt, dW, dWt, dB, dC, dSt, dO;
    const __nv_bfloat16* dx = upload<__nv_bfloat16>(dX, x, static_cast<size_t>(M) * K);
    const float* g = upload<float>(dG, gamma, K);
    const float* bt = upload<float>(dBt, beta, K);
    const float* dw = upload<float>(dW, w, static_cast<size_t>(K) * N);
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    dWt.ensure(static_cast<size_t>(N) * K * 2);
    __nv_bfloat16* wt = static_cast<__nv_bfloat16*>(dWt.p);
    pack_weight_bf16(dw, wt, K, N, K, 0, g);                       // gamma folded into the packed weight rows
    dC.ensure(static_cast<size_t>(N) * 2 * sizeof(float));
    float* c = static_cast<float*>(dC.p);
    ln_fold_consts(dw, wt, K, bt, db, c, c + N, K, N, 0);
    dSt.ensure(static_cast<size_t>(M) * (K / 64) * 2 * sizeof(float));
    float* st = static_cast<float*>(dSt.p);
    dO.ensure(static_cast<size_t>(M) * N * 2);
    __nv_bfloat16* dout = static_cast<__nv_bfloat16*>(dO.p);
    GemmBf16 gm = gemm_bf16_plan(dx, K, wt, K, dout, N, M, N, K, c + N, nullptr, nullptr, 0, gelu != 0);
    gm.ln_c1 = c; gm.ln_stats = st; gm.ln_parts = K / 64; gm.ln_inv_d = 1.0f / static_cast<float>(K);
    timed(iters, elapsed_ms, [&] { row_stats_bf16(dx, K, st, M, K, 0); gemm_bf16_run(gm, 0); });
    download<__nv_bfloat16>(dout, out, static_cast<size_t>(M) * N);
  });
}

int vb_op_gemm(const float* a, int32_t lda, const float* wt, int32_t ldw, int32_t b_rows, const float* bias, const float* scale,
               int32_t gelu, const float* res, int32_t ldr, const float* ln_stats, const float* ln_c1, float* out, int32_t ldc,
               int32_t out_off, int32_t out_f32, float* stats_out, int32_t M, int32_t N, int32_t K, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(a && wt && out && M > 0 && N > 0 && K > 0 && lda >= K && ldw >= K && b_rows >= 0 && b_rows <= N && out_off >= 0 &&
             out_off + N <= ldc, "vb_op_gemm: bad arguments");
    const bool in_place = res != nullptr && res == out;
    VB_CHECK(!in_place || ldr == ldc, "vb_op_gemm: an in-place residual has the output's pitch (ldr == ldc)");
    VB_CHECK(res == nullptr || in_place || ldr >= N, "vb_op_gemm: ldr < N");
    VB_CHECK((ln_stats == nullptr) == (ln_c1 == nullptr), "vb_op_gemm: the folded LayerNorm needs both ln_stats and ln_c1");
    VB_CHECK(ln_c1 == nullptr || (bias != nullptr && K % 64 == 0), "vb_op_gemm: the folded LayerNorm needs the c2 bias and K % 64 == 0");
    DevMem dA, dW, dB, dS, dR, dO, dC1, dLs, dSo;
    const __nv_bfloat16* da = upload<__nv_bfloat16>(dA, a, static_cast<size_t>(M) * lda);
    const __nv_bfloat16* dw = upload<__nv_bfloat16>(dW, wt, static_cast<size_t>(b_rows > 0 ? b_rows : N) * ldw);
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    const float* ds = scale ? upload<float>(dS, scale, N) : nullptr;
    const size_t co = static_cast<size_t>(M) * ldc;
    void* dout = out_f32 ? static_cast<void*>(upload<float>(dO, out, co) + out_off)
                         : static_cast<void*>(upload<__nv_bfloat16>(dO, out, co) + out_off);
    const __nv_bfloat16* dr = in_place ? static_cast<const __nv_bfloat16*>(dout)
                              : res ? upload<__nv_bfloat16>(dR, res, static_cast<size_t>(M) * ldr) : nullptr;
    // the plan exactly as vb_handle::linear / gemm_cached build it
    GemmBf16 g = gemm_bf16_plan(da, lda, dw, ldw, static_cast<__nv_bfloat16*>(dout), ldc, M, N, K, db, ds, dr, ldr, gelu != 0,
                                out_f32 != 0, b_rows);
    if (ln_c1) {
      g.ln_c1 = upload<float>(dC1, ln_c1, N);
      g.ln_stats = upload<float>(dLs, ln_stats, static_cast<size_t>(K / 64) * M * 2);
      g.ln_parts = K / 64;
      g.ln_inv_d = 1.0f / static_cast<float>(K);
    }
    const size_t cs = static_cast<size_t>(N / 64) * M * 2;
    if (stats_out) { dSo.ensure(cs * sizeof(float)); g.stats_out = static_cast<float*>(dSo.p); }
    auto launch = [&] { gemm_bf16_run(g, 0); };
    timed(0, nullptr, launch);                 // the result is the first launch's: an in-place residual accumulates on every launch
    if (out_f32) download<float>(static_cast<const float*>(dO.p), out, co);
    else download<__nv_bfloat16>(static_cast<const __nv_bfloat16*>(dO.p), out, co);
    if (stats_out) download<float>(g.stats_out, stats_out, cs);
    if (iters > 0) timed(iters, elapsed_ms, launch);
  });
}

int vb_op_attention_ex(int32_t precision, int32_t variant, const float* q, int32_t ldq, const float* kv, int32_t ldkv, int32_t k_off,
                       int32_t v_off, const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, float* out,
                       int32_t ldo, int32_t B, int32_t nq, int32_t nk, int32_t heads, int32_t dh, float scale, int32_t iters,
                       float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const bool fused = kv == nullptr;                  // k, v inside the q rows ([q|k|v]) or inside separate [k|v] rows
    const int ldk = fused ? ldq : ldkv;
    const long long inner = static_cast<long long>(heads) * dh;
    VB_CHECK(q && out && B > 0 && nq > 0 && nk > 0 && heads > 0 && dh > 0 && ldq >= inner && ldo >= inner && k_off >= 0 &&
             v_off >= 0 && k_off + inner <= ldk && v_off + inner <= ldk && (!fused || nk == nq), "vb_op_attention_ex: bad arguments");
    VB_CHECK(variant >= 0 && variant <= 2, "vb_op_attention_ex: variant must be 0, 1 or 2");
    DevMem dQ, dKV, dO, dS, dMa, dMb, dG, dBt;
    const float* ma = mix_a ? upload<float>(dMa, mix_a, heads * heads) : nullptr;
    const float* mb = mix_b ? upload<float>(dMb, mix_b, heads * heads) : nullptr;
    const float* g = ln_gamma ? upload<float>(dG, ln_gamma, heads) : nullptr;
    const float* bt = ln_beta ? upload<float>(dBt, ln_beta, heads) : nullptr;
    const MixCacheScope mix_scope{{ma, mb, g, bt}};
    const size_t cq = static_cast<size_t>(B) * nq * ldq, ckv = static_cast<size_t>(B) * nk * ldk, co = static_cast<size_t>(B) * nq * ldo;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* q_d = upload<T>(dQ, q, cq);
      const T* kv_d = fused ? q_d : upload<T>(dKV, kv, ckv);
      T* o_d = upload<T>(dO, out, co);
      dS.ensure(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15) * 4);
      // vb_handle::attention_dispatch without the handle's arena and profiler
      timed(iters, elapsed_ms, [&] {
        if (attention_fast<T>(q_d, ldq, kv_d + k_off, ldk, kv_d + v_off, ldk, o_d, ldo, B, nq, nk, heads, dh, variant, ma, mb, g, bt, 0,
                              scale))
          return;
        VB_CHECK(scale <= 0.f, "vb_op_attention_ex: an explicit softmax scale needs the fused attention kernels");
        attention_generic<T>(q_d, ldq, kv_d + k_off, ldk, kv_d + v_off, ldk, o_d, ldo, static_cast<float*>(dS.p), B, nq, nk, heads, dh,
                             variant, ma, mb, g, bt, 0);
      });
      download<T>(o_d, out, co);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_attention_bias(int32_t precision, const float* q, int32_t ldq, const float* k, int32_t ldk, const float* v, int32_t ldv,
                         const float* pos_bias, float* out, int32_t ldo, int32_t B, int32_t heads, int32_t dh, int32_t fmap,
                         int32_t q_step, float scale, int32_t gelu_out, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const long long inner = static_cast<long long>(heads) * dh;
    VB_CHECK(q && k && v && pos_bias && out && B > 0 && heads > 0 && dh > 0 && fmap > 0 && (q_step == 1 || q_step == 2) && scale > 0.f &&
             ldq >= inner && ldk >= inner && ldv >= inner && ldo >= inner, "vb_op_attention_bias: bad arguments");
    const int f2 = fmap * fmap, nqs = (fmap + q_step - 1) / q_step, nq = nqs * nqs, nk = f2;
    std::vector<float> tab(static_cast<size_t>(heads) * f2);        // [heads][fmap^2] / scale, as vb_finalize packs it
    for (int h = 0; h < heads; ++h)
      for (int e = 0; e < f2; ++e)
        tab[static_cast<size_t>(h) * f2 + e] = static_cast<float>(static_cast<double>(pos_bias[static_cast<size_t>(e) * heads + h]) / scale);
    DevMem dQ, dK, dV, dO, dS, dT;
    dT.ensure(tab.size() * sizeof(float));
    VB_CUDA(cudaMemcpy(dT.p, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
    PosBias pb;
    pb.table = static_cast<const float*>(dT.p); pb.fmap = fmap; pb.step = q_step; pb.gelu_out = gelu_out != 0;
    const size_t cq = static_cast<size_t>(B) * nq * ldq, co = static_cast<size_t>(B) * nq * ldo;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* q_d = upload<T>(dQ, q, cq);
      const T* k_d = upload<T>(dK, k, static_cast<size_t>(B) * nk * ldk);
      const T* v_d = upload<T>(dV, v, static_cast<size_t>(B) * nk * ldv);
      T* o_d = upload<T>(dO, out, co);
      dS.ensure(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15) * 4);
      // vb_handle::attention_bias without the handle's arena and profiler
      timed(iters, elapsed_ms, [&] {
        if (attention_fast<T>(q_d, ldq, k_d, ldk, v_d, ldv, o_d, ldo, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, 0, scale, &pb))
          return;
        attention_generic<T>(q_d, ldq, k_d, ldk, v_d, ldv, o_d, ldo, static_cast<float*>(dS.p), B, nq, nk, heads, dh, 0, nullptr, nullptr,
                             nullptr, nullptr, 0, scale, &pb);
      });
      download<T>(o_d, out, co);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_dwconv(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* ln_gamma, const float* ln_beta,
                 int32_t k, int32_t kv_stride, const float* wq, const float* bn_q, const float* wkv, const float* bn_kv, float* q, float* kv,
                 int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && ln_gamma && ln_beta && wq && bn_q && wkv && bn_kv && q && kv && B > 0 && H > 0 && W > 0 && C > 0 && k >= 1 && k <= 7 &&
             (kv_stride == 1 || kv_stride == 2), "vb_op_dwconv: bad arguments");
    const bool bf = precision == VB_PRECISION_BF16;
    const int Cp = bf ? round_up(C, 64) : C, Ho = (H + kv_stride - 1) / kv_stride, Wo = (W + kv_stride - 1) / kv_stride;
    const size_t M = static_cast<size_t>(B) * H * W, Mk = static_cast<size_t>(B) * Ho * Wo;
    auto vec = [](const float* p, size_t n) { return std::vector<double>(p, p + n); };
    auto fold = [&](const float* w, const float* bn, std::vector<float>& taps, std::vector<float>& shift) {   // as vb_finalize folds
      std::vector<double> wd, sd;
      cvt_fold_dw(vec(w, static_cast<size_t>(k) * k * C), vec(bn, C), vec(bn + C, C), vec(bn + 2 * C, C), vec(bn + 3 * C, C), k, C, Cp, wd, sd);
      taps.assign(wd.begin(), wd.end());
      shift.assign(sd.begin(), sd.end());
    };
    std::vector<float> tq, sq, tkv, skv, xp(M * Cp, 0.f), gp(Cp, 0.f), bp(Cp, 0.f);
    fold(wq, bn_q, tq, sq);
    fold(wkv, bn_kv, tkv, skv);
    for (size_t r = 0; r < M; ++r) std::copy(x + r * C, x + (r + 1) * C, xp.begin() + r * Cp);
    std::copy(ln_gamma, ln_gamma + C, gp.begin());
    std::copy(ln_beta, ln_beta + C, bp.begin());
    DevMem dX, dG, dB, dTq, dSq, dTkv, dSkv, dQ, dKV, dS, dY;
    const float* g_d = upload<float>(dG, gp.data(), Cp);
    const float* b_d = upload<float>(dB, bp.data(), Cp);
    const float* tq_d = upload<float>(dTq, tq.data(), tq.size());
    const float* sq_d = upload<float>(dSq, sq.data(), sq.size());
    const float* tkv_d = upload<float>(dTkv, tkv.data(), tkv.size());
    const float* skv_d = upload<float>(dSkv, skv.data(), skv.size());
    std::vector<float> qh(M * Cp), kvh(Mk * Cp);
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, xp.data(), M * Cp);
      dQ.ensure(M * Cp * sizeof(T));
      dKV.ensure(Mk * Cp * sizeof(T));
      T* q_d = static_cast<T*>(dQ.p);
      T* kv_d = static_cast<T*>(dKV.p);
      // vb_handle::cvt_block's depthwise step, without the handle's arena and profiler
      if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        dS.ensure(M * (Cp / 64) * 2 * sizeof(float));
        float* st = static_cast<float*>(dS.p);
        timed(iters, elapsed_ms, [&] {
          row_stats_bf16(x_d, Cp, st, static_cast<int>(M), Cp, 0);
          dwconv_qkv<T>(x_d, Cp, st, g_d, b_d, C, 1e-5f, tq_d, sq_d, q_d, Cp, tkv_d, skv_d, kv_d, Cp, B, H, W, Cp, k, kv_stride, 0);
        });
      } else {
        dY.ensure(M * Cp * sizeof(T));
        T* y = static_cast<T*>(dY.p);
        timed(iters, elapsed_ms, [&] {
          layernorm<T>(x_d, Cp, g_d, b_d, y, Cp, static_cast<int>(M), C, 0, Cp, 1e-5f);
          dwconv_qkv<T>(y, Cp, nullptr, nullptr, nullptr, C, 1e-5f, tq_d, sq_d, q_d, Cp, tkv_d, skv_d, kv_d, Cp, B, H, W, Cp, k, kv_stride, 0);
        });
      }
      download<T>(q_d, qh.data(), M * Cp);
      download<T>(kv_d, kvh.data(), Mk * Cp);
    };
    if (bf) run(__nv_bfloat16());
    else run(float());
    for (size_t r = 0; r < M; ++r) std::copy(qh.begin() + r * Cp, qh.begin() + r * Cp + C, q + r * C);
    for (size_t r = 0; r < Mk; ++r) std::copy(kvh.begin() + r * Cp, kvh.begin() + r * Cp + C, kv + r * C);
  });
}

int vb_op_window_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t p, int32_t heads,
                           int32_t dh, float* out, int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && out && B > 0 && p > 0 && H > 0 && W > 0 && H % p == 0 && W % p == 0 && heads > 0 && dh > 0 && ld >= 3 * HD && ldo >= HD,
             "vb_op_window_attention: bad arguments");
    Window win;
    win.p = p; win.nx = W / p; win.ny = H / p;
    const int n = p * p, Bw = B * win.nx * win.ny;
    const long long rows = static_cast<long long>(B) * H * W;
    DevMem dX, dO, dW, dOw, dS;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      // vb_handle::attention_dispatch's windowed branch without the handle's arena and profiler
      timed(iters, elapsed_ms, [&] {
        if (attention_fast<T>(x_d, ld, x_d + HD, ld, x_d + 2 * HD, ld, o_d, ldo, Bw, n, n, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, 0, 0.f,
                              nullptr, &win))
          return;
        dW.ensure(static_cast<size_t>(rows) * 3 * HD * sizeof(T));
        dOw.ensure(static_cast<size_t>(rows) * HD * sizeof(T));
        dS.ensure(static_cast<size_t>(Bw) * heads * n * ((n + 15) & ~15) * sizeof(float));
        T* w_d = static_cast<T*>(dW.p);
        T* ow_d = static_cast<T*>(dOw.p);
        window_rows<T>(x_d, ld, w_d, 3 * HD, 3 * HD, win, rows, true, 0);
        attention_generic<T>(w_d, 3 * HD, w_d + HD, 3 * HD, w_d + 2 * HD, 3 * HD, ow_d, HD, static_cast<float*>(dS.p), Bw, n, n, heads, dh, 0,
                             nullptr, nullptr, nullptr, nullptr, 0);
        window_rows<T>(ow_d, HD, o_d, ldo, HD, win, rows, false, 0);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_window_bias_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t wsz,
                                int32_t is_long, int32_t heads, int32_t dh, const float* table, float* out, int32_t ldo, int32_t iters,
                                float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && table && out && B > 0 && wsz > 0 && H > 0 && W > 0 && H % wsz == 0 && W % wsz == 0 && heads > 0 && dh > 0 &&
             ld >= 3 * HD && ldo >= HD, "vb_op_window_bias_attention: bad arguments");
    Window win;
    win.p = wsz; win.nx = W / wsz; win.ny = H / wsz; win.dilated = is_long != 0;
    const int n = wsz * wsz, Bw = B * win.nx * win.ny, t = (2 * wsz - 1) * (2 * wsz - 1);
    const long long rows = static_cast<long long>(B) * H * W;
    DevMem dX, dO, dW, dOw, dS, dT;
    PosBias pb;
    pb.table = upload<float>(dT, table, t); pb.wsz = wsz;
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      // vb_handle::attention_dispatch's windowed branch without the handle's arena and profiler
      timed(iters, elapsed_ms, [&] {
        if (attention_fast<T>(x_d, ld, x_d + HD, ld, x_d + 2 * HD, ld, o_d, ldo, Bw, n, n, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, 0, 0.f,
                              &pb, &win))
          return;
        dW.ensure(static_cast<size_t>(rows) * 3 * HD * sizeof(T));
        dOw.ensure(static_cast<size_t>(rows) * HD * sizeof(T));
        dS.ensure(static_cast<size_t>(Bw) * heads * n * ((n + 15) & ~15) * sizeof(float));
        T* w_d = static_cast<T*>(dW.p);
        T* ow_d = static_cast<T*>(dOw.p);
        window_rows<T>(x_d, ld, w_d, 3 * HD, 3 * HD, win, rows, true, 0);
        attention_generic<T>(w_d, 3 * HD, w_d + HD, 3 * HD, w_d + 2 * HD, 3 * HD, ow_d, HD, static_cast<float*>(dS.p), Bw, n, n, heads, dh, 0,
                             nullptr, nullptr, nullptr, nullptr, 0, 0.f, &pb);
        window_rows<T>(ow_d, HD, o_d, ldo, HD, win, rows, false, 0);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
  });
}

int vb_op_softmax_rows(const float* s, int32_t lds, float* p, int32_t ldp, int32_t rows, int32_t n, int32_t npad, float scale,
                       int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(s && p && rows > 0 && n > 0 && n <= lds && n <= npad && npad <= ldp, "vb_op_softmax_rows: bad arguments");
    DevMem dS, dP;
    const float* s_d = upload<float>(dS, s, static_cast<size_t>(rows) * lds);
    __nv_bfloat16* p_d = upload<__nv_bfloat16>(dP, p, static_cast<size_t>(rows) * ldp);
    const float scale_log2 = scale * 1.4426950408889634f;       // as vb_handle::layer_t2t passes it
    timed(iters, elapsed_ms, [&] { softmax_rows_bf16(s_d, lds, p_d, ldp, rows, n, npad, scale_log2, 0); });
    download<__nv_bfloat16>(p_d, p, static_cast<size_t>(rows) * ldp);
  });
}

}  // extern "C"
