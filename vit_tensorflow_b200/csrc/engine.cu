// libvitb200 engine: weight registry, workspace arena, forward orchestration of ViT / DeepViT / CaiT / CrossViT
// and the extern "C" boundary declared in include/vitb200.h.
//
// The op sequences restate the reference's call graphs (SURVEY.md section 3):
//   ViT / DeepViT  vit.py:159-177, deepvit.py:139-157      CaiT  cait.py:180-194      CrossViT  cross_vit.py:290-303
// with inference semantics (dropout = identity; vb_forward_train masks every Dropout site instead).  T = float runs the
// exact-fp32 SIMT kernels (numerics gate), T = __nv_bfloat16 runs the wgmma GEMM / tensor-core attention kernels with fp32
// accumulation and statistics.
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
  bool silu = false;                 // SiLU instead (MobileViT, mobile_vit.py:33)
  int act() const { return gelu ? ACT_GELU : hswish ? ACT_HSWISH : silu ? ACT_SILU : ACT_NONE; }
  void set_act(int a) { gelu = a == ACT_GELU; hswish = a == ACT_HSWISH; silu = a == ACT_SILU; }
  const float* ln_stats = nullptr;   // (sum, sumsq) partials per 64-column chunk of the A operand's rows for a LayerNorm-folded Dense, [M, K/64, 2]
  float* stats_out = nullptr;        // emit (sum, sumsq) partials of every 64-column chunk of the output rows, [M, N/64, 2]
  DropoutEpi drop;                   // training-mode dropout of the output (vb_handle::dropout)
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
  bool lsa = false;                  // locality self-attention (vit_for_small_dataset.py:88-121): the diagonal masked, scale lsa_scale
  float lsa_scale = 0.f;             // exp(temperature), taken in fp32 as TensorFlow does
  int site_out = -1, site_ff = -1;   // dropout sites (vb_handle::number_dropout_sites): to_out's; the GELU's, fc2's is site_ff + 1
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
struct MlpW { Norm norm; Linear fc1, fc2; int act = ACT_GELU; };   // PreNorm MLP: LayerNorm, fc1, activation (Act), fc2
struct CvtBlockW {
  int dim = 0, dp = 0, heads = 0, k = 0, kv_stride = 1;
  Norm attn_norm;                    // gamma / beta [dp], zero on pad channels
  const float *wq = nullptr, *bq = nullptr, *wkv = nullptr, *bkv = nullptr;
  Linear pw_q, pw_kv, to_out;
  MlpW ff;
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

// One NesT level (nest.py:125-148 and its Aggregate :111-123) on channel rows zero-padded to dp (bf16) / dim (fp32): x +=
// pos_emb[:h w], then `depth` blocks of x = to_out(attention(LN(x))) + x and x = MLP(LN(x)) + x within bs x bs blocks per map,
// then (aggregate) Conv2D(3, SAME) to dim_out, LayerNorm, MaxPool2D(3, 2, SAME).  The bf16 engine folds the PreNorm LayerNorms
// into q|k|v and fc1.  Heads of width dh = dim / heads of the model; inner = heads * dh may be below dim.
struct NestBlockW { Norm attn_norm; Linear qkv, to_out; MlpW ff; };
struct NestLevelW {
  int dim = 0, dp = 0, heads = 0, dh = 0, inner = 0, bs = 1;   // bs: blocks per map side (nest.py:208)
  const float* pos = nullptr;        // pos_emb [seq_len]
  std::vector<NestBlockW> blocks;
  bool aggregate = false;
  int dim_out = 0, dp_out = 0;
  Linear agg;                        // the 3 x 3 convolution as a Dense over unfold_same's (row, column, channel) vectors
  Norm agg_norm;                     // ag_layers.1, [dp_out]
};

// MobileViT (mobile_vit.py:130-206) on channel rows zero-padded to channel_width (bf16) / unpadded (fp32).  Every Conv_NxN_BN and
// MV2 convolution carries its BatchNormalization folded (a Dense with bias, or depthwise taps and a shift).
struct Mv2W {                        // one MV2Block (:130-170)
  int cin = 0, hidden = 0, cout = 0, stride = 1, cp_in = 0, hp = 0, cp_out = 0;
  bool expand = false, residual = false;
  Linear pw1;                        // 1x1 expand + BN, SiLU: [cp_in, hp]
  const float* dw_w = nullptr;       // 3x3 depthwise + BN: taps [9][hp] and shift [hp], zero on pad channels; SiLU
  const float* dw_b = nullptr;
  Linear pw2;                        // 1x1 project + BN: [hp, cp_out]
};
struct MvitLayerW { Norm attn_norm; Linear qkv, to_out; MlpW ff; };
struct MvitBlockW {                  // one MobileViTBlock (:173-206): the concat [conv3 out | block input] lives in one [rows, chp + cp_in] buffer
  int cin = 0, ch = 0, dim = 0, cp_in = 0, chp = 0, dp = 0, k = 3;
  Linear conv1, conv2, conv3, conv4;   // conv1 over unfold_same of the input's cin channels, conv4 over all chp + cp_in columns
  std::vector<MvitLayerW> layers;
};

// ScalableViT (scalable_vit.py:145-304) on channel rows zero-padded to channel_width (bf16) / unpadded (fp32).  q, k and v of each
// attention share one activation head width (SvitStageW::dhs / dhi): the largest of dim_key and dim_value, widened in bf16 to the
// flash kernels' 32 or 64 (or a multiple of 8 above 64) with zero weight columns; the to_out rows and the LIM's input rows and
// output columns follow the same head layout, with zero rows and columns at the pad positions.
struct SvitBlockW {                  // one block, in the order it runs (:236-245)
  Norm ssa_norm, iwsa_norm;          // g / b [dp], zero on pad channels
  Linear ssa_q;                      // [dp, ldq]: q at h * dhs
  Linear ssa_kv;                     // [r * r * dim, ldkv] over unfold's (row, column, channel) vectors: k at h * dhs, v at HS + h * dhs
  Linear ssa_out;                    // [ldq, dp]
  MlpW mlp1, mlp3;                   // construction elements 1 and 3
  const float *peg_w = nullptr, *peg_b = nullptr;   // element 2 (first block only): taps [9][dp] with the residual on the centre tap
  Linear iwsa_qkv;                   // [dp, ldqkv]: q | k | v, each HI = heads * dhi wide
  Linear lim;                        // [9 HI, ldlim] over unfold's vectors of v's HI channels
  Linear iwsa_out;                   // [ldlim, dp]
};
struct SvitStageW {
  int dim = 0, dp = 0, heads = 0, r = 1, window = 0, dhs = 0, dhi = 0;
  int ldq = 0, ldkv = 0, ldqkv = 0, ldlim = 0;   // row pitches of the SSA q (and its output), k|v, IWSA q|k|v and LIM output
  float ssa_scale = 0.f, iwsa_scale = 0.f;       // dim_key^-0.5 of the model
  std::vector<SvitBlockW> blocks;
  Norm norm;                         // the Transformer's LayerNorm (norm_output, :233)
  bool down = false;
  Linear down_conv;                  // Downsample (:71-78): [9 dim, channel_width(2 dim)] over unfold's vectors
};

// NesT's block attention and MobileViT's patch-position attention on the windowed flash kernel (attn_flash.cu): bf16 only, false
// for a shape it does not take.
inline bool block_attention_fast(const float*, int, float*, int, int, int, cudaStream_t, const Window&, float) { return false; }
inline bool block_attention_fast(const __nv_bfloat16* qkv, int ld, __nv_bfloat16* out, int ldo, int heads, int dh, cudaStream_t s,
                                 const Window& win, float scale) {
  return attention_block(qkv, ld, out, ldo, heads, dh, s, scale, win);
}

// One RegionViT stage (regionvit.py:231-240) on channel rows zero-padded to dp (bf16) / dim (fp32): the shared Downsample (s >= 1),
// the PEG (s >= 1 with use_peg), then the R2L layers.  Each layer's one Attention module (4 heads of 32, inner 128) serves the
// regional self-attention and the regional-to-local attention; the bf16 engine folds its LayerNorm (and the MLP's) into q|k|v
// (fc1).
struct RegionLayerW { Norm attn_norm; Linear qkv, to_out; MlpW ff; };
struct RegionStageW {
  int dim = 0, dp = 0;
  bool down = false, peg = false;
  Linear down_conv;                  // Conv2D(3, 2, SAME) as a Dense over unfold_same's (row, column, channel) vectors
  const float* peg_w = nullptr;      // PEG taps [9][dp] with the residual folded into the centre tap, and its bias [dp]
  const float* peg_b = nullptr;
  const float* table = nullptr;      // local_rel_pos_bias as [4][(2 ws - 1)^2], row offset slowest (PosBias::r2l_ws)
  std::vector<RegionLayerW> layers;
};

// RegionViT's Embedding((2 ws - 1)^2, heads) (regionvit.py:126), looked up at row (dr + ws - 1) + (dc + ws - 1) (2 ws - 1) (:152),
// as [heads][(dr + ws - 1) (2 ws - 1) + dc + ws - 1]: the row-offset-slowest convention of the windowed attention kernels
template <typename F>
std::vector<double> r2l_table_from_embedding(const F* emb, int ws, int heads) {
  const int side = 2 * ws - 1;
  std::vector<double> t(static_cast<size_t>(heads) * side * side);
  for (int h = 0; h < heads; ++h)
    for (int a = 0; a < side; ++a)
      for (int c = 0; c < side; ++c) t[(static_cast<size_t>(h) * side + a) * side + c] = emb[(static_cast<size_t>(a) + c * side) * heads + h];
  return t;
}

// RegionViT's regional-to-local attention on its flash kernel (attn_flash.cu): bf16 only, false for a shape it does not take.
inline bool r2l_attention_fast(const float*, int, float*, int, int, int, long long, const PosBias&, const Window&, cudaStream_t) {
  return false;
}
inline bool r2l_attention_fast(const __nv_bfloat16* qkv, int ld, __nv_bfloat16* out, int ldo, int heads, int dh, long long reg_row0,
                               const PosBias& pb, const Window& win, cudaStream_t s) {
  return attention_r2l(qkv, ld, out, ldo, heads, dh, reg_row0, pb, win, s);
}

// res_bias (may be null: patch.bias): what the patch Dense yields on an all-zero (cls) row when that is not its bias -- beta . W +
// bias when a LayerNorm runs before it (SPT, vit_for_small_dataset.py:148-149)
struct EmbedW { Linear patch; const float* pos = nullptr; const float* cls = nullptr; int dim = 0, n_pos = 0; const float* res_bias = nullptr;
               int site = -1; };   // site: the embedding dropout's (vb_handle::number_dropout_sites)
struct CrossW { bool proj = false; Linear project_in, project_out, to_q, to_kv, to_out; Norm norm; int site = -1; };

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
  // Training-mode dropout (vb_set_dropout): the rates, whether a seed is set, and the {seed, draw counter} pair in device memory
  // that the dropout epilogues read.  `training` holds while vb_forward_train issues its launches.
  bool drop_set = false, training = false;
  float drop_rate = 0.f, emb_drop_rate = 0.f;
  DevMem drop_dev;
  static bool dropout_kind(int kind) {
    return kind == VB_KIND_VIT || kind == VB_KIND_DEEPVIT || kind == VB_KIND_CAIT || kind == VB_KIND_CROSSVIT;
  }
  bool dropout_active() const { return training && (drop_rate > 0.f || emb_drop_rate > 0.f); }
  // the epilogue of one site: off unless this is a training forward and the site's rate is > 0
  DropoutEpi dropout(int site, bool emb, int pos) const {
    DropoutEpi d;
    const float rate = emb ? emb_drop_rate : drop_rate;
    if (!training || site < 0 || rate <= 0.f) return d;
    d.pos = pos; d.state = static_cast<const unsigned long long*>(drop_dev.p); d.site = site; d.rate = rate;
    d.scale = static_cast<float>(1.0 / (1.0 - static_cast<double>(rate)));   // tf.nn.dropout: x * (1 / (1 - rate)) kept
    return d;
  }
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> event_pool;
  double prof_ms[PROF_NUM] = {0}, prof_flops[PROF_NUM] = {0}, prof_bytes[PROF_NUM] = {0};
  long long prof_calls[PROF_NUM] = {0};
  // side streams of the per-image T2T soft-split attention (layer_t2t): forked from / joined into the forward's stream with
  // timing-less events, so that the branch is part of a captured graph like everything else
  static constexpr int T2T_MAX_STREAMS = 4;
  cudaStream_t side_streams[T2T_MAX_STREAMS - 1] = {nullptr, nullptr, nullptr};
  cudaEvent_t fork_event = nullptr, join_events[T2T_MAX_STREAMS - 1] = {nullptr, nullptr, nullptr};
  void ensure_side_streams() {
    if (fork_event != nullptr) return;
    VB_CUDA(cudaEventCreateWithFlags(&fork_event, cudaEventDisableTiming));
    for (int i = 0; i < T2T_MAX_STREAMS - 1; ++i) {
      VB_CUDA(cudaStreamCreateWithFlags(&side_streams[i], cudaStreamNonBlocking));
      VB_CUDA(cudaEventCreateWithFlags(&join_events[i], cudaEventDisableTiming));
    }
  }
  void destroy_side_streams() {
    if (fork_event == nullptr) return;
    cudaEventDestroy(fork_event);
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
  // NesT (nest.py:150-216): the patch embedding (`nest_patch`), the levels, the head LayerNorm (`head_norm`) and Dense (`head`)
  vb_nest_config ns{};
  Linear nest_patch;
  std::vector<NestLevelW> nest_levels;
  static std::string nest_pre(int i) { return "nest_layers." + std::to_string(i) + "."; }
  int nest_dim(int i) const { return ns.dim << i; }                  // nest.py:169-172: level i has dim * 2^i channels, heads * 2^i heads
  int nest_last_dim() const { return nest_dim(ns.num_hierarchies - 1); }
  bool nest_aggregates(int i) const { return i != ns.num_hierarchies - 1; }   // is_last (nest.py:188): hierarchies[i] == 0
  // channels of the map the head sees: the last level's output (its Aggregate's when it has one), or the patch embedding's
  int nest_final_dim() const {
    if (ns.levels == 0) return ns.dim;
    return nest_aggregates(ns.levels - 1) ? nest_dim(ns.levels) : nest_dim(ns.levels - 1);
  }
  // RegionViT (regionvit.py:184-263): the local encoder (one 8x8 stride-4 convolution, or three 3x3 with two LayerNorms), the
  // region encoder, the stages, the head LayerNorm (`head_norm`) and Dense (`head`)
  vb_regionvit_config rv{};
  Linear rv_local[3], rv_region;
  Norm rv_local_norm[2];
  std::vector<RegionStageW> rv_stages;
  static std::string rv_pre(int s) { return "region_layers." + std::to_string(s) + "."; }
  int rv_region_patch() const { return rv.local_patch_size * rv.window_size; }   // regionvit.py:204
  static constexpr int kRvHeads = 4, kRvDh = 32, kRvInner = kRvHeads * kRvDh;   // R2LTransformer's defaults (:119, :239)
  struct XBlock { std::vector<LayerW> sm_layers, lg_layers; Norm sm_final, lg_final; std::vector<CrossW> sm_attend_lg, lg_attend_sm; };
  std::vector<XBlock> xblocks;
  // ATS-ViT (ats_vit.py:222-318): ViT's weights and layers; the sampling state of a forward lives in ats_dev (AtsPlan), the
  // Philox key and the 64-bit draw counter in ats_rng
  vb_ats_vit_config ats{};
  DevMem ats_dev, ats_rng;
  // Layer L runs at row pitch P[L]; P[L + 1] = 1 + min(P[L] - 1, K_L).  A layer with P[L] - 1 <= K_L can never sample and launches
  // nothing beyond a ViT layer.  The int state: per slot (one for the embedding, one more per layer that can sample) the live
  // rows of every image (rows, slot-major), C, and the token ids at the slot's pitch; the draws of every layer that can sample;
  // the returned ids [B, P[depth] - 1].
  struct AtsPlan {
    int B = 0;
    std::vector<int> P, slot, slot_P;
    std::vector<bool> can;
    std::vector<size_t> ids, draws;
    size_t rows = 0, C = 0, out = 0, total = 0;
  };
  AtsPlan ats_last;
  AtsPlan ats_plan(int B, int n0) const {
    AtsPlan p;
    p.B = B;
    p.P.push_back(n0); p.slot.push_back(0); p.slot_P.push_back(n0);
    for (int L = 0; L < cfg.depth; ++L) {
      const int P = p.P.back(), K = ats.max_tokens_per_depth[L];
      const bool can = P - 1 > K;
      p.can.push_back(can);
      if (can) p.slot_P.push_back(1 + K);
      p.P.push_back(can ? 1 + K : P);
      p.slot.push_back(static_cast<int>(p.slot_P.size()) - 1);
    }
    const size_t slots = p.slot_P.size();
    size_t off = 0;
    p.rows = off; off += slots * B;
    p.C = off; off += slots;
    for (size_t i = 0; i < slots; ++i) { p.ids.push_back(off); off += static_cast<size_t>(B) * p.slot_P[i]; }
    for (int L = 0; L < cfg.depth; ++L) { p.draws.push_back(off); if (p.can[L]) off += static_cast<size_t>(B) * ats.max_tokens_per_depth[L]; }
    p.out = off; off += static_cast<size_t>(B) * (p.P.back() - 1);
    p.total = off;
    return p;
  }
  unsigned long long* ats_rng_ptr() {
    if (ats_rng.p == nullptr) {
      ats_rng.ensure(2 * sizeof(unsigned long long));
      VB_CUDA(cudaMemset(ats_rng.p, 0, 2 * sizeof(unsigned long long)));
      VB_CUDA(cudaDeviceSynchronize());                // before any forward reads it, on whatever stream that runs
    }
    return static_cast<unsigned long long*>(ats_rng.p);
  }
  // the host side of an ATS forward of a batch of h x w images, before the launches or graph lookup: the state buffer (a new
  // allocation invalidates the captured graphs that point into the old one)
  void ats_prepare(int B, int H, int Wd) {
    VB_CHECK(H % cfg.patch_h == 0 && Wd % cfg.patch_w == 0, "Image dimensions must be divisible by the patch size.");
    const long long np = static_cast<long long>(H / cfg.patch_h) * (Wd / cfg.patch_w);
    VB_CHECK(np + 1 <= ATS_MAX_TOKENS, "ATS-ViT: at most 65,535 patches per image (the sampling noise keys a token by 16 bits)");
    VB_CHECK(np + 1 <= embed.n_pos, "image has more patches than pos_embedding rows");
    ats_last = ats_plan(B, static_cast<int>(np) + 1);
    const void* before = ats_dev.p;
    ats_dev.ensure(ats_last.total * sizeof(int));
    if (before != nullptr && ats_dev.p != before) drop_graphs();
    ats_rng_ptr();
  }
  // MobileViT (mobile_vit.py:209-271): conv1, the seven MV2 blocks (stem 0-3, trunk 4-6), the three MobileViTBlocks, to_logits
  vb_mobilevit_config mv{};
  Linear mv_conv1, mv_logits;
  std::vector<Mv2W> mv_mv2;
  std::vector<MvitBlockW> mv_vit;
  static std::string mv2_pre(int i) { return i < 4 ? "stem." + std::to_string(i) + ".conv." : "trunk." + std::to_string(i - 4) + ".0.conv."; }
  static std::string mvit_pre(int s) { return "trunk." + std::to_string(s) + ".1."; }
  int mvit_cin(int s) const { return mv.channels[4 + 2 * s]; }
  int mvit_ch(int s) const { return mv.channels[5 + 2 * s]; }
  int mvit_mlp(int s) const { return mv.dims[s] * (s == 0 ? 2 : 4); }            // mobile_vit.py:241,246,251
  static constexpr int kMvHeads = 4, kMvDh = 8;                                    // MobileViTBlock's Transformer (:182)
  int mvit_dh() const { return bf16() ? 32 : kMvDh; }                             // bf16: heads widened to the flash kernel's 32
  // ScalableViT (scalable_vit.py:250-319): to_patches (`sv_stem`), the stages, the head LayerNormalization (`head_norm`) and Dense
  vb_scalable_vit_config sv{};
  Linear sv_stem;
  std::vector<SvitStageW> sv_stages;
  static std::string sv_pre(int s) { return "scalable_layers." + std::to_string(s) + "."; }
  int sv_dim(int s) const { return sv.dim[0] << s; }
  // activation head width of an attention whose keys are dk and values dv wide (SvitStageW)
  int sv_head_width(int dk, int dv) const {
    const int m = std::max(dk, dv);
    return !bf16() ? m : m <= 32 ? 32 : m <= 64 ? 64 : round_up(m, 8);
  }
  // PiT (pit.py:158-219): ViT's weights and layers; layer L belongs to stage pit_stage(L) and has that stage's heads
  vb_pit_config pit{};
  int pit_stage(int L) const {
    int s = 0;
    for (int end = pit.depth[0]; L >= end && s + 1 < pit.stages; end += pit.depth[++s]) {}
    return s;
  }
  int layer_heads(int L) const { return cfg.kind == VB_KIND_PIT ? pit.heads[pit_stage(L)] : cfg.heads; }
  // extract_patches(p, stride p / 2, VALID) positions along a side of n pixels (pit.py:16-17,184 for n >= p)
  int pit_side(int n) const { return (n - cfg.patch_h) / (cfg.patch_h / 2) + 1; }
  // MAE / SimMIM (mae.py:49-92, simmim.py:82-129): the encoder ViT's embedding and `layers`; MAE's enc_to_dec (a Dense when
  // dim != decoder_dim), decoder layers and decoder_pos_emb table; both kinds' mask_token and to_pixels.  The mask noise's Philox
  // key, draw counter and the mask kernel's completion counter live in mim_rng; mim_dev holds the permutation [B, n] and the
  // pred / masked_patches outputs [B, num_masked, patch_dim] at stable addresses (a new allocation drops the captured graphs).
  vb_mim_config mim{};
  // MPP (mpp.py:133-218): the encoder ViT with its cls_token, mask_token in pixel space and to_bits (bf16: zero columns up to a
  // multiple of 64, as the wgmma GEMM takes them).  mim_dev also holds the masked ids [B, n + 1], source [B, n] and logits.
  vb_mpp_config mpp{};
  Linear to_bits;
  int to_bits_ld = 0;
  int mpp_classes() const { return 1 << (mpp.output_channel_bits * cfg.channels); }
  std::vector<LayerW> dec_layers;
  Linear enc_to_dec, to_pixels;
  bool enc_to_dec_dense = false;
  const float* mask_token = nullptr;
  const float* dec_pos = nullptr;
  DevMem mim_dev, mim_rng;
  struct MimPlan { int B = 0, n = 0, nm = 0; size_t pred = 0, patches = 0, ids = 0, src = 0; };
  MimPlan mim_last;
  bool is_mim() const { return cfg.kind == VB_KIND_MAE || cfg.kind == VB_KIND_SIMMIM || cfg.kind == VB_KIND_MPP; }
  int mim_dim() const { return cfg.kind == VB_KIND_MAE ? mim.decoder_dim : cfg.dim; }    // width of the rows to_pixels reads
  int patch_dim() const { return cfg.patch_h * cfg.patch_w * cfg.channels; }
  unsigned long long* mim_rng_ptr() {
    if (mim_rng.p == nullptr) {
      mim_rng.ensure(3 * sizeof(unsigned long long));
      VB_CUDA(cudaMemset(mim_rng.p, 0, 3 * sizeof(unsigned long long)));
      VB_CUDA(cudaDeviceSynchronize());                // before any forward reads it, on whatever stream that runs
    }
    return static_cast<unsigned long long*>(mim_rng.p);
  }
  // the host side of a MAE / SimMIM call of a batch of h x w images, before the launches or graph lookup: the shape checks,
  // num_masked = int(masking_ratio * n) in double (mae.py:57, simmim.py:106) and the output buffers
  void mim_prepare(int B, int H, int Wd) {
    VB_CHECK(H % cfg.patch_h == 0 && Wd % cfg.patch_w == 0, "Image dimensions must be divisible by the patch size.");
    const long long n = static_cast<long long>(H / cfg.patch_h) * (Wd / cfg.patch_w);
    VB_CHECK(n + 1 <= embed.n_pos, "MAE / SimMIM: the image has " + std::to_string(n) + " patches but pos_embedding has rows for " +
                                       std::to_string(embed.n_pos - 1));
    VB_CHECK(n <= MIM_MAX_PATCHES, "MAE / SimMIM: the image has " + std::to_string(n) + " patches; the mask kernel takes at most " +
                                       std::to_string(MIM_MAX_PATCHES) + " per image");
    MimPlan p;
    p.B = B; p.n = static_cast<int>(n);
    size_t total = 0;
    if (cfg.kind == VB_KIND_MPP) {
      // mpp.py:80: math.ceil(prob * seq_len) of a double
      const double kd = std::ceil(mpp.mask_prob * static_cast<double>(n));
      VB_CHECK(kd >= 1.0, "MPP: ceil(mask_prob * " + std::to_string(n) + ") is 0: the loss would be a mean over no patches (NaN in the "
                          "reference)");
      VB_CHECK(kd <= static_cast<double>(n), "MPP: ceil(mask_prob * " + std::to_string(n) + ") masks more patches than the image has");
      VB_CHECK(!(mpp.random_patch_prob > 0.0 && mpp.replace_prob == 1.0),
               "MPP: random_patch_prob / (1 - replace_prob) divides by zero (ZeroDivisionError in the reference)");
      p.nm = static_cast<int>(kd);
      p.ids = round_up(B * p.n, 64);                                     // after the top_k permutation [B, n]
      p.src = p.ids + round_up(static_cast<size_t>(B) * (p.n + 1), 64);  // masked ids at pitch n + 1
      p.pred = p.src + round_up(static_cast<size_t>(B) * p.n, 64);         // logits [B, k, K]
      total = p.pred + static_cast<size_t>(B) * p.nm * mpp_classes();
    } else {
      const int nm = static_cast<int>(mim.masking_ratio * static_cast<double>(n));
      VB_CHECK(nm >= 1, "MAE / SimMIM: num_masked = int(masking_ratio * " + std::to_string(n) + ") is 0: the loss would be a mean over no "
                        "patches (NaN in the reference)");
      p.nm = nm;
      const size_t out = static_cast<size_t>(B) * nm * patch_dim();
      p.pred = round_up(B * p.n, 64);
      p.patches = p.pred + out;
      total = p.patches + out;
    }
    mim_last = p;
    const void* before = mim_dev.p;
    mim_dev.ensure(total * sizeof(float));
    if (before != nullptr && mim_dev.p != before) drop_graphs();
    mim_rng_ptr();
  }
  int* mim_idx() const { return static_cast<int*>(mim_dev.p); }
  float* mim_pred() const { return static_cast<float*>(mim_dev.p) + mim_last.pred; }
  float* mim_patches() const { return static_cast<float*>(mim_dev.p) + mim_last.patches; }
  int* mpp_ids() const { return static_cast<int*>(mim_dev.p) + mim_last.ids; }
  int* mpp_src() const { return static_cast<int*>(mim_dev.p) + mim_last.src; }
  // DistillWrapper (distill.py:87-134, vb_create_distill): a ViT / T2TViT student handle that also holds distillation_token and
  // distill_mlp (LayerNorm "distill_mlp.0", Dense "distill_mlp.1").  dw_dev holds one call's float rows at stable addresses:
  // teacher logits, labels, student logits, distill logits [B, K], distill tokens [B, dim], the loss [B], then ce and q [B]
  // (doubles) and the distillation term (a new allocation drops the captured graphs).
  bool distill_wrapper = false;
  Norm dmlp_norm;
  Linear dmlp;
  DevMem dw_dev;
  struct DistillPlan { int B = 0; size_t teacher = 0, labels = 0, student = 0, dlogits = 0, tokens = 0, loss = 0, ce = 0, q = 0, dterm = 0; };
  DistillPlan dw_last;
  void distill_prepare(int B) {
    auto up = [](size_t v) { return (v + 63) / 64 * 64; };
    const size_t rows = up(static_cast<size_t>(B) * cfg.num_classes);
    DistillPlan p;
    p.B = B;
    p.labels = rows;
    p.student = 2 * rows;
    p.dlogits = 3 * rows;
    p.tokens = 4 * rows;
    p.loss = p.tokens + up(static_cast<size_t>(B) * cfg.dim);
    p.ce = p.loss + up(B);                                   // float offsets; ce and q are doubles, 256-byte aligned
    p.q = p.ce + up(2 * static_cast<size_t>(B));
    p.dterm = p.q + up(2 * static_cast<size_t>(B));
    dw_last = p;
    const void* before = dw_dev.p;
    dw_dev.ensure((p.dterm + 64) * sizeof(float));
    if (before != nullptr && dw_dev.p != before) drop_graphs();
  }
  float* dw(size_t off) const { return static_cast<float*>(dw_dev.p) + off; }
  Norm head_norm, sm_head_norm, lg_head_norm;
  Linear head, sm_head, lg_head;
  Norm spt_norm;                     // SPT's LayerNorm over the p^2 * 5 C patch vector (bf16: padded to the GEMM's K, folded into it)

  // cached patch-embedding residual terms, keyed by (embed ptr, batch, rows)
  struct ResKey { const void* e; int B, rows; bool operator<(const ResKey& o) const { return std::tie(e, B, rows) < std::tie(o.e, o.B, o.rows); } };
  std::map<ResKey, std::unique_ptr<DevMem>> embed_res;

  // cached wgmma GEMM plans (TMA descriptors)
  using PlanKey = std::array<uintptr_t, 18>;      // slots 16-17: the dropout epilogue (vb_handle::linear)
  std::map<PlanKey, GemmBf16> plans;

  // Whole-forward CUDA graphs (vb_forward): the launch sequence of one (image pointer, logits pointer, batch, h, w, stream)
  // combination is captured on its SECOND call (the first runs eagerly and does every lazy host-side step: arena growth,
  // kernel attributes, descriptor / residual caches) and replayed from the third on.  Workspace pointers are stable (the
  // arena is reset, never freed, per forward), so a replay touches exactly the memory the eager run would.  Programmatic
  // dependent launches are captured as programmatic edges.  VB_NO_GRAPH=1 disables it; profiling and the legacy default
  // stream (which cannot be captured) always run eagerly.
  struct GraphKey {
    const void* img; void* out; int B, H, W; cudaStream_t s;
    int flags = 0;                                       // vb_forward_mim: which optional outputs the launches write
    // vb_forward_distill_loss: the labels and teacher-logit rows the loss reads, and the bit patterns of T and alpha
    const void* labels = nullptr; const void* teacher = nullptr;
    uint64_t t_bits = 0, alpha_bits = 0;
    bool operator<(const GraphKey& o) const {
      return std::tie(img, out, B, H, W, s, flags, labels, teacher, t_bits, alpha_bits) <
             std::tie(o.img, o.out, o.B, o.H, o.W, o.s, o.flags, o.labels, o.teacher, o.t_bits, o.alpha_bits);
    }
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
    if (kind == VB_KIND_VIT || kind == VB_KIND_DEEPVIT || kind == VB_KIND_ATS_VIT || kind == VB_KIND_SMALL_DATASET_VIT)
      expect_dense(pre + "to_qkv", dim, 3 * inner, false);
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
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_PARALLEL_VIT || c.kind == VB_KIND_ATS_VIT ||
        c.kind == VB_KIND_PIT) {
      const int np = c.kind == VB_KIND_PIT ? pit_side(c.image_h) * pit_side(c.image_w) : (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      expect("pos_embedding", {1, np + 1, c.dim});
      expect("cls_token", {1, 1, c.dim});
      expect_dense("patch", c.patch_h * c.patch_w * C, c.dim);
      for (int L = 0; L < c.depth; ++L) {
        if (c.kind == VB_KIND_PARALLEL_VIT) {   // branch i = (attention fn i, feed-forward fn i) of layer L (parallel_vit.py:109-112)
          for (int i = 0; i < c.parallel_branches; ++i)
            expect_layer("layers." + std::to_string(L) + ".branch" + std::to_string(i) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
        } else {                                // PiT: ViT's layer with its stage's heads, the to_out rule per stage (pit.py:59)
          expect_layer("layers." + std::to_string(L) + ".", c.dim, layer_heads(L), c.dim_head, c.mlp_dim,
                       c.kind == VB_KIND_PIT ? VB_KIND_VIT : c.kind);
        }
      }
      expect_ln("head_norm", c.dim);
      expect_dense("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_MAE || c.kind == VB_KIND_SIMMIM) {   // the encoder ViT without cls_token / mlp_head (mae.py:33-47)
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), pd = patch_dim();
      expect("pos_embedding", {1, np + 1, c.dim});
      expect_dense("patch", pd, c.dim);
      for (int L = 0; L < c.depth; ++L) expect_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
      const int Dd = mim_dim();
      expect("mask_token", {Dd});
      if (c.kind == VB_KIND_MAE) {
        if (c.dim != Dd) expect_dense("enc_to_dec", c.dim, Dd);                        // mae.py:42
        for (int L = 0; L < mim.decoder_depth; ++L)                                    // vit.Transformer (mae.py:44)
          expect_layer("decoder.layers." + std::to_string(L) + ".", Dd, mim.decoder_heads, mim.decoder_dim_head, 4 * Dd, VB_KIND_VIT);
        expect("decoder_pos_emb.embeddings", {np + 1, Dd});                            // Embedding(num_patches, decoder_dim) :45
      }
      expect_dense("to_pixels", Dd, pd);                                               // mae.py:46, simmim.py:86
    } else if (c.kind == VB_KIND_MPP) {                                 // the encoder ViT without mlp_head (mpp.py:149-166, 199-213)
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), pd = patch_dim();
      expect("pos_embedding", {1, np + 1, c.dim});
      expect("cls_token", {1, 1, c.dim});
      expect_dense("patch", pd, c.dim);
      for (int L = 0; L < c.depth; ++L) expect_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT);
      expect("mask_token", {pd});                                        // tf.random.normal([1, 1, channels * patch_size ** 2]) :166
      expect_dense("to_bits", c.dim, mpp_classes());                     // Dense(2 ** (output_channel_bits * channels)) :155
    } else if (c.kind == VB_KIND_SMALL_DATASET_VIT) {                   // vit_for_small_dataset.py:142-195
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), K = c.patch_h * c.patch_w * 5 * C;
      expect("pos_embedding", {1, np + 1, c.dim});
      expect("cls_token", {1, 1, c.dim});
      expect_ln("patch_norm", K);                                        // to_patch_tokens.layers[1]
      expect_dense("patch", K, c.dim);                                   // to_patch_tokens.layers[2]
      for (int L = 0; L < c.depth; ++L) {
        const std::string pre = "layers." + std::to_string(L) + ".";
        expect_layer(pre, c.dim, c.heads, c.dim_head, c.mlp_dim, c.kind);   // to_out always present (no project_out skip, :99-102)
        expect(pre + "temperature", {});                                 // LSA's scalar tf.Variable (:94)
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
    } else if (c.kind == VB_KIND_NEST) {
      auto expect_ln4 = [&](const std::string& n, int d) { expect(n + ".g", {1, 1, 1, d}); expect(n + ".b", {1, 1, 1, d}); };   // :33-34
      const int dh = ns.dim / ns.heads;
      expect("patch_embedding.1.kernel", {1, 1, ns.patch_size * ns.patch_size * c.channels, ns.dim});   // :178-181
      expect("patch_embedding.1.bias", {ns.dim});
      for (int i = 0; i < ns.levels; ++i) {
        const std::string p = nest_pre(i);
        const int d = nest_dim(i), inner = dh * (ns.heads << i), hidden = d * ns.mlp_mult;
        expect(p + "0.pos_emb", {ns.seq_len});                           // Transformer :129
        for (int L = 0; L < ns.block_repeats[i]; ++L) {
          const std::string b = p + "0.layers." + std::to_string(L) + ".";
          expect_ln4(b + "0.norm", d);                                   // PreNorm(Attention) :133, :77-91
          expect(b + "0.fn.to_qkv.kernel", {1, 1, d, 3 * inner});
          expect(b + "0.fn.to_out.0.kernel", {1, 1, inner, d});
          expect(b + "0.fn.to_out.0.bias", {d});
          expect_ln4(b + "1.norm", d);                                   // PreNorm(MLP) :134, :61-72
          expect(b + "1.fn.net.0.kernel", {1, 1, d, hidden});
          expect(b + "1.fn.net.0.bias", {hidden});
          expect(b + "1.fn.net.3.kernel", {1, 1, hidden, d});
          expect(b + "1.fn.net.3.bias", {d});
        }
        if (nest_aggregates(i)) {                                        // Aggregate :111-119
          const int dn = nest_dim(i + 1);
          expect(p + "1.ag_layers.0.kernel", {3, 3, d, dn});
          expect(p + "1.ag_layers.0.bias", {dn});
          expect_ln4(p + "1.ag_layers.1", dn);
        }
      }
      expect_ln4("mlp_head.0", nest_last_dim());                        // :196-200
      expect_dense("mlp_head.2", nest_last_dim(), c.num_classes);
    } else if (c.kind == VB_KIND_REGIONVIT) {
      auto expect_ln = [&](const std::string& n, int d) { expect(n + ".gamma", {d}); expect(n + ".beta", {d}); };
      auto expect_conv = [&](const std::string& n, int k, int cin, int cout) { expect(n + ".kernel", {k, k, cin, cout}); expect(n + ".bias", {cout}); };
      const int d0 = rv.dims[0], p = rv_region_patch(), t = (2 * rv.window_size - 1) * (2 * rv.window_size - 1);
      if (rv.tokenize_local_3_conv) {                                  // regionvit.py:210-219
        expect_conv("local_encoder.0", 3, c.channels, d0);
        expect_ln("local_encoder.1", d0);
        expect_conv("local_encoder.3", 3, d0, d0);
        expect_ln("local_encoder.4", d0);
        expect_conv("local_encoder.6", 3, d0, d0);
      } else {
        expect_conv("local_encoder", 8, c.channels, d0);                // :221
      }
      expect_conv("region_encoder.1", 1, c.channels * p * p, d0);       // :223-226
      for (int s = 0; s < VB_REGIONVIT_STAGES; ++s) {
        const std::string pre = rv_pre(s);
        const int d = rv.dims[s], hidden = d * rv.mlp_mult;
        if (s > 0) expect_conv(pre + "0.conv", 3, rv.dims[s - 1], d);   // Downsample :45-52
        if (s > 0 && rv.use_peg) expect_conv(pre + "1.proj", 3, 1, d);   // PEG :54-61 (groups = dim)
        expect(pre + "2.local_rel_pos_bias.embeddings", {t, kRvHeads});  // :126
        for (int L = 0; L < rv.depth[s]; ++L) {
          const std::string b = pre + "2.layers." + std::to_string(L) + ".";
          expect_ln(b + "0.norm", d);                                    // Attention :79-91
          expect_dense(b + "0.to_qkv", d, 3 * kRvInner, false);
          expect_dense(b + "0.to_out", kRvInner, d);
          expect_ln(b + "1.net.0", d);                                   // MLP :64-74
          expect_dense(b + "1.net.1", d, hidden);
          expect_dense(b + "1.net.4", hidden, d);
        }
      }
      expect_ln("to_logits.1", rv.dims[VB_REGIONVIT_STAGES - 1]);       // :243-247
      expect_dense("to_logits.2", rv.dims[VB_REGIONVIT_STAGES - 1], c.num_classes);
    } else if (c.kind == VB_KIND_MOBILEVIT) {
      auto expect_bn = [&](const std::string& n, int d) {
        for (const char* leaf : {"gamma", "beta", "moving_mean", "moving_variance"}) expect(n + "." + leaf, {d});
      };
      auto expect_cbn = [&](const std::string& n, int k, int cin, int cout) {   // Conv_NxN_BN (:37-49)
        expect(n + ".layers.0.kernel", {k, k, cin, cout});
        expect_bn(n + ".layers.1", cout);
      };
      expect_cbn("conv1", 3, c.channels, mv.channels[0]);
      for (int i = 0; i < VB_MOBILEVIT_MV2; ++i) {                       // MV2Block (:139-164)
        const std::string p = mv2_pre(i);
        const int hid = mv.mv2_hidden[i];
        if (mv.mv2_expand[i]) {
          expect(p + "0.kernel", {1, 1, mv.mv2_in[i], hid}); expect_bn(p + "1", hid);
          expect(p + "3.kernel", {3, 3, 1, hid}); expect_bn(p + "4", hid);
          expect(p + "6.kernel", {1, 1, hid, mv.mv2_out[i]}); expect_bn(p + "7", mv.mv2_out[i]);
        } else {
          expect(p + "0.kernel", {3, 3, 1, hid}); expect_bn(p + "1", hid);
          expect(p + "3.kernel", {1, 1, hid, mv.mv2_out[i]}); expect_bn(p + "4", mv.mv2_out[i]);
        }
      }
      for (int s = 0; s < 3; ++s) {                                      // MobileViTBlock (:173-185)
        const std::string p = mvit_pre(s);
        const int d = mv.dims[s], ch = mvit_ch(s), cin = mvit_cin(s), k = mv.kernel_size, I = kMvHeads * kMvDh;
        expect_cbn(p + "conv1", k, cin, ch);
        expect_cbn(p + "conv2", 1, ch, d);
        for (int L = 0; L < mv.depths[s]; ++L) {                         // Transformer (:110-127)
          const std::string b = p + "transformer.layers." + std::to_string(L) + ".";
          expect_ln(b + "0.norm", d);
          expect_dense(b + "0.fn.to_qkv", d, 3 * I, false);
          expect_dense(b + "0.fn.to_out.0", I, d);
          expect_ln(b + "1.norm", d);
          expect_dense(b + "1.fn.net.0", d, mvit_mlp(s));
          expect_dense(b + "1.fn.net.3", mvit_mlp(s), d);
        }
        expect_cbn(p + "conv3", 1, d, ch);
        expect_cbn(p + "conv4", k, ch + cin, ch);
      }
      expect_cbn("to_logits.0", 1, mv.channels[9], mv.last_dim);         // :254-258
      expect("to_logits.2.kernel", {mv.last_dim, c.num_classes});
    } else if (c.kind == VB_KIND_SCALABLE_VIT) {
      auto expect_ln4 = [&](const std::string& n, int d) { expect(n + ".g", {1, 1, 1, d}); expect(n + ".b", {1, 1, 1, d}); };   // :46-52
      auto expect_conv = [&](const std::string& n, int k, int cin, int cout, bool bias) {
        expect(n + ".kernel", {k, k, cin, cout});
        if (bias) expect(n + ".bias", {cout});
      };
      expect_conv("to_patches", 7, c.channels, sv.dim[0], true);        // :261
      for (int st = 0; st < sv.num_stages; ++st) {
        const int d = sv_dim(st), h = sv.heads[st], r = sv.reduction_factor[st], f = sv.ff_expansion_factor;
        const int sk = sv.ssa_dim_key[st], svv = sv.ssa_dim_value[st], ik = sv.iwsa_dim_key[st], iv = sv.iwsa_dim_value[st];
        for (int L = 0; L < sv.depth[st]; ++L) {
          const std::string b = sv_pre(st) + "0.layers." + std::to_string(L) + ".";
          auto expect_mlp = [&](const std::string& m) {                  // PreNorm(MLP) :61-69, :89-102
            expect_ln4(m + "norm", d);
            expect_conv(m + "fn.net.0", 1, d, f * d, true);
            expect_conv(m + "fn.net.3", 1, f * d, d, true);
          };
          expect_ln4(b + "0.norm", d);                                   // ScalableSelfAttention :104-121
          expect_conv(b + "0.fn.to_q", 1, d, h * sk, false);
          expect_conv(b + "0.fn.to_k", r, d, h * sk, false);
          expect_conv(b + "0.fn.to_v", r, d, h * svv, false);
          expect_conv(b + "0.fn.to_out.0", 1, h * svv, d, true);
          expect_mlp(b + "1.");
          if (L == 0) expect_conv(b + "2.proj", 3, 1, d, true);          // PEG :80-87 (groups = dim)
          expect_mlp(b + "3.");
          expect_ln4(b + "4.norm", d);                                   // InteractiveWindowedSelfAttention :145-163
          expect_conv(b + "4.fn.local_interactive_module", 3, h * iv, h * iv, true);
          expect_conv(b + "4.fn.to_q", 1, d, h * ik, false);
          expect_conv(b + "4.fn.to_k", 1, d, h * ik, false);
          expect_conv(b + "4.fn.to_v", 1, d, h * iv, false);
          expect_conv(b + "4.fn.to_out.0", 1, h * iv, d, true);
        }
        expect_ln4(sv_pre(st) + "0.norm", d);                            // :233
        if (st < sv.num_stages - 1) expect_conv(sv_pre(st) + "1.conv", 3, d, 2 * d, true);   // Downsample :71-78
      }
      const int dl = sv_dim(sv.num_stages - 1);
      expect_ln("mlp_head.1", dl);                                       // :302-306
      expect_dense("mlp_head.2", dl, c.num_classes);
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
    if (distill_wrapper) {                                    // distill.py:101-106, after the student's own weights
      expect("distillation_token", {1, 1, c.dim});
      expect_ln("distill_mlp.0", c.dim);
      expect_dense("distill_mlp.1", c.dim, c.num_classes);
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
    return pack_linear(W(n + ".kernel"), bias ? W(n + ".bias") : nullptr, K, N, std::max(round_up(K, 8), ldw_min), fold);
  }
  // The Dense W [K, N] (device, Keras layout) + bias (may be null); the bf16 engine packs W K-major at pitch ldw and folds the
  // LayerNorm `fold` into it when given
  Linear pack_linear(const float* Wk, const float* bias, int K, int N, int ldw, const Norm* fold) {
    Linear L;
    L.W = Wk;
    L.bias = bias;
    L.K = K; L.N = N; L.ldw = ldw;
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
    if (bf16() && dh < 64 && dh % 8 == 0 && to_out_present && dim % 8 == 0 &&
        (kind == VB_KIND_VIT || kind == VB_KIND_CROSSVIT || kind == VB_KIND_ATS_VIT || kind == VB_KIND_SMALL_DATASET_VIT)) {
      const int dhp = 64;
      auto padded = [&](const std::string& n, int other, int groups, int pad_rows) {
        owned.emplace_back(new DevMem());
        owned.back()->ensure(static_cast<size_t>(other) * groups * heads * dhp * sizeof(float));
        float* wp = static_cast<float*>(owned.back()->p);
        pad_heads_f32(W(n), wp, other, groups, heads, dh, dhp, pad_rows, 0);
        woverride[n] = wp;
      };
      if (kind == VB_KIND_VIT || kind == VB_KIND_ATS_VIT || kind == VB_KIND_SMALL_DATASET_VIT) padded(pre + "to_qkv.kernel", dim, 3, 0);
      else { padded(pre + "to_q.kernel", dim, 1, 0); padded(pre + "to_kv.kernel", dim, 2, 0); }
      padded(pre + "to_out.kernel", dim, 1, 1);
      dh = dhp;
    }
    const int inner = heads * dh;
    l.heads = heads; l.dim_head = dh;
    l.attn_norm = make_norm(pre + "attn_norm", dim);
    l.ff_norm = make_norm(pre + "ff_norm", dim);
    // LayerNorm folding needs every GEMM of the layer on the wgmma path (all widths multiples of 64)
    l.folded = bf16() && fold_ok && dim % 64 == 0 && inner % 64 == 0 && mlp % 64 == 0;
    const Norm* fa = l.folded ? &l.attn_norm : nullptr;
    const Norm* ff = l.folded ? &l.ff_norm : nullptr;
    if (kind == VB_KIND_VIT || kind == VB_KIND_DEEPVIT || kind == VB_KIND_ATS_VIT || kind == VB_KIND_SMALL_DATASET_VIT) {
      l.fused_qkv = true;
      l.to_qkv = make_linear(pre + "to_qkv", dim, 3 * inner, false, fa);
    }
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
    l.folded = bf16() && dim % 64 == 0 && mlp % 64 == 0;   // every GEMM on the wgmma path
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

  // The site of every Dropout layer the reference's call reaches, in its call order from 0 (include/vitb200.h, vb_set_dropout):
  // the embedding's; per layer to_out's (absent without an out-projection, vit.py:53,61-67), the GELU's and fc2's (vit.py:38-44); CaiT's
  // patch stack, then its class stack; CrossViT's small then large embedder, then per block the small tower's layers, the large tower's
  // and the cross-attention rounds, sm_attend_lg before lg_attend_sm (cross_vit.py:187-193,147-160).
  void number_dropout_sites() {
    int s = 0;
    auto layer = [&](LayerW& l) { l.site_out = l.project_out ? s++ : -1; l.site_ff = s; s += 2; };
    if (cfg.kind == VB_KIND_CROSSVIT) {
      sm_embed.site = s++;
      lg_embed.site = s++;
      for (auto& xb : xblocks) {
        for (auto& l : xb.sm_layers) layer(l);
        for (auto& l : xb.lg_layers) layer(l);
        for (size_t R = 0; R < xb.sm_attend_lg.size(); ++R) { xb.sm_attend_lg[R].site = s++; xb.lg_attend_sm[R].site = s++; }
      }
    } else {
      embed.site = s++;
      for (auto& l : layers) layer(l);
      for (auto& l : cls_layers) layer(l);
    }
  }

  void finalize() {
    for (auto& w : weights) VB_CHECK(w.set, "vb_finalize: weight '" + w.name + "' was never set");
    VB_CUDA(cudaSetDevice(device));
    owned.clear(); layers.clear(); cls_layers.clear(); t2t_layers.clear(); xblocks.clear(); plans.clear(); embed_res.clear(); cct_convs.clear();
    lv_stem.clear(); lv_blocks.clear(); cvt_stages.clear(); twins_stages.clear(); cf_stages.clear(); nest_levels.clear(); rv_stages.clear();
    mv_mv2.clear(); mv_vit.clear(); sv_stages.clear(); dec_layers.clear();
    woverride.clear();
    drop_graphs();
    const vb_config& c = cfg;
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_PARALLEL_VIT || c.kind == VB_KIND_ATS_VIT ||
        c.kind == VB_KIND_PIT) {
      const int np = c.kind == VB_KIND_PIT ? pit_side(c.image_h) * pit_side(c.image_w) : (c.image_h / c.patch_h) * (c.image_w / c.patch_w);
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np + 1);
      for (int L = 0; L < c.depth; ++L) {
        if (c.kind == VB_KIND_PARALLEL_VIT) {   // `layers` holds depth x parallel_branches entries, branches of a layer adjacent
          for (int i = 0; i < c.parallel_branches; ++i)
            layers.push_back(make_layer("layers." + std::to_string(L) + ".branch" + std::to_string(i) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
        } else {
          layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, layer_heads(L), c.dim_head, c.mlp_dim,
                                      c.kind == VB_KIND_PIT ? VB_KIND_VIT : c.kind));
        }
      }
      head_norm = make_norm("head_norm", c.dim);
      head = make_linear_f32("head", c.dim, c.num_classes);
    } else if (c.kind == VB_KIND_MAE || c.kind == VB_KIND_SIMMIM) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), Dd = mim_dim();
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np + 1, false);
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
      mask_token = W("mask_token");
      if (c.kind == VB_KIND_MAE) {
        enc_to_dec_dense = has("enc_to_dec.kernel");
        if (enc_to_dec_dense) enc_to_dec = make_linear("enc_to_dec", c.dim, Dd);
        for (int L = 0; L < mim.decoder_depth; ++L)
          dec_layers.push_back(make_layer("decoder.layers." + std::to_string(L) + ".", Dd, mim.decoder_heads, mim.decoder_dim_head, 4 * Dd, VB_KIND_VIT));
        dec_pos = W("decoder_pos_emb.embeddings");
      }
      to_pixels = make_linear("to_pixels", Dd, patch_dim());
    } else if (c.kind == VB_KIND_MPP) {
      const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), K = mpp_classes();
      embed = make_embed("", c.patch_h, c.patch_w, c.dim, np + 1);
      for (int L = 0; L < c.depth; ++L) layers.push_back(make_layer("layers." + std::to_string(L) + ".", c.dim, c.heads, c.dim_head, c.mlp_dim, VB_KIND_VIT));
      mask_token = W("mask_token");
      to_bits_ld = bf16() ? round_up(K, 64) : K;
      to_bits = to_bits_ld == K ? make_linear("to_bits", c.dim, K) : padded_dense("to_bits.padded", "to_bits", c.dim, K, c.dim, to_bits_ld);
    } else if (c.kind == VB_KIND_SMALL_DATASET_VIT) {
      finalize_small_dataset_vit();
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
          if (bf16()) t2t_layers.push_back(make_t2t_layer(pre, st[i].dim));
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
    } else if (c.kind == VB_KIND_NEST) {
      finalize_nest();
    } else if (c.kind == VB_KIND_REGIONVIT) {
      finalize_regionvit();
    } else if (c.kind == VB_KIND_MOBILEVIT) {
      finalize_mobilevit();
    } else if (c.kind == VB_KIND_SCALABLE_VIT) {
      finalize_scalable_vit();
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
    if (dropout_kind(c.kind)) number_dropout_sites();
    if (distill_wrapper) {
      dmlp_norm = make_norm("distill_mlp.0", c.dim);
      dmlp = make_linear_f32("distill_mlp.1", c.dim, c.num_classes);
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
  // The Dense (or Conv2D as a Dense) `name`: its kernel [K, N] as the top-left block of a zero [Kp, Np], its bias (when it has one)
  // padded to Np, packed under `key`.  With `fold`: that LayerNorm (true width K, epsilon eps) folded in by the bf16 engine.
  Linear padded_dense(const std::string& key, const std::string& name, int K, int N, int Kp, int Np, const Norm* fold = nullptr,
                      float eps = 1e-5f) {
    const std::vector<double> bias = has(name + ".bias") ? pad_n(host_weight(name + ".bias"), Np) : std::vector<double>();
    Linear L = linear_from_host(key, pad_kn(host_weight(name + ".kernel"), K, N, Kp, Np), bias, Kp, Np, bf16() ? fold : nullptr);
    if (fold != nullptr) { L.ln_d = K; L.ln_eps = eps; }
    return L;
  }
  // A LayerNorm's gamma / beta [d] (leaves `g` / `b`: the models' own LayerNorm, or Keras' gamma / beta) zero-padded to [dp]
  Norm padded_norm(const std::string& n, int d, int dp, const char* g = ".g", const char* b = ".b") {
    return Norm{upload_owned(pad_n(host_weight(n + g), dp)), upload_owned(pad_n(host_weight(n + b), dp)), d};
  }
  // 'b (h p1) (w p2) c -> b h w (c p1 p2)': the reference's kernel row c p^2 + p1 p + p2 [.., d] is unfold_same's row (p1 p + p2) cin + c
  static std::vector<double> patch_rows_channel_last(const std::vector<double>& wr, int cin, int p, int d) {
    std::vector<double> wp(wr.size());
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < p * p; ++t)
        std::copy(wr.begin() + static_cast<size_t>(c * p * p + t) * d, wr.begin() + static_cast<size_t>(c * p * p + t + 1) * d,
                  wp.begin() + static_cast<size_t>(t * cin + c) * d);
    return wp;
  }
  // PEG: x + dw(x) + b is one depthwise k x k convolution whose centre tap ((k-1)/2, (k-1)/2) has 1 added (TF SAME at stride 1 pads
  // (k-1)/2 on the top / left, so that tap reads the pixel itself).  taps [k*k][d] -> [k*k][dp]
  const float* peg_taps(const std::vector<double>& taps, int k, int d, int dp) {
    std::vector<double> pw(static_cast<size_t>(k) * k * dp, 0.0);
    const int centre = ((k - 1) / 2) * k + (k - 1) / 2;
    for (int t = 0; t < k * k; ++t)
      for (int c = 0; c < d; ++c) pw[static_cast<size_t>(t) * dp + c] = taps[static_cast<size_t>(t) * d + c] + (t == centre ? 1.0 : 0.0);
    return upload_owned(pw);
  }
  // ---- CvT weight packing: channel widths zero-padded (bf16), BatchNormalizations folded into the depthwise taps and a shift
  void finalize_cvt() {
    for (int st = 0; st < VB_CVT_STAGES; ++st) {
      CvtStageW S;
      const std::string p = cvt_pre(st);
      const int d = cv.emb_dim[st], dp = channel_width(d), ke = cv.emb_kernel[st], K = ke * ke * cvt_cin(st);
      S.dim = d; S.dp = dp; S.k = ke; S.stride = cv.emb_stride[st];
      S.conv = padded_dense("cvt." + p + "0", p + "0", K, d, K, dp);
      S.norm = padded_norm(p + "1", d, dp);
      const int inner = 64 * cv.heads[st], k = cv.proj_kernel[st];
      for (int L = 0; L < cv.depth[st]; ++L) {
        const std::string b = p + "2.layers." + std::to_string(L) + ".", key = "cvt." + b;
        CvtBlockW w;
        w.dim = d; w.dp = dp; w.heads = cv.heads[st]; w.k = k; w.kv_stride = cv.kv_proj_stride[st];
        w.attn_norm = padded_norm(b + "0.norm", d, dp);
        for (int kv = 0; kv < 2; ++kv) {
          const std::string n = b + (kv ? "0.fn.to_kv.net." : "0.fn.to_q.net.");
          std::vector<double> taps, shift;
          cvt_fold_dw(host_weight(n + "0.kernel"), host_weight(n + "1.gamma"), host_weight(n + "1.beta"), host_weight(n + "1.moving_mean"),
                      host_weight(n + "1.moving_variance"), k, d, dp, taps, shift);
          const int N = (kv ? 2 : 1) * inner;
          Linear pw = padded_dense(key + (kv ? "pw_kv" : "pw_q"), n + "2", d, N, dp, N);
          if (kv) { w.wkv = upload_owned(taps); w.bkv = upload_owned(shift); w.pw_kv = pw; }
          else { w.wq = upload_owned(taps); w.bq = upload_owned(shift); w.pw_q = pw; }
        }
        w.to_out = padded_dense(key + "to_out", b + "0.fn.to_out.0", inner, d, inner, dp);
        w.ff = prenorm_mlp("cvt.", b + "1.norm", b + "1.fn.net.0", b + "1.fn.net.3", d, dp, cv.mlp_mult[st]);
        S.blocks.push_back(std::move(w));
      }
      cvt_stages.push_back(std::move(S));
    }
    head = make_linear_f32("cvt_layers.3.1", cv.emb_dim[VB_CVT_STAGES - 1], cfg.num_classes);
  }
  // A PreNorm MLP of width mult * d: the LayerNorm `norm` (leaves g / b, epsilon eps), the Dense layers n0 (d -> mult d) and n3
  // (mult d -> d), widths padded, the LayerNorm folded into fc1 in the bf16 engine.  key: the packed copies' own names.
  MlpW prenorm_mlp(const std::string& key, const std::string& norm, const std::string& n0, const std::string& n3, int d, int dp,
                   int mult = 4, float eps = 1e-5f, const char* g = ".g", const char* b = ".b") {
    MlpW w;
    const int hidden = mult * d, hp = channel_width(hidden);
    w.norm = padded_norm(norm, d, dp, g, b);
    w.fc1 = padded_dense(key + n0, n0, d, hidden, dp, hp, &w.norm, eps);
    w.fc2 = padded_dense(key + n3, n3, hidden, d, hp, dp);
    return w;
  }
  // ---- Twins-SVT weight packing: channel widths zero-padded (bf16), the patch kernel's rows permuted, the PEG residual folded
  MlpW twins_mlp(const std::string& m, int d, int dp) {
    return prenorm_mlp("twins.", m + ".fn.norm", m + ".fn.fn.net.0", m + ".fn.fn.net.3", d, dp);
  }
  TwinsLayerW twins_layer_weights(const std::string& b, int st, int d, int dp) {
    TwinsLayerW w;
    const int I = kTwinsInner, kg = tw.global_k[st];
    auto to_out = [&](const std::string& n) { return padded_dense("twins." + n, n, I, d, I, dp); };
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
      w.qkv = linear_from_host("twins." + b + "0.qkv", pad_kn(qkv, d, 3 * I, dp, 3 * I), {}, dp, 3 * I, bf16() ? &w.local_norm : nullptr);
      w.qkv.ln_d = d;
      w.qkv.ln_eps = 1e-5f;                                          // twins_svt.py:46
      w.local_out = to_out(b + "0.fn.fn.to_out.0");
      w.ff1 = twins_mlp(b + "1", d, dp);
    }
    w.global_norm = padded_norm(b + "2.fn.norm", d, dp);
    w.to_q = padded_dense("twins." + b + "2.to_q", b + "2.fn.fn.to_q", d, I, dp, I, &w.global_norm);
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
      const auto wp = patch_rows_channel_last(host_weight(p + "0.proj.kernel"), cin, ps, d);   // twins_svt.py:103
      S.proj = linear_from_host("twins." + p + "0.proj", pad_kn(wp, K, d, K, dp), pad_n(host_weight(p + "0.proj.bias"), dp), K, dp);
      S.peg_w = peg_taps(host_weight(p + "2.proj.fn.kernel"), k, d, dp);                      // PEG (:108-115)
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
    w.to_out = padded_dense("cf." + a + "to_out", a + "to_out", I, d, I, dp);
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
  // ---- NesT weight packing: channel widths zero-padded (bf16), the to_out rows padded to the q|k|v pitch the attention leaves
  void finalize_nest() {
    const int K0 = ns.patch_size * ns.patch_size * cfg.channels, dp0 = channel_width(ns.dim), dh = ns.dim / ns.heads;
    // 'b (h p1) (w p2) c -> b h w (p1 p2 c)' (nest.py:179) is unfold_same's (p1, p2, c) order: the kernel's rows as they are
    nest_patch = padded_dense("nest.patch", "patch_embedding.1", K0, ns.dim, K0, dp0);
    for (int i = 0; i < ns.levels; ++i) {
      NestLevelW V;
      const std::string p = nest_pre(i);
      const int d = nest_dim(i), dp = channel_width(d);
      V.dim = d; V.dp = dp; V.heads = ns.heads << i; V.dh = dh; V.inner = dh * V.heads; V.bs = 1 << (ns.levels - 1 - i);
      V.pos = W(p + "0.pos_emb");
      const int I = V.inner, N = bf16() ? round_up(3 * I, 64) : 3 * I, Ko = bf16() ? round_up(I, 64) : I;
      for (int L = 0; L < ns.block_repeats[i]; ++L) {
        const std::string b = p + "0.layers." + std::to_string(L) + ".", key = "nest." + b;
        NestBlockW w;
        w.attn_norm = padded_norm(b + "0.norm", d, dp);
        w.qkv = padded_dense(key + "qkv", b + "0.fn.to_qkv", d, 3 * I, dp, N, &w.attn_norm);   // nest.py:29: eps 1e-5
        // to_out reads the attention output in place of q: K rows [I, Ko) meet k / v columns and are zero
        w.to_out = padded_dense(key + "to_out", b + "0.fn.to_out.0", I, d, Ko, dp);
        w.ff = prenorm_mlp("nest.", b + "1.norm", b + "1.fn.net.0", b + "1.fn.net.3", d, dp, ns.mlp_mult);
        V.blocks.push_back(std::move(w));
      }
      V.aggregate = nest_aggregates(i);
      if (V.aggregate) {
        const int dn = nest_dim(i + 1), dpn = channel_width(dn);
        V.dim_out = dn; V.dp_out = dpn;
        // [3, 3, d, dn] is the Dense [9 d, dn] over unfold_same's (row, column, channel) vectors of the true d channels
        V.agg = padded_dense("nest." + p + "1.conv", p + "1.ag_layers.0", 9 * d, dn, 9 * d, dpn);
        V.agg_norm = padded_norm(p + "1.ag_layers.1", dn, dpn);
      }
      nest_levels.push_back(std::move(V));
    }
    head_norm = padded_norm("mlp_head.0", nest_last_dim(), channel_width(nest_last_dim()));
    head = make_linear_f32("mlp_head.2", nest_last_dim(), cfg.num_classes);
  }
  // ---- RegionViT weight packing: channel widths zero-padded (bf16), the region kernel's rows permuted, the PEG residual folded,
  // every Attention / MLP LayerNorm (Keras, eps 1e-3) folded into q|k|v / fc1 in the bf16 engine, the window tables transposed
  void finalize_regionvit() {
    const int C = cfg.channels, d0 = rv.dims[0], dp0 = channel_width(d0), p = rv_region_patch(), ws = rv.window_size;
    if (rv.tokenize_local_3_conv) {
      for (int i = 0; i < 3; ++i) {
        const std::string n = "local_encoder." + std::to_string(3 * i);
        const int K = 9 * (i == 0 ? C : d0);
        rv_local[i] = padded_dense("rv." + n, n, K, d0, K, dp0);
      }
      for (int i = 0; i < 2; ++i) rv_local_norm[i] = padded_norm("local_encoder." + std::to_string(3 * i + 1), d0, dp0, ".gamma", ".beta");
    } else {
      rv_local[0] = padded_dense("rv.local_encoder", "local_encoder", 64 * C, d0, 64 * C, dp0);
    }
    const int K = C * p * p;                                             // regionvit.py:224
    rv_region = linear_from_host("rv.region_encoder", pad_kn(patch_rows_channel_last(host_weight("region_encoder.1.kernel"), C, p, d0), K, d0, K, dp0),
                                 pad_n(host_weight("region_encoder.1.bias"), dp0), K, dp0);
    for (int s = 0; s < VB_REGIONVIT_STAGES; ++s) {
      RegionStageW S;
      const std::string pre = rv_pre(s);
      const int d = rv.dims[s], dp = channel_width(d);
      S.dim = d; S.dp = dp; S.down = s > 0; S.peg = s > 0 && rv.use_peg;
      if (S.down) S.down_conv = padded_dense("rv." + pre + "0.conv", pre + "0.conv", 9 * rv.dims[s - 1], d, 9 * rv.dims[s - 1], dp);
      if (S.peg) {                                                      // :54-61, the residual folded
        S.peg_w = peg_taps(host_weight(pre + "1.proj.kernel"), 3, d, dp);
        S.peg_b = upload_owned(pad_n(host_weight(pre + "1.proj.bias"), dp));
      }
      S.table = upload_owned(r2l_table_from_embedding(host_weight(pre + "2.local_rel_pos_bias.embeddings").data(), ws, kRvHeads));
      for (int L = 0; L < rv.depth[s]; ++L) {
        const std::string b = pre + "2.layers." + std::to_string(L) + ".", key = "rv." + b;
        RegionLayerW w;
        w.attn_norm = padded_norm(b + "0.norm", d, dp, ".gamma", ".beta");
        w.qkv = padded_dense(key + "qkv", b + "0.to_qkv", d, 3 * kRvInner, dp, 3 * kRvInner, &w.attn_norm, 1e-3f);
        // to_out reads the attention output in place of q: its K is the inner width, the rows' pitch is that of q|k|v
        w.to_out = padded_dense(key + "to_out", b + "0.to_out", kRvInner, d, kRvInner, dp);
        w.ff = prenorm_mlp("rv.", b + "1.net.0", b + "1.net.1", b + "1.net.4", d, dp, rv.mlp_mult, 1e-3f, ".gamma", ".beta");
        S.layers.push_back(std::move(w));
      }
      rv_stages.push_back(std::move(S));
    }
    const int dl = rv.dims[VB_REGIONVIT_STAGES - 1];
    head_norm = make_norm("to_logits.1", dl);
    head = make_linear_f32("to_logits.2", dl, cfg.num_classes);
  }
  void finalize_levit() {
    const int dh = levit_dh();
    int cin = cfg.channels;
    for (int i = 0; i < 4; ++i) {                                       // stem; the 32-channel map is written 64 wide (zero columns)
      const std::string n = "conv_embedding." + std::to_string(i);
      const int cout = levit_stem_cout(i), np = i == 0 ? 64 : channel_width(cout), K = 9 * cin;
      lv_stem.push_back(padded_dense("levit." + n, n, K, cout, K, np));
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
      b.pos = upload_owned(levit_pos_table(host_weight(a + "pos_bias.embeddings"), p.fmap * p.fmap, H,
                                             std::sqrt(static_cast<double>(dk))));
      const int hidden = p.dim_out * p.mult, hp = channel_width(hidden);
      b.fc1 = padded_dense(key + "fc1", p.pre + "1.net.0", p.dim_out, hidden, dpo, hp);
      b.fc2 = padded_dense(key + "fc2", p.pre + "1.net.3", hidden, p.dim_out, hp, dpo);
      lv_blocks.push_back(std::move(b));
    }
    const int dl = lv.dims[lv.stages - 1];
    head = make_linear_f32("mlp_head", dl, cfg.num_classes);
    if (lv.num_distill_classes > 0) lv_distill = make_linear_f32("distill_head", dl, lv.num_distill_classes);
  }
  // [heads][fmap^2] = embeddings[e, h] * inv_scale, the inverse of the softmax scale dim_key^-0.5 (levit.py:117): the table the
  // attention kernels add
  static std::vector<double> levit_pos_table(const std::vector<double>& emb, int f2, int heads, double inv_scale) {
    std::vector<double> t(static_cast<size_t>(heads) * f2);
    for (int h = 0; h < heads; ++h)
      for (int e = 0; e < f2; ++e) t[static_cast<size_t>(h) * f2 + e] = emb[static_cast<size_t>(e) * heads + h] * inv_scale;
    return t;
  }

  // ---- MobileViT weight packing: every BatchNorm folded on the host, channel widths zero-padded (bf16), heads widened to 32 (bf16)
  // A bias-free Conv2D `conv` [k, k, cin, N] and the BatchNormalization `bn` after it as one Dense: input channel c of tap t at row
  // t * pitch + (c < split ? c : split_at + c - split) (split 0: row t * pitch + c) of a zero [k * k * pitch, Np]
  Linear mv_conv_bn(const std::string& conv, const std::string& bn, int k, int cin, int N, int pitch, int Np, int split = 0, int split_at = 0) {
    auto Wk = host_weight(conv + ".kernel");
    std::vector<double> bias(N, 0.0);
    fold_bn(Wk, bias, k * k * cin, N, bn);
    std::vector<double> Wp(static_cast<size_t>(k) * k * pitch * Np, 0.0);
    for (int t = 0; t < k * k; ++t)
      for (int c = 0; c < cin; ++c) {
        const int row = t * pitch + (split > 0 && c >= split ? split_at + c - split : c);
        for (int n = 0; n < N; ++n) Wp[static_cast<size_t>(row) * Np + n] = Wk[(static_cast<size_t>(t) * cin + c) * N + n];
      }
    return linear_from_host("mv." + conv, Wp, pad_n(bias, Np), k * k * pitch, Np);
  }
  Linear mv_cbn(const std::string& n, int k, int cin, int N, int pitch, int split = 0, int split_at = 0) {   // Conv_NxN_BN `n`
    return mv_conv_bn(n + ".layers.0", n + ".layers.1", k, cin, N, pitch, channel_width(N), split, split_at);
  }
  void finalize_mobilevit() {
    mv_conv1 = mv_cbn("conv1", 3, cfg.channels, mv.channels[0], cfg.channels);
    for (int i = 0; i < VB_MOBILEVIT_MV2; ++i) {
      Mv2W m;
      const std::string p = mv2_pre(i);
      m.cin = mv.mv2_in[i]; m.hidden = mv.mv2_hidden[i]; m.cout = mv.mv2_out[i]; m.stride = mv.mv2_stride[i];
      m.cp_in = channel_width(m.cin); m.hp = channel_width(m.hidden); m.cp_out = channel_width(m.cout);
      m.expand = mv.mv2_expand[i] != 0; m.residual = mv.mv2_residual[i] != 0;
      const std::string dw = m.expand ? "3" : "0", dwbn = m.expand ? "4" : "1", pw = m.expand ? "6" : "3", pwbn = m.expand ? "7" : "4";
      if (m.expand) m.pw1 = mv_conv_bn(p + "0", p + "1", 1, m.cin, m.hidden, m.cp_in, m.hp);
      std::vector<double> taps, shift;
      cvt_fold_dw(host_weight(p + dw + ".kernel"), host_weight(p + dwbn + ".gamma"), host_weight(p + dwbn + ".beta"),
                  host_weight(p + dwbn + ".moving_mean"), host_weight(p + dwbn + ".moving_variance"), 3, m.hidden, m.hp, taps, shift);
      m.dw_w = upload_owned(taps);
      m.dw_b = upload_owned(shift);
      m.pw2 = mv_conv_bn(p + pw, p + pwbn, 1, m.hidden, m.cout, m.hp, m.cp_out);
      mv_mv2.push_back(std::move(m));
    }
    const int dh = mvit_dh(), I = kMvHeads * kMvDh, Ip = kMvHeads * dh;
    for (int s = 0; s < 3; ++s) {
      MvitBlockW v;
      const std::string p = mvit_pre(s);
      v.cin = mvit_cin(s); v.ch = mvit_ch(s); v.dim = mv.dims[s]; v.k = mv.kernel_size;
      v.cp_in = channel_width(v.cin); v.chp = channel_width(v.ch); v.dp = channel_width(v.dim);
      v.conv1 = mv_cbn(p + "conv1", v.k, v.cin, v.ch, v.cin);
      v.conv2 = mv_cbn(p + "conv2", 1, v.ch, v.dim, v.chp);
      for (int L = 0; L < mv.depths[s]; ++L) {
        const std::string b = p + "transformer.layers." + std::to_string(L) + ".", key = "mv." + b;
        MvitLayerW l;
        l.attn_norm = padded_norm(b + "0.norm", v.dim, v.dp, ".gamma", ".beta");
        // head h's 8 columns of q, k and v at g * Ip + h * dh; to_out's rows likewise (zero rows meet the pad columns)
        const auto wq = host_weight(b + "0.fn.to_qkv.kernel"), wo = host_weight(b + "0.fn.to_out.0.kernel");
        std::vector<double> Wqkv(static_cast<size_t>(v.dp) * 3 * Ip, 0.0), Wout(static_cast<size_t>(Ip) * v.dp, 0.0);
        for (int g = 0; g < 3; ++g)
          for (int h = 0; h < kMvHeads; ++h)
            for (int d = 0; d < kMvDh; ++d) {
              for (int r = 0; r < v.dim; ++r)
                Wqkv[static_cast<size_t>(r) * 3 * Ip + g * Ip + h * dh + d] = wq[static_cast<size_t>(r) * 3 * I + g * I + h * kMvDh + d];
              if (g == 0)
                for (int o = 0; o < v.dim; ++o) Wout[static_cast<size_t>(h * dh + d) * v.dp + o] = wo[static_cast<size_t>(h * kMvDh + d) * v.dim + o];
            }
        l.qkv = linear_from_host(key + "qkv", Wqkv, {}, v.dp, 3 * Ip, bf16() ? &l.attn_norm : nullptr);
        l.qkv.ln_d = v.dim;
        l.qkv.ln_eps = 1e-3f;                                          // Keras LayerNormalization (:56)
        l.to_out = linear_from_host(key + "to_out", Wout, pad_n(host_weight(b + "0.fn.to_out.0.bias"), v.dp), Ip, v.dp);
        l.ff = prenorm_mlp("mv.", b + "1.norm", b + "1.fn.net.0", b + "1.fn.net.3", v.dim, v.dp, mvit_mlp(s) / v.dim, 1e-3f, ".gamma", ".beta");
        l.ff.act = ACT_SILU;                                           // MLP (:67-73)
        v.layers.push_back(std::move(l));
      }
      v.conv3 = mv_cbn(p + "conv3", 1, v.dim, v.ch, v.dp);
      v.conv4 = mv_cbn(p + "conv4", v.k, v.ch + v.cin, v.ch, v.chp + v.cp_in, v.ch, v.chp);   // concat([x, y]) (:203)
      mv_vit.push_back(std::move(v));
    }
    mv_logits = mv_cbn("to_logits.0", 1, mv.channels[9], mv.last_dim, channel_width(mv.channels[9]));
    head = Linear();
    head.W = W("to_logits.2.kernel"); head.K = mv.last_dim; head.N = cfg.num_classes; head.ldw = mv.last_dim;   // Dense without bias
  }

  // ---- ScalableViT weight packing: q, k and v in the stage's head layout (SvitStageW), channel widths zero-padded (bf16), the PEG
  // residual folded, the pre-norm LayerNorms (eps 1e-5) folded into the SSA q and IWSA q|k|v GEMMs in the bf16 engine
  // The [K, heads * w] kernel `src` into dst [.., N]: its row k at row rowmap(k), head h's column j at column off + h * dh + j
  template <typename RowMap>
  static void sv_place(const std::vector<double>& src, int K, int heads, int w, std::vector<double>& dst, int N, int off, int dh,
                       RowMap rowmap) {
    for (int k = 0; k < K; ++k)
      for (int h = 0; h < heads; ++h)
        for (int j = 0; j < w; ++j) dst[static_cast<size_t>(rowmap(k)) * N + off + h * dh + j] = src[(static_cast<size_t>(k) * heads + h) * w + j];
  }
  Linear sv_folded(const std::string& key, const std::vector<double>& Wkn, int K, int N, const Norm& norm, int d) {
    Linear L = linear_from_host(key, Wkn, {}, K, N, bf16() ? &norm : nullptr);
    L.ln_d = d;
    L.ln_eps = 1e-5f;                                                // scalable_vit.py:47
    return L;
  }
  // to_out `n` [heads * w, d] + bias as [K, dp]: head h's row j at row h * dh + j, the other rows zero
  Linear sv_head_rows(const std::string& key, const std::string& n, int heads, int w, int dh, int K, int d, int dp) {
    const auto src = host_weight(n + ".kernel");
    std::vector<double> Wo(static_cast<size_t>(K) * dp, 0.0);
    for (int h = 0; h < heads; ++h)
      for (int j = 0; j < w; ++j)
        for (int o = 0; o < d; ++o) Wo[(static_cast<size_t>(h) * dh + j) * dp + o] = src[(static_cast<size_t>(h) * w + j) * d + o];
    return linear_from_host(key, Wo, pad_n(host_weight(n + ".bias"), dp), K, dp);
  }
  void finalize_scalable_vit() {
    const int C = cfg.channels, d0 = sv.dim[0];
    sv_stem = padded_dense("sv.to_patches", "to_patches", 49 * C, d0, 49 * C, channel_width(d0));   // :261
    const auto same = [](int k) { return k; };
    for (int st = 0; st < sv.num_stages; ++st) {
      SvitStageW S;
      const std::string p = sv_pre(st);
      const int d = sv_dim(st), dp = channel_width(d), H = sv.heads[st], r = sv.reduction_factor[st], f = sv.ff_expansion_factor;
      const int sk = sv.ssa_dim_key[st], svv = sv.ssa_dim_value[st], ik = sv.iwsa_dim_key[st], iv = sv.iwsa_dim_value[st];
      S.dim = d; S.dp = dp; S.heads = H; S.r = r; S.window = sv.window[st];
      S.dhs = sv_head_width(sk, svv); S.dhi = sv_head_width(ik, iv);
      const int HS = H * S.dhs, HI = H * S.dhi;
      S.ldq = channel_width(HS); S.ldkv = channel_width(2 * HS); S.ldqkv = channel_width(3 * HI); S.ldlim = channel_width(HI);
      S.ssa_scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(sk)));    // :109, :151
      S.iwsa_scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(ik)));
      for (int L = 0; L < sv.depth[st]; ++L) {
        const std::string b = p + "0.layers." + std::to_string(L) + ".", key = "sv." + b;
        SvitBlockW w;
        w.ssa_norm = padded_norm(b + "0.norm", d, dp);
        std::vector<double> Wq(static_cast<size_t>(dp) * S.ldq, 0.0);
        sv_place(host_weight(b + "0.fn.to_q.kernel"), d, H, sk, Wq, S.ldq, 0, S.dhs, same);
        w.ssa_q = sv_folded(key + "ssa_q", Wq, dp, S.ldq, w.ssa_norm, d);
        std::vector<double> Wkv(static_cast<size_t>(r) * r * d * S.ldkv, 0.0);
        sv_place(host_weight(b + "0.fn.to_k.kernel"), r * r * d, H, sk, Wkv, S.ldkv, 0, S.dhs, same);
        sv_place(host_weight(b + "0.fn.to_v.kernel"), r * r * d, H, svv, Wkv, S.ldkv, HS, S.dhs, same);
        w.ssa_kv = linear_from_host(key + "ssa_kv", Wkv, {}, r * r * d, S.ldkv);
        w.ssa_out = sv_head_rows(key + "ssa_out", b + "0.fn.to_out.0", H, svv, S.dhs, S.ldq, d, dp);
        w.mlp1 = prenorm_mlp("sv.", b + "1.norm", b + "1.fn.net.0", b + "1.fn.net.3", d, dp, f);
        if (L == 0) {
          w.peg_w = peg_taps(host_weight(b + "2.proj.kernel"), 3, d, dp);
          w.peg_b = upload_owned(pad_n(host_weight(b + "2.proj.bias"), dp));
        }
        w.mlp3 = prenorm_mlp("sv.", b + "3.norm", b + "3.fn.net.0", b + "3.fn.net.3", d, dp, f);
        w.iwsa_norm = padded_norm(b + "4.norm", d, dp);
        std::vector<double> Wqkv(static_cast<size_t>(dp) * S.ldqkv, 0.0);
        sv_place(host_weight(b + "4.fn.to_q.kernel"), d, H, ik, Wqkv, S.ldqkv, 0, S.dhi, same);
        sv_place(host_weight(b + "4.fn.to_k.kernel"), d, H, ik, Wqkv, S.ldqkv, HI, S.dhi, same);
        sv_place(host_weight(b + "4.fn.to_v.kernel"), d, H, iv, Wqkv, S.ldqkv, 2 * HI, S.dhi, same);
        w.iwsa_qkv = sv_folded(key + "iwsa_qkv", Wqkv, dp, S.ldqkv, w.iwsa_norm, d);
        // the LIM's input channel c = h iv + j of tap t is row t HI + h dhi + j; its output channels take the same head layout
        std::vector<double> Wl(static_cast<size_t>(9) * HI * S.ldlim, 0.0), bl(S.ldlim, 0.0);
        const int ci = H * iv;
        sv_place(host_weight(b + "4.fn.local_interactive_module.kernel"), 9 * ci, H, iv, Wl, S.ldlim, 0, S.dhi,
                 [&](int k) { return (k / ci) * HI + (k % ci) / iv * S.dhi + k % iv; });
        sv_place(host_weight(b + "4.fn.local_interactive_module.bias"), 1, H, iv, bl, S.ldlim, 0, S.dhi, same);
        w.lim = linear_from_host(key + "lim", Wl, bl, 9 * HI, S.ldlim);
        w.iwsa_out = sv_head_rows(key + "iwsa_out", b + "4.fn.to_out.0", H, iv, S.dhi, S.ldlim, d, dp);
        S.blocks.push_back(std::move(w));
      }
      S.norm = padded_norm(p + "0.norm", d, dp);
      S.down = st < sv.num_stages - 1;
      if (S.down) S.down_conv = padded_dense("sv." + p + "1.conv", p + "1.conv", 9 * d, 2 * d, 9 * d, channel_width(2 * d));
      sv_stages.push_back(std::move(S));
    }
    const int dl = sv_dim(sv.num_stages - 1);
    head_norm = make_norm("mlp_head.1", dl);
    head = make_linear_f32("mlp_head.2", dl, cfg.num_classes);
  }

  // vit_for_small_dataset.ViT (:159-195): SPT (set_spt_patch), then ViT's layers with LSA: the diagonal mask and exp(temperature)
  // as the softmax scale.
  void finalize_small_dataset_vit() {
    const vb_config& c = cfg;
    const int np = (c.image_h / c.patch_h) * (c.image_w / c.patch_w), K = c.patch_h * c.patch_w * 5 * c.channels;
    embed = EmbedW();
    set_spt_patch(host_weight("patch_norm.gamma"), host_weight("patch_norm.beta"), host_weight("patch.kernel"), host_weight("patch.bias"), K,
                  c.dim);
    embed.pos = W("pos_embedding");
    embed.cls = W("cls_token");
    embed.dim = c.dim; embed.n_pos = np + 1;
    for (int L = 0; L < c.depth; ++L) {
      const std::string pre = "layers." + std::to_string(L) + ".";
      layers.push_back(make_layer(pre, c.dim, c.heads, c.dim_head, c.mlp_dim, c.kind));
      layers.back().lsa = true;
      layers.back().lsa_scale = expf(static_cast<float>(host_weight(pre + "temperature")[0]));
    }
    head_norm = make_norm("head_norm", c.dim);
    head = make_linear_f32("head", c.dim, c.num_classes);
  }
  // SPT's LayerNorm gamma / beta [K] (eps 1e-3) and patch Dense W [K, dim] + bias as spt_tokens runs them: the bf16 engine zero-pads
  // K to Kp = round_up(K, 64) and folds the LayerNorm into the wgmma GEMM (dim % 64 == 0); otherwise
  // the LayerNorm kernel runs first.  Either way the Dense yields beta . W + bias on the all-zero cls row, so that is the term the
  // embedding residual takes off (res_bias).
  void set_spt_patch(const std::vector<double>& gamma, const std::vector<double>& beta, const std::vector<double>& Wk,
                     std::vector<double> bias, int K, int dim) {
    const int Kp = bf16() ? round_up(K, 64) : K;
    const bool fold = bf16() && dim % 64 == 0;
    spt_norm = Norm{upload_owned(pad_n(gamma, Kp)), upload_owned(pad_n(beta, Kp)), K};
    embed.patch = linear_from_host("spt.patch", pad_kn(Wk, K, dim, Kp, dim), bias, Kp, dim, fold ? &spt_norm : nullptr);
    if (fold) {
      embed.patch.ln_d = K; embed.patch.ln_eps = 1e-3f;
      embed.res_bias = embed.patch.ln_c2;
    } else {
      for (int k = 0; k < K; ++k)
        for (int n = 0; n < dim; ++n) bias[n] += beta[k] * Wk[static_cast<size_t>(k) * dim + n];
      embed.res_bias = upload_owned(bias);
    }
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
      build_embed_residual<T>(static_cast<T*>(m->p), e.pos, e.cls, e.res_bias != nullptr ? e.res_bias : e.patch.bias, B, rows, e.dim,
                              e.cls != nullptr, s);
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
  // into its residual operand.  cols [B*rows, Kp]: patch vectors, zero in the cls rows and in the pad columns.  ln_stats (bf16, a
  // patch Dense with a LayerNorm folded in): the row statistics of cols.
  template <typename T>
  T* embed_from_cols(const EmbedW& e, const T* col, int Kp, int B, int rows, cudaStream_t s, float** stats_out,
                     const float* ln_stats = nullptr) {
    const int M = B * rows;
    const T* R = embed_residual<T>(e, B, rows, s);
    T* X = arena.get<T>(static_cast<size_t>(M) * e.dim);
    Epi ep; ep.bias = e.patch.bias; ep.res = R; ep.ldr = e.dim;
    ep.drop = dropout(e.site, true, DROP_AFTER_RES);              // vit.py:166: Dropout(emb_dropout) of the sum
    if (ln_stats != nullptr) { ep.ln_stats = ln_stats; ep.bias = e.patch.ln_c2; }
    if (stats_out != nullptr && bf16() && e.dim % 64 == 0) {
      *stats_out = row_stats(M, e.dim);
      ep.stats_out = *stats_out;
    }
    Linear L = e.patch;
    L.K = Kp;  // im2col zero-pads the patch vector to the packed weight pitch
    linear<T>(col, Kp, M, L, X, e.dim, ep, s);
    return X;
  }

  // SPT + cls token + positions (vit_for_small_dataset.py:152-157, 198-203) -> X [B*rows, dim]: spt_rows writes the patch vectors
  // of the image and its four shifts (zero cls rows and pad columns), then the LayerNorm (folded into the GEMM in bf16, from the
  // rows' statistics) and the Dense with cls and positions in its residual operand.
  template <typename T>
  T* spt_tokens(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s, float** stats_out) {
    const int p = cfg.patch_h;
    VB_CHECK(H % p == 0 && Wd % p == 0, "Image dimensions must be divisible by the patch size.");
    const int rows = (H / p) * (Wd / p) + 1, M = B * rows, Kp = embed.patch.K;
    VB_CHECK(rows <= embed.n_pos, "image has more patches than pos_embedding rows");
    T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, 4.0 * B * H * Wd * cfg.channels + static_cast<double>(sizeof(T)) * M * Kp, s);
      spt_rows<T>(img, col, B, H, Wd, cfg.channels, p, Kp, s);
    }
    *rows_out = rows;
    if (embed.patch.ln_c1 != nullptr) {
      float* st = row_stats(M, Kp);
      ensure_stats(col, Kp, st, M, s);
      return embed_from_cols<T>(embed, col, Kp, B, rows, s, stats_out, st);
    }
    T* Y = arena.get<T>(static_cast<size_t>(M) * Kp);
    {
      ProfScope ps(this, PROF_LN, 0.0, 2.0 * sizeof(T) * M * Kp, s);
      layernorm<T>(col, Kp, spt_norm.gamma, spt_norm.beta, Y, Kp, M, spt_norm.D, s, Kp);   // Keras eps 1e-3, pad columns zero
    }
    return embed_from_cols<T>(embed, Y, Kp, B, rows, s, stats_out);
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
      const bool tc = !last && bf16();                                 // tensor-core layer: token rows padded to Dp columns
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

  // PiT.patch_embedding + cls + positions (pit.py:179-182,208-213): extract_patches(p, stride p / 2, VALID) is unfold_same's VALID
  // mode with its (k_row, k_col, c) vectors, written with the zero cls row at the packed weight pitch; the Dense folds cls and
  // positions into its residual operand.
  template <typename T>
  T* embed_pit(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s, float** stats_out) {
    const int p = cfg.patch_h, stride = p / 2;
    VB_CHECK(H >= p && Wd >= p, "PiT: a " + std::to_string(H) + " x " + std::to_string(Wd) + " image is smaller than one " +
                                    std::to_string(p) + " x " + std::to_string(p) + " patch");
    const int rows = pit_side(H) * pit_side(Wd) + 1, Kp = bf16() ? embed.patch.ldw : embed.patch.K;
    VB_CHECK(rows <= embed.n_pos, "PiT: the image gives " + std::to_string(rows - 1) + " patches but pos_embedding has rows for " +
                                      std::to_string(embed.n_pos - 1));
    T* col = arena.get<T>(static_cast<size_t>(B) * rows * Kp);
    UnfoldMode um;
    um.valid = true;
    {
      ProfScope ps(this, PROF_EMBED, 0.0, 4.0 * B * H * Wd * cfg.channels + static_cast<double>(sizeof(T)) * B * rows * Kp, s);
      unfold_same<float, T>(img, col, B, H, Wd, cfg.channels, p, stride, 1, Kp, s, 0, &um);
    }
    *rows_out = rows;
    return embed_from_cols<T>(embed, col, Kp, B, rows, s, stats_out);
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
      const Linear& cw = cct_convs[i];
      const int oh = (mh + c.cct_stride - 1) / c.cct_stride, ow = (mw + c.cct_stride - 1) / c.cct_stride, M = B * oh * ow;
      T* conv_out = arena.get<T>(static_cast<size_t>(M) * cw.N);
      conv<T>(img, map, mc, B, mh, mw, mc, c.cct_kernel, c.cct_stride, cw, conv_out, nullptr, s);   // bias-free
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
      out = arena.get<T>(static_cast<size_t>(B) * rows * cw.N);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, static_cast<double>(sizeof(T)) * (static_cast<double>(M) + static_cast<double>(B) * rows) * cw.N, s);
        maxpool_relu_same<T>(conv_out, out, B, oh, ow, cw.N, c.cct_pool_kernel, c.cct_pool_stride, pos, rows, s);
      }
      map = out; mh = ph; mw = pw; mc = cw.N;
      *rows_out = rows;
    }
    return out;
  }

  // `call` up to the transformer for every kind with one token stream
  template <typename T>
  T* embed_any(const float* img, int B, int H, int Wd, int* rows_out, cudaStream_t s, float** stats_out) {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT has two token streams: no single embedding stage");
    if (cfg.kind == VB_KIND_T2T_VIT) return embed_t2t<T>(img, B, H, Wd, rows_out, s, stats_out);
    if (cfg.kind == VB_KIND_PIT) return embed_pit<T>(img, B, H, Wd, rows_out, s, stats_out);
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
    const int M = B * rows;
    const bool fold = l.folded && stats != nullptr;
    if (fold && !*stats_valid) { ensure_stats(X, dim, stats, M, s); *stats_valid = true; }
    T* Y = arena.get<T>(static_cast<size_t>(M) * dim);
    attend_self<T>(X, B, rows, dim, l, s, fold ? stats : nullptr, Y);
    feed_forward<T>(X, M, dim, l, Y, s, fold ? stats : nullptr);
    // an unfolded layer rewrote X without updating the statistics: a folded layer after it (PiT, whose stages' head counts can
    // fold one stage and not the next) recomputes them
    if (!fold && stats_valid != nullptr) *stats_valid = false;
  }
  // The attention half of layer_self: X += to_out(attention(LN(X))) (the residual carried by to_out's epilogue), with the row
  // statistics `stats` (non-null iff the layer is folded; valid on entry) kept up to date.  Y [M, dim]: LayerNorm scratch of the
  // unfolded layer.  nk_img (may be null): image b's keys >= nk_img[b] masked (ATS-ViT's dead rows).  Returns the fused q|k|v rows
  // (null for separate to_q / to_kv).
  template <typename T>
  const T* attend_self(T* X, int B, int rows, int dim, const LayerW& l, cudaStream_t s, float* stats, T* Y, const int* nk_img = nullptr) {
    const int M = B * rows, inner = l.heads * l.dim_head;
    const bool fold = stats != nullptr;
    const T* qkv = nullptr;
    T* O = arena.get<T>(static_cast<size_t>(M) * inner);
    const T* A = X;
    Epi eq;
    if (fold) eq.ln_stats = stats;
    else { VB_CHECK(!l.folded, "internal: folded layer without statistics"); ln<T>(X, l.attn_norm, Y, M, dim, s); A = Y; }
    if (l.fused_qkv) {
      T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * inner);
      Epi e = eq; e.bias = l.to_qkv.ln_c2;
      linear<T>(A, dim, M, l.to_qkv, QKV, 3 * inner, e, s);
      if (nk_img != nullptr || l.lsa)
        attention_masked_dispatch<T>(QKV, 3 * inner, O, inner, B, rows, l.heads, l.dim_head, l.dh_model,
                                     l.lsa ? l.lsa_scale : 1.0f / sqrtf(static_cast<float>(l.dh_model)),
                                     l.lsa ? ATTN_MASK_DIAG : ATTN_MASK_KEYS, s, nk_img);
      else attention<T>(QKV, 3 * inner, QKV + inner, 3 * inner, QKV + 2 * inner, 3 * inner, O, inner, B, rows, rows, l, s);
      qkv = QKV;
    } else {
      VB_CHECK(nk_img == nullptr, "internal: masked attention reads fused q|k|v rows");
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
      e.drop = dropout(l.site_out, false, DROP_BEFORE_RES);
      if (fold) e.stats_out = stats;
      linear<T>(O, inner, M, l.to_out, X, dim, e, s);
    } else {
      add_tokens<T>(X, O, static_cast<long long>(M) * dim, s);   // vit.py:53: identity out-projection
      if (fold) ensure_stats(X, dim, stats, M, s);
    }
    return qkv;
  }
  // Plain attention over the fused q|k|v rows of `heads` heads of width dh with masked keys: image b's keys >= nk_img[b]
  // (ATTN_MASK_KEYS, ATS-ViT), or the diagonal (ATTN_MASK_DIAG, an LSA layer, with the scale exp(temperature)).  The flash kernels
  // at dh 64 (bf16), else the materialised-scores path with the mask in its softmax, which needs the model's own head width dh_model.
  template <typename T>
  void attention_masked_dispatch(const T* qkv, int ld, T* out, int ldo, int B, int n, int heads, int dh, int dh_model, float scale, int mask,
                                 cudaStream_t s, const int* nk_img) {
    const int HD = heads * dh;
    VB_CHECK(mask != ATTN_MASK_DIAG || n >= 2, "locality self-attention needs at least 2 tokens (every row keeps a key besides its own)");
    ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * n * n * dh, static_cast<double>(sizeof(T)) * B * heads * dh * 4.0 * n, s);
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
      if (attention_masked(qkv, ld, qkv + HD, ld, qkv + 2 * HD, ld, out, ldo, B, n, n, heads, dh, s, scale, nk_img, mask)) return;
    }
    VB_CHECK(dh == dh_model, "internal: a head-padded layer must run on the fused attention kernel");
    float* S = arena.get<float>(static_cast<size_t>(B) * heads * n * n);
    attention_generic_masked<T>(qkv, ld, qkv + HD, ld, qkv + 2 * HD, ld, out, ldo, S, B, n, n, heads, dh, s, scale, nk_img, mask);
  }

  // ATS-ViT's forward (ats_vit.py:300-318, Transformer.call :236-258) in the compact row layout of ats.cu: image b's rows at the
  // layer's pitch P[L] are [cls, its kept tokens in ascending id order, dead rows].  Masked keys get weight exactly 0 in the
  // reference (exp(-FLT_MAX - max) underflows), and its pad rows never reach the cls row or a kept row, so the logits depend on
  // the kept rows alone.  Every decision that depends on the data (whether a layer samples, C > K) is taken on the device.
  template <typename T>
  void ats_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    const vb_config& c = cfg;
    int rows = 0;
    float* stats = nullptr;
    T* X = embed_tokens<T>(embed, img, B, H, Wd, c.patch_h, c.patch_w, &rows, s, &stats);
    const AtsPlan& p = ats_last;
    VB_CHECK(p.B == B && p.P[0] == rows && ats_dev.bytes >= p.total * sizeof(int), "internal: ATS state not prepared for this batch");
    int* st = static_cast<int*>(ats_dev.p);
    unsigned long long* rng = ats_rng_ptr();
    { ProfScope ps(this, PROF_OTHER, 0.0, 4.0 * B * rows, s); ats_init(st + p.rows, st + p.C, st + p.ids[0], B, rows, s); }
    bool sv = stats != nullptr;
    for (int L = 0; L < c.depth; ++L) X = ats_layer<T>(X, B, L, p, st, rng, s, stats, &sv);
    classify<T>(X, p.P[c.depth], c.dim, head_norm, head, B, 0, logits, false, s);
    const int f = p.slot[c.depth];
    ProfScope ps(this, PROF_OTHER, 0.0, 8.0 * B * p.P[c.depth], s);
    ats_ids_out(st + p.ids[f], p.P[c.depth], st + p.rows + static_cast<size_t>(f) * B, st + p.C + f, st + p.out, B, s);
  }
  // One ATS layer (ats_vit.py:246-256): the LayerNorm-folded to_qkv, the masked attention and the residual to_out over all P[L]
  // rows; on a layer that can sample, ats_sample and ats_gather into the next pitch; the MLP over P[L + 1] rows.
  template <typename T>
  T* ats_layer(T* X, int B, int L, const AtsPlan& p, int* st, unsigned long long* rng, cudaStream_t s, float* stats, bool* sv) {
    const LayerW& l = layers[L];
    const int dim = cfg.dim, P = p.P[L], Pn = p.P[L + 1], M = B * P, K = ats.max_tokens_per_depth[L];
    const int si = p.slot[L];
    const int* nk = st + p.rows + static_cast<size_t>(si) * B;
    const bool fold = l.folded && stats != nullptr;
    if (fold && !*sv) { ensure_stats(X, dim, stats, M, s); *sv = true; }
    T* Y = arena.get<T>(static_cast<size_t>(M) * dim);
    const T* qkv = attend_self<T>(X, B, P, dim, l, s, fold ? stats : nullptr, Y, nk);
    if (p.can[L]) {
      const int so = p.slot[L + 1], ld = 3 * l.heads * l.dim_head;
      int* rows_new = st + p.rows + static_cast<size_t>(so) * B;
      int* sel = arena.get<int>(static_cast<size_t>(B) * Pn);
      float* scratch = arena.get<float>(static_cast<size_t>(3) * B * P);
      T* Xn = arena.get<T>(static_cast<size_t>(B) * Pn * dim);
      {
        ProfScope ps(this, PROF_OTHER, 4.0 * B * P * l.heads * l.dim_head + 60.0 * B * K * P,
                     static_cast<double>(sizeof(T)) * B * P * 3 * l.heads * l.dim_head, s);
        ats_sample<T>(qkv, ld, B, P, l.heads, l.dim_head, 1.0f / sqrtf(static_cast<float>(l.dh_model)), nk, st + p.C + si, K, rng,
                      scratch, sel, Pn, rows_new, st + p.draws[L], s);
      }
      {
        ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * B * Pn * dim, s);
        ats_gather<T>(X, P, Xn, Pn, dim, sel, rows_new, st + p.ids[si], st + p.ids[so], B, st + p.C + si, K, st + p.C + so, rng, s);
      }
      X = Xn;
      if (fold) ensure_stats(X, dim, stats, B * Pn, s);
    }
    feed_forward<T>(X, B * Pn, dim, l, Y, s, fold ? stats : nullptr);
    return X;
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
    e1.drop = dropout(l.site_ff, false, DROP_BEFORE_RES);
    linear<T>(A, dim, M, l.fc1, Hb, l.fc1.N, e1, s);
    Epi e2; e2.bias = l.fc2.bias; e2.scale = l.ff_scale; e2.res = X; e2.ldr = dim;
    e2.drop = dropout(l.site_ff < 0 ? -1 : l.site_ff + 1, false, DROP_BEFORE_RES);
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
    e.drop = dropout(l.site_out, false, DROP_BEFORE_RES);
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
      e1.drop = dropout(x.site, false, DROP_BEFORE_RES);           // cross_vit.py:64-67: to_out's Dropout, before project_out
      linear<T>(O, inner, B, x.to_out, a, dctx, e1, s);
      Epi e2; e2.bias = x.project_out.bias; e2.res = cls; e2.ldr = dcls;
      linear<T>(a, dctx, B, x.project_out, cls, dcls, e2, s);
    } else {
      Epi e; e.bias = x.to_out.bias; e.res = cls; e.ldr = dcls;
      e.drop = dropout(x.site, false, DROP_BEFORE_RES);
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

  template <typename T>
  void forward_impl(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    arena.reset();
    const vb_config& c = cfg;
    if (c.kind == VB_KIND_VIT || c.kind == VB_KIND_DEEPVIT || c.kind == VB_KIND_T2T_VIT || c.kind == VB_KIND_PIT) {
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
    } else if (c.kind == VB_KIND_NEST) {
      nest_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_REGIONVIT) {
      regionvit_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_ATS_VIT) {
      ats_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_MOBILEVIT) {
      mobilevit_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_SCALABLE_VIT) {
      svit_forward<T>(img, B, H, Wd, logits, s);
    } else if (c.kind == VB_KIND_SMALL_DATASET_VIT) {     // vit_for_small_dataset.py:197-215, Transformer.call :135-140
      int rows = 0;
      float* stats = nullptr;
      T* X = spt_tokens<T>(img, B, H, Wd, &rows, s, &stats);
      bool sv = stats != nullptr;
      for (const auto& l : layers) layer_self<T>(X, B, rows, c.dim, l, s, stats, &sv);
      classify<T>(X, rows, c.dim, head_norm, head, B, c.pool == VB_POOL_MEAN, logits, false, s);
    } else if (c.kind == VB_KIND_CCT) {                   // CCT.call cct.py:342-345, TransformerClassifier.call :277-305
      int rows = 0;
      T* X = tokenize_cct<T>(img, B, H, Wd, &rows, s);
      float* stats = c.dim % 64 == 0 ? row_stats(static_cast<long long>(B) * rows, c.dim) : nullptr;
      bool sv = false;
      for (const auto& l : layers) layer_cct<T>(X, B, rows, c.dim, l, s, stats, &sv);
      float* z = arena.get<float>(static_cast<size_t>(B) * c.dim);
      {
        ProfScope ps(this, PROF_LN, 4.0 * B * rows * c.dim, static_cast<double>(sizeof(T)) * B * rows * c.dim, s);
        seq_pool<T>(X, rows, c.dim, cct_norm.gamma, cct_norm.beta, cct_pool_w, cct_pool_b, z, B, s);   // :291-299
      }
      dense_head(z, c.dim, head, B, logits, s);                                                         // fc :303
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
      // and joined with timing-less events (part of the captured graph).  Profiling keeps one stream: per-class event timing wants it.
      const bool two = !profiling && bf16();
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
    // after the last site on the forward's stream (CrossViT's side stream joined before the cross-attention), as a plain launch: it
    // starts when every kernel before it has completed, and the next forward's dropout kernels read the counter after it
    if (dropout_active()) { ProfScope ps(this, PROF_OTHER, 0.0, 16.0, s); dropout_advance(static_cast<unsigned long long*>(drop_dev.p), s); }
  }

  float* row_stats(long long M, int dp) {       // (sum, sumsq) partials per 64-column chunk of M rows: bf16 only
    return bf16() ? arena.get<float>(static_cast<size_t>(M) * (dp / 64) * 2) : nullptr;
  }
  // A convolution as unfold_same + GEMM: the fp32 image (map == null, cin channels) or the first cin channels of the token map
  // [B h w, ld], unfolded at the packed weight pitch (`um`: VALID, or the LayerNorm / GELU applied on load), then out [rows, L.N] =
  // act(col W + b) (Act) (+ res [rows, ldr] when given), with the output rows' statistics when stats_out is given
  template <typename T>
  void conv(const float* img, const T* map, int ld, int B, int h, int w, int cin, int k, int stride, const Linear& L, T* out,
            float* stats_out, cudaStream_t s, const UnfoldMode* um = nullptr, int act = ACT_NONE, const T* res = nullptr, int ldr = 0) {
    const bool valid = um != nullptr && um->valid;
    const int oh = valid ? (h - k) / stride + 1 : (h + stride - 1) / stride, ow = valid ? (w - k) / stride + 1 : (w + stride - 1) / stride;
    const int rows = B * oh * ow, Kp = bf16() ? L.ldw : L.K;
    T* col = arena.get<T>(static_cast<size_t>(rows) * Kp);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(map ? sizeof(T) : 4) * B * h * w * cin + static_cast<double>(sizeof(T)) * rows * Kp, s);
      if (map == nullptr) unfold_same<float, T>(img, col, B, h, w, cin, k, stride, 0, Kp, s, 0, um);
      else unfold_same<T, T>(map, col, B, h, w, cin, k, stride, 0, Kp, s, ld, um);
    }
    Linear Lk = L;
    Lk.K = Kp;                      // unfold_same zero-pads the patch vectors to the packed weight pitch
    Epi e; e.bias = L.bias; e.stats_out = stats_out; e.set_act(act); e.res = res; e.ldr = ldr;
    linear<T>(col, Kp, rows, Lk, out, L.N, e, s);
  }
  // The pre-norm sub-blocks x = f(LN(x)) + x over X [M, dp] (true width d).  bf16 folds the LayerNorm into f's first GEMM from
  // the row statistics `stats`, which the residual epilogues keep current; fp32 runs it into the scratch Y first.
  template <typename T>
  struct PreNorm {
    vb_handle& h;
    T* X;
    int M, d, dp;
    float* stats;
    float eps;
    T* Y;                           // fp32 only
    cudaStream_t s;
    PreNorm rows(T* X0, int M0, float* st) const { PreNorm r = *this; r.X = X0; r.M = M0; r.stats = st; return r; }
    const T* norm(const Norm& n) const {          // the A operand of the GEMM that folded_epi's Epi goes with
      if (Y == nullptr) return X;
      ProfScope ps(&h, PROF_LN, 8.0 * M * d, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(X, dp, n.gamma, n.beta, Y, dp, M, d, s, dp, eps);
      return Y;
    }
    Epi folded_epi(const Linear& L) const {
      Epi e;
      if (Y == nullptr) { e.bias = L.ln_c2; e.ln_stats = stats; } else { e.bias = L.bias; }
      return e;
    }
    void residual(const T* A, int lda, const Linear& L) const {   // X = A W + b + X, and X's new row statistics
      Epi e; e.bias = L.bias; e.res = X; e.ldr = dp; e.stats_out = stats;
      h.linear<T>(A, lda, M, L, X, dp, e, s);
    }
    void mlp(const MlpW& m) const {                               // X = fc2(act(fc1(LN(X)))) + X
      const T* a = norm(m.norm);
      T* Hb = h.arena.get<T>(static_cast<size_t>(M) * m.fc1.N);
      Epi e1 = folded_epi(m.fc1);
      e1.set_act(m.act);
      h.linear<T>(a, dp, M, m.fc1, Hb, m.fc1.N, e1, s);
      residual(Hb, m.fc1.N, m.fc2);
    }
  };
  template <typename T>
  PreNorm<T> prenorm(T* X, int M, int d, int dp, float* stats, float eps, cudaStream_t s) {
    return PreNorm<T>{*this, X, M, d, dp, stats, eps, bf16() ? nullptr : arena.get<T>(static_cast<size_t>(M) * dp), s};
  }
  // The mean over each image's `rows` token rows [.., ld] of their first d columns -> z [B, d]
  template <typename T>
  float* mean_pool(const T* X, int rows, int ld, int d, int B, cudaStream_t s) {
    float* z = arena.get<float>(static_cast<size_t>(B) * d);
    ProfScope ps(this, PROF_LN, 1.0 * B * rows * d, static_cast<double>(sizeof(T)) * B * rows * d, s);
    pool_layernorm<T>(X, rows, ld, nullptr, nullptr, z, B, d, 1, s);
    return z;
  }
  void dense_head(const float* z, int d, const Linear& L, int B, float* out, cudaStream_t s) {   // fp32 Dense on pooled rows
    gemm_simt<float, float, float>(z, d, L.W, L.N, 1, out, L.N, B, L.N, d, L.bias, nullptr, nullptr, L.N, 0, s);
  }

  // LeViT.call (levit.py:214-226): stem -> backbone -> GlobalAvgPool2D -> mlp_head (and distill_head when distill != null).
  // The token rows of every block are the NHWC map, pixel-major: row b * fmap^2 + r * fmap + c.
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
      const Linear& L = lv_stem[i];
      const int oh = (mh + 1) / 2, ow = (mw + 1) / 2;
      X = arena.get<T>(static_cast<size_t>(B) * oh * ow * L.N);
      conv<T>(img, map, ld_in, B, mh, mw, mc, 3, 2, L, X, nullptr, s);
      map = X; mh = oh; mw = ow; mc = levit_stem_cout(i); ld_in = L.N;
    }
    int f = fmap;
    for (const auto& b : lv_blocks) {
      X = levit_block<T>(X, B, b, s);
      f = (b.fmap + b.step - 1) / b.step;
    }
    const int dl = lv.dims[lv.stages - 1];
    const float* z = mean_pool<T>(X, f * f, channel_width(dl), dl, B, s);   // GlobalAvgPool2D (levit.py:206-208)
    dense_head(z, dl, head, B, logits, s);
    if (distill != nullptr) dense_head(z, dl, lv_distill, B, distill, s);
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
      attention_bias<T>(QKV, 3 * HD, QKV + HD, 3 * HD, QKV + 2 * HD, 3 * HD, O, HD, B, nq, f2, b.heads, b.dh, b.scale, pb, s);
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
      attention_bias<T>(Q, HD, KV, 2 * HD, KV + HD, 2 * HD, O, HD, B, nq, f2, b.heads, b.dh, b.scale, pb, s);
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
  void attention_bias(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq, int nk, int heads,
                      int dh, float scale, const PosBias& pb, cudaStream_t s) {
    ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * nq * nk * dh, static_cast<double>(sizeof(T)) * B * heads * dh * (2.0 * nq + 2.0 * nk), s);
    if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, s, scale, &pb))
      return;
    float* S = arena.get<float>(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15));
    attention_generic<T>(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, s, scale, &pb);
  }

  // CvT.call (cvt.py:182-202): per stage, Conv2D (SAME, bias) -> LayerNorm -> blocks; then GlobalAvgPool2D -> Dense.  Token rows
  // are the NHWC map, pixel-major, channel widths zero-padded to channel_width.  Any h x w: each SAME stride gives ceil.
  template <typename T>
  void cvt_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    int mh = H, mw = Wd, mc = cfg.channels, ld_in = 0;
    const T* map = nullptr;
    T* X = nullptr;
    for (const CvtStageW& S : cvt_stages) {
      const int oh = (mh + S.stride - 1) / S.stride, ow = (mw + S.stride - 1) / S.stride, M = B * oh * ow;
      T* Y = arena.get<T>(static_cast<size_t>(M) * S.dp);
      conv<T>(img, map, ld_in, B, mh, mw, mc, S.k, S.stride, S.conv, Y, nullptr, s);
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = row_stats(M, S.dp);
      {
        ProfScope ps(this, PROF_LN, 8.0 * M * S.dim, 2.0 * sizeof(T) * M * S.dp, s);
        layernorm<T>(Y, S.dp, S.norm.gamma, S.norm.beta, X, S.dp, M, S.dim, s, S.dp, 1e-5f);   // cvt.py:188
      }
      if (bf16()) ensure_stats<T>(X, S.dp, stats, M, s);               // the first block's PreNorm statistics
      for (const CvtBlockW& b : S.blocks) cvt_block<T>(X, B, oh, ow, b, stats, s);
      map = X; mh = oh; mw = ow; mc = S.dim; ld_in = S.dp;
    }
    const int dl = cv.emb_dim[VB_CVT_STAGES - 1];
    dense_head(mean_pool<T>(X, mh * mw, ld_in, dl, B, s), dl, head, B, logits, s);   // GlobalAvgPool2D cvt.py:196
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
    const PreNorm<T> p = prenorm<T>(X, M, b.dim, dp, stats, 1e-5f, s);
    cvt_dwconv<T>(p, B, H, Wd, b, Qd, KVd, s);
    T* Q = arena.get<T>(static_cast<size_t>(M) * HD);
    T* KV = arena.get<T>(static_cast<size_t>(Mk) * 2 * HD);
    linear<T>(Qd, dp, M, b.pw_q, Q, HD, Epi(), s);                      // cvt.py:86 (no bias)
    linear<T>(KVd, dp, Mk, b.pw_kv, KV, 2 * HD, Epi(), s);
    T* O = arena.get<T>(static_cast<size_t>(M) * HD);
    attention_dispatch<T>(Q, HD, KV, 2 * HD, KV + HD, 2 * HD, O, HD, B, H * Wd, Ho * Wo, b.heads, 64, 0, nullptr, nullptr, nullptr, nullptr, s);
    p.residual(O, HD, b.to_out);
    p.mlp(b.ff);
  }
  // The attention's PreNorm (cvt.py:53) and the depthwise convolutions with their BatchNormalizations (cvt.py:80-85) of a CvT
  // layer over p's rows, the B x H x Wd map: Qd [B H Wd, dp] at stride 1, KVd [B ceil(H / s) ceil(Wd / s), dp] at kv_stride
  template <typename T>
  void cvt_dwconv(const PreNorm<T>& p, int B, int H, int Wd, const CvtBlockW& b, T* Qd, T* KVd, cudaStream_t s) {
    const int dp = b.dp, st = b.kv_stride, M = B * H * Wd, Mk = B * ((H + st - 1) / st) * ((Wd + st - 1) / st);
    const T* a = p.norm(b.attn_norm);
    ProfScope ps(this, PROF_OTHER, 2.0 * b.k * b.k * b.dim * (static_cast<double>(M) + Mk),
                 static_cast<double>(sizeof(T)) * dp * (2.0 * M + Mk) + (p.stats ? 8.0 * M * (dp / 64) : 0.0), s);
    dwconv_qkv<T>(a, dp, p.Y ? nullptr : p.stats, b.attn_norm.gamma, b.attn_norm.beta, b.dim, 1e-5f, b.wq, b.bq, Qd, dp, b.wkv, b.bkv, KVd, dp,
                  B, H, Wd, dp, b.k, st, s);
  }

  // TwinsSVT.call (twins_svt.py:266-268): per stage, PatchEmbedding -> Transformer(1) -> PEG -> Transformer(depth); then
  // GlobalAvgPool2D -> Dense.  Token rows are the NHWC map, pixel-major, channel widths zero-padded to channel_width; no stage
  // permutes its map.  bf16: `stats` holds the (sum, sumsq) partials of X's rows between sub-blocks (emitted by the patch
  // embedding's and the residual GEMMs' epilogues, and after the PEG by a row-statistics pass).
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
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = row_stats(M, S.dp);
      conv<T>(img, map, ld_in, B, mh, mw, mc, S.patch, S.patch, S.proj, X, stats, s);
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
    dense_head(mean_pool<T>(X, mh * mw, ld_in, dl, B, s), dl, head, B, logits, s);   // GlobalAvgPool2D twins_svt.py:262
  }
  // One Transformer layer (twins_svt.py:206-211) in place on X [B*H*W, dp].  bf16: the PreNorm LayerNorms are folded into the
  // fused local q|k|v, the global to_q and the fc1s (from `stats`), and applied on load by the global to_kv's patch gather; fp32:
  // separate LayerNorms.
  template <typename T>
  void twins_layer(T* X, int B, int H, int Wd, const TwinsStageW& S, const TwinsLayerW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, M = B * H * Wd, I = kTwinsInner;
    const PreNorm<T> p = prenorm<T>(X, M, d, dp, stats, 1e-5f, s);   // the MLPs: twins_svt.py:78-92
    T* O = arena.get<T>(static_cast<size_t>(M) * I);
    if (l.local) {                                                    // LocalAttention twins_svt.py:135-156
      const T* a = p.norm(l.local_norm);
      T* QKV = arena.get<T>(static_cast<size_t>(M) * 3 * I);
      linear<T>(a, dp, M, l.qkv, QKV, 3 * I, p.folded_epi(l.qkv), s);
      Window win;
      win.p = S.local; win.nx = Wd / S.local; win.ny = H / S.local;
      const int n = S.local * S.local;
      attention_dispatch<T>(QKV, 3 * I, QKV + I, 3 * I, QKV + 2 * I, 3 * I, O, I, B * win.nx * win.ny, n, n, I / 64, 64, 0, nullptr, nullptr,
                            nullptr, nullptr, s, 0.f, &win);
      p.residual(O, I, l.local_out);
      p.mlp(l.ff1);
    }
    // GlobalAttention twins_svt.py:175-190: q from every pixel, k|v from the VALID k x k stride-k convolution of LN(x)
    const T* a = p.norm(l.global_norm);
    T* Q = arena.get<T>(static_cast<size_t>(M) * I);
    linear<T>(a, dp, M, l.to_q, Q, I, p.folded_epi(l.to_q), s);
    const int k = S.global_k, kh = (H - k) / k + 1, kw = (Wd - k) / k + 1, Mk = B * kh * kw;
    UnfoldMode um;                                                    // bf16: the LayerNorm applied on load
    um.valid = true;
    if (p.Y == nullptr) { um.stats = stats; um.parts = dp / 64; um.d = d; um.eps = 1e-5f; um.gamma = l.global_norm.gamma; um.beta = l.global_norm.beta; }
    T* KV = arena.get<T>(static_cast<size_t>(Mk) * 2 * I);
    conv<T>(nullptr, a, dp, B, H, Wd, d, k, k, l.to_kv, KV, nullptr, s, &um);
    attention_dispatch<T>(Q, I, KV, 2 * I, KV + I, 2 * I, O, I, B, H * Wd, kh * kw, I / 64, 64, 0, nullptr, nullptr, nullptr, nullptr, s);
    p.residual(O, I, l.global_out);
    p.mlp(l.ff2);
  }

  // CrossFormer.call (crossformer.py:263-269): per stage, CrossEmbedLayer -> Transformer; then the mean over the map -> Dense.
  // Token rows are the NHWC map, pixel-major, channel widths zero-padded to channel_width; no stage permutes its map (the windowed
  // attention reads and writes the map's own rows).  bf16: `stats` holds the (sum, sumsq) partials of X's rows between sub-blocks
  // (emitted by the embedding's and the residual GEMMs' epilogues).
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
      X = arena.get<T>(static_cast<size_t>(M) * S.dp);
      float* stats = row_stats(M, S.dp);
      conv<T>(img, map, ld_in, B, mh, mw, mc, S.kmax, S.stride, S.embed, X, stats, s);
      for (const CrossformerLayerW& l : S.layers) crossformer_layer<T>(X, B, oh, ow, S, l, stats, s);
      map = X; mh = oh; mw = ow; mc = S.dim; ld_in = S.dp;
    }
    const int dl = cf.dim[VB_CROSSFORMER_STAGES - 1];
    dense_head(mean_pool<T>(X, mh * mw, ld_in, dl, B, s), dl, head, B, logits, s);   // Reduce('b h w c -> b c', 'mean') crossformer.py:259
  }
  // One Transformer layer (crossformer.py:198-202) in place on X [B*H*W, dp].  bf16: the LayerNorms folded into q|k|v and fc1 (from
  // `stats`); fp32: separate LayerNorms.
  template <typename T>
  void crossformer_layer(T* X, int B, int H, int Wd, const CrossformerStageW& S, const CrossformerLayerW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, M = B * H * Wd, I = 32 * S.heads;
    const PreNorm<T> p = prenorm<T>(X, M, d, dp, stats, 1e-5f, s);   // the MLPs: crossformer.py:89-102
    auto attend = [&](const CrossformerAttnW& at) {                   // crossformer.py:133-180
      const T* a = p.norm(at.norm);
      const int ld = at.qkv.N;
      T* QKV = arena.get<T>(static_cast<size_t>(M) * ld);
      linear<T>(a, dp, M, at.qkv, QKV, ld, p.folded_epi(at.qkv), s);
      if (at.wsz > 1) {                                               // wsz == 1: the output is v itself, which QKV holds
        Window win;
        win.p = at.wsz; win.nx = Wd / at.wsz; win.ny = H / at.wsz; win.dilated = at.dilated;
        PosBias pb;
        pb.table = at.table; pb.wsz = at.wsz;
        const int n = at.wsz * at.wsz;
        attention_dispatch<T>(QKV, ld, QKV + I, ld, QKV + 2 * I, ld, QKV, ld, B * win.nx * win.ny, n, n, S.heads, 32, 0, nullptr, nullptr,
                              nullptr, nullptr, s, 0.f, &win, &pb);
      }
      p.residual(QKV, ld, at.to_out);                                 // to_out reads the I output (or v) columns
    };
    attend(l.short_attn);
    p.mlp(l.ff1);
    attend(l.long_attn);
    p.mlp(l.ff2);
  }

  // NesT.call (nest.py:202-216): the patch embedding, then per level the position add, the Transformer within blocks and the
  // Aggregate; then the head's LayerNorm per pixel, the mean over the map and the Dense.  Token rows are the NHWC map, pixel-major,
  // channel widths zero-padded to channel_width; no level permutes its map (the block attention reads and writes the map's own
  // rows).  The position scalar is added by the kernel that last wrote the rows: a small pass after the patch embedding at level
  // 0, the aggregation tail of the level below otherwise.  bf16: `stats` holds the (sum, sumsq) partials of X's rows between
  // sub-blocks (emitted by those kernels and the residual GEMMs' epilogues).
  // The reference's shape rules (nest.py:179,140-142,209 through einops, and the head LayerNorm's broadcast), checked before
  // anything runs.
  void nest_check_size(int H, int Wd) const {
    const int p = ns.patch_size;
    VB_CHECK(H % p == 0 && Wd % p == 0, "NesT: the " + std::to_string(H) + " x " + std::to_string(Wd) +
                                          " image is not divisible by patch_size " + std::to_string(p));
    int h = H / p, w = Wd / p;
    for (int i = 0; i < ns.levels; ++i) {
      const int bs = 1 << (ns.levels - 1 - i);
      const std::string where = "NesT level " + std::to_string(i) + ": the " + std::to_string(h) + " x " + std::to_string(w) + " map ";
      VB_CHECK(h % bs == 0 && w % bs == 0, where + "is not divisible into " + std::to_string(bs) + " x " + std::to_string(bs) + " blocks");
      VB_CHECK(static_cast<long long>(h / bs) * (w / bs) <= ns.seq_len,
               where + "has blocks of " + std::to_string(h / bs) + " x " + std::to_string(w / bs) + " tokens, more than seq_len " +
                   std::to_string(ns.seq_len) + " positions");
      if (nest_aggregates(i)) { h = (h + 1) / 2; w = (w + 1) / 2; }
    }
    VB_CHECK(nest_final_dim() == nest_last_dim(),
             "NesT: the last map has " + std::to_string(nest_final_dim()) + " channels but the head's LayerNorm has " +
                 std::to_string(nest_last_dim()) + " (block_repeats has fewer than num_hierarchies - 1 entries)");
  }
  template <typename T>
  void nest_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    nest_check_size(H, Wd);
    int mh = H / ns.patch_size, mw = Wd / ns.patch_size, d = ns.dim, dp = channel_width(ns.dim);
    const int M0 = B * mh * mw;
    T* X = arena.get<T>(static_cast<size_t>(M0) * dp);
    float* stats = row_stats(M0, dp);
    conv<T>(img, nullptr, 0, B, H, Wd, cfg.channels, ns.patch_size, ns.patch_size, nest_patch, X, nullptr, s);
    for (size_t i = 0; i < nest_levels.size(); ++i) {
      const NestLevelW& V = nest_levels[i];
      const int M = B * mh * mw;
      if (i == 0) {                                                   // x + pos_emb (nest.py:140-142), in place, and the row statistics
        ProfScope ps(this, PROF_OTHER, 1.0 * M * V.dim, 2.0 * sizeof(T) * M * dp, s);
        nest_pool<T>(X, dp, nullptr, B, mh, mw, V.dim, false, V.pos, mh / V.bs, mw / V.bs, X, dp, stats, s);
      }
      for (const NestBlockW& b : V.blocks) nest_block<T>(X, B, mh, mw, V, b, stats, s);
      if (!V.aggregate) continue;
      // Aggregate (nest.py:111-123): the 3 x 3 SAME convolution as unfold_same + GEMM with the conv rows' statistics, then one pass
      // for the LayerNorm, the max-pool and the next level's position add
      T* Y = arena.get<T>(static_cast<size_t>(M) * V.dp_out);
      float* ystats = row_stats(M, V.dp_out);
      conv<T>(nullptr, X, dp, B, mh, mw, V.dim, 3, 1, V.agg, Y, ystats, s);
      const NestLevelW* next = i + 1 < nest_levels.size() ? &nest_levels[i + 1] : nullptr;
      const int oh = (mh + 1) / 2, ow = (mw + 1) / 2, Mo = B * oh * ow;
      T* Xn = arena.get<T>(static_cast<size_t>(Mo) * V.dp_out);
      float* nstats = row_stats(Mo, V.dp_out);
      nest_aggregate_tail<T>(Y, ystats, B, mh, mw, V.dim_out, V.dp_out, V.agg_norm, next ? next->pos : nullptr, next ? oh / next->bs : 1,
                             next ? ow / next->bs : 1, Xn, nstats, s);
      X = Xn; stats = nstats; mh = oh; mw = ow; d = V.dim_out; dp = V.dp_out;
    }
    if (!nest_levels.empty() && !nest_levels.back().aggregate) { d = nest_levels.back().dim; dp = nest_levels.back().dp; }
    // mlp_head (nest.py:196-200): LayerNorm(last_dim) per pixel, the mean over the map, Dense
    const int M = B * mh * mw;
    T* Y = arena.get<T>(static_cast<size_t>(M) * dp);
    float* z = arena.get<float>(static_cast<size_t>(B) * d);
    {
      ProfScope ps(this, PROF_LN, 9.0 * M * d, static_cast<double>(sizeof(T)) * 3.0 * M * dp, s);
      layernorm<T>(X, dp, head_norm.gamma, head_norm.beta, Y, dp, M, d, s, dp, 1e-5f);
      pool_layernorm<T>(Y, mh * mw, dp, nullptr, nullptr, z, B, d, 1, s);
    }
    dense_head(z, d, head, B, logits, s);
  }
  // Aggregate's tail (nest.py:117-123) on Y [B h w, dp], the convolution's output of true width d: the LayerNorm `norm` (bf16: applied
  // on load from Y's row statistics ystats), then MaxPool2D(3, 2, SAME) with the next level's position add (pos, may be null, over
  // pbh x pbw blocks) -> Xn [B ceil(h / 2) ceil(w / 2), dp] and, bf16, its row statistics nstats
  template <typename T>
  void nest_aggregate_tail(const T* Y, const float* ystats, int B, int h, int w, int d, int dp, const Norm& norm, const float* pos, int pbh,
                           int pbw, T* Xn, float* nstats, cudaStream_t s) {
    const int M = B * h * w, Mo = B * ((h + 1) / 2) * ((w + 1) / 2);
    const T* src = Y;
    NestPoolLn ln;
    if (bf16()) {
      ln.stats = ystats; ln.parts = dp / 64; ln.d = d; ln.eps = 1e-5f; ln.gamma = norm.gamma; ln.beta = norm.beta;
    } else {
      T* Z = arena.get<T>(static_cast<size_t>(M) * dp);
      ProfScope ps(this, PROF_LN, 8.0 * M * d, 2.0 * sizeof(T) * M * dp, s);
      layernorm<T>(Y, dp, norm.gamma, norm.beta, Z, dp, M, d, s, dp, 1e-5f);
      src = Z;
    }
    ProfScope ps(this, PROF_OTHER, 9.0 * Mo * d, static_cast<double>(sizeof(T)) * (static_cast<double>(M) + Mo) * dp, s);
    nest_pool<T>(src, dp, bf16() ? &ln : nullptr, B, h, w, d, true, pos, pbh, pbw, Xn, dp, nstats, s);
  }
  // One Transformer block (nest.py:144-146) in place on X [B*H*W, dp]: attention within the level's bs x bs blocks per map, then
  // the MLP.  bf16: the LayerNorms folded into q|k|v and fc1 (from `stats`); fp32: separate LayerNorms.
  template <typename T>
  void nest_block(T* X, int B, int H, int Wd, const NestLevelW& V, const NestBlockW& l, float* stats, cudaStream_t s) {
    const int dp = V.dp, d = V.dim, M = B * H * Wd;
    const PreNorm<T> p = prenorm<T>(X, M, d, dp, stats, 1e-5f, s);
    const T* a = p.norm(l.attn_norm);                                 // Attention nest.py:93-109
    const int ld = l.qkv.N;
    T* QKV = arena.get<T>(static_cast<size_t>(M) * ld);
    linear<T>(a, dp, M, l.qkv, QKV, ld, p.folded_epi(l.qkv), s);
    Window win;
    win.p = H / V.bs; win.pw = Wd / V.bs; win.nx = V.bs; win.ny = V.bs; win.count = B * V.bs * V.bs;
    block_attention<T>(QKV, ld, QKV, ld, V.heads, V.dh, win, s);      // the output overwrites q
    p.residual(QKV, ld, l.to_out);
    p.mlp(l.ff);                                                      // MLP nest.py:61-75
  }
  // NesT's block attention and MobileViT's patch-position attention: win.count blocks of p x width() tokens of fused q|k|v rows
  // [.., ld], the output rows written to out [.., ldo] pixel-major; scale <= 0: dh^-0.5.  The windowed flash kernel where it serves
  // (bf16, dh 32 or 64), else window_attention_generic.
  template <typename T>
  void block_attention(const T* qkv, int ld, T* out, int ldo, int heads, int dh, const Window& win, cudaStream_t s, float scale = 0.f) {
    const int n = win.p * win.width();
    {
      ProfScope ps(this, PROF_ATTN, 4.0 * win.count * heads * n * n * dh, static_cast<double>(sizeof(T)) * win.count * heads * dh * 4.0 * n, s);
      if (block_attention_fast(qkv, ld, out, ldo, heads, dh, s, win, scale)) return;
    }
    window_attention_generic<T>(qkv, ld, out, ldo, win.count, n, heads, dh, win, nullptr, s, scale);
  }
  // Windowed attention off the flash kernel: B windows of n tokens of fused q|k|v rows [.., ld] (win's layout, with the window
  // bias pb when given) permuted to window-major order, the materialised-scores path, the output rows permuted back to out [.., ldo]
  template <typename T>
  void window_attention_generic(const T* qkv, int ld, T* out, int ldo, int B, int n, int heads, int dh, const Window& win, const PosBias* pb,
                                cudaStream_t s, float scale = 0.f) {
    const int HD = heads * dh;
    const long long rows = static_cast<long long>(B) * n;
    T* qkvw = arena.get<T>(static_cast<size_t>(rows) * 3 * HD);
    T* ow = arena.get<T>(static_cast<size_t>(rows) * HD);
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * 3 * HD, s); window_rows<T>(qkv, ld, qkvw, 3 * HD, 3 * HD, win, rows, true, s); }
    {
      ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * n * n * dh, static_cast<double>(sizeof(T)) * B * heads * dh * 4.0 * n, s);
      float* S = arena.get<float>(static_cast<size_t>(B) * heads * n * ((n + 15) & ~15));
      attention_generic<T>(qkvw, 3 * HD, qkvw + HD, 3 * HD, qkvw + 2 * HD, 3 * HD, ow, HD, S, B, n, n, heads, dh, 0, nullptr, nullptr, nullptr,
                           nullptr, s, scale, pb);
    }
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * HD, s); window_rows<T>(ow, HD, out, ldo, HD, win, rows, false, s); }
  }

  // MobileViT.call (mobile_vit.py:260-271): conv1, the stem, per trunk stage an MV2 block and a MobileViTBlock, then to_logits.
  // Token rows are the NHWC map, pixel-major, channel widths zero-padded to channel_width.  Every SAME stride gives ceil; the
  // reference's regrouping (:196) needs every trunk map divisible by (ph, pw), checked before anything runs.
  void mvit_check_size(int H, int Wd) const {
    int h = (H + 3) / 4, w = (Wd + 3) / 4;                              // conv1 and stem block 1: stride 2 each
    for (int s = 0; s < 3; ++s) {
      h = (h + 1) / 2; w = (w + 1) / 2;
      VB_CHECK(h % mv.ph == 0 && w % mv.pw == 0,
               "MobileViT stage " + std::to_string(s + 1) + ": the " + std::to_string(h) + " x " + std::to_string(w) + " map is not divisible by "
               "patch_size (" + std::to_string(mv.ph) + ", " + std::to_string(mv.pw) + "); every trunk map (1/8, 1/16 and 1/32 of the "
               "image, rounded up) must be");
    }
  }
  template <typename T>
  void mobilevit_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    mvit_check_size(H, Wd);
    int h = (H + 1) / 2, w = (Wd + 1) / 2, ld = mv_conv1.N;
    T* X = arena.get<T>(static_cast<size_t>(B) * h * w * ld);
    conv<T>(img, nullptr, 0, B, H, Wd, cfg.channels, 3, 2, mv_conv1, X, nullptr, s, nullptr, ACT_SILU);   // conv1 (:230)
    for (int i = 0; i < 4; ++i) {                                         // stem (:232-236)
      const Mv2W& m = mv_mv2[i];
      X = mv2_block<T>(X, ld, B, h, w, m, nullptr, 0, s);
      h = (h + m.stride - 1) / m.stride; w = (w + m.stride - 1) / m.stride; ld = m.cp_out;
    }
    for (int st = 0; st < 3; ++st) {
      const Mv2W& m = mv_mv2[4 + st];
      const MvitBlockW& v = mv_vit[st];
      const int oh = (h + 1) / 2, ow = (w + 1) / 2, ldc = v.chp + v.cp_in;
      T* Cat = arena.get<T>(static_cast<size_t>(B) * oh * ow * ldc);      // [conv3 out | y]: the MV2 block writes y, the block's input
      mv2_block<T>(X, ld, B, h, w, m, Cat + v.chp, ldc, s);
      X = mobilevit_block<T>(Cat, B, oh, ow, v, s);
      h = oh; w = ow; ld = v.chp;
    }
    const int M = B * h * w;
    T* Y = arena.get<T>(static_cast<size_t>(M) * mv_logits.N);
    Epi e; e.bias = mv_logits.bias; e.silu = true;
    linear<T>(X, ld, M, mv_logits, Y, mv_logits.N, e, s);               // to_logits.0 (:255)
    dense_head(mean_pool<T>(Y, h * w, mv_logits.N, mv.last_dim, B, s), mv.last_dim, head, B, logits, s);   // Reduce, Dense (:256-257)
  }
  // One MV2Block (mobile_vit.py:166-170) on X [B*h*w, ldx] -> out [B*oh*ow, ldo] (a new buffer when out is null)
  template <typename T>
  T* mv2_block(const T* X, int ldx, int B, int h, int w, const Mv2W& m, T* out, int ldo, cudaStream_t s) {
    const int oh = (h + m.stride - 1) / m.stride, ow = (w + m.stride - 1) / m.stride, M = B * h * w, Mo = B * oh * ow;
    const T* a = X;
    int lda = ldx;
    if (m.expand) {
      T* E = arena.get<T>(static_cast<size_t>(M) * m.hp);
      Epi e; e.bias = m.pw1.bias; e.silu = true;
      linear<T>(X, ldx, M, m.pw1, E, m.hp, e, s);
      a = E; lda = m.hp;
    }
    T* D = arena.get<T>(static_cast<size_t>(Mo) * m.hp);
    {
      ProfScope ps(this, PROF_OTHER, 20.0 * Mo * m.hidden, static_cast<double>(sizeof(T)) * (static_cast<double>(M) * m.hidden + static_cast<double>(Mo) * m.hp), s);
      dwconv_bn_act<T>(a, lda, m.dw_w, m.dw_b, D, m.hp, B, h, w, m.hidden, m.hp, m.stride, s);
    }
    if (out == nullptr) { out = arena.get<T>(static_cast<size_t>(Mo) * m.cp_out); ldo = m.cp_out; }
    Epi e2; e2.bias = m.pw2.bias;
    if (m.residual) { e2.res = X; e2.ldr = ldx; }
    linear<T>(D, m.hp, Mo, m.pw2, out, ldo, e2, s);
    return out;
  }
  // One MobileViTBlock (mobile_vit.py:187-206) on Cat [B*h*w, chp + cp_in] whose right half holds its input y -> a new [B*h*w, chp]
  template <typename T>
  T* mobilevit_block(T* Cat, int B, int h, int w, const MvitBlockW& v, cudaStream_t s) {
    const int ldc = v.chp + v.cp_in, M = B * h * w, dh = mvit_dh(), ld = 3 * kMvHeads * dh;
    T* Y1 = arena.get<T>(static_cast<size_t>(M) * v.chp);
    conv<T>(nullptr, Cat + v.chp, ldc, B, h, w, v.cin, v.k, 1, v.conv1, Y1, nullptr, s, nullptr, ACT_SILU);
    T* X = arena.get<T>(static_cast<size_t>(M) * v.dp);
    float* stats = row_stats(M, v.dp);
    Epi e2; e2.bias = v.conv2.bias; e2.silu = true; e2.stats_out = stats;
    linear<T>(Y1, v.chp, M, v.conv2, X, v.dp, e2, s);
    // 'b (h ph) (w pw) d -> b (ph pw) (h w) d': the pixels of one patch position are a dilated h/ph x w/pw window of the map
    Window win;
    win.p = h / mv.ph; win.pw = w / mv.pw; win.ny = mv.ph; win.nx = mv.pw; win.dilated = 1; win.count = B * mv.ph * mv.pw;
    const float scale = 1.0f / sqrtf(static_cast<float>(kMvDh));
    for (const MvitLayerW& l : v.layers) {
      const PreNorm<T> p = prenorm<T>(X, M, v.dim, v.dp, stats, 1e-3f, s);
      const T* a = p.norm(l.attn_norm);
      T* QKV = arena.get<T>(static_cast<size_t>(M) * ld);
      linear<T>(a, v.dp, M, l.qkv, QKV, ld, p.folded_epi(l.qkv), s);
      block_attention<T>(QKV, ld, QKV, ld, kMvHeads, dh, win, s, scale);   // the output overwrites q
      p.residual(QKV, ld, l.to_out);
      p.mlp(l.ff);
    }
    Epi e3; e3.bias = v.conv3.bias; e3.silu = true;
    linear<T>(X, v.dp, M, v.conv3, Cat, ldc, e3, s);                     // the concat's left half
    T* out = arena.get<T>(static_cast<size_t>(M) * v.chp);
    conv<T>(nullptr, Cat, ldc, B, h, w, ldc, v.k, 1, v.conv4, out, nullptr, s, nullptr, ACT_SILU);
    return out;
  }

  // ScalableViT.call (scalable_vit.py:308-319): to_patches, per stage the Transformer (its blocks, then its LayerNorm) and the
  // Downsample, then the mean over the map, LayerNormalization and Dense.  Token rows are the NHWC map, pixel-major, channel widths
  // zero-padded to channel_width; no step permutes the map (the windowed attention reads and writes the map's own rows).  bf16:
  // `stats` holds the (sum, sumsq) partials of X's rows between sub-blocks (emitted by to_patches', the Downsample's and the
  // residual GEMMs' epilogues, and after the PEG by a row-statistics pass).
  // The reference's shape rules, checked before anything runs: the SSA's VALID r x r convolution needs a map of at least r on each
  // side, and IWSA asserts that its window divides the map (:171).  The SAME stride-4 stem and stride-2 Downsamples give ceil.
  void svit_check_size(int H, int Wd) const {
    int h = (H + 3) / 4, w = (Wd + 3) / 4;
    for (int st = 0; st < sv.num_stages; ++st) {
      if (st > 0) { h = (h + 1) / 2; w = (w + 1) / 2; }
      if (sv.depth[st] == 0) continue;
      const int r = sv.reduction_factor[st], wh = sv.window[st] > 0 ? sv.window[st] : h, ww = sv.window[st] > 0 ? sv.window[st] : w;
      const std::string where = "ScalableViT stage " + std::to_string(st + 1) + ": ";
      VB_CHECK(h >= r && w >= r, where + "the " + std::to_string(h) + " x " + std::to_string(w) + " map is smaller than reduction_factor " +
                                     std::to_string(r) + " (a VALID convolution)");
      VB_CHECK(h % wh == 0 && w % ww == 0, where + "height (" + std::to_string(h) + ") or width (" + std::to_string(w) +
                                               ") of feature map is not divisible by the window size (" + std::to_string(wh) + ", " +
                                               std::to_string(ww) + ")");
    }
  }
  template <typename T>
  void svit_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    svit_check_size(H, Wd);
    int h = (H + 3) / 4, w = (Wd + 3) / 4;
    T* X = arena.get<T>(static_cast<size_t>(B) * h * w * sv_stages[0].dp);
    float* stats = row_stats(static_cast<long long>(B) * h * w, sv_stages[0].dp);
    conv<T>(img, nullptr, 0, B, H, Wd, cfg.channels, 7, 4, sv_stem, X, stats, s);       // to_patches (:310)
    for (const SvitStageW& S : sv_stages) {
      const int M = B * h * w;
      for (const SvitBlockW& l : S.blocks) X = svit_block<T>(X, B, h, w, S, l, stats, s);
      const PreNorm<T> p = prenorm<T>(X, M, S.dim, S.dp, stats, 1e-5f, s);
      if (!S.down) {                                                   // the last stage's LayerNorm, the mean, mlp_head (:302-306)
        const T* a = p.norm(S.norm);
        if (p.Y == nullptr) {
          T* Y = arena.get<T>(static_cast<size_t>(M) * S.dp);
          ProfScope ps(this, PROF_LN, 8.0 * M * S.dim, 2.0 * sizeof(T) * M * S.dp, s);
          layernorm<T>(X, S.dp, S.norm.gamma, S.norm.beta, Y, S.dp, M, S.dim, s, S.dp, 1e-5f);
          a = Y;
        }
        float* z = arena.get<float>(static_cast<size_t>(B) * S.dim);
        {
          ProfScope ps(this, PROF_LN, 2.0 * M * S.dim, static_cast<double>(sizeof(T)) * M * S.dp, s);
          pool_layernorm<T>(a, h * w, S.dp, head_norm.gamma, head_norm.beta, z, B, S.dim, 1, s);
        }
        dense_head(z, S.dim, head, B, logits, s);
        return;
      }
      // Downsample (:71-78) of the Transformer's LayerNorm output: bf16 applies that LayerNorm on load from the row statistics
      UnfoldMode um;
      um.stats = stats; um.parts = S.dp / 64; um.d = S.dim; um.eps = 1e-5f; um.gamma = S.norm.gamma; um.beta = S.norm.beta;
      const T* a = p.norm(S.norm);
      const int oh = (h + 1) / 2, ow = (w + 1) / 2, dpn = S.down_conv.N;
      T* Xn = arena.get<T>(static_cast<size_t>(B) * oh * ow * dpn);
      stats = row_stats(static_cast<long long>(B) * oh * ow, dpn);
      conv<T>(nullptr, a, S.dp, B, h, w, S.dim, 3, 2, S.down_conv, Xn, stats, s, p.Y == nullptr ? &um : nullptr);
      X = Xn; h = oh; w = ow;
    }
  }
  // One block (scalable_vit.py:237-245) on X [B*h*w, dp]; returns the block's output rows (a new buffer after the PEG).  bf16: the
  // LayerNorms folded into the SSA q, the MLPs' fc1 and the IWSA q|k|v (from `stats`), and applied on load by the SSA's k|v unfold;
  // fp32: separate LayerNorms.
  template <typename T>
  T* svit_block(T* X, int B, int h, int w, const SvitStageW& S, const SvitBlockW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, M = B * h * w, HS = S.heads * S.dhs, HI = S.heads * S.dhi;
    const PreNorm<T> p0 = prenorm<T>(X, M, d, dp, stats, 1e-5f, s);
    {                                                                 // ScalableSelfAttention (:121-143)
      const T* a = p0.norm(l.ssa_norm);
      T* Q = arena.get<T>(static_cast<size_t>(M) * S.ldq);
      linear<T>(a, dp, M, l.ssa_q, Q, S.ldq, p0.folded_epi(l.ssa_q), s);
      const int kh = h / S.r, kw = w / S.r;
      UnfoldMode um;                                                  // to_k | to_v: the VALID r x r stride-r convolution
      um.valid = true;
      if (p0.Y == nullptr) { um.stats = stats; um.parts = dp / 64; um.d = d; um.eps = 1e-5f; um.gamma = l.ssa_norm.gamma; um.beta = l.ssa_norm.beta; }
      T* KV = arena.get<T>(static_cast<size_t>(B) * kh * kw * S.ldkv);
      conv<T>(nullptr, a, dp, B, h, w, d, S.r, S.r, l.ssa_kv, KV, nullptr, s, &um);
      attention_dispatch<T>(Q, S.ldq, KV, S.ldkv, KV + HS, S.ldkv, Q, S.ldq, B, h * w, kh * kw, S.heads, S.dhs, 0, nullptr, nullptr, nullptr,
                            nullptr, s, S.ssa_scale);               // the output overwrites q
      p0.residual(Q, S.ldq, l.ssa_out);
    }
    p0.mlp(l.mlp1);
    if (l.peg_w != nullptr) {                                         // PEG (:85-87), the residual folded into the centre tap
      T* Y = arena.get<T>(static_cast<size_t>(M) * dp);               // the halo reads the unmodified map
      {
        ProfScope ps(this, PROF_OTHER, 18.0 * M * d, 2.0 * sizeof(T) * M * dp, s);
        dwconv_qkv<T>(X, dp, nullptr, nullptr, nullptr, d, 1e-5f, l.peg_w, l.peg_b, Y, dp, nullptr, nullptr, nullptr, dp, B, h, w, dp, 3, 1, s);
      }
      X = Y;
      if (bf16()) ensure_stats<T>(X, dp, stats, M, s);
    }
    const PreNorm<T> p = p0.rows(X, M, stats);
    p.mlp(l.mlp3);
    {                                                                 // InteractiveWindowedSelfAttention (:165-198)
      const T* a = p.norm(l.iwsa_norm);
      T* QKV = arena.get<T>(static_cast<size_t>(M) * S.ldqkv);
      linear<T>(a, dp, M, l.iwsa_qkv, QKV, S.ldqkv, p.folded_epi(l.iwsa_qkv), s);
      Window win;                                                     // window 0 (None): one window per image
      win.p = S.window > 0 ? S.window : h; win.pw = S.window > 0 ? S.window : w;
      win.ny = h / win.p; win.nx = w / win.pw; win.count = B * win.nx * win.ny;
      block_attention<T>(QKV, S.ldqkv, QKV, S.ldqkv, S.heads, S.dhi, win, s, S.iwsa_scale);   // the output overwrites q
      // LIM(v) + the attention output: the 3x3 convolution over v's columns of the same rows, the output as its residual
      T* LO = arena.get<T>(static_cast<size_t>(M) * S.ldlim);
      conv<T>(nullptr, QKV + 2 * HI, S.ldqkv, B, h, w, HI, 3, 1, l.lim, LO, nullptr, s, nullptr, ACT_NONE, QKV, S.ldqkv);
      p.residual(LO, S.ldlim, l.iwsa_out);
    }
    return X;
  }

  // RegionViT.call (regionvit.py:249-263): the local and region encoders, then per stage the shared Downsample of both maps, the
  // PEG of the local map and the R2L layers; then the mean over the regional tokens, LayerNorm and Dense.  Each stage keeps its
  // local rows (the pixel-major B x lh x lw map) followed by its regional rows (the B x rh x rw map) in one arena, so every
  // token-wise step is one launch over both; the R2L attention reads and writes both in place.  Channel widths are zero-padded to
  // channel_width.  bf16: `stats` holds the (sum, sumsq) partials of all rows between sub-blocks, pitch M.
  // The reference's shape rules (the call-time asserts :251-252, the window rearranges and concat :163-168, the bias Embedding
  // :153), checked before anything runs.  The local encoder's SAME stride 4 (or two SAME stride 2) gives ceil(H / 4).
  void rv_check_size(int H, int Wd) const {
    const int p = rv_region_patch(), lp = rv.local_patch_size, ws = rv.window_size;
    VB_CHECK(H % p == 0 && Wd % p == 0, "height and width must be divisible by region patch size");
    VB_CHECK(H % lp == 0 && Wd % lp == 0, "height and width must be divisible by local patch size");
    int lh = (H + 3) / 4, lw = (Wd + 3) / 4, rh = H / p, rw = Wd / p;
    for (int s = 0; s < VB_REGIONVIT_STAGES; ++s) {
      if (s > 0) { lh = (lh + 1) / 2; lw = (lw + 1) / 2; rh = (rh + 1) / 2; rw = (rw + 1) / 2; }
      const std::string where = "RegionViT stage " + std::to_string(s + 1) + ": the " + std::to_string(lh) + " x " + std::to_string(lw) +
                                " local map and the " + std::to_string(rh) + " x " + std::to_string(rw) + " region map ";
      VB_CHECK(lh >= rh && lw >= rw && lh % rh == 0 && lw % rw == 0,
               where + "do not make whole windows (the local map must be the region map times the window)");
      VB_CHECK(lh / rh <= ws && lw / rw <= ws, where + "make " + std::to_string(lh / rh) + " x " + std::to_string(lw / rw) +
                                                   " windows, larger than window_size " + std::to_string(ws) +
                                                   " (the relative-position table's reach)");
    }
  }
  // The row statistics of the regional rows at pitch M, after their own residual update (bf16; the fp32 engine keeps none).
  template <typename T>
  void rv_region_stats(const T* Xr, int dp, float* stats, int Mr, long long pitch, cudaStream_t s) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
      ProfScope ps(this, PROF_LN, 0.0, 2.0 * Mr * dp, s);
      row_stats_bf16(Xr, dp, stats, Mr, dp, s, pitch);
    }
  }
  template <typename T>
  void regionvit_forward(const float* img, int B, int H, int Wd, float* logits, cudaStream_t s) {
    rv_check_size(H, Wd);
    const int C = cfg.channels, p = rv_region_patch();
    int lh = (H + 3) / 4, lw = (Wd + 3) / 4, rh = H / p, rw = Wd / p;
    int Ml = B * lh * lw, Mr = B * rh * rw, M = Ml + Mr, d = rv.dims[0], dp = rv_stages[0].dp;
    T* X = arena.get<T>(static_cast<size_t>(M) * dp);
    float* stats = row_stats(M, dp);
    if (rv.tokenize_local_3_conv) {                                  // regionvit.py:211-218: the LayerNorm + GELU applied on load
      int h = H, w = Wd;
      const T* src = nullptr;
      for (int i = 0; i < 3; ++i) {
        const int stride = i < 2 ? 2 : 1, oh = (h + stride - 1) / stride, ow = (w + stride - 1) / stride, rows = B * oh * ow;
        UnfoldMode um;
        um.gelu = true;
        if (i > 0 && bf16()) {
          um.stats = stats; um.parts = dp / 64; um.d = d; um.eps = 1e-3f; um.gamma = rv_local_norm[i - 1].gamma; um.beta = rv_local_norm[i - 1].beta;
        } else if (i > 0) {
          T* Z = arena.get<T>(static_cast<size_t>(B) * h * w * dp);
          ProfScope ps(this, PROF_LN, 8.0 * B * h * w * d, 2.0 * sizeof(T) * B * h * w * dp, s);
          layernorm<T>(src, dp, rv_local_norm[i - 1].gamma, rv_local_norm[i - 1].beta, Z, dp, B * h * w, d, s, dp, 1e-3f);
          src = Z;
        }
        T* out = i == 2 ? X : arena.get<T>(static_cast<size_t>(rows) * dp);
        float* st = i < 2 ? row_stats(rows, dp) : nullptr;
        conv<T>(img, src, dp, B, h, w, i == 0 ? C : d, 3, stride, rv_local[i], out, st, s, i > 0 ? &um : nullptr);
        src = out; h = oh; w = ow;
        if (st != nullptr) stats = st;                               // the next unfold's LayerNorm statistics
      }
      stats = row_stats(M, dp);
    } else {
      conv<T>(img, nullptr, 0, B, H, Wd, C, 8, 4, rv_local[0], X, nullptr, s);   // :221
    }
    conv<T>(img, nullptr, 0, B, H, Wd, C, p, p, rv_region, X + static_cast<size_t>(Ml) * dp, nullptr, s);   // :223-226
    if (bf16()) ensure_stats<T>(X, dp, stats, M, s);
    for (const RegionStageW& S : rv_stages) {
      if (S.down) {          // :258: one Conv2D(3, 2, SAME) for both maps, both unfolded into one column buffer, one GEMM
        const int olh = (lh + 1) / 2, olw = (lw + 1) / 2, orh = (rh + 1) / 2, orw = (rw + 1) / 2;
        const int nMl = B * olh * olw, nMr = B * orh * orw, nM = nMl + nMr, Kp = bf16() ? S.down_conv.ldw : S.down_conv.K;
        T* col = arena.get<T>(static_cast<size_t>(nM) * Kp);
        {
          ProfScope ps(this, PROF_EMBED, 0.0, static_cast<double>(sizeof(T)) * (static_cast<double>(M) * dp + static_cast<double>(nM) * Kp), s);
          unfold_same<T, T>(X, col, B, lh, lw, d, 3, 2, 0, Kp, s, dp);
          unfold_same<T, T>(X + static_cast<size_t>(Ml) * dp, col + static_cast<size_t>(nMl) * Kp, B, rh, rw, d, 3, 2, 0, Kp, s, dp);
        }
        T* Xn = arena.get<T>(static_cast<size_t>(nM) * S.dp);
        stats = row_stats(nM, S.dp);
        Linear L = S.down_conv;
        L.K = Kp;
        Epi e; e.bias = S.down_conv.bias; e.stats_out = S.peg ? nullptr : stats;
        linear<T>(col, Kp, nM, L, Xn, S.dp, e, s);
        X = Xn; lh = olh; lw = olw; rh = orh; rw = orw; Ml = nMl; Mr = nMr; M = nM; d = S.dim; dp = S.dp;
      }
      if (S.peg) {           // :259: the local map only; the halo reads the unmodified map, so the result goes to a new arena
        T* Y = arena.get<T>(static_cast<size_t>(M) * dp);
        {
          ProfScope ps(this, PROF_OTHER, 18.0 * Ml * d, 2.0 * sizeof(T) * Ml * dp, s);
          dwconv_qkv<T>(X, dp, nullptr, nullptr, nullptr, d, 1e-5f, S.peg_w, S.peg_b, Y, dp, nullptr, nullptr, nullptr, dp, B, lh, lw, dp, 3, 1, s);
        }
        VB_CUDA(cudaMemcpyAsync(Y + static_cast<size_t>(Ml) * dp, X + static_cast<size_t>(Ml) * dp, static_cast<size_t>(Mr) * dp * sizeof(T),
                                cudaMemcpyDeviceToDevice, s));
        X = Y;
        if (bf16()) ensure_stats<T>(X, dp, stats, M, s);
      }
      for (const RegionLayerW& l : S.layers) regionvit_layer<T>(X, B, lh, lw, rh, rw, S, l, stats, s);
    }
    // to_logits (:243-247): the mean over the regional tokens, then LayerNorm, then Dense
    float* z = arena.get<float>(static_cast<size_t>(B) * d);
    {
      ProfScope ps(this, PROF_LN, 1.0 * Mr * d + 8.0 * B * d, static_cast<double>(sizeof(T)) * Mr * dp, s);
      pool_layernorm<T>(X + static_cast<size_t>(Ml) * dp, rh * rw, dp, head_norm.gamma, head_norm.beta, z, B, d, 1, s);
    }
    dense_head(z, d, head, B, logits, s);
  }
  // One R2L layer (regionvit.py:158-172) in place on X [M, dp], M = B lh lw local rows + B rh rw regional rows: the regional
  // self-attention on the regional rows, then the R2L attention and the MLP over all rows.  bf16: the LayerNorms folded into q|k|v
  // and fc1 (from `stats`, and for the regional q|k|v from the regional rows' own statistics at pitch Mr); fp32: separate
  // LayerNorms.
  template <typename T>
  void regionvit_layer(T* X, int B, int lh, int lw, int rh, int rw, const RegionStageW& S, const RegionLayerW& l, float* stats, cudaStream_t s) {
    const int dp = S.dp, d = S.dim, Ml = B * lh * lw, Mr = B * rh * rw, M = Ml + Mr, ld = l.qkv.N;
    T* Xr = X + static_cast<size_t>(Ml) * dp;
    const PreNorm<T> p = prenorm<T>(X, M, d, dp, stats, 1e-3f, s);
    T* QKV = arena.get<T>(static_cast<size_t>(M) * ld);
    // region_tokens = attn(region_tokens) + region_tokens (:159): all rh x rw regional tokens of an image attend together, their
    // LayerNorm folded from the regional rows' own statistics
    float* rstats = row_stats(Mr, dp);
    if (bf16()) rv_region_stats<T>(Xr, dp, rstats, Mr, Mr, s);
    const PreNorm<T> pr = p.rows(Xr, Mr, rstats);
    linear<T>(pr.norm(l.attn_norm), dp, Mr, l.qkv, QKV, ld, pr.folded_epi(l.qkv), s);
    Window rwin;
    rwin.p = rh; rwin.pw = rw; rwin.nx = 1; rwin.ny = 1; rwin.count = B;
    block_attention<T>(QKV, ld, QKV, ld, kRvHeads, kRvDh, rwin, s);     // the output overwrites q
    p.rows(Xr, Mr, nullptr).residual(QKV, ld, l.to_out);               // its statistics: the next pass, at pitch M
    if (bf16()) rv_region_stats<T>(Xr, dp, stats + static_cast<size_t>(Ml) * 2, Mr, M, s);
    // [r; window] = attn([r; window], rel_pos_bias) + [r; window] (:168-169), each window with its regional token
    linear<T>(p.norm(l.attn_norm), dp, M, l.qkv, QKV, ld, p.folded_epi(l.qkv), s);
    Window win;
    win.p = lh / rh; win.pw = lw / rw; win.nx = rw; win.ny = rh; win.count = Mr;
    PosBias pb;
    pb.table = S.table; pb.r2l_ws = rv.window_size; pb.r2l_h = win.p; pb.r2l_w = win.pw;
    r2l_attention<T>(QKV, ld, QKV, ld, Ml, pb, win, s);
    p.residual(QKV, ld, l.to_out);
    p.mlp(l.ff);                                                        // ff(.) + . (:172)
  }
  // RegionViT's R2L attention: win.count windows of p x width() local rows, each with its regional row reg_row0 + (window index),
  // fused q|k|v rows [.., ld], the output rows written in place to out [.., ldo].  The R2L flash kernel where it serves (bf16, dh
  // 32, tables up to its shared-memory size); otherwise the windows gathered window-major with the regional row first, the
  // materialised-scores path with the R2L bias, and the output rows scattered back.
  template <typename T>
  void r2l_attention(const T* qkv, int ld, T* out, int ldo, long long reg_row0, const PosBias& pb, const Window& win, cudaStream_t s,
                     int heads = kRvHeads, int dh = kRvDh) {
    const int n = 1 + win.p * win.width(), HD = heads * dh;
    const long long Bw = win.count, rows = Bw * n;
    const double fl = 4.0 * Bw * heads * n * n * dh, by = static_cast<double>(sizeof(T)) * Bw * heads * dh * 4.0 * n;
    {
      ProfScope ps(this, PROF_ATTN, fl, by, s);
      if (r2l_attention_fast(qkv, ld, out, ldo, heads, dh, reg_row0, pb, win, s)) return;
    }
    T* qkvw = arena.get<T>(static_cast<size_t>(rows) * 3 * HD);
    T* ow = arena.get<T>(static_cast<size_t>(rows) * HD);
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * 3 * HD, s); r2l_rows<T>(qkv, ld, qkvw, 3 * HD, 3 * HD, win, reg_row0, true, s); }
    {
      ProfScope ps(this, PROF_ATTN, fl, by, s);
      float* Sc = arena.get<float>(static_cast<size_t>(Bw) * heads * n * ((n + 15) & ~15));
      attention_generic<T>(qkvw, 3 * HD, qkvw + HD, 3 * HD, qkvw + 2 * HD, 3 * HD, ow, HD, Sc, static_cast<int>(Bw), n, n, heads, dh, 0, nullptr,
                           nullptr, nullptr, nullptr, s, 0.f, &pb);
    }
    { ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * rows * HD, s); r2l_rows<T>(ow, HD, out, ldo, HD, win, reg_row0, false, s); }
  }

  // MAE.call (mae.py:49-92) and SimMIM.call (simmim.py:82-129) as mim_prepare planned them, writing the loss to `loss` (device)
  // and, per `flags` (1: pred, 2: masked_patches), the outputs to mim_pred() / mim_patches().  The masks come from the device's
  // own noise counter; every step after them is a fixed launch sequence.
  template <typename T>
  void mim_forward(const float* img, int B, int H, int Wd, float* loss, int flags, cudaStream_t s) {
    const vb_config& c = cfg;
    const MimPlan& p = mim_last;
    VB_CHECK(p.B == B && p.n == (H / c.patch_h) * (Wd / c.patch_w) && mim_dev.p != nullptr, "internal: MIM state not prepared for this batch");
    arena.reset();
    const bool mae = c.kind == VB_KIND_MAE;
    const int n = p.n, nm = p.nm, nk = n - nm, dim = c.dim, pd = patch_dim(), Dd = mim_dim();
    int* idx = mim_idx();
    {
      ProfScope ps(this, PROF_OTHER, 0.0, 4.0 * B * n, s);
      mim_mask(B, n, mae ? 0 : 1, mim_rng_ptr(), idx, s);
    }
    // the patch embedding of the kept rows (MAE: per row the reference's embed-then-gather) or of all rows (SimMIM)
    const int rows = mae ? nk : n, M = B * rows, Kp = bf16() ? embed.patch.ldw : embed.patch.K;
    T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
    T* R = arena.get<T>(static_cast<size_t>(M) * dim);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, 4.0 * M * pd + static_cast<double>(sizeof(T)) * M * (Kp + dim), s);
      mim_patch_rows<T>(img, B, H, Wd, c.channels, c.patch_h, c.patch_w, mae ? idx : nullptr, n, nm, rows, col, Kp, embed.pos, R, dim, s);
    }
    T* X = arena.get<T>(static_cast<size_t>(M) * dim);
    float* stats = nullptr;
    {
      Epi ep; ep.bias = embed.patch.bias; ep.res = R; ep.ldr = dim;
      if (mae && bf16() && dim % 64 == 0) { stats = row_stats(M, dim); ep.stats_out = stats; }
      Linear L = embed.patch;
      L.K = Kp;
      linear<T>(col, Kp, M, L, X, dim, ep, s);
    }
    if (!mae) {
      ProfScope ps(this, PROF_OTHER, 0.0, static_cast<double>(sizeof(T)) * B * nm * dim, s);
      mim_mask_tokens<T>(X, idx, B, n, nm, mask_token, embed.pos, dim, s);
      stats = dim % 64 == 0 ? row_stats(M, dim) : nullptr;   // recomputed by the first layer: the mask rows replaced the GEMM's
    }
    bool sv = mae && stats != nullptr;
    for (const auto& l : layers) layer_self<T>(X, B, rows, dim, l, s, stats, &sv);
    const T* Xp = X;                                            // the rows to_pixels reads, nm per image
    if (mae) {
      const T* E = X;
      if (enc_to_dec_dense) {
        T* Ed = arena.get<T>(static_cast<size_t>(M) * Dd);
        Epi e; e.bias = enc_to_dec.bias;
        linear<T>(X, dim, M, enc_to_dec, Ed, Dd, e, s);
        E = Ed;
      }
      T* Z = arena.get<T>(static_cast<size_t>(B) * n * Dd);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, static_cast<double>(sizeof(T)) * B * (nk + n) * Dd + 4.0 * B * n * Dd, s);
        mim_decoder_rows<T>(E, idx, B, n, nm, mask_token, dec_pos, Z, Dd, s);
      }
      float* dstats = Dd % 64 == 0 ? row_stats(static_cast<long long>(B) * n, Dd) : nullptr;
      bool dsv = false;
      for (const auto& l : dec_layers) layer_self<T>(Z, B, n, Dd, l, s, dstats, &dsv);
      T* Zm = arena.get<T>(static_cast<size_t>(B) * nm * Dd);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * B * nm * Dd, s);
        mim_take_rows<T>(Z, n, nullptr, Zm, B, nm, Dd, s);   // the mask rows: first in every image (mae.py:84)
      }
      Xp = Zm;
    } else {
      T* Xm = arena.get<T>(static_cast<size_t>(B) * nm * dim);
      {
        ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * B * nm * dim, s);
        mim_take_rows<T>(X, n, idx, Xm, B, nm, dim, s);      // simmim.py:119: the encoded rows at the masked ids, top_k order
      }
      Xp = Xm;
    }
    const long long Mp = static_cast<long long>(B) * nm;
    T* P = arena.get<T>(static_cast<size_t>(Mp) * pd);
    {
      Epi e; e.bias = to_pixels.bias;
      linear<T>(Xp, Dd, static_cast<int>(Mp), to_pixels, P, pd, e, s);
    }
    double* partial = arena.get<double>(static_cast<size_t>(mim_loss_blocks(Mp)));
    {
      ProfScope ps(this, PROF_OTHER, 3.0 * Mp * pd, static_cast<double>(sizeof(T)) * Mp * pd + (mae ? 0.0 : 4.0 * Mp * pd), s);
      mim_loss<T>(P, pd, B, nm, mae ? nullptr : img, H, Wd, c.channels, c.patch_h, c.patch_w, idx, n, partial, loss, s);
    }
    if (flags & 1) {
      ProfScope ps(this, PROF_OTHER, 0.0, (static_cast<double>(sizeof(T)) + 4.0) * Mp * pd, s);
      to_f32<T>(P, mim_pred(), Mp * pd, s);
    }
    if (flags & 2) {
      ProfScope ps(this, PROF_OTHER, 0.0, 8.0 * Mp * pd, s);
      mim_patch_rows<float>(img, B, H, Wd, c.channels, c.patch_h, c.patch_w, idx, n, 0, nm, mim_patches(), pd, nullptr, nullptr, 0, s);
    }
  }

  // MPP.call (mpp.py:168-218) as mim_prepare planned it, writing the loss to `loss` (device) and, when `want_logits`, the logits of
  // the masked rows to mim_pred().  The mask and the corruption draws come from the device's own counter; every step after them is a
  // fixed launch sequence.
  template <typename T>
  void mpp_forward(const float* img, int B, int H, int Wd, float* loss, bool want_logits, cudaStream_t s) {
    const vb_config& c = cfg;
    const MimPlan& p = mim_last;
    VB_CHECK(p.B == B && p.n == (H / c.patch_h) * (Wd / c.patch_w) && mim_dev.p != nullptr, "internal: MPP state not prepared for this batch");
    arena.reset();
    const int n = p.n, k = p.nm, rows = n + 1, dim = c.dim, pd = patch_dim(), K = mpp_classes();
    int* idx = mim_idx();
    {
      ProfScope ps(this, PROF_OTHER, 0.0, 4.0 * B * n, s);
      mim_mask(B, n, 1, mim_rng_ptr(), idx, s);                       // mpp.py:78-88: the top_k of the noise
    }
    {
      ProfScope ps(this, PROF_OTHER, 0.0, 4.0 * B * (n + k + n), s);
      const double p_rand = mpp.random_patch_prob > 0.0 ? mpp.random_patch_prob / (1.0 - mpp.replace_prob) : 0.0;   // mpp.py:185
      mpp_draws(B, n, k, idx, mim_rng_ptr(), mpp.random_patch_prob, p_rand, mpp.replace_prob, mpp_src(), mpp_ids(), rows, s);
    }
    // the patch Dense of the corrupted patches with cls and positions in its residual operand (mpp.py:199-208)
    const int M = B * rows, Kp = bf16() ? embed.patch.ldw : embed.patch.K;
    T* col = arena.get<T>(static_cast<size_t>(M) * Kp);
    T* R = arena.get<T>(static_cast<size_t>(M) * dim);
    {
      ProfScope ps(this, PROF_EMBED, 0.0, 4.0 * M * pd + static_cast<double>(sizeof(T)) * M * (Kp + dim), s);
      mim_patch_rows<T>(img, B, H, Wd, c.channels, c.patch_h, c.patch_w, nullptr, n, 0, rows, col, Kp, embed.pos, R, dim, s, mpp_src(),
                        mask_token, embed.cls, embed.patch.bias);
    }
    T* X = arena.get<T>(static_cast<size_t>(M) * dim);
    float* stats = nullptr;
    {
      Epi ep; ep.bias = embed.patch.bias; ep.res = R; ep.ldr = dim;
      if (bf16() && dim % 64 == 0) { stats = row_stats(M, dim); ep.stats_out = stats; }
      Linear L = embed.patch;
      L.K = Kp;
      linear<T>(col, Kp, M, L, X, dim, ep, s);
    }
    bool sv = stats != nullptr;
    for (const auto& l : layers) layer_self<T>(X, B, rows, dim, l, s, stats, &sv);
    // to_bits on the masked rows only, ids ascending (predicted_patches[mask], mpp.py:128)
    const long long Mk = static_cast<long long>(B) * k;
    T* Xm = arena.get<T>(static_cast<size_t>(Mk) * dim);
    {
      ProfScope ps(this, PROF_OTHER, 0.0, 2.0 * sizeof(T) * Mk * dim, s);
      mim_take_rows<T>(X + dim, rows, mpp_ids(), Xm, B, k, dim, s);   // row 1 + j of each image, the ids at pitch n + 1
    }
    T* Lg = arena.get<T>(static_cast<size_t>(Mk) * to_bits_ld);
    {
      Epi e; e.bias = to_bits.bias;
      linear<T>(Xm, dim, static_cast<int>(Mk), to_bits, Lg, to_bits_ld, e, s);
    }
    double* partial = arena.get<double>(static_cast<size_t>(mim_loss_blocks(Mk)));
    {
      ProfScope ps(this, PROF_OTHER, static_cast<double>(Mk) * K, static_cast<double>(sizeof(T)) * Mk * K, s);
      mpp_loss<T>(Lg, to_bits_ld, K, Mk, partial, loss, s);
    }
    if (want_logits) {
      ProfScope ps(this, PROF_OTHER, 0.0, (static_cast<double>(sizeof(T)) + 4.0) * Mk * K, s);
      convert_rows<T, float>(Lg, to_bits_ld, mim_pred(), K, Mk, K, s);
    }
  }

  // DistillMixin.call (distill.py:16-45) on top of a ViT or a T2TViT: embed (the patch Dense, or T2T's soft splits and their
  // one-layer transformers, as vb_forward runs them) -> append the distillation token as the LAST row -> transformer over
  // n + 2 rows -> head on the first n + 1 rows, and the last row returned as is.
  template <typename T>
  void distill_impl(const float* img, int B, int H, int Wd, const float* distill_token, float* logits, float* distill_out, cudaStream_t s) {
    const vb_config& c = cfg;
    VB_CHECK(c.kind == VB_KIND_VIT || c.kind == VB_KIND_T2T_VIT, "vb_forward_distill supports ViT and T2TViT (distill.py:47, :61)");
    VB_CHECK(c.kind != VB_KIND_T2T_VIT || c.depth > 0,
             "vb_forward_distill: this T2TViT was built for an injected transformer (depth 0) and holds no main transformer; "
             "run vb_forward_embed, the injected transformer over the rows with the token appended, and vb_forward_head");
    arena.reset();
    int rows = 0;
    T* E = embed_any<T>(img, B, H, Wd, &rows, s, nullptr);
    const int rd = rows + 1;
    T* X = arena.get<T>(static_cast<size_t>(B) * rd * c.dim);
    copy_tokens<T>(E, rows, 0, X, rd, 0, rows, B, c.dim, s);
    T* last = X + static_cast<size_t>(rows) * c.dim;                 // row `rows` of image 0; image pitch rd rows
    broadcast_row<T>(distill_token, last, rd, B, c.dim, s);
    float* stats = c.dim % 64 == 0 ? row_stats(static_cast<long long>(B) * rd, c.dim) : nullptr;
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

  // DistillWrapper.call after the teacher (distill.py:116-134): the student over the handle's own distillation token, distill_mlp
  // on the token's row, and the loss from the labels and teacher logits at `labels` / `tlog` [B, num_classes] into loss [B]
  template <typename T>
  void distill_loss_forward(const float* img, int B, int H, int Wd, const float* labels, const float* tlog, double temperature,
                            double alpha, float* loss, cudaStream_t s) {
    const DistillPlan& p = dw_last;
    distill_impl<T>(img, B, H, Wd, W("distillation_token"), dw(p.student), dw(p.tokens), s);
    classify<float>(dw(p.tokens), 1, cfg.dim, dmlp_norm, dmlp, B, 0, dw(p.dlogits), false, s);
    distill_loss(dw(p.student), labels, tlog, B, cfg.num_classes, temperature, alpha, reinterpret_cast<double*>(dw(p.ce)),
                 reinterpret_cast<double*>(dw(p.q)), dw(p.dterm), loss, s);
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
    float* stats = cfg.dim % 64 == 0 ? row_stats(static_cast<long long>(B) * n, cfg.dim) : nullptr;
    bool sv = false;
    for (const auto& l : layers) layer_self<T>(X, B, n, cfg.dim, l, s, stats, &sv);
    if (sizeof(T) == 4) VB_CUDA(cudaMemcpyAsync(out, X, count * 4, cudaMemcpyDeviceToDevice, s));
    else convert<__nv_bfloat16, float>(reinterpret_cast<const __nv_bfloat16*>(X), out, count, s);
  }

  // ---------------------------------------------------------------- stage entries (vb_forward_embed / _head / vb_patch_to_emb)
  // The kinds that run as a whole forward only refuse the stage entries (and vb_forward_tokens) with a message of their own
  static const char* whole_forward_only(int kind) {
    switch (kind) {
      case VB_KIND_CCT: return "CCT runs as a whole forward only: its tokenizer / classifier stages have no entry of their own";
      case VB_KIND_LEVIT: return "LeViT runs as a whole forward only: its stem / backbone / head stages have no entry of their own";
      case VB_KIND_CVT: return "CvT runs as a whole forward only: its stem / stage / head steps have no entry of their own";
      case VB_KIND_TWINS_SVT: return "Twins-SVT runs as a whole forward only: its patch-embedding / stage / head steps have no entry of their own";
      case VB_KIND_CROSSFORMER: return "CrossFormer runs as a whole forward only: its embedding / stage / head steps have no entry of their own";
      case VB_KIND_NEST: return "NesT runs as a whole forward only: its patch-embedding / level / head steps have no entry of their own";
      case VB_KIND_REGIONVIT: return "RegionViT runs as a whole forward only: its encoder / stage / head steps have no entry of their own";
      case VB_KIND_ATS_VIT: return "ATS-ViT runs as a whole forward only: its token count changes inside the transformer, so its stages have no entry of their own";
      case VB_KIND_SMALL_DATASET_VIT: return "the small-dataset ViT runs as a whole forward only: its SPT embedding / transformer / head steps have no entry of their own";
      case VB_KIND_MOBILEVIT: return "MobileViT runs as a whole forward only: its stem / trunk / head steps have no entry of their own";
      case VB_KIND_SCALABLE_VIT: return "ScalableViT runs as a whole forward only: its patch-embedding / stage / head steps have no entry of their own";
      case VB_KIND_PIT: return "PiT runs as a whole forward only: it has no `transformer` attribute, so its patch-embedding / stage / head steps have no entry of their own";
      case VB_KIND_MAE: return "MAE runs through vb_forward_mim only: its encoder and decoder steps have no entry of their own";
      case VB_KIND_SIMMIM: return "SimMIM runs through vb_forward_mim only: its encoder steps have no entry of their own";
      case VB_KIND_MPP: return "MPP runs through vb_forward_mpp only: its encoder steps have no entry of their own";
      default: return nullptr;
    }
  }
  void check_stage_entries() const {
    const char* msg = whole_forward_only(cfg.kind);
    VB_CHECK(msg == nullptr, msg);
  }
  int embed_rows(int H, int Wd) const {
    VB_CHECK(cfg.kind != VB_KIND_CROSSVIT, "CrossViT has two token streams: no single embedding stage");
    check_stage_entries();
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
    check_stage_entries();
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
    check_stage_entries();
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
                                 static_cast<const float*>(e.res), e.ldr, e.act(), s, e.drop);
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
    if (e.drop.pos != DROP_NONE) {                  // a dropout epilogue: its position, site and rate
      uint32_t rate_bits = 0;
      std::memcpy(&rate_bits, &e.drop.rate, sizeof rate_bits);
      key[16] = static_cast<uintptr_t>(e.drop.pos) | static_cast<uintptr_t>(e.drop.site) << 8;
      key[17] = rate_bits;
    }
    auto it = plans.find(key);
    if (it == plans.end()) {
      if (plans.size() > 8192) plans.clear();      // shape sweeps: bounded host memory (a plan is four 128-byte tensor maps)
      GemmBf16 g = gemm_bf16_plan(A, lda, L.Wt, L.ldw, out, ldc, M, L.N, K, e.bias, e.scale, res, e.ldr, e.act(), false, 0,
                                  e.drop.pos != DROP_NONE);
      if (folded) { g.ln_c1 = L.ln_c1; g.ln_stats = e.ln_stats; g.ln_parts = K / 64; g.ln_inv_d = 1.0f / static_cast<float>(L.ln_d > 0 ? L.ln_d : K);
                    g.ln_eps = L.ln_eps; }
      if (e.stats_out) { g.stats_out = e.stats_out; }
      g.drop = e.drop;
      it = plans.emplace(key, g).first;
    }
    gemm_bf16_run(it->second, s);
  } else {
    gemm_simt<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(A, lda, L.Wt, 1, L.ldw, out, ldc, M, L.N, K, e.bias, e.scale, res,
                                                           e.ldr, e.act(), s, e.drop);
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
  int ns = std::min(s_elems * 6 > (48u << 20) ? 2 : T2T_MAX_STREAMS, B);
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
    VB_CHECK(k == q + HD && v == q + 2 * HD && ldk == ldq && ldv == ldq && nq == nk && variant == 0,
             "internal: windowed attention reads fused q|k|v rows");
    {
      ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * nq * nk * dh, static_cast<double>(sizeof(T)) * B * heads * dh * (2.0 * nq + 2.0 * nk), s);
      if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, s, 0.f, pb, win))
        return;
    }
    window_attention_generic<T>(q, ldq, out, ldo, B, nq, heads, dh, *win, pb, s);
    return;
  }
  ProfScope ps(this, PROF_ATTN, 4.0 * B * heads * nq * nk * dh + (variant == 1 ? 2.0 : variant == 2 ? 4.0 : 0.0) * B * nq * nk * heads * heads,
               static_cast<double>(sizeof(T)) * B * heads * dh * (2.0 * nq + 2.0 * nk), s);
  if (attention_fast<T>(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, variant, mix_a, mix_b, g, b, s, scale)) return;
  float* S = arena.get<float>(static_cast<size_t>(B) * heads * nq * ((nk + 15) & ~15));   // row pitch padded for the bf16-P path
  attention_generic<T>(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, heads, dh, variant, mix_a, mix_b, g, b, s, scale);
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
  VB_CHECK(c.kind != VB_KIND_NEST, "NesT: create the handle with vb_create_nest (its levels are a vb_nest_config)");
  VB_CHECK(c.kind != VB_KIND_REGIONVIT, "RegionViT: create the handle with vb_create_regionvit (its stages are a vb_regionvit_config)");
  VB_CHECK(c.kind != VB_KIND_ATS_VIT, "ATS-ViT: create the handle with vb_create_ats_vit (its token counts are a vb_ats_vit_config)");
  VB_CHECK(c.kind != VB_KIND_MOBILEVIT, "MobileViT: create the handle with vb_create_mobilevit (its blocks are a vb_mobilevit_config)");
  VB_CHECK(c.kind != VB_KIND_SCALABLE_VIT, "ScalableViT: create the handle with vb_create_scalable_vit (its stages are a vb_scalable_vit_config)");
  VB_CHECK(c.kind != VB_KIND_PIT, "PiT: create the handle with vb_create_pit (its stages' depths and heads are a vb_pit_config)");
  VB_CHECK(c.kind != VB_KIND_MAE, "MAE: create the handle with vb_create_mim (its masking ratio and decoder are a vb_mim_config)");
  VB_CHECK(c.kind != VB_KIND_SIMMIM, "SimMIM: create the handle with vb_create_mim (its masking ratio is a vb_mim_config)");
  VB_CHECK(c.kind != VB_KIND_MPP, "MPP: create the handle with vb_create_mim (its probabilities and bits are a vb_mpp_config)");
  VB_CHECK((c.kind >= VB_KIND_VIT && c.kind <= VB_KIND_CCT) || c.kind == VB_KIND_SMALL_DATASET_VIT, "unknown model kind");
  if (c.kind == VB_KIND_SMALL_DATASET_VIT) {
    // SPT's Rearrange takes one patch size for both sides (vit_for_small_dataset.py:147) and shift() one image of 3 channels
    VB_CHECK(c.patch_h == c.patch_w, "the small-dataset ViT takes one integer patch_size (SPT's Rearrange uses it for both sides)");
    VB_CHECK(c.channels == 3, "the small-dataset ViT takes images of 3 channels");
  }
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

void validate_nest(const vb_config& c, const vb_nest_config& n) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0, "NesT: bad channel / class configuration");
  VB_CHECK(n.num_hierarchies >= 1 && n.num_hierarchies <= VB_NEST_MAX_LEVELS,
           "NesT: num_hierarchies " + std::to_string(n.num_hierarchies) + " is not supported (1 to VB_NEST_MAX_LEVELS = " +
               std::to_string(VB_NEST_MAX_LEVELS) + ")");
  VB_CHECK(n.levels >= 0 && n.levels <= n.num_hierarchies, "NesT: levels must be in [0, num_hierarchies] (the zip with block_repeats)");
  VB_CHECK(n.patch_size > 0 && n.heads > 0 && n.dim >= n.heads && n.mlp_mult > 0 && n.seq_len > 0,
           "NesT: bad patch_size / dim / heads / mlp_mult / seq_len");
  VB_CHECK((static_cast<long long>(n.dim) << (n.num_hierarchies - 1)) <= 65536, "NesT: dim * 2^(num_hierarchies - 1) is too large");
  for (int i = 0; i < n.levels; ++i) VB_CHECK(n.block_repeats[i] >= 0, "NesT: block_repeats must not be negative");
}

// ats_vit.py:225-227 (the reference's assert messages) on top of ViT's checks
void validate_ats(const vb_config& c, const vb_ats_vit_config& a) {
  vb_config v = c;
  v.kind = VB_KIND_VIT;
  v.pool = VB_POOL_CLS;
  validate(v);
  VB_CHECK(c.depth >= 1 && c.depth <= VB_ATS_MAX_DEPTH, "ATS-ViT: depth must be in [1, 64]");
  for (int L = 1; L < c.depth; ++L)
    VB_CHECK(a.max_tokens_per_depth[L] <= a.max_tokens_per_depth[L - 1], "max_tokens_per_depth must be in decreasing order");
  for (int L = 0; L < c.depth; ++L)
    VB_CHECK(a.max_tokens_per_depth[L] > 0, "max_tokens_per_depth must have at least 1 token at any layer");
  VB_CHECK(c.dim_head <= ATS_MAX_DH, "ATS-ViT: dim_head must be at most 256");
}

// pit.py:173 and ViT's checks on the model the stages make: one stream of width dim, the depths summed, every stage's heads in [1, 32]
void validate_pit(const vb_config& c, const vb_pit_config& p) {
  VB_CHECK(p.stages >= 0 && p.stages <= VB_PIT_MAX_STAGES, "PiT: stages must be in [0, " + std::to_string(VB_PIT_MAX_STAGES) + "]");
  VB_CHECK(c.image_h == c.image_w && c.patch_h == c.patch_w, "PiT takes one integer image_size and one integer patch_size");
  VB_CHECK(c.patch_h >= 2, "PiT: patch_size must be at least 2 (the patch stride is patch_size // 2)");
  vb_config v = c;
  v.kind = VB_KIND_VIT;
  v.pool = VB_POOL_CLS;
  v.heads = 1;
  v.depth = 0;
  for (int s = 0; s < p.stages; ++s) {
    VB_CHECK(p.depth[s] >= 0 && p.heads[s] >= 1 && p.heads[s] <= 32, "PiT: every stage needs depth >= 0 and 1 to 32 heads");
    v.depth += p.depth[s];
  }
  validate(v);
}

// mae.py:28 / simmim.py:74 (the reference's assert message) and the decoder's Transformer on top of ViT's checks of the encoder
void validate_mim(const vb_config& c, const vb_mim_config& m) {
  vb_config v = c;
  v.kind = VB_KIND_VIT;
  v.pool = VB_POOL_CLS;
  v.num_classes = 1;                                     // the encoder's mlp_head is not part of the model
  validate(v);
  VB_CHECK(m.masking_ratio > 0.0 && m.masking_ratio < 1.0, "masking ratio must be kept between 0 and 1");
  if (c.kind == VB_KIND_MAE) {
    VB_CHECK(m.decoder_dim > 0 && m.decoder_depth >= 0 && m.decoder_heads > 0 && m.decoder_dim_head > 0, "MAE: bad decoder dimensions");
    VB_CHECK(m.decoder_heads <= 32, "MAE: at most 32 decoder heads");
  }
}

// mpp.py's constructor arguments the engine takes: channels 3 (its Bucketize / bin_mask read three channels), at most 2^16 classes
void validate_mpp(const vb_config& c, const vb_mpp_config& m) {
  vb_config v = c;
  v.kind = VB_KIND_VIT;
  v.pool = VB_POOL_CLS;
  v.num_classes = 1;
  validate(v);
  VB_CHECK(c.channels == 3, "MPP: images of 3 channels");
  VB_CHECK(m.output_channel_bits >= 1 && m.output_channel_bits * c.channels <= 16,
           "MPP: output_channel_bits * channels must be 1 to 16 (to_bits has 2^(bits * channels) classes)");
  VB_CHECK(std::isfinite(m.mask_prob) && std::isfinite(m.replace_prob) && std::isfinite(m.random_patch_prob), "MPP: probabilities must be finite");
}

void validate_regionvit(const vb_config& c, const vb_regionvit_config& r) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.num_classes > 0, "RegionViT: bad channel / class configuration");
  for (int s = 0; s < VB_REGIONVIT_STAGES; ++s)
    VB_CHECK(r.dims[s] > 0 && r.dims[s] <= 65536 && r.depth[s] >= 0, "RegionViT: dims must be positive and depth not negative");
  VB_CHECK(r.window_size > 0 && r.local_patch_size > 0 && r.mlp_mult > 0, "RegionViT: bad window_size / local_patch_size / mlp_mult");
  VB_CHECK(static_cast<long long>(r.local_patch_size) * r.window_size <= 4096, "RegionViT: the region patch size is too large");
  VB_CHECK(r.window_size <= 1024, "RegionViT: window_size is too large");
}

// The widths the host computed must chain as mobile_vit.py:230-252 wires the blocks
void validate_mobilevit(const vb_config& c, const vb_mobilevit_config& m) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels == 3 && c.num_classes > 0, "MobileViT: images of 3 channels and a positive num_classes");
  for (int i = 0; i < 10; ++i) VB_CHECK(m.channels[i] > 0 && m.channels[i] <= 65536, "MobileViT: channels must be positive");
  VB_CHECK(m.last_dim > 0 && m.last_dim <= 65536, "MobileViT: channels[-1] must be positive");
  for (int s = 0; s < 3; ++s) VB_CHECK(m.dims[s] > 0 && m.dims[s] <= 65536 && m.depths[s] >= 0, "MobileViT: dims must be positive and depths not negative");
  VB_CHECK(m.kernel_size >= 1 && m.kernel_size <= 15 && m.ph > 0 && m.pw > 0, "MobileViT: bad kernel_size / patch_size");
  const int in[VB_MOBILEVIT_MV2] = {m.channels[0], m.channels[1], m.channels[2], m.channels[3], m.channels[3], m.channels[5], m.channels[7]};
  const int out[VB_MOBILEVIT_MV2] = {m.channels[1], m.channels[2], m.channels[3], m.channels[3], m.channels[4], m.channels[6], m.channels[8]};
  const int stride[VB_MOBILEVIT_MV2] = {1, 2, 1, 1, 2, 2, 2};
  for (int i = 0; i < VB_MOBILEVIT_MV2; ++i) {
    const std::string b = "MobileViT MV2 block " + std::to_string(i) + ": ";
    VB_CHECK(m.mv2_in[i] == in[i] && m.mv2_out[i] == out[i] && m.mv2_stride[i] == stride[i], b + "widths or stride do not chain");
    VB_CHECK(m.mv2_hidden[i] > 0 && m.mv2_hidden[i] <= 262144, b + "bad hidden width");
    VB_CHECK(m.mv2_expand[i] || m.mv2_hidden[i] == m.mv2_in[i], b + "without the expand convolution the depthwise step needs hidden == input width");
    VB_CHECK(!m.mv2_residual[i] || (stride[i] == 1 && in[i] == out[i]), b + "a residual needs stride 1 and equal widths");
  }
}

void validate_scalable_vit(const vb_config& c, const vb_scalable_vit_config& v) {
  VB_CHECK(c.precision == VB_PRECISION_FP32 || c.precision == VB_PRECISION_BF16, "unknown precision");
  VB_CHECK(c.channels > 0 && c.channels <= 64 && c.num_classes > 0, "ScalableViT: bad channel / class configuration");
  VB_CHECK(v.num_stages >= 1 && v.num_stages <= VB_SCALABLE_VIT_STAGES, "ScalableViT: num_stages must be in [1, 4]");
  VB_CHECK(v.ff_expansion_factor >= 1 && v.ff_expansion_factor <= 64, "ScalableViT: bad ff_expansion_factor");
  VB_CHECK(v.dim[0] > 0 && (static_cast<long long>(v.dim[0]) << (v.num_stages - 1)) <= 8192, "ScalableViT: bad dim");
  for (int st = 0; st < v.num_stages; ++st) {
    const std::string stage = "ScalableViT stage " + std::to_string(st + 1) + ": ";
    VB_CHECK(v.dim[st] == v.dim[0] << st, stage + "dim must be dim[0] * 2^s");
    VB_CHECK(v.depth[st] >= 0 && v.depth[st] <= 256, stage + "bad depth");
    VB_CHECK(v.heads[st] >= 1 && v.heads[st] <= 64, stage + "bad heads");
    VB_CHECK(v.ssa_dim_key[st] >= 1 && v.ssa_dim_value[st] >= 1 && v.iwsa_dim_key[st] >= 1 && v.iwsa_dim_value[st] >= 1 &&
             v.ssa_dim_key[st] <= 512 && v.ssa_dim_value[st] <= 512 && v.iwsa_dim_key[st] <= 512 && v.iwsa_dim_value[st] <= 512,
             stage + "bad key / value widths");
    VB_CHECK(v.reduction_factor[st] >= 1 && v.reduction_factor[st] <= 64, stage + "bad reduction_factor");
    VB_CHECK(v.window[st] >= 0, stage + "bad window");
  }
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
// f(h, T()) with T the element type of `precision` (float for fp32, __nv_bfloat16 otherwise) and h a scratch handle of that
// precision, on which an op entry runs the forward's own members: no weights, profiling off, its arena the entry's scratch.  A
// timed iteration resets the arena first, so the scratch pointers, and the GEMM plans cached on them, stay the same.
template <typename F>
void with_precision(int32_t precision, F&& f) {
  vb_handle h{};
  if (precision == VB_PRECISION_FP32) {
    h.cfg.precision = VB_PRECISION_FP32;
    f(h, float());
  } else {
    h.cfg.precision = VB_PRECISION_BF16;
    f(h, __nv_bfloat16());
  }
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
// vb_create, and vb_create_distill (distill_wrapper: a ViT / T2TViT student handle that also registers DistillWrapper's weights)
int create_base(const char* fn, const vb_config* cfg, int device, vb_handle** out, bool distill_wrapper) {
  const std::string f(fn);
  return guarded(nullptr, [&] {
    VB_CHECK(cfg != nullptr && out != nullptr, f + ": null argument");
    // a client of the ABI-7 struct without the CCT fields passes the shorter size: read only its bytes, zero the rest
    const int32_t size = cfg->struct_size;
    VB_CHECK(size == static_cast<int32_t>(sizeof(vb_config)) || size == VB_CONFIG_SIZE_ABI7, "vb_config.struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, cfg, static_cast<size_t>(size));
    if (distill_wrapper) {
      VB_CHECK(c.kind == VB_KIND_VIT || c.kind == VB_KIND_T2T_VIT, f + " supports ViT and T2TViT (distill.py:47, :61)");
      VB_CHECK(c.kind != VB_KIND_T2T_VIT || c.depth > 0,
               f + ": this T2TViT was built for an injected transformer (depth 0); its distillation call is composed on the host");
    }
    validate(c);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, f + ": no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, f + ": bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, f + ": libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    h->device = device;
    h->distill_wrapper = distill_wrapper;
    h->build_expected();
    *out = h.release();
  });
}
// an extension config's struct_size: its first field, or (vb_mpp_config) that of the vb_mim_config it begins with
template <typename Ext> int32_t ext_struct_size(const Ext& e) { return e.struct_size; }
int32_t ext_struct_size(const vb_mpp_config& e) { return e.mim.struct_size; }
// vb_create_<kind> for the kinds whose stages come in an extension config: `fn` and `ext_name` name the entry point and the
// config struct in the messages; `validate` checks the config against the base, `adopt` stores it in the handle and sets cfg.dim.
template <typename Ext, typename Validate, typename Adopt>
int create_with(const char* fn, const char* ext_name, int kind, const char* kind_name, const vb_config* base, const Ext* ext, int device,
                vb_handle** out, Validate validate, Adopt adopt) {
  const std::string f(fn);
  return guarded(nullptr, [&] {
    VB_CHECK(base != nullptr && ext != nullptr && out != nullptr, f + ": null argument");
    VB_CHECK(base->struct_size == static_cast<int32_t>(sizeof(vb_config)) || base->struct_size == VB_CONFIG_SIZE_ABI7,
             "vb_config.struct_size mismatch (ABI)");
    VB_CHECK(ext_struct_size(*ext) == static_cast<int32_t>(sizeof(Ext)), std::string(ext_name) + ".struct_size mismatch (ABI)");
    vb_config c;
    memset(&c, 0, sizeof c);
    memcpy(&c, base, static_cast<size_t>(base->struct_size));
    VB_CHECK(c.kind == kind, f + ": base.kind must be " + kind_name);
    validate(c, *ext);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VB_CHECK(e == cudaSuccess && ndev > 0, f + ": no CUDA device available -- libvitb200 has no CPU fallback");
    VB_CHECK(device >= 0 && device < ndev, f + ": bad device index");
    VB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    VB_CUDA(cudaGetDeviceProperties(&prop, device));
    VB_CHECK(prop.major == 9 && prop.minor == 0, f + ": libvitb200 is built for sm_90a (Hopper H100) only");
    std::unique_ptr<vb_handle> h(new vb_handle());
    h->cfg = c;
    adopt(*h);
    h->device = device;
    h->build_expected();
    *out = h.release();
  });
}
// The whole-forward CUDA graph of vb_forward / vb_forward_mim (see vb_handle::graphs): the key's second call on a capturable stream
// is captured and launched, later calls replay it; otherwise, and when the capture fails, run_eager runs the launches directly.
template <typename F>
void run_graphed(vb_handle* h, const vb_handle::GraphKey& key, F&& run_eager) {
  cudaStream_t s = key.s;
  static const bool graphs_off = getenv("VB_NO_GRAPH") != nullptr;
  const bool graphable = !graphs_off && !h->profiling && s != nullptr && s != cudaStreamLegacy;
  bool done = false;
  if (graphable) {
    if (h->graphs.size() > 64) h->drop_graphs();                         // shape / pointer sweeps: bounded
    vb_handle::GraphEntry& ge = h->graphs[key];
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
}

}  // namespace

extern "C" {

int vb_abi_version(void) { return VB_ABI_VERSION; }

int vb_create(const vb_config* cfg, int device, vb_handle** out) { return create_base("vb_create", cfg, device, out, false); }

int vb_create_distill(const vb_config* student, int device, vb_handle** out) {
  return create_base("vb_create_distill", student, device, out, true);
}

int vb_create_levit(const vb_config* base, const vb_levit_config* lv, int device, vb_handle** out) {
  return create_with("vb_create_levit", "vb_levit_config", VB_KIND_LEVIT, "VB_KIND_LEVIT", base, lv, device, out,
                                      validate_levit, [&](vb_handle& h) { h.lv = *lv; h.cfg.dim = lv->dims[lv->stages - 1]; });
}
int vb_create_cvt(const vb_config* base, const vb_cvt_config* cvt, int device, vb_handle** out) {
  return create_with("vb_create_cvt", "vb_cvt_config", VB_KIND_CVT, "VB_KIND_CVT", base, cvt, device, out, validate_cvt,
                                    [&](vb_handle& h) { h.cv = *cvt; h.cfg.dim = cvt->emb_dim[VB_CVT_STAGES - 1]; });
}
int vb_create_twins_svt(const vb_config* base, const vb_twins_svt_config* tw, int device, vb_handle** out) {
  return create_with("vb_create_twins_svt", "vb_twins_svt_config", VB_KIND_TWINS_SVT, "VB_KIND_TWINS_SVT", base, tw,
                                          device, out, validate_twins,
                                          [&](vb_handle& h) { h.tw = *tw; h.cfg.dim = tw->emb_dim[VB_TWINS_STAGES - 1]; });
}
int vb_create_crossformer(const vb_config* base, const vb_crossformer_config* cfc, int device, vb_handle** out) {
  return create_with("vb_create_crossformer", "vb_crossformer_config", VB_KIND_CROSSFORMER, "VB_KIND_CROSSFORMER",
                                            base, cfc, device, out, validate_crossformer,
                                            [&](vb_handle& h) { h.cf = *cfc; h.cfg.dim = cfc->dim[VB_CROSSFORMER_STAGES - 1]; });
}
int vb_create_nest(const vb_config* base, const vb_nest_config* nc, int device, vb_handle** out) {
  return create_with("vb_create_nest", "vb_nest_config", VB_KIND_NEST, "VB_KIND_NEST", base, nc, device, out, validate_nest,
                                     [&](vb_handle& h) { h.ns = *nc; h.cfg.dim = h.nest_last_dim(); });
}
int vb_create_ats_vit(const vb_config* base, const vb_ats_vit_config* ac, int device, vb_handle** out) {
  return create_with("vb_create_ats_vit", "vb_ats_vit_config", VB_KIND_ATS_VIT, "VB_KIND_ATS_VIT", base, ac, device, out, validate_ats,
                     [&](vb_handle& h) { h.ats = *ac; h.cfg.pool = VB_POOL_CLS; });
}

int vb_ats_set_seed(vb_handle* h, uint64_t seed) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CHECK(h->cfg.kind == VB_KIND_ATS_VIT, "vb_ats_set_seed: not an ATS-ViT handle");
    VB_CUDA(cudaSetDevice(h->device));
    VB_CUDA(cudaDeviceSynchronize());                  // no forward in flight reads the old key and counter
    const unsigned long long v[2] = {static_cast<unsigned long long>(seed), 0ull};
    VB_CUDA(cudaMemcpy(h->ats_rng_ptr(), v, sizeof v, cudaMemcpyHostToDevice));
    VB_CUDA(cudaDeviceSynchronize());                  // a pageable copy may return before it lands
  });
}

int vb_forward_ats(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
                   int32_t* token_ids, int32_t* count, void* stream) {
  const int rc = guarded(h, [&] {
    VB_CHECK(h != nullptr && token_ids != nullptr && count != nullptr, "vb_forward_ats: null argument");
    VB_CHECK(h->cfg.kind == VB_KIND_ATS_VIT, "vb_forward_ats: not an ATS-ViT handle");
  });
  if (rc != 0) return rc;
  const int fr = vb_forward(h, img, img_mem, batch, img_h, img_w, logits, VB_MEM_HOST, stream);
  if (fr != 0) return fr;
  return guarded(h, [&] {
    const vb_handle::AtsPlan& p = h->ats_last;
    const int* st = static_cast<const int*>(h->ats_dev.p);
    const int depth = h->cfg.depth, f = p.slot[depth];
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VB_CUDA(cudaMemcpyAsync(token_ids, st + p.out, static_cast<size_t>(batch) * (p.P[depth] - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(count, st + p.C + f, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
  });
}

int vb_ats_last_draws(vb_handle* h, int32_t layer, int32_t* draws, int32_t* counts, int32_t* sampled) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && draws != nullptr && counts != nullptr && sampled != nullptr, "vb_ats_last_draws: null argument");
    VB_CHECK(h->cfg.kind == VB_KIND_ATS_VIT, "vb_ats_last_draws: not an ATS-ViT handle");
    const vb_handle::AtsPlan& p = h->ats_last;
    VB_CHECK(p.B > 0, "vb_ats_last_draws: no forward has run");
    VB_CHECK(layer >= 0 && layer < h->cfg.depth && p.can[layer], "vb_ats_last_draws: layer " + std::to_string(layer) + " never samples");
    VB_CUDA(cudaSetDevice(h->device));
    VB_CUDA(cudaDeviceSynchronize());
    const int* st = static_cast<const int*>(h->ats_dev.p);
    const int K = h->ats.max_tokens_per_depth[layer];
    VB_CUDA(cudaMemcpy(draws, st + p.draws[layer], static_cast<size_t>(p.B) * K * sizeof(int), cudaMemcpyDeviceToHost));
    VB_CUDA(cudaMemcpy(counts, st + p.rows + static_cast<size_t>(p.slot[layer + 1]) * p.B, static_cast<size_t>(p.B) * sizeof(int),
                       cudaMemcpyDeviceToHost));
    for (int b = 0; b < p.B; ++b) counts[b] -= 1;      // live rows -> kept tokens
    int C_in = 0;
    VB_CUDA(cudaMemcpy(&C_in, st + p.C + p.slot[layer], sizeof(int), cudaMemcpyDeviceToHost));
    *sampled = C_in > K ? 1 : 0;                       // ats_vit.py:213 on the batch's padded length
    if (!*sampled) std::fill(draws, draws + static_cast<size_t>(p.B) * K, -1);
  });
}

int vb_op_ats_sample(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t P, int32_t heads, int32_t dh, float scale,
                     const int32_t* rows, int32_t K, uint64_t seed, uint64_t counter, int32_t* sel, int32_t* rows_new, int32_t* draws) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(qkv && rows && sel && rows_new && draws && B > 0 && P > 1 && heads > 0 && dh > 0 && ld >= 3 * heads * dh && K > 0,
             "vb_op_ats_sample: bad arguments");
    int C = 0;
    for (int b = 0; b < B; ++b) {
      VB_CHECK(rows[b] >= 2 && rows[b] <= P, "vb_op_ats_sample: rows[b] must be in [2, P]");
      C = std::max(C, rows[b] - 1);
    }
    const int Pn = 1 + std::min(P - 1, K);
    DevMem dX, dI, dR, dS, dF;
    const size_t nint = static_cast<size_t>(B) + 1 + static_cast<size_t>(B) * Pn + B + static_cast<size_t>(B) * K;
    dI.ensure(nint * sizeof(int));
    int* i_d = static_cast<int*>(dI.p);
    int *rows_d = i_d, *C_d = i_d + B, *sel_d = C_d + 1, *rn_d = sel_d + static_cast<size_t>(B) * Pn, *dr_d = rn_d + B;
    VB_CUDA(cudaMemcpy(rows_d, rows, static_cast<size_t>(B) * sizeof(int), cudaMemcpyHostToDevice));
    VB_CUDA(cudaMemcpy(C_d, &C, sizeof(int), cudaMemcpyHostToDevice));
    VB_CUDA(cudaMemset(dr_d, 0xff, static_cast<size_t>(B) * K * sizeof(int)));
    const unsigned long long rng[2] = {static_cast<unsigned long long>(seed), static_cast<unsigned long long>(counter)};
    dR.ensure(sizeof rng);
    VB_CUDA(cudaMemcpy(dR.p, rng, sizeof rng, cudaMemcpyHostToDevice));
    dF.ensure(static_cast<size_t>(3) * B * P * sizeof(float));
    auto run = [&](auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(B) * P * ld);
      ats_sample<T>(x_d, ld, B, P, heads, dh, scale, rows_d, C_d, K, static_cast<const unsigned long long*>(dR.p), static_cast<float*>(dF.p),
                    sel_d, Pn, rn_d, dr_d, 0);
    };
    if (precision == VB_PRECISION_FP32) run(float());
    else run(__nv_bfloat16());
    VB_CUDA(cudaDeviceSynchronize());
    VB_CUDA(cudaMemcpy(sel, sel_d, static_cast<size_t>(B) * Pn * sizeof(int), cudaMemcpyDeviceToHost));
    VB_CUDA(cudaMemcpy(rows_new, rn_d, static_cast<size_t>(B) * sizeof(int), cudaMemcpyDeviceToHost));
    VB_CUDA(cudaMemcpy(draws, dr_d, static_cast<size_t>(B) * K * sizeof(int), cudaMemcpyDeviceToHost));
  });
}

int vb_op_masked_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t n, int32_t heads, int32_t dh,
                           const int32_t* nk_img, float* out, int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && nk_img && out && B > 0 && n > 0 && heads > 0 && dh > 0 && ld >= 3 * HD && ldo >= HD, "vb_op_masked_attention: bad arguments");
    for (int b = 0; b < B; ++b) VB_CHECK(nk_img[b] >= 1 && nk_img[b] <= n, "vb_op_masked_attention: nk_img[b] must be in [1, n]");
    DevMem dX, dO, dN;
    dN.ensure(static_cast<size_t>(B) * sizeof(int));
    VB_CUDA(cudaMemcpy(dN.p, nk_img, static_cast<size_t>(B) * sizeof(int), cudaMemcpyHostToDevice));
    const int* nk_d = static_cast<const int*>(dN.p);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(B) * n * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(B) * n * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_masked_dispatch<T>(x_d, ld, o_d, ldo, B, n, heads, dh, dh, 1.0f / sqrtf(static_cast<float>(dh)), ATTN_MASK_KEYS, 0, nk_d);
      });
      download<T>(o_d, out, static_cast<size_t>(B) * n * ldo);
    });
  });
}

int vb_op_spt(int32_t precision, const float* img, int32_t B, int32_t H, int32_t W, int32_t p, int32_t dim, const float* gamma,
              const float* beta, const float* kernel, const float* bias, const float* cls, const float* pos, float* out) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(img && gamma && beta && kernel && bias && out && B > 0 && H > 0 && W > 0 && p > 0 && dim > 0, "vb_op_spt: bad arguments");
    VB_CHECK(H % p == 0 && W % p == 0, "Image dimensions must be divisible by the patch size.");
    const int C = 3, K = p * p * 5 * C, rows = 1 + (H / p) * (W / p);
    auto host = [](const float* a, size_t n) { return a ? std::vector<double>(a, a + n) : std::vector<double>(n, 0.0); };
    DevMem dI;
    const float* img_d = upload<float>(dI, img, static_cast<size_t>(B) * H * W * C);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      h.cfg.patch_h = p;
      h.cfg.channels = C;
      h.set_spt_patch(host(gamma, K), host(beta, K), host(kernel, static_cast<size_t>(K) * dim), host(bias, dim), K, dim);
      h.embed.cls = h.upload_owned(host(cls, dim));                // zero cls and positions when not given
      h.embed.pos = h.upload_owned(host(pos, static_cast<size_t>(rows) * dim));
      h.embed.dim = dim;
      h.embed.n_pos = rows;
      int r = 0;
      const T* o_d = h.spt_tokens<T>(img_d, B, H, W, &r, 0, nullptr);
      download<T>(o_d, out, static_cast<size_t>(B) * rows * dim);
    });
    VB_CUDA(cudaDeviceSynchronize());
  });
}

int vb_op_lsa_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t n, int32_t heads, int32_t dh, float scale,
                        float* out, int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && out && B > 0 && n > 0 && heads > 0 && dh > 0 && ld >= 3 * HD && ldo >= HD && scale > 0.f,
             "vb_op_lsa_attention: bad arguments");
    VB_CHECK(n >= 2, "vb_op_lsa_attention: locality self-attention needs n >= 2 (every row keeps a key besides its own)");
    // bf16 heads narrower than 64 run widened with zero columns, as make_layer widens an LSA layer's to_qkv / to_out
    const bool widen = precision == VB_PRECISION_BF16 && dh < 64 && dh % 8 == 0;
    const int dw = widen ? 64 : dh, HW = heads * dw, ldw = widen ? 3 * HW : ld, ldow = widen ? HW : ldo;
    std::vector<float> wide, wout;
    const float* src = qkv;
    if (widen) {
      wide.assign(static_cast<size_t>(B) * n * ldw, 0.f);
      for (size_t r = 0; r < static_cast<size_t>(B) * n; ++r)
        for (int g = 0; g < 3; ++g)
          for (int h = 0; h < heads; ++h)
            std::copy(qkv + r * ld + g * HD + h * dh, qkv + r * ld + g * HD + h * dh + dh, wide.begin() + r * ldw + g * HW + h * dw);
      wout.assign(static_cast<size_t>(B) * n * ldow, 0.f);
      src = wide.data();
    }
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, src, static_cast<size_t>(B) * n * ldw);
      T* o_d = upload<T>(dO, widen ? wout.data() : out, static_cast<size_t>(B) * n * ldow);
      timed(iters, elapsed_ms, [&] {                  // the scale is explicit, so the widened heads run as the model's own
        h.arena.reset();
        h.attention_masked_dispatch<T>(x_d, ldw, o_d, ldow, B, n, heads, dw, dw, scale, ATTN_MASK_DIAG, 0, nullptr);
      });
      download<T>(o_d, widen ? wout.data() : out, static_cast<size_t>(B) * n * ldow);
    });
    if (widen)
      for (size_t r = 0; r < static_cast<size_t>(B) * n; ++r)
        for (int h = 0; h < heads; ++h)
          std::copy(wout.begin() + r * ldow + h * dw, wout.begin() + r * ldow + h * dw + dh, out + r * ldo + h * dh);
  });
}

int vb_create_mobilevit(const vb_config* base, const vb_mobilevit_config* mc, int device, vb_handle** out) {
  return create_with("vb_create_mobilevit", "vb_mobilevit_config", VB_KIND_MOBILEVIT, "VB_KIND_MOBILEVIT", base, mc, device, out,
                     validate_mobilevit, [&](vb_handle& h) { h.mv = *mc; h.cfg.dim = mc->last_dim; });
}

int vb_create_scalable_vit(const vb_config* base, const vb_scalable_vit_config* sc, int device, vb_handle** out) {
  return create_with("vb_create_scalable_vit", "vb_scalable_vit_config", VB_KIND_SCALABLE_VIT, "VB_KIND_SCALABLE_VIT", base, sc, device,
                     out, validate_scalable_vit, [&](vb_handle& h) { h.sv = *sc; h.cfg.dim = sc->dim[sc->num_stages - 1]; });
}

int vb_create_pit(const vb_config* base, const vb_pit_config* pc, int device, vb_handle** out) {
  return create_with("vb_create_pit", "vb_pit_config", VB_KIND_PIT, "VB_KIND_PIT", base, pc, device, out, validate_pit, [&](vb_handle& h) {
    h.pit = *pc;
    h.cfg.depth = 0;
    for (int s = 0; s < pc->stages; ++s) h.cfg.depth += pc->depth[s];
    h.cfg.heads = pc->stages > 0 ? pc->heads[0] : 1;
    h.cfg.pool = VB_POOL_CLS;
  });
}

int vb_create_mim(const vb_config* encoder, const vb_mim_config* mc, int device, vb_handle** out) {
  const int rc = guarded(nullptr, [&] {
    VB_CHECK(encoder != nullptr && mc != nullptr && out != nullptr, "vb_create_mim: null argument");
    VB_CHECK(encoder->kind == VB_KIND_MAE || encoder->kind == VB_KIND_SIMMIM || encoder->kind == VB_KIND_MPP,
             "vb_create_mim: encoder.kind must be VB_KIND_MAE or VB_KIND_SIMMIM (or VB_KIND_MPP)");
  });
  if (rc != 0) return rc;
  if (encoder->kind == VB_KIND_MPP) {                    // the vb_mpp_config begins with the vb_mim_config whose struct_size it sets
    const vb_mpp_config* mp = reinterpret_cast<const vb_mpp_config*>(mc);
    return create_with("vb_create_mim", "vb_mpp_config", VB_KIND_MPP, "VB_KIND_MPP", encoder, mp, device, out, validate_mpp,
                       [&](vb_handle& h) { h.mpp = *mp; h.mim = mp->mim; h.cfg.pool = VB_POOL_CLS; });
  }
  return create_with("vb_create_mim", "vb_mim_config", encoder->kind, encoder->kind == VB_KIND_MAE ? "VB_KIND_MAE" : "VB_KIND_SIMMIM", encoder,
                     mc, device, out, validate_mim, [&](vb_handle& h) { h.mim = *mc; h.cfg.pool = VB_POOL_CLS; });
}

int vb_mim_set_seed(vb_handle* h, uint64_t seed) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CHECK(h->is_mim(), "vb_mim_set_seed: not a MAE / SimMIM / MPP handle");
    VB_CUDA(cudaSetDevice(h->device));
    VB_CUDA(cudaDeviceSynchronize());                  // no forward in flight reads the old key and counter
    const unsigned long long v[3] = {static_cast<unsigned long long>(seed), 0ull, 0ull};
    VB_CUDA(cudaMemcpy(h->mim_rng_ptr(), v, sizeof v, cudaMemcpyHostToDevice));
    VB_CUDA(cudaDeviceSynchronize());                  // a pageable copy may return before it lands
  });
}

int vb_forward_mim(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* loss, float* pred,
                   float* masked_patches, int32_t* indices, int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && loss != nullptr, "vb_forward_mim: null argument");
    VB_CHECK(h->is_mim() && h->cfg.kind != VB_KIND_MPP, "vb_forward_mim: not a MAE / SimMIM handle (MPP runs through vb_forward_mpp)");
    VB_CHECK(h->finalized, "vb_forward_mim: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward_mim: bad batch / image size");
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const size_t img_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const float* img_d = img;
    if (img_mem == VB_MEM_HOST) {
      h->img_dev.ensure(img_bytes);
      VB_CUDA(cudaMemcpyAsync(h->img_dev.p, img, img_bytes, cudaMemcpyHostToDevice, s));
      img_d = static_cast<const float*>(h->img_dev.p);
    }
    float* loss_d = loss;
    if (out_mem == VB_MEM_HOST) {
      h->logits_dev.ensure(sizeof(float));
      loss_d = static_cast<float*>(h->logits_dev.p);
    }
    h->mim_prepare(batch, img_h, img_w);
    const int flags = (pred != nullptr ? 1 : 0) | (masked_patches != nullptr ? 2 : 0);
    vb_handle::GraphKey key{img_d, loss_d, batch, img_h, img_w, s};
    key.flags = flags;
    run_graphed(h, key, [&] {
      if (h->bf16()) h->mim_forward<__nv_bfloat16>(img_d, batch, img_h, img_w, loss_d, flags, s);
      else h->mim_forward<float>(img_d, batch, img_h, img_w, loss_d, flags, s);
    });
    h->last_launches = launch_counter() - before;
    const vb_handle::MimPlan& p = h->mim_last;
    const size_t out_bytes = static_cast<size_t>(batch) * p.nm * h->patch_dim() * sizeof(float);
    const cudaMemcpyKind kind = out_mem == VB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (pred != nullptr) VB_CUDA(cudaMemcpyAsync(pred, h->mim_pred(), out_bytes, kind, s));
    if (masked_patches != nullptr) VB_CUDA(cudaMemcpyAsync(masked_patches, h->mim_patches(), out_bytes, kind, s));
    if (indices != nullptr) VB_CUDA(cudaMemcpyAsync(indices, h->mim_idx(), static_cast<size_t>(batch) * p.n * sizeof(int), kind, s));
    if (out_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(loss, loss_d, sizeof(float), cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_op_mim_mask(int32_t descending, int32_t B, int32_t n, uint64_t seed, uint64_t counter, int32_t* indices) {
  return guarded(nullptr, [&] {
    VB_CHECK(indices != nullptr && B > 0 && (descending == 0 || descending == 1), "vb_op_mim_mask: bad arguments");
    VB_CHECK(n >= 1 && n <= MIM_MAX_PATCHES, "vb_op_mim_mask: n = " + std::to_string(n) + " is outside 1 .. " + std::to_string(MIM_MAX_PATCHES) +
                                                 " (the patches per image the mask kernel sorts)");
    require_gpu();
    DevMem rng, idx;
    rng.ensure(3 * sizeof(unsigned long long));
    const unsigned long long v[3] = {static_cast<unsigned long long>(seed), static_cast<unsigned long long>(counter), 0ull};
    VB_CUDA(cudaMemcpy(rng.p, v, sizeof v, cudaMemcpyHostToDevice));
    idx.ensure(static_cast<size_t>(B) * n * sizeof(int));
    mim_mask(B, n, descending, static_cast<unsigned long long*>(rng.p), static_cast<int*>(idx.p), 0);
    VB_CUDA(cudaMemcpy(indices, idx.p, static_cast<size_t>(B) * n * sizeof(int), cudaMemcpyDeviceToHost));
    unsigned long long after[3];
    VB_CUDA(cudaMemcpy(after, rng.p, sizeof after, cudaMemcpyDeviceToHost));
    VB_CHECK(after[1] == counter + 1 && after[2] == 0, "vb_op_mim_mask: the mask kernel did not advance its counter once");
  });
}

int vb_forward_mpp(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* loss, float* logits,
                   int32_t* mask_ids, int32_t* source, int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && loss != nullptr, "vb_forward_mpp: null argument");
    VB_CHECK(h->cfg.kind == VB_KIND_MPP, "vb_forward_mpp: not a MPP handle");
    VB_CHECK(h->finalized, "vb_forward_mpp: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward_mpp: bad batch / image size");
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const size_t img_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const float* img_d = img;
    if (img_mem == VB_MEM_HOST) {
      h->img_dev.ensure(img_bytes);
      VB_CUDA(cudaMemcpyAsync(h->img_dev.p, img, img_bytes, cudaMemcpyHostToDevice, s));
      img_d = static_cast<const float*>(h->img_dev.p);
    }
    float* loss_d = loss;
    if (out_mem == VB_MEM_HOST) {
      h->logits_dev.ensure(sizeof(float));
      loss_d = static_cast<float*>(h->logits_dev.p);
    }
    h->mim_prepare(batch, img_h, img_w);
    const bool want_logits = logits != nullptr;
    vb_handle::GraphKey key{img_d, loss_d, batch, img_h, img_w, s};
    key.flags = want_logits ? 1 : 0;
    run_graphed(h, key, [&] {
      if (h->bf16()) h->mpp_forward<__nv_bfloat16>(img_d, batch, img_h, img_w, loss_d, want_logits, s);
      else h->mpp_forward<float>(img_d, batch, img_h, img_w, loss_d, want_logits, s);
    });
    h->last_launches = launch_counter() - before;
    const vb_handle::MimPlan& p = h->mim_last;
    const cudaMemcpyKind kind = out_mem == VB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (logits != nullptr)
      VB_CUDA(cudaMemcpyAsync(logits, h->mim_pred(), static_cast<size_t>(batch) * p.nm * h->mpp_classes() * sizeof(float), kind, s));
    if (mask_ids != nullptr)
      VB_CUDA(cudaMemcpy2DAsync(mask_ids, static_cast<size_t>(p.nm) * sizeof(int), h->mpp_ids(), static_cast<size_t>(p.n + 1) * sizeof(int),
                                static_cast<size_t>(p.nm) * sizeof(int), batch, kind, s));
    if (source != nullptr) VB_CUDA(cudaMemcpyAsync(source, h->mpp_src(), static_cast<size_t>(batch) * p.n * sizeof(int), kind, s));
    if (out_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(loss, loss_d, sizeof(float), cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_op_mpp_draws(int32_t B, int32_t n, int32_t k, double replace_prob, double random_patch_prob, uint64_t seed, uint64_t counter,
                    int32_t* mask_ids, int32_t* source) {
  return guarded(nullptr, [&] {
    VB_CHECK(mask_ids != nullptr && source != nullptr && B > 0, "vb_op_mpp_draws: bad arguments");
    VB_CHECK(n >= 1 && n <= MIM_MAX_PATCHES && k >= 1 && k <= n, "vb_op_mpp_draws: need 1 <= k <= n <= " + std::to_string(MIM_MAX_PATCHES));
    VB_CHECK(!(random_patch_prob > 0.0 && replace_prob == 1.0), "vb_op_mpp_draws: random_patch_prob / (1 - replace_prob) divides by zero");
    require_gpu();
    DevMem rng, idx, ids, src;
    rng.ensure(3 * sizeof(unsigned long long));
    const unsigned long long v[3] = {static_cast<unsigned long long>(seed), static_cast<unsigned long long>(counter), 0ull};
    VB_CUDA(cudaMemcpy(rng.p, v, sizeof v, cudaMemcpyHostToDevice));
    idx.ensure(static_cast<size_t>(B) * n * sizeof(int));
    ids.ensure(static_cast<size_t>(B) * k * sizeof(int));
    src.ensure(static_cast<size_t>(B) * n * sizeof(int));
    unsigned long long* r = static_cast<unsigned long long*>(rng.p);
    mim_mask(B, n, 1, r, static_cast<int*>(idx.p), 0);
    const double p_rand = random_patch_prob > 0.0 ? random_patch_prob / (1.0 - replace_prob) : 0.0;
    mpp_draws(B, n, k, static_cast<const int*>(idx.p), r, random_patch_prob, p_rand, replace_prob, static_cast<int*>(src.p),
              static_cast<int*>(ids.p), k, 0);
    VB_CUDA(cudaMemcpy(mask_ids, ids.p, static_cast<size_t>(B) * k * sizeof(int), cudaMemcpyDeviceToHost));
    VB_CUDA(cudaMemcpy(source, src.p, static_cast<size_t>(B) * n * sizeof(int), cudaMemcpyDeviceToHost));
  });
}

int vb_create_regionvit(const vb_config* base, const vb_regionvit_config* rc, int device, vb_handle** out) {
  return create_with("vb_create_regionvit", "vb_regionvit_config", VB_KIND_REGIONVIT, "VB_KIND_REGIONVIT", base, rc,
                                          device, out, validate_regionvit,
                                          [&](vb_handle& h) { h.rv = *rc; h.cfg.dim = rc->dims[VB_REGIONVIT_STAGES - 1]; });
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

namespace {
// vb_forward and vb_forward_train: `train` runs every dropout site with a rate > 0 (vb_handle::dropout) and advances the draw counter
int forward_entry(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
                  int32_t logits_mem, void* stream, bool train) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && logits != nullptr, "vb_forward: null argument");
    VB_CHECK(h->finalized, "vb_forward: call vb_finalize after setting the weights");
    VB_CHECK(!train || h->drop_set, "vb_forward_train: call vb_set_dropout first");
    VB_CHECK(!h->is_mim(), h->whole_forward_only(h->cfg.kind));
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
    if (h->cfg.kind == VB_KIND_ATS_VIT) h->ats_prepare(batch, img_h, img_w);
    vb_handle::GraphKey key{img_d, out_d, batch, img_h, img_w, s};
    struct Training {                                      // the flag holds while the launches are issued, exceptions included
      vb_handle* h;
      Training(vb_handle* hh, bool on) : h(hh) { h->training = on; }
      ~Training() { h->training = false; }
    } tr(h, train);
    key.flags = h->dropout_active() ? 2 : 0;               // all rates 0: the inference forward and its graph
    run_graphed(h, key, [&] {
      if (h->bf16()) h->forward_impl<__nv_bfloat16>(img_d, batch, img_h, img_w, out_d, s);
      else h->forward_impl<float>(img_d, batch, img_h, img_w, out_d, s);
    });
    h->last_launches = launch_counter() - before;
    if (logits_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(logits, out_d, out_bytes, cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}
}  // namespace

int vb_forward(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
               int32_t logits_mem, void* stream) {
  return forward_entry(h, img, img_mem, batch, img_h, img_w, logits, logits_mem, stream, false);
}

int vb_forward_train(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
                     int32_t logits_mem, void* stream) {
  return forward_entry(h, img, img_mem, batch, img_h, img_w, logits, logits_mem, stream, true);
}

int vb_set_dropout(vb_handle* h, float dropout, float emb_dropout, uint64_t seed) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr, "null handle");
    VB_CHECK(vb_handle::dropout_kind(h->cfg.kind) && !h->distill_wrapper,
             "vb_set_dropout: training-mode dropout runs on ViT, DeepViT, CaiT and CrossViT handles only");
    VB_CHECK(dropout >= 0.f && dropout < 1.f, "vb_set_dropout: dropout = " + std::to_string(dropout) + " is outside [0, 1)");
    VB_CHECK(emb_dropout >= 0.f && emb_dropout < 1.f, "vb_set_dropout: emb_dropout = " + std::to_string(emb_dropout) + " is outside [0, 1)");
    VB_CUDA(cudaSetDevice(h->device));
    VB_CUDA(cudaDeviceSynchronize());                    // no forward in flight reads the old key, counter or rates
    h->drop_dev.ensure(2 * sizeof(unsigned long long));
    const unsigned long long v[2] = {static_cast<unsigned long long>(seed), 0ull};
    VB_CUDA(cudaMemcpy(h->drop_dev.p, v, sizeof v, cudaMemcpyHostToDevice));
    VB_CUDA(cudaDeviceSynchronize());                    // a pageable copy may return before it lands
    h->drop_rate = dropout;
    h->emb_drop_rate = emb_dropout;
    h->drop_set = true;
    h->drop_graphs();                                    // the captured launches carry the rates
  });
}

int vb_op_dropout_mask(uint64_t seed, uint32_t draw, uint32_t site, int32_t M, int32_t N, float rate, uint8_t* keep) {
  return guarded(nullptr, [&] {
    VB_CHECK(keep != nullptr && M > 0 && N > 0, "vb_op_dropout_mask: bad arguments");
    VB_CHECK(rate >= 0.f && rate < 1.f, "vb_op_dropout_mask: rate outside [0, 1)");
    require_gpu();
    DevMem out;
    const size_t n = static_cast<size_t>(M) * N;
    out.ensure(n);
    dropout_mask(static_cast<unsigned long long>(seed), draw, site, M, N, rate, static_cast<uint8_t*>(out.p), 0);
    VB_CUDA(cudaMemcpy(keep, out.p, n, cudaMemcpyDeviceToHost));
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
    VB_CHECK(h->cfg.kind != VB_KIND_NEST, "vb_forward_distill: NesT has no distillation head");
    VB_CHECK(h->cfg.kind != VB_KIND_REGIONVIT, "vb_forward_distill: RegionViT has no distillation head");
    VB_CHECK(h->cfg.kind != VB_KIND_ATS_VIT, h->whole_forward_only(VB_KIND_ATS_VIT));
    VB_CHECK(h->cfg.kind != VB_KIND_SMALL_DATASET_VIT, h->whole_forward_only(VB_KIND_SMALL_DATASET_VIT));
    VB_CHECK(h->cfg.kind != VB_KIND_MOBILEVIT, h->whole_forward_only(VB_KIND_MOBILEVIT));
    VB_CHECK(h->cfg.kind != VB_KIND_SCALABLE_VIT, h->whole_forward_only(VB_KIND_SCALABLE_VIT));
    VB_CHECK(h->cfg.kind != VB_KIND_PIT, h->whole_forward_only(VB_KIND_PIT));
    VB_CHECK(!h->is_mim(), h->whole_forward_only(h->cfg.kind));
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

int vb_forward_distill_loss(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                            const float* labels, vb_handle* teacher, const float* teacher_logits, int32_t in_mem, double temperature,
                            double alpha, float* loss, float* student_logits, float* distill_logits, float* teacher_logits_out,
                            int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && img != nullptr && labels != nullptr && loss != nullptr, "vb_forward_distill_loss: null argument");
    VB_CHECK(h->distill_wrapper, "vb_forward_distill_loss: not a DistillWrapper handle (create it with vb_create_distill)");
    VB_CHECK(h->finalized, "vb_forward_distill_loss: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && img_h > 0 && img_w > 0, "vb_forward_distill_loss: bad batch / image size");
    VB_CHECK((teacher != nullptr) != (teacher_logits != nullptr), "vb_forward_distill_loss: pass exactly one of teacher and teacher_logits");
    VB_CHECK(temperature != 0.0, "DistillWrapper: temperature 0 divides the logits by zero (inf / NaN in the reference)");
    if (teacher != nullptr) {
      VB_CHECK(teacher != h, "vb_forward_distill_loss: the teacher must be another handle");
      VB_CHECK(teacher->device == h->device, "vb_forward_distill_loss: the teacher handle is on another device");
      VB_CHECK(!teacher->is_mim() && !teacher->distill_wrapper, "vb_forward_distill_loss: the teacher must be a classifier handle");
      VB_CHECK(teacher->cfg.num_classes == h->cfg.num_classes,
               "vb_forward_distill_loss: the teacher has " + std::to_string(teacher->cfg.num_classes) +
                   " classes; the teacher logits must be [b, num_classes] with num_classes = " + std::to_string(h->cfg.num_classes));
    }
    VB_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long before = launch_counter();
    const size_t img_bytes = static_cast<size_t>(batch) * img_h * img_w * h->cfg.channels * sizeof(float);
    const size_t row_bytes = static_cast<size_t>(batch) * h->cfg.num_classes * sizeof(float);
    const float* img_d = img;
    if (img_mem == VB_MEM_HOST) {                             // uploaded once: the teacher and the student read the same copy
      h->img_dev.ensure(img_bytes);
      VB_CUDA(cudaMemcpyAsync(h->img_dev.p, img, img_bytes, cudaMemcpyHostToDevice, s));
      img_d = static_cast<const float*>(h->img_dev.p);
    }
    h->distill_prepare(batch);
    const vb_handle::DistillPlan& p = h->dw_last;
    const float* labels_d = labels;
    if (in_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(h->dw(p.labels), labels, row_bytes, cudaMemcpyHostToDevice, s));
      labels_d = h->dw(p.labels);
    }
    const float* tlog_d = teacher_logits;
    if (teacher != nullptr) {
      // the teacher's own vb_forward, under its own graph rules, outside this handle's graph: a teacher that re-finalizes or
      // grows its arena cannot leave a stale capture here
      const int rc = vb_forward(teacher, img_d, VB_MEM_DEVICE, batch, img_h, img_w, h->dw(p.teacher), VB_MEM_DEVICE, stream);
      if (rc != 0) throw Error(rc, "vb_forward_distill_loss: the teacher's forward failed: " + teacher->error);
      tlog_d = h->dw(p.teacher);
    } else if (in_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(h->dw(p.teacher), teacher_logits, row_bytes, cudaMemcpyHostToDevice, s));
      tlog_d = h->dw(p.teacher);
    }
    float* loss_d = out_mem == VB_MEM_HOST ? h->dw(p.loss) : loss;
    // the optional outputs are copied from dw_dev after the launches, so they do not change what is captured
    vb_handle::GraphKey key{img_d, loss_d, batch, img_h, img_w, s};
    key.labels = labels_d;
    key.teacher = tlog_d;
    memcpy(&key.t_bits, &temperature, sizeof temperature);
    memcpy(&key.alpha_bits, &alpha, sizeof alpha);
    run_graphed(h, key, [&] {
      if (h->bf16()) h->distill_loss_forward<__nv_bfloat16>(img_d, batch, img_h, img_w, labels_d, tlog_d, temperature, alpha, loss_d, s);
      else h->distill_loss_forward<float>(img_d, batch, img_h, img_w, labels_d, tlog_d, temperature, alpha, loss_d, s);
    });
    h->last_launches = launch_counter() - before;
    const cudaMemcpyKind kind = out_mem == VB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (student_logits != nullptr) VB_CUDA(cudaMemcpyAsync(student_logits, h->dw(p.student), row_bytes, kind, s));
    if (distill_logits != nullptr) VB_CUDA(cudaMemcpyAsync(distill_logits, h->dw(p.dlogits), row_bytes, kind, s));
    if (teacher_logits_out != nullptr) VB_CUDA(cudaMemcpyAsync(teacher_logits_out, tlog_d, row_bytes, kind, s));
    if (out_mem == VB_MEM_HOST) {
      VB_CUDA(cudaMemcpyAsync(loss, loss_d, static_cast<size_t>(batch) * sizeof(float), cudaMemcpyDeviceToHost, s));
      VB_CUDA(cudaStreamSynchronize(s));
    }
  });
}

int vb_op_distill_loss(const float* student_logits, const float* labels, const float* teacher_logits, int32_t B, int32_t K,
                       double temperature, double alpha, float* out) {
  return guarded(nullptr, [&] {
    VB_CHECK(student_logits && labels && teacher_logits && out && B > 0 && K > 0, "vb_op_distill_loss: bad arguments");
    VB_CHECK(temperature != 0.0, "DistillWrapper: temperature 0 divides the logits by zero (inf / NaN in the reference)");
    require_gpu();
    const size_t rows = static_cast<size_t>(B) * K;
    DevMem dS, dY, dT, dw;
    const float* s_d = upload<float>(dS, student_logits, rows);
    const float* y_d = upload<float>(dY, labels, rows);
    const float* t_d = upload<float>(dT, teacher_logits, rows);
    dw.ensure(2 * static_cast<size_t>(B) * sizeof(double) + (static_cast<size_t>(B) + 64) * sizeof(float));
    double* ce = static_cast<double*>(dw.p);
    float* dterm = reinterpret_cast<float*>(ce + 2 * static_cast<size_t>(B));
    float* o_d = dterm + 64;
    distill_loss(s_d, y_d, t_d, B, K, temperature, alpha, ce, ce + B, dterm, o_d, 0);
    VB_CUDA(cudaMemcpy(out, o_d, static_cast<size_t>(B) * sizeof(float), cudaMemcpyDeviceToHost));
  });
}

int vb_forward_tokens(vb_handle* h, const float* tokens, int32_t tokens_mem, int32_t batch, int32_t n, float* out,
                      int32_t out_mem, void* stream) {
  return guarded(h, [&] {
    VB_CHECK(h != nullptr && tokens != nullptr && out != nullptr, "vb_forward_tokens: null argument");
    VB_CHECK(h->finalized, "vb_forward_tokens: call vb_finalize after setting the weights");
    VB_CHECK(batch > 0 && n > 0, "vb_forward_tokens: bad shape");
    h->check_stage_entries();
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
    VB_CHECK(h->cfg.kind != VB_KIND_SMALL_DATASET_VIT, h->whole_forward_only(VB_KIND_SMALL_DATASET_VIT));
    VB_CHECK(h->cfg.kind != VB_KIND_MOBILEVIT, h->whole_forward_only(VB_KIND_MOBILEVIT));
    VB_CHECK(h->cfg.kind != VB_KIND_SCALABLE_VIT, h->whole_forward_only(VB_KIND_SCALABLE_VIT));
    VB_CHECK(h->cfg.kind != VB_KIND_PIT, h->whole_forward_only(VB_KIND_PIT));
    VB_CHECK(!h->is_mim(), h->whole_forward_only(h->cfg.kind));
    VB_CHECK(h->cfg.kind != VB_KIND_CROSSVIT && h->cfg.kind != VB_KIND_T2T_VIT && h->cfg.kind != VB_KIND_CCT &&
             h->cfg.kind != VB_KIND_LEVIT && h->cfg.kind != VB_KIND_CVT && h->cfg.kind != VB_KIND_TWINS_SVT &&
             h->cfg.kind != VB_KIND_CROSSFORMER && h->cfg.kind != VB_KIND_NEST && h->cfg.kind != VB_KIND_REGIONVIT,
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
    h->check_stage_entries();
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
    DevMem dA, dW, dB, dS, dR, dO;
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    const float* ds = scale ? upload<float>(dS, scale, N) : nullptr;
    const float* dw = upload<float>(dW, w, static_cast<size_t>(K) * N);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      if (h.bf16()) VB_CHECK(gemm_bf16_supported(M, N, K, K, K, N), "vb_op_linear(bf16): need N % 64 == 0 and K % 8 == 0");
      const T* da = upload<T>(dA, a, static_cast<size_t>(M) * K);
      Epi e;
      e.bias = db; e.scale = ds; e.gelu = gelu != 0; e.ldr = N;
      e.res = res ? upload<T>(dR, res, static_cast<size_t>(M) * N) : nullptr;
      const Linear L = h.pack_linear(dw, db, K, N, K, nullptr);
      dO.ensure(static_cast<size_t>(M) * N * sizeof(T));
      T* dout = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] { h.linear<T>(da, K, M, L, dout, N, e, 0); });
      download<T>(dout, out, static_cast<size_t>(M) * N);
    });
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
    DevMem dQ, dK, dV, dO, dMa, dMb, dG, dBt;
    const float* ma = mix_a ? upload<float>(dMa, mix_a, heads * heads) : nullptr;
    const float* mb = mix_b ? upload<float>(dMb, mix_b, heads * heads) : nullptr;
    const float* g = ln_gamma ? upload<float>(dG, ln_gamma, heads) : nullptr;
    const float* bt = ln_beta ? upload<float>(dBt, ln_beta, heads) : nullptr;
    const MixCacheScope mix_scope{{ma, mb, g, bt}};
    const size_t cq = static_cast<size_t>(B) * nq * inner, ck = static_cast<size_t>(B) * nk * inner;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* q_d = upload<T>(dQ, q, cq);
      const T* k_d = upload<T>(dK, k, ck);
      const T* v_d = upload<T>(dV, v, ck);
      dO.ensure(cq * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_dispatch<T>(q_d, inner, k_d, inner, v_d, inner, o_d, inner, B, nq, nk, heads, dim_head, variant, ma, mb, g, bt, 0);
      });
      download<T>(o_d, out, cq);
    });
  });
}

int vb_op_patch_merger(int32_t precision, const float* x, const float* gamma, const float* beta, const float* queries, float* out,
                       int32_t B, int32_t n, int32_t D, int32_t nt, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && queries && out && B > 0 && n > 0 && D > 0 && nt > 0, "vb_op_patch_merger: bad arguments");
    DevMem dX, dG, dB, dQf;
    const Norm norm{upload<float>(dG, gamma, D), upload<float>(dB, beta, D), D};
    const float* qf = upload<float>(dQf, queries, static_cast<size_t>(nt) * D);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, static_cast<size_t>(B) * n * D);
      const T* o_d = nullptr;
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        o_d = h.patch_merge<T>(x_d, B, n, D, norm, qf, nt, 0);
      });
      download<T>(o_d, out, static_cast<size_t>(B) * nt * D);
    });
  });
}

int vb_op_layernorm(int32_t precision, const float* x, const float* gamma, const float* beta, float* out, int32_t M, int32_t D,
                    int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && out && M > 0 && D > 0, "vb_op_layernorm: bad arguments");
    DevMem dX, dG, dB, dO;
    const Norm norm{upload<float>(dG, gamma, D), upload<float>(dB, beta, D), D};
    const size_t cnt = static_cast<size_t>(M) * D;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, cnt);
      dO.ensure(cnt * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] { h.ln<T>(x_d, norm, o_d, M, D, 0); });
      download<T>(o_d, out, cnt);
    });
  });
}

int vb_op_ln_linear(const float* x, const float* gamma, const float* beta, const float* w, const float* bias, int32_t gelu,
                    float* out, int32_t M, int32_t N, int32_t K, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && w && out && M > 0 && N > 0 && K > 0, "vb_op_ln_linear: bad arguments");
    VB_CHECK(N % 64 == 0 && K % 64 == 0, "vb_op_ln_linear: the folded form needs N % 64 == 0 and K % 64 == 0");
    using bf = __nv_bfloat16;
    vb_handle h{};
    h.cfg.precision = VB_PRECISION_BF16;
    DevMem dX, dG, dBt, dW, dB, dO;
    const bf* dx = upload<bf>(dX, x, static_cast<size_t>(M) * K);
    const Norm norm{upload<float>(dG, gamma, K), upload<float>(dBt, beta, K), K};
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    const Linear L = h.pack_linear(upload<float>(dW, w, static_cast<size_t>(K) * N), db, K, N, K, &norm);
    float* st = h.row_stats(M, K);
    dO.ensure(static_cast<size_t>(M) * N * 2);
    bf* dout = static_cast<bf*>(dO.p);
    Epi e;
    e.bias = L.ln_c2; e.ln_stats = st; e.gelu = gelu != 0;
    timed(iters, elapsed_ms, [&] { h.ensure_stats<bf>(dx, K, st, M, 0); h.linear<bf>(dx, K, M, L, dout, N, e, 0); });
    download<bf>(dout, out, static_cast<size_t>(M) * N);
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
    const int act = gelu == 0 ? ACT_NONE : gelu == ACT_SILU ? ACT_SILU : ACT_GELU;   // any other nonzero value: GELU, as it always was
    GemmBf16 g = gemm_bf16_plan(da, lda, dw, ldw, static_cast<__nv_bfloat16*>(dout), ldc, M, N, K, db, ds, dr, ldr, act,
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
    DevMem dQ, dKV, dO, dMa, dMb, dG, dBt;
    const float* ma = mix_a ? upload<float>(dMa, mix_a, heads * heads) : nullptr;
    const float* mb = mix_b ? upload<float>(dMb, mix_b, heads * heads) : nullptr;
    const float* g = ln_gamma ? upload<float>(dG, ln_gamma, heads) : nullptr;
    const float* bt = ln_beta ? upload<float>(dBt, ln_beta, heads) : nullptr;
    const MixCacheScope mix_scope{{ma, mb, g, bt}};
    const size_t cq = static_cast<size_t>(B) * nq * ldq, ckv = static_cast<size_t>(B) * nk * ldk, co = static_cast<size_t>(B) * nq * ldo;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* q_d = upload<T>(dQ, q, cq);
      const T* kv_d = fused ? q_d : upload<T>(dKV, kv, ckv);
      T* o_d = upload<T>(dO, out, co);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_dispatch<T>(q_d, ldq, kv_d + k_off, ldk, kv_d + v_off, ldk, o_d, ldo, B, nq, nk, heads, dh, variant, ma, mb, g, bt, 0,
                                scale);
      });
      download<T>(o_d, out, co);
    });
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
    DevMem dQ, dK, dV, dO;
    const size_t cq = static_cast<size_t>(B) * nq * ldq, co = static_cast<size_t>(B) * nq * ldo;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      PosBias pb;
      pb.table = h.upload_owned(vb_handle::levit_pos_table(std::vector<double>(pos_bias, pos_bias + static_cast<size_t>(f2) * heads), f2, heads,
                                                           1.0 / scale));
      pb.fmap = fmap; pb.step = q_step; pb.gelu_out = gelu_out != 0;
      const T* q_d = upload<T>(dQ, q, cq);
      const T* k_d = upload<T>(dK, k, static_cast<size_t>(B) * nk * ldk);
      const T* v_d = upload<T>(dV, v, static_cast<size_t>(B) * nk * ldv);
      T* o_d = upload<T>(dO, out, co);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_bias<T>(q_d, ldq, k_d, ldk, v_d, ldv, o_d, ldo, B, nq, nk, heads, dh, scale, pb, 0);
      });
      download<T>(o_d, out, co);
    });
  });
}

int vb_op_dwconv(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* ln_gamma, const float* ln_beta,
                 int32_t k, int32_t kv_stride, const float* wq, const float* bn_q, const float* wkv, const float* bn_kv, float* q, float* kv,
                 int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && ln_gamma && ln_beta && wq && bn_q && wkv && bn_kv && q && kv && B > 0 && H > 0 && W > 0 && C > 0 && k >= 1 && k <= 7 &&
             (kv_stride == 1 || kv_stride == 2), "vb_op_dwconv: bad arguments");
    const bool bf = precision != VB_PRECISION_FP32;               // as with_precision picks the element type
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
    DevMem dX, dG, dB, dTq, dSq, dTkv, dSkv, dQ, dKV;
    CvtBlockW b;
    b.dim = C; b.dp = Cp; b.k = k; b.kv_stride = kv_stride;
    b.attn_norm = Norm{upload<float>(dG, gp.data(), Cp), upload<float>(dB, bp.data(), Cp), C};
    b.wq = upload<float>(dTq, tq.data(), tq.size());
    b.bq = upload<float>(dSq, sq.data(), sq.size());
    b.wkv = upload<float>(dTkv, tkv.data(), tkv.size());
    b.bkv = upload<float>(dSkv, skv.data(), skv.size());
    std::vector<float> qh(M * Cp), kvh(Mk * Cp);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      T* x_d = upload<T>(dX, xp.data(), M * Cp);
      dQ.ensure(M * Cp * sizeof(T));
      dKV.ensure(Mk * Cp * sizeof(T));
      T* q_d = static_cast<T*>(dQ.p);
      T* kv_d = static_cast<T*>(dKV.p);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        float* st = h.row_stats(static_cast<long long>(M), Cp);
        h.ensure_stats<T>(x_d, Cp, st, static_cast<int>(M), 0);
        h.cvt_dwconv<T>(h.prenorm<T>(x_d, static_cast<int>(M), C, Cp, st, 1e-5f, 0), B, H, W, b, q_d, kv_d, 0);
      });
      download<T>(q_d, qh.data(), M * Cp);
      download<T>(kv_d, kvh.data(), Mk * Cp);
    });
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
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_dispatch<T>(x_d, ld, x_d + HD, ld, x_d + 2 * HD, ld, o_d, ldo, Bw, n, n, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, 0,
                                0.f, &win);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    });
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
    DevMem dX, dO, dT;
    PosBias pb;
    pb.table = upload<float>(dT, table, t); pb.wsz = wsz;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.attention_dispatch<T>(x_d, ld, x_d + HD, ld, x_d + 2 * HD, ld, o_d, ldo, Bw, n, n, heads, dh, 0, nullptr, nullptr, nullptr, nullptr, 0,
                                0.f, &win, &pb);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    });
  });
}

int vb_op_block_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t bh, int32_t bw,
                          int32_t heads, int32_t dh, float* out, int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && out && B > 0 && bh > 0 && bw > 0 && H > 0 && W > 0 && H % bh == 0 && W % bw == 0 && heads > 0 && dh > 0 && ld >= 3 * HD &&
             ldo >= HD, "vb_op_block_attention: bad arguments");
    Window win;
    win.p = bh; win.pw = bw; win.nx = W / bw; win.ny = H / bh; win.count = B * win.nx * win.ny;
    const long long rows = static_cast<long long>(B) * H * W;
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.block_attention<T>(x_d, ld, o_d, ldo, heads, dh, win, 0);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    });
  });
}

int vb_op_mv2_dwconv(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, const float* w,
                     const float* bn, float* out, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && w && bn && out && B > 0 && H > 0 && W > 0 && C > 0 && (stride == 1 || stride == 2), "vb_op_mv2_dwconv: bad arguments");
    const bool bf = precision != VB_PRECISION_FP32;               // as with_precision picks the element type
    const int Cp = bf ? round_up(C, 64) : C, Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    const size_t M = static_cast<size_t>(B) * H * W, Mo = static_cast<size_t>(B) * Ho * Wo;
    auto vec = [](const float* p, size_t n) { return std::vector<double>(p, p + n); };
    std::vector<double> wd, sd;                                   // as vb_finalize folds it
    cvt_fold_dw(vec(w, static_cast<size_t>(9) * C), vec(bn, C), vec(bn + C, C), vec(bn + 2 * C, C), vec(bn + 3 * C, C), 3, C, Cp, wd, sd);
    const std::vector<float> taps(wd.begin(), wd.end()), shift(sd.begin(), sd.end());
    std::vector<float> xp(M * Cp, 0.f);
    for (size_t r = 0; r < M; ++r) std::copy(x + r * C, x + (r + 1) * C, xp.begin() + r * Cp);
    DevMem dX, dT, dS, dO;
    const float* t_d = upload<float>(dT, taps.data(), taps.size());
    const float* s_d = upload<float>(dS, shift.data(), shift.size());
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, xp.data(), M * Cp);
      dO.ensure(Mo * Cp * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] { dwconv_bn_act<T>(x_d, Cp, t_d, s_d, o_d, Cp, B, H, W, C, Cp, stride, 0); });
      (void)h;
      download<T>(o_d, out, Mo * Cp);
    });
  });
}

int vb_op_patch_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t ph, int32_t pw,
                          int32_t heads, int32_t dh, float scale, float* out, int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh;
    VB_CHECK(qkv && out && B > 0 && ph > 0 && pw > 0 && H > 0 && W > 0 && H % ph == 0 && W % pw == 0 && heads > 0 && dh > 0 && ld >= 3 * HD &&
             ldo >= HD, "vb_op_patch_attention: bad arguments");
    Window win;                                                   // as mobilevit_block builds it
    win.p = H / ph; win.pw = W / pw; win.ny = ph; win.nx = pw; win.dilated = 1; win.count = B * ph * pw;
    const long long rows = static_cast<long long>(B) * H * W;
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.block_attention<T>(x_d, ld, o_d, ldo, heads, dh, win, 0, scale);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    });
  });
}

int vb_op_r2l_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t lh, int32_t lw, int32_t rh, int32_t rw,
                        int32_t heads, int32_t dh, const float* table, int32_t window_size, float* out, int32_t ldo, int32_t iters,
                        float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    const int HD = heads * dh, ws = window_size;
    VB_CHECK(qkv && table && out && B > 0 && lh > 0 && lw > 0 && rh > 0 && rw > 0 && lh % rh == 0 && lw % rw == 0 && heads > 0 && dh > 0 &&
             ws > 0 && ws <= 1024 && lh / rh <= ws && lw / rw <= ws && ld >= 3 * HD && ldo >= HD, "vb_op_r2l_attention: bad arguments");
    Window win;
    win.p = lh / rh; win.pw = lw / rw; win.nx = rw; win.ny = rh; win.count = B * rh * rw;
    const long long Ml = static_cast<long long>(B) * lh * lw, rows = Ml + static_cast<long long>(B) * rh * rw;
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      PosBias pb;
      pb.table = h.upload_owned(r2l_table_from_embedding(table, ws, heads));   // transposed as vb_finalize does
      pb.r2l_ws = ws; pb.r2l_h = win.p; pb.r2l_w = win.pw;
      const T* x_d = upload<T>(dX, qkv, static_cast<size_t>(rows) * ld);
      T* o_d = upload<T>(dO, out, static_cast<size_t>(rows) * ldo);
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        h.r2l_attention<T>(x_d, ld, o_d, ldo, Ml, pb, win, 0, heads, dh);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * ldo);
    });
  });
}

int vb_op_nest_aggregate(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* gamma, const float* beta,
                         const float* pos, int32_t bh, int32_t bw, float* out, float* stats_out, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && out && B > 0 && H > 0 && W > 0 && C > 0, "vb_op_nest_aggregate: bad arguments");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    VB_CHECK(pos == nullptr || (bh > 0 && bw > 0 && Ho % bh == 0 && Wo % bw == 0), "vb_op_nest_aggregate: the pooled map is not whole blocks");
    const bool bf = precision != VB_PRECISION_FP32;               // as with_precision picks the element type
    const int Cp = bf ? round_up(C, 64) : C;
    const size_t M = static_cast<size_t>(B) * H * W, Mo = static_cast<size_t>(B) * Ho * Wo;
    std::vector<float> xp(M * Cp, 0.f), gp(Cp, 0.f), bp(Cp, 0.f), oh(Mo * Cp), sh(Mo * (Cp / 64 + 1) * 2, 0.f);
    for (size_t r = 0; r < M; ++r) std::copy(x + r * C, x + (r + 1) * C, xp.begin() + r * Cp);
    std::copy(gamma, gamma + C, gp.begin());
    std::copy(beta, beta + C, bp.begin());
    DevMem dX, dG, dB, dP, dO;
    const Norm norm{upload<float>(dG, gp.data(), Cp), upload<float>(dB, bp.data(), Cp), C};
    const float* p_d = pos ? upload<float>(dP, pos, static_cast<size_t>(bh) * bw) : nullptr;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, xp.data(), M * Cp);
      dO.ensure(Mo * Cp * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      float* so = nullptr;
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        float* st = h.row_stats(static_cast<long long>(M), Cp);
        so = h.row_stats(static_cast<long long>(Mo), Cp);
        h.ensure_stats<T>(x_d, Cp, st, static_cast<int>(M), 0);
        h.nest_aggregate_tail<T>(x_d, st, B, H, W, C, Cp, norm, p_d, bh, bw, o_d, so, 0);
      });
      if (so) VB_CUDA(cudaMemcpy(sh.data(), so, Mo * (Cp / 64) * 2 * sizeof(float), cudaMemcpyDeviceToHost));
      download<T>(o_d, oh.data(), Mo * Cp);
    });
    for (size_t r = 0; r < Mo; ++r) std::copy(oh.begin() + r * Cp, oh.begin() + r * Cp + C, out + r * C);
    if (bf && stats_out != nullptr) std::copy(sh.begin(), sh.begin() + Mo * (Cp / 64) * 2, stats_out);
  });
}

int vb_op_conv2d(int32_t precision, const float* x, int32_t image, int32_t B, int32_t H, int32_t W, int32_t cin, int32_t ld, int32_t off,
                 const float* kernel, const float* bias, int32_t N, int32_t k, int32_t stride, int32_t valid, const float* ln_gamma,
                 const float* ln_beta, float ln_eps, int32_t gelu_in, int32_t act, const float* res, int32_t ldr, float* out,
                 float* stats_out, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && kernel && out && B > 0 && H > 0 && W > 0 && cin > 0 && N > 0 && k > 0 && stride > 0, "vb_op_conv2d: bad arguments");
    VB_CHECK(image ? (ld == cin && off == 0) : (off >= 0 && ld >= off + cin), "vb_op_conv2d: the map's channels [off, off + cin) exceed ld");
    VB_CHECK((ln_gamma == nullptr) == (ln_beta == nullptr), "vb_op_conv2d: the LayerNorm needs both gamma and beta");
    const bool ln = ln_gamma != nullptr;
    VB_CHECK(!image || (!ln && !gelu_in), "vb_op_conv2d: the LayerNorm and GELU on load read a token map, not the image");
    VB_CHECK(!ln || (off == 0 && ln_eps > 0.f), "vb_op_conv2d: the LayerNorm needs off == 0 and eps > 0");
    VB_CHECK(act >= ACT_NONE && act <= ACT_SILU, "vb_op_conv2d: act must be 0 (none), 1 (GELU), 2 (hard-swish) or 3 (SiLU)");
    VB_CHECK(!valid || (H >= k && W >= k), "vb_op_conv2d: a VALID window larger than the map");
    const bool bf = precision != VB_PRECISION_FP32;               // as with_precision picks the element type
    VB_CHECK(res == nullptr || ldr >= N, "vb_op_conv2d: ldr < N");
    VB_CHECK(stats_out == nullptr || !bf || N % 64 == 0, "vb_op_conv2d: output statistics need N % 64 == 0");
    const long long M = static_cast<long long>(B) * H * W;
    // the token map at the pitch the engine's zero-padded rows have: whole 64-column chunks in bf16, as row_stats reads them
    const int P = image ? cin : bf ? round_up(ld, 64) : ld;
    if (ln)                                                       // the row statistics sum every column: past cin, the pad's zeros
      for (long long r = 0; r < M; ++r)
        for (int c = cin; c < ld; ++c) VB_CHECK(x[r * ld + c] == 0.f, "vb_op_conv2d: with the LayerNorm, columns [cin, ld) must be zero");
    const int oh = valid ? (H - k) / stride + 1 : (H + stride - 1) / stride, ow = valid ? (W - k) / stride + 1 : (W + stride - 1) / stride;
    const long long rows = static_cast<long long>(B) * oh * ow;
    const int K = k * k * cin;
    std::vector<float> xp(static_cast<size_t>(M) * P, 0.f);
    for (long long r = 0; r < M; ++r) std::copy(x + r * (image ? cin : ld), x + (r + 1) * (image ? cin : ld), xp.begin() + r * P);
    DevMem dX, dW, dB, dG, dBt, dR, dO;
    const float* dw = upload<float>(dW, kernel, static_cast<size_t>(K) * N);
    const float* db = bias ? upload<float>(dB, bias, N) : nullptr;
    const float* g_d = ln ? upload<float>(dG, ln_gamma, cin) : nullptr;
    const float* b_d = ln ? upload<float>(dBt, ln_beta, cin) : nullptr;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const Linear L = h.pack_linear(dw, db, K, N, round_up(K, 8), nullptr);   // as make_linear packs it
      const float* img_d = image ? upload<float>(dX, xp.data(), xp.size()) : nullptr;
      const T* map_d = image ? nullptr : upload<T>(dX, xp.data(), xp.size());
      const T* r_d = res ? upload<T>(dR, res, static_cast<size_t>(rows) * ldr) : nullptr;
      dO.ensure(static_cast<size_t>(rows) * N * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      float* so = nullptr;
      timed(iters, elapsed_ms, [&] {
        h.arena.reset();
        UnfoldMode um;
        um.valid = valid != 0;
        um.gelu = gelu_in != 0;
        const T* src = map_d ? map_d + off : nullptr;
        if (ln && h.bf16()) {                                     // the LayerNorm on load from the map's row statistics
          float* st = h.row_stats(M, P);
          h.ensure_stats<T>(map_d, P, st, static_cast<int>(M), 0);
          um.stats = st; um.parts = P / 64; um.d = cin; um.eps = ln_eps; um.gamma = g_d; um.beta = b_d;
        } else if (ln) {                                          // fp32: a separate LayerNorm into scratch first
          T* Z = h.arena.get<T>(static_cast<size_t>(M) * P);
          layernorm<T>(map_d, P, g_d, b_d, Z, P, static_cast<int>(M), cin, 0, P, ln_eps);
          src = Z;
        }
        so = stats_out && h.bf16() ? h.row_stats(rows, N) : nullptr;
        h.conv<T>(img_d, src, P, B, H, W, cin, k, stride, L, o_d, so, 0, &um, act, r_d, ldr);
      });
      download<T>(o_d, out, static_cast<size_t>(rows) * N);
      if (so) VB_CUDA(cudaMemcpy(stats_out, so, static_cast<size_t>(N / 64) * rows * 2 * sizeof(float), cudaMemcpyDeviceToHost));
    });
  });
}

int vb_op_cct_pool(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, int32_t stride,
                   const float* pos, int32_t rows, float* out, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && out && B > 0 && H > 0 && W > 0 && C > 0 && k > 0 && stride > 0 && rows > 0, "vb_op_cct_pool: bad arguments");
    const int oh = (H + stride - 1) / stride, ow = (W + stride - 1) / stride;
    VB_CHECK(rows >= oh * ow, "vb_op_cct_pool: fewer output rows than pooled positions");
    const size_t ci = static_cast<size_t>(B) * H * W * C, co = static_cast<size_t>(B) * rows * C;
    DevMem dX, dP, dO;
    const float* p_d = pos ? upload<float>(dP, pos, static_cast<size_t>(oh) * ow * C) : nullptr;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, ci);
      dO.ensure(co * sizeof(T));
      T* o_d = static_cast<T*>(dO.p);
      timed(iters, elapsed_ms, [&] { maxpool_relu_same<T>(x_d, o_d, B, H, W, C, k, stride, p_d, rows, 0); });
      (void)h;
      download<T>(o_d, out, co);
    });
  });
}

int vb_op_seq_pool(int32_t precision, const float* x, int32_t B, int32_t n, int32_t D, const float* gamma, const float* beta,
                   const float* pw, const float* pb, float* z, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && gamma && beta && pw && pb && z && B > 0 && n >= 0 && D > 0, "vb_op_seq_pool: bad arguments");
    DevMem dX, dG, dB, dPw, dPb, dZ;
    const float* g_d = upload<float>(dG, gamma, D);
    const float* b_d = upload<float>(dB, beta, D);
    const float* pw_d = upload<float>(dPw, pw, D);
    const float* pb_d = upload<float>(dPb, pb, 1);
    dZ.ensure(static_cast<size_t>(B) * D * sizeof(float));
    float* z_d = static_cast<float*>(dZ.p);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, static_cast<size_t>(B) * n * D);
      timed(iters, elapsed_ms, [&] { seq_pool<T>(x_d, n, D, g_d, b_d, pw_d, pb_d, z_d, B, 0); });   // refuses D > 1024 and n == 0
      (void)h;
    });
    download<float>(z_d, z, static_cast<size_t>(B) * D);
  });
}

int vb_op_pool_layernorm(int32_t precision, const float* x, int32_t B, int32_t n, int32_t ldx, int32_t D, const float* gamma,
                         const float* beta, int32_t mean_pool, float* z, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && z && B > 0 && n > 0 && D > 0 && ldx >= D, "vb_op_pool_layernorm: bad arguments");
    VB_CHECK((gamma == nullptr) == (beta == nullptr), "vb_op_pool_layernorm: the LayerNorm needs both gamma and beta");
    DevMem dX, dG, dB, dZ;
    const float* g_d = gamma ? upload<float>(dG, gamma, D) : nullptr;
    const float* b_d = beta ? upload<float>(dB, beta, D) : nullptr;
    dZ.ensure(static_cast<size_t>(B) * D * sizeof(float));
    float* z_d = static_cast<float*>(dZ.p);
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, static_cast<size_t>(B) * n * ldx);
      timed(iters, elapsed_ms, [&] { pool_layernorm<T>(x_d, n, ldx, g_d, b_d, z_d, B, D, mean_pool != 0, 0); });
      (void)h;
    });
    download<float>(z_d, z, static_cast<size_t>(B) * D);
  });
}

int vb_op_gather_grid(int32_t precision, const float* x, int32_t ldi, int32_t B, int32_t H, int32_t W, int32_t C, int32_t step, float* out,
                      int32_t ldo, int32_t iters, float* elapsed_ms) {
  return guarded(nullptr, [&] {
    require_gpu();
    VB_CHECK(x && out && B > 0 && H > 0 && W > 0 && C > 0 && step > 0 && ldi >= C && ldo >= C, "vb_op_gather_grid: bad arguments");
    const size_t ci = static_cast<size_t>(B) * H * W * ldi, co = static_cast<size_t>(B) * ((H + step - 1) / step) * ((W + step - 1) / step) * ldo;
    DevMem dX, dO;
    with_precision(precision, [&](vb_handle& h, auto tag) {
      using T = decltype(tag);
      const T* x_d = upload<T>(dX, x, ci);
      T* o_d = upload<T>(dO, out, co);
      timed(iters, elapsed_ms, [&] { gather_grid<T>(x_d, ldi, o_d, ldo, B, H, W, C, step, 0); });
      (void)h;
      download<T>(o_d, out, co);
    });
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
