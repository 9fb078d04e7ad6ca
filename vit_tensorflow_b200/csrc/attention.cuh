// Attention entry points: the generic materialised-scores path (any shape / variant, both precisions) and the
// fused fast path (bf16; returns false when the shape is not covered so the caller falls back to generic).
#pragma once
#include "common.h"

#include <vector>

namespace vb {

// Which branch of the dispatch ran the most recent attention call of the calling thread (vb_last_attention_path): every
// branch notes itself when it launches, so a test can tell which kernels served a shape.  Values as in include/vitb200.h.
enum AttentionPath { ATTN_PATH_NONE = 0, ATTN_PATH_FLASH = 1, ATTN_PATH_CLS = 2, ATTN_PATH_ROWS = 3, ATTN_PATH_MID_FUSED = 4,
                     ATTN_PATH_SIMT = 5 };
void note_attention_path(AttentionPath p);
int take_last_attention_path();                  // and reset it to ATTN_PATH_NONE

// variant 0: softmax(QK^T*scale)V                   (vit.py:77-82, cross_vit.py:87-91)
// variant 1: DeepViT re-attention: softmax -> head mix (mix_a [h,h]) -> LayerNorm over heads (deepvit.py:79-87)
// variant 2: CaiT talking heads: mix_a before softmax, mix_b after (cait.py:121-127)
// scale: softmax scale; <= 0 means dh^-0.5 (vit.py:57).  A layer whose heads were zero-padded to the kernels' head width
// (engine.cu: dh 48 -> 64) passes its true dim_head^-0.5 here.  pb (variant 0 only, may be null): LeViT's relative-position
// bias and output GELU (common.h), or CrossFormer's window table (PosBias::wsz > 0, B windows of nq == nk == wsz^2 window-major
// rows).  win (attention_fast only, may be null): windowed attention in the map's own rows, B = the number of windows and
// nq == nk == p^2 (common.h); with pb (the window-table form, dh 32 or 64) CrossFormer's windowed-bias flash kernel.
template <typename T>
void attention_generic(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, float* S, int B, int nq,
                       int nk, int heads, int dh, int variant, const float* mix_a, const float* mix_b, const float* ln_gamma,
                       const float* ln_beta, cudaStream_t s, float scale = 0.f, const PosBias* pb = nullptr);

template <typename T>
bool attention_fast(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, int B, int nq, int nk,
                    int heads, int dh, int variant, const float* mix_a, const float* mix_b, const float* ln_gamma,
                    const float* ln_beta, cudaStream_t s, float scale = 0.f, const PosBias* pb = nullptr,
                    const Window* win = nullptr);

// The talking-heads / re-attention path keeps host copies of the head-mix weights keyed by their device pointers (one process-
// wide cache for all handles); whoever frees or rewrites such weights (vb_finalize, vb_destroy, the op-level test entries) must
// erase the entries that name any of those pointers -- and only those: another handle's entries must survive, because a miss
// inside that handle's graph capture would make the capture fail.
void attention_mix_cache_erase(const std::vector<const void*>& ptrs);

// Tensor-core (mma.sync) + fused-middle version of attention_generic for the bf16 engine; false if the shape is not covered.
bool attention_generic_mma(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                           __nv_bfloat16* out, int ldo, float* S, int B, int nq, int nk, int heads, int dh, int variant,
                           const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, cudaStream_t s,
                           float scale = 0.f, const PosBias* pb = nullptr);

// Head-mix weights as kernel parameters (heads <= 16): wa = pre-softmax mix (CaiT) / re-attention weights (DeepViT), wb = CaiT's
// post-softmax mix, both [h][g] with row pitch `heads`; gamma / beta = DeepViT's LayerNorm over heads.
struct MixParams {
  float wa[256];
  float wb[256];
  float gamma[16], beta[16];
};
bool attention_mix_params(const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, int heads,
                          cudaStream_t s, MixParams* out);

// One-kernel attention for a single query row per image (CaiT class attention, CrossViT cross attention; any variant):
// attn_cls.cu.  false if the shape is not covered.
bool attention_cls(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                   __nv_bfloat16* out, int ldo, int B, int nk, int heads, int dh, int variant, const float* mix_a,
                   const float* mix_b, const float* ln_gamma, const float* ln_beta, cudaStream_t s, float scale = 0.f);

}  // namespace vb
