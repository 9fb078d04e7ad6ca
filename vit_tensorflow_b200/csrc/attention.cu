// Generic attention through materialised fp32 scores (the reference's own dataflow, vit.py:77-82): used by the
// exact-fp32 gate path and as the fallback of the bf16 path for shapes the fused kernels do not cover.
#include "attention.cuh"
#include "kernels.cuh"
#include <cmath>

namespace vb {

namespace {
thread_local int t_last_attention_path = ATTN_PATH_NONE;
}  // namespace

void note_attention_path(AttentionPath p) { t_last_attention_path = p; }

int take_last_attention_path() {
  const int p = t_last_attention_path;
  t_last_attention_path = ATTN_PATH_NONE;
  return p;
}

template <typename T>
void attention_generic(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, float* S, int B, int nq,
                       int nk, int heads, int dh, int variant, const float* mix_a, const float* mix_b, const float* ln_gamma,
                       const float* ln_beta, cudaStream_t s, float scale, const PosBias* pb) {
  note_attention_path(ATTN_PATH_SIMT);
  VB_CHECK(pb == nullptr || variant == 0, "attention: the position bias is for plain softmax attention only");
  attn_scores<T>(q, ldq, k, ldk, S, B, heads, nq, nk, dh, scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh)), s);
  if (pb != nullptr) attn_pos_bias(S, *pb, B, heads, nq, nk, s);                              // levit.py:131
  if (variant == 2) attn_head_mix(S, mix_a, nullptr, nullptr, B, heads, nq, nk, s);            // cait.py:123
  attn_softmax(S, static_cast<long long>(B) * heads * nq, nk, s);
  if (variant == 1) attn_head_mix(S, mix_a, ln_gamma, ln_beta, B, heads, nq, nk, s);           // deepvit.py:83-84
  if (variant == 2) attn_head_mix(S, mix_b, nullptr, nullptr, B, heads, nq, nk, s);            // cait.py:125
  attn_pv<T>(S, v, ldv, out, ldo, B, heads, nq, nk, dh, s, pb != nullptr && pb->gelu_out);
}

template <>
void attention_generic<__nv_bfloat16>(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                                      __nv_bfloat16* out, int ldo, float* S, int B, int nq, int nk, int heads, int dh, int variant,
                                      const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta,
                                      cudaStream_t s, float scale, const PosBias* pb) {
  if (attention_generic_mma(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, heads, dh, variant, mix_a, mix_b, ln_gamma, ln_beta, s,
                            scale, pb))
    return;
  note_attention_path(ATTN_PATH_SIMT);
  VB_CHECK(pb == nullptr || variant == 0, "attention: the position bias is for plain softmax attention only");
  attn_scores<__nv_bfloat16>(q, ldq, k, ldk, S, B, heads, nq, nk, dh, scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh)), s);
  if (pb != nullptr) attn_pos_bias(S, *pb, B, heads, nq, nk, s);
  if (variant == 2) attn_head_mix(S, mix_a, nullptr, nullptr, B, heads, nq, nk, s);
  attn_softmax(S, static_cast<long long>(B) * heads * nq, nk, s);
  if (variant == 1) attn_head_mix(S, mix_a, ln_gamma, ln_beta, B, heads, nq, nk, s);
  if (variant == 2) attn_head_mix(S, mix_b, nullptr, nullptr, B, heads, nq, nk, s);
  attn_pv<__nv_bfloat16>(S, v, ldv, out, ldo, B, heads, nq, nk, dh, s, pb != nullptr && pb->gelu_out);
}

template void attention_generic<float>(const float*, int, const float*, int, const float*, int, float*, int, float*, int, int, int,
                                       int, int, int, const float*, const float*, const float*, const float*, cudaStream_t, float,
                                       const PosBias*);

template <typename T>
void attention_generic_masked(const T* q, int ldq, const T* k, int ldk, const T* v, int ldv, T* out, int ldo, float* S, int B, int nq,
                              int nk, int heads, int dh, cudaStream_t s, float scale, const int* nk_img, int mask) {
  note_attention_path(ATTN_PATH_SIMT);
  attn_scores<T>(q, ldq, k, ldk, S, B, heads, nq, nk, dh, scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh)), s);
  const bool diag = mask == ATTN_MASK_DIAG;
  attn_softmax_masked(S, static_cast<long long>(B) * heads * nq, nk, static_cast<long long>(heads) * nq, diag ? nullptr : nk_img, s,
                      diag ? nq : 0);
  attn_pv<T>(S, v, ldv, out, ldo, B, heads, nq, nk, dh, s);
}
template void attention_generic_masked<float>(const float*, int, const float*, int, const float*, int, float*, int, float*, int, int, int,
                                              int, int, cudaStream_t, float, const int*, int);
template void attention_generic_masked<__nv_bfloat16>(const __nv_bfloat16*, int, const __nv_bfloat16*, int, const __nv_bfloat16*, int,
                                                      __nv_bfloat16*, int, float*, int, int, int, int, int, cudaStream_t, float, const int*,
                                                      int);


template <>
bool attention_fast<float>(const float*, int, const float*, int, const float*, int, float*, int, int, int, int, int, int, int,
                           const float*, const float*, const float*, const float*, cudaStream_t, float, const PosBias*,
                           const Window*) {
  return false;  // the fp32 gate path always takes the exact SIMT kernels
}

}  // namespace vb
