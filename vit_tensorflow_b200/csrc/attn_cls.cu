// Single-query attention (nq == 1) in one kernel: the CaiT class-attention stage (cait.py:109-131 with x = the cls token,
// context = [LN(cls) ; patches], talking heads) and CrossViT's cross-attention (cross_vit.py:69-93,152-163: the cls token of
// one branch attends over the other branch's patches).
//
// With one query row per image there is nothing for a tensor core to do (M = 1): the op is a read of K and V
// (B * nk * 2 * heads * dh bf16 values, 38.7 MB at the CaiT-S36 cls stage, B = 128) plus O(heads^2 nk) arithmetic per image.
// One CTA per image, everything between the loads in shared memory:
//   1. scores   S[h][j] = scale * q_h . k_{j,h}        thread = (key j, head h), 16-byte loads along the head's slice of the K row
//   2. variant 2: S <- mix_pre^T S (cait.py:123)        thread = key j
//   3. softmax over j per head                          warp = head (shuffle reductions, exp2 on pre-scaled scores)
//   4. variant 2: P <- mix_post^T P (cait.py:125); variant 1: P <- LN_heads(W^T P) (deepvit.py:83-84)     thread = key j
//   5. out[h*dh + d] = sum_j P[h][j] v[j][h*dh + d]     thread = two adjacent output columns, coalesced V reads
// The [b, h, 1, nk] score tensor never leaves the SM.  Algorithmic bytes: 2 * B * nk * heads * dh * 2 (K, V) + the q / out rows.
#include "attention.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace vb {
namespace {

constexpr int CLS_THREADS = 256;

__global__ void __launch_bounds__(CLS_THREADS)
attn_cls_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k, int ldk,
                const __nv_bfloat16* __restrict__ v, int ldv, __nv_bfloat16* __restrict__ out, int ldo, int nk, int heads, int dh,
                int variant, const float* __restrict__ mix_a, const float* __restrict__ mix_b, const float* __restrict__ ln_g,
                const float* __restrict__ ln_b, float scale_log2) {
  extern __shared__ float sm[];
  const int inner = heads * dh;
  float* sq = sm;                                  // [inner] query row, fp32
  float* sA = sq + inner;                          // [heads][nk] scores / probabilities
  float* sB = sA + heads * nk;                     // [heads][nk] second buffer for the head mixes (variants 1, 2)
  float* sWa = sB + (variant != 0 ? heads * nk : 0);   // [heads][heads]
  float* sWb = sWa + heads * heads;
  float* sG = sWb + heads * heads;                 // [heads] gamma, beta
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_wait();
  pdl_launch_dependents();
  for (int e = tid; e < inner; e += CLS_THREADS) sq[e] = __bfloat162float(q[static_cast<size_t>(b) * ldq + e]);
  if (variant != 0) {
    for (int e = tid; e < heads * heads; e += CLS_THREADS) {
      sWa[e] = mix_a[e];
      if (variant == 2) sWb[e] = mix_b[e];
    }
    if (variant == 1) for (int e = tid; e < heads; e += CLS_THREADS) { sG[e] = ln_g[e]; sG[heads + e] = ln_b[e]; }
  }
  __syncthreads();
  // ---- 1. scores (in log2 units: scale * log2(e) folded in; the pre-softmax mix is linear, so it commutes with the factor)
  // thread = (key j, head h), adjacent threads = adjacent heads of one key: a warp's eight 16-byte loads per thread sweep four
  // whole K rows (4 KB, L1-resident), all issued before the arithmetic, instead of 64 dependent loads along one 1 KB row per
  // thread.
  const int chunks = dh >> 3;
  for (int idx = tid; idx < nk * heads; idx += CLS_THREADS) {
    const int j = idx / heads, h = idx - j * heads;
    const uint4* kr = reinterpret_cast<const uint4*>(k + (static_cast<size_t>(b) * nk + j) * ldk) + h * chunks;
    const float* qh = sq + h * dh;
    float acc = 0.f;
    for (int c0 = 0; c0 < chunks; c0 += 8) {
      uint4 w[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) w[c] = (c0 + c < chunks) ? __ldg(kr + c0 + c) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c0 + c < chunks) {
          const float* qq = qh + (c0 + c) * 8;
          acc = fmaf(bf16_lo(w[c].x), qq[0], acc); acc = fmaf(bf16_hi(w[c].x), qq[1], acc);
          acc = fmaf(bf16_lo(w[c].y), qq[2], acc); acc = fmaf(bf16_hi(w[c].y), qq[3], acc);
          acc = fmaf(bf16_lo(w[c].z), qq[4], acc); acc = fmaf(bf16_hi(w[c].z), qq[5], acc);
          acc = fmaf(bf16_lo(w[c].w), qq[6], acc); acc = fmaf(bf16_hi(w[c].w), qq[7], acc);
        }
      }
    }
    sA[h * nk + j] = acc * scale_log2;
  }
  __syncthreads();
  float* cur = sA;
  // ---- 2. CaiT: dots = einsum('b h i j, h g -> b g i j', dots, mix_heads_pre_attn)
  if (variant == 2) {
    for (int j = tid; j < nk; j += CLS_THREADS)
      for (int g = 0; g < heads; ++g) {
        float acc = 0.f;
        for (int h = 0; h < heads; ++h) acc = fmaf(sWa[h * heads + g], sA[h * nk + j], acc);
        sB[g * nk + j] = acc;
      }
    __syncthreads();
    cur = sB;
  }
  // ---- 3. softmax over the keys, one warp per head
  for (int h = warp; h < heads; h += CLS_THREADS / 32) {
    float* row = cur + h * nk;
    float m = -INFINITY;
    for (int j = lane; j < nk; j += 32) m = fmaxf(m, row[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float l = 0.f;
    for (int j = lane; j < nk; j += 32) { const float p = ex2_approx(row[j] - m); row[j] = p; l += p; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    const float il = 1.0f / l;
    for (int j = lane; j < nk; j += 32) row[j] *= il;
  }
  __syncthreads();
  // ---- 4. post-softmax head mix (CaiT mix_post) / DeepViT re-attention + LayerNorm over the head axis (eps 1e-3)
  if (variant != 0) {
    float* dst = (cur == sA) ? sB : sA;
    const float* W = (variant == 2) ? sWb : sWa;
    for (int j = tid; j < nk; j += CLS_THREADS) {
      float s1 = 0.f, s2 = 0.f;
      for (int g = 0; g < heads; ++g) {
        float acc = 0.f;
        for (int h = 0; h < heads; ++h) acc = fmaf(W[h * heads + g], cur[h * nk + j], acc);
        dst[g * nk + j] = acc;
        s1 += acc;
      }
      if (variant == 1) {
        const float mu = s1 / static_cast<float>(heads);
        for (int g = 0; g < heads; ++g) { const float d = dst[g * nk + j] - mu; s2 = fmaf(d, d, s2); }
        const float rstd = rsqrtf(s2 / static_cast<float>(heads) + 1e-3f);
        for (int g = 0; g < heads; ++g) dst[g * nk + j] = (dst[g * nk + j] - mu) * rstd * sG[g] + sG[heads + g];
      }
    }
    __syncthreads();
    cur = dst;
  }
  // ---- 5. out = P . V  (fp32 probabilities; two adjacent columns per thread)
  for (int e2 = tid; e2 < (inner >> 1); e2 += CLS_THREADS) {
    const int e = e2 * 2, h = e / dh;
    const float* p = cur + h * nk;
    const __nv_bfloat16* vc = v + static_cast<size_t>(b) * nk * ldv + e;
    // eight independent row loads in flight per thread (the two-deep form was latency-bound: nk / 2 dependent L2 round trips)
    float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
    int j = 0;
    for (; j + 7 < nk; j += 8) {
      uint32_t w[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) w[u] = __ldg(reinterpret_cast<const uint32_t*>(vc + static_cast<size_t>(j + u) * ldv));
#pragma unroll
      for (int u = 0; u < 8; u += 2) {
        a0 = fmaf(p[j + u], bf16_lo(w[u]), a0); a1 = fmaf(p[j + u], bf16_hi(w[u]), a1);
        c0 = fmaf(p[j + u + 1], bf16_lo(w[u + 1]), c0); c1 = fmaf(p[j + u + 1], bf16_hi(w[u + 1]), c1);
      }
    }
    for (; j < nk; ++j) {                                          // even keys -> (a0, a1), odd keys -> (c0, c1), as in the main loop
      const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(vc + static_cast<size_t>(j) * ldv));
      if (j & 1) { c0 = fmaf(p[j], bf16_lo(w0), c0); c1 = fmaf(p[j], bf16_hi(w0), c1); }
      else { a0 = fmaf(p[j], bf16_lo(w0), a0); a1 = fmaf(p[j], bf16_hi(w0), a1); }
    }
    *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(b) * ldo + e) = pack_bf16x2(a0 + c0, a1 + c1);
  }
}

}  // namespace

// false when the shape is not covered (the caller falls back to the general path)
bool attention_cls(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                   __nv_bfloat16* out, int ldo, int B, int nk, int heads, int dh, int variant, const float* mix_a,
                   const float* mix_b, const float* ln_g, const float* ln_b, cudaStream_t s, float scale) {
  if (dh % 8 != 0 || heads < 1 || nk < 1) return false;
  if ((ldk % 8) || (ldv % 2) || (ldo % 2)) return false;
  if ((reinterpret_cast<uintptr_t>(k) % 16) || (reinterpret_cast<uintptr_t>(v) % 4) || (reinterpret_cast<uintptr_t>(out) % 4)) return false;
  if (variant == 1 && (mix_a == nullptr || ln_g == nullptr || ln_b == nullptr)) return false;
  if (variant == 2 && (mix_a == nullptr || mix_b == nullptr)) return false;
  const size_t smem = (static_cast<size_t>(heads) * dh + static_cast<size_t>(variant != 0 ? 2 : 1) * heads * nk + 2 * heads * heads +
                       2 * heads) * sizeof(float);
  if (smem > 200 * 1024) return false;
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(attn_cls_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(B);
  cfg.blockDim = dim3(CLS_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VB_CUDA(cudaLaunchKernelEx(&cfg, attn_cls_kernel, q, ldq, k, ldk, v, ldv, out, ldo, nk, heads, dh, variant, mix_a, mix_b, ln_g, ln_b,
                             scale_log2));
  count_launch();
  note_attention_path(ATTN_PATH_CLS);
  return true;
}

}  // namespace vb
