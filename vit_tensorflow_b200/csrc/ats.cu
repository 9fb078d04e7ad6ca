// Adaptive token sampling (ats_vit.py:77-132, 191-258) on the device, in the compact row layout of the engine's ATS forward:
// image b keeps its rows at pitch P as [cls, c_b kept tokens in ascending id order, dead rows].  The batch maximum C of the
// counts decides on the device whether a layer samples (C > K, ats_vit.py:213), so the whole forward is one fixed launch
// sequence that a CUDA graph can replay.  See kernels.cuh for the contracts.
#include "kernels.cuh"
#include "philox.cuh"

#include <cmath>

namespace vb {
namespace {

template <typename T> __device__ __forceinline__ float ats_f(T v);
template <> __device__ __forceinline__ float ats_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float ats_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

__device__ __forceinline__ float ats_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int ATS_THREADS = 256;
constexpr int ATS_WARPS = ATS_THREADS / 32;

// block-wide reduction through `red` (ATS_WARPS floats); every thread gets the result
template <bool MAX>
__device__ float ats_block_reduce(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, w) : v + w;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                       // `red` may still be read from the previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < ATS_WARPS; ++w) r = MAX ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

__global__ void ats_init_kernel(int* rows, int* C, int* ids, int B, int P) {
  const long long total = static_cast<long long>(B) * P;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(e % P);
    ids[e] = t;
    if (t == 0) rows[e / P] = P;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *C = P - 1;
}

template <typename T>
__global__ void __launch_bounds__(ATS_THREADS)
ats_sample_kernel(const T* __restrict__ qkv, int ld, int P, int heads, int dh, float scale, const int* __restrict__ rows,
                  const int* __restrict__ Cp, int K, const unsigned long long* __restrict__ rng, float* __restrict__ scratch,
                  int* __restrict__ sel, int Pn, int* __restrict__ rows_new, int* __restrict__ draws) {
  __shared__ float qs[ATS_MAX_DH];
  __shared__ float red[ATS_WARPS];
  __shared__ uint32_t bits[ATS_MAX_TOKENS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int c = rows[b] - 1, C = *Cp;
  if (C <= K) {                                              // ats_vit.py:213: the layer keeps every row
    for (int t = tid; t <= c; t += ATS_THREADS) sel[static_cast<size_t>(b) * Pn + t] = t;
    if (tid == 0) rows_new[b] = c + 1;
    return;
  }
  const int HD = heads * dh;
  const T* base = qkv + static_cast<size_t>(b) * P * ld;
  float* acc = scratch + static_cast<size_t>(b) * 3 * P;     // per token: the head sum, then the pseudo-logit
  float* sc = acc + P;                                       // per key of the current head: the score, the value norm
  float* vn = sc + P;
  for (int i = tid; i <= c; i += ATS_THREADS) acc[i] = 0.f;
  for (int w = tid; w < ATS_MAX_TOKENS / 32; w += ATS_THREADS) bits[w] = 0u;
  for (int h = 0; h < heads; ++h) {
    __syncthreads();
    for (int d = tid; d < dh; d += ATS_THREADS) qs[d] = ats_f(base[h * dh + d]);
    __syncthreads();
    // the cls query's scores over the valid keys 0..c (cls included, ats_vit.py:81) and the value norms (:84), a warp per key
    for (int i = warp; i <= c; i += ATS_WARPS) {
      const T* row = base + static_cast<size_t>(i) * ld + h * dh;
      float dot = 0.f, v2 = 0.f;
      for (int d = lane; d < dh; d += 32) {
        dot = fmaf(qs[d], ats_f(row[HD + d]), dot);
        const float v = ats_f(row[2 * HD + d]);
        v2 = fmaf(v, v, v2);
      }
      dot = ats_warp_sum(dot);
      v2 = ats_warp_sum(v2);
      if (lane == 0) { sc[i] = dot * scale; vn[i] = sqrtf(v2); }
    }
    __syncthreads();
    float m = -INFINITY;
    for (int i = tid; i <= c; i += ATS_THREADS) m = fmaxf(m, sc[i]);
    m = ats_block_reduce<true>(m, red);
    float sum = 0.f;
    for (int i = tid; i <= c; i += ATS_THREADS) sum += expf(sc[i] - m);
    const float inv = 1.0f / ats_block_reduce<false>(sum, red);
    for (int i = 1 + tid; i <= c; i += ATS_THREADS) acc[i] += expf(sc[i] - m) * inv * vn[i];   // einsum over heads (:87)
  }
  __syncthreads();
  float tot = 0.f;
  for (int i = 1 + tid; i <= c; i += ATS_THREADS) tot += acc[i];
  tot = ats_block_reduce<false>(tot, red);
  for (int i = 1 + tid; i <= c; i += ATS_THREADS) acc[i] = logf(acc[i] / (tot + 1e-6f) + 1e-6f);   // :90-93
  __syncthreads();
  // K Gumbel-max draws (:101-105), a warp per draw.  The noise of compact token i is the reference's column j = (C - c) + i - 1
  // of its left-padded [b, K, n - 1] tensor; masked columns never win, so only the c valid ones are visited.
  const uint32_t k0 = static_cast<uint32_t>(rng[0]), k1 = static_cast<uint32_t>(rng[0] >> 32);
  const unsigned long long dctr = rng[1];
  const int off = C - c;
  for (int k = warp; k < K; k += ATS_WARPS) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = 1 + lane; i <= c; i += 32) {
      const uint32_t j = static_cast<uint32_t>(off + i - 1);
      const uint4 x = philox4x32_10(make_uint4(j | (static_cast<uint32_t>(k) << 16), static_cast<uint32_t>(b),
                                               static_cast<uint32_t>(dctr), static_cast<uint32_t>(dctr >> 32)), k0, k1);
      const float u = static_cast<float>(x.x >> 8) * 5.9604644775390625e-8f;   // 2^-24
      const float g = -logf(-logf(u + 1e-6f) + 1e-6f);
      const float v = acc[i] + g;
      if (v > best) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {                       // argmax, the first index on ties (tf.argmax)
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (bi > c) bi = c;                                      // no candidate compared greater (NaN scores): stay inside the set
    if (lane == 0) {
      draws[static_cast<size_t>(b) * K + k] = off + bi;      // argmax + 1: the position in the padded layout
      atomicOr(&bits[bi >> 5], 1u << (bi & 31));
    }
  }
  __syncthreads();
  if (tid == 0) {                                            // tf.unique + tf.sort (:110-113): the set bits in order
    int t = 0;
    sel[static_cast<size_t>(b) * Pn] = 0;
    for (int w = 0; w <= (c >> 5); ++w)
      for (uint32_t word = bits[w]; word != 0u; word &= word - 1u) sel[static_cast<size_t>(b) * Pn + (++t)] = w * 32 + __ffs(word) - 1;
    rows_new[b] = t + 1;
  }
}

// Xn row t of image b = X row sel[b, t] for t < rows_new[b], zero after; ids likewise (0 on dead rows).  Block 0 also
// publishes the new batch maximum and advances the noise counter when the layer sampled.
template <typename T>
__global__ void __launch_bounds__(128)
ats_gather_kernel(const T* __restrict__ X, int P, T* __restrict__ Xn, int Pn, int dim, const int* __restrict__ sel,
                  const int* __restrict__ rows_new, const int* __restrict__ ids, int* __restrict__ ids_n, int B,
                  const int* __restrict__ C_old, int K, int* __restrict__ C_new, unsigned long long* __restrict__ rng) {
  const long long r = blockIdx.x;
  const int b = static_cast<int>(r / Pn), t = static_cast<int>(r % Pn);
  const bool live = t < rows_new[b];
  const int src = live ? sel[static_cast<size_t>(b) * Pn + t] : 0;
  const T* xs = X + (static_cast<size_t>(b) * P + src) * dim;
  T* xd = Xn + static_cast<size_t>(r) * dim;
  if ((dim * sizeof(T)) % 16 == 0) {
    const int nv = static_cast<int>(dim * sizeof(T) / 16);
    const uint4* vs = reinterpret_cast<const uint4*>(xs);
    uint4* vd = reinterpret_cast<uint4*>(xd);
    for (int e = threadIdx.x; e < nv; e += blockDim.x) vd[e] = live ? vs[e] : make_uint4(0u, 0u, 0u, 0u);
  } else {
    for (int e = threadIdx.x; e < dim; e += blockDim.x) xd[e] = live ? xs[e] : T(0.f);
  }
  if (threadIdx.x == 0) ids_n[r] = live ? ids[static_cast<size_t>(b) * P + src] : 0;
  if (r == 0 && threadIdx.x == 0) {
    int m = 0;
    for (int i = 0; i < B; ++i) m = max(m, rows_new[i]);
    *C_new = m - 1;
    if (*C_old > K) rng[1] += 1ull;                          // one noise draw per sampling event (tf.random.uniform call)
  }
}

// out[b, j] = (the reference's token_ids[:, 1:] - 1) column j (ats_vit.py:315): left-padded with -1 to C; -1 beyond C
__global__ void ats_ids_out_kernel(const int* __restrict__ ids, int P, const int* __restrict__ rows, const int* __restrict__ Cp,
                                   int* __restrict__ out, int B) {
  const int W = P - 1, C = *Cp;
  const long long total = static_cast<long long>(B) * W;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(e / W), j = static_cast<int>(e % W), off = C + 1 - rows[b];
    out[e] = (j < off || j >= C) ? -1 : ids[static_cast<size_t>(b) * P + 1 + j - off] - 1;
  }
}

// Row softmax of materialised scores with the keys j >= nk_img[row / rows_per_img] (nk_img non-null) and the key j == row % diag_nq
// (diag_nq > 0) masked: weight exactly 0
__global__ void attn_softmax_masked_kernel(float* __restrict__ S, long long rows, int nk, long long rows_per_img,
                                           const int* __restrict__ nk_img, int diag_nq) {
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31, valid = nk_img != nullptr ? min(nk, nk_img[row / rows_per_img]) : nk;
  const int dj = diag_nq > 0 ? static_cast<int>(row % diag_nq) : -1;
  float* r = S + row * nk;
  float mx = -INFINITY;
  for (int j = lane; j < valid; j += 32) if (j != dj) mx = fmaxf(mx, r[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < valid; j += 32) { const float e = j != dj ? expf(r[j] - mx) : 0.f; r[j] = e; sum += e; }
  const float inv = 1.0f / ats_warp_sum(sum);
  for (int j = lane; j < nk; j += 32) r[j] = j < valid ? r[j] * inv : 0.f;
}

int ats_grid(long long total) {
  const long long g = (total + 255) / 256, cap = static_cast<long long>(sm_count()) * 8;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

void ats_init(int* rows, int* C, int* ids, int B, int P, cudaStream_t s) {
  ats_init_kernel<<<ats_grid(static_cast<long long>(B) * P), 256, 0, s>>>(rows, C, ids, B, P);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void ats_sample(const T* qkv, int ld, int B, int P, int heads, int dh, float scale, const int* rows, const int* C, int K,
                const unsigned long long* rng, float* scratch, int* sel, int Pn, int* rows_new, int* draws, cudaStream_t s) {
  VB_CHECK(dh <= ATS_MAX_DH && P <= ATS_MAX_TOKENS, "adaptive token sampling: dim_head <= 256 and at most 65,535 patches");
  ats_sample_kernel<T><<<B, ATS_THREADS, 0, s>>>(qkv, ld, P, heads, dh, scale, rows, C, K, rng, scratch, sel, Pn, rows_new, draws);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void ats_gather(const T* X, int P, T* Xn, int Pn, int dim, const int* sel, const int* rows_new, const int* ids, int* ids_n, int B,
                const int* C_old, int K, int* C_new, unsigned long long* rng, cudaStream_t s) {
  const long long blocks = static_cast<long long>(B) * Pn;
  VB_CHECK(blocks <= 0x7fffffffLL, "adaptive token sampling: too many rows");
  ats_gather_kernel<T><<<static_cast<unsigned>(blocks), 128, 0, s>>>(X, P, Xn, Pn, dim, sel, rows_new, ids, ids_n, B, C_old, K, C_new, rng);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

void ats_ids_out(const int* ids, int P, const int* rows, const int* C, int* out, int B, cudaStream_t s) {
  ats_ids_out_kernel<<<ats_grid(static_cast<long long>(B) * (P - 1)), 256, 0, s>>>(ids, P, rows, C, out, B);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

void attn_softmax_masked(float* S, long long rows, int nk, long long rows_per_img, const int* nk_img, cudaStream_t s, int diag_nq) {
  const int warps = 8;
  attn_softmax_masked_kernel<<<static_cast<unsigned>((rows + warps - 1) / warps), warps * 32, 0, s>>>(S, rows, nk, rows_per_img, nk_img,
                                                                                                       diag_nq);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template void ats_sample<float>(const float*, int, int, int, int, int, float, const int*, const int*, int, const unsigned long long*,
                                float*, int*, int, int*, int*, cudaStream_t);
template void ats_sample<__nv_bfloat16>(const __nv_bfloat16*, int, int, int, int, int, float, const int*, const int*, int,
                                        const unsigned long long*, float*, int*, int, int*, int*, cudaStream_t);
template void ats_gather<float>(const float*, int, float*, int, int, const int*, const int*, const int*, int*, int, const int*, int, int*,
                                unsigned long long*, cudaStream_t);
template void ats_gather<__nv_bfloat16>(const __nv_bfloat16*, int, __nv_bfloat16*, int, int, const int*, const int*, const int*, int*, int,
                                        const int*, int, int*, unsigned long long*, cudaStream_t);

}  // namespace vb
