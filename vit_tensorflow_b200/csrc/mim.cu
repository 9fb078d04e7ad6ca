// Masked image modelling on the device (MAE, mae.py:49-92; SimMIM, simmim.py:82-129): the patch masks drawn from the engine's
// Philox noise, the kept-patch gather straight out of the NHWC image, the rows the encoder / decoder hand each other, and the two
// reconstruction losses as fixed-order reductions.  See kernels.cuh for the contracts.
#include "kernels.cuh"
#include "philox.cuh"

namespace vb {
namespace {

template <typename T> __device__ __forceinline__ float mim_f(T v);
template <> __device__ __forceinline__ float mim_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float mim_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

constexpr int MIM_MASK_THREADS = 1024;
constexpr int MIM_LOSS_THREADS = 256;
constexpr int MIM_LOSS_BLOCKS = 1024;
constexpr int MPP_DRAW_THREADS = 256;

// One CTA per image: u[b, j] = (Philox4x32-10 word 0 >> 8) for j < n with counter (j, b, d_lo, d_hi), sorted as the 64-bit keys
// (u << 32 | j) ascending (MAE's stable argsort) or ((2^24 - 1 - u) << 32 | j) ascending (SimMIM's top_k: u descending, ties to
// the smaller j) by a bitonic network in shared memory.  The CTA that finishes last advances d, after every CTA has read it.
__global__ void __launch_bounds__(MIM_MASK_THREADS)
mim_mask_kernel(int n, int descending, unsigned long long* rng, unsigned int* done, int* __restrict__ idx) {
  __shared__ unsigned long long key[MIM_MAX_PATCHES];
  __shared__ unsigned long long kd[2];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) { kd[0] = rng[0]; kd[1] = rng[1]; }
  __syncthreads();
  const uint32_t k0 = static_cast<uint32_t>(kd[0]), k1 = static_cast<uint32_t>(kd[0] >> 32);
  const unsigned long long d = kd[1];
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  for (int j = tid; j < np2; j += MIM_MASK_THREADS) {
    if (j < n) {
      const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>(j), static_cast<uint32_t>(b), static_cast<uint32_t>(d),
                                               static_cast<uint32_t>(d >> 32)), k0, k1);
      const uint32_t u = x.x >> 8;
      key[j] = (static_cast<unsigned long long>(descending ? 0xFFFFFFu - u : u) << 32) | static_cast<uint32_t>(j);
    } else {
      key[j] = ~0ull;                                        // padding sorts last
    }
  }
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    for (int s = k >> 1; s > 0; s >>= 1) {
      for (int i = tid; i < np2; i += MIM_MASK_THREADS) {
        const int p = i ^ s;
        if (p > i) {
          const unsigned long long a = key[i], c = key[p];
          if ((a > c) == ((i & k) == 0)) { key[i] = c; key[p] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int j = tid; j < n; j += MIM_MASK_THREADS) idx[static_cast<size_t>(b) * n + j] = static_cast<int>(key[j] & 0xFFFFFFFFull);
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(done, 1u) == gridDim.x - 1) {              // every CTA has read d: one draw per forward
      rng[1] = d + 1ull;
      *done = 0u;
      __threadfence();
    }
  }
}

// Row r = b * count + i of `out` [B * count, ldo]: the (p1, p2, c) vector of patch j = idx[b * n + off + i] (j = i without idx),
// zero in the columns [pd, ldo); with R, R row r = pos[1 + j] (the patch GEMM's residual operand).  MPP's corrupted rows (cls
// non-null): each image's row 0 is the cls row (A zero, R = pos[0] + cls - bias, which the GEMM's bias completes to cls + pos[0],
// as the ViT embedding's residual does); row 1 + j reads its pixels from patch src[b * n + j] rather than j, or mask_row where
// that is -1, and keeps R = pos[1 + j].  MPP is a template flag, so MAE's and SimMIM's instances carry none of its branches.
template <typename T, bool MPP>
__global__ void __launch_bounds__(128)
mim_patch_rows_kernel(const float* __restrict__ img, int H, int W, int C, int ph, int pw, const int* __restrict__ idx, int n, int off,
                      int count, T* __restrict__ out, int ldo, const float* __restrict__ pos, T* __restrict__ R, int dim, long long rows,
                      const int* __restrict__ src, const float* __restrict__ mask_row, const float* __restrict__ cls,
                      const float* __restrict__ bias) {
  const int pd = ph * pw * C, gw = W / pw;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int b = static_cast<int>(r / count), i = static_cast<int>(r % count);
    T* o = out + r * ldo;
    if (MPP && i == 0) {
      for (int e = threadIdx.x; e < ldo; e += blockDim.x) o[e] = T(0.f);
      T* rr = R + r * dim;
      for (int e = threadIdx.x; e < dim; e += blockDim.x) rr[e] = T(pos[e] + cls[e] - bias[e]);
      continue;
    }
    const int t = MPP ? i - 1 : i;
    const int j = idx != nullptr ? idx[static_cast<size_t>(b) * n + off + t] : t;
    const int sj = MPP ? src[static_cast<size_t>(b) * n + j] : j;
    const int gy = sj / gw, gx = sj % gw;
    const float* base = img + ((static_cast<size_t>(b) * H + static_cast<size_t>(gy) * ph) * W + static_cast<size_t>(gx) * pw) * C;
    for (int e = threadIdx.x; e < ldo; e += blockDim.x) {
      float v = 0.f;
      if (e < pd) {
        const int p1 = e / (pw * C), rem = e - p1 * pw * C;
        v = MPP && sj < 0 ? mask_row[e] : base[static_cast<size_t>(p1) * W * C + rem];   // rem = p2 * C + c: contiguous along the image row
      }
      o[e] = T(v);
    }
    if (R != nullptr) {
      const float* pr = pos + static_cast<size_t>(1 + j) * dim;
      T* rr = R + r * dim;
      for (int e = threadIdx.x; e < dim; e += blockDim.x) rr[e] = T(pr[e]);
    }
  }
}

// MPP's corruption draws (mpp.py:178-197), one CTA per image, after mim_mask_kernel drew this call's mask at counter d = rng[1] - 1
// (it has advanced rng[1] since).  The first k ids of idx (the top_k) become a bitmap.  Per masked position j, words 1-3 of
// Philox4x32-10 at counter (j, b, d_lo, d_hi) give the random-patch coin u1 < p_rand (when use_rand), the random id
// (word 2 * n) >> 32 and the replace coin u3 < p_repl, with u = (word >> 8) 2^-24 compared in float32.  source[b, j] is j, the
// random id where the random-patch coin is true, or -1 (the mask token) where the replace coin is true.  mask_ids[b * ldm + i],
// i < k: the masked ids ascending (the order of predicted_patches[mask]).
__global__ void __launch_bounds__(MPP_DRAW_THREADS)
mpp_draws_kernel(int n, int k, const int* __restrict__ idx, const unsigned long long* __restrict__ rng, int use_rand, float p_rand,
                 float p_repl, int* __restrict__ source, int* __restrict__ mask_ids, int ldm) {
  constexpr int WORDS = MIM_MAX_PATCHES / 32;
  __shared__ uint32_t bits[WORDS];
  __shared__ int before[WORDS];
  const int b = blockIdx.x, tid = threadIdx.x, nw = (n + 31) / 32;
  for (int w = tid; w < WORDS; w += MPP_DRAW_THREADS) bits[w] = 0u;
  __syncthreads();
  for (int i = tid; i < k; i += MPP_DRAW_THREADS) {
    const int j = idx[static_cast<size_t>(b) * n + i];
    atomicOr(&bits[j >> 5], 1u << (j & 31));
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int w = 0; w < nw; ++w) { before[w] = run; run += __popc(bits[w]); }
  }
  __syncthreads();
  const uint32_t k0 = static_cast<uint32_t>(rng[0]), k1 = static_cast<uint32_t>(rng[0] >> 32);
  const unsigned long long d = rng[1] - 1ull;
  for (int j = tid; j < n; j += MPP_DRAW_THREADS) {
    const uint32_t word = bits[j >> 5], bit = 1u << (j & 31);
    int s = j;
    if (word & bit) {
      const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>(j), static_cast<uint32_t>(b), static_cast<uint32_t>(d),
                                               static_cast<uint32_t>(d >> 32)), k0, k1);
      const float u1 = static_cast<float>(x.y >> 8) * 0x1p-24f, u3 = static_cast<float>(x.w >> 8) * 0x1p-24f;
      if (use_rand && u1 < p_rand) s = static_cast<int>((static_cast<unsigned long long>(x.z) * static_cast<unsigned>(n)) >> 32);
      if (u3 < p_repl) s = -1;
      mask_ids[static_cast<size_t>(b) * ldm + before[j >> 5] + __popc(word & (bit - 1u))] = j;
    }
    source[static_cast<size_t>(b) * n + j] = s;
  }
}

// MAE's decoder input, image b's rows at pitch n: row t < nm = mask_token + dpe[idx[b, t]], row t >= nm = E[b * (n - nm) + t - nm]
// + dpe[idx[b, t]] (mae.py:72-80: the mask tokens first, then the kept rows in argsort order)
template <typename T>
__global__ void __launch_bounds__(128)
mim_decoder_rows_kernel(const T* __restrict__ E, const int* __restrict__ idx, int n, int nm, const float* __restrict__ mask_token,
                        const float* __restrict__ dpe, T* __restrict__ Z, int D, long long rows) {
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int b = static_cast<int>(r / n), t = static_cast<int>(r % n);
    const int j = idx[r];
    const float* pe = dpe + static_cast<size_t>(j) * D;
    T* z = Z + r * D;
    if (t < nm) {
      for (int e = threadIdx.x; e < D; e += blockDim.x) z[e] = T(mask_token[e] + pe[e]);
    } else {
      const T* x = E + (static_cast<size_t>(b) * (n - nm) + (t - nm)) * D;
      for (int e = threadIdx.x; e < D; e += blockDim.x) z[e] = T(mim_f(x[e]) + pe[e]);
    }
  }
}

// SimMIM: image b's row j = idx[b, i], i < nm, becomes mask_token + pos[1 + j] (simmim.py:98-110)
template <typename T>
__global__ void __launch_bounds__(128)
mim_mask_tokens_kernel(T* __restrict__ X, const int* __restrict__ idx, int n, int nm, const float* __restrict__ mask_token,
                       const float* __restrict__ pos, int D, long long rows) {
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int b = static_cast<int>(r / nm), i = static_cast<int>(r % nm);
    const int j = idx[static_cast<size_t>(b) * n + i];
    const float* pe = pos + static_cast<size_t>(1 + j) * D;
    T* x = X + (static_cast<size_t>(b) * n + j) * D;
    for (int e = threadIdx.x; e < D; e += blockDim.x) x[e] = T(mask_token[e] + pe[e]);
  }
}

// out row b * count + i = X row b * n + (idx ? idx[b * n + i] : i)
template <typename T>
__global__ void __launch_bounds__(128)
mim_take_rows_kernel(const T* __restrict__ X, int n, const int* __restrict__ idx, T* __restrict__ out, int count, int D, long long rows) {
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int b = static_cast<int>(r / count), i = static_cast<int>(r % count);
    const int src = idx != nullptr ? idx[static_cast<size_t>(b) * n + i] : i;
    const T* x = X + (static_cast<size_t>(b) * n + src) * D;
    T* o = out + r * D;
    for (int e = threadIdx.x; e < D; e += blockDim.x) o[e] = x[e];
  }
}

__device__ double mim_block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = MIM_LOSS_THREADS / 2; s > 0; s >>= 1) {      // a fixed tree: the same bits on every call
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  return red[0];
}

// Block g's partial sum over the rows g, g + G, ... of pred [rows, pd] (rows = B * nm): pred^2 (MAE), or |pred - patch| with the
// patch of row b * nm + i read from the image at id idx[b * n + i] (SimMIM)
template <typename T>
__global__ void __launch_bounds__(MIM_LOSS_THREADS)
mim_loss_partial_kernel(const T* __restrict__ pred, int pd, long long rows, const float* __restrict__ img, int H, int W, int C, int ph,
                        int pw, const int* __restrict__ idx, int n, int nm, double* __restrict__ partial) {
  __shared__ double red[MIM_LOSS_THREADS];
  double acc = 0.0;
  const int gw = W / pw;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const T* p = pred + r * pd;
    if (img == nullptr) {
      for (int e = threadIdx.x; e < pd; e += MIM_LOSS_THREADS) { const double v = mim_f(p[e]); acc += v * v; }
    } else {
      const int b = static_cast<int>(r / nm), i = static_cast<int>(r % nm);
      const int j = idx[static_cast<size_t>(b) * n + i], gy = j / gw, gx = j % gw;
      const float* base = img + ((static_cast<size_t>(b) * H + static_cast<size_t>(gy) * ph) * W + static_cast<size_t>(gx) * pw) * C;
      for (int e = threadIdx.x; e < pd; e += MIM_LOSS_THREADS) {
        const int p1 = e / (pw * C), rem = e - p1 * pw * C;
        acc += fabs(static_cast<double>(mim_f(p[e])) - static_cast<double>(base[static_cast<size_t>(p1) * W * C + rem]));
      }
    }
  }
  const double s = mim_block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(MIM_LOSS_THREADS)
mim_loss_final_kernel(const double* __restrict__ partial, int G, double scale, float* __restrict__ loss) {
  __shared__ double red[MIM_LOSS_THREADS];
  double acc = 0.0;
  for (int g = threadIdx.x; g < G; g += MIM_LOSS_THREADS) acc += partial[g];
  const double s = mim_block_sum(acc, red);
  if (threadIdx.x == 0) *loss = static_cast<float>(s * scale);
}

// MPP: block g's partial sum of the logits over the rows g, g + G, ... of L [rows, ldl], columns [0, K)
template <typename T>
__global__ void __launch_bounds__(MIM_LOSS_THREADS)
mpp_logit_sum_kernel(const T* __restrict__ L, int ldl, int K, long long rows, double* __restrict__ partial) {
  __shared__ double red[MIM_LOSS_THREADS];
  double acc = 0.0;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const T* l = L + r * ldl;
    for (int e = threadIdx.x; e < K; e += MIM_LOSS_THREADS) acc += static_cast<double>(mim_f(l[e]));
  }
  const double s = mim_block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

unsigned mim_grid(long long rows) {
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<unsigned>(rows < 1 ? 1 : (rows > cap ? cap : rows));
}

}  // namespace

void mim_mask(int B, int n, int descending, unsigned long long* rng, int* idx, cudaStream_t s) {
  VB_CHECK(n >= 1 && n <= MIM_MAX_PATCHES, "MAE / SimMIM: an image has " + std::to_string(n) + " patches; the mask kernel takes 1 to " +
                                               std::to_string(MIM_MAX_PATCHES) + " per image");
  VB_CHECK(B >= 1 && B <= 0x7fffffff, "MAE / SimMIM: bad batch");
  mim_mask_kernel<<<B, MIM_MASK_THREADS, 0, s>>>(n, descending, rng, reinterpret_cast<unsigned int*>(rng + 2), idx);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void mim_patch_rows(const float* img, int B, int H, int W, int C, int ph, int pw, const int* idx, int n, int off, int count, T* out, int ldo,
                    const float* pos, T* R, int dim, cudaStream_t s, const int* src, const float* mask_row, const float* cls,
                    const float* bias) {
  const long long rows = static_cast<long long>(B) * count;
  if (cls != nullptr)
    mim_patch_rows_kernel<T, true><<<mim_grid(rows), 128, 0, s>>>(img, H, W, C, ph, pw, idx, n, off, count, out, ldo, pos, R, dim, rows,
                                                                  src, mask_row, cls, bias);
  else
    mim_patch_rows_kernel<T, false><<<mim_grid(rows), 128, 0, s>>>(img, H, W, C, ph, pw, idx, n, off, count, out, ldo, pos, R, dim, rows,
                                                                   src, mask_row, cls, bias);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

void mpp_draws(int B, int n, int k, const int* idx, const unsigned long long* rng, double random_patch_prob, double p_rand,
               double replace_prob, int* source, int* mask_ids, int ldm, cudaStream_t s) {
  VB_CHECK(n >= 1 && n <= MIM_MAX_PATCHES && k >= 1 && k <= n && ldm >= k, "MPP: bad draw shape");
  // the coins compare float32 noise with the probabilities as TF converts a Python float: rounded to float32
  mpp_draws_kernel<<<B, MPP_DRAW_THREADS, 0, s>>>(n, k, idx, rng, random_patch_prob > 0.0 ? 1 : 0, static_cast<float>(p_rand),
                                                  static_cast<float>(replace_prob), source, mask_ids, ldm);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void mim_decoder_rows(const T* E, const int* idx, int B, int n, int nm, const float* mask_token, const float* dpe, T* Z, int D, cudaStream_t s) {
  const long long rows = static_cast<long long>(B) * n;
  mim_decoder_rows_kernel<T><<<mim_grid(rows), 128, 0, s>>>(E, idx, n, nm, mask_token, dpe, Z, D, rows);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void mim_mask_tokens(T* X, const int* idx, int B, int n, int nm, const float* mask_token, const float* pos, int D, cudaStream_t s) {
  const long long rows = static_cast<long long>(B) * nm;
  mim_mask_tokens_kernel<T><<<mim_grid(rows), 128, 0, s>>>(X, idx, n, nm, mask_token, pos, D, rows);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void mim_take_rows(const T* X, int n, const int* idx, T* out, int B, int count, int D, cudaStream_t s) {
  const long long rows = static_cast<long long>(B) * count;
  mim_take_rows_kernel<T><<<mim_grid(rows), 128, 0, s>>>(X, n, idx, out, count, D, rows);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

int mim_loss_blocks(long long rows) { return static_cast<int>(rows < MIM_LOSS_BLOCKS ? rows : MIM_LOSS_BLOCKS); }

void mim_loss_final(const double* partial, int G, double scale, float* loss, cudaStream_t s) {
  mim_loss_final_kernel<<<1, MIM_LOSS_THREADS, 0, s>>>(partial, G, scale, loss);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template <typename T>
void mim_loss(const T* pred, int pd, int B, int nm, const float* img, int H, int W, int C, int ph, int pw, const int* idx, int n,
              double* partial, float* loss, cudaStream_t s) {
  const long long rows = static_cast<long long>(B) * nm;
  const int G = mim_loss_blocks(rows);
  mim_loss_partial_kernel<T><<<G, MIM_LOSS_THREADS, 0, s>>>(pred, pd, rows, img, H, W, C, ph, pw, idx, n, nm, partial);
  VB_CUDA(cudaGetLastError());
  count_launch();
  double scale = 1.0 / (static_cast<double>(rows) * pd);
  if (img != nullptr) scale /= nm;                           // simmim.py:128: the mean divided by num_masked once more
  mim_loss_final(partial, G, scale, loss, s);
}

template <typename T>
void mpp_loss(const T* logits, int ldl, int K, long long rows, double* partial, float* loss, cudaStream_t s) {
  const int G = mim_loss_blocks(rows);
  mpp_logit_sum_kernel<T><<<G, MIM_LOSS_THREADS, 0, s>>>(logits, ldl, K, rows, partial);
  VB_CUDA(cudaGetLastError());
  count_launch();
  // mpp.py:128-129 as TF computes it: every row's cross-entropy is ln(K) times the sum of its logits (see vitb200.h)
  mim_loss_final(partial, G, std::log(static_cast<double>(K)) / static_cast<double>(rows), loss, s);
}

#define VB_MIM_INSTANTIATE(T)                                                                                                   \
  template void mim_patch_rows<T>(const float*, int, int, int, int, int, int, const int*, int, int, int, T*, int, const float*, T*, \
                                  int, cudaStream_t, const int*, const float*, const float*, const float*);                    \
  template void mpp_loss<T>(const T*, int, int, long long, double*, float*, cudaStream_t);                                     \
  template void mim_decoder_rows<T>(const T*, const int*, int, int, int, const float*, const float*, T*, int, cudaStream_t);     \
  template void mim_mask_tokens<T>(T*, const int*, int, int, int, const float*, const float*, int, cudaStream_t);                \
  template void mim_take_rows<T>(const T*, int, const int*, T*, int, int, int, cudaStream_t);                                   \
  template void mim_loss<T>(const T*, int, int, int, const float*, int, int, int, int, int, const int*, int, double*, float*,     \
                            cudaStream_t);
VB_MIM_INSTANTIATE(float)
VB_MIM_INSTANTIATE(__nv_bfloat16)
#undef VB_MIM_INSTANTIATE

}  // namespace vb
