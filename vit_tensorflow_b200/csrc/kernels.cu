// Non-tensor-core kernels: vectorised HBM-bound ops (im2col, LayerNorm, pooling, copies) for both precisions
// and the exact-fp32 SIMT GEMM / attention used by the fp32 numerics gate (BASELINE config 1) and as the
// general fallback of the bf16 path.  See kernels.cuh for the contracts and the reference lines replaced.
#include "kernels.cuh"
#include "philox.cuh"
#include <atomic>

namespace vb {

namespace {

std::atomic<long long> g_launches{0};

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

inline int blocks_for(long long work, int per_block) { return static_cast<int>((work + per_block - 1) / per_block); }

// ------------------------------------------------------------------------------------------ im2col
// One thread per 4 consecutive output elements of a patch row segment (pw*C contiguous floats in the image); the VEC4 form
// keeps four independent 16-byte loads in flight per thread before the first store (ncu: 2.95 TB/s with one).
template <typename T, bool VEC4>
__global__ void im2col_kernel(const float* __restrict__ img, T* __restrict__ out, int B, int H, int W, int C, int ph, int pw,
                              int cls_row, int ldo) {
  const int gh = H / ph, gw = W / pw;
  const int rows = cls_row + gh * gw;
  const int seg = pw * C;                 // contiguous run shared by input and output
  const int K = ph * seg;
  constexpr int V = VEC4 ? 4 : 1;
  constexpr int U = VEC4 ? 4 : 1;         // units per thread per sweep
  const int units_per_row = ldo / V;      // ldo % 4 == 0 when VEC4
  const long long total = static_cast<long long>(B) * rows * units_per_row;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long base = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; base < total; base += stride * U) {
    float v[U][V];
    T* dst[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long idx = base + u * stride;
#pragma unroll
      for (int i = 0; i < V; ++i) v[u][i] = 0.f;
      dst[u] = nullptr;
      if (idx < total) {
        const int un = static_cast<int>(idx % units_per_row);
        const long long r = idx / units_per_row;
        const int t = static_cast<int>(r % rows);
        const int b = static_cast<int>(r / rows);
        const int col = un * V;
        dst[u] = out + r * ldo + col;
        if (t >= cls_row && col < K) {
          const int p = t - cls_row;
          const int py = p / gw, px = p % gw;
          const int p1 = col / seg, off = col % seg;
          const float* src = img + ((static_cast<long long>(b) * H + py * ph + p1) * W + px * pw) * C + off;
          if (VEC4) {
            const float4 f = *reinterpret_cast<const float4*>(src);   // seg % 4 == 0 -> never straddles a segment
            v[u][0] = f.x; v[u][1 % V] = f.y; v[u][2 % V] = f.z; v[u][3 % V] = f.w;
          } else {
            v[u][0] = *src;
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (dst[u] == nullptr) continue;
      if (VEC4) {
        if (sizeof(T) == 4) {
          *reinterpret_cast<float4*>(dst[u]) = make_float4(v[u][0], v[u][1 % V], v[u][2 % V], v[u][3 % V]);
        } else {
          __nv_bfloat162 lo = __floats2bfloat162_rn(v[u][0], v[u][1 % V]);
          __nv_bfloat162 hi = __floats2bfloat162_rn(v[u][2 % V], v[u][3 % V]);
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&lo);
          pk.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(dst[u]) = pk;
        }
      } else {
        dst[u][0] = from_f<T>(v[u][0]);
      }
    }
  }
}

template <typename T>
__global__ void embed_residual_kernel(T* __restrict__ R, const float* __restrict__ pos, const float* __restrict__ cls,
                                      const float* __restrict__ bias, int B, int rows, int dim, int has_cls) {
  const long long total = static_cast<long long>(B) * rows * dim;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(idx % dim);
    const int t = static_cast<int>((idx / dim) % rows);
    float v = pos[static_cast<long long>(t) * dim + d];
    if (has_cls && t == 0) v += cls[d] - bias[d];
    R[idx] = from_f<T>(v);
  }
}

// ------------------------------------------------------------------------------------------ LayerNorm
// One warp per row, row cached in registers (8-element chunks: 16-byte bf16 / 2x16-byte fp32 accesses).
template <typename T, int MAXC>
__global__ void layernorm_kernel(const T* __restrict__ x, int ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 T* __restrict__ out, int ldo, int M, int D, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const int nchunks = D >> 3;              // D % 8 == 0
  const T* xr = x + static_cast<long long>(row) * ldx;
  float v[MAXC][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXC; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      if (sizeof(T) == 2) {
        const uint4 pk = *reinterpret_cast<const uint4*>(xr + c * 8);
        const uint32_t w4[4] = {pk.x, pk.y, pk.z, pk.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          v[i][2 * j] = __uint_as_float(w4[j] << 16);
          v[i][2 * j + 1] = __uint_as_float(w4[j] & 0xFFFF0000u);
        }
      } else {
        const float4 a = *reinterpret_cast<const float4*>(xr + c * 8);
        const float4 b = *reinterpret_cast<const float4*>(xr + c * 8 + 4);
        v[i][0] = a.x; v[i][1] = a.y; v[i][2] = a.z; v[i][3] = a.w;
        v[i][4] = b.x; v[i][5] = b.y; v[i][6] = b.z; v[i][7] = b.w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[i][j];
    }
  }
  const float mean = warp_sum(sum) / D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXC; ++i) {
    if (lane + 32 * i < nchunks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; sq += d * d; }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / D + eps);
  T* orow = out + static_cast<long long>(row) * ldo;
#pragma unroll
  for (int i = 0; i < MAXC; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      float y[8];
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c * 8));
      const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c * 8 + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + c * 8 + 4));
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = (v[i][j] - mean) * rstd * g[j] + bb[j];
      if (sizeof(T) == 2) {
        uint4 pk;
        __nv_bfloat162 p0 = __floats2bfloat162_rn(y[0], y[1]), p1 = __floats2bfloat162_rn(y[2], y[3]);
        __nv_bfloat162 p2 = __floats2bfloat162_rn(y[4], y[5]), p3 = __floats2bfloat162_rn(y[6], y[7]);
        pk.x = *reinterpret_cast<uint32_t*>(&p0); pk.y = *reinterpret_cast<uint32_t*>(&p1);
        pk.z = *reinterpret_cast<uint32_t*>(&p2); pk.w = *reinterpret_cast<uint32_t*>(&p3);
        *reinterpret_cast<uint4*>(orow + c * 8) = pk;
      } else {
        *reinterpret_cast<float4*>(orow + c * 8) = make_float4(y[0], y[1], y[2], y[3]);
        *reinterpret_cast<float4*>(orow + c * 8 + 4) = make_float4(y[4], y[5], y[6], y[7]);
      }
    }
  }
}

// Any D / alignment: one warp per row, three passes over the (L1-resident) row.
template <typename T>
__global__ void layernorm_generic_kernel(const T* __restrict__ x, int ldx, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, T* __restrict__ out, int ldo, int M, int D, int pad_to,
                                         float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const T* xr = x + static_cast<long long>(row) * ldx;
  float sum = 0.f;
  for (int d = lane; d < D; d += 32) sum += to_f(xr[d]);
  const float mean = warp_sum(sum) / D;
  float sq = 0.f;
  for (int d = lane; d < D; d += 32) { const float t = to_f(xr[d]) - mean; sq += t * t; }
  const float rstd = rsqrtf(warp_sum(sq) / D + eps);
  T* orow = out + static_cast<long long>(row) * ldo;
  for (int d = lane; d < D; d += 32) orow[d] = from_f<T>((to_f(xr[d]) - mean) * rstd * gamma[d] + beta[d]);
  for (int d = D + lane; d < pad_to; d += 32) orow[d] = from_f<T>(0.f);     // zero pad columns [D, pad_to) (pitch-padded token rows)
}

// Row softmax of materialised fp32 scores -> bf16 probabilities (the T2T soft-split attention, t2t.py:35: one head of width
// 147 / 1323 over 3136 / 784 tokens, far outside the fused kernels' head widths).  One block per row, the row in registers;
// S holds q.k (unscaled), scale_log2 = dim_head^-0.5 * log2(e); columns [n, npad) of P are zeroed (the PV GEMM's K padding).
constexpr int SM_THREADS = 256, SM_MAXE = 16;
__global__ void __launch_bounds__(SM_THREADS)
softmax_rows_bf16_kernel(const float* __restrict__ S, int lds, __nv_bfloat16* __restrict__ P, int ldp, int n, int npad, float scale_log2) {
  __shared__ float red[SM_THREADS / 32];
  const long long row = blockIdx.x;
  const float* sr = S + row * lds;
  float v[SM_MAXE];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < SM_MAXE; ++i) {
    const int e = threadIdx.x + SM_THREADS * i;
    v[i] = e < n ? sr[e] * scale_log2 : -INFINITY;
    m = fmaxf(m, v[i]);
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < SM_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float l = 0.f;
#pragma unroll
  for (int i = 0; i < SM_MAXE; ++i) { v[i] = exp2f(v[i] - m); l += v[i]; }
  l = warp_sum(l);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  l = 0.f;
#pragma unroll
  for (int w = 0; w < SM_THREADS / 32; ++w) l += red[w];
  const float il = 1.0f / l;
  __nv_bfloat16* pr = P + row * ldp;
#pragma unroll
  for (int i = 0; i < SM_MAXE; ++i) {
    const int e = threadIdx.x + SM_THREADS * i;
    if (e < npad) pr[e] = __float2bfloat16_rn(e < n ? v[i] * il : 0.f);
  }
}

// any row length: three passes over the (L2-resident) row
__global__ void __launch_bounds__(SM_THREADS)
softmax_rows_bf16_big_kernel(const float* __restrict__ S, int lds, __nv_bfloat16* __restrict__ P, int ldp, int n, int npad, float scale_log2) {
  __shared__ float red[SM_THREADS / 32];
  const long long row = blockIdx.x;
  const float* sr = S + row * lds;
  float m = -INFINITY;
  for (int e = threadIdx.x; e < n; e += SM_THREADS) m = fmaxf(m, sr[e] * scale_log2);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < SM_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float l = 0.f;
  for (int e = threadIdx.x; e < n; e += SM_THREADS) l += exp2f(sr[e] * scale_log2 - m);
  l = warp_sum(l);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  l = 0.f;
  for (int w = 0; w < SM_THREADS / 32; ++w) l += red[w];
  const float il = 1.0f / l;
  __nv_bfloat16* pr = P + row * ldp;
  for (int e = threadIdx.x; e < npad; e += SM_THREADS) pr[e] = __float2bfloat16_rn(e < n ? exp2f(sr[e] * scale_log2 - m) * il : 0.f);
}

// out[b, c, j] = in[b, j, c] (bf16), c < cols, j < npad with zeros for j >= n: V -> V^T for the K-major B operand of the PV GEMM
__global__ void transpose_rows_bf16_kernel(const __nv_bfloat16* __restrict__ in, int ldi, long long in_batch, __nv_bfloat16* __restrict__ out,
                                           int ldo, long long out_batch, int n, int npad, int cols) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int jt = (npad + 31) / 32, ct = (cols + 31) / 32;            // flat grid, j tile fastest: no 65 535 limit on B
  const int tile_idx = static_cast<int>(blockIdx.x % (jt * ct)), b = static_cast<int>(blockIdx.x / (jt * ct));
  const int j0 = (tile_idx % jt) * 32, c0 = (tile_idx / jt) * 32;
  const __nv_bfloat16* ib = in + b * in_batch;
  __nv_bfloat16* ob = out + b * out_batch;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int j = j0 + r, c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (j < n && c < cols) ? ib[static_cast<long long>(j) * ldi + c] : __float2bfloat16_rn(0.f);
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r, j = j0 + threadIdx.x;
    if (c < cols && j < npad) ob[static_cast<long long>(c) * ldo + j] = tile[threadIdx.x][r];
  }
}

// ------------------------------------------------------------------------------------------ SIMT GEMM
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// (16*TM)x64 output tile, 16x16 threads x (TM x 4) micro-tile, BK = 16; exact fp32 FMA accumulation in k order.
// TM = 4: 64-row tiles; TM = 1: 16-row tiles for small-M problems (the classifier head) so the grid still fills the GPU.
// SILU: the SiLU epilogue (act is then ignored), an instance of its own so that the others keep their registers.
// DROP: training-mode dropout (DropPos), instances of their own likewise.
template <typename TA, typename TW, typename TO, int TM, bool SILU = false, int DROP = DROP_NONE>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const TA* __restrict__ A, int lda, const TW* __restrict__ W, int wsk, int wsn, TO* out, int ldc, int M, int N,
                 int K, const float* __restrict__ bias, const float* __restrict__ scale, const TO* res, int ldr, int act,
                 DropoutEpi drop) {
  constexpr int BMT = 16 * TM;
  __shared__ float As[16][BMT + 1];
  __shared__ __align__(16) float Ws[16][64 + 4];   // pitch 68 floats: 16-byte aligned rows, one LDS.128 per thread and k
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int n_tiles = (N + 63) / 64;                                // flat grid, n fastest: no 65 535 limit on the row tiles
  const int m0 = static_cast<int>(blockIdx.x / n_tiles) * BMT, n0 = static_cast<int>(blockIdx.x % n_tiles) * 64;
  float acc[TM][4];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  unsigned long long drop_seed = 0;
  uint32_t drop_d = 0;
  if constexpr (DROP != DROP_NONE) { drop_seed = drop.state[0]; drop_d = static_cast<uint32_t>(drop.state[1]); }
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int e = threadIdx.x; e < 16 * 64; e += 256) {
      if (e < 16 * BMT) {  // A tile: consecutive threads along k (contiguous in memory)
        const int kk = e & 15, mm = e >> 4;
        const int m = m0 + mm, k = k0 + kk;
        As[kk][mm] = (m < M && k < K) ? to_f(A[static_cast<long long>(m) * lda + k]) : 0.f;
      }
      {  // W tile: consecutive threads along the contiguous axis of W
        int kk, nn;
        if (wsn == 1) { nn = e & 63; kk = e >> 6; } else { kk = e & 15; nn = e >> 4; }
        const int n = n0 + nn, k = k0 + kk;
        Ws[kk][nn] = (n < N && k < K) ? to_f(W[static_cast<long long>(k) * wsk + static_cast<long long>(n) * wsn]) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[TM];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
      // the thread's four W columns in one 128-bit read (16 lanes x 16 B = two conflict-free wavefronts per warp; four
      // scalar reads at pitch 65 cost eight): the TM = 1 classifier-head GEMM was shared-memory-bandwidth bound
      const float4 w4 = *reinterpret_cast<const float4*>(&Ws[kk][tx * 4]);
      const float w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      if (SILU) v = silu(v);                                                      // mobile_vit.py:33
      else if (act == ACT_GELU) v = gelu_erf_f(v);
      else if (act == ACT_HSWISH) v = v * fminf(fmaxf(v + 3.0f, 0.0f), 6.0f) / 6.0f;   // levit.py:37
      const bool keep = DROP == DROP_NONE || dropout_keep_at(drop_seed, drop_d, drop.site, m, n, drop.rate);
      if (DROP == DROP_BEFORE_RES) v = keep ? v * drop.scale : 0.f;
      if (scale) v *= scale[n];
      if (res) v += to_f(res[static_cast<long long>(m) * ldr + n]);
      if (DROP == DROP_AFTER_RES) v = keep ? v * drop.scale : 0.f;
      out[static_cast<long long>(m) * ldc + n] = from_f<TO>(v);
    }
  }
}

// ------------------------------------------------------------------------------------------ generic attention
// S[b,h,i,j] = scale * sum_d q[b,i,h,d] k[b,j,h,d];  32x32 tile per block, 16x16 threads x (2x2).
template <typename T>
__global__ void __launch_bounds__(256)
attn_scores_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ k, int ldk, float* __restrict__ S, int heads, int nq,
                   int nk, int dh, float scale) {
  __shared__ float Qs[32][33];
  __shared__ float Ks[32][33];
  const int kt = (nk + 31) / 32, qt = (nq + 31) / 32;              // flat grid, key tile fastest: no 65 535 limit on B * heads
  const int bh = blockIdx.x / (kt * qt), b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x / kt % qt) * 32, j0 = (blockIdx.x % kt) * 32;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int d0 = 0; d0 < dh; d0 += 32) {
    for (int e = threadIdx.x; e < 32 * 32; e += 256) {
      const int dd = e & 31, rr = e >> 5;
      const int d = d0 + dd;
      const int i = i0 + rr, j = j0 + rr;
      Qs[rr][dd] = (i < nq && d < dh) ? to_f(q[(static_cast<long long>(b) * nq + i) * ldq + h * dh + d]) : 0.f;
      Ks[rr][dd] = (j < nk && d < dh) ? to_f(k[(static_cast<long long>(b) * nk + j) * ldk + h * dh + d]) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int dd = 0; dd < 32; ++dd) {
      const float a0 = Qs[ty * 2][dd], a1 = Qs[ty * 2 + 1][dd];
      const float b0 = Ks[tx * 2][dd], b1 = Ks[tx * 2 + 1][dd];
      acc[0][0] = fmaf(a0, b0, acc[0][0]); acc[0][1] = fmaf(a0, b1, acc[0][1]);
      acc[1][0] = fmaf(a1, b0, acc[1][0]); acc[1][1] = fmaf(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int i = i0 + ty * 2 + a, j = j0 + tx * 2 + c;
      if (i < nq && j < nk) S[(static_cast<long long>(bh) * nq + i) * nk + j] = acc[a][c] * scale;
    }
}

constexpr int MAX_HEADS = 32;
// one thread per (b,i,j): y[g] = sum_h x[h] W[h,g]; optional LayerNorm over g (eps 1e-3)
__global__ void attn_head_mix_kernel(float* __restrict__ S, const float* __restrict__ Wmix, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, int B, int heads, long long plane /* nq*nk */) {
  __shared__ float Wm[MAX_HEADS * MAX_HEADS];
  for (int e = threadIdx.x; e < heads * heads; e += blockDim.x) Wm[e] = Wmix[e];
  __syncthreads();
  const long long total = static_cast<long long>(B) * plane;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = idx / plane, ij = idx % plane;
    float* base = S + b * heads * plane + ij;
    float x[MAX_HEADS], y[MAX_HEADS];
    for (int h = 0; h < heads; ++h) x[h] = base[h * plane];
    for (int g = 0; g < heads; ++g) {
      float a = 0.f;
      for (int h = 0; h < heads; ++h) a = fmaf(x[h], Wm[h * heads + g], a);
      y[g] = a;
    }
    if (gamma != nullptr) {
      float mean = 0.f;
      for (int g = 0; g < heads; ++g) mean += y[g];
      mean /= heads;
      float var = 0.f;
      for (int g = 0; g < heads; ++g) { const float d = y[g] - mean; var += d * d; }
      const float rstd = rsqrtf(var / heads + 1e-3f);
      for (int g = 0; g < heads; ++g) y[g] = (y[g] - mean) * rstd * gamma[g] + beta[g];
    }
    for (int g = 0; g < heads; ++g) base[g * plane] = y[g];
  }
}

__global__ void attn_softmax_kernel(float* __restrict__ S, long long rows, int nk) {
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float* r = S + row * nk;
  float mx = -INFINITY;
  for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, r[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nk; j += 32) { const float e = expf(r[j] - mx); r[j] = e; sum += e; }
  const float inv = 1.0f / warp_sum(sum);
  for (int j = lane; j < nk; j += 32) r[j] *= inv;
}

// out[b,i,h,d] = sum_j S[b,h,i,j] v[b,j,h,d];  32(i) x 32(d) tile per block
template <typename T>
__global__ void __launch_bounds__(256)
attn_pv_kernel(const float* __restrict__ S, const T* __restrict__ v, int ldv, T* __restrict__ out, int ldo, int heads, int nq, int nk,
               int dh, int gelu_out) {
  __shared__ float Ps[32][33];
  __shared__ float Vs[32][33];
  const int dt = (dh + 31) / 32, qt = (nq + 31) / 32;              // flat grid, column tile fastest
  const int bh = blockIdx.x / (dt * qt), b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x / dt % qt) * 32, d0 = (blockIdx.x % dt) * 32;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int j0 = 0; j0 < nk; j0 += 32) {
    for (int e = threadIdx.x; e < 32 * 32; e += 256) {
      const int cc = e & 31, rr = e >> 5;
      const int i = i0 + rr, j = j0 + cc;
      Ps[rr][cc] = (i < nq && j < nk) ? S[(static_cast<long long>(bh) * nq + i) * nk + j] : 0.f;
      const int jj = j0 + rr, d = d0 + cc;
      Vs[rr][cc] = (jj < nk && d < dh) ? to_f(v[(static_cast<long long>(b) * nk + jj) * ldv + h * dh + d]) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int jj = 0; jj < 32; ++jj) {
      const float a0 = Ps[ty * 2][jj], a1 = Ps[ty * 2 + 1][jj];
      const float b0 = Vs[jj][tx * 2], b1 = Vs[jj][tx * 2 + 1];
      acc[0][0] = fmaf(a0, b0, acc[0][0]); acc[0][1] = fmaf(a0, b1, acc[0][1]);
      acc[1][0] = fmaf(a1, b0, acc[1][0]); acc[1][1] = fmaf(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int i = i0 + ty * 2 + a, d = d0 + tx * 2 + c;
      if (i < nq && d < dh) out[(static_cast<long long>(b) * nq + i) * ldo + h * dh + d] = from_f<T>(gelu_out ? gelu_exact(acc[a][c]) : acc[a][c]);
    }
}

// S[b,h,i,j] += table[h, pos_bias_index(i, j)]  (materialised scores, row pitch nk)
__global__ void attn_pos_bias_kernel(float* __restrict__ S, const float* __restrict__ table, int heads, int nq, int nk, int fmap,
                                     int step, long long total) {
  const int nqs = (fmap + step - 1) / step;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % nk);
    const long long r = idx / nk;
    const int i = static_cast<int>(r % nq), h = static_cast<int>((r / nq) % heads);
    S[idx] += table[static_cast<long long>(h) * fmap * fmap + pos_bias_index(i, j, fmap, step, nqs)];
  }
}

// S[w,h,i,j] += table[window_bias_index(i, j, wsz)]  (CrossFormer's window table, shared by the heads; row pitch nk = wsz^2)
__global__ void attn_window_bias_kernel(float* __restrict__ S, const float* __restrict__ table, int nk, int wsz, long long total) {
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % nk), i = static_cast<int>((idx / nk) % nk);
    S[idx] += table[window_bias_index(i, j, wsz)];
  }
}

// S[w,h,i,j] += table[h, r2l_bias_index(i, j)] for i, j > 0  (RegionViT's window table; row pitch nk = 1 + wh * ww)
__global__ void attn_r2l_bias_kernel(float* __restrict__ S, const float* __restrict__ table, int heads, int nk, int ww, int ws,
                                     long long total) {
  const int t2 = (2 * ws - 1) * (2 * ws - 1);
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % nk);
    const long long r = idx / nk;
    const int i = static_cast<int>(r % nk), h = static_cast<int>((r / nk) % heads);
    if (i > 0 && j > 0) S[idx] += table[static_cast<long long>(h) * t2 + r2l_bias_index(i, j, ww, ws)];
  }
}

// One CTA per window-major row t = bw * n + i: i == 0 is the regional row reg_row0 + bw, i > 0 the local row win.row(bw, i - 1).
template <typename T>
__global__ void r2l_rows_kernel(const T* __restrict__ in, int ldi, T* __restrict__ out, int ldo, int cols, Window win, int n,
                                long long reg_row0, bool to_window) {
  const long long t = blockIdx.x, bw = t / n;
  const int i = static_cast<int>(t - bw * n);
  const long long px = i == 0 ? reg_row0 + bw : win.row(bw, i - 1);
  const T* __restrict__ src = in + (to_window ? px : t) * ldi;
  T* __restrict__ dst = out + (to_window ? t : px) * ldo;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) dst[c] = src[c];
}

// out[b, r*ow + c, :] = in[b, (step*r)*W + step*c, :]  (16-byte vectors when C, ld are multiples of the vector width)
template <typename T>
__global__ void gather_grid_kernel(const T* __restrict__ in, int ldi, T* __restrict__ out, int ldo, int H, int W, int C, int step,
                                   int oh, int ow, long long total_vec, int vec) {
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total_vec;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = C / vec;
    const int c = static_cast<int>(idx % cv) * vec;
    const long long p = idx / cv;
    const int pc = static_cast<int>(p % ow), pr = static_cast<int>((p / ow) % oh);
    const long long b = p / (static_cast<long long>(ow) * oh);
    const T* src = in + ((b * H + static_cast<long long>(pr) * step) * W + static_cast<long long>(pc) * step) * ldi + c;
    T* dst = out + p * ldo + c;
    if (vec * sizeof(T) == 16) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    else for (int e = 0; e < vec; ++e) dst[e] = src[e];
  }
}

// ------------------------------------------------------------------------------------------ pooling + head LN
template <typename T>
__global__ void pool_layernorm_kernel(const T* __restrict__ X, int n, int ldx, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, float* __restrict__ out, int D, int mean_pool) {
  extern __shared__ float z[];  // [D] pooled vector
  __shared__ float red[32];
  const int b = blockIdx.x;
  const T* xb = X + static_cast<long long>(b) * n * ldx;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float v;
    if (mean_pool) {
      float s = 0.f;
      for (int t = 0; t < n; ++t) s += to_f(xb[static_cast<long long>(t) * ldx + d]);
      v = s / n;
    } else {
      v = to_f(xb[d]);
    }
    z[d] = v;
  }
  __syncthreads();
  if (gamma == nullptr) {                                           // GlobalAvgPool2D alone (levit.py:206-208)
    for (int d = threadIdx.x; d < D; d += blockDim.x) out[static_cast<long long>(b) * D + d] = z[d];
    return;
  }
  auto block_sum = [&](float v) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
      t = warp_sum(t);
      if (threadIdx.x == 0) red[0] = t;
    }
    __syncthreads();
    const float total = red[0];
    __syncthreads();
    return total;
  };
  float s = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) s += z[d];
  const float mean = block_sum(s) / D;
  float sq = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) { const float t = z[d] - mean; sq += t * t; }
  const float rstd = rsqrtf(block_sum(sq) / D + 1e-3f);
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    out[static_cast<long long>(b) * D + d] = (z[d] - mean) * rstd * gamma[d] + beta[d];
}

template <typename T>
__global__ void copy_tokens_kernel(const T* __restrict__ src, int src_rows, int soff, T* __restrict__ dst, int dst_rows, int doff,
                                   int count, int B, int D) {
  const long long total = static_cast<long long>(B) * count * D;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(idx % D);
    const int t = static_cast<int>((idx / D) % count);
    const long long b = idx / (static_cast<long long>(D) * count);
    dst[(b * dst_rows + doff + t) * D + d] = src[(b * src_rows + soff + t) * D + d];
  }
}

template <typename T>
__global__ void broadcast_row_kernel(const float* __restrict__ vec, T* __restrict__ dst, int dst_rows, int B, int D) {
  const long long total = static_cast<long long>(B) * D;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(idx % D);
    const long long b = idx / D;
    dst[b * dst_rows * D + d] = from_f<T>(vec[d]);
  }
}

// dst[b, t, :] = vec[t, :] (fp32 [nt, D]) for every b: learned query rows shared by all images
template <typename T>
__global__ void broadcast_rows_kernel(const float* __restrict__ vec, T* __restrict__ dst, int B, int nt, int D) {
  const long long per = static_cast<long long>(nt) * D, total = per * B;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[idx] = from_f<T>(vec[idx % per]);
}

// Soft split of T2T: tf.image.extract_patches(sizes k x k, strides s, rates 1, padding SAME) (t2t.py:43) followed by
// 'b h w c -> b (h w) c' (:44).  Taps outside the image read 0; the patch vector is (k_row, k_col, channel) with the channel
// fastest.  One CTA per output row (b, t): no 64-bit index arithmetic and no division per element (one thread per output
// element would cost six divisions each, two of them 64-bit).
// C >= 32 (the 147-channel layers): the threads walk the k*k taps and copy each tap's C contiguous channels;
// small C (the image, C = 3): one thread per column with 32-bit divisions.
// stats (UnfoldMode, may be null): the pixel's LayerNorm from its (sum, sumsq) partials, applied on load.
__device__ __forceinline__ float2 unfold_ln(const float2* __restrict__ stats, int parts, long long M, long long pix, float inv_d, float eps) {
  float s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < parts; ++j) {
    const float2 v = __ldg(stats + j * M + pix);
    s1 += v.x;
    s2 += v.y;
  }
  const float m = s1 * inv_d;
  return make_float2(m, rsqrtf(fmaxf(s2 * inv_d - m * m, 0.f) + eps));
}
template <typename TI, typename TO>
__global__ void unfold_same_kernel(const TI* __restrict__ in, int ldi, TO* __restrict__ out, int B, int H, int W, int C, int k, int stride,
                                   int oh, int ow, int pad_top, int pad_left, int cls_row, int ldo, const float2* __restrict__ stats,
                                   int parts, float inv_d, float eps, const float* __restrict__ gamma, const float* __restrict__ beta,
                                   int gelu) {
  const int rows = cls_row + oh * ow;
  const int K = k * k * C;
  const int r = blockIdx.x;                                    // (b, t): B * rows CTAs
  const int b = r / rows, t = r - b * rows;
  TO* __restrict__ orow = out + static_cast<size_t>(r) * ldo;
  if (t < cls_row) {                                           // reserved rows (cls slots): zero, the caller fills them
    for (int col = threadIdx.x; col < ldo; col += blockDim.x) orow[col] = from_f<TO>(0.f);
    return;
  }
  const int p = t - cls_row;
  const int oy = p / ow, ox = p - oy * ow;
  const int y0 = oy * stride - pad_top, x0 = ox * stride - pad_left;
  const TI* __restrict__ img = in + static_cast<size_t>(b) * H * W * ldi;
  if (C >= 32) {
    for (int tap = 0; tap < k * k; ++tap) {
      const int ky = tap / k, kx = tap - ky * k;
      const int y = y0 + ky, x = x0 + kx;
      const bool inside = y >= 0 && y < H && x >= 0 && x < W;
      const TI* __restrict__ src = img + (static_cast<size_t>(inside ? y : 0) * W + (inside ? x : 0)) * ldi;
      TO* __restrict__ dst = orow + tap * C;
      if (stats != nullptr && inside) {
        const float2 mr = unfold_ln(stats, parts, static_cast<long long>(B) * H * W, (static_cast<long long>(b) * H + y) * W + x, inv_d, eps);
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
          const float v = (to_f(src[c]) - mr.x) * mr.y * gamma[c] + beta[c];
          dst[c] = from_f<TO>(gelu ? gelu_exact(v) : v);
        }
      } else {
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
          const float v = inside ? to_f(src[c]) : 0.f;
          dst[c] = from_f<TO>(gelu && inside ? gelu_exact(v) : v);
        }
      }
    }
  } else {
    const int kC = k * C;
    for (int col = threadIdx.x; col < K; col += blockDim.x) {
      const int ky = col / kC, rem = col - ky * kC;
      const int kx = rem / C, c = rem - kx * C;
      const int y = y0 + ky, x = x0 + kx;
      float v = 0.f;
      if (y >= 0 && y < H && x >= 0 && x < W) {
        v = to_f(img[(static_cast<size_t>(y) * W + x) * ldi + c]);
        if (stats != nullptr) {
          const float2 mr = unfold_ln(stats, parts, static_cast<long long>(B) * H * W, (static_cast<long long>(b) * H + y) * W + x, inv_d, eps);
          v = (v - mr.x) * mr.y * gamma[c] + beta[c];
        }
        if (gelu) v = gelu_exact(v);
      }
      orow[col] = from_f<TO>(v);
    }
  }
  for (int col = K + threadIdx.x; col < ldo; col += blockDim.x) orow[col] = from_f<TO>(0.f);   // pitch padding
}

// One CTA per window-major row.
template <typename T>
__global__ void window_rows_kernel(const T* __restrict__ in, int ldi, T* __restrict__ out, int ldo, int cols, Window win, int n,
                                   bool to_window) {
  const long long t = blockIdx.x, px = win.row(t / n, static_cast<int>(t % n));
  const T* __restrict__ src = in + (to_window ? px : t) * ldi;
  T* __restrict__ dst = out + (to_window ? t : px) * ldo;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) dst[c] = src[c];
}

// One warp per output pixel, lane l holding columns 64 j + 2 l and 64 j + 2 l + 1 of chunk j: each tap's LayerNorm (mean, rstd)
// comes from that input pixel's statistics once per tap, and the chunk's (sum, sumsq) by a warp reduction of the stored values.
// `in` may alias `out` when pool == 0 (every element is read and written by the same lane).
constexpr int NEST_POOL_WARPS = 8;
template <typename T>
__global__ void __launch_bounds__(NEST_POOL_WARPS * 32, 4)
nest_pool_kernel(const T* in, int ldi, const float2* __restrict__ stats, int parts, float inv_d, float eps,
                 const float* __restrict__ gamma, const float* __restrict__ beta, int C, int H, int W, int pool, int oh, int ow,
                 int pad_top, int pad_left, const float* __restrict__ pos, int bh, int bw, T* out, int ldo,
                 float2* __restrict__ stats_out, long long pixels) {
  const long long px = static_cast<long long>(blockIdx.x) * NEST_POOL_WARPS + (threadIdx.x >> 5);
  if (px >= pixels) return;
  const int lane = threadIdx.x & 31;
  const long long b = px / (static_cast<long long>(oh) * ow);
  const int t = static_cast<int>(px - b * oh * ow), oy = t / ow, ox = t - oy * ow;
  const long long in_pixels = static_cast<long long>(pixels / (static_cast<long long>(oh) * ow)) * H * W;
  const int k = pool ? 3 : 1, st = pool ? 2 : 1;
  const int y0 = oy * st - pad_top, x0 = ox * st - pad_left;
  const float p = pos != nullptr ? __ldg(pos + (oy % bh) * bw + (ox % bw)) : 0.f;
  for (int c0 = 0; c0 < ldo; c0 += 64) {
    const int c = c0 + 2 * lane;
    float m0 = -INFINITY, m1 = -INFINITY;
    for (int ky = 0; ky < k; ++ky) {
      const int y = y0 + ky;
      if (y < 0 || y >= H) continue;                               // TF SAME: padded taps never win
      for (int kx = 0; kx < k; ++kx) {
        const int x = x0 + kx;
        if (x < 0 || x >= W) continue;
        const long long ip = (b * H + y) * W + x;
        const T* src = in + ip * ldi;
        float v0 = c < C ? to_f(src[c]) : 0.f, v1 = c + 1 < C ? to_f(src[c + 1]) : 0.f;
        if (stats != nullptr) {
          float s1 = 0.f, s2 = 0.f;
          for (int j = 0; j < parts; ++j) {
            const float2 sv = __ldg(stats + j * in_pixels + ip);
            s1 += sv.x;
            s2 += sv.y;
          }
          const float mean = s1 * inv_d, rstd = rsqrtf(fmaxf(s2 * inv_d - mean * mean, 0.f) + eps);
          if (c < C) v0 = (v0 - mean) * rstd * gamma[c] + beta[c];
          if (c + 1 < C) v1 = (v1 - mean) * rstd * gamma[c + 1] + beta[c + 1];
        }
        m0 = fmaxf(m0, v0);
        m1 = fmaxf(m1, v1);
      }
    }
    // the position scalar goes to the true channels only; pad channels stay zero
    const T o0 = from_f<T>(c < C ? m0 + p : 0.f), o1 = from_f<T>(c + 1 < C ? m1 + p : 0.f);
    T* dst = out + px * ldo;
    if (c < ldo) dst[c] = o0;
    if (c + 1 < ldo) dst[c + 1] = o1;
    if (stats_out != nullptr) {
      const float f0 = to_f(o0), f1 = to_f(o1);
      float s1 = f0 + f1, s2 = f0 * f0 + f1 * f1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      }
      if (lane == 0) stats_out[(c0 / 64) * pixels + px] = make_float2(s1, s2);
    }
  }
}

// One thread per output element (b, t, c), c fastest: the k*k taps of a thread are C apart, so a warp reads whole channel runs.
template <typename T>
__global__ void maxpool_relu_same_kernel(const T* __restrict__ in, T* __restrict__ out, int H, int W, int C, int k, int stride, int oh,
                                         int ow, int pad_top, int pad_left, const float* __restrict__ pos, int rows, long long total) {
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % C);
    const long long r = idx / C;
    const int t = static_cast<int>(r % rows);
    const long long b = r / rows;
    float v = 0.f;
    if (t < oh * ow) {
      const int oy = t / ow, ox = t - oy * ow;
      const int y0 = oy * stride - pad_top, x0 = ox * stride - pad_left;
      const T* __restrict__ img = in + b * H * W * C + c;
      float m = -INFINITY;
      for (int ky = 0; ky < k; ++ky) {
        const int y = y0 + ky;
        if (y < 0 || y >= H) continue;
        for (int kx = 0; kx < k; ++kx) {
          const int x = x0 + kx;
          if (x >= 0 && x < W) m = fmaxf(m, to_f(img[(static_cast<long long>(y) * W + x) * C]));
        }
      }
      v = fmaxf(m, 0.f);
      if (pos != nullptr) v += pos[static_cast<long long>(t) * C + c];
    }
    out[idx] = from_f<T>(v);
  }
}

// One CTA per image, 8 warps; warp w takes rows w, w + 8, ...: LayerNorm of the row in registers (lane holds columns
// lane + 32 j), score by a warp reduction, and a running (max, sum, weighted row sum) per warp; the warps' partial states are
// merged through shared memory at the end.  The LayerNorm affine is taken out of the loop: with x^ the standardised row,
// score = x^ . (gamma * pw) + (beta . pw + pb), and since the weights sum to one, z = gamma * sum_t w_t x^_t + beta.
constexpr int SEQ_POOL_WARPS = 8;
template <typename T, int J>
__global__ void __launch_bounds__(SEQ_POOL_WARPS * 32)
seq_pool_kernel(const T* __restrict__ X, int n, int D, const float* __restrict__ gamma, const float* __restrict__ beta,
                const float* __restrict__ pw, const float* __restrict__ pb, float* __restrict__ z) {
  extern __shared__ float sp[];                  // [SEQ_POOL_WARPS][D] partial sums, then [2][SEQ_POOL_WARPS] (max, sum)
  float* acc_s = sp;
  float* ml = sp + SEQ_POOL_WARPS * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const T* __restrict__ xb = X + static_cast<long long>(blockIdx.x) * n * D;
  float gw[J], acc[J], cb = 0.f;
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int d = lane + 32 * j;
    const bool in = d < D;
    gw[j] = in ? gamma[d] * pw[d] : 0.f;
    if (in) cb = fmaf(beta[d], pw[d], cb);
    acc[j] = 0.f;
  }
  const float bias = warp_sum(cb) + pb[0], inv_d = 1.0f / static_cast<float>(D);
  float m = -INFINITY, l = 0.f;
  for (int t = warp; t < n; t += SEQ_POOL_WARPS) {
    const T* __restrict__ row = xb + static_cast<long long>(t) * D;
    float v[J];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int d = lane + 32 * j;
      v[j] = d < D ? to_f(row[d]) : 0.f;
      s += v[j];
    }
    const float mean = warp_sum(s) * inv_d;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const float e = lane + 32 * j < D ? v[j] - mean : 0.f;
      q += e * e;
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_d + 1e-3f);
    float sc = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      v[j] = (v[j] - mean) * rstd;
      sc = fmaf(v[j], gw[j], sc);                    // gw = 0 beyond D
    }
    sc = warp_sum(sc) + bias;
    const float m_new = fmaxf(m, sc);
    const float corr = expf(m - m_new), p = expf(sc - m_new);
    l = l * corr + p;
#pragma unroll
    for (int j = 0; j < J; ++j) acc[j] = fmaf(acc[j], corr, p * v[j]);
    m = m_new;
  }
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int d = lane + 32 * j;
    if (d < D) acc_s[warp * D + d] = acc[j];
  }
  if (lane == 0) { ml[warp] = m; ml[SEQ_POOL_WARPS + warp] = l; }
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < SEQ_POOL_WARPS; ++w) M = fmaxf(M, ml[w]);
  float f[SEQ_POOL_WARPS], L = 0.f;
#pragma unroll
  for (int w = 0; w < SEQ_POOL_WARPS; ++w) {
    f[w] = ml[SEQ_POOL_WARPS + w] > 0.f ? expf(ml[w] - M) : 0.f;   // warps without rows hold (-inf, 0)
    L = fmaf(ml[SEQ_POOL_WARPS + w], f[w], L);
  }
  const float inv_l = 1.0f / L;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < SEQ_POOL_WARPS; ++w) a = fmaf(acc_s[w * D + d], f[w], a);
    z[static_cast<long long>(blockIdx.x) * D + d] = fmaf(gamma[d], a * inv_l, beta[d]);
  }
}

// out[r, c] = in[r, c] for c < cols, 0 for cols <= c < ldo (row-pitch change with conversion)
template <typename TI, typename TO>
__global__ void convert_rows_kernel(const TI* __restrict__ in, int ldi, TO* __restrict__ out, int ldo, long long rows, int cols) {
  const long long total = rows * ldo;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % ldo);
    const long long r = idx / ldo;
    out[idx] = from_f<TO>(c < cols ? to_f(in[r * ldi + c]) : 0.f);
  }
}

template <typename TI, typename TO>
__global__ void convert_kernel(const TI* __restrict__ in, TO* __restrict__ out, long long count) {
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < count;
       idx += static_cast<long long>(gridDim.x) * blockDim.x)
    out[idx] = from_f<TO>(to_f(in[idx]));
}

__global__ void add_inplace_kernel(float* __restrict__ a, const float* __restrict__ b, long long count) {
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < count;
       idx += static_cast<long long>(gridDim.x) * blockDim.x)
    a[idx] += b[idx];
}

// 32x32 smem-transposed: reads W[k,n] coalesced along n, writes Wt[n,k] coalesced along k
__global__ void pack_weight_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ Wt, int K, int N, int ldw,
                                   const float* __restrict__ row_scale) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int k = k0 + r, n = n0 + threadIdx.x;
    float v = (k < K && n < N) ? W[static_cast<long long>(k) * N + n] : 0.f;
    if (row_scale != nullptr && k < K) v *= row_scale[k];
    tile[r][threadIdx.x] = v;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int n = n0 + r, k = k0 + threadIdx.x;
    if (n < N && k < ldw) Wt[static_cast<long long>(n) * ldw + k] = __float2bfloat16_rn(tile[threadIdx.x][r]);
  }
}

// one warp per output column n
__global__ void ln_fold_consts_kernel(const float* __restrict__ W, const __nv_bfloat16* __restrict__ Wt, int ldw,
                                      const float* __restrict__ beta, const float* __restrict__ bias, float* __restrict__ c1,
                                      float* __restrict__ c2, int K, int N) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const int lane = threadIdx.x & 31;
  float a = 0.f, b = 0.f;
  for (int k = lane; k < K; k += 32) {
    a += __bfloat162float(Wt[static_cast<long long>(n) * ldw + k]);
    b = fmaf(beta[k], W[static_cast<long long>(k) * N + n], b);
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) { c1[n] = a; c2[n] = b + (bias ? bias[n] : 0.f); }
}

// one thread per (row, 64-column chunk)
__global__ void row_stats_kernel(const __nv_bfloat16* __restrict__ X, int ldx, float2* __restrict__ stats, int M, int parts,
                                 long long pitch) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(M) * parts) return;
  const int c = static_cast<int>(idx % parts);
  const long long m = idx / parts;
  const uint4* p = reinterpret_cast<const uint4*>(X + m * ldx + c * 64);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 v = p[i];
    const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = __uint_as_float(w4[j] << 16), b = __uint_as_float(w4[j] & 0xFFFF0000u);
      s1 += a + b;
      s2 = fmaf(a, a, fmaf(b, b, s2));
    }
  }
  stats[c * pitch + m] = make_float2(s1, s2);      // [part][pitch], the layout the GEMM epilogue emits (pitch M)
}

__global__ void pad_heads_kernel(const float* __restrict__ W, float* __restrict__ Wp, int other, int groups, int heads, int dh, int dhp,
                                 int pad_rows) {
  const long long total = static_cast<long long>(other) * groups * heads * dhp;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int wide = groups * heads * dhp, narrow = groups * heads * dh;
    long long o; int c;                              // o: index along the untouched dimension, c: padded (g, h, d) index
    if (pad_rows) { c = static_cast<int>(idx / other); o = idx % other; } else { o = idx / wide; c = static_cast<int>(idx % wide); }
    const int d = c % dhp, gh = c / dhp;
    float v = 0.f;
    if (d < dh) v = pad_rows ? W[static_cast<long long>(gh * dh + d) * other + o] : W[o * narrow + gh * dh + d];
    Wp[idx] = v;
  }
}

// ------------------------------------------------------------------------------------------ CvT depthwise convolutions
// One CTA: a DW_T x DW_T tile of the stride-1 (q) output map x DW_CG channels of one image.  The input tile with its halo
// (DW_T + K - 1 square, zero outside the map) is read once into shared memory -- LayerNormed on load from the rows' (sum,
// sumsq) partials when `stats` is given, so the halo holds zeros of the NORMALISED map, as the reference's SAME padding of
// LN(x) does -- and both convolutions read it: warp w computes row w of the q tile (DW_T outputs per lane, one channel per
// lane), and for the k|v map the outputs r whose 2r (stride 2) or r (stride 1) falls in the tile.  With TF SAME padding the
// stride-2 map's top / left padding is the stride-1 one's or one less (kv_dy / kv_dx), so its windows lie inside the halo.
constexpr int DW_T = 8, DW_CG = 32, DW_THREADS = DW_CG * DW_T, DW_MAXK = 7;
// One row of DW_T stride-1 outputs of lane's channel: tile rows row .. row + K - 1; out points at the row's first output, n_valid
// of them inside the map.
template <typename T, int K>
__device__ __forceinline__ void dw_conv_row(const float (*tile)[DW_CG], const float (*taps)[DW_CG], float shift, T* out, int ld, int row,
                                            int lane, int n_valid) {
  constexpr int TS = DW_T + K - 1;
  float acc[DW_T];
#pragma unroll
  for (int xx = 0; xx < DW_T; ++xx) acc[xx] = 0.f;
#pragma unroll
  for (int i = 0; i < K; ++i) {
    float xr[TS];
#pragma unroll
    for (int j = 0; j < TS; ++j) xr[j] = tile[(row + i) * TS + j][lane];
#pragma unroll
    for (int j = 0; j < K; ++j) {
      const float w = taps[i * K + j][lane];
#pragma unroll
      for (int xx = 0; xx < DW_T; ++xx) acc[xx] = fmaf(xr[xx + j], w, acc[xx]);
    }
  }
#pragma unroll
  for (int xx = 0; xx < DW_T; ++xx)
    if (xx < n_valid) out[static_cast<long long>(xx) * ld] = from_f<T>(acc[xx] + shift);
}
template <typename T, int K>
__global__ void __launch_bounds__(DW_THREADS)
dwconv_qkv_kernel(const T* __restrict__ x, int ldx, const float2* __restrict__ stats, int parts, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float inv_d, float eps, const float* __restrict__ wq, const float* __restrict__ bq,
                  T* __restrict__ q, int ldq, const float* __restrict__ wkv, const float* __restrict__ bkv, T* __restrict__ kv, int ldkv,
                  int H, int W, int C, int kv_stride, int Ho, int Wo, int kv_dy, int kv_dx, int tiles_x, int tiles_y, int groups,
                  long long M) {
  constexpr int TS = DW_T + K - 1, P = TS * TS, PAD = (K - 1) / 2;
  __shared__ float tile[P][DW_CG];
  __shared__ float mu_s[P], rs_s[P];
  __shared__ float tq[K * K][DW_CG], tkv[K * K][DW_CG];
  long long bid = blockIdx.x;
  const int tx = static_cast<int>(bid % tiles_x); bid /= tiles_x;
  const int ty = static_cast<int>(bid % tiles_y); bid /= tiles_y;
  const int g = static_cast<int>(bid % groups);
  const long long b = bid / groups;
  const int y0 = ty * DW_T, x0 = tx * DW_T, c0 = g * DW_CG;
  const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;
  const int c = c0 + lane;
  const bool cok = c < C;
  for (int i = threadIdx.x; i < K * K * DW_CG; i += DW_THREADS) {
    const int t = i / DW_CG, cc = c0 + i % DW_CG;
    tq[t][i % DW_CG] = cc < C ? __ldg(wq + static_cast<size_t>(t) * C + cc) : 0.f;
    tkv[t][i % DW_CG] = (wkv != nullptr && cc < C) ? __ldg(wkv + static_cast<size_t>(t) * C + cc) : 0.f;
  }
  if (stats != nullptr) {
    for (int p = threadIdx.x; p < P; p += DW_THREADS) {
      const int iy = y0 - PAD + p / TS, ix = x0 - PAD + p % TS;
      float m = 0.f, r = 0.f;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const long long pix = (b * H + iy) * W + ix;
        float s1 = 0.f, s2 = 0.f;
        for (int j = 0; j < parts; ++j) {
          const float2 v = __ldg(stats + j * M + pix);
          s1 += v.x;
          s2 += v.y;
        }
        m = s1 * inv_d;
        r = rsqrtf(fmaxf(s2 * inv_d - m * m, 0.f) + eps);
      }
      mu_s[p] = m;
      rs_s[p] = r;
    }
    __syncthreads();
  }
  const float ga = (stats != nullptr && cok) ? __ldg(gamma + c) : 1.f, be = (stats != nullptr && cok) ? __ldg(beta + c) : 0.f;
  for (int p = row; p < P; p += DW_T) {
    const int iy = y0 - PAD + p / TS, ix = x0 - PAD + p % TS;
    float v = 0.f;
    if (cok && iy >= 0 && iy < H && ix >= 0 && ix < W) {
      v = to_f(x[((b * H + iy) * W + ix) * ldx + c]);
      if (stats != nullptr) v = (v - mu_s[p]) * rs_s[p] * ga + be;
    }
    tile[p][lane] = v;
  }
  __syncthreads();
  const int oy = y0 + row;
  if (oy < H && cok) dw_conv_row<T, K>(tile, tq, bq[c], q + ((b * H + oy) * W + x0) * ldq + c, ldq, row, lane, W - x0);
  if (kv == nullptr) {
  } else if (kv_stride == 1) {
    if (oy < H && cok) dw_conv_row<T, K>(tile, tkv, bkv[c], kv + ((b * H + oy) * W + x0) * ldkv + c, ldkv, row, lane, W - x0);
  } else if (row < DW_T / 2 && cok) {                            // stride 2: outputs (y0/2 + row, x0/2 + xx), xx < DW_T/2
    const int r = y0 / 2 + row;
    if (r < Ho) {
      float acc[DW_T / 2];
#pragma unroll
      for (int xx = 0; xx < DW_T / 2; ++xx) acc[xx] = 0.f;
#pragma unroll
      for (int i = 0; i < K; ++i) {
        const int tr = (2 * row + kv_dy + i) * TS + kv_dx;
#pragma unroll
        for (int j = 0; j < K; ++j) {
          const float w = tkv[i * K + j][lane];
#pragma unroll
          for (int xx = 0; xx < DW_T / 2; ++xx) acc[xx] = fmaf(tile[tr + 2 * xx + j][lane], w, acc[xx]);
        }
      }
      const float sh = __ldg(bkv + c);
#pragma unroll
      for (int xx = 0; xx < DW_T / 2; ++xx)
        if (x0 / 2 + xx < Wo) kv[((b * Ho + r) * Wo + x0 / 2 + xx) * ldkv + c] = from_f<T>(acc[xx] + sh);
    }
  }
}

inline int grid_1d(long long total, int block = 256) {
  long long g = (total + block - 1) / block;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

long long launch_counter() { return g_launches.load(); }
void count_launch(int n) { g_launches.fetch_add(n); }

#define VB_LAUNCHED()          \
  do {                         \
    VB_CUDA(cudaGetLastError()); \
    count_launch();            \
  } while (0)

template <typename T>
void im2col(const float* img, T* out, int B, int H, int W, int C, int ph, int pw, int cls_row, int ldo, cudaStream_t s) {
  const int rows = cls_row + (H / ph) * (W / pw);
  const bool vec = ((pw * C) % 4 == 0) && (ldo % 4 == 0) && (reinterpret_cast<uintptr_t>(img) % 16 == 0) &&
                   (reinterpret_cast<uintptr_t>(out) % (4 * sizeof(T)) == 0);
  if (vec) {
    const long long total = static_cast<long long>(B) * rows * (ldo / 4);
    im2col_kernel<T, true><<<grid_1d(total), 256, 0, s>>>(img, out, B, H, W, C, ph, pw, cls_row, ldo);
  } else {
    const long long total = static_cast<long long>(B) * rows * ldo;
    im2col_kernel<T, false><<<grid_1d(total), 256, 0, s>>>(img, out, B, H, W, C, ph, pw, cls_row, ldo);
  }
  VB_LAUNCHED();
}

void softmax_rows_bf16(const float* S, int lds, __nv_bfloat16* P, int ldp, long long rows, int n, int npad, float scale_log2, cudaStream_t s) {
  VB_CHECK(n <= npad, "softmax_rows_bf16: n <= npad");
  if (npad <= SM_THREADS * SM_MAXE) softmax_rows_bf16_kernel<<<static_cast<unsigned>(rows), SM_THREADS, 0, s>>>(S, lds, P, ldp, n, npad, scale_log2);
  else softmax_rows_bf16_big_kernel<<<static_cast<unsigned>(rows), SM_THREADS, 0, s>>>(S, lds, P, ldp, n, npad, scale_log2);
  VB_LAUNCHED();
}

void transpose_rows_bf16(const __nv_bfloat16* in, int ldi, long long in_batch, __nv_bfloat16* out, int ldo, long long out_batch, int B,
                         int n, int npad, int cols, cudaStream_t s) {
  const unsigned grid = flat_blocks(static_cast<long long>((npad + 31) / 32) * ((cols + 31) / 32), B, "transpose_rows_bf16");
  transpose_rows_bf16_kernel<<<grid, dim3(32, 8), 0, s>>>(in, ldi, in_batch, out, ldo, out_batch, n, npad, cols);
  VB_LAUNCHED();
}

void pad_heads_f32(const float* W, float* Wp, int other, int groups, int heads, int dh, int dhp, int pad_rows, cudaStream_t s) {
  const long long total = static_cast<long long>(other) * groups * heads * dhp;
  pad_heads_kernel<<<grid_1d(total), 256, 0, s>>>(W, Wp, other, groups, heads, dh, dhp, pad_rows);
  VB_LAUNCHED();
}

template <typename T>
void build_embed_residual(T* R, const float* pos, const float* cls, const float* bias, int B, int rows, int dim, int has_cls,
                          cudaStream_t s) {
  const long long total = static_cast<long long>(B) * rows * dim;
  embed_residual_kernel<T><<<grid_1d(total), 256, 0, s>>>(R, pos, cls, bias, B, rows, dim, has_cls);
  VB_LAUNCHED();
}

template <typename T>
void layernorm(const T* x, int ldx, const float* gamma, const float* beta, T* out, int ldo, int M, int D, cudaStream_t s, int pad_to,
               float eps) {
  const int warps = 8;
  const int blocks = (M + warps - 1) / warps;
  const bool aligned = (pad_to <= D) && (D % 8 == 0) && (ldx % 8 == 0) && (ldo % 8 == 0) &&
                       (reinterpret_cast<uintptr_t>(x) % 16 == 0) && (reinterpret_cast<uintptr_t>(out) % 16 == 0) &&
                       (reinterpret_cast<uintptr_t>(gamma) % 16 == 0) && (reinterpret_cast<uintptr_t>(beta) % 16 == 0);
  if (aligned && D <= 8 * 32 * 2) {
    layernorm_kernel<T, 2><<<blocks, warps * 32, 0, s>>>(x, ldx, gamma, beta, out, ldo, M, D, eps);
  } else if (aligned && D <= 8 * 32 * 4) {
    layernorm_kernel<T, 4><<<blocks, warps * 32, 0, s>>>(x, ldx, gamma, beta, out, ldo, M, D, eps);
  } else {
    layernorm_generic_kernel<T><<<blocks, warps * 32, 0, s>>>(x, ldx, gamma, beta, out, ldo, M, D, pad_to, eps);
  }
  VB_LAUNCHED();
}

template <typename TA, typename TW, typename TO>
void gemm_simt(const TA* A, int lda, const TW* W, int wsk, int wsn, TO* out, int ldc, int M, int N, int K, const float* bias,
               const float* scale, const TO* res, int ldr, int act, cudaStream_t s, const DropoutEpi& drop) {
  VB_CHECK(drop.pos == DROP_NONE || act != ACT_SILU, "gemm_simt: no dropout instance with the SiLU epilogue");
  VB_CHECK(drop.pos != DROP_AFTER_RES || res != nullptr, "gemm_simt: dropout after the residual needs one");
  if (static_cast<long long>((N + 63) / 64) * ((M + 63) / 64) >= 2 * sm_count()) {
    const unsigned grid = flat_blocks((N + 63) / 64, (M + 63) / 64, "gemm_simt");
    if (act == ACT_SILU) gemm_simt_kernel<TA, TW, TO, 4, true><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else if (drop.pos == DROP_BEFORE_RES) gemm_simt_kernel<TA, TW, TO, 4, false, DROP_BEFORE_RES><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else if (drop.pos == DROP_AFTER_RES) gemm_simt_kernel<TA, TW, TO, 4, false, DROP_AFTER_RES><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else gemm_simt_kernel<TA, TW, TO, 4><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
  } else {
    const unsigned grid = flat_blocks((N + 63) / 64, (M + 15) / 16, "gemm_simt");
    if (act == ACT_SILU) gemm_simt_kernel<TA, TW, TO, 1, true><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else if (drop.pos == DROP_BEFORE_RES) gemm_simt_kernel<TA, TW, TO, 1, false, DROP_BEFORE_RES><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else if (drop.pos == DROP_AFTER_RES) gemm_simt_kernel<TA, TW, TO, 1, false, DROP_AFTER_RES><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
    else gemm_simt_kernel<TA, TW, TO, 1><<<grid, 256, 0, s>>>(A, lda, W, wsk, wsn, out, ldc, M, N, K, bias, scale, res, ldr, act, drop);
  }
  VB_LAUNCHED();
}

// The draw counter's advance after a training-mode forward's last site (one thread; the launches after it wait for it)
__global__ void dropout_advance_kernel(unsigned long long* state) { state[1] = static_cast<uint32_t>(state[1] + 1); }
void dropout_advance(unsigned long long* state, cudaStream_t s) {
  dropout_advance_kernel<<<1, 1, 0, s>>>(state);
  VB_LAUNCHED();
}

// keep[m, n] of site `site` at draw d (vb_op_dropout_mask), by the function the epilogues use
__global__ void dropout_mask_kernel(unsigned long long seed, uint32_t d, uint32_t site, int M, int N, float rate, uint8_t* __restrict__ keep) {
  const long long total = static_cast<long long>(M) * N;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint32_t m = static_cast<uint32_t>(i / N), n = static_cast<uint32_t>(i % N);
    keep[i] = dropout_keep_at(seed, d, site, m, n, rate) ? 1 : 0;
  }
}
void dropout_mask(unsigned long long seed, uint32_t d, uint32_t site, int M, int N, float rate, uint8_t* keep, cudaStream_t s) {
  dropout_mask_kernel<<<grid_1d(static_cast<long long>(M) * N), 256, 0, s>>>(seed, d, site, M, N, rate, keep);
  VB_LAUNCHED();
}

template <typename T>
void attn_scores(const T* q, int ldq, const T* k, int ldk, float* S, int B, int heads, int nq, int nk, int dh, float scale,
                 cudaStream_t s) {
  const long long blocks = static_cast<long long>((nk + 31) / 32) * ((nq + 31) / 32) * B * heads;
  VB_CHECK(blocks <= 0x7fffffffLL, "attention scores: grid of " + std::to_string(blocks) + " blocks exceeds 2^31 - 1");
  attn_scores_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(q, ldq, k, ldk, S, heads, nq, nk, dh, scale);
  VB_LAUNCHED();
}

void attn_head_mix(float* S, const float* Wmix, const float* gamma, const float* beta, int B, int heads, int nq, int nk,
                   cudaStream_t s) {
  VB_CHECK(heads <= MAX_HEADS, "attention head mixing supports at most 32 heads");
  const long long plane = static_cast<long long>(nq) * nk;
  attn_head_mix_kernel<<<grid_1d(B * plane, 128), 128, 0, s>>>(S, Wmix, gamma, beta, B, heads, plane);
  VB_LAUNCHED();
}

void attn_softmax(float* S, long long rows, int nk, cudaStream_t s) {
  const int warps = 8;
  attn_softmax_kernel<<<static_cast<unsigned>((rows + warps - 1) / warps), warps * 32, 0, s>>>(S, rows, nk);
  VB_LAUNCHED();
}

template <typename T>
void attn_pv(const float* S, const T* v, int ldv, T* out, int ldo, int B, int heads, int nq, int nk, int dh, cudaStream_t s, int gelu_out) {
  const long long blocks = static_cast<long long>((dh + 31) / 32) * ((nq + 31) / 32) * B * heads;
  VB_CHECK(blocks <= 0x7fffffffLL, "attention PV: grid of " + std::to_string(blocks) + " blocks exceeds 2^31 - 1");
  attn_pv_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(S, v, ldv, out, ldo, heads, nq, nk, dh, gelu_out);
  VB_LAUNCHED();
}

void attn_pos_bias(float* S, const PosBias& pb, int B, int heads, int nq, int nk, cudaStream_t s) {
  const long long total = static_cast<long long>(B) * heads * nq * nk;
  if (pb.r2l_ws > 0) {
    VB_CHECK(nq == 1 + pb.r2l_h * pb.r2l_w && nk == nq && pb.r2l_h <= pb.r2l_ws && pb.r2l_w <= pb.r2l_ws,
             "attention: the R2L window table needs nq == nk == 1 + wh * ww with wh, ww <= window_size");
    attn_r2l_bias_kernel<<<grid_1d(total, 256), 256, 0, s>>>(S, pb.table, heads, nk, pb.r2l_w, pb.r2l_ws, total);
    VB_LAUNCHED();
    return;
  }
  if (pb.wsz > 0) {
    VB_CHECK(nq == pb.wsz * pb.wsz && nk == nq, "attention: the window table needs nq == nk == wsz^2");
    attn_window_bias_kernel<<<grid_1d(total, 256), 256, 0, s>>>(S, pb.table, nk, pb.wsz, total);
    VB_LAUNCHED();
    return;
  }
  attn_pos_bias_kernel<<<grid_1d(total, 256), 256, 0, s>>>(S, pb.table, heads, nq, nk, pb.fmap, pb.step, total);
  VB_LAUNCHED();
}

template <typename T>
void gather_grid(const T* in, int ldi, T* out, int ldo, int B, int H, int W, int C, int step, cudaStream_t s) {
  const int oh = (H + step - 1) / step, ow = (W + step - 1) / step;
  const int vec = (C % (16 / sizeof(T)) == 0 && ldi % (16 / sizeof(T)) == 0 && ldo % (16 / sizeof(T)) == 0 &&
                   (reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) % 16 == 0) ? 16 / sizeof(T) : 1;
  const long long total = static_cast<long long>(B) * oh * ow * (C / vec);
  gather_grid_kernel<T><<<grid_1d(total, 256), 256, 0, s>>>(in, ldi, out, ldo, H, W, C, step, oh, ow, total, vec);
  VB_LAUNCHED();
}

template <typename T>
void pool_layernorm(const T* X, int n, int ldx, const float* gamma, const float* beta, float* out, int B, int D, int mean_pool,
                    cudaStream_t s) {
  pool_layernorm_kernel<T><<<B, 256, D * sizeof(float), s>>>(X, n, ldx, gamma, beta, out, D, mean_pool);
  VB_LAUNCHED();
}

template <typename T>
void copy_tokens(const T* src, int src_rows, int soff, T* dst, int dst_rows, int doff, int count, int B, int D, cudaStream_t s) {
  const long long total = static_cast<long long>(B) * count * D;
  if (total == 0) return;
  copy_tokens_kernel<T><<<grid_1d(total), 256, 0, s>>>(src, src_rows, soff, dst, dst_rows, doff, count, B, D);
  VB_LAUNCHED();
}

template <typename T>
void broadcast_row(const float* vec, T* dst, int dst_rows, int B, int D, cudaStream_t s) {
  broadcast_row_kernel<T><<<grid_1d(static_cast<long long>(B) * D), 256, 0, s>>>(vec, dst, dst_rows, B, D);
  VB_LAUNCHED();
}

template <typename T>
void broadcast_rows(const float* vec, T* dst, int B, int nt, int D, cudaStream_t s) {
  broadcast_rows_kernel<T><<<grid_1d(static_cast<long long>(B) * nt * D), 256, 0, s>>>(vec, dst, B, nt, D);
  VB_LAUNCHED();
}

template <typename TI, typename TO>
void unfold_same(const TI* in, TO* out, int B, int H, int W, int C, int k, int stride, int cls_row, int ldo, cudaStream_t s, int ldi,
                 const UnfoldMode* mode) {
  if (ldi <= 0) ldi = C;
  const bool valid = mode != nullptr && mode->valid;
  const int oh = valid ? (H - k) / stride + 1 : (H + stride - 1) / stride, ow = valid ? (W - k) / stride + 1 : (W + stride - 1) / stride;
  VB_CHECK(!valid || (H >= k && W >= k), "unfold_same: a VALID window larger than the map");
  const int ph = !valid && (oh - 1) * stride + k > H ? (oh - 1) * stride + k - H : 0;
  const int pw = !valid && (ow - 1) * stride + k > W ? (ow - 1) * stride + k - W : 0;
  const long long rows_total = static_cast<long long>(B) * (cls_row + oh * ow);
  VB_CHECK(rows_total > 0 && rows_total < (1ll << 31), "unfold_same: B * rows out of range");
  const float2* stats = mode != nullptr ? reinterpret_cast<const float2*>(mode->stats) : nullptr;
  VB_CHECK(stats == nullptr || (mode->parts > 0 && mode->d > 0 && mode->gamma != nullptr && mode->beta != nullptr),
           "unfold_same: LayerNorm statistics without their width / gamma / beta");
  const int threads = C >= 128 ? 160 : (C >= 32 ? 64 : (k * k * C >= 128 ? 160 : 64));
  unfold_same_kernel<TI, TO><<<static_cast<unsigned>(rows_total), threads, 0, s>>>(
      in, ldi, out, B, H, W, C, k, stride, oh, ow, ph / 2, pw / 2, cls_row, ldo, stats, stats ? mode->parts : 0,
      stats ? 1.0f / static_cast<float>(mode->d) : 0.f, stats ? mode->eps : 0.f, stats ? mode->gamma : nullptr, stats ? mode->beta : nullptr,
      mode != nullptr && mode->gelu ? 1 : 0);
  VB_LAUNCHED();
}

template <typename T>
void window_rows(const T* in, int ldi, T* out, int ldo, int cols, const Window& win, long long rows, bool to_window, cudaStream_t s) {
  const int n = win.p * win.width();
  VB_CHECK(n > 0 && rows % n == 0 && rows < (1ll << 31), "window_rows: rows must be whole windows, fewer than 2^31");
  if (rows == 0) return;
  window_rows_kernel<T><<<static_cast<unsigned>(rows), cols >= 256 ? 256 : 128, 0, s>>>(in, ldi, out, ldo, cols, win, n, to_window);
  VB_LAUNCHED();
}

template <typename T>
void r2l_rows(const T* in, int ldi, T* out, int ldo, int cols, const Window& win, long long reg_row0, bool to_window, cudaStream_t s) {
  const int n = 1 + win.p * win.width();
  const long long rows = static_cast<long long>(win.count) * n;
  VB_CHECK(win.count >= 0 && rows < (1ll << 31), "r2l_rows: fewer than 2^31 window-major rows");
  if (rows == 0) return;
  r2l_rows_kernel<T><<<static_cast<unsigned>(rows), cols >= 256 ? 256 : 128, 0, s>>>(in, ldi, out, ldo, cols, win, n, reg_row0, to_window);
  VB_LAUNCHED();
}

template <typename T>
void maxpool_relu_same(const T* in, T* out, int B, int H, int W, int C, int k, int stride, const float* pos, int rows, cudaStream_t s) {
  const int oh = (H + stride - 1) / stride, ow = (W + stride - 1) / stride;
  VB_CHECK(rows >= oh * ow, "maxpool_relu_same: fewer output rows than pooled positions");
  const int ph = std::max((oh - 1) * stride + k - H, 0), pw = std::max((ow - 1) * stride + k - W, 0);
  const long long total = static_cast<long long>(B) * rows * C;
  maxpool_relu_same_kernel<T><<<grid_1d(total), 256, 0, s>>>(in, out, H, W, C, k, stride, oh, ow, ph / 2, pw / 2, pos, rows, total);
  VB_LAUNCHED();
}

template <typename T>
void nest_pool(const T* in, int ldi, const NestPoolLn* ln, int B, int H, int W, int C, bool pool, const float* pos, int bh, int bw,
               T* out, int ldo, float* stats_out, cudaStream_t s) {
  const int oh = pool ? (H + 1) / 2 : H, ow = pool ? (W + 1) / 2 : W;
  const int ph = pool ? std::max((oh - 1) * 2 + 3 - H, 0) : 0, pw = pool ? std::max((ow - 1) * 2 + 3 - W, 0) : 0;
  const long long pixels = static_cast<long long>(B) * oh * ow;
  VB_CHECK(pixels > 0 && (pixels + NEST_POOL_WARPS - 1) / NEST_POOL_WARPS < (1ll << 31) && C <= ldo && C <= ldi,
           "nest_pool: bad shape");
  VB_CHECK(stats_out == nullptr || ldo % 64 == 0, "nest_pool: row statistics need a multiple of 64 columns");
  VB_CHECK(pos == nullptr || (bh > 0 && bw > 0 && oh % bh == 0 && ow % bw == 0), "nest_pool: the map is not whole blocks");
  VB_CHECK(ln == nullptr || (ln->stats != nullptr && ln->parts > 0 && ln->d > 0 && ln->gamma != nullptr && ln->beta != nullptr),
           "nest_pool: LayerNorm statistics without their width / gamma / beta");
  VB_CHECK(pool || ln == nullptr, "nest_pool: the LayerNorm on load is for the pooling form");
  const unsigned grid = static_cast<unsigned>((pixels + NEST_POOL_WARPS - 1) / NEST_POOL_WARPS);
  nest_pool_kernel<T><<<grid, NEST_POOL_WARPS * 32, 0, s>>>(
      in, ldi, ln ? reinterpret_cast<const float2*>(ln->stats) : nullptr, ln ? ln->parts : 0, ln ? 1.0f / static_cast<float>(ln->d) : 0.f,
      ln ? ln->eps : 0.f, ln ? ln->gamma : nullptr, ln ? ln->beta : nullptr, C, H, W, pool ? 1 : 0, oh, ow, ph / 2, pw / 2, pos, bh, bw,
      out, ldo, reinterpret_cast<float2*>(stats_out), pixels);
  VB_LAUNCHED();
}

template <typename T>
void seq_pool(const T* X, int n, int D, const float* gamma, const float* beta, const float* pw, const float* pb, float* z, int B,
              cudaStream_t s) {
  VB_CHECK(D > 0 && D <= 1024 && n > 0, "seq_pool: needs 0 < dim <= 1024 and at least one token");
  const size_t smem = (static_cast<size_t>(SEQ_POOL_WARPS) * D + 2 * SEQ_POOL_WARPS) * sizeof(float);
  const dim3 block(SEQ_POOL_WARPS * 32);
  if (D <= 128) seq_pool_kernel<T, 4><<<B, block, smem, s>>>(X, n, D, gamma, beta, pw, pb, z);
  else if (D <= 256) seq_pool_kernel<T, 8><<<B, block, smem, s>>>(X, n, D, gamma, beta, pw, pb, z);
  else if (D <= 512) seq_pool_kernel<T, 16><<<B, block, smem, s>>>(X, n, D, gamma, beta, pw, pb, z);
  else seq_pool_kernel<T, 32><<<B, block, smem, s>>>(X, n, D, gamma, beta, pw, pb, z);
  VB_LAUNCHED();
}

template <typename TI, typename TO>
void convert_rows(const TI* in, int ldi, TO* out, int ldo, long long rows, int cols, cudaStream_t s) {
  if (rows == 0) return;
  convert_rows_kernel<TI, TO><<<grid_1d(rows * ldo), 256, 0, s>>>(in, ldi, out, ldo, rows, cols);
  VB_LAUNCHED();
}

template <typename TI, typename TO>
void convert(const TI* in, TO* out, long long count, cudaStream_t s) {
  if (count == 0) return;
  convert_kernel<TI, TO><<<grid_1d(count), 256, 0, s>>>(in, out, count);
  VB_LAUNCHED();
}

void add_inplace_f32(float* a, const float* b, long long count, cudaStream_t s) {
  add_inplace_kernel<<<grid_1d(count), 256, 0, s>>>(a, b, count);
  VB_LAUNCHED();
}

void pack_weight_bf16(const float* W, __nv_bfloat16* Wt, int K, int N, int ldw, cudaStream_t s, const float* row_scale) {
  dim3 grid((N + 31) / 32, (ldw + 31) / 32);
  pack_weight_kernel<<<grid, dim3(32, 8), 0, s>>>(W, Wt, K, N, ldw, row_scale);
  VB_LAUNCHED();
}

void ln_fold_consts(const float* W, const __nv_bfloat16* Wt, int ldw, const float* beta, const float* bias, float* c1, float* c2,
                    int K, int N, cudaStream_t s) {
  ln_fold_consts_kernel<<<(N + 7) / 8, 256, 0, s>>>(W, Wt, ldw, beta, bias, c1, c2, K, N);
  VB_LAUNCHED();
}

void row_stats_bf16(const __nv_bfloat16* X, int ldx, float* stats, int M, int D, cudaStream_t s, long long pitch) {
  VB_CHECK(D % 64 == 0 && ldx % 8 == 0, "row_stats_bf16: D must be a multiple of 64");
  VB_CHECK(pitch == 0 || pitch >= M, "row_stats_bf16: the statistics pitch is below M");
  const int parts = D / 64;
  const long long total = static_cast<long long>(M) * parts;
  row_stats_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(X, ldx, reinterpret_cast<float2*>(stats), M, parts,
                                                                             pitch > 0 ? pitch : M);
  VB_LAUNCHED();
}

template <typename T>
void dwconv_qkv(const T* x, int ldx, const float* stats, const float* gamma, const float* beta, int D, float eps, const float* wq,
                const float* bq, T* q, int ldq, const float* wkv, const float* bkv, T* kv, int ldkv, int B, int H, int W, int C, int k,
                int kv_stride, cudaStream_t s) {
  VB_CHECK(k >= 1 && k <= DW_MAXK && (kv_stride == 1 || kv_stride == 2), "dwconv_qkv: kernel size 1..7 and stride 1 or 2 only");
  VB_CHECK(stats == nullptr || C % 64 == 0, "dwconv_qkv: LayerNorm statistics need a channel width that is a multiple of 64");
  const int Ho = (H + kv_stride - 1) / kv_stride, Wo = (W + kv_stride - 1) / kv_stride;
  const int pad = (k - 1) / 2;
  const int kv_dy = pad - std::max((Ho - 1) * kv_stride + k - H, 0) / 2, kv_dx = pad - std::max((Wo - 1) * kv_stride + k - W, 0) / 2;
  VB_CHECK(kv_dy >= 0 && kv_dy <= 1 && kv_dx >= 0 && kv_dx <= 1, "dwconv_qkv: internal: k|v window outside the tile halo");
  const int tiles_x = (W + DW_T - 1) / DW_T, tiles_y = (H + DW_T - 1) / DW_T, groups = (C + DW_CG - 1) / DW_CG;
  const unsigned grid = flat_blocks(static_cast<long long>(tiles_x) * tiles_y * groups, B, "dwconv_qkv");
  const long long M = static_cast<long long>(B) * H * W;
  const float2* st = reinterpret_cast<const float2*>(stats);
#define VB_DW_CASE(KS)                                                                                                        \
  case KS:                                                                                                                    \
    dwconv_qkv_kernel<T, KS><<<grid, DW_THREADS, 0, s>>>(x, ldx, st, C / 64, gamma, beta, 1.0f / static_cast<float>(D), eps, wq, bq, \
                                                         q, ldq, wkv, bkv, kv, ldkv, H, W, C, kv_stride, Ho, Wo, kv_dy, kv_dx,     \
                                                         tiles_x, tiles_y, groups, M);                                        \
    break;
  switch (k) { VB_DW_CASE(1) VB_DW_CASE(2) VB_DW_CASE(3) VB_DW_CASE(4) VB_DW_CASE(5) VB_DW_CASE(6) VB_DW_CASE(7) }
#undef VB_DW_CASE
  VB_LAUNCHED();
}

// ------------------------------------------------------------------------------------------ MV2 depthwise convolution
namespace {
// V channels of one pixel: 8 bf16 in one 16-byte access, or one float (the fp32 engine's unpadded widths); load(const float*)
// reads V fp32 taps or shifts (two 16-byte accesses for V = 8: Cp and c0 are multiples of 8, w and shift 16-byte aligned)
template <typename T, int V> struct DwVec;
template <> struct DwVec<__nv_bfloat16, 8> {
  static __device__ __forceinline__ void load(const float* p, float (&v)[8]) {   // 8 fp32 taps / shifts, 32-byte aligned
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float (&v)[8]) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float (&v)[8]) {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};
template <> struct DwVec<float, 1> {
  static __device__ __forceinline__ void load(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
  static __device__ __forceinline__ void store(float* p, const float (&v)[1]) { *p = v[0]; }
};

// One thread per (output pixel, V channels), channel groups fastest so that a warp reads whole pixel rows.  Taps [9][Cp] and the
// shift [Cp] carry the folded BatchNorm and are zero on the pad channels; groups wholly past C store zeros without reading.
template <typename T, int V>
__global__ void __launch_bounds__(256)
dwconv_bn_act_kernel(const T* __restrict__ x, int ldx, const float* __restrict__ w, const float* __restrict__ shift, T* __restrict__ out,
                     int ldo, int H, int W, int C, int Cp, int stride, int Ho, int Wo, int pt, int pl, long long total) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int G = Cp / V, g = static_cast<int>(idx % G), c0 = g * V;
  const long long pix = idx / G;
  const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>(pix / Wo % Ho);
  const long long b = pix / (static_cast<long long>(Wo) * Ho);
  float acc[V];
  if (c0 >= C) {
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = 0.f;
    DwVec<T, V>::store(out + pix * ldo + c0, acc);
    return;
  }
  DwVec<T, V>::load(shift + c0, acc);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * stride - pt + ky;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * stride - pl + kx;
      if (ix < 0 || ix >= W) continue;
      float xv[V];
      DwVec<T, V>::load(x + ((b * H + iy) * W + ix) * ldx + c0, xv);
      float tap[V];
      DwVec<T, V>::load(w + (ky * 3 + kx) * Cp + c0, tap);
#pragma unroll
      for (int v = 0; v < V; ++v) acc[v] = fmaf(xv[v], tap[v], acc[v]);
    }
  }
#pragma unroll
  for (int v = 0; v < V; ++v) acc[v] = silu(acc[v]);
  DwVec<T, V>::store(out + pix * ldo + c0, acc);
}
}  // namespace

template <typename T>
void dwconv_bn_act(const T* x, int ldx, const float* w, const float* shift, T* out, int ldo, int B, int H, int W, int C, int Cp, int stride,
                   cudaStream_t s) {
  constexpr int V = sizeof(T) == 2 ? 8 : 1;
  VB_CHECK(stride == 1 || stride == 2, "dwconv_bn_act: stride 1 or 2 only");
  VB_CHECK(C > 0 && Cp >= C && Cp % V == 0 && ldx >= Cp && ldo >= Cp, "dwconv_bn_act: bad channel widths");
  VB_CHECK(V == 1 || (ldx % 8 == 0 && ldo % 8 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) |
                                                       reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(shift)) % 16) == 0),
           "dwconv_bn_act: bf16 rows need 16-byte aligned pitches and pointers");
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  const int pt = std::max((Ho - 1) * stride + 3 - H, 0) / 2, pl = std::max((Wo - 1) * stride + 3 - W, 0) / 2;   // TF SAME, smaller half first
  const long long total = static_cast<long long>(B) * Ho * Wo * (Cp / V);
  dwconv_bn_act_kernel<T, V><<<flat_blocks((total + 255) / 256, 1, "dwconv_bn_act"), 256, 0, s>>>(x, ldx, w, shift, out, ldo, H, W, C, Cp, stride,
                                                                                               Ho, Wo, pt, pl, total);
  VB_LAUNCHED();
}

// ------------------------------------------------------------------------------------------ instantiations
#define VB_INST_T(T)                                                                                                         \
  template void im2col<T>(const float*, T*, int, int, int, int, int, int, int, int, cudaStream_t);                          \
  template void build_embed_residual<T>(T*, const float*, const float*, const float*, int, int, int, int, cudaStream_t);    \
  template void layernorm<T>(const T*, int, const float*, const float*, T*, int, int, int, cudaStream_t, int, float);            \
  template void attn_scores<T>(const T*, int, const T*, int, float*, int, int, int, int, int, float, cudaStream_t);         \
  template void attn_pv<T>(const float*, const T*, int, T*, int, int, int, int, int, int, cudaStream_t, int);               \
  template void gather_grid<T>(const T*, int, T*, int, int, int, int, int, int, cudaStream_t);                              \
  template void pool_layernorm<T>(const T*, int, int, const float*, const float*, float*, int, int, int, cudaStream_t);     \
  template void copy_tokens<T>(const T*, int, int, T*, int, int, int, int, int, cudaStream_t);                              \
  template void broadcast_row<T>(const float*, T*, int, int, int, cudaStream_t);                                            \
  template void broadcast_rows<T>(const float*, T*, int, int, int, cudaStream_t);                                           \
  template void unfold_same<float, T>(const float*, T*, int, int, int, int, int, int, int, int, cudaStream_t, int, const UnfoldMode*); \
  template void window_rows<T>(const T*, int, T*, int, int, const Window&, long long, bool, cudaStream_t);                   \
  template void r2l_rows<T>(const T*, int, T*, int, int, const Window&, long long, bool, cudaStream_t);                      \
  template void convert_rows<float, T>(const float*, int, T*, int, long long, int, cudaStream_t);                           \
  template void maxpool_relu_same<T>(const T*, T*, int, int, int, int, int, int, const float*, int, cudaStream_t);         \
  template void nest_pool<T>(const T*, int, const NestPoolLn*, int, int, int, int, bool, const float*, int, int, T*, int, float*,   \
                             cudaStream_t);                                                                                  \
  template void seq_pool<T>(const T*, int, int, const float*, const float*, const float*, const float*, float*, int, cudaStream_t); \
  template void dwconv_qkv<T>(const T*, int, const float*, const float*, const float*, int, float, const float*, const float*, T*, int, \
                              const float*, const float*, T*, int, int, int, int, int, int, int, cudaStream_t);            \
  template void dwconv_bn_act<T>(const T*, int, const float*, const float*, T*, int, int, int, int, int, int, int, cudaStream_t);
VB_INST_T(float)
VB_INST_T(__nv_bfloat16)

template void gemm_simt<float, float, float>(const float*, int, const float*, int, int, float*, int, int, int, int, const float*,
                                             const float*, const float*, int, int, cudaStream_t, const DropoutEpi&);
template void gemm_simt<__nv_bfloat16, __nv_bfloat16, __nv_bfloat16>(const __nv_bfloat16*, int, const __nv_bfloat16*, int, int,
                                                                     __nv_bfloat16*, int, int, int, int, const float*,
                                                                     const float*, const __nv_bfloat16*, int, int, cudaStream_t,
                                                                     const DropoutEpi&);
template void unfold_same<__nv_bfloat16, __nv_bfloat16>(const __nv_bfloat16*, __nv_bfloat16*, int, int, int, int, int, int, int, int,
                                                        cudaStream_t, int, const UnfoldMode*);
template void convert_rows<__nv_bfloat16, float>(const __nv_bfloat16*, int, float*, int, long long, int, cudaStream_t);
template void convert<float, __nv_bfloat16>(const float*, __nv_bfloat16*, long long, cudaStream_t);
template void convert<__nv_bfloat16, float>(const __nv_bfloat16*, float*, long long, cudaStream_t);

}  // namespace vb
