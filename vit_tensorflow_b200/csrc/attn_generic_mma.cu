// Second-tier attention path for the bf16 engine: shapes / variants the fused kernel (attn_flash.cu) does not cover
// (DeepViT re-attention deepvit.py:83-84, CaiT talking heads cait.py:121-127, dim_head != 64, 1-row class-attention
// queries).  The score tensor is still materialised (fp32, like the reference does), but
//   * QK^T and PV run on the tensor cores through mma.sync.m16n8k16 (legacy HMMA path: simple, any dh % 16 == 0),
//   * pre-mix -> softmax -> post-mix / LayerNorm-over-heads is ONE kernel (one read + one write of the scores
//     instead of three full passes).
// (DeepViT re-attention and CaiT talking heads are served here: the head mix couples every head of a query row.)
#include "attention.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <map>
#include <set>
#include <tuple>
#include <vector>

namespace vb {
namespace {

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

constexpr int MAXDH = 128;
constexpr int PITCH = MAXDH + 8;   // bf16 elements; +8 keeps the fragment loads bank-conflict free

// Every kernel of this file takes its (tile, b * heads + h) item from a flat blockIdx.x, tile index fastest, so B * heads is
// not bounded by the 65 535 of gridDim.y / gridDim.z; flat_blocks() (common.h) checks the product against gridDim.x's 2^31 - 1.

// S[bh, i, j] = scale * sum_d q[b,i,h,d] k[b,j,h,d];  block: 64 x 64 tile, 4 warps x (16 rows x 64 cols)
__global__ void __launch_bounds__(128)
scores_mma_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k, int ldk, float* __restrict__ S,
                  int heads, int nq, int nk, int dh, float scale, int lds) {
  __shared__ __align__(16) __nv_bfloat16 Qs[64][PITCH];
  __shared__ __align__(16) __nv_bfloat16 Ks[64][PITCH];
  const int kt = (nk + 63) / 64, qt = (nq + 63) / 64;
  const int bh = blockIdx.x / (kt * qt), b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x / kt % qt) * 64, j0 = (blockIdx.x % kt) * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int vec = dh >> 3;                                        // 16-byte vectors per row
  for (int e = threadIdx.x; e < 64 * vec; e += 128) {
    const int r = e / vec, c = (e % vec) * 8;
    uint4 vq = make_uint4(0, 0, 0, 0), vk = make_uint4(0, 0, 0, 0);
    if (i0 + r < nq) vq = *reinterpret_cast<const uint4*>(q + (static_cast<size_t>(b) * nq + i0 + r) * ldq + h * dh + c);
    if (j0 + r < nk) vk = *reinterpret_cast<const uint4*>(k + (static_cast<size_t>(b) * nk + j0 + r) * ldk + h * dh + c);
    *reinterpret_cast<uint4*>(&Qs[r][c]) = vq;
    *reinterpret_cast<uint4*>(&Ks[r][c]) = vk;
  }
  __syncthreads();
  float acc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) { acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f; }
  const int ar = warp * 16 + (lane >> 2), ac = 2 * (lane & 3);
  for (int kk = 0; kk < dh; kk += 16) {
    uint32_t a[4];
    a[0] = *reinterpret_cast<const uint32_t*>(&Qs[ar][kk + ac]);
    a[1] = *reinterpret_cast<const uint32_t*>(&Qs[ar + 8][kk + ac]);
    a[2] = *reinterpret_cast<const uint32_t*>(&Qs[ar][kk + ac + 8]);
    a[3] = *reinterpret_cast<const uint32_t*>(&Qs[ar + 8][kk + ac + 8]);
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      uint32_t bb[2];
      bb[0] = *reinterpret_cast<const uint32_t*>(&Ks[n * 8 + (lane >> 2)][kk + ac]);
      bb[1] = *reinterpret_cast<const uint32_t*>(&Ks[n * 8 + (lane >> 2)][kk + ac + 8]);
      mma_bf16_16816(acc[n], a, bb);
    }
  }
  const int r0 = i0 + ar;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const int c0 = j0 + n * 8 + ac;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int r = r0 + half * 8;
      if (r < nq) {
        float* dst = S + (static_cast<size_t>(bh) * nq + r) * lds + c0;
        if (c0 < nk) dst[0] = acc[n][2 * half] * scale;
        if (c0 + 1 < nk) dst[1] = acc[n][2 * half + 1] * scale;
      }
    }
  }
}

// out[b,i,h,d] = sum_j P[bh,i,j] v[b,j,h,d];  block: 64 query rows x dh, keys in chunks of 64.
// SPLIT: P is fed as bf16 hi + bf16 lo (two MMAs, ~2^-17 relative): DeepViT's re-attention weights are LayerNorm
// outputs of magnitude up to 1/sqrt(eps) with mixed signs, and a single bf16 rounding of them costs ~1e-1 absolute
// on the output, outside the bf16 tolerance of the parity tests.
template <bool SPLIT>
__global__ void __launch_bounds__(128)
pv_mma_kernel(const float* __restrict__ P, const __nv_bfloat16* __restrict__ v, int ldv, __nv_bfloat16* __restrict__ out, int ldo,
              int heads, int nq, int nk, int dh, int gelu_out) {
  __shared__ __align__(16) __nv_bfloat16 Ps[64][64 + 8];
  __shared__ __align__(16) __nv_bfloat16 Pl[SPLIT ? 64 : 1][64 + 8];
  __shared__ __align__(16) __nv_bfloat16 Vt[MAXDH][64 + 8];        // transposed: Vt[d][j]
  const int qt = (nq + 63) / 64;
  const int bh = blockIdx.x / qt, b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x % qt) * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = dh >> 3;
  float acc[MAXDH / 8][4];
#pragma unroll
  for (int n = 0; n < MAXDH / 8; ++n) { acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f; }
  const int ar = warp * 16 + (lane >> 2), ac = 2 * (lane & 3);
  for (int j0 = 0; j0 < nk; j0 += 64) {
    for (int e = threadIdx.x; e < 64 * 64; e += 128) {
      const int r = e >> 6, c = e & 63;
      float p = 0.f;
      if (i0 + r < nq && j0 + c < nk) p = P[(static_cast<size_t>(bh) * nq + i0 + r) * nk + j0 + c];
      const __nv_bfloat16 hi = __float2bfloat16_rn(p);
      Ps[r][c] = hi;
      if (SPLIT) Pl[r][c] = __float2bfloat16_rn(p - __bfloat162float(hi));
    }
    for (int e = threadIdx.x; e < 64 * dh; e += 128) {
      const int r = e / dh, c = e % dh;
      __nv_bfloat16 x = __float2bfloat16_rn(0.f);
      if (j0 + r < nk) x = v[(static_cast<size_t>(b) * nk + j0 + r) * ldv + h * dh + c];
      Vt[c][r] = x;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 64; kk += 16) {
      uint32_t a[4];
      a[0] = *reinterpret_cast<const uint32_t*>(&Ps[ar][kk + ac]);
      a[1] = *reinterpret_cast<const uint32_t*>(&Ps[ar + 8][kk + ac]);
      a[2] = *reinterpret_cast<const uint32_t*>(&Ps[ar][kk + ac + 8]);
      a[3] = *reinterpret_cast<const uint32_t*>(&Ps[ar + 8][kk + ac + 8]);
      uint32_t al[4] = {0, 0, 0, 0};
      if (SPLIT) {
        al[0] = *reinterpret_cast<const uint32_t*>(&Pl[ar][kk + ac]);
        al[1] = *reinterpret_cast<const uint32_t*>(&Pl[ar + 8][kk + ac]);
        al[2] = *reinterpret_cast<const uint32_t*>(&Pl[ar][kk + ac + 8]);
        al[3] = *reinterpret_cast<const uint32_t*>(&Pl[ar + 8][kk + ac + 8]);
      }
#pragma unroll
      for (int n = 0; n < MAXDH / 8; ++n) {
        if (n < ntiles) {
          uint32_t bb[2];
          bb[0] = *reinterpret_cast<const uint32_t*>(&Vt[n * 8 + (lane >> 2)][kk + ac]);
          bb[1] = *reinterpret_cast<const uint32_t*>(&Vt[n * 8 + (lane >> 2)][kk + ac + 8]);
          mma_bf16_16816(acc[n], a, bb);
          if (SPLIT) mma_bf16_16816(acc[n], al, bb);
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int n = 0; n < MAXDH / 8; ++n) {
    if (n < ntiles) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = i0 + ar + half * 8;
        if (r < nq) {
          const float o0 = acc[n][2 * half], o1 = acc[n][2 * half + 1];
          __nv_bfloat162 o = gelu_out ? __floats2bfloat162_rn(gelu_exact(o0), gelu_exact(o1)) : __floats2bfloat162_rn(o0, o1);
          *reinterpret_cast<__nv_bfloat162*>(out + (static_cast<size_t>(b) * nq + r) * ldo + h * dh + n * 8 + ac) = o;
        }
      }
    }
  }
}

constexpr int MIX_MAX_HEADS = 32;
// One block per (query row i, batch b): all heads' score rows in shared memory.
//   variant 2: pre-softmax head mix -> softmax -> post-softmax head mix      (cait.py:123-125)
//   variant 1: softmax -> head mix -> LayerNorm across heads (eps 1e-3)       (deepvit.py:80-84)
//   variant 0: softmax
__global__ void __launch_bounds__(256)
mid_fused_kernel(float* __restrict__ S, const float* __restrict__ mix_a, const float* __restrict__ mix_b, const float* __restrict__ gamma,
                 const float* __restrict__ beta, int heads, int nq, int nk, int variant, const float* __restrict__ pos_tab, int fmap,
                 int step) {
  extern __shared__ float buf[];                    // [heads][nk] then 2 x [heads*heads] mix matrices
  float* Wa = buf + heads * nk;
  float* Wb = Wa + heads * heads;
  const int i = blockIdx.x % nq, b = blockIdx.x / nq;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const size_t plane = static_cast<size_t>(nq) * nk;
  float* base = S + (static_cast<size_t>(b) * heads * nq + i) * nk;        // head h row at base + h * plane
  for (int e = threadIdx.x; e < heads * heads; e += blockDim.x) {
    Wa[e] = mix_a ? mix_a[e] : 0.f;
    Wb[e] = mix_b ? mix_b[e] : 0.f;
  }
  const int nqs = (fmap + step - 1) / step;
  for (int h = 0; h < heads; ++h)
    for (int j = threadIdx.x; j < nk; j += blockDim.x)                 // + LeViT's relative-position bias (levit.py:131)
      buf[h * nk + j] = base[h * plane + j] + (pos_tab != nullptr ? pos_tab[h * fmap * fmap + pos_bias_index(i, j, fmap, step, nqs)] : 0.f);
  __syncthreads();
  auto mix = [&](const float* W, bool ln) {
    for (int j = threadIdx.x; j < nk; j += blockDim.x) {
      float x[MIX_MAX_HEADS], y[MIX_MAX_HEADS];
      for (int h = 0; h < heads; ++h) x[h] = buf[h * nk + j];
      for (int g = 0; g < heads; ++g) {
        float a = 0.f;
        for (int h = 0; h < heads; ++h) a = fmaf(x[h], W[h * heads + g], a);
        y[g] = a;
      }
      if (ln) {
        float mean = 0.f;
        for (int g = 0; g < heads; ++g) mean += y[g];
        mean /= heads;
        float var = 0.f;
        for (int g = 0; g < heads; ++g) { const float d = y[g] - mean; var += d * d; }
        const float rstd = rsqrtf(var / heads + 1e-3f);
        for (int g = 0; g < heads; ++g) y[g] = (y[g] - mean) * rstd * gamma[g] + beta[g];
      }
      for (int g = 0; g < heads; ++g) buf[g * nk + j] = y[g];
    }
  };
  if (variant == 2) { mix(Wa, false); __syncthreads(); }
  for (int h = warp; h < heads; h += nwarps) {      // softmax over keys, one warp per head row
    float* r = buf + h * nk;
    float mx = -INFINITY;
    for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, r[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < nk; j += 32) { const float e = expf(r[j] - mx); r[j] = e; sum += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    for (int j = lane; j < nk; j += 32) r[j] *= inv;
  }
  __syncthreads();
  if (variant == 1) { mix(Wa, true); __syncthreads(); }
  if (variant == 2) { mix(Wb, false); __syncthreads(); }
  for (int h = 0; h < heads; ++h)
    for (int j = threadIdx.x; j < nk; j += blockDim.x) base[h * plane + j] = buf[h * nk + j];
}


// Scores for the row path: one block per (64-query-row stripe, b, h).  The stripe's Q rows and ALL keys of the head go to
// shared memory once (cp.async), then each warp sweeps its 16 rows over the keys 8 at a time: ldmatrix fragments,
// dh/16 MMAs and two 8-byte stores per step.  Against the 64x64-tile kernel above this loads Q once instead of once
// per key tile and has one load/barrier phase per 64 x nk outputs instead of per 64 x 64.
__global__ void __launch_bounds__(128)
scores_stripe_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k, int ldk, float* __restrict__ S,
                     int heads, int nq, int nk, int dh, float scale, int lds) {
  extern __shared__ __align__(16) uint8_t sc_smem[];
  const int pitch = dh + 8;                                         // bf16; rows stay 16-byte aligned and conflict free
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(sc_smem);    // [64][pitch]
  __nv_bfloat16* Ks = Qs + 64 * pitch;                              // [nk8][pitch]
  const int qt = (nq + 63) / 64;
  const int bh = blockIdx.x / qt, b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x % qt) * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int vec = dh >> 3, nk8 = (nk + 7) & ~7;
  // (per-row 1-D bulk/TMA copies were tried here and in the PV kernel: 96-832 byte copies issued by one warp were
  //  1.5-1.8x slower than these per-thread 16-byte cp.async requests)
  for (int e = threadIdx.x; e < 64 * vec; e += 128) {
    const int r = e / vec, c = (e % vec) * 8;
    const int ri = min(i0 + r, nq - 1);                             // rows past nq: any valid row, never stored
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(Qs + r * pitch + c));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(q + (static_cast<size_t>(b) * nq + ri) * ldq + h * dh + c) : "memory");
  }
  for (int e = threadIdx.x; e < nk8 * vec; e += 128) {
    const int r = e / vec, c = (e % vec) * 8;
    const int rj = min(r, nk - 1);
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(Ks + r * pitch + c));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(k + (static_cast<size_t>(b) * nk + rj) * ldk + h * dh + c) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  uint32_t a[MAXDH / 16][4];
  const uint32_t qa = static_cast<uint32_t>(__cvta_generic_to_shared(Qs + (warp * 16 + (lane & 15)) * pitch + 8 * (lane >> 4)));
#pragma unroll
  for (int ks = 0; ks < MAXDH / 16; ++ks)
    if (ks * 16 < dh)
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                   : "=r"(a[ks][0]), "=r"(a[ks][1]), "=r"(a[ks][2]), "=r"(a[ks][3]) : "r"(qa + ks * 32));
  // B fragments of one 8-key tile, two 16-wide k steps per ldmatrix.x4: lanes 0-7 / 8-15 / 16-23 / 24-31 address the
  // tile's key rows at d offsets 0 / 8 / 16 / 24
  const uint32_t ka = static_cast<uint32_t>(__cvta_generic_to_shared(Ks + (lane & 7) * pitch + 8 * (lane >> 3)));
  const int fr = lane >> 2, fc = 2 * (lane & 3);
  const int r0 = i0 + warp * 16 + fr, r1 = r0 + 8;
  float* s0 = S + (static_cast<size_t>(bh) * nq + r0) * lds;
  float* s1 = S + (static_cast<size_t>(bh) * nq + r1) * lds;
  for (int nt = 0; nt < nk8 / 8; ++nt) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kp = 0; kp < MAXDH / 32; ++kp) {
      if (kp * 32 < dh) {
        uint32_t b0[2], b1[2];
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(b0[0]), "=r"(b0[1]), "=r"(b1[0]), "=r"(b1[1]) : "r"(ka + (nt * 8 * pitch + kp * 32) * 2));
        mma_bf16_16816(acc, a[2 * kp], b0);
        if (kp * 32 + 16 < dh) mma_bf16_16816(acc, a[2 * kp + 1], b1);
      }
    }
    const int c0 = nt * 8 + fc;                                     // c0 even, lds even: 8-byte aligned; columns < nkp exist
    if (r0 < nq) *reinterpret_cast<float2*>(s0 + c0) = make_float2(acc[0] * scale, acc[1] * scale);
    if (r1 < nq) *reinterpret_cast<float2*>(s1 + c0) = make_float2(acc[2] * scale, acc[3] * scale);
  }
}

// ------------------------------------------------------------------------------------------ row-per-warp middle + bf16 PV
// The cross-head steps (CaiT talking heads cait.py:123-125, DeepViT re-attention + LayerNorm over heads
// deepvit.py:83-84) need, for one (image, query row), the score rows of ALL heads.  One warp owns such a row set:
// lane l holds keys l, l+32, l+64, ... of every head in registers (JS slots x H heads), so the head mixes are
// register FMAs against weights that sit in the kernel-parameter constant bank, the softmax reductions are warp
// shuffles, and there is no shared memory and no block barrier.  Rows are read as fp32 scores and rewritten IN PLACE
// (row pitch `lds` floats >= 16-aligned nk) as bf16 probabilities: hi plane in the first nkp bf16 of the row, and for
// DeepViT the lo plane (p - hi) in the next nkp, so the PV product can feed them to mma.sync without conversion.

template <int H>
__device__ __forceinline__ float tree_sum(const float (&v)[H]) {           // pairwise: depth log2(H) instead of H
  float t[H];
#pragma unroll
  for (int g = 0; g < H; ++g) t[g] = v[g];
#pragma unroll
  for (int w = H / 2; w > 0; w >>= 1)
#pragma unroll
    for (int g = 0; g < w; ++g) t[g] += t[g + w];
  return t[0];
}

// WPR = warps per row: with 16 heads one warp would need 7 x 16 score registers (255 registers, 8 warps per SM), so two
// warps split the key slots (slot ts = WPR * t + w) and exchange their per-head (max, sum) once through shared memory.
template <int H, int JS, int VARIANT, int WPR>
__global__ void __launch_bounds__(256)
mid_rows_kernel(float* __restrict__ S, const __grid_constant__ MixParams P, int nq, int nk, int lds, int nkp, long long rows) {
  constexpr int RPB = 8 / WPR;                                                            // rows per block
  __shared__ float2 stat[WPR > 1 ? RPB : 1][WPR][H];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int w = warp % WPR, rl = warp / WPR;
  const long long row_raw = static_cast<long long>(blockIdx.x) * RPB + rl;                // (b, i)
  const bool live = row_raw < rows;
  const long long row = live ? row_raw : rows - 1;                                        // dead warps shadow a valid row, no stores
  const long long b = row / nq;
  const int i = static_cast<int>(row % nq);
  float* base = S + (b * H * nq + i) * lds;                                               // head h at + h * nq * lds
  const size_t plane = static_cast<size_t>(nq) * lds;
  float x[JS][H];                                                                         // key lane + 32 (WPR t + w) of every head
#pragma unroll
  for (int t = 0; t < JS; ++t) {
    const int j = lane + 32 * (WPR * t + w);
#pragma unroll
    for (int h = 0; h < H; ++h) x[t][h] = j < nk ? base[h * plane + j] : 0.f;
  }
  auto mix = [&](float (&v)[H], const float* W) {                                          // v[g] <- sum_h v[h] W[h][g]
    float y[H];
#pragma unroll
    for (int g = 0; g < H; ++g) y[g] = 0.f;
#pragma unroll
    for (int h = 0; h < H; ++h)
#pragma unroll
      for (int g = 0; g < H; ++g) y[g] = fmaf(v[h], W[h * H + g], y[g]);
#pragma unroll
    for (int g = 0; g < H; ++g) v[g] = y[g];
  };
  if (VARIANT == 2) {
#pragma unroll
    for (int t = 0; t < JS; ++t) mix(x[t], P.wa);
  }
  // softmax over the keys, per head: this warp's (max, sum of exp relative to it), merged across the row's warps
  float fac[H];
#pragma unroll
  for (int h = 0; h < H; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < JS; ++t)
      if (lane + 32 * (WPR * t + w) < nk) mx = fmaxf(mx, x[t][h]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < JS; ++t) {
      const float ex = (lane + 32 * (WPR * t + w) < nk) ? __expf(x[t][h] - mx) : 0.f;     // a warp without valid keys: mx = -inf, all 0
      x[t][h] = ex;
      sum += ex;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (WPR == 1) fac[h] = 1.0f / sum;
    else {
      if (lane == 0) stat[rl][w][h] = make_float2(mx, sum);
      fac[h] = mx;
    }
  }
  if (WPR > 1) {
    __syncthreads();
#pragma unroll
    for (int h = 0; h < H; ++h) {
      float m = -INFINITY;
#pragma unroll
      for (int u = 0; u < WPR; ++u) m = fmaxf(m, stat[rl][u][h].x);
      float l = 0.f;
#pragma unroll
      for (int u = 0; u < WPR; ++u) l += stat[rl][u][h].y * __expf(stat[rl][u][h].x - m);
      fac[h] = __expf(fac[h] - m) / l;                                                     // exp(x - m_w) * fac = exp(x - m) / l
    }
  }
#pragma unroll
  for (int t = 0; t < JS; ++t) {
#pragma unroll
    for (int h = 0; h < H; ++h) x[t][h] *= fac[h];
    if (VARIANT == 2) mix(x[t], P.wb);
    if (VARIANT == 1) {
      mix(x[t], P.wa);
      const float mean = tree_sum<H>(x[t]) * (1.0f / H);
      float d2[H];
#pragma unroll
      for (int g = 0; g < H; ++g) { x[t][g] -= mean; d2[g] = x[t][g] * x[t][g]; }
      const float rstd = rsqrtf(tree_sum<H>(d2) * (1.0f / H) + 1e-3f);
#pragma unroll
      for (int g = 0; g < H; ++g) x[t][g] = fmaf(x[t][g] * rstd, P.gamma[g], P.beta[g]);
    }
  }
  // every warp of the row has read everything it needs from these rows (block barrier above, or the single warp's own
  // program order): rewrite them as bf16 (hi | lo planes), zero padded to nkp
  if (WPR > 1) __syncthreads(); else __syncwarp();
  if (!live) return;
#pragma unroll
  for (int t = 0; t < JS; ++t) {
    const int j = lane + 32 * (WPR * t + w);
    if (j < nkp) {
#pragma unroll
      for (int h = 0; h < H; ++h) {
        const float p = j < nk ? x[t][h] : 0.f;
        const __nv_bfloat16 hi = __float2bfloat16_rn(p);
        __nv_bfloat16* prow = reinterpret_cast<__nv_bfloat16*>(base + h * plane);
        prow[j] = hi;
        if (VARIANT == 1) prow[nkp + j] = __float2bfloat16_rn(p - __bfloat162float(hi));
      }
    }
  }
}

// out[b,i,h,d] = sum_j P[bh,i,j] v[b,j,h,d] with P in the bf16 row format written by mid_rows_kernel.
// Block: 64 query rows of one (b, h), 4 warps x 16 rows; keys in chunks of 64 through a two-stage cp.async ring;
// A fragments by ldmatrix, B fragments by ldmatrix.trans from the row-major V tile.
template <bool SPLIT>
__global__ void __launch_bounds__(128)
pv_rows_kernel(const float* __restrict__ S, int lds, int nkp, const __nv_bfloat16* __restrict__ v, int ldv, __nv_bfloat16* __restrict__ out,
               int ldo, int heads, int nq, int nk, int dh) {
  constexpr int PP = 64 + 8;                                        // P tile pitch (bf16)
  constexpr int VP = MAXDH + 8;                                     // V tile pitch (bf16)
  extern __shared__ __align__(16) uint8_t pv_smem[];
  // per stage: P hi [64][PP], (P lo [64][PP]), V [64][VP]
  constexpr int P_ELEMS = 64 * PP, V_ELEMS = 64 * VP;
  constexpr int STAGE_ELEMS = (SPLIT ? 2 : 1) * P_ELEMS + V_ELEMS;
  __nv_bfloat16* sm = reinterpret_cast<__nv_bfloat16*>(pv_smem);
  const int qt = (nq + 63) / 64;
  const int bh = blockIdx.x / qt, b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x % qt) * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = dh >> 3, vec = dh >> 3;
  const int nchunks = (nk + 63) / 64;
  auto stage = [&](int c) {
    if (c < nchunks) {
      __nv_bfloat16* st = sm + (c & 1) * STAGE_ELEMS;
      const int j0 = c * 64;
      for (int e = threadIdx.x; e < 64 * 8; e += 128) {             // P: 64 rows x 8 x 16 bytes (x2 planes)
        const int r = e >> 3, cc = (e & 7) * 8;
        const int ri = min(i0 + r, nq - 1);                         // rows past nq: any valid row, results discarded
        const __nv_bfloat16* prow = reinterpret_cast<const __nv_bfloat16*>(S + (static_cast<size_t>(bh) * nq + ri) * lds);
        const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(st + r * PP + cc));
        if (j0 + cc < nkp) {
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(prow + j0 + cc) : "memory");
          if (SPLIT) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + P_ELEMS * 2), "l"(prow + nkp + j0 + cc) : "memory");
        } else {
          *reinterpret_cast<uint4*>(st + r * PP + cc) = make_uint4(0, 0, 0, 0);
          if (SPLIT) *reinterpret_cast<uint4*>(st + P_ELEMS + r * PP + cc) = make_uint4(0, 0, 0, 0);
        }
      }
      __nv_bfloat16* vs = st + (SPLIT ? 2 : 1) * P_ELEMS;
      for (int e = threadIdx.x; e < 64 * vec; e += 128) {
        const int r = e / vec, cc = (e % vec) * 8;
        if (j0 + r < nk) {
          const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(vs + r * VP + cc));
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(v + (static_cast<size_t>(b) * nk + j0 + r) * ldv + h * dh + cc) : "memory");
        } else {
          *reinterpret_cast<uint4*>(vs + r * VP + cc) = make_uint4(0, 0, 0, 0);
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  float acc[MAXDH / 8][4];
#pragma unroll
  for (int n = 0; n < MAXDH / 8; ++n) { acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f; }
  stage(0);
  for (int c = 0; c < nchunks; ++c) {
    stage(c + 1);
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    const __nv_bfloat16* st = sm + (c & 1) * STAGE_ELEMS;
    const __nv_bfloat16* vs = st + (SPLIT ? 2 : 1) * P_ELEMS;
    const uint32_t pa = static_cast<uint32_t>(__cvta_generic_to_shared(st + (warp * 16 + (lane & 15)) * PP + 8 * (lane >> 4)));
    const uint32_t va = static_cast<uint32_t>(__cvta_generic_to_shared(vs + (lane & 15) * VP));
#pragma unroll
    for (int kk = 0; kk < 64; kk += 16) {
      uint32_t a[4], al[4] = {0, 0, 0, 0};
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                   : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(pa + kk * 2));
      if (SPLIT)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(al[0]), "=r"(al[1]), "=r"(al[2]), "=r"(al[3]) : "r"(pa + P_ELEMS * 2 + kk * 2));
#pragma unroll
      for (int n = 0; n < MAXDH / 8; ++n) {
        if (n < ntiles) {
          uint32_t bb[2];
          asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
                       : "=r"(bb[0]), "=r"(bb[1]) : "r"(va + (kk * VP + n * 8) * 2));
          mma_bf16_16816(acc[n], a, bb);
          if (SPLIT) mma_bf16_16816(acc[n], al, bb);
        }
      }
    }
    __syncthreads();                       // the next iteration's prefetch overwrites the other stage only after this
  }
  const int ar = warp * 16 + (lane >> 2), ac = 2 * (lane & 3);
#pragma unroll
  for (int n = 0; n < MAXDH / 8; ++n) {
    if (n < ntiles) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = i0 + ar + half * 8;
        if (r < nq)
          *reinterpret_cast<__nv_bfloat162*>(out + (static_cast<size_t>(b) * nq + r) * ldo + h * dh + n * 8 + ac) =
              __floats2bfloat162_rn(acc[n][2 * half], acc[n][2 * half + 1]);
      }
    }
  }
}

struct MixKey {
  const float *a, *b, *g, *be;
  bool operator<(const MixKey& o) const { return std::tie(a, b, g, be) < std::tie(o.a, o.b, o.g, o.be); }
};
std::map<MixKey, MixParams>& mix_cache() {
  static std::map<MixKey, MixParams> c;
  return c;
}

template <int H, int JS, int WPR>
void launch_mid_rows(float* S, const MixParams& P, int nq, int nk, int lds, int nkp, long long rows, int variant, cudaStream_t s) {
  constexpr int RPB = 8 / WPR;
  const unsigned blocks = static_cast<unsigned>((rows + RPB - 1) / RPB);
  if (variant == 1) mid_rows_kernel<H, JS, 1, WPR><<<blocks, 256, 0, s>>>(S, P, nq, nk, lds, nkp, rows);
  else mid_rows_kernel<H, JS, 2, WPR><<<blocks, 256, 0, s>>>(S, P, nq, nk, lds, nkp, rows);
}

// Talking-heads / re-attention path for heads in {8, 16} and nk <= 256 (every BASELINE config); false otherwise.
// The mix weights are tiny and constant per layer: they are read back once per (pointer set) and then travel as
// kernel parameters.  S must hold B * heads * nq * round_up(nk, 16) floats.
bool attention_rows_path(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                         __nv_bfloat16* out, int ldo, float* S, int B, int nq, int nk, int heads, int dh, int variant,
                         const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, cudaStream_t s) {
  if (variant != 1 && variant != 2) return false;
  if ((heads != 8 && heads != 16) || nk > 256 || dh > MAXDH) return false;
  if (reinterpret_cast<uintptr_t>(v) % 16 != 0 || reinterpret_cast<uintptr_t>(S) % 16 != 0) return false;
  const int nkp = (nk + 15) & ~15;
  const int lds = nkp;
  MixParams mixp;
  if (!attention_mix_params(mix_a, mix_b, ln_gamma, ln_beta, heads, s, &mixp)) return false;
  const float scale = 1.0f / sqrtf(static_cast<float>(dh));
  {
    const int sc_smem = (64 + ((nk + 7) & ~7)) * (dh + 8) * 2 + 32;   // +32: the last ldmatrix.x4 of a dh = 48 row touches its pad
    static int configured[256] = {0};                               // per device: the attribute is device state
    int dev = 0;
    VB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(global_cache_mutex());
    if (sc_smem > configured[dev & 255]) {
      VB_CUDA(cudaFuncSetAttribute(scores_stripe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sc_smem));
      configured[dev & 255] = sc_smem;
    }
    scores_stripe_kernel<<<flat_blocks((nq + 63) / 64, static_cast<long long>(B) * heads), 128, sc_smem, s>>>(q, ldq, k, ldk, S, heads, nq,
                                                                                                             nk, dh, scale, lds);
  }
  VB_CUDA(cudaGetLastError());
  const long long rows = static_cast<long long>(B) * nq;
  const int js = (nkp + 31) / 32;                                // key slots of 32 per row: 7 for n = 196 / 197
  if (heads == 8) {
    if (js <= 4) launch_mid_rows<8, 4, 1>(S, mixp, nq, nk, lds, nkp, rows, variant, s);
    else if (js <= 7) launch_mid_rows<8, 7, 1>(S, mixp, nq, nk, lds, nkp, rows, variant, s);
    else launch_mid_rows<8, 8, 1>(S, mixp, nq, nk, lds, nkp, rows, variant, s);
  } else {
    if (js <= 4) launch_mid_rows<16, 2, 2>(S, mixp, nq, nk, lds, nkp, rows, variant, s);
    else launch_mid_rows<16, 4, 2>(S, mixp, nq, nk, lds, nkp, rows, variant, s);
  }
  VB_CUDA(cudaGetLastError());
  const unsigned grid = flat_blocks((nq + 63) / 64, static_cast<long long>(B) * heads);
  if (variant == 1) {
    constexpr int smem = 2 * (2 * 64 * 72 + 64 * (MAXDH + 8)) * 2;
    static unsigned long long seen[4] = {0, 0, 0, 0};
    if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(pv_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    pv_rows_kernel<true><<<grid, 128, smem, s>>>(S, lds, nkp, v, ldv, out, ldo, heads, nq, nk, dh);
  } else {
    constexpr int smem = 2 * (64 * 72 + 64 * (MAXDH + 8)) * 2;
    static unsigned long long seen[4] = {0, 0, 0, 0};
    if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(pv_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    pv_rows_kernel<false><<<grid, 128, smem, s>>>(S, lds, nkp, v, ldv, out, ldo, heads, nq, nk, dh);
  }
  VB_CUDA(cudaGetLastError());
  count_launch(3);
  note_attention_path(ATTN_PATH_ROWS);
  return true;
}

}  // namespace

void attention_mix_cache_erase(const std::vector<const void*>& ptrs) {
  std::set<const void*> gone(ptrs.begin(), ptrs.end());
  gone.erase(nullptr);                                            // an absent operand (DeepViT has no mix_b) names nothing
  if (gone.empty()) return;
  std::lock_guard<std::mutex> lock(global_cache_mutex());
  auto& cache = mix_cache();
  for (auto it = cache.begin(); it != cache.end();) {
    const MixKey& k = it->first;
    if (gone.count(k.a) || gone.count(k.b) || gone.count(k.g) || gone.count(k.be)) it = cache.erase(it);
    else ++it;
  }
}

// The head-mix weights are tiny and constant per layer: they are read back from the device once per pointer set and then travel
// as kernel parameters (constant-bank operands).  The value is copied out under the lock: handles on other threads may erase
// their own entries.  The first use of a pointer set synchronises the stream, which a stream capture does not allow: the first
// call of a graph key is eager and fills the entry, and the entries of a handle are erased only by that handle (vb_finalize,
// vb_destroy), which drops its graphs at the same time.
bool attention_mix_params(const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, int heads,
                          cudaStream_t s, MixParams* out) {
  if (heads > 16 || heads < 1) return false;
  const MixKey key{mix_a, mix_b, ln_gamma, ln_beta};
  {
    std::lock_guard<std::mutex> lock(global_cache_mutex());       // weights are immutable while their entries exist
    auto& cache = mix_cache();
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return true; }
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  VB_CUDA(cudaStreamIsCapturing(s, &cs));
  VB_CHECK(cs == cudaStreamCaptureStatusNone, "attention_mix_params: head-mix weights first used inside a stream capture "
                                              "(their host copies were erased after the eager call of this key)");
  MixParams P = {};
  const size_t hh = static_cast<size_t>(heads) * heads * sizeof(float);
  VB_CUDA(cudaStreamSynchronize(s));
  if (mix_a) VB_CUDA(cudaMemcpy(P.wa, mix_a, hh, cudaMemcpyDeviceToHost));
  if (mix_b) VB_CUDA(cudaMemcpy(P.wb, mix_b, hh, cudaMemcpyDeviceToHost));
  if (ln_gamma) VB_CUDA(cudaMemcpy(P.gamma, ln_gamma, heads * sizeof(float), cudaMemcpyDeviceToHost));
  if (ln_beta) VB_CUDA(cudaMemcpy(P.beta, ln_beta, heads * sizeof(float), cudaMemcpyDeviceToHost));
  *out = P;
  std::lock_guard<std::mutex> lock(global_cache_mutex());
  mix_cache()[key] = P;
  return true;
}

bool attention_generic_mma(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                           __nv_bfloat16* out, int ldo, float* S, int B, int nq, int nk, int heads, int dh, int variant,
                           const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta, cudaStream_t s,
                           float scale, const PosBias* pb) {
  if (dh % 16 != 0 || dh > MAXDH || heads > MIX_MAX_HEADS) return false;
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2)) return false;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k)) % 16) return false;
  if (pb != nullptr && (variant != 0 || pb->wsz > 0 || pb->r2l_ws > 0)) return false;   // the window tables: the SIMT kernels (attn_pos_bias)
  if (pb == nullptr && attention_rows_path(q, ldq, k, ldk, v, ldv, out, ldo, S, B, nq, nk, heads, dh, variant, mix_a, mix_b, ln_gamma, ln_beta, s)) return true;
  const size_t smem = (static_cast<size_t>(heads) * nk + 2 * heads * heads) * sizeof(float);
  if (smem > 200 * 1024) return false;
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(mid_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  if (scale <= 0.f) scale = 1.0f / sqrtf(static_cast<float>(dh));
  const long long items = static_cast<long long>(B) * heads;
  scores_mma_kernel<<<flat_blocks(static_cast<long long>((nk + 63) / 64) * ((nq + 63) / 64), items), 128, 0, s>>>(q, ldq, k, ldk, S, heads,
                                                                                                                  nq, nk, dh, scale, nk);
  VB_CUDA(cudaGetLastError());
  mid_fused_kernel<<<flat_blocks(nq, B), 256, smem, s>>>(S, mix_a, mix_b, ln_gamma, ln_beta, heads, nq, nk, variant,
                                                         pb ? pb->table : nullptr, pb ? pb->fmap : 1, pb ? pb->step : 1);
  VB_CUDA(cudaGetLastError());
  const unsigned pv_grid = flat_blocks((nq + 63) / 64, items);
  const int gelu_out = pb != nullptr && pb->gelu_out;
  if (variant == 1) pv_mma_kernel<true><<<pv_grid, 128, 0, s>>>(S, v, ldv, out, ldo, heads, nq, nk, dh, gelu_out);
  else pv_mma_kernel<false><<<pv_grid, 128, 0, s>>>(S, v, ldv, out, ldo, heads, nq, nk, dh, gelu_out);
  VB_CUDA(cudaGetLastError());
  count_launch(3);
  note_attention_path(ATTN_PATH_MID_FUSED);
  return true;
}

}  // namespace vb
