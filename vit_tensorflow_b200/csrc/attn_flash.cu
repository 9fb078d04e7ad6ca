// Tensor-core multi-head attention for the bf16 engine (bf16 operands, fp32 accumulation, dim_head = 64; 32 in the windowed-bias and
// block forms and in the plain streaming form).
//
//   out[b, i, h, :] = softmax_j( scale * q[b,i,h,:] . k[b,j,h,:] ) @ v[b,j,h,:]        (vit.py:77-82)
//
// The [b,h,n,n] score tensor the reference materialises twice in memory (dots, attn) lives only in registers.
// One CTA per (64 query rows, b, h) on a flat grid index (no 65535 limit on B*h), 4 warps of 16 query rows each.  Q, K and
// V are read straight out of the row-major projection output ([B, n, 3*h*dh] for the fused to_qkv), so the head split 'b n (h d) -> b h n d' (vit.py:74) costs
// nothing; 64-key blocks of K and V stream through a two-stage cp.async ring.  Per block and warp:
//   S = Q K^T       mma.sync m16n8k16 (Q fragments loaded once, K fragments from the row-major K tile),
//   online softmax  row max / exp2 / row sum on the S fragments (a row lives in the 4 lanes of a quad),
//   O += P V        the S fragments, rounded to bf16, ARE the A fragments of the next product; V fragments by
//                   ldmatrix.trans from the row-major V tile.
// Final 1/l normalisation and bf16 stores in 'b n (h d)' order (the merge-heads rearrange, vit.py:82).
//
// BIAS (LeViT, levit.py:114-117,94): the head's [fmap^2] relative-position table sits in shared memory (in log2 units); every
// score gets table[pos_bias_index(i, j)] added before the online softmax, and the stored rows optionally go through GELU.
// With BIAS the scores are moved to log2 units as soon as they are computed, so the softmax below runs with a unit scale.
//
// WIN (Twins-SVT local attention, twins_svt.py:135-156): the flat batch index is a p x p window of a pixel-major map (Window,
// common.h), nq == nk == p^2.  Q, K and V rows are loaded from, and the output rows stored to, the map's own pixel rows, so the
// window split and merge rearranges (:141,153) cost no copies.  p^2 > 64 takes several query tiles and key blocks as any n does.
//
// BIAS and WIN (CrossFormer, crossformer.py:104-180; head width 32 or 64): windows as WIN, contiguous or dilated (Window), every
// score plus the window table of PosBias::wsz (one (2p-1)^2 table for all heads, in log2 units in shared memory).  Windows of up
// to 32 tokens share a 64-row query tile floor(64 / p^2) at a time, a block-diagonal mask keeping each to its own keys: the
// 4-token windows of CrossFormer's stage-3 long attention then fill 16 times fewer CTAs.
//
// WIN alone at head width 32 (NesT's block attention, nest.py:93-109; attention_block below): the same windowed form over
// rectangular bh x bw blocks (Window::pw), reached only through attention_block.  NesT's 14 x 14 blocks of 196 tokens take four
// query tiles and four key blocks each.  MobileViT's patch-position groups (mobile_vit.py:196-199) are dilated rectangular windows
// of the same form: the kernel reads every row through Window::row.
//
// Plain attention at head width 32 (ScalableViT's scalable self-attention, scalable_vit.py:123-143: h x w queries against the keys of
// an r x r stride-r convolution, nq != nk) runs the streaming form above, attn_flash_kernel<32, false, false>; the resident form
// below stays at 64.
//
// RegionViT's regional-to-local attention (attn_r2l_kernel, attention_r2l below) is a kernel of its own with the same tiles and
// online softmax: each window attends together with one regional row from elsewhere in the rows, under a per-head window table.
#include "attention.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cmath>

namespace vb {
namespace {

constexpr int DH = 64;             // head width of every path but the windowed-bias one (which also runs 32)
constexpr int FQ = 64;             // query rows per CTA
constexpr int FK = 64;             // keys per block

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

constexpr int FLASH_BIAS_MAX = 4096;   // fmap^2 of the largest relative-position table (16 KB of shared memory)

// MASK (attention.cuh's AttnMask): ATTN_MASK_KEYS masks image b's keys >= nk_img[b] and runs only the key blocks that hold a
// valid key; ATTN_MASK_DIAG masks key j == query i (plain attention, nq == nk).
template <int D, bool BIAS, bool WIN, int MASK = ATTN_MASK_NONE>
__global__ void __launch_bounds__(128)
attn_flash_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k, int ldk,
                  const __nv_bfloat16* __restrict__ v, int ldv, __nv_bfloat16* __restrict__ out, int ldo, int heads, int nq, int nk,
                  float scale_log2, const float* __restrict__ pos_tab, int fmap, int step, int gelu_out, Window win,
                  const int* __restrict__ nk_img) {
  constexpr int FP = D + 8;          // smem row pitch (bf16): +16 bytes keeps the fragment loads bank-conflict free
  constexpr bool WB = BIAS && WIN;   // the windowed-bias form (below)
  extern __shared__ float tab[];     // BIAS: [fmap^2] of this head / WB: the (2p-1)^2 window table; times log2(e)
  __shared__ __align__(16) __nv_bfloat16 Qs[FQ][FP];
  __shared__ __align__(16) __nv_bfloat16 Ks[2][FK][FP];
  __shared__ __align__(16) __nv_bfloat16 Vs[2][FK][FP];
  const int qtiles = (nq + FQ - 1) / FQ;
  const int bh = blockIdx.x / qtiles, b = bh / heads, h = bh % heads;
  const int i0 = (blockIdx.x % qtiles) * FQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int nblk = (nk + FK - 1) / FK;
  // WB: batch entry b is windows [b * G, b * G + G) of the win.count windows, G = floor(64 / p^2) for p^2 <= 32 and 1 above, so
  // nq == nk == G * p^2; token t of the entry is token t % p^2 of window b * G + t / p^2.  The last entry may hold fewer windows:
  // nqv / nkv are the entry's live tokens.
  const int wn = WB ? win.p * win.p : 1, G = WB ? (wn <= 32 ? FQ / wn : 1) : 1;
  const int nqv = WB ? min(nq, (win.count - b * G) * wn) : nq;
  int nkv = WB ? nqv : nk;
  // row of token i of this CTA's batch entry in the q / k / v / out matrices
  auto qrow_of = [&](int i) -> size_t {
    if (WB) return static_cast<size_t>(win.row(static_cast<long long>(b) * G + i / wn, i % wn));
    return WIN ? static_cast<size_t>(win.row(b, i)) : static_cast<size_t>(b) * nq + i;
  };
  auto krow_of = [&](int i) -> size_t {
    if (WB) return static_cast<size_t>(win.row(static_cast<long long>(b) * G + i / wn, i % wn));
    return WIN ? static_cast<size_t>(win.row(b, i)) : static_cast<size_t>(b) * nk + i;
  };

  pdl_wait();                 // Q/K/V come from the previous kernel of the stream
  pdl_launch_dependents();
  if (MASK == ATTN_MASK_KEYS) {   // keys >= nk_img[b] masked: only the blocks that hold a valid key (at least one: the cls row)
    nkv = min(nk, nk_img[b]);
    nblk = (nkv + FK - 1) / FK;
  }

  // rows past n are zero-filled (never read from the next image); D / 8 16-byte vectors per row
  constexpr int VR = D / 8, VS = D == 64 ? 3 : 2;                  // VR = 2^VS
  for (int e = threadIdx.x; e < FQ * VR; e += 128) {
    const int r = e >> VS, c = (e & (VR - 1)) * 8;
    if (i0 + r < nqv) cp_async16(smem_u32(&Qs[r][c]), q + qrow_of(i0 + r) * ldq + h * D + c);
    else *reinterpret_cast<uint4*>(&Qs[r][c]) = make_uint4(0, 0, 0, 0);
  }
  auto stage = [&](int j) {
    if (j < nblk) {
      const int s = j & 1, j0 = j * FK;
      for (int e = threadIdx.x; e < FK * VR; e += 128) {
        const int r = e >> VS, c = (e & (VR - 1)) * 8;
        if (j0 + r < nkv) {
          const size_t row = krow_of(j0 + r);
          cp_async16(smem_u32(&Ks[s][r][c]), k + row * ldk + h * D + c);
          cp_async16(smem_u32(&Vs[s][r][c]), v + row * ldv + h * D + c);
        } else {                                                     // zero V rows: 0 * garbage could be NaN
          *reinterpret_cast<uint4*>(&Ks[s][r][c]) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(&Vs[s][r][c]) = make_uint4(0, 0, 0, 0);
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  stage(0);
  int nqs = 1, qrow[2] = {0, 0};
  int qwin[2] = {0, 0}, qy[2] = {0, 0}, qx[2] = {0, 0};             // WB: window and in-window position of the two rows
  if (WB) {
    const int p = win.p, t2 = (2 * p - 1) * (2 * p - 1);
    for (int e = threadIdx.x; e < t2; e += 128) tab[e] = pos_tab[e] * 1.4426950408889634f;
    for (int r = 0; r < 2; ++r) {
      const int t = min(i0 + warp * 16 + (lane >> 2) + 8 * r, nqv - 1);   // rows past nqv: any live row
      qwin[r] = t / wn;
      qy[r] = (t - qwin[r] * wn) / p;
      qx[r] = t - qwin[r] * wn - qy[r] * p;
    }
  } else if (BIAS) {
    const int f2 = fmap * fmap;
    for (int e = threadIdx.x; e < f2; e += 128) tab[e] = pos_tab[static_cast<size_t>(h) * f2 + e] * 1.4426950408889634f;
    nqs = (fmap + step - 1) / step;
    for (int r = 0; r < 2; ++r) qrow[r] = min(i0 + warp * 16 + (lane >> 2) + 8 * r, nq - 1);   // rows past nq: any valid index
  }

  const int qr = lane >> 2, qc = 2 * (lane & 3);                     // fragment row (and row + 8) / column pair of this lane
  uint32_t qf[D / 16][4];
  float o[D / 8][4];
#pragma unroll
  for (int n = 0; n < D / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};    // running max (log2 units) / partial row sums

  for (int j = 0; j < nblk; ++j) {
    stage(j + 1);
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    if (j == 0) {
      const uint32_t qa = smem_u32(&Qs[warp * 16 + (lane & 15)][8 * (lane >> 4)]);
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(qf[kk][0]), "=r"(qf[kk][1]), "=r"(qf[kk][2]), "=r"(qf[kk][3]) : "r"(qa + kk * 32));
    }
    const int s = j & 1;
    // ---- S = Q K^T for this warp's 16 rows x 64 keys
    float sc[FK / 8][4];
#pragma unroll
    for (int n = 0; n < FK / 8; ++n) {
      sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Ks[s][n * 8 + qr][kk * 16 + qc]);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Ks[s][n * 8 + qr][kk * 16 + qc + 8]);
        mma_bf16_16816(sc[n], qf[kk], b0, b1);
      }
    }
    // ---- online softmax (rows qr and qr + 8 of the warp's tile)
    const int valid = nkv - j * FK;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < FK / 8; ++n) {
      int kwin[2] = {0, 0}, ky[2] = {0, 0}, kx[2] = {0, 0};          // WB: window and in-window position of the two key columns
      if (WB) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int u = j * FK + n * 8 + qc + c;
          kwin[c] = u / wn;
          ky[c] = (u - kwin[c] * wn) / win.p;
          kx[c] = u - kwin[c] * wn - ky[c] * win.p;
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (WB) {                                                    // the block-diagonal mask, then the window table
          const int c = e & 1, r = e >> 1;
          if (kwin[c] != qwin[r]) sc[n][e] = -INFINITY;
          else sc[n][e] = fmaf(sc[n][e], scale_log2, tab[(qy[r] - ky[c] + win.p - 1) * (2 * win.p - 1) + qx[r] - kx[c] + win.p - 1]);
        } else if (BIAS && n * 8 + qc + (e & 1) < valid)
          sc[n][e] = fmaf(sc[n][e], scale_log2, tab[pos_bias_index(qrow[e >> 1], j * FK + n * 8 + qc + (e & 1), fmap, step, nqs)]);
        if (n * 8 + qc + (e & 1) >= valid) sc[n][e] = -INFINITY;
        if (MASK == ATTN_MASK_DIAG && j * FK + n * 8 + qc + (e & 1) == i0 + warp * 16 + qr + 8 * (e >> 1)) sc[n][e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], sc[n][e]);
      }
    }
    const float sl = BIAS ? 1.0f : scale_log2;                      // BIAS: the scores are already in log2 units
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r] * sl);       // every block holds at least one valid key: finite
      alpha[r] = ex2_approx(m_run[r] - m_new);                       // first block: 2^-inf = 0
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
#pragma unroll
    for (int n = 0; n < D / 8; ++n) {
      o[n][0] *= alpha[0]; o[n][1] *= alpha[0];
      o[n][2] *= alpha[1]; o[n][3] *= alpha[1];
    }
    uint32_t pf[FK / 16][4];                                         // P as the A fragments of the PV product
#pragma unroll
    for (int n = 0; n < FK / 8; ++n) {
      const float p0 = ex2_approx(fmaf(sc[n][0], sl, -m_run[0]));
      const float p1 = ex2_approx(fmaf(sc[n][1], sl, -m_run[0]));
      const float p2 = ex2_approx(fmaf(sc[n][2], sl, -m_run[1]));
      const float p3 = ex2_approx(fmaf(sc[n][3], sl, -m_run[1]));
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pf[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      pf[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    // ---- O += P V
    const uint32_t va = smem_u32(&Vs[s][lane & 15][0]);
#pragma unroll
    for (int kk = 0; kk < FK / 16; ++kk) {
#pragma unroll
      for (int n = 0; n < D / 8; ++n) {
        uint32_t b0, b1;
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
                     : "=r"(b0), "=r"(b1) : "r"(va + (kk * 16 * FP + n * 8) * 2));
        mma_bf16_16816(o[n], pf[kk], b0, b1);
      }
    }
    __syncthreads();                       // the next iteration's prefetch overwrites this stage only after every warp is done
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    l_run[r] = 1.0f / l_run[r];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = i0 + warp * 16 + qr + 8 * r;
    if (row >= nqv) continue;
    __nv_bfloat16* orow = out + qrow_of(row) * ldo + h * D + qc;
#pragma unroll
    for (int n = 0; n < D / 8; ++n) {
      float a0 = o[n][2 * r] * l_run[r], a1 = o[n][2 * r + 1] * l_run[r];
      if (BIAS && gelu_out) { a0 = gelu_exact(a0); a1 = gelu_exact(a1); }
      *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_bf16x2(a0, a1);
    }
  }
}

// ---- Resident-head form (plain attention, nk <= 256): the whole of a head's K and V fits in shared memory, so a CTA loads each
// (b, h, query chunk) unit's Q, K and V once, by TMA, and runs its query rows against all of them.  The streaming kernel above
// instead gives each 64-row query tile its own CTA, which reloads the head's K and V, and computes whole 64-key blocks.
//   Persistent: one CTA per SM walks the units (head fastest, then query chunk of up to RQ rows, then image).  A producer
//   thread issues the next unit's three TMA boxes into the other of two unit buffers while RW compute warps work on this one.
//   Tensor maps {64 columns, token row, image} over the row-major projection output; rows past the image's n are out of bounds
//   and TMA fills them with zeros, so no row of the next image is read and the zero V rows keep 0 * P finite.
//   Compute warps take the 16-row query slices of a unit round-robin, continuing the rotation across units so that no warp
//   always takes the odd slice.  Keys run to round_up(nk, 16): each 64-key block computes only the 8-key S groups and 16-key
//   PV steps that hold a valid key, with the same online softmax (log2 units, ex2.approx, P rounded to bf16) as above.
//   A warp stages its 16 finished output rows in its own Q rows (swizzled) and stores them as 16-byte row segments.
constexpr int RQ = 256;                  // query rows per unit, and the most keys the resident form holds (one TMA box each)
constexpr int RW = 8;                    // compute warps; warp RW is the producer
constexpr int RTILE = RQ * DH * 2;       // bytes of one 256-row x 64-column bf16 tile (128-byte rows, 128-byte swizzle)
constexpr int RBUF = 3 * RTILE;          // Q | K | V of one unit
constexpr int RSMEM = 2 * RBUF + 1024 + 32;   // two unit buffers, 1024-byte alignment slack, four mbarriers

// byte address of 16-byte chunk `chunk` of row `row` in a 128-byte-swizzled tile that starts 1024-byte aligned
__device__ __forceinline__ uint32_t sw128(uint32_t tile, int row, int chunk) {
  return tile + row * 128 + ((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// mma.sync m16n8k16 without `volatile`: a pure register operation, so the compiler may interleave independent products
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One 64-key block of a 16-row query slice: S = Q K^T, the online-softmax update, O += P V.  PART (the last block, nk % 64
// keys): only the 8-key S groups and 16-key PV steps that hold a valid key, keys >= nk masked to -inf.  Full blocks take no
// per-group branch, so the products of all eight groups are in flight together.  DIAG: key qrow (this lane's first row) and
// qrow + 8 (its second) masked to -inf as well.
template <bool PART, bool DIAG = false>
__device__ __forceinline__ void resident_block(const uint32_t (&qf)[DH / 16][4], float (&o)[DH / 8][4], float (&m_run)[2],
                                               float (&l_run)[2], uint32_t tK, uint32_t tV, int j0, int nk, float scale_log2,
                                               int lane, int qrow = 0) {
  const int qc = 2 * (lane & 3);
  float sc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) {                 // K fragments of all 8 groups for dims [16 kk, 16 kk + 16), then 8 products
    uint32_t kf[8][2];
#pragma unroll
    for (int n = 0; n < 8; n += 2) {
      uint32_t r[4];                                     // b0, b1 of groups n and n + 1
      if (!PART || j0 + n * 8 < nk) ldsm_x4(r, sw128(tK, j0 + (n + (lane >> 4)) * 8 + (lane & 7), 2 * kk + ((lane >> 3) & 1)));
      kf[n][0] = r[0]; kf[n][1] = r[1]; kf[n + 1][0] = r[2]; kf[n + 1][1] = r[3];
    }
#pragma unroll
    for (int n = 0; n < 8; ++n)
      if (!PART || j0 + n * 8 < nk) mma_16816(sc[n], qf[kk], kf[n][0], kf[n][1]);
  }
  // ---- online softmax (rows lane / 4 and lane / 4 + 8 of the slice)
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (PART && j0 + n * 8 + qc + (e & 1) >= nk) sc[n][e] = -INFINITY;
      if (DIAG && j0 + n * 8 + qc + (e & 1) == qrow + 8 * (e >> 1)) sc[n][e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], sc[n][e]);
    }
  float alpha[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float m_new = fmaxf(m_run[r], mx[r] * scale_log2);    // every block holds at least one valid key: finite
    alpha[r] = ex2_approx(m_run[r] - m_new);                      // first block: 2^-inf = 0
    m_run[r] = m_new;
    l_run[r] *= alpha[r];
  }
#pragma unroll
  for (int n = 0; n < DH / 8; ++n) {
    o[n][0] *= alpha[0]; o[n][1] *= alpha[0];
    o[n][2] *= alpha[1]; o[n][3] *= alpha[1];
  }
  uint32_t pf[4][4];                                              // P as the A fragments of the PV product
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const float p0 = ex2_approx(fmaf(sc[n][0], scale_log2, -m_run[0]));
    const float p1 = ex2_approx(fmaf(sc[n][1], scale_log2, -m_run[0]));
    const float p2 = ex2_approx(fmaf(sc[n][2], scale_log2, -m_run[1]));
    const float p3 = ex2_approx(fmaf(sc[n][3], scale_log2, -m_run[1]));
    l_run[0] += p0 + p1;
    l_run[1] += p2 + p3;
    pf[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p0, p1);
    pf[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p2, p3);
  }
  // ---- O += P V
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    if (PART && j0 + kk * 16 >= nk) continue;
#pragma unroll
    for (int n = 0; n < DH / 8; n += 2) {
      uint32_t vf[4];                                             // b0, b1 of column groups n and n + 1
      ldsm_x4_trans(vf, sw128(tV, j0 + kk * 16 + (lane & 15), n + (lane >> 4)));
      mma_16816(o[n], pf[kk], vf[0], vf[1]);
      mma_16816(o[n + 1], pf[kk], vf[2], vf[3]);
    }
  }
}

// MASK (AttnMask): ATTN_MASK_KEYS masks image b's keys >= nk_img[b] and runs only the key blocks that hold a valid key;
// ATTN_MASK_DIAG masks key j == query i.
template <int MASK>
__global__ void __launch_bounds__((RW + 1) * 32, 1)
attn_resident_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                     const __grid_constant__ CUtensorMap tv, __nv_bfloat16* __restrict__ out, int ldo, int heads, int nq, int nk,
                     int qbox, int kbox, long long units, float scale_log2, const int* __restrict__ nk_img) {
  extern __shared__ __align__(16) uint8_t rsmem[];
  const uint32_t base = (smem_u32(rsmem) + 1023) & ~1023u;
  const uint32_t bars = base + 2 * RBUF;   // full[0], full[1], empty[0], empty[1]
  auto full_bar = [&](int s) { return bars + 8 * s; };
  auto empty_bar = [&](int s) { return bars + 16 + 8 * s; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunks = (nq + RQ - 1) / RQ;
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), RW);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();                 // Q/K/V come from the previous kernel of the stream, which may also still read `out`
  pdl_launch_dependents();

  if (warp == RW) {
    if (lane == 0) {
      tma_prefetch_desc(&tq);
      tma_prefetch_desc(&tk);
      tma_prefetch_desc(&tv);
      const uint32_t bytes = static_cast<uint32_t>(qbox + 2 * kbox) * DH * 2;
      int it = 0;
      for (long long u = blockIdx.x; u < units; u += gridDim.x, ++it) {
        const int s = it & 1;
        if (it >= 2) mbar_wait(empty_bar(s), ((it >> 1) + 1) & 1);
        const int h = static_cast<int>(u % heads);
        const long long bc = u / heads;
        const int c = static_cast<int>(bc % chunks), b = static_cast<int>(bc / chunks);
        const uint32_t t = base + s * RBUF;
        mbar_arrive_expect_tx(full_bar(s), bytes);
        tma_load_3d(t, &tq, full_bar(s), h * DH, c * RQ, b);
        tma_load_3d(t + RTILE, &tk, full_bar(s), h * DH, 0, b);
        tma_load_3d(t + 2 * RTILE, &tv, full_bar(s), h * DH, 0, b);
      }
    }
    return;
  }

  const int qr = lane >> 2, qc = 2 * (lane & 3);   // fragment row (and row + 8) / column pair of this lane
  int it = 0, rot = 0;                             // rot: the warp that takes slice 0 of this unit
  for (long long u = blockIdx.x; u < units; u += gridDim.x, ++it) {
    const int s = it & 1;
    const int h = static_cast<int>(u % heads);
    const long long bc = u / heads;
    const int c = static_cast<int>(bc % chunks), b = static_cast<int>(bc / chunks);
    const int i0 = c * RQ, slices = (min(RQ, nq - i0) + 15) / 16;
    const uint32_t tQ = base + s * RBUF, tK = tQ + RTILE, tV = tQ + 2 * RTILE;
    const int nkb = MASK == ATTN_MASK_KEYS ? min(nk, nk_img[b]) : nk;
    mbar_wait(full_bar(s), (it >> 1) & 1);
    for (int sl = (warp - rot + RW) % RW; sl < slices; sl += RW) {
      const int r16 = sl * 16;
      uint32_t qf[DH / 16][4];
#pragma unroll
      for (int kk = 0; kk < DH / 16; ++kk) ldsm_x4(qf[kk], sw128(tQ, r16 + (lane & 15), 2 * kk + (lane >> 4)));
      float o[DH / 8][4];
#pragma unroll
      for (int n = 0; n < DH / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

      constexpr bool DG = MASK == ATTN_MASK_DIAG;
      const int qrow = i0 + r16 + qr;
      for (int j0 = 0; j0 + 64 <= nkb; j0 += 64) resident_block<false, DG>(qf, o, m_run, l_run, tK, tV, j0, nkb, scale_log2, lane, qrow);
      if (nkb % 64) resident_block<true, DG>(qf, o, m_run, l_run, tK, tV, nkb & ~63, nkb, scale_log2, lane, qrow);

#pragma unroll
      for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
        l_run[r] = 1.0f / l_run[r];
      }
      // stage the 16 output rows in the slice's own Q rows (their fragments are in registers), then 16-byte row segments
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int n = 0; n < DH / 8; ++n) {
          const uint32_t val = pack_bf16x2(o[n][2 * r] * l_run[r], o[n][2 * r + 1] * l_run[r]);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(sw128(tQ, r16 + qr + 8 * r, n) + qc * 2), "r"(val) : "memory");
        }
      __syncwarp();
#pragma unroll
      for (int e = lane; e < 16 * 8; e += 32) {
        const int row = e >> 3, ch = e & 7, i = i0 + r16 + row;
        uint4 val;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(val.x), "=r"(val.y), "=r"(val.z), "=r"(val.w) : "r"(sw128(tQ, r16 + row, ch)) : "memory");
        if (i < nq) *reinterpret_cast<uint4*>(out + (static_cast<size_t>(b) * nq + i) * ldo + h * DH + ch * 8) = val;
      }
    }
    fence_proxy_async_smem();                      // the staging writes come before the next TMA load into this buffer
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(s));
    rot = (rot + slices) % RW;
  }
}

// The resident-head form of attention_fast's plain case; false (nothing launched) when the shape is not one it covers.
// mask (AttnMask) and nk_img (attention_masked): ATTN_MASK_KEYS takes the per-image key counts nk_img.
bool attention_resident(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                        __nv_bfloat16* out, int ldo, int B, int nq, int nk, int heads, float scale_log2, cudaStream_t s,
                        const int* nk_img = nullptr, int mask = ATTN_MASK_NONE) {
  if (nk > RQ || (ldo % 8)) return false;
  const int qbox = std::min(RQ, (nq + 15) & ~15), kbox = (nk + 15) & ~15;
  const uint64_t inner = static_cast<uint64_t>(heads) * DH;
  const CUtensorMap tq = make_tmap_3d(q, inner, nq, B, static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(nq) * ldq * 2, DH, qbox);
  const CUtensorMap tk = make_tmap_3d(k, inner, nk, B, static_cast<uint64_t>(ldk) * 2, static_cast<uint64_t>(nk) * ldk * 2, DH, kbox);
  const CUtensorMap tv = make_tmap_3d(v, inner, nk, B, static_cast<uint64_t>(ldv) * 2, static_cast<uint64_t>(nk) * ldv * 2, DH, kbox);
  const long long units = static_cast<long long>(B) * heads * ((nq + RQ - 1) / RQ);
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) {
    VB_CUDA(cudaFuncSetAttribute(attn_resident_kernel<ATTN_MASK_NONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, RSMEM));
    VB_CUDA(cudaFuncSetAttribute(attn_resident_kernel<ATTN_MASK_KEYS>, cudaFuncAttributeMaxDynamicSharedMemorySize, RSMEM));
    VB_CUDA(cudaFuncSetAttribute(attn_resident_kernel<ATTN_MASK_DIAG>, cudaFuncAttributeMaxDynamicSharedMemorySize, RSMEM));
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(units < sm_count() ? units : sm_count()));
  cfg.blockDim = dim3((RW + 1) * 32);
  cfg.dynamicSmemBytes = RSMEM;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (mask == ATTN_MASK_KEYS)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_resident_kernel<ATTN_MASK_KEYS>, tq, tk, tv, out, ldo, heads, nq, nk, qbox, kbox, units, scale_log2,
                               nk_img));
  else if (mask == ATTN_MASK_DIAG)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_resident_kernel<ATTN_MASK_DIAG>, tq, tk, tv, out, ldo, heads, nq, nk, qbox, kbox, units, scale_log2,
                               static_cast<const int*>(nullptr)));
  else
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_resident_kernel<ATTN_MASK_NONE>, tq, tk, tv, out, ldo, heads, nq, nk, qbox, kbox, units, scale_log2,
                               static_cast<const int*>(nullptr)));
  return true;
}

template <int D>
void launch_window_bias(cudaLaunchConfig_t& cfg, const __nv_bfloat16* q, int ldq, __nv_bfloat16* out, int ldo, int heads, int n,
                        float scale_log2, const PosBias& pb, const Window& win) {
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen))
    VB_CUDA(cudaFuncSetAttribute(attn_flash_kernel<D, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FLASH_BIAS_MAX * 4));
  const int HD = heads * D;
  VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<D, true, true>, q, ldq, q + HD, ldq, q + 2 * HD, ldq, out, ldo, heads, n, n,
                             scale_log2, pb.table, 0, 1, 0, win, static_cast<const int*>(nullptr)));
}

// CrossFormer's attention: windows of B = win.count images' maps, q | k | v at columns [0, HD), [HD, 2 HD), [2 HD, 3 HD) of the
// fused rows (HD = heads * dh), the window table of pb added to every score.  p^2 <= 32 packs floor(64 / p^2) windows into a
// tile; 32 < p^2 <= 64 is one window per tile; larger windows take several query tiles and key blocks.
bool attention_window_bias(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                           __nv_bfloat16* out, int ldo, int B, int nq, int nk, int heads, int dh, cudaStream_t s, float scale,
                           const PosBias& pb, const Window& win) {
  const int n = win.p * win.p, HD = heads * dh;
  if (pb.wsz != win.p || nq != n || nk != n || (dh != 32 && dh != 64)) return false;
  if ((2 * win.p - 1) * (2 * win.p - 1) > FLASH_BIAS_MAX) return false;
  if (k != q + HD || v != q + 2 * HD || ldk != ldq || ldv != ldq || (ldq % 8) || (ldo % 2)) return false;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(out)) % 16) return false;
  const int G = n <= 32 ? FQ / n : 1, tile = G * n;
  const long long entries = (static_cast<long long>(B) + G - 1) / G;
  const long long blocks = entries * heads * ((tile + FQ - 1) / FQ);
  if (blocks > 0x7fffffffLL || B <= 0) return false;
  Window w = win;
  w.count = B;
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(blocks));
  cfg.blockDim = dim3(128);
  cfg.stream = s;
  cfg.dynamicSmemBytes = static_cast<size_t>(2 * win.p - 1) * (2 * win.p - 1) * sizeof(float);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (dh == 32) launch_window_bias<32>(cfg, q, ldq, out, ldo, heads, tile, scale_log2, pb, w);
  else launch_window_bias<64>(cfg, q, ldq, out, ldo, heads, tile, scale_log2, pb, w);
  count_launch();
  note_attention_path(ATTN_PATH_FLASH);
  return true;
}

// ---- RegionViT's regional-to-local attention (regionvit.py:163-177; attention_r2l below), head width 32.  One CTA per (64 query
// rows, window, head) as attn_flash_kernel, over the n = 1 + p q tokens of window bw = (b, wy, wx): token 0 is the regional row
// reg_row0 + bw of the fused q|k|v rows ((b * rh + wy) * rw + wx: the region map's own pixel order), token t > 0 the window's
// local row win.row(bw, t - 1).  Scores are moved to log2 units as computed, plus (i, j > 0) the head's table entry of the
// window offset (PosBias::r2l_ws, common.h); row 0 and column 0 take no bias.  Output row 0 goes to the regional row, the others
// to the local rows, so nothing is gathered, scattered or materialised.  n > 64 (14 x 14 windows: 197 tokens) takes several
// query tiles and key blocks.
__global__ void __launch_bounds__(128)
attn_r2l_kernel(const __nv_bfloat16* __restrict__ qkv, int ld, __nv_bfloat16* __restrict__ out, int ldo, int heads, long long reg_row0,
                float scale_log2, const float* __restrict__ table, int ws, Window win) {
  constexpr int D = 32, FP = D + 8, VR = D / 8;
  extern __shared__ float tab[];     // this head's (2 ws - 1)^2 table, times log2(e)
  __shared__ __align__(16) __nv_bfloat16 Qs[FQ][FP];
  __shared__ __align__(16) __nv_bfloat16 Ks[2][FK][FP];
  __shared__ __align__(16) __nv_bfloat16 Vs[2][FK][FP];
  const int ww = win.width(), n = 1 + win.p * ww, HD = heads * D, side = 2 * ws - 1;
  const int qtiles = (n + FQ - 1) / FQ;
  const long long wh = blockIdx.x / qtiles, bw = wh / heads;
  const int h = static_cast<int>(wh - bw * heads);
  const int i0 = (blockIdx.x % qtiles) * FQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nblk = (n + FK - 1) / FK;
  auto row_of = [&](int t) -> size_t { return static_cast<size_t>(t == 0 ? reg_row0 + bw : win.row(bw, t - 1)); };

  pdl_wait();                 // q|k|v come from the previous kernel of the stream
  pdl_launch_dependents();

  for (int e = threadIdx.x; e < FQ * VR; e += 128) {
    const int r = e >> 2, c = (e & (VR - 1)) * 8;
    if (i0 + r < n) cp_async16(smem_u32(&Qs[r][c]), qkv + row_of(i0 + r) * ld + h * D + c);
    else *reinterpret_cast<uint4*>(&Qs[r][c]) = make_uint4(0, 0, 0, 0);
  }
  auto stage = [&](int j) {
    if (j < nblk) {
      const int s = j & 1, j0 = j * FK;
      for (int e = threadIdx.x; e < FK * VR; e += 128) {
        const int r = e >> 2, c = (e & (VR - 1)) * 8;
        if (j0 + r < n) {
          const __nv_bfloat16* src = qkv + row_of(j0 + r) * ld + h * D + c;
          cp_async16(smem_u32(&Ks[s][r][c]), src + HD);
          cp_async16(smem_u32(&Vs[s][r][c]), src + 2 * HD);
        } else {                                                     // zero V rows: 0 * garbage could be NaN
          *reinterpret_cast<uint4*>(&Ks[s][r][c]) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(&Vs[s][r][c]) = make_uint4(0, 0, 0, 0);
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  stage(0);
  for (int e = threadIdx.x; e < side * side; e += 128) tab[e] = table[static_cast<size_t>(h) * side * side + e] * 1.4426950408889634f;
  int qy[2], qx[2];                                                  // window position of the lane's two rows; qy = -1: the regional row
  for (int r = 0; r < 2; ++r) {
    const int t = min(i0 + warp * 16 + (lane >> 2) + 8 * r, n - 1);  // rows past n: any live row
    qy[r] = t == 0 ? -1 : (t - 1) / ww;
    qx[r] = t == 0 ? 0 : t - 1 - qy[r] * ww;
  }

  const int qr = lane >> 2, qc = 2 * (lane & 3);
  uint32_t qf[D / 16][4];
  float o[D / 8][4];
#pragma unroll
  for (int k = 0; k < D / 8; ++k) o[k][0] = o[k][1] = o[k][2] = o[k][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int j = 0; j < nblk; ++j) {
    stage(j + 1);
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    if (j == 0) {
      const uint32_t qa = smem_u32(&Qs[warp * 16 + (lane & 15)][8 * (lane >> 4)]);
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(qf[kk][0]), "=r"(qf[kk][1]), "=r"(qf[kk][2]), "=r"(qf[kk][3]) : "r"(qa + kk * 32));
    }
    const int s = j & 1;
    float sc[FK / 8][4];
#pragma unroll
    for (int g = 0; g < FK / 8; ++g) {
      sc[g][0] = sc[g][1] = sc[g][2] = sc[g][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Ks[s][g * 8 + qr][kk * 16 + qc]);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Ks[s][g * 8 + qr][kk * 16 + qc + 8]);
        mma_bf16_16816(sc[g], qf[kk], b0, b1);
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int g = 0; g < FK / 8; ++g) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int u = j * FK + g * 8 + qc + c;
        const int ky = u > 0 ? (u - 1) / ww : -1, kx = u > 0 ? u - 1 - ky * ww : 0;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float& v = sc[g][2 * r + c];
          if (u >= n) v = -INFINITY;
          else v = v * scale_log2 + (qy[r] >= 0 && ky >= 0 ? tab[(qy[r] - ky + ws - 1) * side + qx[r] - kx + ws - 1] : 0.f);
          mx[r] = fmaxf(mx[r], v);
        }
      }
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);                    // every block holds at least one valid key: finite
      alpha[r] = ex2_approx(m_run[r] - m_new);
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
#pragma unroll
    for (int k = 0; k < D / 8; ++k) {
      o[k][0] *= alpha[0]; o[k][1] *= alpha[0];
      o[k][2] *= alpha[1]; o[k][3] *= alpha[1];
    }
    uint32_t pf[FK / 16][4];
#pragma unroll
    for (int g = 0; g < FK / 8; ++g) {
      const float p0 = ex2_approx(sc[g][0] - m_run[0]), p1 = ex2_approx(sc[g][1] - m_run[0]);
      const float p2 = ex2_approx(sc[g][2] - m_run[1]), p3 = ex2_approx(sc[g][3] - m_run[1]);
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pf[g >> 1][(g & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      pf[g >> 1][(g & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    const uint32_t va = smem_u32(&Vs[s][lane & 15][0]);
#pragma unroll
    for (int kk = 0; kk < FK / 16; ++kk) {
#pragma unroll
      for (int k = 0; k < D / 8; ++k) {
        uint32_t b0, b1;
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];"
                     : "=r"(b0), "=r"(b1) : "r"(va + (kk * 16 * FP + k * 8) * 2));
        mma_bf16_16816(o[k], pf[kk], b0, b1);
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    l_run[r] = 1.0f / l_run[r];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = i0 + warp * 16 + qr + 8 * r;
    if (row >= n) continue;
    __nv_bfloat16* orow = out + row_of(row) * ldo + h * D + qc;
#pragma unroll
    for (int k = 0; k < D / 8; ++k)
      *reinterpret_cast<uint32_t*>(orow + k * 8) = pack_bf16x2(o[k][2 * r] * l_run[r], o[k][2 * r + 1] * l_run[r]);
  }
}

}  // namespace

bool attention_r2l(const __nv_bfloat16* qkv, int ld, __nv_bfloat16* out, int ldo, int heads, int dh, long long reg_row0,
                   const PosBias& pb, const Window& win, cudaStream_t s, float scale) {
  const int ws = pb.r2l_ws, side = 2 * ws - 1, n = 1 + win.p * win.width();
  if (dh != 32 || ws <= 0 || side * side > FLASH_BIAS_MAX || win.dilated || win.count <= 0 || n <= 1) return false;
  if (pb.r2l_h != win.p || pb.r2l_w != win.width() || win.p > ws || win.width() > ws) return false;
  if ((ld % 8) || (ldo % 2) || ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) % 16)) return false;
  const long long blocks = static_cast<long long>(win.count) * heads * ((n + FQ - 1) / FQ);
  if (blocks > 0x7fffffffLL) return false;
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(blocks));
  cfg.blockDim = dim3(128);
  cfg.dynamicSmemBytes = static_cast<size_t>(side) * side * sizeof(float);   // with the 25.6 KB static tiles: under 48 KB
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VB_CUDA(cudaLaunchKernelEx(&cfg, attn_r2l_kernel, qkv, ld, out, ldo, heads, reg_row0, scale_log2, pb.table, ws, win));
  count_launch();
  note_attention_path(ATTN_PATH_FLASH);
  return true;
}

bool attention_block(const __nv_bfloat16* qkv, int ld, __nv_bfloat16* out, int ldo, int heads, int dh, cudaStream_t s, float scale,
                     const Window& win) {
  const int n = win.p * win.width();
  const long long B = static_cast<long long>(win.count);
  if ((dh != 32 && dh != 64) || n <= 0 || B <= 0) return false;
  if ((ld % 8) || (ldo % 2) || ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) % 16)) return false;
  const long long blocks = B * heads * ((n + FQ - 1) / FQ);
  if (blocks > 0x7fffffffLL) return false;
  const int HD = heads * dh;
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(blocks));
  cfg.blockDim = dim3(128);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (dh == 32)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<32, false, true>, qkv, ld, qkv + HD, ld, qkv + 2 * HD, ld, out, ldo, heads, n, n,
                               scale_log2, static_cast<const float*>(nullptr), 0, 1, 0, win, static_cast<const int*>(nullptr)));
  else
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<64, false, true>, qkv, ld, qkv + HD, ld, qkv + 2 * HD, ld, out, ldo, heads, n, n,
                               scale_log2, static_cast<const float*>(nullptr), 0, 1, 0, win, static_cast<const int*>(nullptr)));
  count_launch();
  note_attention_path(ATTN_PATH_FLASH);
  return true;
}

template <>
bool attention_fast<__nv_bfloat16>(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                                   __nv_bfloat16* out, int ldo, int B, int nq, int nk, int heads, int dh, int variant,
                                   const float* mix_a, const float* mix_b, const float* ln_g, const float* ln_b, cudaStream_t s,
                                   float scale, const PosBias* pb, const Window* win) {
  if (win != nullptr && pb != nullptr) return attention_window_bias(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, dh, s, scale, *pb, *win);
  if (pb != nullptr && pb->wsz > 0) return false;
  if (win != nullptr && (nq != win->p * win->p || nk != nq)) return false;
  if (nq == 1 && pb == nullptr && win == nullptr && attention_cls(q, ldq, k, ldk, v, ldv, out, ldo, B, nk, heads, dh, variant, mix_a, mix_b, ln_g, ln_b, s, scale)) return true;
  // DeepViT re-attention / CaiT talking heads: the materialised-scores path (attn_generic_mma.cu) -- a fused form with all heads'
  // scores of a 16-row tile in shared memory measured 9-11 % slower on the H100 (one CTA per SM at 16 heads)
  const bool narrow = dh == 32 && pb == nullptr && win == nullptr;   // plain attention at head width 32: the streaming kernel
  if (variant != 0 || (dh != DH && !narrow) || (nq < 2 && pb == nullptr)) return false;
  if (pb != nullptr && (pb->fmap * pb->fmap > FLASH_BIAS_MAX || nk != pb->fmap * pb->fmap || nq != pb->q_side() * pb->q_side())) return false;
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2)) return false;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
       reinterpret_cast<uintptr_t>(out)) % 16) return false;
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  if (pb == nullptr && win == nullptr && !narrow && attention_resident(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, scale_log2, s)) {
    count_launch();
    note_attention_path(ATTN_PATH_FLASH);
    return true;
  }
  cudaLaunchConfig_t cfg = {};
  const long long blocks = static_cast<long long>(B) * heads * ((nq + FQ - 1) / FQ);
  if (blocks > 0x7fffffffLL) return false;
  cfg.gridDim = dim3(static_cast<unsigned>(blocks));
  cfg.blockDim = dim3(128);
  cfg.stream = s;
  if (pb != nullptr) {
    static unsigned long long seen[4] = {0, 0, 0, 0};
    if (first_use_on_this_device(seen))
      VB_CUDA(cudaFuncSetAttribute(attn_flash_kernel<DH, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FLASH_BIAS_MAX * 4));
    cfg.dynamicSmemBytes = static_cast<size_t>(pb->fmap) * pb->fmap * sizeof(float);
  }
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (pb != nullptr)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<DH, true, false>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk, scale_log2,
                               pb->table, pb->fmap, pb->step, static_cast<int>(pb->gelu_out), Window(),
                               static_cast<const int*>(nullptr)));
  else if (win != nullptr)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<DH, false, true>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk, scale_log2,
                               static_cast<const float*>(nullptr), 0, 1, 0, *win, static_cast<const int*>(nullptr)));
  else if (narrow)
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<32, false, false>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk, scale_log2,
                               static_cast<const float*>(nullptr), 0, 1, 0, Window(), static_cast<const int*>(nullptr)));
  else
    VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<DH, false, false>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk, scale_log2,
                               static_cast<const float*>(nullptr), 0, 1, 0, Window(), static_cast<const int*>(nullptr)));
  count_launch();
  note_attention_path(ATTN_PATH_FLASH);
  return true;
}

bool attention_masked(const __nv_bfloat16* q, int ldq, const __nv_bfloat16* k, int ldk, const __nv_bfloat16* v, int ldv,
                      __nv_bfloat16* out, int ldo, int B, int nq, int nk, int heads, int dh, cudaStream_t s, float scale,
                      const int* nk_img, int mask) {
  if (dh != DH || nq < 1 || nk < 1 || B < 1 || (ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 2)) return false;
  if (mask == ATTN_MASK_DIAG && (nq != nk || nk < 2)) return false;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
       reinterpret_cast<uintptr_t>(out)) % 16) return false;
  const float scale_log2 = (scale > 0.f ? scale : 1.0f / sqrtf(static_cast<float>(dh))) * 1.4426950408889634f;
  if (!attention_resident(q, ldq, k, ldk, v, ldv, out, ldo, B, nq, nk, heads, scale_log2, s, nk_img, mask)) {
    const long long blocks = static_cast<long long>(B) * heads * ((nq + FQ - 1) / FQ);
    if (blocks > 0x7fffffffLL) return false;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(blocks));
    cfg.blockDim = dim3(128);
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (mask == ATTN_MASK_DIAG)
      VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<DH, false, false, ATTN_MASK_DIAG>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk,
                                 scale_log2, static_cast<const float*>(nullptr), 0, 1, 0, Window(), static_cast<const int*>(nullptr)));
    else
      VB_CUDA(cudaLaunchKernelEx(&cfg, attn_flash_kernel<DH, false, false, ATTN_MASK_KEYS>, q, ldq, k, ldk, v, ldv, out, ldo, heads, nq, nk,
                                 scale_log2, static_cast<const float*>(nullptr), 0, 1, 0, Window(), nk_img));
  }
  count_launch();
  note_attention_path(ATTN_PATH_FLASH);
  return true;
}

}  // namespace vb
