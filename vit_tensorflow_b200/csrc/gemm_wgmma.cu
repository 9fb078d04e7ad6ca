// Warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   out[M,N] (bf16) = epi( A[M,K] (bf16, K-major) x Wt[N,K]^T (bf16, K-major) ),  fp32 accumulation in registers
//   epi(v) = (+bias[n]) -> exact-erf GELU, hard-swish or SiLU -> (*scale[n]) -> (+res[m,n])
//
// Replaces, on the reference's hot path, every nn.Dense: patch embedding (vit.py:143), to_qkv (vit.py:59,72),
// to_out + residual (vit.py:62-69,101), MLP fc1+GELU / fc2 + residual (vit.py:38-44,102), CaiT to_q/to_kv
// (cait.py:94-95) with LayerScale folded in (cait.py:48).
//
// Structure: persistent, one CTA of 384 threads per SM; CTA b computes the 128 x BN output tiles b, b + gridDim.x, ...
// of the flat tile order (n fastest).  BN = 192 where it divides N and N >= 1536 (ViT-B/16's to_qkv and fc1), else 128
// (gemm_bf16_plan states the rule): a 128 x 192 k-block brings 40 KB from L2 for 3.1 MFLOP against 32 KB for 2.1, and
// each tile's fixed cost (epilogue, handover) is spread over 1.5x the work.  192 is the widest N at which one consumer
// warpgroup still holds a whole tile's accumulators (2 x 96 fp32 registers per thread).
//   producer        warpgroup 0 (its registers handed to the consumers by setmaxnreg).  Thread 0 streams the A (128 x 64)
//                   and B (BN x 64) k-blocks of the CTA's tiles, one tile after the other, into a STAGES-deep ring of
//                   128B-swizzled tiles (mbarrier full / empty pairs; 4 x 32 KB at BN = 128, 3 x 40 KB at 192).  Warps 1-3
//                   prepare each tile's epilogue operands ahead of it, in the buffers of the consumer warpgroup that will
//                   run it: the residual tile (TMA loads into the warpgroup's output staging tile), the bias / ln_c1 /
//                   scale of its columns and the folded LayerNorm's (rstd, -mu rstd) of its rows (mbarrier epi_full /
//                   epi_empty pair per warpgroup).
//   2 consumer warpgroups, ping-pong: warpgroup w computes the CTA's tiles i = w (mod 2), each whole: two wgmma
//                   m64 x BN x 16 per k16 step (rows 0-63 and 64-127 of the tile) into register accumulators, one k-block
//                   in flight while the previous one's stage is released; then the epilogue from the accumulator
//                   registers (bias / folded LayerNorm / GELU / LayerScale / residual, optional per-64-column row
//                   statistics of the stored values), reading its operands from shared memory only.  A bf16 tile is
//                   written into the staging tile (over its residual) by stmatrix and leaves by one TMA store per 64 x 128 half; an
//                   fp32 tile is stored straight from registers.  Two named barriers pass the main loop from one
//                   warpgroup to the other, so the main loops take turns on the tensor cores and one tile's epilogue runs
//                   under the next tile's main loop.
#include <type_traits>

#include "common.h"
#include "kernels.cuh"
#include "philox.cuh"
#include "ptx.cuh"

namespace vb {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;             // 64 bf16 = 128 bytes = one swizzle row
constexpr int THREADS = 384;
constexpr int A_BYTES = BM * BK * 2;
constexpr int HALF_BYTES = BM * 64 * 2;      // 64 columns of an output tile: 128 rows of 128 bytes, 128B-swizzled
constexpr int EPI_THREADS = 96;    // producer warps 1-3

// Everything that follows the tile width BN (128 or 192).
template <int BN>
struct Tile {
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // of the 227 KB a CTA may use: 4 x 32 KB ring + 2 x 32 KB output staging, or 3 x 40 KB + 2 x 48 KB.  Both rings hold
  // about the same tensor-core time (8.4 and 9.4 MFLOP), and a stage is refilled while the two after it are computed.
  static constexpr int STAGES = BN == 128 ? 4 : 3;
  static constexpr int STG_BYTES = BN / 64 * HALF_BYTES;   // per consumer warpgroup: its bf16 output tile (and residual
                                                          // tile before it), one 128B-swizzled box per 64-column half
  static constexpr int PARAM_FLOATS = 3 * BN + 2 * BM;    // per consumer warpgroup: bias, ln_c1, scale of its tile's
                                                          // columns; the folded LayerNorm's rstd and -mu rstd of its rows
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * STG_BYTES + 256 /*barriers*/ + 2 * PARAM_FLOATS * 4 + 1024 /*align*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "ring does not fit in shared memory");
};
// setmaxnreg: the launch gives every thread 168 registers (65,536 / 384, rounded down to a multiple of 8); the producer
// warpgroup hands what it does not need to the consumers, whose accumulators take BN fp32 registers per thread.  At BN = 192
// the 192 accumulators and the epilogue's state fit in 232 without spilling; the producer's warps need 40.
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 168 * THREADS, "setmaxnreg exceeds the CTA's registers");

// Exact-erf GELU (vit.py:34), written as  gelu(x) = x/2 - |x| * (E(|x|) - 1/2),  E(a) = erfc(a/sqrt2) / 2  (for x > 0
// this is x - x E, for x < 0 it is x E), with E evaluated as 2^q(a): q is a degree-5 polynomial (weighted minimax fit
// of log2(erfc(a/sqrt2)/2) on a in [0, 6], constant term exactly -1; tools/gelu_error.py refits and checks it).  Its
// leading coefficient is negative and q is monotone beyond the fit range, so no clamp is needed: for |x| > 6 the tail
// term |x| 2^q is below 6 * 2^-29 and shrinks.  Max abs error of the GELU 5.7e-7 = 0.003 bf16 ulp of the result for
// every finite x; gelu(+inf) = +inf and gelu(-inf) = NaN as in the reference's x * Phi(x).
// It takes h = x / 2, which the epilogue's bias / folded-LayerNorm FMAs produce at no cost (their operands are staged
// halved), and returns  h - |h| (2 E - 1)  with q's k-th coefficient scaled by 2^k for the argument -|h|.  Every scaling
// is by a power of two, so each rounding is the one  x/2 - |x| (E - 1/2)  makes from x (outside the subnormal range),
// without its multiply by 1/2.
__device__ __forceinline__ float gelu_erf_half(float h) {
  const float na = -fabsf(h);                                        // -|x| / 2
  float q = fmaf(4.881368368e-04f * 32.f, na, 7.198925130e-03f * 16.f);   // odd coefficients negated: q(-2 na)
  q = fmaf(q, na, 5.214704946e-02f * 8.f);
  q = fmaf(q, na, -4.595955014e-01f * 4.f);
  q = fmaf(q, na, 1.151000619e+00f * 2.f);
  q = fmaf(q, na, -1.0f);
  const float e = ex2_approx(q);                                     // erfc(|x|/sqrt2) / 2
  return fmaf(na, fmaf(2.f, e, -1.f), h);
}

// levit.py:37: x * relu6(x + 3) / 6, rounded in the reference's order
__device__ __forceinline__ float hard_swish(float x) { return __fdiv_rn(x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f), 6.0f); }

// Advance a ring position (stage, phase) by n k-blocks.
template <int STAGES>
__device__ __forceinline__ void ring_advance(int& stage, uint32_t& phase, int n) {
  stage += n % STAGES;
  phase ^= static_cast<uint32_t>(n / STAGES) & 1u;
  if (stage >= STAGES) { stage -= STAGES; phase ^= 1u; }
}

// EPI: 0 = no per-column addend, 1 = + bias[n], 2 = folded LayerNorm (c1 = ln_c1, c2 = bias)
// DROP: training-mode dropout (DropPos), its own instances; DROP_NONE compiles the epilogue without it
template <int BN, int ACT, bool RES, int EPI, bool OF32, int DROP = DROP_NONE>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_res, int M, int N, int K,
                 float* __restrict__ out_f32, int ldc, const float* __restrict__ bias, const float* __restrict__ scale,
                 const float* __restrict__ ln_c1, const float2* ln_stats, int ln_parts, float ln_inv_d, float ln_eps,
                 float2* __restrict__ stats_out, const unsigned long long* drop_state, uint32_t drop_site, float drop_rate,
                 float drop_scale) {
  static_assert(!OF32 || (ACT == ACT_NONE && !RES && EPI != 2), "fp32 output: plain / bias epilogue only");
  static_assert(DROP == DROP_NONE || (!OF32 && (DROP == DROP_BEFORE_RES || RES)), "dropout: bf16 output; after the residual needs one");
  static_assert(BN == 128 || BN == 192, "tile width");
  using T = Tile<BN>;
  constexpr int STAGES = T::STAGES, STAGE_BYTES = T::STAGE_BYTES, STG_BYTES = T::STG_BYTES, PARAM_FLOATS = T::PARAM_FLOATS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t stg_base = smem_base + STAGES * STAGE_BYTES;     // consumer warpgroup w's staging tile at + w STG_BYTES
  const uint32_t bar_base = stg_base + 2 * STG_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto epi_full = [&](int w) { return bar_base + 8u * (2 * STAGES + w); };        // warpgroup w's epilogue operands staged
  auto epi_empty = [&](int w) { return bar_base + 8u * (2 * STAGES + 2 + w); };   // ... and consumed (staging tile stored)
  uint8_t* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  float* const params = reinterpret_cast<float*>(smem + (bar_base + 256 - smem_base));   // [2][PARAM_FLOATS]

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  // flat tile order, n fastest: the tiles that share an A row block run together; 64-bit, so neither M nor the tile count
  // is bounded by a grid dimension
  const int n_tiles = (N + BN - 1) / BN;
  const long long tiles = static_cast<long long>(n_tiles) * ((M + BM - 1) / BM);
  const int num_kb = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (!OF32) tma_prefetch_desc(&tmap_out);
    if (RES) tma_prefetch_desc(&tmap_res);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);                                  // released by the warpgroup that consumed the stage
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(epi_full(w), EPI_THREADS);
      mbar_init(epi_empty(w), 1);                                  // thread 0 of the consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Everything above overlapped the previous kernel's tail (PDL); from here on we touch its outputs.
  pdl_wait();
  pdl_launch_dependents();

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (tid == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int n0 = static_cast<int>(t % n_tiles) * BN;
        const int m0 = static_cast<int>(t / n_tiles) * BM;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), STAGE_BYTES);     // out-of-range box elements are zero-filled and counted
          tma_load_2d(sa, &tmap_a, full_bar(stage), kb * BK, m0);
          tma_load_2d(sa + A_BYTES, &tmap_b, full_bar(stage), kb * BK, n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (tid >= 32) {
      // ------------------------------------------------------------------- epilogue operands of the CTA's tiles, in order:
      // tile i goes to consumer warpgroup w = i % 2 as soon as that warpgroup's tile i - 2 has left its buffers, i.e.
      // while the other warpgroup runs tile i - 1's main loop, well before tile i's epilogue needs them
      const int pt = tid - 32;
      // the GELU epilogue computes x / 2 (gelu_erf_half's argument): the bias (c2) and the rows' rstd, -mu rstd are staged
      // halved, which leaves every rounding of the bias / folded-LayerNorm FMAs as it is, halved
      constexpr float HALF = ACT == ACT_GELU ? 0.5f : 1.f;
      int i = 0;
      for (long long t = blockIdx.x; t < tiles; t += gridDim.x, ++i) {
        const int w = i & 1;
        const int n0 = static_cast<int>(t % n_tiles) * BN;
        const int m0 = static_cast<int>(t / n_tiles) * BM;
        mbar_wait(epi_empty(w), ((i >> 1) & 1) ^ 1);
        if (RES && pt == 0) {
          // rows >= M are zero-filled; N % 64 == 0, so a 64-column half is entirely in or out
          const int halves = (N - n0 >= BN ? BN : N - n0) / 64;
          const uint32_t stg = stg_base + w * STG_BYTES;
          fence_proxy_async_smem();
          mbar_expect_tx(epi_full(w), halves * HALF_BYTES);
          for (int c = 0; c < halves; ++c) tma_load_2d(stg + c * HALF_BYTES, &tmap_res, epi_full(w), n0 + 64 * c, m0);
        }
        float* const par = params + w * PARAM_FLOATS;
        for (int c = pt; c < BN; c += EPI_THREADS) {
          float b = 0.f, c1 = 0.f, s = 1.f;
          if (n0 + c < N) {
            if (EPI >= 1) b = __ldg(bias + n0 + c);
            if (EPI == 2) c1 = __ldg(ln_c1 + n0 + c);
            if (scale != nullptr) s = __ldg(scale + n0 + c);
          }
          par[c] = b * HALF;
          par[BN + c] = c1;
          par[2 * BN + c] = s;
        }
        // folded LayerNorm of the A operand: y = rstd * acc + (-rstd * mu) * c1[n] + c2[n]   (c2 arrives through `bias`); the
        // rows' statistics arrive as `ln_parts` (sum, sumsq) partials [part][M], reduced in a fixed order
        if (EPI == 2) {
          for (int r = pt; r < BM; r += EPI_THREADS) {
            const int m = m0 + r;
            float rstd = 0.f, nmr = 0.f;
            if (m < M) {
              float s1 = 0.f, s2 = 0.f;
#pragma unroll 4
              for (int p = 0; p < ln_parts; ++p) {
                const float2 v = __ldg(ln_stats + static_cast<size_t>(p) * M + m);
                s1 += v.x;
                s2 += v.y;
              }
              const float mu = s1 * ln_inv_d;
              rstd = rsqrtf(fmaxf(fmaf(s2, ln_inv_d, -__fmul_rn(mu, mu)), 0.f) + ln_eps);
              nmr = -mu * rstd;
            }
            par[3 * BN + r] = rstd * HALF;
            par[3 * BN + BM + r] = nmr * HALF;
          }
        }
        mbar_arrive(epi_full(w));
      }
    }
    return;
  }

  // ===================================================================== consumers
  setmaxnreg_inc<CONSUMER_REGS>();
  const int cw = wg - 1;                                           // takes the CTA's tiles i = cw (mod 2)
  const int warp = tid >> 5, lane = tid & 31;
  const int col_t = 2 * (lane & 3);
  // Named barrier 1 + w: warpgroup w waits there for its turn at the main loop, which the other warpgroup hands over
  // (bar.arrive) when it has issued its own.  The turns alternate, so the ring's k-blocks are consumed in the order the
  // producer fills them and a warpgroup never waits on a stage more than one ring lap ahead of the producer.
  const uint32_t my_turn = 1 + cw, other_turn = 2 - cw, epi_done = 3 + cw;
  const float* const par = params + cw * PARAM_FLOATS;
  uint8_t* const stg = smem + STAGES * STAGE_BYTES + cw * STG_BYTES;
  const int row_l = warp * 16 + (lane >> 2);                       // this thread's accumulator rows in the tile: row_l +
                                                                   // 64 hm + 8 h; all = lane / 4 (mod 8)
  int stage = 0;
  uint32_t phase = 0, epi_phase = 0;
  ring_advance<STAGES>(stage, phase, cw * num_kb);                 // warpgroup 1 starts after tile 0's k-blocks
  // the dropout key and draw counter, read after griddepcontrol.wait (the kernel that advances the counter has completed)
  unsigned long long drop_seed = 0;
  uint32_t drop_d = 0;
  if constexpr (DROP != DROP_NONE) { drop_seed = drop_state[0]; drop_d = static_cast<uint32_t>(drop_state[1]); }

  for (long long t = blockIdx.x + static_cast<long long>(cw) * gridDim.x; t < tiles; t += 2LL * gridDim.x) {
    const int n0 = static_cast<int>(t % n_tiles) * BN;
    const int m0 = static_cast<int>(t / n_tiles) * BM;

    // the CTA's first tile starts at once
    if (cw == 1 || t != blockIdx.x) named_bar_sync(my_turn, 256);
    float acc[2][BN / 2];                                          // [64-row half of the tile][wgmma fragment]
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    wgmma_fence_operand(acc[0]);
    wgmma_fence_operand(acc[1]);
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * STAGE_BYTES;
      const uint64_t da = make_wgmma_desc_sw128(sa);
      const uint64_t db = make_wgmma_desc_sw128(sa + A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // advance 16 bf16 = 32 bytes along K inside the 128-byte swizzle row: +2 in the 16-byte address field; rows 64-127
        // start 64 x 128 bytes = +512 further
        const uint32_t acc_on = (kb | k) != 0 ? 1u : 0u;
        if constexpr (BN == 128) {
          wgmma_m64n128k16_bf16(acc[0], da + 2u * k, db + 2u * k, acc_on);
          wgmma_m64n128k16_bf16(acc[1], da + 512u + 2u * k, db + 2u * k, acc_on);
        } else {
          wgmma_m64n192k16_bf16(acc[0], da + 2u * k, db + 2u * k, acc_on);
          wgmma_m64n192k16_bf16(acc[1], da + 512u + 2u * k, db + 2u * k, acc_on);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                             // the previous k-block's products have retired
      if (kb > 0 && tid == 0) mbar_arrive(empty_bar(stage == 0 ? STAGES - 1 : stage - 1));
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if (t + gridDim.x < tiles) named_bar_arrive(other_turn, 256);  // the CTA's next tile may start its main loop
    wgmma_wait<0>();
    wgmma_fence_operand(acc[0]);
    wgmma_fence_operand(acc[1]);
    if (tid == 0) mbar_arrive(empty_bar(stage == 0 ? STAGES - 1 : stage - 1));
    ring_advance<STAGES>(stage, phase, num_kb);                    // skip the other warpgroup's tile

    // =================================================================== epilogue, 64-column chunks
    mbar_wait(epi_full(cw), epi_phase);                            // operands (and residual tile) staged by warps 1-3
    epi_phase ^= 1;
    // The tile in groups of 8 accumulators per thread: two 8-column blocks jj = 2 jp, 2 jp + 1 of one 64-column chunk c, in
    // the rows row_l + 64 hm + 8 h (h = 0, 1) of one 64-row half hm.  A group's 8 elements are independent from the
    // accumulator to the store, so the activation's dependent chains (about eight FP32 operations and one MUFU each) overlap
    // each other, and the group leaves as the four 8 x 8 matrices of one stmatrix.x4 (its residual arrives by the matching
    // ldmatrix.x4).  The halves go one after the other, so only their two rows' LayerNorm terms are held in registers.
    // LEAN: neither LayerScale nor row statistics, decided once per tile instead of paying a multiply by 1 and the
    // predicated statistics on every element (fc1 and to_qkv run LEAN).
    auto epilogue = [&](auto lean) {
      constexpr bool LEAN = decltype(lean)::value;
      const bool has_scale = !LEAN && scale != nullptr, has_stats = !LEAN && stats_out != nullptr;
#pragma unroll
      for (int hm = 0; hm < 2; ++hm) {
        float ln_rstd[2] = {0.f, 0.f}, ln_nmr[2] = {0.f, 0.f};   // rows row_l + 64 hm + 8 h
        if (EPI == 2) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            ln_rstd[h] = par[3 * BN + row_l + 64 * hm + 8 * h];
            ln_nmr[h] = par[3 * BN + BM + row_l + 64 * hm + 8 * h];
          }
        }
#pragma unroll
        for (int c = 0; c < BN / 64; ++c) {
          const int nc = n0 + c * 64;
          if (nc >= N) break;                                      // N % 64 == 0: a chunk is entirely in or out
          float st1[2] = {0.f, 0.f}, st2[2] = {0.f, 0.f};          // (sum, sumsq) of the stored bf16 outputs, per row
          // the staging tile in TMA's 128B-swizzled layout: 16-byte chunk k of row r at chunk k ^ (r % 8), so the 8 rows a
          // matrix's lanes address hit 8 distinct 16-byte bank groups.  Lane t addresses row t % 8 of matrix i = t / 8 of a
          // group: row warp 16 + 64 hm + 8 (i % 2) + t % 8, 16-byte chunk 2 jp + i / 2, so r[i] holds (h, jj) = (i % 2, 2 jp + i / 2)
          const uint32_t rows = smem_u32(stg) + c * HALF_BYTES + (warp * 16 + 64 * hm + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128;
          const uint32_t swz = (lane >> 4) ^ (lane & 7);
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            float v[4][2];                                         // [i = 2 u + h][column 0 / 1]
#pragma unroll
            for (int u = 0; u < 2; ++u) {                          // columns (2 jp + u) 8 + col_t, + 1 of the chunk
              const int cn = c * 64 + (2 * jp + u) * 8 + col_t;
              float cb[2] = {0.f, 0.f}, c1[2] = {0.f, 0.f};
              if (EPI >= 1) { const float2 b2 = *reinterpret_cast<const float2*>(par + cn); cb[0] = b2.x; cb[1] = b2.y; }
              if (EPI == 2) { const float2 c2 = *reinterpret_cast<const float2*>(par + BN + cn); c1[0] = c2.x; c1[1] = c2.y; }
#pragma unroll
              for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  float x = acc[hm][4 * (c * 8 + 2 * jp + u) + 2 * h + e];
                  if (EPI == 2) x = fmaf(x, ln_rstd[h], fmaf(c1[e], ln_nmr[h], cb[e]));
                  else if (EPI == 1) x = ACT == ACT_GELU ? fmaf(x, 0.5f, cb[e]) : x + cb[e];
                  else if (ACT == ACT_GELU) x *= 0.5f;
                  v[2 * u + h][e] = x;
                }
              }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (ACT == ACT_GELU) v[i][e] = gelu_erf_half(v[i][e]);   // of 2 v: see the staging of par
                if (ACT == ACT_HSWISH) v[i][e] = hard_swish(v[i][e]);
                if (ACT == ACT_SILU) v[i][e] = silu(v[i][e]);
              }
            }
            // the group's two 2 x 2 fragments (columns u = 0, 1) are one Philox block each: words 2 h + e
            auto drop_mask = [&]() {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                const uint4 x = dropout_block(drop_seed, drop_d, drop_site, static_cast<uint32_t>(m0 + row_l + 64 * hm),
                                              static_cast<uint32_t>(nc + (2 * jp + u) * 8 + col_t));
                const uint32_t wd[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                  for (int e = 0; e < 2; ++e)
                    v[2 * u + h][e] = dropout_keep(wd[2 * h + e], drop_rate) ? v[2 * u + h][e] * drop_scale : 0.f;
              }
            };
            if constexpr (DROP == DROP_BEFORE_RES) drop_mask();
            if (has_scale) {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                const float2 s2 = *reinterpret_cast<const float2*>(par + 2 * BN + c * 64 + (2 * jp + u) * 8 + col_t);
                // rounded on its own, as the reference's LayerScale is, never fused with the residual add into one FMA
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  v[2 * u + h][0] = __fmul_rn(v[2 * u + h][0], s2.x);
                  v[2 * u + h][1] = __fmul_rn(v[2 * u + h][1], s2.y);
                }
              }
            }
            if (OF32) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int rl = row_l + 64 * hm + 8 * (i & 1);
                if (m0 + rl < M)
                  *reinterpret_cast<float2*>(out_f32 + static_cast<size_t>(m0 + rl) * ldc + nc + (2 * jp + (i >> 1)) * 8 + col_t) =
                      make_float2(v[i][0], v[i][1]);
              }
            } else {
              const uint32_t addr = rows + (((2u * jp) ^ swz) << 4);
              uint32_t r[4];
              // the residual (zero in rows >= M, which the store clips) is read here and overwritten by the output, by the
              // same warp
              if (RES) ldmatrix_x4(addr, r);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                if (RES) {
                  v[i][0] += bf16_lo(r[i]);
                  v[i][1] += bf16_hi(r[i]);
                }
              }
              if constexpr (DROP == DROP_AFTER_RES) drop_mask();
#pragma unroll
              for (int i = 0; i < 4; ++i) r[i] = pack_bf16x2(v[i][0], v[i][1]);
              stmatrix_x4(addr, r);
              if (has_stats) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const float a0 = bf16_lo(r[i]), a1 = bf16_hi(r[i]);
                  st1[i & 1] += a0 + a1;
                  st2[i & 1] = fmaf(a0, a0, fmaf(a1, a1, st2[i & 1]));
                }
              }
            }
          }
          if (has_stats) {                                         // the row's 64 columns are spread over the 4 lanes of a quad
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              st1[h] += __shfl_xor_sync(0xffffffffu, st1[h], 1);
              st2[h] += __shfl_xor_sync(0xffffffffu, st2[h], 1);
              st1[h] += __shfl_xor_sync(0xffffffffu, st1[h], 2);
              st2[h] += __shfl_xor_sync(0xffffffffu, st2[h], 2);
              const int r = m0 + row_l + 64 * hm + 8 * h;
              if ((lane & 3) == 0 && r < M) stats_out[static_cast<size_t>(nc >> 6) * M + r] = make_float2(st1[h], st2[h]);   // [part][M]
            }
          }
        }
      }
    };
    if constexpr (OF32) epilogue(std::true_type{});
    else if (scale == nullptr && stats_out == nullptr) epilogue(std::true_type{});
    else epilogue(std::false_type{});
    // The staged bf16 tile leaves by TMA (rows >= M clipped); once it has been read out, the buffers go back to warps 1-3.
    // `res` may alias `out`: the tile's residual was loaded before this store, and no other tile touches these elements.
    if (!OF32) fence_proxy_async_smem();
    named_bar_sync(epi_done, 128);
    if (tid == 0) {
      if (!OF32) {
        const uint32_t s = stg_base + cw * STG_BYTES;
#pragma unroll
        for (int c = 0; c < BN / 64; ++c)
          if (n0 + 64 * c < N) tma_store_2d(&tmap_out, s + c * HALF_BYTES, n0 + 64 * c, m0);
        bulk_commit_group();
        // the CTA's stores are complete before it exits (a dependent kernel's griddepcontrol.wait waits for the grid's
        // exit only): after its last tile the warpgroup waits for the store's writes, not just its reads.  (Waiting after
        // the loop instead costs the 192-wide instances their registers: ptxas then spills the accumulators.)
        if (t + 2LL * gridDim.x < tiles) bulk_wait_group_read<0>();
        else bulk_wait_group<0>();
      }
      mbar_arrive(epi_empty(cw));
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static const EncodeTiledFn fn = [] {             // C++11 magic static: initialised once, thread-safe
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    VB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    VB_CHECK(p != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available from the driver");
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

template <int BN, int ACT, bool RES, int EPI, bool OF32 = false, int DROP = DROP_NONE>
void launch(const GemmBf16& g, cudaStream_t stream) {
  auto kern = gemm_bf16_kernel<BN, ACT, RES, EPI, OF32, DROP>;
  constexpr int smem = Tile<BN>::SMEM_BYTES;
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long tiles = static_cast<long long>((g.N + BN - 1) / BN) * ((g.M + BM - 1) / BM);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(tiles < sm_count() ? tiles : sm_count()));
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VB_CUDA(cudaLaunchKernelEx(&cfg, kern, g.tmap_a, g.tmap_b, g.tmap_out, g.tmap_res, g.M, g.N, g.K,
                             OF32 ? reinterpret_cast<float*>(g.out) : nullptr, g.ldc, g.bias, g.scale, g.ln_c1,
                             reinterpret_cast<const float2*>(g.ln_stats), g.ln_parts, g.ln_inv_d, g.ln_eps,
                             reinterpret_cast<float2*>(g.stats_out), g.drop.state, static_cast<uint32_t>(g.drop.site), g.drop.rate,
                             g.drop.scale));
  count_launch();
}

template <int BN>
void dispatch(const GemmBf16& g, bool res, int epi, cudaStream_t stream) {
  if constexpr (BN == 128) {                                          // fp32 output: 128-wide only (gemm_bf16_plan)
    if (g.out_f32) {
      if (epi == 0) return launch<BN, ACT_NONE, false, 0, true>(g, stream);
      return launch<BN, ACT_NONE, false, 1, true>(g, stream);
    }
  }
  VB_CHECK(!g.out_f32, "gemm_bf16: fp32 output runs the 128-wide tile only");
  VB_CHECK(g.drop.pos == DROP_NONE || BN == 128, "gemm_bf16: dropout runs the 128-wide tile only");
  if constexpr (BN == 128) if (g.drop.pos != DROP_NONE) {              // the dropout sites of ViT / DeepViT / CaiT / CrossViT
#define VB_GEMM_DROP(A, R, E, D) if (g.act == A && res == R && epi == E && g.drop.pos == D) return launch<BN, A, R, E, false, D>(g, stream)
    VB_GEMM_DROP(ACT_NONE, true, 1, DROP_BEFORE_RES);                   // to_out, fc2 (+ residual)
    VB_GEMM_DROP(ACT_NONE, false, 1, DROP_BEFORE_RES);                  // CrossViT's projected to_out
    VB_GEMM_DROP(ACT_GELU, false, 1, DROP_BEFORE_RES);                  // fc1 + GELU
    VB_GEMM_DROP(ACT_GELU, false, 2, DROP_BEFORE_RES);                  // fc1 + GELU, LayerNorm folded
    VB_GEMM_DROP(ACT_NONE, true, 1, DROP_AFTER_RES);                    // patch embedding + positions
#undef VB_GEMM_DROP
    VB_CHECK(false, "gemm_bf16: no dropout instance for this epilogue (activation " + std::to_string(g.act) + ")");
  }
#define VB_GEMM_CASE(A, R, E) if (g.act == A && res == R && epi == E) return launch<BN, A, R, E>(g, stream)
  VB_GEMM_CASE(ACT_NONE, false, 0); VB_GEMM_CASE(ACT_NONE, false, 1); VB_GEMM_CASE(ACT_NONE, false, 2);
  VB_GEMM_CASE(ACT_GELU, false, 0); VB_GEMM_CASE(ACT_GELU, false, 1); VB_GEMM_CASE(ACT_GELU, false, 2);
  VB_GEMM_CASE(ACT_NONE, true, 0);  VB_GEMM_CASE(ACT_NONE, true, 1);  VB_GEMM_CASE(ACT_NONE, true, 2);
  VB_GEMM_CASE(ACT_GELU, true, 0);  VB_GEMM_CASE(ACT_GELU, true, 1);  VB_GEMM_CASE(ACT_GELU, true, 2);
  VB_GEMM_CASE(ACT_HSWISH, false, 1);                                  // LeViT MLP fc1 (levit.py:53-54)
  VB_GEMM_CASE(ACT_SILU, false, 1);                                    // MobileViT Conv_NxN_BN, MV2 expand (mobile_vit.py:41-45,152-155)
  VB_GEMM_CASE(ACT_SILU, false, 2);                                    // MobileViT MLP fc1, LayerNorm folded (mobile_vit.py:67-70)
#undef VB_GEMM_CASE
  VB_CHECK(false, "gemm_bf16: no kernel instance for this epilogue (activation " + std::to_string(g.act) + ")");
}

}  // namespace

int sm_count() {                                  // of the CURRENT device (one process may hold handles on several GPUs)
  static int n[64] = {0};
  int dev = 0;
  VB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(global_cache_mutex());
  int& v = n[dev & 63];
  if (v == 0) VB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
  return v;
}

CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes, uint32_t box_inner,
                         uint32_t box_outer, bool swizzle128, bool f32) {
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {outer_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(&m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(2d) failed with CUresult " + std::to_string(static_cast<int>(r)));
  return m;
}

CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes, uint64_t stride2_bytes,
                         uint32_t box0, uint32_t box1) {
  CUtensorMap m;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(3d) failed with CUresult " + std::to_string(static_cast<int>(r)));
  return m;
}

bool gemm_bf16_supported(int M, int N, int K, int lda, int ldw, int ldc) {
  return M > 0 && N > 0 && K > 0 && (N % 64 == 0) && (K % 8 == 0) && (lda % 8 == 0) && (ldw % 8 == 0) && (ldc % 8 == 0);
}

GemmBf16 gemm_bf16_plan(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, __nv_bfloat16* out, int ldc, int M,
                        int N, int K, const float* bias, const float* scale, const __nv_bfloat16* res, int ldr, int act,
                        bool out_f32, int b_rows, bool dropout) {
  VB_CHECK(gemm_bf16_supported(M, N, K, lda, ldw, ldc), "gemm_bf16: unsupported shape (need N%64==0, K%8==0, ld%8==0)");
  VB_CHECK(res == nullptr || ldr % 8 == 0, "gemm_bf16: residual leading dimension must be a multiple of 8");
  VB_CHECK((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Wt) | reinterpret_cast<uintptr_t>(out) |
            reinterpret_cast<uintptr_t>(res)) % 16 == 0, "gemm_bf16: operands must be 16-byte aligned");
  GemmBf16 g;
  g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.scale = scale; g.res = res; g.ldr = ldr; g.act = act;
  g.out = out; g.ldc = ldc; g.out_f32 = out_f32;
  // The wider tile where it covers N exactly (no half-empty last column of tiles) in at least 8 column tiles.  Measured on
  // an H100 at ViT-B/16's shapes, it takes N = 2304 / 3072 at K = 768 from 0.320 / 0.448 ms to 0.281 / 0.423-0.433, but
  // N = 768 (4 column tiles) runs no faster at K = 768 and 3 % slower at K = 3072, so those keep the 128-wide tile.
  // An fp32 output (the classifier heads) keeps it too: its 64-bit row addresses next to 192 accumulators make ptxas spill; so
  // does a dropout epilogue, whose Philox rounds need registers beyond the 232 the 192 accumulators leave.
  g.bn = N % 192 == 0 && N >= 8 * 192 && !out_f32 && !dropout ? 192 : 128;
  g.tmap_a = make_tmap_2d(A, K, M, static_cast<uint64_t>(lda) * 2, BK, BM);
  // b_rows: rows of Wt that exist (< N when the output is column-padded: TMA zero-fills the rest instead of reading on)
  g.tmap_b = make_tmap_2d(Wt, K, b_rows > 0 ? b_rows : N, static_cast<uint64_t>(ldw) * 2, BK, g.bn);
  // bf16 output and residual tiles move as 64-column halves; TMA clips the store and zero-fills the load past row M
  if (!out_f32) g.tmap_out = make_tmap_2d(out, N, M, static_cast<uint64_t>(ldc) * 2, 64, BM);
  if (res != nullptr) g.tmap_res = make_tmap_2d(res, N, M, static_cast<uint64_t>(ldr) * 2, 64, BM);
  return g;
}

void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream) {
  const bool res = g.res != nullptr;
  const int epi = g.ln_c1 != nullptr ? 2 : g.bias != nullptr ? 1 : 0;
  VB_CHECK(epi != 2 || (g.bias != nullptr && g.ln_stats != nullptr && g.ln_parts > 0), "folded LayerNorm needs c1, c2 and the row statistics");
  if (g.out_f32)
    VB_CHECK(g.act == ACT_NONE && !res && epi != 2 && g.scale == nullptr && g.stats_out == nullptr, "fp32-output GEMM: plain or bias epilogue only");
  if (g.bn == 192) return dispatch<192>(g, res, epi, stream);
  VB_CHECK(g.bn == 128, "gemm_bf16: tile width " + std::to_string(g.bn) + " has no kernel");
  dispatch<128>(g, res, epi, stream);
}

}  // namespace vb
