// Warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   out[M,N] (bf16) = epi( A[M,K] (bf16, K-major) x Wt[N,K]^T (bf16, K-major) ),  fp32 accumulation in registers
//   epi(v) = (+bias[n]) -> exact-erf GELU or hard-swish -> (*scale[n]) -> (+res[m,n])
//
// Replaces, on the reference's hot path, every nn.Dense: patch embedding (vit.py:143), to_qkv (vit.py:59,72),
// to_out + residual (vit.py:62-69,101), MLP fc1+GELU / fc2 + residual (vit.py:38-44,102), CaiT to_q/to_kv
// (cait.py:94-95) with LayerScale folded in (cait.py:48).
//
// Structure: persistent, one CTA of 384 threads per SM; CTA b computes the 128 x 128 output tiles b, b + gridDim.x, ...
// of the flat tile order (n fastest).
//   producer        warpgroup 0 (its registers handed to the consumers by setmaxnreg); one thread streams the A (128 x 64)
//                   and B (128 x 64) k-blocks of the CTA's tiles, one tile after the other, into a STAGES-deep ring of
//                   128B-swizzled tiles (mbarrier full / empty pairs).
//   2 consumer warpgroups, ping-pong: warpgroup w computes the CTA's tiles i = w (mod 2), each whole: two wgmma
//                   m64 x 128 x 16 per k16 step (rows 0-63 and 64-127 of the tile) into register accumulators, one k-block
//                   in flight while the previous one's stage is released; then the epilogue straight from the accumulator
//                   registers (bias / folded LayerNorm / GELU / LayerScale / residual, bf16 or fp32 stores, optional
//                   per-64-column row statistics of the stored values).  Two named barriers pass the main loop from one
//                   warpgroup to the other, so the main loops take turns on the tensor cores and one tile's epilogue
//                   runs under the next tile's main loop.
#include "common.h"
#include "kernels.cuh"
#include "ptx.cuh"

namespace vb {

namespace {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;             // 64 bf16 = 128 bytes = one swizzle row
constexpr int THREADS = 384;
constexpr int A_BYTES = BM * BK * 2;
constexpr int B_BYTES = BN * BK * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int STAGES = 6;          // 6 x 32 KB of the 227 KB a CTA may use
constexpr int COLS_BYTES = 2 * 3 * BN * 4;   // per consumer warpgroup: bias, ln_c1 and scale of its tile's columns
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 /*barriers*/ + COLS_BYTES + 1024 /*align*/;
static_assert(SMEM_BYTES <= 227 * 1024, "ring does not fit in shared memory");

// Exact-erf GELU (vit.py:34), written as  gelu(x) = x/2 - |x| * (E(|x|) - 1/2),  E(a) = erfc(a/sqrt2) / 2  (for x > 0
// this is x - x E, for x < 0 it is x E), with E evaluated as 2^q(a): q is a degree-5 polynomial (weighted minimax fit
// of log2(erfc(a/sqrt2)/2) on a in [0, 6], constant term exactly -1; tools/gelu_error.py refits and checks it).  Its
// leading coefficient is negative and q is monotone beyond the fit range, so no clamp is needed: for |x| > 6 the tail
// term |x| 2^q is below 6 * 2^-29 and shrinks.  Max abs error of the GELU 5.7e-7 = 0.003 bf16 ulp of the result for
// every finite x; gelu(+inf) = +inf and gelu(-inf) = NaN as in the reference's x * Phi(x).
__device__ __forceinline__ float gelu_erf(float x) {
  const float na = -fabsf(x);
  float q = fmaf(4.881368368e-04f, na, 7.198925130e-03f);          // odd coefficients negated: q(-na)
  q = fmaf(q, na, 5.214704946e-02f);
  q = fmaf(q, na, -4.595955014e-01f);
  q = fmaf(q, na, 1.151000619e+00f);
  q = fmaf(q, na, -1.0f);
  const float e = ex2_approx(q);                                     // erfc(|x|/sqrt2) / 2
  return fmaf(na, e + -0.5f, x * 0.5f);
}

// levit.py:37: x * relu6(x + 3) / 6, rounded in the reference's order
__device__ __forceinline__ float hard_swish(float x) { return __fdiv_rn(x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f), 6.0f); }

// Advance a ring position (stage, phase) by n k-blocks.
__device__ __forceinline__ void ring_advance(int& stage, uint32_t& phase, int n) {
  stage += n % STAGES;
  phase ^= static_cast<uint32_t>(n / STAGES) & 1u;
  if (stage >= STAGES) { stage -= STAGES; phase ^= 1u; }
}

// EPI: 0 = no per-column addend, 1 = + bias[n], 2 = folded LayerNorm (c1 = ln_c1, c2 = bias)
template <int ACT, bool RES, int EPI, bool OF32>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
                 void* __restrict__ out, int ldc, const float* __restrict__ bias, const float* __restrict__ scale,
                 const __nv_bfloat16* res, int ldr, const float* __restrict__ ln_c1, const float2* ln_stats, int ln_parts,
                 float ln_inv_d, float ln_eps, float2* __restrict__ stats_out) {
  static_assert(!OF32 || (ACT == ACT_NONE && !RES && EPI != 2), "fp32 output: plain / bias epilogue only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

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
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);                                  // released by the warpgroup that consumed the stage
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Everything above overlapped the previous kernel's tail (PDL); from here on we touch its outputs.
  pdl_wait();
  pdl_launch_dependents();

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<40>();
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
    }
    return;
  }

  // ===================================================================== consumers
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                                           // takes the CTA's tiles i = cw (mod 2)
  const int warp = tid >> 5, lane = tid & 31;
  const int col_t = 2 * (lane & 3);
  // Named barrier 1 + w: warpgroup w waits there for its turn at the main loop, which the other warpgroup hands over
  // (bar.arrive) when it has issued its own.  The turns alternate, so the ring's k-blocks are consumed in the order the
  // producer fills them and a warpgroup never waits on a stage more than one ring lap ahead of the producer.
  const uint32_t my_turn = 1 + cw, other_turn = 2 - cw, cols_ready = 3 + cw;
  // The tile's per-column epilogue parameters, staged in shared memory: loaded before the main loop, so the epilogue
  // does not wait on a global load for every 8 columns.
  float* cols = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - smem_u32(smem_raw))) + cw * 3 * BN;
  int stage = 0;
  uint32_t phase = 0;
  ring_advance(stage, phase, cw * num_kb);                         // warpgroup 1 starts after tile 0's k-blocks

  for (long long t = blockIdx.x + static_cast<long long>(cw) * gridDim.x; t < tiles; t += 2LL * gridDim.x) {
    const int n0 = static_cast<int>(t % n_tiles) * BN;
    const int m0 = static_cast<int>(t / n_tiles) * BM;
    const int row_a = m0 + warp * 16 + (lane >> 2);                // this thread's accumulator rows: row_a + 64 hm + 8 h,
                                                                   // q = 2 hm + h below

    // folded LayerNorm of the A operand: y = rstd * acc + (-rstd * mu) * c1[n] + c2[n]   (c2 arrives through `bias`); the
    // rows' statistics arrive as `ln_parts` (sum, sumsq) partials [part][M], reduced here in a fixed order while the other
    // warpgroup runs its main loop
    float ln_rstd[4] = {0.f, 0.f, 0.f, 0.f}, ln_nmr[4] = {0.f, 0.f, 0.f, 0.f};   // rows row_a + 64 (q / 2) + 8 (q % 2)
    if (EPI == 2) {
      float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int i = 0; i < ln_parts; ++i)                           // the four rows' loads in flight together
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = row_a + 64 * (q >> 1) + 8 * (q & 1);
          if (r < M) {
            const float2 v = __ldg(ln_stats + static_cast<size_t>(i) * M + r);
            s1[q] += v.x;
            s2[q] += v.y;
          }
        }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float mu = s1[q] * ln_inv_d;
        const float rstd = rsqrtf(fmaxf(s2[q] * ln_inv_d - mu * mu, 0.f) + ln_eps);
        ln_rstd[q] = rstd;
        ln_nmr[q] = -mu * rstd;
      }
    }

    float col_b = 0.f, col_c1 = 0.f, col_s = 1.f;
    if (n0 + tid < N) {
      if (EPI >= 1) col_b = __ldg(bias + n0 + tid);
      if (EPI == 2) col_c1 = __ldg(ln_c1 + n0 + tid);
      if (scale != nullptr) col_s = __ldg(scale + n0 + tid);
    }

    // the CTA's first tile starts at once; for the others, this also means the warpgroup's previous epilogue is done
    // with `cols`
    if (cw == 1 || t != blockIdx.x) named_bar_sync(my_turn, 256);
    float acc[2][64];                                              // [64-row half of the tile][wgmma fragment]
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
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
        wgmma_m64n128k16_bf16(acc[0], da + 2u * k, db + 2u * k, acc_on);
        wgmma_m64n128k16_bf16(acc[1], da + 512u + 2u * k, db + 2u * k, acc_on);
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
    ring_advance(stage, phase, num_kb);                            // skip the other warpgroup's tile
    cols[tid] = col_b;
    cols[BN + tid] = col_c1;
    cols[2 * BN + tid] = col_s;
    named_bar_sync(cols_ready, 128);

    // =================================================================== epilogue, 64-column chunks
#pragma unroll
    for (int c = 0; c < BN / 64; ++c) {
      const int nc = n0 + c * 64;
      if (nc >= N) break;                                          // N % 64 == 0: a chunk is entirely in or out
      float st1[4] = {0.f, 0.f, 0.f, 0.f}, st2[4] = {0.f, 0.f, 0.f, 0.f};   // (sum, sumsq) of the stored bf16 outputs, per row
      // The chunk's residuals, all loaded before its first store: one memory round trip instead of one per store.  `res`
      // may alias `out`; each element is still read before it is written, by the thread that writes it.
      uint32_t rw[8][4];
      if (RES) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int r = row_a + 64 * (q >> 1) + 8 * (q & 1);
            rw[jj][q] = r < M ? *reinterpret_cast<const uint32_t*>(res + static_cast<size_t>(r) * ldr + nc + jj * 8 + col_t) : 0u;
          }
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = c * 8 + jj;
        const int n = nc + jj * 8 + col_t;
        float cb0 = 0.f, cb1 = 0.f, c10 = 0.f, c11 = 0.f, sc0 = 1.f, sc1 = 1.f;
        if (EPI >= 1) { const float2 b2 = *reinterpret_cast<const float2*>(cols + (n - n0)); cb0 = b2.x; cb1 = b2.y; }
        if (EPI == 2) { const float2 c2 = *reinterpret_cast<const float2*>(cols + BN + (n - n0)); c10 = c2.x; c11 = c2.y; }
        if (scale != nullptr) { const float2 s2 = *reinterpret_cast<const float2*>(cols + 2 * BN + (n - n0)); sc0 = s2.x; sc1 = s2.y; }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = row_a + 64 * (q >> 1) + 8 * (q & 1);
          float v0 = acc[q >> 1][4 * j + 2 * (q & 1)], v1 = acc[q >> 1][4 * j + 2 * (q & 1) + 1];
          if (EPI == 2) {
            v0 = fmaf(v0, ln_rstd[q], fmaf(c10, ln_nmr[q], cb0));
            v1 = fmaf(v1, ln_rstd[q], fmaf(c11, ln_nmr[q], cb1));
          } else if (EPI == 1) {
            v0 += cb0;
            v1 += cb1;
          }
          if (ACT == ACT_GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
          if (ACT == ACT_HSWISH) { v0 = hard_swish(v0); v1 = hard_swish(v1); }
          // rounded on its own, as the reference's LayerScale is, never fused with the residual add into one FMA
          if (scale != nullptr) { v0 = __fmul_rn(v0, sc0); v1 = __fmul_rn(v1, sc1); }
          if (r >= M) continue;
          if (RES) {
            v0 += bf16_lo(rw[jj][q]);
            v1 += bf16_hi(rw[jj][q]);
          }
          if (OF32) {
            *reinterpret_cast<float2*>(static_cast<float*>(out) + static_cast<size_t>(r) * ldc + n) = make_float2(v0, v1);
          } else {
            const uint32_t pk = pack_bf16x2(v0, v1);
            *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(out) + static_cast<size_t>(r) * ldc + n) = pk;
            if (stats_out != nullptr) {
              const float a0 = bf16_lo(pk), a1 = bf16_hi(pk);
              st1[q] += a0 + a1;
              st2[q] = fmaf(a0, a0, fmaf(a1, a1, st2[q]));
            }
          }
        }
      }
      if (stats_out != nullptr) {                                  // the row's 64 columns are spread over the 4 lanes of a quad
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          st1[q] += __shfl_xor_sync(0xffffffffu, st1[q], 1);
          st2[q] += __shfl_xor_sync(0xffffffffu, st2[q], 1);
          st1[q] += __shfl_xor_sync(0xffffffffu, st1[q], 2);
          st2[q] += __shfl_xor_sync(0xffffffffu, st2[q], 2);
          const int r = row_a + 64 * (q >> 1) + 8 * (q & 1);
          if ((lane & 3) == 0 && r < M) stats_out[static_cast<size_t>(nc >> 6) * M + r] = make_float2(st1[q], st2[q]);   // [part][M]
        }
      }
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

template <int ACT, bool RES, int EPI, bool OF32 = false>
void launch(const GemmBf16& g, cudaStream_t stream) {
  auto kern = gemm_bf16_kernel<ACT, RES, EPI, OF32>;
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  const long long tiles = static_cast<long long>((g.N + BN - 1) / BN) * ((g.M + BM - 1) / BM);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(tiles < sm_count() ? tiles : sm_count()));
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VB_CUDA(cudaLaunchKernelEx(&cfg, kern, g.tmap_a, g.tmap_b, g.M, g.N, g.K, static_cast<void*>(g.out), g.ldc, g.bias, g.scale, g.res,
                             g.ldr, g.ln_c1, reinterpret_cast<const float2*>(g.ln_stats), g.ln_parts, g.ln_inv_d,
                             g.ln_eps, reinterpret_cast<float2*>(g.stats_out)));
  count_launch();
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
                        bool out_f32, int b_rows) {
  VB_CHECK(gemm_bf16_supported(M, N, K, lda, ldw, ldc), "gemm_bf16: unsupported shape (need N%64==0, K%8==0, ld%8==0)");
  VB_CHECK(res == nullptr || ldr % 8 == 0, "gemm_bf16: residual leading dimension must be a multiple of 8");
  VB_CHECK((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Wt) | reinterpret_cast<uintptr_t>(out) |
            reinterpret_cast<uintptr_t>(res)) % 16 == 0, "gemm_bf16: operands must be 16-byte aligned");
  GemmBf16 g;
  g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.scale = scale; g.res = res; g.ldr = ldr; g.act = act;
  g.out = out; g.ldc = ldc; g.out_f32 = out_f32;
  g.tmap_a = make_tmap_2d(A, K, M, static_cast<uint64_t>(lda) * 2, BK, BM);
  // b_rows: rows of Wt that exist (< N when the output is column-padded: TMA zero-fills the rest instead of reading on)
  g.tmap_b = make_tmap_2d(Wt, K, b_rows > 0 ? b_rows : N, static_cast<uint64_t>(ldw) * 2, BK, BN);
  return g;
}

void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream) {
  const bool res = g.res != nullptr;
  const int epi = g.ln_c1 != nullptr ? 2 : g.bias != nullptr ? 1 : 0;
  VB_CHECK(epi != 2 || (g.bias != nullptr && g.ln_stats != nullptr && g.ln_parts > 0), "folded LayerNorm needs c1, c2 and the row statistics");
  if (g.out_f32) {
    VB_CHECK(g.act == ACT_NONE && !res && epi != 2 && g.scale == nullptr && g.stats_out == nullptr, "fp32-output GEMM: plain or bias epilogue only");
    if (epi == 0) return launch<ACT_NONE, false, 0, true>(g, stream);
    return launch<ACT_NONE, false, 1, true>(g, stream);
  }
#define VB_GEMM_CASE(A, R, E) if (g.act == A && res == R && epi == E) return launch<A, R, E>(g, stream)
  VB_GEMM_CASE(ACT_NONE, false, 0); VB_GEMM_CASE(ACT_NONE, false, 1); VB_GEMM_CASE(ACT_NONE, false, 2);
  VB_GEMM_CASE(ACT_GELU, false, 0); VB_GEMM_CASE(ACT_GELU, false, 1); VB_GEMM_CASE(ACT_GELU, false, 2);
  VB_GEMM_CASE(ACT_NONE, true, 0);  VB_GEMM_CASE(ACT_NONE, true, 1);  VB_GEMM_CASE(ACT_NONE, true, 2);
  VB_GEMM_CASE(ACT_GELU, true, 0);  VB_GEMM_CASE(ACT_GELU, true, 1);  VB_GEMM_CASE(ACT_GELU, true, 2);
  VB_GEMM_CASE(ACT_HSWISH, false, 1);                                  // LeViT MLP fc1 (levit.py:53-54)
#undef VB_GEMM_CASE
  VB_CHECK(false, "gemm_bf16: no kernel instance for this epilogue (activation " + std::to_string(g.act) + ")");
}

}  // namespace vb
