// Warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   out[M,N] (bf16) = epi( A[M,K] (bf16, K-major) x Wt[N,K]^T (bf16, K-major) ),  fp32 accumulation in registers
//   epi(v) = (+bias[n]) -> exact-erf GELU -> (*scale[n]) -> (+res[m,n])
//
// Replaces, on the reference's hot path, every nn.Dense: patch embedding (vit.py:143), to_qkv (vit.py:59,72),
// to_out + residual (vit.py:62-69,101), MLP fc1+GELU / fc2 + residual (vit.py:38-44,102), CaiT to_q/to_kv
// (cait.py:94-95) with LayerScale folded in (cait.py:48).
//
// Structure: one CTA per 128 x BN output tile (flat grid, n fastest); BN = 128 tiles run two CTAs per SM (see Cfg).
//   producer        one thread streams A (128 x 64) and B (BN x 64) k-blocks into a STAGES-deep ring of 128B-swizzled
//                   tiles (mbarrier full / empty pairs).
//   2 consumer warpgroups, 64 rows each: wgmma m64 x BN x 16 from shared memory into register accumulators, one
//                   k-block in flight while the previous one's stage is released; then the epilogue straight from the
//                   accumulator registers (bias / folded LayerNorm / GELU / LayerScale / residual, bf16 or fp32 stores,
//                   optional per-64-column row statistics of the stored values).
#include "common.h"
#include "kernels.cuh"
#include "ptx.cuh"

namespace vb {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;             // 64 bf16 = 128 bytes = one swizzle row

// BN = 128 runs two CTAs per SM, so that one CTA's epilogue and pipeline fill overlap the other's main loop; BN = 256
// (128 fp32 accumulators per consumer thread) fills the register file with one CTA.
//   one CTA per SM:  warpgroup 0 is the producer (its registers handed to the consumers by setmaxnreg), 1-2 the consumers;
//   two CTAs per SM: warpgroups 0-1 are the consumers and a single warp 8 the producer, 288 threads at up to 96
//                    registers (ptxas holds the whole kernel to the launch-bound cap, and 384 threads x 2 CTAs would
//                    leave 80, too few for a 64-accumulator wgmma).
template <int BN>
struct Cfg {
  static constexpr int CTAS_PER_SM = BN == 128 ? 2 : 1;
  static constexpr int THREADS = CTAS_PER_SM == 1 ? 384 : 288;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // 228 KB of shared memory per SM, 1 KB of it reserved per CTA
  static constexpr int STAGES_FIT = ((228 * 1024) / CTAS_PER_SM - 1024 - 256 - 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;   // 3 x 32 KB (BN = 128), 4 x 48 KB (BN = 256)
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 /*barriers*/ + 1024 /*align*/;
};

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

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_m64n256k16_bf16(d, da, db, accumulate);
  else wgmma_m64n128k16_bf16(d, da, db, accumulate);
}

// EPI: 0 = no per-column addend, 1 = + bias[n], 2 = folded LayerNorm (c1 = ln_c1, c2 = bias)
template <int BN, bool GELU, bool RES, int EPI, bool OF32>
__global__ void __launch_bounds__(Cfg<BN>::THREADS, Cfg<BN>::CTAS_PER_SM)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N, int K,
                 void* __restrict__ out, int ldc, const float* __restrict__ bias, const float* __restrict__ scale,
                 const __nv_bfloat16* res, int ldr, const float* __restrict__ ln_c1, const float2* ln_stats, int ln_parts,
                 float ln_inv_d, float2* __restrict__ stats_out) {
  using C = Cfg<BN>;
  static_assert(!OF32 || (!GELU && !RES && EPI != 2), "fp32 output: plain / bias epilogue only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + C::STAGES * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  // flat grid, n fastest: the CTAs that share an A row block run together, and M is not bounded by gridDim.y's 65 535 tiles
  const int n_tiles = (N + BN - 1) / BN;
  const int n0 = static_cast<int>(blockIdx.x % n_tiles) * BN;
  const int m0 = static_cast<int>(blockIdx.x / n_tiles) * BM;
  const int num_kb = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);                                  // one release per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Everything above overlapped the previous kernel's tail (PDL); from here on we touch its outputs.
  pdl_wait();
  pdl_launch_dependents();

  if (wg == (C::CTAS_PER_SM == 1 ? 0 : 2)) {
    // ===================================================================== TMA producer
    if (C::CTAS_PER_SM == 1) setmaxnreg_dec<40>();
    if (tid == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1);
        const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
        mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);   // out-of-range box elements are zero-filled and counted
        tma_load_2d(sa, &tmap_a, full_bar(stage), kb * BK, m0);
        tma_load_2d(sa + C::A_BYTES, &tmap_b, full_bar(stage), kb * BK, n0);
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================================================================== consumers
  if (C::CTAS_PER_SM == 1) setmaxnreg_inc<232>();
  const int cw = C::CTAS_PER_SM == 1 ? wg - 1 : wg;                // 64-row half of the tile
  const int warp = tid >> 5, lane = tid & 31;
  const int row_a = m0 + cw * 64 + warp * 16 + (lane >> 2);        // this thread's two accumulator rows: row_a, row_a + 8
  const int col_t = 2 * (lane & 3);

  // folded LayerNorm of the A operand: y = rstd * acc + (-rstd * mu) * c1[n] + c2[n]   (c2 arrives through `bias`); the rows'
  // statistics arrive as `ln_parts` (sum, sumsq) partials [part][M], reduced here in a fixed order before the main loop
  float ln_rstd[2] = {0.f, 0.f}, ln_nmr[2] = {0.f, 0.f};
  if (EPI == 2) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_a + 8 * h;
      if (r < M) {
        float s1 = 0.f, s2 = 0.f;
        for (int i = 0; i < ln_parts; ++i) {
          const float2 v = __ldg(ln_stats + static_cast<size_t>(i) * M + r);
          s1 += v.x;
          s2 += v.y;
        }
        const float mu = s1 * ln_inv_d;
        const float rstd = rsqrtf(fmaxf(s2 * ln_inv_d - mu * mu, 0.f) + 1e-3f);
        ln_rstd[h] = rstd;
        ln_nmr[h] = -mu * rstd;
      }
    }
  }

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    int stage = 0;
    uint32_t phase = 0;
    wgmma_fence_operand(acc);
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
      const uint64_t da = make_wgmma_desc_sw128(sa + cw * 64 * 128);
      const uint64_t db = make_wgmma_desc_sw128(sa + C::A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        // advance 16 bf16 = 32 bytes along K inside the 128-byte swizzle row: +2 in the 16-byte address field
        wgmma_tile<BN>(acc, da + 2u * k, db + 2u * k, (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                                             // the previous k-block's products have retired
      if (kb > 0 && tid == 0) mbar_arrive(empty_bar(stage == 0 ? C::STAGES - 1 : stage - 1));
      if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    if (tid == 0) mbar_arrive(empty_bar(stage == 0 ? C::STAGES - 1 : stage - 1));
  }

  // ===================================================================== epilogue, 64-column chunks
#pragma unroll
  for (int c = 0; c < BN / 64; ++c) {
    const int nc = n0 + c * 64;
    if (nc >= N) break;                                            // N % 64 == 0: a chunk is entirely in or out
    float st1[2] = {0.f, 0.f}, st2[2] = {0.f, 0.f};                // (sum, sum of squares) of the stored bf16 outputs
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = c * 8 + jj;
      const int n = nc + jj * 8 + col_t;
      float cb0 = 0.f, cb1 = 0.f, c10 = 0.f, c11 = 0.f, sc0 = 1.f, sc1 = 1.f;
      if (EPI >= 1) { const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n)); cb0 = b2.x; cb1 = b2.y; }
      if (EPI == 2) { const float2 c2 = __ldg(reinterpret_cast<const float2*>(ln_c1 + n)); c10 = c2.x; c11 = c2.y; }
      if (scale != nullptr) { const float2 s2 = __ldg(reinterpret_cast<const float2*>(scale + n)); sc0 = s2.x; sc1 = s2.y; }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row_a + 8 * h;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (EPI == 2) {
          v0 = fmaf(v0, ln_rstd[h], fmaf(c10, ln_nmr[h], cb0));
          v1 = fmaf(v1, ln_rstd[h], fmaf(c11, ln_nmr[h], cb1));
        } else if (EPI == 1) {
          v0 += cb0;
          v1 += cb1;
        }
        if (GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
        if (scale != nullptr) { v0 *= sc0; v1 *= sc1; }
        if (r >= M) continue;
        if (RES) {
          const uint32_t w = *reinterpret_cast<const uint32_t*>(res + static_cast<size_t>(r) * ldr + n);   // may alias out
          v0 += bf16_lo(w);
          v1 += bf16_hi(w);
        }
        if (OF32) {
          *reinterpret_cast<float2*>(static_cast<float*>(out) + static_cast<size_t>(r) * ldc + n) = make_float2(v0, v1);
        } else {
          const uint32_t pk = pack_bf16x2(v0, v1);
          *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(out) + static_cast<size_t>(r) * ldc + n) = pk;
          if (stats_out != nullptr) {
            const float a0 = bf16_lo(pk), a1 = bf16_hi(pk);
            st1[h] += a0 + a1;
            st2[h] = fmaf(a0, a0, fmaf(a1, a1, st2[h]));
          }
        }
      }
    }
    if (stats_out != nullptr) {                                    // the row's 64 columns are spread over the 4 lanes of a quad
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        st1[h] += __shfl_xor_sync(0xffffffffu, st1[h], 1);
        st2[h] += __shfl_xor_sync(0xffffffffu, st2[h], 1);
        st1[h] += __shfl_xor_sync(0xffffffffu, st1[h], 2);
        st2[h] += __shfl_xor_sync(0xffffffffu, st2[h], 2);
        const int r = row_a + 8 * h;
        if ((lane & 3) == 0 && r < M) stats_out[static_cast<size_t>(nc >> 6) * M + r] = make_float2(st1[h], st2[h]);   // [part][M]
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

template <int BN, bool GELU, bool RES, int EPI, bool OF32 = false>
void launch(const GemmBf16& g, cudaStream_t stream) {
  auto kern = gemm_bf16_kernel<BN, GELU, RES, EPI, OF32>;
  static unsigned long long seen[4] = {0, 0, 0, 0};
  if (first_use_on_this_device(seen)) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM_BYTES));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(flat_blocks((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, "gemm_bf16"));
  cfg.blockDim = dim3(Cfg<BN>::THREADS);
  cfg.dynamicSmemBytes = Cfg<BN>::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VB_CUDA(cudaLaunchKernelEx(&cfg, kern, g.tmap_a, g.tmap_b, g.M, g.N, g.K, static_cast<void*>(g.out), g.ldc, g.bias, g.scale, g.res,
                             g.ldr, g.ln_c1, reinterpret_cast<const float2*>(g.ln_stats), g.ln_parts, g.ln_inv_d,
                             reinterpret_cast<float2*>(g.stats_out)));
  count_launch();
}

template <int BN>
void launch_epi(const GemmBf16& g, cudaStream_t stream) {
  const bool res = g.res != nullptr;
  const int epi = g.ln_c1 != nullptr ? 2 : g.bias != nullptr ? 1 : 0;
  VB_CHECK(epi != 2 || (g.bias != nullptr && g.ln_stats != nullptr && g.ln_parts > 0), "folded LayerNorm needs c1, c2 and the row statistics");
  if (g.out_f32) {
    VB_CHECK(!g.gelu && !res && epi != 2 && g.scale == nullptr && g.stats_out == nullptr, "fp32-output GEMM: plain or bias epilogue only");
    if (epi == 0) return launch<BN, false, false, 0, true>(g, stream);
    return launch<BN, false, false, 1, true>(g, stream);
  }
#define VB_GEMM_CASE(G, R, E) if (g.gelu == G && res == R && epi == E) return launch<BN, G, R, E>(g, stream)
  VB_GEMM_CASE(false, false, 0); VB_GEMM_CASE(false, false, 1); VB_GEMM_CASE(false, false, 2);
  VB_GEMM_CASE(true, false, 0);  VB_GEMM_CASE(true, false, 1);  VB_GEMM_CASE(true, false, 2);
  VB_GEMM_CASE(false, true, 0);  VB_GEMM_CASE(false, true, 1);  VB_GEMM_CASE(false, true, 2);
  VB_GEMM_CASE(true, true, 0);   VB_GEMM_CASE(true, true, 1);   VB_GEMM_CASE(true, true, 2);
#undef VB_GEMM_CASE
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

bool gemm_bf16_supported(int M, int N, int K, int lda, int ldw, int ldc) {
  return M > 0 && N > 0 && K > 0 && (N % 64 == 0) && (K % 8 == 0) && (lda % 8 == 0) && (ldw % 8 == 0) && (ldc % 8 == 0);
}

GemmBf16 gemm_bf16_plan(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, __nv_bfloat16* out, int ldc, int M,
                        int N, int K, const float* bias, const float* scale, const __nv_bfloat16* res, int ldr, bool gelu,
                        bool out_f32, int b_rows) {
  VB_CHECK(gemm_bf16_supported(M, N, K, lda, ldw, ldc), "gemm_bf16: unsupported shape (need N%64==0, K%8==0, ld%8==0)");
  VB_CHECK(res == nullptr || ldr % 8 == 0, "gemm_bf16: residual leading dimension must be a multiple of 8");
  VB_CHECK((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Wt) | reinterpret_cast<uintptr_t>(out) |
            reinterpret_cast<uintptr_t>(res)) % 16 == 0, "gemm_bf16: operands must be 16-byte aligned");
  GemmBf16 g;
  g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.scale = scale; g.res = res; g.ldr = ldr; g.gelu = gelu;
  g.out = out; g.ldc = ldc; g.out_f32 = out_f32;
  // Each tile pays a fixed cost (pipeline fill, epilogue) of about as much as a 12-k-block main loop.  128-wide tiles run
  // two CTAs per SM, so that cost overlaps the other CTA's main loop; 256-wide tiles (one CTA per SM, half the A re-reads)
  // are faster only once the main loop is long.  On an H100 (400 W) at M = 50 432: K = 768 128-wide 0.24-0.77 ms against
  // 0.28-0.90 ms 256-wide, K = 3072 (N = 768) 0.651 ms against 0.609 ms.
  g.block_n = (N % 256 == 0 && K >= 2048) ? 256 : 128;
  g.tmap_a = make_tmap_2d(A, K, M, static_cast<uint64_t>(lda) * 2, BK, BM);
  // b_rows: rows of Wt that exist (< N when the output is column-padded: TMA zero-fills the rest instead of reading on)
  g.tmap_b = make_tmap_2d(Wt, K, b_rows > 0 ? b_rows : N, static_cast<uint64_t>(ldw) * 2, BK, g.block_n);
  return g;
}

void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream) {
  if (g.block_n == 256) launch_epi<256>(g, stream); else launch_epi<128>(g, stream);
}

}  // namespace vb
