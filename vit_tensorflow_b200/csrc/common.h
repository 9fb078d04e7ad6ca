// Host-side common definitions for libvitb200: error plumbing, TMA tensor-map encoding, launch interfaces
// of the kernels (implemented in the .cu files of this directory).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <mutex>
#include <stdexcept>
#include <string>

namespace vb {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define VB_CUDA(expr)                                                                                   \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess)                                                                              \
      throw ::vb::Error(2, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" + __FILE__ + \
                               ":" + std::to_string(__LINE__) + ")");                                   \
  } while (0)

#define VB_CHECK(cond, msg)                                       \
  do {                                                            \
    if (!(cond)) throw ::vb::Error(1, std::string(msg));          \
  } while (0)

int sm_count();

// Kernel function attributes (opt-in shared memory) are per DEVICE, and one process may hold handles on several GPUs:
// true the first time the calling site runs on the current device.
// Thread-safe: distinct handles may be driven from distinct threads (include/vitb200.h), and every process-wide cache of
// this library (this bitmap, sm_count, the attention TMA-plan and head-mix caches) is guarded by a mutex.
inline std::mutex& global_cache_mutex() {
  static std::mutex m;
  return m;
}
inline bool first_use_on_this_device(unsigned long long (&seen)[4]) {
  std::lock_guard<std::mutex> lock(global_cache_mutex());
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return true;
  unsigned long long& word = seen[(dev >> 6) & 3];
  const unsigned long long bit = 1ull << (dev & 63);
  if (word & bit) return false;
  word |= bit;
  return true;
}

// Kernels whose grid counts images, rows or (image, head) items take their (tile, item) from a flat blockIdx.x, tile index
// fastest: gridDim.y and gridDim.z stop at 65 535, gridDim.x at 2^31 - 1.  The block count of such a grid, checked.
inline unsigned flat_blocks(long long tiles, long long items, const char* what = "attention") {
  const long long n = tiles * items;
  VB_CHECK(n > 0 && n <= 0x7fffffffLL, std::string(what) + ": grid of " + std::to_string(n) + " blocks exceeds 2^31 - 1");
  return static_cast<unsigned>(n);
}

// 2-D bf16 (or fp32) tensor map (innermost dimension first), 128-byte swizzle unless swizzle128 == false.
CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                         uint32_t box_inner, uint32_t box_outer, bool swizzle128 = true, bool f32 = false);

// ------------------------------------------------------------------------------------------ wgmma GEMM
// out[M,N] = epilogue(A[M,K] * Wt[N,K]^T): bf16 operands (K-major), fp32 accumulation in registers.
// epilogue: (+bias[n]) -> (exact-erf GELU) -> (*scale[n]) -> (+res[m,n]); out bf16.
struct GemmBf16 {
  CUtensorMap tmap_a, tmap_b;           // A, B (weights)
  int M = 0, N = 0, K = 0;
  __nv_bfloat16* out = nullptr;         // [M, ldc] (the epilogue stores rows straight from registers)
  int ldc = 0;
  bool out_f32 = false;                 // `out` is float* (ldc in floats): plain / bias epilogue only
  const float* bias = nullptr;          // [N] or null
  const float* scale = nullptr;         // [N] or null (LayerScale)
  const __nv_bfloat16* res = nullptr;   // [M, ldr] or null (may alias out)
  int ldr = 0;
  bool gelu = false;
  // Folded LayerNorm of the A operand (Wt must hold gamma-scaled weights, bias the beta.W + b term):
  //   out = rstd[m] * (acc - mu[m] * ln_c1[n]) + bias[n], with (mu, rstd) of row m reduced in the epilogue from the
  //   ln_parts (sum, sumsq) partials of that row (the stats_out format below) over 1 / ln_inv_d elements.
  const float* ln_c1 = nullptr;
  const float* ln_stats = nullptr;      // [ln_parts, M, 2]
  int ln_parts = 0;
  float ln_inv_d = 0.f;
  // Emit (sum, sumsq) of every 64-column chunk of the stored bf16 output rows: [N/64, M, 2]
  float* stats_out = nullptr;
};
// lda/ldw/ldc/ldr in elements; all must be multiples of 8 (16-byte TMA strides); N % 64 == 0.
GemmBf16 gemm_bf16_plan(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, __nv_bfloat16* out, int ldc,
                        int M, int N, int K, const float* bias, const float* scale, const __nv_bfloat16* res, int ldr,
                        bool gelu, bool out_f32 = false, int b_rows = 0);
void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream);
bool gemm_bf16_supported(int M, int N, int K, int lda, int ldw, int ldc);

}  // namespace vb
