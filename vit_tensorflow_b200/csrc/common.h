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

// LeViT attention (levit.py:100-117,94): an additive relative-position bias on the scores and GELU on the output rows.
//   score(b, h, i, j) += table[h * fmap^2 + |qr - kr| * fmap + |qc - kc|]
// with key j at grid position (kr, kc) = (j / fmap, j % fmap) and query i at (qr, qc) = step * (i / nqs, i % nqs), nqs =
// ceil(fmap / step): the queries of a stride-2 "shrink" attention sit on the even pixels of the key grid.  `table` is fp32
// [heads][fmap^2] in the units of the scaled scores (the reference adds pos_bias / scale, levit.py:117).  nk == fmap^2, nq == nqs^2.
//
// wsz > 0 (CrossFormer, crossformer.py:126-131,158-165) replaces that form: within a wsz x wsz window, token i at (i / wsz, i % wsz)
// and key j at (j / wsz, j % wsz) give the signed offsets (dr, dc), and every head adds
//   table[(dr + wsz - 1) * (2 wsz - 1) + (dc + wsz - 1)]
// from one shared fp32 table of (2 wsz - 1)^2 entries, in the units of the scaled scores.  nq == nk == wsz^2; fmap / step unused.
struct PosBias {
  const float* table = nullptr;
  int fmap = 0, step = 1;
  bool gelu_out = false;                  // levit.py:94: to_out starts with an exact-erf GELU of the attention output
  int wsz = 0;
  __host__ __device__ int q_side() const { return (fmap + step - 1) / step; }
};
__host__ __device__ __forceinline__ int window_bias_index(int i, int j, int wsz) {
  const int ri = i / wsz, rj = j / wsz;
  return (ri - rj + wsz - 1) * (2 * wsz - 1) + (i - ri * wsz) - (j - rj * wsz) + wsz - 1;
}
__device__ __forceinline__ int pos_bias_index(int i, int j, int fmap, int step, int nqs) {
  const int qr = (i / nqs) * step, qc = (i % nqs) * step, kr = j / fmap, kc = j - kr * fmap;
  return abs(qr - kr) * fmap + abs(qc - kc);
}
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Windowed attention on a pixel-major [B, H, W] map: each window of p x p tokens attends within itself.  The flat batch index of
// the attention is (image, window row, window column) over nx x ny windows (W = nx * p, H = ny * p), and token i < p^2 of window
// bw = (b, wy, wx), at (r, c) = (i / p, i % p) in the window, is the map's row (b * H + y) * W + x with
//   y = wy * oy + r * sy,  x = wx * ox + c * sx,
//   contiguous blocks (dilated == 0; Twins-SVT twins_svt.py:141, CrossFormer's short attention crossformer.py:144):
//     oy = ox = p, sy = sx = 1;
//   dilated windows (dilated != 0; CrossFormer's long attention, crossformer.py:146 'b (l1 h) (l2 w) d -> (b h w) l1 l2 d'):
//     oy = ox = 1, sy = ny, sx = nx.
// nq == nk == p^2.
struct Window {
  int p = 0, nx = 0, ny = 0;
  int dilated = 0;
  int count = 0;                          // windows in the batch: the windowed-bias flash kernel packs several into one query tile
  __host__ __device__ long long row(long long bw, int i) const {
    const long long per = static_cast<long long>(nx) * ny, b = bw / per;
    const int w = static_cast<int>(bw - b * per), wy = w / nx, wx = w - wy * nx, r = i / p, c = i - r * p;
    const int oy = dilated ? 1 : p, sy = dilated ? ny : 1, ox = dilated ? 1 : p, sx = dilated ? nx : 1;
    return (b * ny * p + wy * oy + r * sy) * (static_cast<long long>(nx) * p) + wx * ox + c * sx;
  }
};

// 2-D bf16 (or fp32) tensor map (innermost dimension first), 128-byte swizzle unless swizzle128 == false.
CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                         uint32_t box_inner, uint32_t box_outer, bool swizzle128 = true, bool f32 = false);
// 3-D bf16 tensor map {d0, d1, d2} (innermost first; strides of d1 and d2 in bytes), box {box0, box1, 1}, 128-byte swizzle.
// Coordinates past d1 read as zero.
CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes, uint64_t stride2_bytes,
                         uint32_t box0, uint32_t box1);

// Activation of a GEMM epilogue: exact-erf GELU (vit.py:34) or hard-swish x * relu6(x + 3) / 6 (levit.py:36-38).  ACT_GELU is 1,
// so the `gelu` flags (bool / int 0-1) of the older entry points convert to it unchanged.
enum Act { ACT_NONE = 0, ACT_GELU = 1, ACT_HSWISH = 2 };

// ------------------------------------------------------------------------------------------ wgmma GEMM
// out[M,N] = epilogue(A[M,K] * Wt[N,K]^T): bf16 operands (K-major), fp32 accumulation in registers.
// epilogue: (+bias[n]) -> (activation) -> (*scale[n]) -> (+res[m,n]); out bf16.
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
  int act = ACT_NONE;                   // Act
  // Folded LayerNorm of the A operand (Wt must hold gamma-scaled weights, bias the beta.W + b term):
  //   out = rstd[m] * (acc - mu[m] * ln_c1[n]) + bias[n], with (mu, rstd) of row m reduced in the epilogue from the
  //   ln_parts (sum, sumsq) partials of that row (the stats_out format below) over 1 / ln_inv_d elements, rstd =
  //   1 / sqrt(var + ln_eps) (Keras LayerNormalization: 1e-3; CvT's own LayerNorm: 1e-5).
  const float* ln_c1 = nullptr;
  const float* ln_stats = nullptr;      // [ln_parts, M, 2]
  int ln_parts = 0;
  float ln_inv_d = 0.f;
  float ln_eps = 1e-3f;
  // Emit (sum, sumsq) of every 64-column chunk of the stored bf16 output rows: [N/64, M, 2]
  float* stats_out = nullptr;
};
// lda/ldw/ldc/ldr in elements; all must be multiples of 8 (16-byte TMA strides); N % 64 == 0.
GemmBf16 gemm_bf16_plan(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, __nv_bfloat16* out, int ldc,
                        int M, int N, int K, const float* bias, const float* scale, const __nv_bfloat16* res, int ldr,
                        int act, bool out_f32 = false, int b_rows = 0);
void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream);
bool gemm_bf16_supported(int M, int N, int K, int lda, int ldw, int ldc);

}  // namespace vb
