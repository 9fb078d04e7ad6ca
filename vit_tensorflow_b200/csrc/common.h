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
//
// r2l_ws > 0 (RegionViT's regional-to-local attention, regionvit.py:143-155,168-169) replaces both: token 0 is the regional token
// and tokens 1 .. r2l_h * r2l_w the r2l_h x r2l_w local window, token t > 0 at (r, c) = ((t - 1) / r2l_w, (t - 1) % r2l_w).  For
// i, j > 0 head h adds
//   table[h * (2 ws - 1)^2 + (dr + ws - 1) * (2 ws - 1) + (dc + ws - 1)]     (ws = r2l_ws; r2l_h, r2l_w <= ws)
// and row 0 / column 0 get nothing.  The table is [heads][(2 ws - 1)^2], in the units of the scaled scores.  nq == nk == 1 + r2l_h r2l_w.
struct PosBias {
  const float* table = nullptr;
  int fmap = 0, step = 1;
  bool gelu_out = false;                  // levit.py:94: to_out starts with an exact-erf GELU of the attention output
  int wsz = 0;
  int r2l_ws = 0, r2l_h = 0, r2l_w = 0;
  __host__ __device__ int q_side() const { return (fmap + step - 1) / step; }
};
__host__ __device__ __forceinline__ int r2l_bias_index(int i, int j, int ww, int ws) {   // i, j > 0
  const int ri = (i - 1) / ww, ci = i - 1 - ri * ww, rj = (j - 1) / ww, cj = j - 1 - rj * ww;
  return (ri - rj + ws - 1) * (2 * ws - 1) + ci - cj + ws - 1;
}
__host__ __device__ __forceinline__ int window_bias_index(int i, int j, int wsz) {
  const int ri = i / wsz, rj = j / wsz;
  return (ri - rj + wsz - 1) * (2 * wsz - 1) + (i - ri * wsz) - (j - rj * wsz) + wsz - 1;
}
__device__ __forceinline__ int pos_bias_index(int i, int j, int fmap, int step, int nqs) {
  const int qr = (i / nqs) * step, qc = (i % nqs) * step, kr = j / fmap, kc = j - kr * fmap;
  return abs(qr - kr) * fmap + abs(qc - kc);
}
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Windowed attention on a pixel-major [B, H, W] map: each window of p x q tokens (p rows, q = width() columns) attends within
// itself.  The flat batch index of the attention is (image, window row, window column) over nx x ny windows (W = nx * q,
// H = ny * p), and token i < p q of window bw = (b, wy, wx), at (r, c) = (i / q, i % q) in the window, is the map's row
// (b * H + y) * W + x with
//   y = wy * oy + r * sy,  x = wx * ox + c * sx,
//   contiguous blocks (dilated == 0; Twins-SVT twins_svt.py:141, CrossFormer's short attention crossformer.py:144, NesT's
//   rectangular blocks nest.py:209):
//     oy = p, ox = q, sy = sx = 1;
//   dilated windows (dilated != 0; CrossFormer's long attention, crossformer.py:146 'b (l1 h) (l2 w) d -> (b h w) l1 l2 d', and
//   MobileViT's patch positions, mobile_vit.py:196 'b (h ph) (w pw) d -> b (ph pw) (h w) d' with p = h, q = w, ny = ph, nx = pw):
//     oy = ox = 1, sy = ny, sx = nx.
// nq == nk == p q.  pw == 0 means a square window (q = p): every caller but NesT's block attention and MobileViT's.
struct Window {
  int p = 0, nx = 0, ny = 0;
  int dilated = 0;
  int count = 0;                          // windows in the batch: the windowed-bias flash kernel packs several into one query tile
  int pw = 0;                             // the window's width q when it differs from p (NesT's rectangular blocks)
  __host__ __device__ int width() const { return pw > 0 ? pw : p; }
  __host__ __device__ long long row(long long bw, int i) const {
    const int q = width();
    const long long per = static_cast<long long>(nx) * ny, b = bw / per;
    const int w = static_cast<int>(bw - b * per), wy = w / nx, wx = w - wy * nx, r = i / q, c = i - r * q;
    const int oy = dilated ? 1 : p, sy = dilated ? ny : 1, ox = dilated ? 1 : q, sx = dilated ? nx : 1;
    return (b * ny * p + wy * oy + r * sy) * (static_cast<long long>(nx) * q) + wx * ox + c * sx;
  }
};

// 2-D bf16 (or fp32) tensor map (innermost dimension first), 128-byte swizzle unless swizzle128 == false.
CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                         uint32_t box_inner, uint32_t box_outer, bool swizzle128 = true, bool f32 = false);
// 3-D bf16 tensor map {d0, d1, d2} (innermost first; strides of d1 and d2 in bytes), box {box0, box1, 1}, 128-byte swizzle.
// Coordinates past d1 read as zero.
CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes, uint64_t stride2_bytes,
                         uint32_t box0, uint32_t box1);

// Activation of a GEMM epilogue: exact-erf GELU (vit.py:34), hard-swish x * relu6(x + 3) / 6 (levit.py:36-38) or SiLU / Keras
// swish x * sigmoid(x) (mobile_vit.py:33).  ACT_GELU is 1, so the `gelu` flags (bool / int 0-1) of the older entry points convert
// to it unchanged.
enum Act { ACT_NONE = 0, ACT_GELU = 1, ACT_HSWISH = 2, ACT_SILU = 3 };

#ifdef __CUDACC__
// SiLU, x * sigmoid(x) = x / (1 + e^-x), the one definition every kernel applying it uses (the GEMM epilogues, dwconv_bn_act).  The
// fast intrinsics: __expf is within 2 + 1.17 |x| ulp, __fdividef within 2 ulp while 1 + e^-x < 2^126 and 0 beyond (x < -87, where
// SiLU is below 1e-36); a few ulp of fp32 against bf16 storage or the fp32 engine's 1e-5 relative bound.  The IEEE expf and division
// add a slow path whose registers make the 192-wide LayerNorm-folded wgmma instance spill.
__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
#endif

// Training-mode dropout in a GEMM epilogue (philox.cuh dropout_block; include/vitb200.h states the stream): site `site` masks the
// [M, N] output at rate `rate` and scales the kept values by `scale` = fp32(1 / (1 - rate)).  DROP_BEFORE_RES masks after the
// activation, before LayerScale and the residual; DROP_AFTER_RES masks the sum.  state: the handle's {seed, draw counter} in
// device memory, read by the kernel.
enum DropPos { DROP_NONE = 0, DROP_BEFORE_RES = 1, DROP_AFTER_RES = 2 };
struct DropoutEpi {
  int pos = DROP_NONE;
  const unsigned long long* state = nullptr;
  int site = 0;
  float rate = 0.f, scale = 1.f;
};

// ------------------------------------------------------------------------------------------ wgmma GEMM
// out[M,N] = epilogue(A[M,K] * Wt[N,K]^T): bf16 operands (K-major), fp32 accumulation in registers.
// epilogue: (+bias[n]) -> (activation) -> (dropout) -> (*scale[n]) -> (+res[m,n]) -> (dropout); out bf16.
struct GemmBf16 {
  CUtensorMap tmap_a, tmap_b;           // A, B (weights)
  CUtensorMap tmap_out = {}, tmap_res = {};   // bf16 out and res, which the epilogue stores and loads by TMA
  int M = 0, N = 0, K = 0;
  int bn = 128;                         // tile width, 128 or 192 (gemm_bf16_plan's rule); the B tensor map's box follows it
  __nv_bfloat16* out = nullptr;         // [M, ldc] (fp32: stored straight from the accumulator registers)
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
  DropoutEpi drop;
};
// lda/ldw/ldc/ldr in elements; all must be multiples of 8 (16-byte TMA strides); N % 64 == 0.
GemmBf16 gemm_bf16_plan(const __nv_bfloat16* A, int lda, const __nv_bfloat16* Wt, int ldw, __nv_bfloat16* out, int ldc,
                        int M, int N, int K, const float* bias, const float* scale, const __nv_bfloat16* res, int ldr,
                        int act, bool out_f32 = false, int b_rows = 0, bool dropout = false);
void gemm_bf16_run(const GemmBf16& g, cudaStream_t stream);
bool gemm_bf16_supported(int M, int N, int K, int lda, int ldw, int ldc);

}  // namespace vb
