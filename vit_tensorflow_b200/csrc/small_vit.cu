// Shifted patch tokens (vit_for_small_dataset.py:15-47, 142-157) on the device: the image is read once and the five views of
// SPT's channel concat -- the image and its four one-pixel shifts with zero fill -- are formed on the fly while the patch rows
// are written.  See kernels.cuh for the layout.
#include "kernels.cuh"

namespace vb {
namespace {

// element k of patch row t of image b (t >= 1, k < 5 C p^2)
__device__ __forceinline__ float spt_value(const float* __restrict__ img, long long b, int t, int k, int H, int W, int C, int p, int gw) {
  const int c = k % C, rest = k / C, view = rest % 5, pix = rest / 5;
  int y = ((t - 1) / gw) * p + pix / p, x = ((t - 1) % gw) * p + pix % p;
  // shift() order (:21-45): width +1, width -1, height +1, height -1
  if (view == 1) --x;
  else if (view == 2) ++x;
  else if (view == 3) --y;
  else if (view == 4) ++y;
  return (y >= 0 && y < H && x >= 0 && x < W) ? __ldg(img + ((b * H + y) * W + x) * C + c) : 0.f;
}

// One thread per VEC consecutive columns of a row (VEC = 8: one 16-byte bf16 store, two fp32 ones; ldo % 8 == 0)
template <typename T, int VEC>
__global__ void spt_rows_kernel(const float* __restrict__ img, T* __restrict__ out, int B, int H, int W, int C, int p, int ldo) {
  const int gw = W / p, rows = 1 + (H / p) * gw, kd = 5 * C * p * p, chunks = ldo / VEC;
  const long long total = static_cast<long long>(B) * rows * chunks;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / chunks;
    const int k0 = static_cast<int>(e - r * chunks) * VEC, t = static_cast<int>(r % rows);
    const long long b = r / rows;
    float v[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i)                            // the cls row and the pad columns stay zero
      v[i] = (t > 0 && k0 + i < kd) ? spt_value(img, b, t, k0 + i, H, W, C, p, gw) : 0.f;
    T* dst = out + r * ldo + k0;
    if constexpr (VEC == 8 && sizeof(T) == 2) {
      uint4 u;
      uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<const uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(dst) = u;
    } else if constexpr (VEC == 8) {
      reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) dst[i] = static_cast<T>(v[i]);
    }
  }
}

}  // namespace

template <typename T>
void spt_rows(const float* img, T* out, int B, int H, int W, int C, int p, int ldo, cudaStream_t s) {
  VB_CHECK(p > 0 && H % p == 0 && W % p == 0 && ldo >= 5 * C * p * p, "spt_rows: bad shape");
  const bool vec = ldo % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
  const long long total = static_cast<long long>(B) * (1 + static_cast<long long>(H / p) * (W / p)) * (vec ? ldo / 8 : ldo);
  const long long g = (total + 255) / 256, cap = static_cast<long long>(sm_count()) * 16;
  const unsigned grid = static_cast<unsigned>(g < 1 ? 1 : (g > cap ? cap : g));
  if (vec) spt_rows_kernel<T, 8><<<grid, 256, 0, s>>>(img, out, B, H, W, C, p, ldo);
  else spt_rows_kernel<T, 1><<<grid, 256, 0, s>>>(img, out, B, H, W, C, p, ldo);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

template void spt_rows<float>(const float*, float*, int, int, int, int, int, int, cudaStream_t);
template void spt_rows<__nv_bfloat16>(const float*, __nv_bfloat16*, int, int, int, int, int, int, cudaStream_t);

}  // namespace vb
