// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants): the counter-based generator behind every engine-defined noise
// stream (ATS-ViT's Gumbel-max draws, MAE / SimMIM's patch masks; include/vitb200.h states each stream's key and counter).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

}  // namespace vb
