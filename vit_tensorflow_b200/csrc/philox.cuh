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

// Training-mode dropout (include/vitb200.h states the stream): site s's element (m, n) of its [M, N] view, draw d, key = the 64-bit
// seed.  One Philox block covers rows {m, m + 8} x columns {n, n + 1} for m % 16 < 8 and n even: the 2 x 2 fragment one thread of
// the wgmma epilogue holds.  Word 2 ((m >> 3) & 1) + (n & 1) is the element's.
__device__ __forceinline__ uint4 dropout_block(unsigned long long seed, uint32_t d, uint32_t site, uint32_t m, uint32_t n) {
  return philox4x32_10(make_uint4(n >> 1, ((m >> 4) << 3) | (m & 7u), site, d), static_cast<uint32_t>(seed),
                       static_cast<uint32_t>(seed >> 32));
}
// Keras' keep test, random_uniform >= rate, on the 24-bit uniform (word >> 8) 2^-24 the ATS / MIM streams use (exact in fp32)
__device__ __forceinline__ bool dropout_keep(uint32_t word, float rate) {
  return static_cast<float>(word >> 8) * 5.9604644775390625e-8f >= rate;
}
__device__ __forceinline__ uint32_t dropout_word(uint4 x, uint32_t m, uint32_t n) {
  const uint32_t i = 2u * ((m >> 3) & 1u) + (n & 1u);
  return i == 0 ? x.x : i == 1 ? x.y : i == 2 ? x.z : x.w;
}
// The element form (the SIMT GEMM epilogue and vb_op_dropout_mask)
__device__ __forceinline__ bool dropout_keep_at(unsigned long long seed, uint32_t d, uint32_t site, uint32_t m, uint32_t n, float rate) {
  return dropout_keep(dropout_word(dropout_block(seed, d, site, m, n), m, n), rate);
}

}  // namespace vb
