// Philox4x32-10, the counter-based RNG behind every dropout mask of the library: bsmm_dropout_mask (ewops.cuh) and the
// fused attention kernels with dropout (tc_bst_attn.cuh, tc_bst_attn_bwd.cuh) draw element e of a mask from word e % 4
// of philox4x32_10(counter = (e / 4 as 64 bits, call as 64 bits), key = seed), so one definition keeps them in step.
#pragma once
#include <cstdint>

namespace bsmm {

// Philox4x32-10 (Salmon et al., SC'11; the constants of Random123's philox4x32)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
    const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Keep bits of the 4 elements 4g .. 4g + 3 of mask `call` under key `seed`: bit w set iff word w < thr (thr =
// floor(keep_prob * 2^32), compared in 64 bits).
__device__ __forceinline__ uint32_t philox_keep4(unsigned long long g, unsigned long long call, uint2 key,
                                                 unsigned long long thr) {
  const uint4 r = philox4x32_10(make_uint4((unsigned)g, (unsigned)(g >> 32), (unsigned)call, (unsigned)(call >> 32)), key);
  return (uint32_t)(r.x < thr) | (uint32_t)(r.y < thr) << 1 | (uint32_t)(r.z < thr) << 2 | (uint32_t)(r.w < thr) << 3;
}

}  // namespace bsmm
