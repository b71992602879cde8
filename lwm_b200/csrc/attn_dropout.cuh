// Attention dropout: the keep/drop decision of one (batch row, head, query, key) entry, made from a counter-based
// generator so that the forward and backward tile kernels regenerate the same mask without ever storing it.
//
// The mask function (restated bit for bit in numpy by tests/attn_dropout_model.py):
//   generator  Philox4x32-10 (Salmon et al., SC'11; the generator of curand and torch)
//   key        (seed & 0xffffffff, seed >> 32)
//   counter    (c0(k), q & ~8, h, b) with c0(k) = ((k >> 4) << 2) | ((k >> 1) & 3)
//   entry      16-bit half (k & 1) of word 2 ((q >> 3) & 1) + ((k >> 3) & 1) of the call's four 32-bit words (half 0 =
//              low bits)
//   dropped    iff that u16 < thr, thr = min(65535, round(p * 65536))
// q and k are GLOBAL token positions, h the head and b the GLOBAL batch row. One call covers the 2 x 4 entries
// {q, q + 8} x {k, k + 1, k + 8, k + 9} (q, k with bit 3 and k with bit 0 clear). That shape fits both kernels' register
// fragments: a forward thread holds rows r and r + 8 against keys 8 g + 2 quad + {0, 1}, so a call serves 8 of its
// entries (8 calls per thread per 128-key tile); a backward thread holds S^T, keys kr and kr + 8 against query columns
// 8 g + 2 quad + {0, 1}, so a call serves 4 (8 calls per thread per 64-row Q tile). Both rely on q_pos0 and k_pos0
// being multiples of 128 (checked by the entry points), which keeps a thread's r / r + 8 and kr / kr + 8 in one call.
#pragma once
#include "attn_common.cuh"

namespace lwm {

LWM_DEVICE uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

struct DropParams {
  uint32_t seed_lo, seed_hi;   // Philox key
  uint32_t thr;                // 1 .. 65535: drop iff u16 < thr
  uint32_t batch0;             // global batch row of the launch's batch row 0 (blockIdx.z / the CTA's b is added)
};

LWM_DEVICE uint32_t drop_ctr0(uint32_t k) { return ((k >> 4) << 2) | ((k >> 1) & 3u); }

// The Philox block of queries {q, q + 8} and keys {k, k + 1, k + 8, k + 9} (bit 3 of q and bits 0, 3 of k ignored);
// b is the launch-local batch row
LWM_DEVICE uint4 drop_block(const DropParams& d, uint32_t q, uint32_t k, uint32_t h, uint32_t b) {
  return philox4x32_10(make_uint4(drop_ctr0(k), q & ~8u, h, d.batch0 + b), d.seed_lo, d.seed_hi);
}

// The decision of the entry with query bit 3 = qb, key bit 3 = kb and key bit 0 = half in block r
LWM_DEVICE bool drop_pick(uint4 r, uint32_t qb, uint32_t kb, uint32_t half, uint32_t thr) {
  const uint32_t j = 2 * qb + kb;
  const uint32_t wd = j == 0 ? r.x : j == 1 ? r.y : j == 2 ? r.z : r.w;
  return ((wd >> (16 * half)) & 0xffffu) < thr;
}

}  // namespace lwm
