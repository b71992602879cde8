// The row bodies of the KV-cache writes, in one place: the writes at a host row (lwm_kv_cache_write_rope in
// attn_rope.cu, lwm_kv_cache_write_q8 in kv_q8.cu) and the decode write at a device cursor (lwm_kv_cache_write_at in
// kv_write_at.cu) all run these, so that every write stores the same bits for the same row.
// Token t of the B*n new rows is (b, i) = (t / n, t % n): source row b*n_src + src0 + i of k / v [B,n_src,H,128],
// destination row b*L + dst0 + i of the cache shards [B,L,H,128]. Each body is one CTA of 256 threads serving the
// kRopePos tokens from tok0.
#pragma once
#include "attn_common.cuh"
#include "kv_q8.cuh"
#include "rope_common.cuh"

#include <type_traits>

namespace lwm {

// bf16 / fp32 cache: k rotated at position_ids[b*n_src + src0 + i] and rounded to T (rope_kernel<T, T>'s bits) when
// kRope, else copied; v copied bit for bit.
template <typename T, bool kRope>
__device__ __forceinline__ void kv_write_rows(const T* __restrict__ k_new, const T* __restrict__ v_new,
                                              T* __restrict__ cache_k, T* __restrict__ cache_v,
                                              const int* __restrict__ position_ids, const float* __restrict__ inv_freq,
                                              int n_src, long long src0, int n, int L, long long dst0, int H,
                                              long long n_tok, long long tok0) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  if constexpr (kRope) {
    const int p = threadIdx.x >> 6, j = threadIdx.x & 63;
    const long long tok = tok0 + p;
    if (tok < n_tok) {
      const long long b = tok / n, i = tok - b * n;
      cs[p][j] = rope_cos_sin(position_ids, inv_freq, b * n_src + src0 + i, j, 1.0f);
    }
    __syncthreads();
  }
  const int vh = H * (kRopeDim / 8), vt = 2 * vh;      // 8-element vectors of one row of k (then of v)
  constexpr int kBatch = Raw8<T>::kBatch;
  const int total = kRopePos * vt;
  for (int base = threadIdx.x; base < total; base += kBatch * blockDim.x) {
    Raw8<T> raw[kBatch];
    long long src[kBatch], dst[kBatch];
    int cs_idx[kBatch];
    bool live[kBatch], is_k[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int v = base + u * blockDim.x;
      const int p = v / vt, r = v - p * vt;
      const long long tok = tok0 + p;
      live[u] = v < total && tok < n_tok;
      is_k[u] = r < vh;
      const int rr = is_k[u] ? r : r - vh;
      const long long b = tok / n, i = tok - b * n;
      src[u] = (b * n_src + src0 + i) * H * kRopeDim + rr * 8;
      dst[u] = (b * L + dst0 + i) * H * kRopeDim + rr * 8;
      cs_idx[u] = p * kRopePairs + (rr & 15) * 4;
      if (live[u]) raw[u].load((is_k[u] ? k_new : v_new) + src[u]);
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (!live[u]) continue;
      if (kRope && is_k[u]) {
        float x[8], y[8];
        raw[u].unpack(x);
        rope_rotate8(x, y, &cs[0][0], cs_idx[u]);
        store8<T>(cache_k + dst[u], y);
      } else {
        raw[u].store((is_k[u] ? cache_k : cache_v) + dst[u]);
      }
    }
  }
}

constexpr int kQ8Warps = 8;
constexpr int kQ8Batch = 4;   // rows loaded per warp before the first is quantized

// lane's 4 elements [4l, 4l+4) of a fp32 or bf16 row, as floats
template <typename T>
__device__ __forceinline__ void load4(const T* row, int lane, float (&x)[4]) {
  if constexpr (std::is_same<T, float>::value) {
    const float4 f = reinterpret_cast<const float4*>(row)[lane];
    x[0] = f.x; x[1] = f.y; x[2] = f.z; x[3] = f.w;
  } else {
    const uint2 r = reinterpret_cast<const uint2*>(row)[lane];
    x[0] = __uint_as_float(r.x << 16); x[1] = __uint_as_float(r.x & 0xffff0000u);
    x[2] = __uint_as_float(r.y << 16); x[3] = __uint_as_float(r.y & 0xffff0000u);
  }
}

// 8-bit cache: rows quantized into codes data [B,L,H,128] and exponent words exp [B,H,L] (word (b*H + h)*L + dst0 + i),
// k first rotated and rounded to T as kv_write_rows stores it when kRope. One warp per (token, tensor, head) row in the
// decode kernel's lane layout: lane l owns elements [4l, 4l+4), the group maximum is a shuffle max over the group's 8
// lanes, and each lane stores its codes as one 32-bit word.
template <typename T, bool kRope>
__device__ __forceinline__ void kv_write_q8_rows(const T* __restrict__ k_src, const T* __restrict__ v_src,
                                                 signed char* __restrict__ k_data, unsigned* __restrict__ k_exp,
                                                 signed char* __restrict__ v_data, unsigned* __restrict__ v_exp,
                                                 const int* __restrict__ position_ids,
                                                 const float* __restrict__ inv_freq, int n_src, long long src0, int n,
                                                 int L, long long dst0, int H, long long n_tok, long long tok0) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  if constexpr (kRope) {
    const int p = threadIdx.x >> 6, j = threadIdx.x & 63;
    const long long tok = tok0 + p;
    if (tok < n_tok) {
      const long long b = tok / n, i = tok - b * n;
      cs[p][j] = rope_cos_sin(position_ids, inv_freq, b * n_src + src0 + i, j, 1.0f);
    }
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = kRopePos * 2 * H;          // (token, k/v, head), heads fastest
  for (int r0 = warp; r0 < rows; r0 += kQ8Warps * kQ8Batch) {
    float x[kQ8Batch][4];
    bool live[kQ8Batch];
#pragma unroll
    for (int u = 0; u < kQ8Batch; ++u) {
      const int r = r0 + u * kQ8Warps;
      const int p = r / (2 * H), h = r % H;
      const bool is_k = (r / H) % 2 == 0;
      const long long tok = tok0 + p;
      live[u] = r < rows && tok < n_tok;   // warp-uniform
      if (live[u]) {
        const long long b = tok / n, i = tok - b * n;
        load4<T>((is_k ? k_src : v_src) + ((b * n_src + src0 + i) * H + h) * kHeadDim, lane, x[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < kQ8Batch; ++u) {
      if (!live[u]) continue;
      const int r = r0 + u * kQ8Warps;
      const int p = r / (2 * H), h = r % H;
      const bool is_k = (r / H) % 2 == 0;
      const long long tok = tok0 + p, b = tok / n, i = tok - b * n;
      float y[4] = {x[u][0], x[u][1], x[u][2], x[u][3]};
      if (kRope && is_k) {
        // pairs (2l, 2l+1) with rope_rotate8's separately rounded products, rounded to T as the rope write stores them
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float2 f = cs[p][2 * lane + e];
          y[2 * e] = __fsub_rn(__fmul_rn(x[u][2 * e], f.x), __fmul_rn(x[u][2 * e + 1], f.y));
          y[2 * e + 1] = __fadd_rn(__fmul_rn(x[u][2 * e], f.y), __fmul_rn(x[u][2 * e + 1], f.x));
        }
        if constexpr (!std::is_same<T, float>::value) {
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = __bfloat162float(__float2bfloat16_rn(y[e]));
        }
      }
      const int e = q8_group_exp(y);
      const unsigned codes = q8_pack4(y, e);
      const long long dst = b * L + dst0 + i;
      reinterpret_cast<unsigned*>((is_k ? k_data : v_data) + (dst * H + h) * kHeadDim)[lane] = codes;
      // the row's 4 exponents (groups at lanes 0, 8, 16, 24) as one word
      unsigned w = 0;
#pragma unroll
      for (int g = 0; g < 4; ++g) w |= (unsigned(__shfl_sync(0xffffffffu, e, 8 * g)) & 0xffu) << (8 * g);
      if (lane == 0) (is_k ? k_exp : v_exp)[(b * H + h) * (long long)L + dst0 + i] = w;
    }
  }
}

}  // namespace lwm
