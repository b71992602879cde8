// Rotary position embedding arithmetic shared by the stand-alone rotation (attn_rope.cu: rope_kernel) and the
// operand passes of the attention op that rotate q / k on the fly (attn_misc.cu: the *_rope kernels). One definition,
// so that both produce the same bits for the same (position, element):
//   angle   = float32(float64(pos) * float64(inv_freq[j]))      (np.outer of an int64 and a float32 vector)
//   (c, s)  = cos / sin of that angle taken in double and rounded once to float32
//   y       = (a + ib)(c + is) on the interleaved pair (2j, 2j+1), every product and sum separately rounded as in a
//             plain complex64 multiply; the conjugate rotation flips the sign of s.
#pragma once
#include <cuda_bf16.h>

namespace lwm {

constexpr int kRopeDim = 128;
constexpr int kRopePairs = kRopeDim / 2;
constexpr int kRopePos = 4;   // token positions per CTA (and per (cos, sin) table in shared memory)

// (cos, sin_sign * sin) of the rotation of pair j at the position of token tok
__device__ __forceinline__ float2 rope_cos_sin(const int* __restrict__ position_ids, const float* __restrict__ inv_freq,
                                               long long tok, int j, float sin_sign) {
  const float angle = (float)((double)position_ids[tok] * (double)inv_freq[j]);
  double s, c;
  sincos((double)angle, &s, &c);
  return make_float2((float)c, sin_sign * (float)s);
}

// y = x rotated pairwise: 8 consecutive elements (4 pairs) of one row, cs[idx + i] = (cos, sin) of pair i
__device__ __forceinline__ void rope_rotate8(const float (&x)[8], float (&y)[8], const float2* cs, int idx) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = cs[idx + i];
    // (a + ib)(c + is) = (ac - bs) + i(as + bc), separately rounded products as in a plain complex64 multiply
    y[2 * i] = __fsub_rn(__fmul_rn(x[2 * i], f.x), __fmul_rn(x[2 * i + 1], f.y));
    y[2 * i + 1] = __fadd_rn(__fmul_rn(x[2 * i], f.y), __fmul_rn(x[2 * i + 1], f.x));
  }
}

// cs[p][j] for the kRopePos tokens from tok0, one (p, j) per thread: the CTA has exactly kRopePos * kRopePairs = 256
// threads. Tokens >= n_tok are skipped.
__device__ __forceinline__ void rope_fill_table(float2 (*cs)[kRopePairs], const int* __restrict__ position_ids,
                                                const float* __restrict__ inv_freq, long long tok0, long long n_tok,
                                                float sin_sign) {
  const int p = threadIdx.x >> 6, j = threadIdx.x & 63;
  const long long tok = tok0 + p;
  if (tok < n_tok) cs[p][j] = rope_cos_sin(position_ids, inv_freq, tok, j, sin_sign);
}

// 8 consecutive elements as loaded (kept raw until use, so that a batch of loads costs few registers)
template <typename T>
struct Raw8;
template <>
struct Raw8<float> {
  float4 a, b;
  static constexpr int kBatch = 4;
  __device__ __forceinline__ void load(const float* p) {
    a = reinterpret_cast<const float4*>(p)[0];
    b = reinterpret_cast<const float4*>(p)[1];
  }
  __device__ __forceinline__ void store(float* p) const {
    reinterpret_cast<float4*>(p)[0] = a;
    reinterpret_cast<float4*>(p)[1] = b;
  }
  __device__ __forceinline__ void unpack(float (&x)[8]) const {
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  }
};
template <>
struct Raw8<__nv_bfloat16> {
  uint4 a;
  static constexpr int kBatch = 8;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { a = reinterpret_cast<const uint4*>(p)[0]; }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { reinterpret_cast<uint4*>(p)[0] = a; }
  __device__ __forceinline__ void unpack(float (&x)[8]) const {
    const unsigned w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      x[2 * i] = __uint_as_float(w[i] << 16);
      x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
};

// round 8 floats to T and back (the value a store8<T> / load of T would round-trip): identity for float
template <typename T>
__device__ __forceinline__ void round8(float (&y)[8]);
template <>
__device__ __forceinline__ void round8<float>(float (&)[8]) {}
template <>
__device__ __forceinline__ void round8<__nv_bfloat16>(float (&y)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) y[i] = __bfloat162float(__float2bfloat16_rn(y[i]));
}

template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&y)[8]);
template <>
__device__ __forceinline__ void store8<float>(float* p, const float (&y)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(y[0], y[1], y[2], y[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(y[4], y[5], y[6], y[7]);
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&y)[8]) {
  uint4 o;
  unsigned* w = reinterpret_cast<unsigned*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(y[2 * i], y[2 * i + 1]);
    w[i] = *reinterpret_cast<const unsigned*>(&v);
  }
  reinterpret_cast<uint4*>(p)[0] = o;
}

}  // namespace lwm
