// The 8-bit KV-cache format (DESIGN.md §5 "8-bit KV cache"), in one place: the quantizing cache write (kv_q8.cu),
// the exact dequantization (kv_q8.cu) and the GEMV decode kernel reading the cache (attn_decode.cu) all use these.
//   row    one (batch, position, head) vector of 128 values: int8 codes data [B,L,H,128] plus one power-of-two exponent
//          per 32-element group, exp int8 [B,H,L,4] (head-major: the 4 exponents of a row are one 32-bit word, and
//          consecutive keys of one head are consecutive words)
//   e      floor(log2(m)) - 6 for the group's largest FINITE |x| = m, clamped to [-126, 121]; 0 when m = 0
//   code   clamp(round_half_even(x / 2^e), -127, 127); -128 for NaN and +-inf (reads back as NaN)
//   value  code * 2^e: exact in fp32 and bf16 (at most 7 significant bits, 127 * 2^121 < 2^128)
// In the GEMV layout lane l owns elements [4l, 4l+4) of a row, so group g is lanes [8g, 8g+8) and each lane's codes
// are one 32-bit word of the row.
#pragma once
#include <cuda_runtime.h>

namespace lwm {

constexpr int kQ8Group = 32;          // elements per exponent
constexpr int kQ8ExpMin = -126, kQ8ExpMax = 121;
constexpr int kQ8NanCode = -128;

// 2^e as a float, e in [kQ8ExpMin, kQ8ExpMax] (a normal number)
__device__ __forceinline__ float q8_pow2(int e) { return __int_as_float((e + 127) << 23); }

// exponent of lane's group (lanes [8g, 8g+8)) from the lane's own 4 values: the shuffle max over the group's 8 lanes
__device__ __forceinline__ int q8_group_exp(const float (&x)[4]) {
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) m = fmaxf(m, isfinite(x[i]) ? fabsf(x[i]) : 0.f);
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (m == 0.f) return 0;
  // floor(log2(m)) - 6 from the biased exponent field; a subnormal m (field 0) lands below the clamp
  const int e = int((__float_as_uint(m) >> 23) & 0xffu) - 127 - 6;
  return min(max(e, kQ8ExpMin), kQ8ExpMax);
}

// the 4 codes of x at exponent e, packed little-endian (element 4l + i in byte i). x * 2^-e is exact wherever the
// product is a normal number, and a product below that rounds to code 0 either way.
__device__ __forceinline__ unsigned q8_pack4(const float (&x)[4], int e) {
  const float inv = q8_pow2(-e);      // -e in [-121, 126]
  unsigned w = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = isfinite(x[i]) ? min(max(__float2int_rn(x[i] * inv), -127), 127) : kQ8NanCode;
    w |= (unsigned(c) & 0xffu) << (8 * i);
  }
  return w;
}

// one code (byte i of w) at scale 2^e -> its exact value; the NaN code -> NaN
__device__ __forceinline__ float q8_value(unsigned w, int i, float scale) {
  const int c = int(w << (24 - 8 * i)) >> 24;
  return c == kQ8NanCode ? __int_as_float(0x7fffffff) : __int2float_rn(c) * scale;
}

// lane's 4 values of a row from its code word and the row's exponent word (the exponent of group lane / 8)
__device__ __forceinline__ float4 q8_dequant4(unsigned w, unsigned exps, int lane) {
  const float scale = q8_pow2(int(exps << (24 - 8 * (lane >> 3))) >> 24);
  return make_float4(q8_value(w, 0, scale), q8_value(w, 1, scale), q8_value(w, 2, scale), q8_value(w, 3, scale));
}

}  // namespace lwm
