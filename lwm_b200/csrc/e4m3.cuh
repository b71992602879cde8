// Conversion of fp32 values to e4m3 bytes, shared by every pass that writes the fp8 mode's operand copies (attn_misc.cu,
// kv_q8.cu), so that each copy holds the same bytes whichever source it was staged from.
#pragma once
#include <cuda_fp8.h>
#include <stdint.h>

namespace lwm {

// e4m3 (RN) of two fp32 values, x in the low byte. The callers' power-of-two scales keep every finite value below 256,
// so nothing saturates; NaN and +-inf become the NaN byte (sign | 0x7f, what torch's cast to float8_e4m3fn gives; a
// NaN's sign is whatever the scaling multiply left): e4m3fn has no infinity, and the hardware conversion alone
// (satfinite) would turn +-inf into +-448.
__device__ __forceinline__ uint32_t pack_e4m3x2(float lo, float hi) {
  uint32_t r = __nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, __NV_E4M3);
  const uint32_t a = __float_as_uint(lo), b = __float_as_uint(hi);
  if ((a & 0x7fffffffu) >= 0x7f800000u) r = (r & 0xff00u) | ((a >> 24) & 0x80u) | 0x7fu;
  if ((b & 0x7fffffffu) >= 0x7f800000u) r = (r & 0x00ffu) | ((((b >> 24) & 0x80u) | 0x7fu) << 8);
  return r;
}
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  return pack_e4m3x2(a, b) | (pack_e4m3x2(c, d) << 16);
}

}  // namespace lwm
