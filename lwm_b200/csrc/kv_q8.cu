// The 8-bit KV cache of the generation path (format: kv_q8.cuh, DESIGN.md §5 "8-bit KV cache"):
//   kv_write_q8_kernel   quantizes new k / v rows as they are written into this rank's cache shard, the keys optionally
//                        rotated first (the rotation of lwm_kv_cache_write_rope, rounded to the source dtype). One warp
//                        per (token, tensor, head) row in the decode kernel's lane layout: lane l owns elements
//                        [4l, 4l+4), the group maximum is a shuffle max over the group's 8 lanes, and each lane stores
//                        its codes as one 32-bit word. One CTA serves kRopePos tokens with one (cos, sin) table.
//   kv_dequant_q8_kernel cache rows -> fp32 or bf16 values (exact), one warp per row.
//   kv_q8_absmax_kernel  largest finite |value| of the cache rows, as lwm_attn_absmax over their dequantized values.
//   kv_q8_stage_kernel   cache rows -> the scaled fp16 / e4m3 operand copies of the tensor-core paths, the same bytes as
//                        lwm_attn_to_f16_scaled / lwm_attn_to_e4m3_scaled write from the dequantized rows, without them.
#include "attn_common.cuh"
#include "capi_internal.h"
#include "e4m3.cuh"
#include "kv_q8.cuh"
#include "kv_write.cuh"
#include "rope_common.cuh"

#include <algorithm>
#include <type_traits>

namespace lwm {

// kv_write.cuh: kv_write_q8_rows; one CTA serves kRopePos tokens with one (cos, sin) table
template <typename T, bool kRope>
__global__ void __launch_bounds__(kQ8Warps * 32)
kv_write_q8_kernel(const T* __restrict__ k_src, const T* __restrict__ v_src, signed char* __restrict__ k_data,
                   unsigned* __restrict__ k_exp, signed char* __restrict__ v_data, unsigned* __restrict__ v_exp,
                   const int* __restrict__ position_ids, const float* __restrict__ inv_freq, int n_src, long long src0,
                   int n, int L, long long dst0, int H, long long n_tok) {
  kv_write_q8_rows<T, kRope>(k_src, v_src, k_data, k_exp, v_data, v_exp, position_ids, inv_freq, n_src, src0, n, L,
                             dst0, H, n_tok, (long long)blockIdx.x * kRopePos);
}

// lane's 4 exact values of row `row` (over B*L*H) of data [B,L,H,128] / exp [B,H,L,4]
__device__ __forceinline__ float4 q8_row_values(const signed char* __restrict__ data, const unsigned* __restrict__ exp,
                                                int L, int H, long long row, int lane) {
  const long long h = row % H, bl = row / H, b = bl / L, l = bl - b * L;
  const unsigned w = reinterpret_cast<const unsigned*>(data + row * kHeadDim)[lane];
  return q8_dequant4(w, exp[(b * H + h) * L + l], lane);
}

// rows = B*L*H rows of data [B,L,H,128] / exp [B,H,L,4] -> out [B,L,H,128] in T
template <typename T>
__global__ void __launch_bounds__(256) kv_dequant_q8_kernel(const signed char* __restrict__ data,
                                                            const unsigned* __restrict__ exp, T* __restrict__ out,
                                                            int L, int H, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    const float4 f = q8_row_values(data, exp, L, H, row, lane);
    if constexpr (std::is_same<T, float>::value)
      reinterpret_cast<float4*>(out + row * kHeadDim)[lane] = f;
    else
      reinterpret_cast<uint2*>(out + row * kHeadDim)[lane] = make_uint2(pack_bf16x2(f.x, f.y), pack_bf16x2(f.z, f.w));
  }
}

// atomicMax of the finite |value| bit patterns into *out_bits (the NaN code reads back as NaN and is skipped)
__global__ void __launch_bounds__(256) kv_q8_absmax_kernel(const signed char* __restrict__ data,
                                                           const unsigned* __restrict__ exp,
                                                           unsigned* __restrict__ out_bits, int L, int H,
                                                           long long rows) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  unsigned m = 0;
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    const float4 f = q8_row_values(data, exp, L, H, row, lane);
    m = max(max(m, finite_abs_bits(__float_as_uint(f.x))),
            max(finite_abs_bits(__float_as_uint(f.y)),
                max(finite_abs_bits(__float_as_uint(f.z)), finite_abs_bits(__float_as_uint(f.w)))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0 && m) atomicMax(out_bits, m);
}

// dst = fp16(value / *scale) (kDst 2) or e4m3(value / *scale) (kDst 3), [B,L,H,128] like the rows. The exact fp32 value
// is formed first and then multiplied by 1 / *scale, as the *_by_scale kernels of attn_misc.cu do with the dequantized
// value: folding 2^e into the multiplier would round differently where the product falls below fp16's normal range.
template <int kDst>
__global__ void __launch_bounds__(256) kv_q8_stage_kernel(const signed char* __restrict__ data,
                                                          const unsigned* __restrict__ exp, void* __restrict__ dst,
                                                          const float* __restrict__ scale, int L, int H, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  const float inv = 1.0f / *scale;
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    const float4 f = q8_row_values(data, exp, L, H, row, lane);
    if constexpr (kDst == 3)
      reinterpret_cast<uint32_t*>(dst)[row * (kHeadDim / 4) + lane] =
          pack_e4m3x4(f.x * inv, f.y * inv, f.z * inv, f.w * inv);
    else
      reinterpret_cast<uint2*>(dst)[row * (kHeadDim / 4) + lane] =
          make_uint2(pack_f16x2(f.x * inv, f.y * inv), pack_f16x2(f.z * inv, f.w * inv));
  }
}

}  // namespace lwm

using namespace lwm;

static bool aligned4(const void* p) { return (reinterpret_cast<size_t>(p) & 3) == 0; }

extern "C" int lwm_kv_cache_write_q8(const void* k_src, const void* v_src, int src_dtype, signed char* k_data,
                                     signed char* k_exp, signed char* v_data, signed char* v_exp,
                                     const int* position_ids, const float* inv_freq, int B, int n_src, long long src0,
                                     int n, int L, long long dst0, int H, int D, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_q8: head_dim must be 128");
  if (B <= 0 || n <= 0 || H <= 0 || n_src <= 0 || L <= 0) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_q8: bad sizes");
  if (src0 < 0 || src0 + n > n_src || dst0 < 0 || dst0 + n > L)
    return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_q8: rows out of range");
  if (!k_src || !v_src || !k_data || !k_exp || !v_data || !v_exp)
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_q8: null pointer");
  if (!position_ids != !inv_freq) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_q8: null position_ids / inv_freq");
  if (src_dtype != 0 && src_dtype != 1)
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_q8: dtype codes are 0 (fp32) or 1 (bf16)");
  if (!aligned4(k_data) || !aligned4(k_exp) || !aligned4(v_data) || !aligned4(v_exp))
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_q8: data and exp must be 4-byte aligned");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long n_tok = (long long)B * n;
  const unsigned blocks = unsigned((n_tok + kRopePos - 1) / kRopePos);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* ke = reinterpret_cast<unsigned*>(k_exp);
  auto* vexp = reinterpret_cast<unsigned*>(v_exp);
  const bool rope = position_ids != nullptr;
  if (src_dtype == 0) {
    auto* kernel = rope ? kv_write_q8_kernel<float, true> : kv_write_q8_kernel<float, false>;
    kernel<<<blocks, kQ8Warps * 32, 0, st>>>(reinterpret_cast<const float*>(k_src), reinterpret_cast<const float*>(v_src),
                                             k_data, ke, v_data, vexp, position_ids, inv_freq, n_src, src0, n, L, dst0,
                                             H, n_tok);
  } else {
    auto* kernel = rope ? kv_write_q8_kernel<__nv_bfloat16, true> : kv_write_q8_kernel<__nv_bfloat16, false>;
    kernel<<<blocks, kQ8Warps * 32, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(k_src),
                                             reinterpret_cast<const __nv_bfloat16*>(v_src), k_data, ke, v_data, vexp,
                                             position_ids, inv_freq, n_src, src0, n, L, dst0, H, n_tok);
  }
  return lwm_check_launch("kv_write_q8_kernel");
}

extern "C" int lwm_kv_dequant_q8(const signed char* data, const signed char* exp, void* out, int out_dtype, int B,
                                 int L, int H, int D, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "kv_dequant_q8: head_dim must be 128");
  if (B <= 0 || L <= 0 || H <= 0) return lwm_fail(LWM_ERR_SHAPE, "kv_dequant_q8: bad sizes");
  if (!data || !exp || !out) return lwm_fail(LWM_ERR_ARG, "kv_dequant_q8: null pointer");
  if (out_dtype != 0 && out_dtype != 1)
    return lwm_fail(LWM_ERR_ARG, "kv_dequant_q8: dtype codes are 0 (fp32) or 1 (bf16)");
  if (!aligned4(data) || !aligned4(exp)) return lwm_fail(LWM_ERR_ARG, "kv_dequant_q8: data and exp must be 4-byte aligned");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long rows = (long long)B * L * H;
  const unsigned blocks = unsigned(std::min<long long>((rows + 7) / 8, 132 * 16));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* e = reinterpret_cast<const unsigned*>(exp);
  if (out_dtype == 0)
    kv_dequant_q8_kernel<float><<<blocks, 256, 0, st>>>(data, e, reinterpret_cast<float*>(out), L, H, rows);
  else
    kv_dequant_q8_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(data, e, reinterpret_cast<__nv_bfloat16*>(out), L, H,
                                                               rows);
  return lwm_check_launch("kv_dequant_q8_kernel");
}

static unsigned q8_row_blocks(long long rows) { return unsigned(std::min<long long>((rows + 7) / 8, 132 * 16)); }

extern "C" int lwm_kv_q8_absmax(const signed char* data, const signed char* exp, int B, int L, int H, int D,
                                unsigned* out_bits, void* stream) {
  if (!data || !exp || !out_bits) return lwm_fail(LWM_ERR_ARG, "kv_q8_absmax: null pointer");
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "kv_q8_absmax: head_dim must be 128");
  if (B <= 0 || L <= 0 || H <= 0) return lwm_fail(LWM_ERR_SHAPE, "kv_q8_absmax: bad sizes");
  if (!aligned4(data) || !aligned4(exp)) return lwm_fail(LWM_ERR_ARG, "kv_q8_absmax: data and exp must be 4-byte aligned");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long rows = (long long)B * L * H;
  kv_q8_absmax_kernel<<<q8_row_blocks(rows), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      data, reinterpret_cast<const unsigned*>(exp), out_bits, L, H, rows);
  return lwm_check_launch("kv_q8_absmax_kernel");
}

extern "C" int lwm_kv_q8_stage(const signed char* data, const signed char* exp, void* dst, int dst_dtype,
                               const float* scale, int B, int L, int H, int D, void* stream) {
  if (!data || !exp || !dst || !scale) return lwm_fail(LWM_ERR_ARG, "kv_q8_stage: null pointer");
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "kv_q8_stage: head_dim must be 128");
  if (dst_dtype != 2 && dst_dtype != 3)
    return lwm_fail(LWM_ERR_ARG, "kv_q8_stage: dst dtype codes are 2 (scaled fp16) or 3 (scaled e4m3)");
  if (B <= 0 || L <= 0 || H <= 0) return lwm_fail(LWM_ERR_SHAPE, "kv_q8_stage: bad sizes");
  if (!aligned4(data) || !aligned4(exp)) return lwm_fail(LWM_ERR_ARG, "kv_q8_stage: data and exp must be 4-byte aligned");
  if (reinterpret_cast<size_t>(dst) & (dst_dtype == 2 ? 7 : 3))
    return lwm_fail(LWM_ERR_ARG, "kv_q8_stage: dst must be 8-byte (fp16) or 4-byte (e4m3) aligned");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long rows = (long long)B * L * H;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const auto* e = reinterpret_cast<const unsigned*>(exp);
  if (dst_dtype == 3)
    kv_q8_stage_kernel<3><<<q8_row_blocks(rows), 256, 0, st>>>(data, e, dst, scale, L, H, rows);
  else
    kv_q8_stage_kernel<2><<<q8_row_blocks(rows), 256, 0, st>>>(data, e, dst, scale, L, H, rows);
  return lwm_check_launch("kv_q8_stage_kernel");
}
