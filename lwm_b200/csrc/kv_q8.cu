// The 8-bit KV cache of the generation path (format: kv_q8.cuh, DESIGN.md §5 "8-bit KV cache"):
//   kv_write_q8_kernel   quantizes new k / v rows as they are written into this rank's cache shard, the keys optionally
//                        rotated first (the rotation of lwm_kv_cache_write_rope, rounded to the source dtype). One warp
//                        per (token, tensor, head) row in the decode kernel's lane layout: lane l owns elements
//                        [4l, 4l+4), the group maximum is a shuffle max over the group's 8 lanes, and each lane stores
//                        its codes as one 32-bit word. One CTA serves kRopePos tokens with one (cos, sin) table.
//   kv_dequant_q8_kernel cache rows -> fp32 or bf16 values (exact), one warp per row.
#include "attn_common.cuh"
#include "capi_internal.h"
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

// rows = B*L*H rows of data [B,L,H,128] / exp [B,H,L,4] -> out [B,L,H,128] in T
template <typename T>
__global__ void __launch_bounds__(256) kv_dequant_q8_kernel(const signed char* __restrict__ data,
                                                            const unsigned* __restrict__ exp, T* __restrict__ out,
                                                            int L, int H, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += stride) {
    const long long h = row % H, bl = row / H, b = bl / L, l = bl - b * L;
    const unsigned w = reinterpret_cast<const unsigned*>(data + row * kHeadDim)[lane];
    const float4 f = q8_dequant4(w, exp[(b * H + h) * L + l], lane);
    if constexpr (std::is_same<T, float>::value)
      reinterpret_cast<float4*>(out + row * kHeadDim)[lane] = f;
    else
      reinterpret_cast<uint2*>(out + row * kHeadDim)[lane] = make_uint2(pack_bf16x2(f.x, f.y), pack_bf16x2(f.z, f.w));
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
