// The capturable decode step (DESIGN.md §3.6 "Decode in a CUDA graph"): nothing on it depends on a host value that
// changes from token to token, so one recorded step can be replayed token after token.
//   kv_write_at_kernel      the decode write of one new row per batch entry at the global slot held in a device cursor
//                           (int32 [2]: the slot, then an arrival counter that is zero between calls). Every rank
//                           launches it; only the owner of the slot (lo <= slot < lo + L) writes, with the row bodies
//                           of the host-row writes (kv_write.cuh), so the cache holds the same bits. The last CTA to
//                           arrive advances the slot by one. A slot >= max_length or a position outside
//                           [0, max_position) writes nothing and ORs an LWM_DEVICE_ERR_* bit into a sticky error word.
//   check_positions_kernel  the same position check for q's positions, on its own (the GEMV decode kernel's arguments
//                           are fixed). A position is never used as an index (the angle is pos * inv_freq), so an
//                           out-of-range one is a wrong answer, not a wild access: the check reports it.
#include "capi_internal.h"
#include "kv_write.cuh"
#include "../../include/lwm_b200.h"

#include <algorithm>
#include <type_traits>

namespace lwm {

template <typename T, bool kQ8, bool kRope>
__global__ void __launch_bounds__(256, 1)   // (without the 1, ptxas caps the q8 + rope instances at 64 registers and spills)
kv_write_at_kernel(const T* __restrict__ k_new, const T* __restrict__ v_new, void* cache_k, void* cache_v,
                   unsigned* k_exp, unsigned* v_exp, const int* __restrict__ position_ids,
                   const float* __restrict__ inv_freq, int max_position, int* cursor, long long lo, int L,
                   int max_length, int B, int H, int* err) {
  __shared__ int s_slot;
  if (threadIdx.x == 0) s_slot = cursor[0];
  bool bad_pos = false;
  if constexpr (kRope) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      const int p = position_ids[b];
      bad_pos |= p < 0 || p >= max_position;
    }
  }
  // every CTA checks the whole step, so that a bad step writes nothing anywhere; the barrier also publishes s_slot
  bad_pos = __syncthreads_or(bad_pos);
  const int slot = s_slot;
  const bool bad_slot = slot < 0 || slot >= max_length;
  const long long dst0 = slot - lo;
  if (!bad_slot && !bad_pos && dst0 >= 0 && dst0 < L) {
    const long long tok0 = (long long)blockIdx.x * kRopePos;
    if constexpr (kQ8)
      kv_write_q8_rows<T, kRope>(k_new, v_new, static_cast<signed char*>(cache_k), k_exp,
                                 static_cast<signed char*>(cache_v), v_exp, position_ids, inv_freq, 1, 0, 1, L, dst0, H,
                                 B, tok0);
    else
      kv_write_rows<T, kRope>(k_new, v_new, static_cast<T*>(cache_k), static_cast<T*>(cache_v), position_ids, inv_freq,
                              1, 0, 1, L, dst0, H, B, tok0);
  }
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0 && (bad_slot || bad_pos))
      atomicOr(err, (bad_slot ? LWM_DEVICE_ERR_SLOT : 0) | (bad_pos ? LWM_DEVICE_ERR_POSITION : 0));
    // this CTA's read of the slot is complete (it is in s_slot): the last CTA to arrive may advance it
    if (atomicAdd(cursor + 1, 1) == int(gridDim.x) - 1) {
      cursor[1] = 0;
      cursor[0] = slot + 1;
    }
  }
}

__global__ void __launch_bounds__(256) check_positions_kernel(const int* __restrict__ position_ids, long long n,
                                                              int max_position, int* err) {
  bool bad = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int p = position_ids[i];
    bad |= p < 0 || p >= max_position;
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(err, LWM_DEVICE_ERR_POSITION);
}

}  // namespace lwm

using namespace lwm;

static bool aligned4(const void* p) { return (reinterpret_cast<size_t>(p) & 3) == 0; }

extern "C" int lwm_kv_cache_write_at(const void* k_new, const void* v_new, int src_dtype, void* cache_k, void* cache_v,
                                     signed char* k_exp, signed char* v_exp, const int* position_ids,
                                     const float* inv_freq, int max_position, int* cursor, long long lo, int L,
                                     int max_length, int B, int H, int D, int* err, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_at: head_dim must be 128");
  if (B <= 0 || H <= 0 || L <= 0 || max_length <= 0) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_at: bad sizes");
  if (lo < 0 || lo + L > max_length) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_at: shard rows out of range");
  if (!k_new || !v_new || !cache_k || !cache_v || !cursor || !err)
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: null pointer");
  if (!k_exp != !v_exp) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: k_exp and v_exp go together");
  if (!position_ids != !inv_freq) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: null position_ids / inv_freq");
  if (position_ids && max_position <= 0) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: max_position must be > 0");
  if (src_dtype != 0 && src_dtype != 1)
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: dtype codes are 0 (fp32) or 1 (bf16)");
  const bool q8 = k_exp != nullptr;
  if (q8 && !(aligned4(cache_k) && aligned4(k_exp) && aligned4(cache_v) && aligned4(v_exp)))
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: the 8-bit cache's data and exp must be 4-byte aligned");
  if (!aligned4(cursor) || !aligned4(err)) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_at: cursor and err must be aligned");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const unsigned blocks = unsigned((B + kRopePos - 1) / kRopePos);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto* ke = reinterpret_cast<unsigned*>(k_exp);
  auto* ve = reinterpret_cast<unsigned*>(v_exp);
  return with_flags(
      [&](auto is_f32, auto kq8, auto rope) {
        using T = std::conditional_t<decltype(is_f32)::value, float, __nv_bfloat16>;
        kv_write_at_kernel<T, decltype(kq8)::value, decltype(rope)::value><<<blocks, 256, 0, st>>>(
            static_cast<const T*>(k_new), static_cast<const T*>(v_new), cache_k, cache_v, ke, ve, position_ids,
            inv_freq, max_position, cursor, lo, L, max_length, B, H, err);
        return lwm_check_launch("kv_write_at_kernel");
      },
      src_dtype == 0, q8, position_ids != nullptr);
}

extern "C" int lwm_rope_check_positions(const int* position_ids, long long n, int max_position, int* err,
                                        void* stream) {
  if (n <= 0) return lwm_fail(LWM_ERR_SHAPE, "rope_check_positions: bad sizes");
  if (!position_ids || !err) return lwm_fail(LWM_ERR_ARG, "rope_check_positions: null pointer");
  if (max_position <= 0) return lwm_fail(LWM_ERR_ARG, "rope_check_positions: max_position must be > 0");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const unsigned blocks = unsigned(std::min<long long>((n + 255) / 256, kNumSMs));
  check_positions_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(position_ids, n, max_position,
                                                                                     err);
  return lwm_check_launch("check_positions_kernel");
}
