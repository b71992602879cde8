// The attention-dropout mask of one region, written out from the device function the tile kernels use
// (attn_dropout.cuh): lets the mask be compared with its restatement bit for bit, without attention arithmetic.
#include "attn_dropout.cuh"
#include "capi_internal.h"

namespace lwm {

__global__ void dropout_mask_kernel(DropParams d, uint32_t b, uint32_t h, long long q_pos0, long long k_pos0, int n_q,
                                    int n_k, uint8_t* __restrict__ out) {
  const long long n = (long long)n_q * n_k;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t q = uint32_t(q_pos0 + i / n_k), k = uint32_t(k_pos0 + i % n_k);
    out[i] = drop_pick(drop_block(d, q, k, h, b), (q >> 3) & 1u, (k >> 3) & 1u, k & 1u, d.thr) ? 1 : 0;
  }
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_attn_dropout_mask(long long seed, unsigned drop_threshold, int b, int h, long long q_pos0,
                                     long long k_pos0, int n_q, int n_k, unsigned char* out, void* stream) {
  if (drop_threshold == 0 || drop_threshold > 65535)
    return lwm_fail(LWM_ERR_ARG, "attn_dropout_mask: drop_threshold must be in [1, 65535]");
  if (!out) return lwm_fail(LWM_ERR_ARG, "attn_dropout_mask: null out");
  if (b < 0 || h < 0 || n_q <= 0 || n_k <= 0 || q_pos0 < 0 || k_pos0 < 0 || q_pos0 + n_q > 0x7fffffffLL ||
      k_pos0 + n_k > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_dropout_mask: b, h >= 0, n_q, n_k >= 1 and positions in [0, 2^31)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const DropParams d = {uint32_t(uint64_t(seed)), uint32_t(uint64_t(seed) >> 32), drop_threshold, 0u};
  const long long want = ((long long)n_q * n_k + 255) / 256;
  dropout_mask_kernel<<<unsigned(want < 4096 ? want : 4096), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      d, uint32_t(b), uint32_t(h), q_pos0, k_pos0, n_q, n_k, out);
  return lwm_check_launch("dropout_mask_kernel");
}
