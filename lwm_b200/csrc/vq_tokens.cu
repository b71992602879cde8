// Vision token framing around the VQGAN (SURVEY.md §8f next-row 4): the wire format that turns codebook indices
// into language-model tokens and back.
//   lwm_vq_frame_tokens    codes [clips, T_in, P] -> tokens [clips, T_out, P+1]: the P codes of every kept frame
//                          followed by eof (8192), or by eov (8193) after the last frame of the clip
//                          (lwm/vision_chat.py:97-104, lwm/data.py:193-212); optional uniform frame selection
//                          (data.py:196-202: np.linspace(0, n-1, max_n_frames).astype(int), built by the host)
//   lwm_vq_unframe_tokens  tokens [n, P+1] -> codes [n, P] (drops the delimiter of every frame, as
//                          lwm/vision_generation.py:160,221 does with `[..., :-1]` before VQGAN.decode)
// Pure index movement, bit-exact by construction; one int32 per thread, coalesced both ways.
#include "capi_internal.h"

namespace lwm {

__global__ void frame_tokens_kernel(const int* __restrict__ codes, const int* __restrict__ frame_idx,
                                    int* __restrict__ tokens, long long total, int T_in, int T_out, int P, int eof,
                                    int eov) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = int(i % (P + 1));
    const long long f = i / (P + 1);
    const int t = int(f % T_out);
    const long long clip = f / T_out;
    const int src_t = frame_idx ? frame_idx[t] : t;
    tokens[i] = p < P ? codes[(clip * T_in + src_t) * P + p] : (t == T_out - 1 ? eov : eof);
  }
}

__global__ void unframe_tokens_kernel(const int* __restrict__ tokens, int* __restrict__ codes, long long total, int P) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long f = i / P;
    codes[i] = tokens[f * (P + 1) + (i - f * P)];
  }
}

static unsigned grid_for(long long total) {
  const long long want = (total + 255) / 256;
  return unsigned(want < kNumSMs * 16 ? want : kNumSMs * 16);
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_vq_frame_tokens(const int* codes, const int* frame_idx, int* tokens, int n_clips, int T_in, int T_out,
                                   int tokens_per_frame, int eof_token, int eov_token, void* stream) {
  if (!codes || !tokens) return lwm_fail(LWM_ERR_ARG, "vq_frame_tokens: null pointer");
  if (n_clips < 0 || T_in <= 0 || T_out <= 0 || tokens_per_frame <= 0)
    return lwm_fail(LWM_ERR_SHAPE, "vq_frame_tokens: a clip needs at least one frame");  // data.py:205 asserts n_frames > 0
  if (!frame_idx && T_in != T_out) return lwm_fail(LWM_ERR_SHAPE, "vq_frame_tokens: T_out != T_in needs frame_idx");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (n_clips == 0) return LWM_OK;
  const long long total = (long long)n_clips * T_out * (tokens_per_frame + 1);
  frame_tokens_kernel<<<grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      codes, frame_idx, tokens, total, T_in, T_out, tokens_per_frame, eof_token, eov_token);
  return lwm_check_launch("frame_tokens_kernel");
}

extern "C" int lwm_vq_unframe_tokens(const int* tokens, int* codes, long long n_frames, int tokens_per_frame, void* stream) {
  if (!tokens || !codes) return lwm_fail(LWM_ERR_ARG, "vq_unframe_tokens: null pointer");
  if (n_frames < 0 || tokens_per_frame <= 0) return lwm_fail(LWM_ERR_SHAPE, "vq_unframe_tokens: bad sizes");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (n_frames == 0) return LWM_OK;
  const long long total = n_frames * tokens_per_frame;
  unframe_tokens_kernel<<<grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(tokens, codes, total,
                                                                                          tokens_per_frame);
  return lwm_check_launch("unframe_tokens_kernel");
}
