// Frame preprocessing in front of the VQGAN encoder (lwm/vision_chat.py:59-74 `Sampler._process_frame`):
// PIL.Image.resize(new_size) with Pillow's default bicubic filter, the centre crop, then x / 127.5 - 1 in fp32.
// Bit-identical to Pillow's 8-bit path: the host builds Pillow's fixed-point coefficient tables
// (lwm_b200/vision_frames.py::pass_tables), and each pass is the same integer multiply-accumulate Pillow runs
// (accumulator starts at 1 << 21, >> 22, clipped to [0, 255]); the image between the passes is uint8.
//
// One launch per clip. A block owns one band of kBandRows output rows of one frame:
//   1. horizontal pass over the input rows the band's vertical support touches, crop columns only, into shared memory
//      as uint8 [rows][crop_w * 3];
//   2. vertical pass from shared memory, then the two separately rounded fp32 operations numpy performs.
// Neighbouring bands recompute the rows their supports share; that costs (band rows * scale + ky) / (band rows *
// scale), e.g. 1.3x of the horizontal pass at 1080p, and keeps every block independent.
// Tables come from the caller: indices taken from them are clamped so that no table can make a read leave the frame
// or the shared-memory band.
#include "capi_internal.h"

namespace lwm {

constexpr int kFramesThreads = 256;
constexpr int kFramesPrecisionBits = 22;                      // Pillow: 32 - 8 (uint8) - 2
constexpr int kFramesSmemTarget = 100 * 1024;                 // two blocks per SM
constexpr int kFramesSmemMax = 227 * 1024;

__device__ __forceinline__ int clip8_shift(int acc) {
  const int v = acc >> kFramesPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(kFramesThreads)
frames_prep_kernel(const unsigned char* __restrict__ frames, int H, int W, const int* __restrict__ x_bounds,
                   const int* __restrict__ x_coeffs, int kx, const int* __restrict__ y_bounds,
                   const int* __restrict__ y_coeffs, int ky, int left, int top, int crop_w, int crop_h, int band_rows,
                   int n_bands, int max_rows, float* __restrict__ out) {
  extern __shared__ unsigned char s_rows[];                   // [max_rows][crop_w * 3]
  const int t = blockIdx.x / n_bands;
  const int r0 = (blockIdx.x % n_bands) * band_rows;
  const int r1 = min(r0 + band_rows, crop_h);
  const int row_bytes = crop_w * 3;

  // input rows touched by the band: bounds are non-decreasing in the output row, but take the extremes anyway
  int y0 = H, y1 = 0;
  for (int r = r0; r < r1; ++r) {
    const int ymin = y_bounds[2 * (top + r)], n = y_bounds[2 * (top + r) + 1];
    y0 = min(y0, ymin);
    y1 = max(y1, ymin + n);
  }
  y0 = max(y0, 0);
  const int rows = max(0, min(min(y1, H) - y0, max_rows));

  // 1. horizontal pass
  const unsigned char* frame = frames + (size_t)t * H * W * 3;
  for (int i = threadIdx.x; i < rows * row_bytes; i += kFramesThreads) {
    const int row = i / row_bytes, col3 = i - row * row_bytes;
    const int c = col3 / 3, ch = col3 - c * 3;
    const int xmin = x_bounds[2 * (left + c)], n = min(x_bounds[2 * (left + c) + 1], kx);
    const int* k = x_coeffs + (size_t)(left + c) * kx;
    const unsigned char* src = frame + (size_t)(y0 + row) * W * 3 + ch;
    int acc = 1 << (kFramesPrecisionBits - 1);
    for (int j = 0; j < n; ++j) {
      const int x = min(max(xmin + j, 0), W - 1);
      acc += int(__ldg(src + x * 3)) * __ldg(k + j);
    }
    s_rows[i] = (unsigned char)clip8_shift(acc);
  }
  __syncthreads();

  // 2. vertical pass + scaling to [-1, 1] as numpy does it on float32: (x / 127.5f) - 1.0f, each op rounded
  float* dst = out + ((size_t)t * crop_h + r0) * row_bytes;
  for (int i = threadIdx.x; i < (r1 - r0) * row_bytes; i += kFramesThreads) {
    const int r = i / row_bytes, col3 = i - r * row_bytes;
    const int ymin = y_bounds[2 * (top + r0 + r)], n = min(y_bounds[2 * (top + r0 + r) + 1], ky);
    const int* k = y_coeffs + (size_t)(top + r0 + r) * ky;
    int acc = 1 << (kFramesPrecisionBits - 1);
    for (int j = 0; j < n; ++j) {
      const int row = min(max(ymin + j - y0, 0), max(rows - 1, 0));
      acc += int(s_rows[row * row_bytes + col3]) * __ldg(k + j);
    }
    dst[i] = __fsub_rn(__fdiv_rn(float(clip8_shift(acc)), 127.5f), 1.0f);
  }
}

// Upper bound on the input rows that a band of `band_rows` output rows touches: the supports of output rows r0 and r1
// start at int(c_r0 - s + 0.5) >= c_r0 - s - 0.5 and end at int(c_r1 + s + 0.5) <= c_r1 + s + 0.5, with
// c_r1 - c_r0 = (band_rows - 1) * H / out_h and 2s + 1 <= ky; one more row covers the rounding of c_r.
static long long frames_band_rows_bound(int band_rows, int H, int out_h, int ky) {
  const long long span = ((long long)(band_rows - 1) * H + out_h - 1) / out_h + ky + 1;
  return span < H ? span : H;
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_vq_frames_prep(const unsigned char* frames, int T, int H, int W, int C, const int* x_bounds,
                                  const int* x_coeffs, int out_w, int kx, const int* y_bounds, const int* y_coeffs,
                                  int out_h, int ky, int left, int top, int crop_w, int crop_h, float* out,
                                  void* stream) {
  if (!frames || !x_bounds || !x_coeffs || !y_bounds || !y_coeffs || !out)
    return lwm_fail(LWM_ERR_ARG, "vq_frames_prep: null pointer");
  if (C != 3) return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: only 3-channel (RGB) uint8 frames are accepted");
  if (T < 0 || H <= 0 || W <= 0) return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: bad frame sizes");
  if (out_w <= 0 || out_h <= 0 || kx <= 0 || ky <= 0)
    return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: bad resampling tables");
  if (left < 0 || top < 0 || crop_w <= 0 || crop_h <= 0 || crop_w > out_w - left || crop_h > out_h - top)
    return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: crop window outside the resized frame");
  int band_rows = 16;
  long long rows = frames_band_rows_bound(band_rows, H, out_h, ky);
  while (band_rows > 1 && rows * crop_w * 3 > kFramesSmemTarget)
    rows = frames_band_rows_bound(band_rows /= 2, H, out_h, ky);
  const long long smem = rows * crop_w * 3;
  if (smem > kFramesSmemMax) return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: one band does not fit in shared memory");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (T == 0) return LWM_OK;
  const int n_bands = (crop_h + band_rows - 1) / band_rows;
  if ((long long)T * n_bands > 0x7fffffffLL) return lwm_fail(LWM_ERR_SHAPE, "vq_frames_prep: too many frames");
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_set_dev[64] = {};                          // function attributes are per device
  if (!attr_set_dev[dev & 63]) {
    if (cudaFuncSetAttribute(frames_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFramesSmemMax) !=
        cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "vq_frames_prep: cannot raise dynamic shared memory limit");
    attr_set_dev[dev & 63] = true;
  }
  frames_prep_kernel<<<unsigned(T * n_bands), kFramesThreads, size_t(smem), reinterpret_cast<cudaStream_t>(stream)>>>(
      frames, H, W, x_bounds, x_coeffs, kx, y_bounds, y_coeffs, ky, left, top, crop_w, crop_h, band_rows, n_bands,
      int(rows), out);
  return lwm_check_launch("frames_prep_kernel");
}
