// Mask preparation for the tensor-core inference path (attn_fwd_kernel<true, true>): the boolean
// mask [B,1,Q,K] of `ringattention_inference` becomes
//   * bits      [slab][B][Q][n_kt * 4] uint32: bit j of word w <=> key 32 w + j of the slab, 1 = attend; every row
//               is padded to whole 128-key tiles with zeros. A rank packs its query rows once per key slab (one
//               slab per rank of the ring), so each slab can be sent to the rank that holds those keys.
//   * row_any   [B][Q] int32: 1 iff the row has a true entry in any packed slab (the "fully masked" test).
//   * the tile map: per (b, 128-row Q tile) the ascending list of KV tiles to visit, each entry kt * 2 + mixed.
//     A tile is skipped only if every entry of its valid rows is false and no valid row of the Q tile is fully
//     masked (globally: row_any is all-gathered first). It is full (no mask read) if every entry is true and all
//     its keys are < Sk. Fully masked rows make every tile of their Q tile visited and mixed, so they average all
//     keys with the masked logit, as the reference's finfo.min does.
// The source mask is read through its strides: a batch-broadcast mask is never materialised.
#include "attn_common.cuh"
#include "capi_internal.h"

namespace lwm {

constexpr int kPackThreads = 256;

__global__ void __launch_bounds__(kPackThreads)
mask_pack_kernel(const unsigned char* __restrict__ mask, long long sb, long long sq, long long sk, int B, int Q,
                 long long col0, int ncols, int kw, uint32_t* __restrict__ bits, int* __restrict__ row_any) {
  const int q = blockIdx.x, b = blockIdx.y, slab = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned char* src = mask + (long long)b * sb + (long long)q * sq + (col0 + (long long)slab * ncols) * sk;
  uint32_t* dst = bits + (((long long)slab * B + b) * Q + q) * kw;
  int any = 0;
  for (int w = warp; w < kw; w += kPackThreads / 32) {
    const int c = w * 32 + lane;
    const unsigned word = __ballot_sync(0xffffffffu, c < ncols && src[(long long)c * sk] != 0);
    if (lane == 0) dst[w] = word;
    any |= word != 0u;
  }
  if (__syncthreads_or(any) && threadIdx.x == 0) atomicOr(row_any + (long long)b * Q + q, 1);
}

__global__ void __launch_bounds__(kTile)
infer_tilemap_kernel(const uint32_t* __restrict__ bits, const int* __restrict__ row_any, int Q, int Sk, int n_kt,
                     int* __restrict__ tiles, int* __restrict__ tile_count) {
  const int qt = blockIdx.x, b = blockIdx.y;
  const int n_qt = gridDim.x;
  const int row = qt * kTile + threadIdx.x;
  const bool valid = row < Q;
  const bool visit_all = __syncthreads_or(valid && row_any && row_any[(long long)b * Q + row] == 0);
  const uint4* rb = (bits && valid) ? reinterpret_cast<const uint4*>(bits + ((long long)b * Q + row) * (n_kt * 4)) : nullptr;
  int* out = tiles + ((long long)b * n_qt + qt) * n_kt;
  int n = 0;
  for (int kt = 0; kt < n_kt; ++kt) {
    int any_t = valid, all_t = 1;      // no mask: every valid row sees every key
    if (rb) {
      const uint4 w = rb[kt];
      any_t = (w.x | w.y | w.z | w.w) != 0u;
      all_t = (w.x & w.y & w.z & w.w) == ~0u;
    }
    const int any = __syncthreads_or(any_t);
    const int all = __syncthreads_and(all_t);
    if (threadIdx.x == 0 && (any || visit_all)) {
      const bool tail = (kt + 1) * kTile > Sk;
      out[n++] = kt * 2 + ((tail || visit_all || !all) ? 1 : 0);
    }
  }
  if (threadIdx.x == 0) tile_count[(long long)b * n_qt + qt] = n;
}

// The backward's map, transposed: per (b, 128-key tile) the ascending list of 64-row Q tiles, entries t * 2 + mixed.
// Only live rows count (row < Q and row_any set): a fully masked row contributes nothing to any gradient, so it forces
// no visit and does not stop a tile from being clean. A pair is skipped when no live row has a true bit in the tile,
// clean when every live row's bits are all true and every key is < Sk, mixed otherwise.
constexpr int kBwdMapRows = 64;

__global__ void __launch_bounds__(kBwdMapRows)
infer_bwd_tilemap_kernel(const uint32_t* __restrict__ bits, const int* __restrict__ row_any, int Q, int Sk, int n_kt,
                         int n_qt, int* __restrict__ tiles, int* __restrict__ tile_count) {
  const int kt = blockIdx.x, b = blockIdx.y;
  const bool tail = (kt + 1) * kTile > Sk;
  int* out = tiles + ((long long)b * n_kt + kt) * n_qt;
  int n = 0;
  for (int t = 0; t < n_qt; ++t) {
    const int row = t * kBwdMapRows + threadIdx.x;
    const bool live = row < Q && (!row_any || row_any[(long long)b * Q + row] != 0);
    int any_t = live, all_t = 1;      // no mask: every live row sees every key
    if (live && bits) {
      const uint4 w = *reinterpret_cast<const uint4*>(bits + ((long long)b * Q + row) * (n_kt * 4) + kt * 4);
      any_t = (w.x | w.y | w.z | w.w) != 0u;
      all_t = (w.x & w.y & w.z & w.w) == ~0u;
    }
    const int any = __syncthreads_or(any_t);
    const int all = __syncthreads_and(all_t);
    if (threadIdx.x == 0 && any) out[n++] = t * 2 + ((tail || !all) ? 1 : 0);
  }
  if (threadIdx.x == 0) tile_count[(long long)b * n_kt + kt] = n;
}

}  // namespace lwm

using namespace lwm;

// mask: uint8/bool element (b, q, k) at mask[b*stride_b + q*stride_q + k*stride_k] (nonzero = attend; stride_b = 0
// broadcasts one mask over the batch). Packs key columns [col0 + s*ncols, col0 + (s+1)*ncols) for s < n_slabs into
// bits [n_slabs][B][Q][ceil(ncols/128)*4] and row_any [B][Q] (zeroed here, then OR over the slabs).
extern "C" int lwm_attn_mask_pack(const unsigned char* mask, long long stride_b, long long stride_q, long long stride_k,
                                  int B, int Q, long long col0, int ncols, int n_slabs, unsigned* bits, int* row_any,
                                  void* stream) {
  if (!mask || !bits || !row_any) return lwm_fail(LWM_ERR_ARG, "attn_mask_pack: null pointer");
  if (B <= 0 || Q <= 0 || ncols <= 0 || n_slabs <= 0 || B > 65535 || n_slabs > 65535 || col0 < 0 || stride_b < 0 ||
      stride_q < 0 || stride_k <= 0)
    return lwm_fail(LWM_ERR_SHAPE, "attn_mask_pack: bad shape or strides");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(row_any, 0, sizeof(int) * (size_t)B * Q, st) != cudaSuccess)
    return lwm_fail(LWM_ERR_CUDA, "attn_mask_pack: memset failed");
  const int kw = (ncols + kTile - 1) / kTile * 4;
  mask_pack_kernel<<<dim3(Q, B, n_slabs), kPackThreads, 0, st>>>(mask, stride_b, stride_q, stride_k, B, Q, col0, ncols,
                                                                 kw, bits, row_any);
  return lwm_check_launch("mask_pack_kernel");
}

// bits [B][Q][ceil(Sk/128)*4] or null (every key visible); row_any [B][Q] (global over the ring) or null ->
// tiles [B][ceil(Q/128)][ceil(Sk/128)], tile_count [B][ceil(Q/128)] for lwm_attn_infer_partial.
extern "C" int lwm_attn_infer_tilemap(const unsigned* bits, const int* row_any, int B, int Q, int Sk, int* tiles,
                                      int* tile_count, void* stream) {
  if (!tiles || !tile_count) return lwm_fail(LWM_ERR_ARG, "attn_infer_tilemap: null pointer");
  if (B <= 0 || Q <= 0 || Sk <= 0 || B > 65535) return lwm_fail(LWM_ERR_SHAPE, "attn_infer_tilemap: bad shape");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  infer_tilemap_kernel<<<dim3((Q + kTile - 1) / kTile, B), kTile, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      bits, row_any, Q, Sk, (Sk + kTile - 1) / kTile, tiles, tile_count);
  return lwm_check_launch("infer_tilemap_kernel");
}

// bits [B][Q][ceil(Sk/128)*4] or null (every key visible); row_any [B][Q] (global over the ring) or null (every row
// live) -> tiles [B][ceil(Sk/128)][ceil(Q/64)], tile_count [B][ceil(Sk/128)] for lwm_attn_infer_bwd.
extern "C" int lwm_attn_infer_bwd_tilemap(const unsigned* bits, const int* row_any, int B, int Q, int Sk, int* tiles,
                                          int* tile_count, void* stream) {
  if (!tiles || !tile_count) return lwm_fail(LWM_ERR_ARG, "attn_infer_bwd_tilemap: null pointer");
  if (B <= 0 || Q <= 0 || Sk <= 0 || B > 65535 || Q > 0x7fffffff - kBwdMapRows)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd_tilemap: bad shape");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const int n_kt = (Sk + kTile - 1) / kTile, n_qt = (Q + kBwdMapRows - 1) / kBwdMapRows;
  infer_bwd_tilemap_kernel<<<dim3(n_kt, B), kBwdMapRows, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      bits, row_any, Q, Sk, n_kt, n_qt, tiles, tile_count);
  return lwm_check_launch("infer_bwd_tilemap_kernel");
}
