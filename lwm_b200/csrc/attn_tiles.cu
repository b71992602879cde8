// Block map of one training ring step with a padding bias and/or segment ids: which (Q tile, KV tile) pairs the
// forward and backward tile kernels visit, and which of those need the per-element mask (DESIGN §3.6, §5).
//
// Pass 1 (tile_summary_kernel) summarises every 64-row Q block and every 128-key K tile of the step:
//   Q block: min / max segment id, and "proven": every row sees its own key in this step (the bias at the row's own
//            global position is +-0 and that position is one of the step's keys), so its running max is a real logit.
//   K tile:  min / max segment id, and the bias class: zero (every value +-0), masked (every value has
//            bias * log2(e) < kMaskedLogit, the kernels' own test, in fp32) or other.
// Pass 2 (tile_lists_kernel) writes one ascending list per (b, Q tile) for the forward and per (b, K tile) for the
// backward, entries t * 2 + mixed, over the causal range only. A pair is skipped when the K tile is masked or the two
// segment ranges are disjoint (every entry of the pair is masked); it is clean (no bias or segment read) when the bias
// is zero or absent and the segments are absent or one single id; mixed otherwise. A forward Q tile with a row that is
// not proven visits its whole causal range as mixed: such a row may see no key at all and must then average every
// visited key with the masked logit. The backward skips for every row: a masked entry has P = 0 there.
#include "attn_common.cuh"
#include "capi_internal.h"
#include <climits>

namespace lwm {

constexpr int kSumThreads = 128;
constexpr int kBQBlock = 64;   // query rows per backward Q tile
enum { kBiasZero = 0, kBiasMasked = 1, kBiasOther = 2 };

LWM_DEVICE int block_min(int v, int* red) {
  v = __reduce_min_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return min(min(red[0], red[1]), min(red[2], red[3]));
}

LWM_DEVICE int block_max(int v, int* red) {
  v = __reduce_max_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return max(max(red[0], red[1]), max(red[2], red[3]));
}

// blockIdx.x < n_q64: Q block blockIdx.x (threads >= 64 idle) ; else K tile blockIdx.x - n_q64. One int4 each:
// (seg min, seg max, proven | bias class, 0).
__global__ void __launch_bounds__(kSumThreads)
tile_summary_kernel(const float* __restrict__ bias, long long bias_stride, const int* __restrict__ seg,
                    long long seg_stride, int q_pos0, int k_pos0, int Sk, int n_q64, int n_kt,
                    int4* __restrict__ qsum, int4* __restrict__ ksum) {
  __shared__ int red[kSumThreads / 32];
  const int blk = blockIdx.x, b = blockIdx.y;
  const bool is_q = blk < n_q64;
  const bool active = !is_q || threadIdx.x < kBQBlock;
  const int pos = is_q ? q_pos0 + blk * kBQBlock + int(threadIdx.x) : k_pos0 + (blk - n_q64) * kTile + int(threadIdx.x);
  const float* bias_row = bias ? bias + (long long)b * bias_stride : nullptr;
  const int sid = (seg && active) ? seg[(long long)b * seg_stride + pos] : 0;
  const int smin = block_min(active ? sid : INT_MAX, red);
  const int smax = block_max(active ? sid : INT_MIN, red);
  if (is_q) {
    // the own key is checked against the step's key range before the bias is read: bias_stride >= k_pos0 + Sk only
    const bool own = pos >= k_pos0 && pos < k_pos0 + Sk && (!bias_row || bias_row[pos] == 0.f);
    const int proven = __syncthreads_and(!active || own);
    if (threadIdx.x == 0) qsum[(long long)b * n_q64 + blk] = make_int4(smin, smax, proven, 0);
  } else {
    const float bv = bias_row ? bias_row[pos] : 0.f;
    const int all_zero = __syncthreads_and(bv == 0.f);
    const int all_masked = __syncthreads_and(bias_row && __fmul_rn(bv, kLog2e) < kMaskedLogit);
    const int cls = all_zero ? kBiasZero : all_masked ? kBiasMasked : kBiasOther;
    if (threadIdx.x == 0) ksum[(long long)b * n_kt + (blk - n_q64)] = make_int4(smin, smax, cls, 0);
  }
}

// 0 skip, 1 clean, 2 mixed
LWM_DEVICE int classify(int4 q, int4 k, bool has_seg) {
  if (k.z == kBiasMasked || (has_seg && (q.y < k.x || k.y < q.x))) return 0;
  if (k.z == kBiasZero && (!has_seg || (q.x == q.y && k.x == k.y && q.x == k.x))) return 1;
  return 2;
}

// one warp per list; blockIdx.x < n_qt: forward list of Q tile blockIdx.x ; else backward list of K tile
// blockIdx.x - n_qt. Either half may be absent (null outputs).
__global__ void __launch_bounds__(32)
tile_lists_kernel(const int4* __restrict__ qsum, const int4* __restrict__ ksum, int has_seg, int q_pos0, int k_pos0,
                  int causal, int n_q64, int n_kt, int* __restrict__ fwd_tiles, int* __restrict__ fwd_count,
                  int* __restrict__ bwd_tiles, int* __restrict__ bwd_count) {
  const int lane = threadIdx.x, b = blockIdx.y;
  const int n_qt = fwd_tiles ? n_q64 / 2 : 0;
  const int4* qs = qsum + (long long)b * n_q64;
  const int4* ks = ksum + (long long)b * n_kt;
  int n = 0;
  if ((int)blockIdx.x < n_qt) {
    const int t = blockIdx.x;
    const int4 a = qs[2 * t], c = qs[2 * t + 1];
    const int4 q = make_int4(min(a.x, c.x), max(a.y, c.y), a.z & c.z, 0);
    int n_vis = n_kt;   // KV tiles any row of the Q tile can see: as attn_fwd_kernel computes it
    if (causal) {
      const long long vis = (long long)q_pos0 + (long long)t * kTile + kTile - 1 - k_pos0;
      n_vis = vis < 0 ? 0 : (int)min((long long)n_kt, vis / kTile + 1);
    }
    int* out = fwd_tiles + ((long long)b * n_qt + t) * n_kt;
    for (int base = 0; base < n_vis; base += 32) {
      const int kt = base + lane;
      const int cls = kt < n_vis ? (q.z ? classify(q, ks[kt], has_seg) : 2) : 0;
      const unsigned keep = __ballot_sync(0xffffffffu, cls != 0);
      if (cls) out[n + __popc(keep & ((1u << lane) - 1u))] = kt * 2 + (cls == 2);
      n += __popc(keep);
    }
    if (lane == 0) fwd_count[(long long)b * n_qt + t] = n;
  } else {
    const int kt = blockIdx.x - n_qt;
    int i_start = 0;   // first Q tile with a row that can see key 0 of this K tile: as attn_bwd_kernel computes it
    if (causal) {
      const long long diff = (long long)k_pos0 + (long long)kt * kTile - q_pos0;
      i_start = diff <= 0 ? 0 : (int)min(diff / kBQBlock, (long long)n_q64);
    }
    const int4 k = ks[kt];
    int* out = bwd_tiles + ((long long)b * n_kt + kt) * n_q64;
    for (int base = i_start; base < n_q64; base += 32) {
      const int qi = base + lane;
      const int cls = qi < n_q64 ? classify(qs[qi], k, has_seg) : 0;
      const unsigned keep = __ballot_sync(0xffffffffu, cls != 0);
      if (cls) out[n + __popc(keep & ((1u << lane) - 1u))] = qi * 2 + (cls == 2);
      n += __popc(keep);
    }
    if (lane == 0) bwd_count[(long long)b * n_kt + kt] = n;
  }
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_attn_step_tilemap(const float* bias, long long bias_stride, const int* segment_ids,
                                     long long seg_stride, int B, int Sq, int Sk, long long q_pos0, long long k_pos0,
                                     int causal, int* fwd_tiles, int* fwd_count, int* bwd_tiles, int* bwd_count,
                                     void* workspace, void* stream) {
  if (!bias && !segment_ids) return lwm_fail(LWM_ERR_ARG, "attn_step_tilemap: bias or segment_ids required");
  if (!fwd_tiles != !fwd_count || !bwd_tiles != !bwd_count || (!fwd_tiles && !bwd_tiles) || !workspace)
    return lwm_fail(LWM_ERR_ARG, "attn_step_tilemap: null pointer (tiles and counts of a map go together)");
  if (B <= 0 || B > 65535 || Sq <= 0 || Sk <= 0 || Sq % kTile || Sk % kTile)
    return lwm_fail(LWM_ERR_SHAPE, "attn_step_tilemap: Sq and Sk must be positive multiples of 128, B <= 65535");
  if (q_pos0 < 0 || k_pos0 < 0 || q_pos0 + Sq > 0x7fffffffLL || k_pos0 + Sk > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_step_tilemap: global positions must be >= 0 and fit in int32");
  if (bias && bias_stride < k_pos0 + Sk)
    return lwm_fail(LWM_ERR_SHAPE, "attn_step_tilemap: bias is indexed by GLOBAL key position: bias_stride < k_pos0 + Sk");
  if (segment_ids && (seg_stride < q_pos0 + Sq || seg_stride < k_pos0 + Sk))
    return lwm_fail(LWM_ERR_SHAPE, "attn_step_tilemap: segment_ids is indexed by GLOBAL position: seg_stride < max(q_pos0 + Sq, k_pos0 + Sk)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n_q64 = Sq / kBQBlock, n_kt = Sk / kTile;
  int4* qsum = reinterpret_cast<int4*>(workspace);
  int4* ksum = qsum + (long long)B * n_q64;
  tile_summary_kernel<<<dim3(n_q64 + n_kt, B), kSumThreads, 0, st>>>(bias, bias_stride, segment_ids, seg_stride,
                                                                    int(q_pos0), int(k_pos0), Sk, n_q64, n_kt, qsum, ksum);
  const int st1 = lwm_check_launch("tile_summary_kernel");
  if (st1) return st1;
  const int n_lists = (fwd_tiles ? Sq / kTile : 0) + (bwd_tiles ? n_kt : 0);
  tile_lists_kernel<<<dim3(n_lists, B), 32, 0, st>>>(qsum, ksum, segment_ids != nullptr, int(q_pos0), int(k_pos0),
                                                     causal, n_q64, n_kt, fwd_tiles, fwd_count, bwd_tiles, bwd_count);
  return lwm_check_launch("tile_lists_kernel");
}
