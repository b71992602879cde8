// Ring-attention backward tile kernel for sm_90a.
//
// One launch = one ring step of the reference's custom_vjp backward (SURVEY.md Appendix A `bwd`;
// the op is bound at lwm/llama.py:541): for the held K/V block, recompute P from (q, k, lse) and
// accumulate dV += P^T dO, dK += dS^T Q / sqrt(D), dQ += dS K / sqrt(D) with
// dS = P o (dO V^T - rowsum(dO o O)).
//
// Mapping to the hardware (K/V-stationary, everything computed TRANSPOSED so that the key index is
// the M dimension and P^T / dS^T feed the dV / dK wgmmas straight from registers):
//   CTA = one 128-key tile of one (batch, head); loop over the 64-row Q tiles that can see it.
//   warpgroups 0 / 1 own keys [0,64) / [64,128) of the tile; per Q tile each runs (bf16 or fp16 in,
//   fp32 accumulators in registers):
//     S^T  = K  Q^T     m64n64   both operands K-major in shared memory
//     dP^T = V  dO^T    m64n64   both operands K-major in shared memory
//     dV  += P^T dO     m64n128  A = P^T from registers, dO read MN-major
//     dK  += dS^T Q     m64n128  A = dS^T from registers, Q read MN-major
//     dQ   = dS  K      m64n64   A = the shared dS^T tile read MN-major (all 128 keys), B = this
//                                warpgroup's 64 columns of K read MN-major; staged in shared memory
//                                as fp32 and added to dq_acc by a TMA reduction.
//   warp 8: TMA loads (K, V once; Q + dO + lse + delta double-buffered).
//   warp 9: dQ reductions (cp.reduce.async.bulk.tensor add, from a double-buffered fp32 staging tile).
//   warps 10, 11: idle.
// Inside an iteration each wgmma group is waited for only where its result is needed: exp(S^T) runs under
// dP^T, dS^T under dV, and the dS^T handoff between the warpgroups under dK.
// The softmax scale is folded into dS before it is rounded, so dK and dQ need no epilogue scaling.
// dk_acc / dv_acc are accumulated read-modify-write by the one CTA that owns the tile.
#include "attn_common.cuh"
#include "attn_dropout.cuh"
#include "tmap.h"
#include "capi_internal.h"
#include <type_traits>

namespace lwm {

struct BwdParams {
  int B, H, Sq, Sk;
  float scale;       // softmax_scale
  float scale_log2;  // softmax_scale * log2(e)
  MaskParams mask;
  const float* lse;    // [B,H,Sq] PRE-SCALED: -lse*log2(e) (lwm_attn_bwd_lse), -inf for rows without any unmasked key
  const float* delta;  // [B,H,Sq]
  float* dq_acc;       // [B,Sq,H,D] fp32
  float* dk_acc;       // [B,Sk,H,D] fp32
  float* dv_acc;       // [B,Sk,H,D] fp32
  const float *scale_q, *scale_k, *scale_v, *scale_do;   // fp16 mode: device scalars (x = x16 * scale); else null
  int dkv_init;        // 1: dk_acc/dv_acc rows of this launch are WRITTEN (first visit of the block), 0: accumulated
  // kMap (a bias or segment ids): the backward map of lwm_attn_step_tilemap, per (b, K tile) the ascending list of
  // 64-row Q tiles, entries qt * 2 + mixed
  const int* tiles;       // [B, Sk/128, Sq/64]
  const int* tile_count;  // [B, Sk/128]
  // kBits (the backward of ringattention_inference): Sq is the query length rounded up to 64 (the row stride of lse,
  // delta and the lists), q_rows the real one; Sk is the real key length (any value, K tiles = gridDim.x). bits is the
  // forward's mask, [B, q_rows, gridDim.x * 4] words (bit j of word w <=> key 32 w + j; 1 = attend), or null.
  const uint32_t* bits;
  int q_rows;
  // kOrdered: order_ws = [ticket, error flag, dQ semaphores [B][H][Sq/64]] (zeroed by the entry point); with kMap,
  // turns [B, Sk/128, Sq/64] holds each list entry's turn (dq_turns_kernel)
  int* order_ws;
  const int* turns;
  DropParams drop;     // kDrop: the attention-dropout mask (attn_dropout.cuh)
};

constexpr int kBQ = 64;                         // query rows per inner iteration
constexpr int kBwdThreads = 384;                // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kBwdConsumerWarps = 8;
constexpr int kTB = kTile * kHeadDim * 2;       // 32 KB: a 128-row bf16 tile
constexpr int kQB = kBQ * kHeadDim * 2;         // 16 KB: a 64-row bf16 tile
constexpr int kDSB = kTile * kBQ * 2;           // 16 KB: dS^T of one Q tile (128 keys x 64 queries, 16 bit)
constexpr int kDQB = kBQ * kHeadDim * 4;        // 32 KB: fp32 dQ tile (64 queries x 128 columns)
constexpr int kDQBox = kBQ * 32 * 4;            // 8 KB: one 32-column box of the dQ tile (128 B rows, swizzled)
// smem map (bytes): K | V | Q0 Q1 | dO0 dO1 | dS^T 0 1 | dQ 0 1 | lse[2] | delta[2] | barriers
constexpr int kOffK = 0, kOffV = kTB, kOffQ = 2 * kTB, kOffDO = kOffQ + 2 * kQB, kOffDS = kOffDO + 2 * kQB;
constexpr int kOffDQ = kOffDS + 2 * kDSB;
constexpr int kOffLse = kOffDQ + 2 * kDQB, kOffDelta = kOffLse + 2 * kBQ * 4, kOffBars = kOffDelta + 2 * kBQ * 4;
constexpr int kBwdSmemBytes = kOffBars + 128;
static_assert(kBwdSmemBytes <= 227 * 1024, "attn_bwd: shared memory over the sm_90 per-block limit");
static_assert(kOffDQ % 1024 == 0, "128B-swizzled TMA tiles need 1024-byte alignment");

struct BwdBarriers {
  uint64_t kv_full;
  uint64_t q_full[2], q_empty[2];   // Q + dO + lse + delta of one Q tile
  uint64_t dq_full[2], dq_empty[2]; // fp32 dQ staging tile: written by the consumers, reduced by warp 9
};
// kMap: the list entry of the Q tile in stage st, written by the producer before it arms q_full[st] (the consumers read
// it there instead of holding a pointer into the list across their loop)
constexpr int kOffEntry = kOffBars + 96;
// kOrdered: the (n, h, b) of the CTA's ticket, written by thread 0
constexpr int kOffTicket = kOffEntry + 2 * 4;
static_assert(sizeof(BwdBarriers) <= 96 && 96 + 5 * 4 <= 128, "attn_bwd: barrier block layout");

// ---- kOrdered: dQ reduced in a fixed key-tile order (lwm_attn_bwd_step_ordered, lwm_attn_infer_bwd_ordered)
// Every element of dQ tile (b, h, 64-row Q tile i) receives the contributions of its key tiles in ascending key-tile
// order, so dQ is the same bits on every run. Each (b, h, i) has a semaphore, the number of key tiles that have added
// into the tile. Warp 9 of key tile n waits until it equals n's turn, the number of key tiles below n that reduce into
// tile i (without a map they are a prefix, as i_start is monotone in n: the turn is n), issues its four reductions,
// waits for them to complete, and increments the semaphore.
// Forward progress does not rest on the order in which CTAs are dispatched: each CTA takes a ticket with one atomicAdd
// when it starts and works on the (n, h, b) the ticket names, h fastest, then b, then n. A CTA only waits on key tiles
// below its own, whose tickets are smaller; their CTAs have started, so they are resident or finished, and by induction
// on the ticket every wait ends. (With n fastest, neighbouring key tiles of one head would run together and each would
// stall behind the one before it.)
// Memory ordering (PTX memory consistency model): the reductions are async-proxy writes of global memory. The
// signaller waits for their completion (cp.async.bulk.wait_group 0: the writes are performed, not only the smem source
// read), orders them before its generic-proxy accesses with fence.proxy.async.global, and publishes with a release
// increment at gpu scope. The waiter's ld.acquire.gpu that reads the new count synchronises with that release, and its
// fence.proxy.async.global orders the acquire before its own async-proxy reductions. So the previous key tile's adds
// happen before the next one's, element for element.
constexpr int kOrderHeader = 2;                          // order_ws[0] ticket, order_ws[1] error flag
constexpr unsigned long long kTurnTimeoutNs = 4000000000ull;

LWM_DEVICE void take_ticket(int* counter, int H, int B, volatile int* s_nhb) {
  if (threadIdx.x == 0) {
    const int t = atomicAdd(counter, 1);
    s_nhb[0] = t / (H * B);
    s_nhb[1] = t % H;
    s_nhb[2] = t / H % B;
  }
  __syncthreads();
}

// Spin until *sem == turn. A wait longer than kTurnTimeoutNs is a bug (a turn that never comes): it sets the error flag
// and carries on with the reduction, so it shows up as a flag the caller reads and never as a hang.
LWM_DEVICE void dq_wait_turn(const int* sem, int turn, int* err) {
  if (ld_acquire_gpu(sem) != turn) {
    const uint64_t t0 = globaltimer_ns();
    uint32_t ns = 32;
    while (ld_acquire_gpu(sem) != turn) {
      __nanosleep(ns);
      ns = min(ns * 2, 1024u);
      if (globaltimer_ns() - t0 > kTurnTimeoutNs) {
        atomicOr(err, 1);
        break;
      }
    }
  }
  fence_proxy_async_global();
}

LWM_DEVICE void dq_pass_turn(int* sem) {
  tma_wait_group<0>();
  fence_proxy_async_global();
  red_release_gpu_add(sem, 1);
}

LWM_DEVICE void load_tile_nb(uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int h, int row0, int b, int half_bytes) {
  tma_load_4d(dst, tm, bar, 0, h, row0, b);
  tma_load_4d(dst + half_bytes, tm, bar, 64, h, row0, b);
}

// kF16: fp16 operands (exact scaled copies of the bf16 inputs), P^T and dS^T kept in fp16. dS^T is rounded in the
// units of the fp16 operands, i.e. divided by scale_do * scale_v, so its magnitude does not depend on how large dO and
// V are (real upstream gradients are 1e-6 .. 1e-10 of unit scale): with |dO16|, |V16| < 2^13 and D = 128,
// |dP16 - delta16| <= 2 * 128 * 2^13 * 2^13 = 2^34 and P <= 1, so softmax_scale * P * (dP16 - delta16) * 2^-15 stays
// below 2^15.5 < 65504 for any input. Every scale factor is undone in fp32 where the results leave the tensor cores
// (dQ atomics, dK/dV epilogue); all of them are powers of two, so the gradients scale exactly with dO and V.
constexpr float kDsNorm = 1.0f / 32768.0f;
// P^T = exp(s - lse) is a NORMALISED probability: at 128K .. 1M keys a typical entry is 1e-5 .. 1e-6, below fp16's
// smallest normal (6.1e-5), where it would lose its 11 bits. The fp16 kernel therefore works on P * 2^14 (<= 16384,
// never overflows; normal down to 3.7e-9): the host folds the +14 into the pre-scaled lse (lwm_attn_bwd_lse,
// offset_log2 = LWM_ATTN_F16_P_BOOST_LOG2) and the factor is undone in fp32 in the dV epilogue and in the dS scale.
constexpr float kPBoostInv = 1.0f / 16384.0f;

// kMap: the CTA walks its K tile's list of Q tiles instead of i_start .. n_q_tiles (pairs whose entries are all masked
// are not in it: they would add exact zeros); mixed tiles run the per-element mask, clean tiles the same branch with no
// bias or segment read.
// kBits (with kMap): the backward of the inference op. The lists come from lwm_attn_infer_bwd_tilemap; clean tiles take
// the unmasked path, mixed tiles read one mask word per query column and give masked entries and keys >= Sk P = 0.
// Rows >= q_rows and rows without any visible key carry lse = -inf (P = 0, dS = 0). Q / dO rows past q_rows and K / V
// rows past Sk are zero-filled by TMA, the dQ reduction clips rows >= q_rows, and dK / dV rows >= Sk are not written.
// kOrdered: dQ is reduced in ascending key-tile order (above); the grid's shape is the same, blockIdx is not used.
// kDrop (training instances): attention dropout. Every visited tile runs the per-element branch, which regenerates the
// forward's mask and gives a dropped entry the masked logit (P = 0, dS = 0). Rows the forward left without a surviving
// key arrive with lse = -inf.
template <bool kF16, bool kMap = false, bool kBits = false, bool kOrdered = false>
__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  constexpr bool kDrop = false;
#include "attn_bwd_body.cuh"
}

template <bool kF16, bool kMap, bool kOrdered>
__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_dropout_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                        const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  constexpr bool kBits = false, kDrop = true;
#include "attn_bwd_body.cuh"
}

static bool make_bf16_tmap(CUtensorMap* tm, const void* ptr, int B, int S, int H, int box_rows) {
  uint64_t dims[4] = {uint64_t(kHeadDim), uint64_t(H), uint64_t(S), uint64_t(B)};
  uint64_t strides[3] = {uint64_t(kHeadDim) * 2, uint64_t(H) * kHeadDim * 2, uint64_t(S) * H * kHeadDim * 2};
  uint32_t box[4] = {64, 1, uint32_t(box_rows), 1};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// fp32 [B, S, H, 128] accumulator, boxes of 32 columns (128 B, swizzled) x box_rows rows: the dQ reduction target
static bool make_f32_tmap(CUtensorMap* tm, const void* ptr, int B, int S, int H, int box_rows) {
  uint64_t dims[4] = {uint64_t(kHeadDim), uint64_t(H), uint64_t(S), uint64_t(B)};
  uint64_t strides[3] = {uint64_t(kHeadDim) * 4, uint64_t(H) * kHeadDim * 4, uint64_t(S) * H * kHeadDim * 4};
  uint32_t box[4] = {32, 1, uint32_t(box_rows), 1};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// turns[b][n][pos] = #{n' < n : the list of K tile n' holds Q tile tiles[b][n][pos] >> 1}, over the backward lists of
// lwm_attn_step_tilemap and lwm_attn_infer_bwd_tilemap (the same format): the turn of each list entry in the ordered dQ
// reduction. One warp per (b, Q tile) walks the K tiles 32 at a time, finds the Q tile in each ascending list by
// binary search and numbers the lists that hold it in key-tile order. Entries past a list's count are not written.
constexpr int kTurnThreads = 128;
__global__ void __launch_bounds__(kTurnThreads)
dq_turns_kernel(const int* __restrict__ tiles, const int* __restrict__ counts, int n_kt, int n_q64,
                int* __restrict__ turns) {
  const int qt = int((blockIdx.x * kTurnThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31, b = blockIdx.y;
  if (qt >= n_q64) return;   // whole warps
  int turn = 0;
  for (int base = 0; base < n_kt; base += 32) {
    const int kt = base + lane;
    int pos = -1;
    if (kt < n_kt) {
      const long long lt = (long long)b * n_kt + kt;
      const int* list = tiles + lt * n_q64;
      const int cnt = counts[lt];
      int lo = 0, hi = cnt;   // first entry whose Q tile is >= qt
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((list[mid] >> 1) < qt) lo = mid + 1;
        else hi = mid;
      }
      if (lo < cnt && (list[lo] >> 1) == qt) pos = lo;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, pos >= 0);
    if (pos >= 0) turns[((long long)b * n_kt + kt) * n_q64 + pos] = turn + __popc(hit & ((1u << lane) - 1u));
    turn += __popc(hit);
  }
}

template <bool kF16, bool kMap, bool kBits, bool kOrdered, bool kDrop = false>
static int launch_bwd(dim3 grid, cudaStream_t st, const CUtensorMap (&tm)[5], const BwdParams& p, const char* what) {
  void (*kernel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, BwdParams);
  if constexpr (kDrop) kernel = attn_bwd_dropout_kernel<kF16, kMap, kOrdered>;
  else kernel = attn_bwd_kernel<kF16, kMap, kBits, kOrdered>;
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63];      // function attributes are per device
  if (!attr_set) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmemBytes) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "attn_bwd: cannot raise dynamic shared memory limit");
    attr_set = true;
  }
  kernel<<<grid, kBwdThreads, kBwdSmemBytes, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], p);
  return lwm_check_launch(what);
}

// The ordered launches' set-up on the call's stream: the ticket, the error flag and n_sem dQ semaphores are zeroed, and
// with a block map its turns are written after the semaphores.
static int order_prologue(int* order_ws, long long n_sem, const int* tiles, const int* tile_count, int B, int n_kt,
                          int n_q64, cudaStream_t st, BwdParams& p) {
  if (cudaMemsetAsync(order_ws, 0, (kOrderHeader + n_sem) * sizeof(int), st) != cudaSuccess)
    return lwm_fail(LWM_ERR_CUDA, "attn_bwd (ordered): cudaMemsetAsync of order_ws failed");
  p.order_ws = order_ws;
  p.turns = nullptr;
  if (!tiles) return LWM_OK;
  int* turns = order_ws + kOrderHeader + n_sem;
  constexpr int kWarps = kTurnThreads / 32;
  dq_turns_kernel<<<dim3((n_q64 + kWarps - 1) / kWarps, B), kTurnThreads, 0, st>>>(tiles, tile_count, n_kt, n_q64,
                                                                                    turns);
  p.turns = turns;
  return lwm_check_launch("dq_turns_kernel");
}

// Size checks of the ordered launches: semaphore indices, tickets and turn indices are int32.
static bool order_fits(int B, int H, int n_kt, int n_q64, bool map) {
  const long long sem = (long long)B * H * n_q64, tickets = (long long)B * H * n_kt;
  const long long turns = map ? (long long)B * n_kt * n_q64 : 0;
  return B <= 65535 && H <= 65535 && kOrderHeader + sem + turns <= 0x7fffffffLL && tickets <= 0x7fffffffLL;
}

}  // namespace lwm

using namespace lwm;

// One ring step; order_ws null: the unordered reduction of lwm_attn_bwd_step, else lwm_attn_bwd_step_ordered's.
static int bwd_step(const void* q, const void* k, const void* v, const void* dout, const float* scale_q,
                    const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                    const float* delta, float* dq_acc, float* dk_acc, float* dv_acc, int B, int H, int Sq, int Sk,
                    int D, long long q_pos0, long long k_pos0, int causal, const float* bias, long long bias_stride,
                    const int* segment_ids, long long seg_stride, float softmax_scale, int dkv_init, const int* tiles,
                    const int* tile_count, int* order_ws, const DropParams* drop, void* stream) {
  if (!scale_k != !scale_q || !scale_v != !scale_q || !scale_do != !scale_q)
    return lwm_fail(LWM_ERR_ARG, "attn_bwd: scales are all given (fp16 operands) or all null (bf16)");
  if (!tiles != !tile_count) return lwm_fail(LWM_ERR_ARG, "attn_bwd: tiles and tile_count are both given or both null");
  if (tiles && !bias && !segment_ids) return lwm_fail(LWM_ERR_ARG, "attn_bwd: a block map needs bias or segment_ids");
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: head_dim must be 128");
  if (B <= 0 || H <= 0 || Sq <= 0 || Sk <= 0 || Sq % kTile || Sk % kTile)
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: Sq and Sk must be positive multiples of 128");
  if (!q || !k || !v || !dout || !lse || !delta || !dq_acc || !dk_acc || !dv_acc)
    return lwm_fail(LWM_ERR_ARG, "attn_bwd: null pointer");
  if (q_pos0 + Sq > 0x7fffffffLL || k_pos0 + Sk > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: global positions must fit in int32");
  if (bias && bias_stride < k_pos0 + Sk)
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: bias is indexed by GLOBAL key position: bias_stride < k_pos0 + Sk");
  if (segment_ids && (seg_stride < q_pos0 + Sq || seg_stride < k_pos0 + Sk))
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: segment_ids is indexed by GLOBAL position: seg_stride < max(q_pos0 + Sq, k_pos0 + Sk)");
  if (tiles && (long long)B * (Sk / kTile) * (Sq / kBQ) > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd: B * Sk/128 * Sq/64 must fit in int32 with a block map");
  if (order_ws && !order_fits(B, H, Sk / kTile, Sq / kBQ, tiles != nullptr))
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd_ordered: B, H <= 65535 and the order_ws words, B * H * Sk/128 must fit in int32");
  if (drop && (q_pos0 % kTile || k_pos0 % kTile))
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd_dropout: q_pos0 and k_pos0 must each be a multiple of 128");
  if (drop && (B > 65535 || H > 65535 || (long long)drop->batch0 + B > 0x7fffffffLL))
    return lwm_fail(LWM_ERR_SHAPE, "attn_bwd_dropout: B, H <= 65535 and batch0 + B < 2^31");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tm[5];   // q, k, v, dout, dq_acc
  if (!make_bf16_tmap(&tm[0], q, B, Sq, H, kBQ) || !make_bf16_tmap(&tm[1], k, B, Sk, H, kTile) ||
      !make_bf16_tmap(&tm[2], v, B, Sk, H, kTile) || !make_bf16_tmap(&tm[3], dout, B, Sq, H, kBQ) ||
      !make_f32_tmap(&tm[4], dq_acc, B, Sq, H, kBQ))
    return lwm_fail(LWM_ERR_CUDA, "attn_bwd: cuTensorMapEncodeTiled failed (pointers must be 16B aligned)");
  BwdParams p{};
  p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk;
  p.scale = softmax_scale;
  p.scale_log2 = softmax_scale * kLog2e;
  p.mask.q_pos0 = int(q_pos0); p.mask.k_pos0 = int(k_pos0); p.mask.causal = causal;
  p.mask.bias = bias; p.mask.bias_stride = bias_stride;
  p.mask.seg = segment_ids; p.mask.seg_stride = seg_stride;
  p.lse = lse; p.delta = delta; p.dq_acc = dq_acc; p.dk_acc = dk_acc; p.dv_acc = dv_acc;
  p.scale_q = scale_q; p.scale_k = scale_k; p.scale_v = scale_v; p.scale_do = scale_do;
  p.dkv_init = dkv_init ? 1 : 0;
  p.tiles = tiles; p.tile_count = tile_count;
  p.order_ws = nullptr; p.turns = nullptr;
  dim3 grid(Sk / kTile, H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (order_ws) {
    const int s = order_prologue(order_ws, (long long)B * H * (Sq / kBQ), tiles, tile_count, B, Sk / kTile, Sq / kBQ,
                                 st, p);
    if (s) return s;
    if (drop) {
      p.drop = *drop;
      if (tiles)
        return scale_q ? launch_bwd<true, true, false, true, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (ordered, block map)")
                       : launch_bwd<false, true, false, true, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (ordered, block map)");
      return scale_q ? launch_bwd<true, false, false, true, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (ordered)")
                     : launch_bwd<false, false, false, true, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (ordered)");
    }
    if (tiles)
      return scale_q ? launch_bwd<true, true, false, true>(grid, st, tm, p, "attn_bwd_kernel (ordered, block map)")
                     : launch_bwd<false, true, false, true>(grid, st, tm, p, "attn_bwd_kernel (ordered, block map)");
    return scale_q ? launch_bwd<true, false, false, true>(grid, st, tm, p, "attn_bwd_kernel (ordered)")
                   : launch_bwd<false, false, false, true>(grid, st, tm, p, "attn_bwd_kernel (ordered)");
  }
  if (drop) {
    p.drop = *drop;
    if (tiles)
      return scale_q ? launch_bwd<true, true, false, false, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (block map)")
                     : launch_bwd<false, true, false, false, true>(grid, st, tm, p, "attn_bwd_dropout_kernel (block map)");
    return scale_q ? launch_bwd<true, false, false, false, true>(grid, st, tm, p, "attn_bwd_dropout_kernel")
                   : launch_bwd<false, false, false, false, true>(grid, st, tm, p, "attn_bwd_dropout_kernel");
  }
  if (tiles)
    return scale_q ? launch_bwd<true, true, false, false>(grid, st, tm, p, "attn_bwd_kernel (block map)")
                   : launch_bwd<false, true, false, false>(grid, st, tm, p, "attn_bwd_kernel (block map)");
  return scale_q ? launch_bwd<true, false, false, false>(grid, st, tm, p, "attn_bwd_kernel")
                 : launch_bwd<false, false, false, false>(grid, st, tm, p, "attn_bwd_kernel");
}

// One ring step (include/lwm_b200.h): the scales select the fp16-operand kernel, tiles / tile_count the block map.
extern "C" int lwm_attn_bwd_step(const void* q, const void* k, const void* v, const void* dout, const float* scale_q,
                                 const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                                 const float* delta, float* dq_acc, float* dk_acc, float* dv_acc, int B, int H,
                                 int Sq, int Sk, int D, long long q_pos0, long long k_pos0, int causal,
                                 const float* bias, long long bias_stride, const int* segment_ids,
                                 long long seg_stride, float softmax_scale, int dkv_init, const int* tiles,
                                 const int* tile_count, void* stream) {
  return bwd_step(q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc, dk_acc, dv_acc, B, H, Sq, Sk,
                  D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale, dkv_init, tiles,
                  tile_count, nullptr, nullptr, stream);
}

// lwm_attn_bwd_step with dQ reduced in ascending key-tile order (include/lwm_b200.h)
extern "C" int lwm_attn_bwd_step_ordered(const void* q, const void* k, const void* v, const void* dout,
                                         const float* scale_q, const float* scale_k, const float* scale_v,
                                         const float* scale_do, const float* lse, const float* delta, float* dq_acc,
                                         float* dk_acc, float* dv_acc, int B, int H, int Sq, int Sk, int D,
                                         long long q_pos0, long long k_pos0, int causal, const float* bias,
                                         long long bias_stride, const int* segment_ids, long long seg_stride,
                                         float softmax_scale, int dkv_init, const int* tiles, const int* tile_count,
                                         int* order_ws, void* stream) {
  if (!order_ws) return lwm_fail(LWM_ERR_ARG, "attn_bwd_ordered: null order_ws");
  return bwd_step(q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc, dk_acc, dv_acc, B, H, Sq, Sk,
                  D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale, dkv_init, tiles,
                  tile_count, order_ws, nullptr, stream);
}

// lwm_attn_bwd_step (order_ws null) or lwm_attn_bwd_step_ordered (order_ws given) with attention dropout
// (include/lwm_b200.h)
extern "C" int lwm_attn_bwd_step_dropout(const void* q, const void* k, const void* v, const void* dout,
                                         const float* scale_q, const float* scale_k, const float* scale_v,
                                         const float* scale_do, const float* lse, const float* delta, float* dq_acc,
                                         float* dk_acc, float* dv_acc, int B, int H, int Sq, int Sk, int D,
                                         long long q_pos0, long long k_pos0, int causal, const float* bias,
                                         long long bias_stride, const int* segment_ids, long long seg_stride,
                                         float softmax_scale, int dkv_init, const int* tiles, const int* tile_count,
                                         int* order_ws, long long seed, unsigned drop_threshold, int batch0,
                                         void* stream) {
  if (drop_threshold == 0 || drop_threshold > 65535)
    return lwm_fail(LWM_ERR_ARG, "attn_bwd_dropout: drop_threshold must be in [1, 65535] (0 is lwm_attn_bwd_step)");
  if (batch0 < 0) return lwm_fail(LWM_ERR_ARG, "attn_bwd_dropout: batch0 must be >= 0");
  const DropParams d = {uint32_t(uint64_t(seed)), uint32_t(uint64_t(seed) >> 32), drop_threshold, uint32_t(batch0)};
  return bwd_step(q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc, dk_acc, dv_acc, B, H, Sq, Sk,
                  D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale, dkv_init, tiles,
                  tile_count, order_ws, &d, stream);
}

// Backward of ringattention_inference (attn_bwd_kernel<true, true, true>): any Q and Sk. q16 / dout16 [B,Q,H,128],
// k16 / v16 [B,Sk,H,128] scaled fp16 copies with their device scales; lse (pre-scaled by lwm_attn_bwd_lse with the fp16
// offset, -inf for rows without a visible key) and delta [B,H,Qp], Qp = Q rounded up to 64, rows >= Q: lse = -inf;
// bits [B,Q,ceil(Sk/128)*4] or null; tiles / tile_count from lwm_attn_infer_bwd_tilemap. dq_acc [B,Q,H,128] fp32 is
// accumulated into (zero it first); dk_acc / dv_acc [B,Sk,H,128] fp32 are written. order_ws: as in bwd_step.
static int infer_bwd(const void* q16, const void* k16, const void* v16, const void* dout16, const float* scale_q,
                     const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                     const float* delta, const unsigned* bits, const int* tiles, const int* tile_count, float* dq_acc,
                     float* dk_acc, float* dv_acc, int B, int H, int Q, int Sk, int D, float softmax_scale,
                     int* order_ws, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: head_dim must be 128");
  if (!q16 || !k16 || !v16 || !dout16 || !scale_q || !scale_k || !scale_v || !scale_do || !lse || !delta || !tiles ||
      !tile_count || !dq_acc || !dk_acc || !dv_acc)
    return lwm_fail(LWM_ERR_ARG, "attn_infer_bwd: null pointer");
  if (B <= 0 || H <= 0 || Q <= 0 || Sk <= 0 || B > 65535 || H > 65535)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: bad shape (B, H <= 65535; Q, Sk >= 1)");
  const int n_kt = (Sk + kTile - 1) / kTile, qp = (Q + kBQ - 1) / kBQ * kBQ;
  if ((long long)B * n_kt * (qp / kBQ) > 0x7fffffffLL || (long long)Q + kBQ > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: B * ceil(Sk/128) * ceil(Q/64) must fit in int32");
  if (order_ws && !order_fits(B, H, n_kt, qp / kBQ, true))
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd_ordered: the order_ws words and B * H * ceil(Sk/128) must fit in int32");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tm[5];
  if (!make_bf16_tmap(&tm[0], q16, B, Q, H, kBQ) || !make_bf16_tmap(&tm[1], k16, B, Sk, H, kTile) ||
      !make_bf16_tmap(&tm[2], v16, B, Sk, H, kTile) || !make_bf16_tmap(&tm[3], dout16, B, Q, H, kBQ) ||
      !make_f32_tmap(&tm[4], dq_acc, B, Q, H, kBQ))
    return lwm_fail(LWM_ERR_CUDA, "attn_infer_bwd: cuTensorMapEncodeTiled failed (pointers must be 16B aligned)");
  BwdParams p{};
  p.B = B; p.H = H; p.Sq = qp; p.Sk = Sk;
  p.scale = softmax_scale;
  p.scale_log2 = softmax_scale * kLog2e;
  p.lse = lse; p.delta = delta; p.dq_acc = dq_acc; p.dk_acc = dk_acc; p.dv_acc = dv_acc;
  p.scale_q = scale_q; p.scale_k = scale_k; p.scale_v = scale_v; p.scale_do = scale_do;
  p.dkv_init = 1;
  p.tiles = tiles; p.tile_count = tile_count;
  p.bits = bits; p.q_rows = Q;
  const dim3 grid(n_kt, H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (order_ws) {
    const int s = order_prologue(order_ws, (long long)B * H * (qp / kBQ), tiles, tile_count, B, n_kt, qp / kBQ, st, p);
    if (s) return s;
    return launch_bwd<true, true, true, true>(grid, st, tm, p, "attn_bwd_kernel (inference, ordered)");
  }
  return launch_bwd<true, true, true, false>(grid, st, tm, p, "attn_bwd_kernel (inference)");
}

extern "C" int lwm_attn_infer_bwd(const void* q16, const void* k16, const void* v16, const void* dout16,
                                  const float* scale_q, const float* scale_k, const float* scale_v,
                                  const float* scale_do, const float* lse, const float* delta, const unsigned* bits,
                                  const int* tiles, const int* tile_count, float* dq_acc, float* dk_acc, float* dv_acc,
                                  int B, int H, int Q, int Sk, int D, float softmax_scale, void* stream) {
  return infer_bwd(q16, k16, v16, dout16, scale_q, scale_k, scale_v, scale_do, lse, delta, bits, tiles, tile_count,
                   dq_acc, dk_acc, dv_acc, B, H, Q, Sk, D, softmax_scale, nullptr, stream);
}

// lwm_attn_infer_bwd with dQ reduced in ascending key-tile order (include/lwm_b200.h)
extern "C" int lwm_attn_infer_bwd_ordered(const void* q16, const void* k16, const void* v16, const void* dout16,
                                          const float* scale_q, const float* scale_k, const float* scale_v,
                                          const float* scale_do, const float* lse, const float* delta,
                                          const unsigned* bits, const int* tiles, const int* tile_count,
                                          float* dq_acc, float* dk_acc, float* dv_acc, int B, int H, int Q, int Sk,
                                          int D, float softmax_scale, int* order_ws, void* stream) {
  if (!order_ws) return lwm_fail(LWM_ERR_ARG, "attn_infer_bwd_ordered: null order_ws");
  return infer_bwd(q16, k16, v16, dout16, scale_q, scale_k, scale_v, scale_do, lse, delta, bits, tiles, tile_count,
                   dq_acc, dk_acc, dv_acc, B, H, Q, Sk, D, softmax_scale, order_ws, stream);
}
