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
static_assert(sizeof(BwdBarriers) <= 96 && 96 + 2 * 4 <= 128, "attn_bwd: barrier block layout");

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
template <bool kF16, bool kMap = false, bool kBits = false>
__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  // no static shared memory in this kernel: the dynamic window starts 1024-aligned (checked below)
  extern __shared__ __align__(1024) uint8_t smem[];
  float (*s_lse)[kBQ] = reinterpret_cast<float (*)[kBQ]>(smem + kOffLse);
  float (*s_delta)[kBQ] = reinterpret_cast<float (*)[kBQ]>(smem + kOffDelta);
  BwdBarriers& bars = *reinterpret_cast<BwdBarriers*>(smem + kOffBars);
  if (smem_u32(smem) & 1023u) __trap();

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x;  // kv tile (ascending = heaviest first under causal masking)
  const int h = blockIdx.y, b = blockIdx.z;
  const int n_q_tiles = p.Sq / kBQ;
  // first Q tile with a row that can see key 0 of this tile
  int i_start = 0;
  if (p.mask.causal) {
    const long long diff = (long long)p.mask.k_pos0 + (long long)n * kTile - p.mask.q_pos0;
    i_start = diff <= 0 ? 0 : int(min(diff / kBQ, (long long)n_q_tiles));
  }
  int nq = n_q_tiles - i_start;
  int list0 = 0;   // kMap: offset of this K tile's list in p.tiles (B * Sk/128 * Sq/64 < 2^31: checked on the host)
  if constexpr (kMap) {
    const int lt = b * gridDim.x + n;
    nq = p.tile_count[lt];
    list0 = lt * n_q_tiles;
  }
  int* s_entry = reinterpret_cast<int*>(smem + kOffEntry);
  // Q tile of list position it (producer warps)
  auto q_tile = [&](int it) { return kMap ? (p.tiles[list0 + it] >> 1) : i_start + it; };
  // kMap: the count is re-read where each role starts its loop rather than held across setmaxnreg (no spill)
  auto loop_count = [&]() { return kMap ? p.tile_count[b * gridDim.x + n] : nq; };
  if (nq <= 0) {  // this key tile is invisible to the whole q shard: dk/dv unchanged (zero when this launch initialises them)
    if (p.dkv_init) {
      const long long base = (((long long)b * p.Sk + (long long)n * kTile) * p.H + h) * kHeadDim;
      for (int i = threadIdx.x; i < kTile * kHeadDim / 4; i += kBwdThreads) {
        if (kBits && n * kTile + i / (kHeadDim / 4) >= p.Sk) break;   // rows past the cache: not ours to write
        const long long off = base + (long long)(i / (kHeadDim / 4)) * p.H * kHeadDim + (i % (kHeadDim / 4)) * 4;
        *reinterpret_cast<float4*>(p.dk_acc + off) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(p.dv_acc + off) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    return;
  }

  if (threadIdx.x == 0) {
    mbar_init(&bars.kv_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars.q_full[s], 1);
      mbar_init(&bars.q_empty[s], kBwdConsumerWarps);
      mbar_init(&bars.dq_full[s], kBwdConsumerWarps * 32);
      mbar_init(&bars.dq_empty[s], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<24>();
    if (warp == 9 && lane == 0) {
      // dQ reductions: one fp32 add per dQ element per (key tile, Q tile), four 32-column boxes per tile
      tma_prefetch_desc(&tmDQ);
      const int nql = loop_count();
      for (int it = 0; it < nql; ++it) {
        const int st = it & 1;
        const int row0 = q_tile(it) * kBQ;
        mbar_wait(&bars.dq_full[st], (it >> 1) & 1);
#pragma unroll
        for (int j = 0; j < kHeadDim / 32; ++j)
          tma_reduce_add_4d(&tmDQ, smem + kOffDQ + st * kDQB + j * kDQBox, 32 * j, h, row0, b);
        tma_commit_group();
        tma_wait_group_read<0>();
        mbar_arrive(&bars.dq_empty[st]);
      }
      tma_wait_group<0>();
    }
    if (warp == 8 && lane == 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      tma_prefetch_desc(&tmDO);
      mbar_arrive_expect_tx(&bars.kv_full, 2 * kTB);
      load_tile_nb(smem + kOffK, &tmK, &bars.kv_full, h, n * kTile, b, kTB / 2);
      load_tile_nb(smem + kOffV, &tmV, &bars.kv_full, h, n * kTile, b, kTB / 2);
      const long long ml_base = ((long long)b * p.H + h) * p.Sq;
      const int nql = loop_count();
      for (int it = 0; it < nql; ++it) {
        const int st = it & 1;
        const int row0 = q_tile(it) * kBQ;
        mbar_wait(&bars.q_empty[st], ((it >> 1) & 1) ^ 1);
        if constexpr (kMap) s_entry[st] = p.tiles[list0 + it];
        mbar_arrive_expect_tx(&bars.q_full[st], 2 * kQB + 2 * kBQ * 4);
        load_tile_nb(smem + kOffQ + st * kQB, &tmQ, &bars.q_full[st], h, row0, b, kQB / 2);
        load_tile_nb(smem + kOffDO + st * kQB, &tmDO, &bars.q_full[st], h, row0, b, kQB / 2);
        bulk_load_1d(s_lse[st], p.lse + ml_base + row0, kBQ * 4, &bars.q_full[st]);
        bulk_load_1d(s_delta[st], p.delta + ml_base + row0, kBQ * 4, &bars.q_full[st]);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;      // keys [64 wg, 64 wg + 64) of the tile
  const int w = warp & 3;
  const int quad = lane & 3;
  const int kr0 = wg * 64 + w * 16 + (lane >> 2);   // this thread's key rows in the tile: kr0, kr0 + 8
  const bool has_bias = p.mask.bias != nullptr, has_seg = p.mask.seg != nullptr;
  // fp16 mode: logits scale picks up scale_q*scale_k; dP = dO16 V16^T stays in operand units (the absolute delta is
  // brought into them instead) and the dS scale dp_mul = scale_do*scale_v is undone with the dQ / dK scales
  const float scale_log2 = p.scale_log2 * (kF16 ? (*p.scale_q) * (*p.scale_k) : 1.0f);
  const float delta_mul = kF16 ? 1.0f / ((*p.scale_do) * (*p.scale_v)) : 1.0f;   // exact: a power of two
  const float ds_mul = p.scale * (kF16 ? kDsNorm * kPBoostInv : 1.0f);    // P holds P * 2^14 in fp16 mode
  // positions fit in int32 (checked on the host); int keeps the loop under the register budget
  const int wg_k_last = p.mask.k_pos0 + n * kTile + wg * 64 + 63;

  const uint32_t aK = smem_u32(smem + kOffK), aV = smem_u32(smem + kOffV), aDS = smem_u32(smem + kOffDS);
  const uint64_t dK_k = desc_kmajor_sw128(aK + wg * 64 * 128), dV_k = desc_kmajor_sw128(aV + wg * 64 * 128);
  const uint64_t dK_n = desc_mnmajor_sw128(aK + wg * (kTB / 2), kTB / 2);   // this warpgroup's 64 columns of K
  uint8_t* sDQ = smem + kOffDQ;

  float dk[64], dv[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dk[i] = dv[i] = 0.f;

  mbar_wait(&bars.kv_full, 0);
  const int nql = loop_count();
  for (int it = 0; it < nql; ++it) {
    const int st = it & 1;
    const uint32_t aQ = smem_u32(smem + kOffQ + st * kQB), aDO = smem_u32(smem + kOffDO + st * kQB);
    const uint64_t dQ_k = desc_kmajor_sw128(aQ), dDO_k = desc_kmajor_sw128(aDO);
    const uint64_t dQ_n = desc_mnmajor_sw128(aQ, kQB / 2), dDO_n = desc_mnmajor_sw128(aDO, kQB / 2);
    const uint64_t dDS_m = desc_mnmajor_sw128(aDS + st * kDSB, kDSB);
    uint8_t* sDS = smem + kOffDS + st * kDSB;
    mbar_wait(&bars.q_full[st], (it >> 1) & 1);
    const int entry = kMap ? s_entry[st] : 0;

    // ---- S^T = K Q^T, dP^T = V dO^T: two groups, so that exp(S^T) runs while dP^T is on the tensor cores
    float sacc[32], dpacc[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kHeadDim / 16; ++ks) {
      const uint32_t ka = (ks >> 2) * (kTB / 2) + (ks & 3) * 32, kb = (ks >> 2) * (kQB / 2) + (ks & 3) * 32;
      wgmma_ss<64, kF16, 0, 0>(sacc, desc_advance(dK_k, ka), desc_advance(dQ_k, kb), ks > 0);
    }
    wgmma_commit();
#pragma unroll
    for (int ks = 0; ks < kHeadDim / 16; ++ks) {
      const uint32_t ka = (ks >> 2) * (kTB / 2) + (ks & 3) * 32, kb = (ks >> 2) * (kQB / 2) + (ks & 3) * 32;
      wgmma_ss<64, kF16, 0, 0>(dpacc, desc_advance(dV_k, ka), desc_advance(dDO_k, kb), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<1>();
    reg_fence(sacc);

    // ---- P^T = exp2(S^T * scale_log2 (+bias) - lse2)
    const int q_tile_pos = p.mask.q_pos0 + (kMap ? entry >> 1 : i_start + it) * kBQ;
    // kMap: clean tiles keep the masked path's rounding (fmaf(s, scale, 0)): bit-identical to the step without a map
    const bool need_mask =
        kBits ? bool(entry & 1) : (kMap || has_bias || has_seg || (p.mask.causal && q_tile_pos < wg_k_last));
    const bool mixed = kMap ? (entry & 1) : true;   // the tile reads bias and segment ids
    uint32_t pk[4][4], dsk[4][4];   // P^T and dS^T as A fragments, one 16-query slice per entry
    float pr[4][8];
    // the mask test is hoisted out of the element loop: one branch per tile keeps the fragment in registers
    if (!need_mask) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = (i >> 2) * 8 + quad * 2 + (i & 1);   // query column in the tile
        pr[i >> 3][i & 7] = ex2f(fmaf(sacc[i], scale_log2, s_lse[st][col]));   // -lse*log2e (or -inf): lwm_attn_bwd_lse
      }
    } else if constexpr (kBits) {
      // keys kr0 and kr0 + 8 sit in one 32-bit word of every query row's bits (bits sh and sh + 8). Rows past q_rows
      // read the last row instead: their lse is -inf, whatever the bits say. Masked entries and keys >= Sk get P = 0.
      const int key0 = n * kTile + kr0;
      const int sh = key0 & 31;
      const int kw = gridDim.x * 4;
      const uint32_t* wcol = p.bits ? p.bits + (long long)b * p.q_rows * kw + (key0 >> 5) : nullptr;
      const bool key_in[2] = {key0 < p.Sk, key0 + 8 < p.Sk};
#pragma unroll
      for (int g = 0; g < 8; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = g * 8 + quad * 2 + e;
          const uint32_t word = wcol ? wcol[(long long)min(q_tile_pos + col, p.q_rows - 1) * kw] : ~0u;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int i = 4 * g + 2 * hh + e;
            const bool vis = key_in[hh] && ((word >> (sh + 8 * hh)) & 1u);
            pr[i >> 3][i & 7] = vis ? ex2f(fmaf(sacc[i], scale_log2, s_lse[st][col])) : 0.f;
          }
        }
    } else {
      // per-key mask inputs, reloaded per masked tile (L1 hits) rather than held in registers across the loop
      const bool use_bias = has_bias && mixed, use_seg = has_seg && mixed;
      const int* seg_row = use_seg ? p.mask.seg + (long long)b * p.mask.seg_stride : nullptr;
      const int k_pos = p.mask.k_pos0 + n * kTile + kr0;   // this thread's keys: k_pos, k_pos + 8
      int my_seg[2];
      float bias_t[2] = {0.f, 0.f};
      bool key_masked[2] = {false, false};
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        my_seg[hh] = use_seg ? seg_row[k_pos + 8 * hh] : 0;
        if (use_bias) {
          bias_t[hh] = p.mask.bias[(long long)b * p.mask.bias_stride + k_pos + 8 * hh] * kLog2e;
          key_masked[hh] = bias_t[hh] < kMaskedLogit;
        }
      }
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int hh = (i >> 1) & 1;
        const int col = (i >> 2) * 8 + quad * 2 + (i & 1);
        float tv = key_masked[hh] ? kMaskedLogit : fmaf(sacc[i], scale_log2, bias_t[hh]);
        const int q_pos = q_tile_pos + col;
        if (use_seg && seg_row[q_pos] != my_seg[hh]) tv = kMaskedLogit;
        if (p.mask.causal && q_pos < k_pos + 8 * hh) tv = kMaskedLogit;
        pr[i >> 3][i & 7] = ex2f(tv + s_lse[st][col]);
      }
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int t = 0; t < 4; ++t)
        pk[kk][t] = kF16 ? pack_f16x2(pr[kk][2 * t], pr[kk][2 * t + 1]) : pack_bf16x2(pr[kk][2 * t], pr[kk][2 * t + 1]);

    // ---- dV += P^T dO, on the tensor cores while dS^T is computed
    reg_fence(dv);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs128<kF16, 1>(dv, pk[kk], desc_advance(dDO_n, kk * 2048), 1);
    wgmma_commit();

    // ---- dS^T = P^T o (dP^T - delta) * scale (waits for dP^T only)
    wgmma_wait<1>();
    reg_fence(dpacc);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      float ds[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int i = 8 * kk + t;
        const int col = (i >> 2) * 8 + quad * 2 + (i & 1);
        ds[t] = (pr[kk][t] * ds_mul) * fmaf(-s_delta[st][col], delta_mul, dpacc[i]);
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) dsk[kk][t] = kF16 ? pack_f16x2(ds[2 * t], ds[2 * t + 1]) : pack_bf16x2(ds[2 * t], ds[2 * t + 1]);
    }

    // ---- dS^T -> shared memory stage st (128B-swizzled, key rows of 64 queries) for the dQ wgmma of both
    // warpgroups. The stage was last read by the dQ wgmmas of tile it - 2, which both warpgroups waited for
    // before they passed the barrier of tile it - 1.
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const uint32_t row = kr0 + 8 * (t & 1);
        const uint32_t col = kk * 16 + (t >> 1) * 8 + quad * 2;
        *reinterpret_cast<uint32_t*>(sDS + swz128_offset(row, col >> 3) + (col & 7) * 2) = dsk[kk][t];
      }
    fence_proxy_async_smem();

    // ---- dK += dS^T Q, running while the other warpgroup's half of dS^T arrives
    reg_fence(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs128<kF16, 1>(dk, dsk[kk], desc_advance(dQ_n, kk * 2048), 1);
    wgmma_commit();

    // ---- dQ = dS K over all 128 keys (the barrier: both halves of dS^T are in shared memory)
    named_bar_sync(1, 256);
    float dq[32];
#pragma unroll
    for (int ks = 0; ks < kTile / 16; ++ks)
      wgmma_ss<64, kF16, 1, 1>(dq, desc_advance(dDS_m, ks * 2048), desc_advance(dK_n, ks * 2048), ks > 0);
    wgmma_commit();
    wgmma_wait<1>();   // dV and dK: the last reads of Q, dO, lse and delta of this stage
    reg_fence(dv);
    reg_fence(dk);
    if (lane == 0) mbar_arrive(&bars.q_empty[st]);

    // dQ tile (64 queries x this warpgroup's 64 columns, scaled to fp32 gradient units) -> staging tile st, as
    // two 32-column boxes of 128-byte rows, 16-byte chunks XOR-swizzled by row (conflict-free float2 stores)
    mbar_wait(&bars.dq_empty[st], ((it >> 1) & 1) ^ 1);
    wgmma_wait<0>();
    reg_fence(dq);
    // dQ = dS16 K16 * scale_k * dp_mul / norm with dp_mul = scale_do * scale_v (re-read here: no register held across the loop)
    const float dq_mul = kF16 ? (*p.scale_k) * ((*p.scale_do) * (*p.scale_v)) * (1.0f / kDsNorm) : 1.0f;
    uint8_t* sdq = sDQ + st * kDQB + wg * 2 * kDQBox + (quad & 1) * 8;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const uint32_t row = w * 16 + (lane >> 2) + 8 * hh;
#pragma unroll
      for (int g = 0; g < 8; ++g)
        *reinterpret_cast<float2*>(sdq + (g >> 2) * kDQBox + swz128_offset(row, (g & 3) * 2 + (quad >> 1))) =
            make_float2(dq[4 * g + 2 * hh] * dq_mul, dq[4 * g + 2 * hh + 1] * dq_mul);
    }
    fence_proxy_async_smem();
    mbar_arrive(&bars.dq_full[st]);
  }

  // ------------------------------------------------------------------ epilogue: dK, dV
  // dK = dS16^T Q16 * scale_q * dp_mul / norm ; dV = P^T dO16 * scale_do
  const float dk_mul = kF16 ? (*p.scale_q) * ((*p.scale_do) * (*p.scale_v)) * (1.0f / kDsNorm) : 1.0f;
  const float dv_mul = kF16 ? (*p.scale_do) * kPBoostInv : 1.0f;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (kBits && n * kTile + kr0 + 8 * hh >= p.Sk) continue;   // key rows past the cache are not written
    const long long row = ((((long long)b * p.Sk + (long long)n * kTile + kr0 + 8 * hh) * p.H + h) * kHeadDim);
#pragma unroll
    for (int g = 0; g < kHeadDim / 8; ++g) {
      const int c = g * 8 + quad * 2;
      float2* pk2 = reinterpret_cast<float2*>(p.dk_acc + row + c);
      float2* pv2 = reinterpret_cast<float2*>(p.dv_acc + row + c);
      float2 ck = p.dkv_init ? make_float2(0.f, 0.f) : *pk2;
      float2 cv = p.dkv_init ? make_float2(0.f, 0.f) : *pv2;
      ck.x = fmaf(dk[4 * g + 2 * hh], dk_mul, ck.x);
      ck.y = fmaf(dk[4 * g + 2 * hh + 1], dk_mul, ck.y);
      cv.x = fmaf(dv[4 * g + 2 * hh], dv_mul, cv.x);
      cv.y = fmaf(dv[4 * g + 2 * hh + 1], dv_mul, cv.y);
      *pk2 = ck;
      *pv2 = cv;
    }
  }
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

}  // namespace lwm

using namespace lwm;

// One ring step (include/lwm_b200.h): the scales select the fp16-operand kernel, tiles / tile_count the block map.
extern "C" int lwm_attn_bwd_step(const void* q, const void* k, const void* v, const void* dout, const float* scale_q,
                                 const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                                 const float* delta, float* dq_acc, float* dk_acc, float* dv_acc, int B, int H,
                                 int Sq, int Sk, int D, long long q_pos0, long long k_pos0, int causal,
                                 const float* bias, long long bias_stride, const int* segment_ids,
                                 long long seg_stride, float softmax_scale, int dkv_init, const int* tiles,
                                 const int* tile_count, void* stream) {
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
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tq, tk, tv, tdo, tdq;
  if (!make_bf16_tmap(&tq, q, B, Sq, H, kBQ) || !make_bf16_tmap(&tk, k, B, Sk, H, kTile) ||
      !make_bf16_tmap(&tv, v, B, Sk, H, kTile) || !make_bf16_tmap(&tdo, dout, B, Sq, H, kBQ) ||
      !make_f32_tmap(&tdq, dq_acc, B, Sq, H, kBQ))
    return lwm_fail(LWM_ERR_CUDA, "attn_bwd: cuTensorMapEncodeTiled failed (pointers must be 16B aligned)");
  BwdParams p;
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
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63];      // function attributes are per device
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmemBytes) !=
            cudaSuccess ||
        cudaFuncSetAttribute(attn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmemBytes) !=
            cudaSuccess ||
        cudaFuncSetAttribute(attn_bwd_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             kBwdSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(attn_bwd_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             kBwdSmemBytes) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "attn_bwd: cannot raise dynamic shared memory limit");
    attr_set = true;
  }
  dim3 grid(Sk / kTile, H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (tiles) {
    if (scale_q) attn_bwd_kernel<true, true><<<grid, kBwdThreads, kBwdSmemBytes, st>>>(tq, tk, tv, tdo, tdq, p);
    else attn_bwd_kernel<false, true><<<grid, kBwdThreads, kBwdSmemBytes, st>>>(tq, tk, tv, tdo, tdq, p);
    return lwm_check_launch("attn_bwd_kernel (block map)");
  }
  if (scale_q) attn_bwd_kernel<true><<<grid, kBwdThreads, kBwdSmemBytes, st>>>(tq, tk, tv, tdo, tdq, p);
  else attn_bwd_kernel<false><<<grid, kBwdThreads, kBwdSmemBytes, st>>>(tq, tk, tv, tdo, tdq, p);
  return lwm_check_launch("attn_bwd_kernel");
}

// Backward of ringattention_inference (attn_bwd_kernel<true, true, true>): any Q and Sk. q16 / dout16 [B,Q,H,128],
// k16 / v16 [B,Sk,H,128] scaled fp16 copies with their device scales; lse (pre-scaled by lwm_attn_bwd_lse with the fp16
// offset, -inf for rows without a visible key) and delta [B,H,Qp], Qp = Q rounded up to 64, rows >= Q: lse = -inf;
// bits [B,Q,ceil(Sk/128)*4] or null; tiles / tile_count from lwm_attn_infer_bwd_tilemap. dq_acc [B,Q,H,128] fp32 is
// accumulated into (zero it first); dk_acc / dv_acc [B,Sk,H,128] fp32 are written.
extern "C" int lwm_attn_infer_bwd(const void* q16, const void* k16, const void* v16, const void* dout16,
                                  const float* scale_q, const float* scale_k, const float* scale_v,
                                  const float* scale_do, const float* lse, const float* delta, const unsigned* bits,
                                  const int* tiles, const int* tile_count, float* dq_acc, float* dk_acc, float* dv_acc,
                                  int B, int H, int Q, int Sk, int D, float softmax_scale, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: head_dim must be 128");
  if (!q16 || !k16 || !v16 || !dout16 || !scale_q || !scale_k || !scale_v || !scale_do || !lse || !delta || !tiles ||
      !tile_count || !dq_acc || !dk_acc || !dv_acc)
    return lwm_fail(LWM_ERR_ARG, "attn_infer_bwd: null pointer");
  if (B <= 0 || H <= 0 || Q <= 0 || Sk <= 0 || B > 65535 || H > 65535)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: bad shape (B, H <= 65535; Q, Sk >= 1)");
  const int n_kt = (Sk + kTile - 1) / kTile, qp = (Q + kBQ - 1) / kBQ * kBQ;
  if ((long long)B * n_kt * (qp / kBQ) > 0x7fffffffLL || (long long)Q + kBQ > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_bwd: B * ceil(Sk/128) * ceil(Q/64) must fit in int32");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tq, tk, tv, tdo, tdq;
  if (!make_bf16_tmap(&tq, q16, B, Q, H, kBQ) || !make_bf16_tmap(&tk, k16, B, Sk, H, kTile) ||
      !make_bf16_tmap(&tv, v16, B, Sk, H, kTile) || !make_bf16_tmap(&tdo, dout16, B, Q, H, kBQ) ||
      !make_f32_tmap(&tdq, dq_acc, B, Q, H, kBQ))
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
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63];
  if (!attr_set) {
    if (cudaFuncSetAttribute(attn_bwd_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             kBwdSmemBytes) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "attn_infer_bwd: cannot raise dynamic shared memory limit");
    attr_set = true;
  }
  attn_bwd_kernel<true, true, true><<<dim3(n_kt, H, B), kBwdThreads, kBwdSmemBytes,
                                      reinterpret_cast<cudaStream_t>(stream)>>>(tq, tk, tv, tdo, tdq, p);
  return lwm_check_launch("attn_bwd_kernel (inference)");
}
