// Ring-attention forward tile kernel for sm_90a.
//
// One launch = one ring step of SURVEY.md Appendix A `blockwise_fwd`: the local query shard
// [B,Sq,H,128] attends to the currently held K/V block [B,Sk,H,128]; the running
// (numerator, denominator, max) carry of the reference (ringattention fwd, bound at
// lwm/llama.py:541) is merged in the epilogue, so the ring loop on the host only rotates K/V.
//
// Mapping to the hardware:
//   * CTA = one 128-row Q tile of one (batch, head); CTAs are ordered heaviest (latest rows) first.
//   * warp 8 streams K/V tiles with TMA (128B swizzle) through a 4-slot ring (K0 V0 K1 V1).
//   * warpgroups 0 and 1 each own 64 query rows: S = Q K^T with wgmma (both operands K-major in
//     shared memory, fp32 logits in registers), online softmax in the log2 domain on the register
//     fragment (a row is spread over the 4 lanes of a quad), then O += P V with P taken straight
//     from registers as the A fragment and V read MN-major from the TMA tile (no transpose).
//   * the consumer loop is software-pipelined: iteration j issues S_j = Q K_j^T and O += P_{j-1} V_{j-1} as two
//     commit groups, waits for S_j only, and runs tile j's softmax while the PV group is on the tensor cores. The
//     two warpgroups take turns issuing (named barriers 1 and 2), so one's softmax also runs under the other's GEMMs.
//   * causal masking by global token position; KV tiles entirely above the diagonal are never
//     loaded; only diagonal tiles pay for the mask.
#include "attn_common.cuh"
#include "attn_dropout.cuh"
#include "tmap.h"
#include "capi_internal.h"

namespace lwm {

struct FwdParams {
  int B, H, Sq, Sk;
  float scale_log2;  // softmax_scale * log2(e)
  MaskParams mask;
  __nv_bfloat16* out;  // [B,Sq,H,D]   written when last
  float* out_f32;      // optional un-rounded copy of `out` (fp16 precision mode residual), written when last
  float* lse;          // [B,H,Sq]     natural-log LSE, written when last
  float* acc_o;        // [B,Sq,H,D]   fp32 numerator carry (relative to acc_m)
  float* acc_m;        // [B,H,Sq]     running max, log2 domain
  float* acc_l;        // [B,H,Sq]     running denominator
  int first, last;
  const float *scale_q, *scale_k, *scale_v;   // fp16 mode: device scalars, x = x16 * scale; null => bf16 operands
  // list modes: the (b, Q tile) lists of KV tiles. Inference (ringattention_inference, Sq = Q rows, any Q and Sk):
  // from the mask bits (attn_infer.cu). Training with a bias or segment ids: from lwm_attn_step_tilemap (attn_tiles.cu).
  const uint32_t* bits;   // inference: [B, Sq, n_kt * 4] mask bits (bit j of word w <=> key 32 w + j; 1 = attend) or null
  const int* tiles;       // [B, ceil(Sq/128), n_kt]: kt * 2 + mixed, ascending kt
  const int* tile_count;  // [B, ceil(Sq/128)]
  int n_kt, splits;       // KV tiles of the shard; inference: CTAs per Q tile, each takes a contiguous slice of the list
  float* o_part;          // [B*Sq*H, splits, 128] un-normalised numerators (in V's units)
  float* ml_part;         // [B*Sq*H, splits, 2] (max in the log2 domain, denominator)
  DropParams drop;        // kDrop: the attention-dropout mask (attn_dropout.cuh)
};

constexpr int kFwdStages = 4;
constexpr int kFwdTileBytes = kTile * kHeadDim * 2;  // 32 KB
constexpr int kFwdThreads = 384;  // 2 consumer warpgroups + 1 producer warpgroup (one TMA warp, 3 idle warps)
constexpr int kFwdConsumerWarps = 8;
constexpr int kFwdSmemBytes = (1 + kFwdStages) * kFwdTileBytes + 1024;
// fp16 P is packed as p * 2^15 (p <= 1, so at most 32768 < 65504): normal down to p = 2^-29 instead of 2^-14. A row
// whose max sits on a sink key ~10+ nats above the rest otherwise packs the bulk of its mass as fp16 subnormals or
// zeros while l_run keeps it (DESIGN.md §5). The boost enters the exponent; l_run adds s * 2^-15 (= p), and the
// epilogues fold 2^-15 into their power-of-two V factor, so m_run, l_run, the carries and lse stay in units of p.
constexpr float kPBoostLog2 = 15.f, kPBoostInv = 1.f / 32768.f;

struct FwdBarriers {
  uint64_t q_full;
  uint64_t kv_full[kFwdStages];
  uint64_t kv_empty[kFwdStages];
};

LWM_DEVICE void load_tile(uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int h, int row0, int b) {
  mbar_arrive_expect_tx(bar, kFwdTileBytes);
  tma_load_4d(dst, tm, bar, 0, h, row0, b);
  tma_load_4d(dst + kFwdTileBytes / 2, tm, bar, 64, h, row0, b);
}

LWM_DEVICE float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
LWM_DEVICE float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// kF16: operands are IEEE fp16 (exact, scaled copies of the bf16 inputs) and P is kept in fp16
// (11 significant bits instead of 8) — the precision mode that meets 1e-3 on white-noise inputs.
// kInfer: the inference mode. A CTA walks its slice of its Q tile's KV tile list (built from a bit mask by
// attn_infer.cu); only tiles marked mixed read mask bits, keys >= Sk get -inf, rows >= Sq are padding. The epilogue
// writes the CTA's un-normalised partial for decode_merge_kernel instead of a carry.
// kMap: the training step with a bias or segment ids, over the block map of lwm_attn_step_tilemap: the CTA walks its
// Q tile's list of KV tiles (masked ones are not in it); mixed tiles run the per-element mask, clean tiles the same
// branch with no bias or segment read (the causal compare stays). The epilogue is the training one.
// kDrop (training instances): attention dropout. Every visited tile runs the per-element branch, which gives a dropped
// entry the masked logit; a row left without a surviving key writes out = 0 and an lse at the masked level.
// The kernel body; attn_fwd_kernel (no dropout) and attn_fwd_dropout_kernel are its entry points.
template <bool kF16, bool kInfer, bool kMap, bool kDrop>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                              const FwdParams& p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                   // 32 KB: d [0,64) | d [64,128), 128 rows each
  uint8_t* sKV = smem + kFwdTileBytes;  // ring of 32 KB slots: K0 V0 K1 V1
  __shared__ FwdBarriers bars;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_q_tiles = kInfer ? (p.Sq + kTile - 1) / kTile : p.Sq / kTile;
  // heaviest (latest rows) first under causal masking
  const int tile = n_q_tiles - 1 - int(kInfer ? blockIdx.x / p.splits : blockIdx.x);
  const int h = blockIdx.y, b = blockIdx.z;
  const int m0 = tile * kTile;

  // number of KV tiles any row of this CTA can see
  int n_kv = p.Sk / kTile;
  const int* list = nullptr;   // kInfer: this CTA's slice of the tile list
  if constexpr (kInfer) {
    const long long lt = (long long)b * n_q_tiles + tile;
    const int cnt = p.tile_count[lt];
    const int per = (cnt + p.splits - 1) / p.splits;
    const int beg = min(cnt, int(blockIdx.x % p.splits) * per);
    n_kv = min(cnt, beg + per) - beg;
    list = p.tiles + lt * p.n_kt + beg;
  } else if constexpr (kMap) {
    const long long lt = (long long)b * n_q_tiles + tile;
    n_kv = p.tile_count[lt];
    list = p.tiles + lt * p.n_kt;
  } else if (p.mask.causal) {
    const long long last_q = (long long)p.mask.q_pos0 + m0 + kTile - 1;
    const long long vis = last_q - p.mask.k_pos0;  // largest visible local key index
    n_kv = vis < 0 ? 0 : min((long long)n_kv, vis / kTile + 1);
  }
  if (n_kv == 0 && !p.first && !p.last) return;  // nothing visible: the carry is unchanged

  if (threadIdx.x == 0) {
    mbar_init(&bars.q_full, 1);
    for (int i = 0; i < kFwdStages; ++i) {
      mbar_init(&bars.kv_full[i], 1);
      mbar_init(&bars.kv_empty[i], kFwdConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<24>();
    if (warp == 8 && lane == 0 && n_kv > 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      load_tile(sQ, &tmQ, &bars.q_full, h, m0, b);
      for (int i = 0; i < 2 * n_kv; ++i) {
        const int slot = i % kFwdStages;
        const uint32_t ph = (i / kFwdStages) & 1;
        mbar_wait(&bars.kv_empty[slot], ph ^ 1);
        const int kt = (kInfer || kMap) ? (list[i >> 1] >> 1) : (i >> 1);
        load_tile(sKV + slot * kFwdTileBytes, (i & 1) ? &tmV : &tmK, &bars.kv_full[slot], h, kt * kTile, b);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;   // rows [64 wg, 64 wg + 64) of the Q tile
  const int w = warp & 3;
  const int quad = lane & 3;
  // this thread's two rows: r0 and r0 + 8 (accumulator fragment of wgmma m64nNk16)
  const int r0 = m0 + wg * 64 + w * 16 + (lane >> 2);
  const float scale = p.scale_log2 * (p.scale_q ? (*p.scale_q) * (*p.scale_k) : 1.0f);
  const bool has_bias = p.mask.bias != nullptr, has_seg = p.mask.seg != nullptr;

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  if (n_kv > 0) {
    mbar_wait(&bars.q_full, 0);
    const uint64_t q_desc = desc_kmajor_sw128(smem_u32(sQ + wg * 64 * 128));
    const uint32_t kv_base = smem_u32(sKV);
    // positions fit in int32 (checked on the host); int keeps the loop under the register budget
    const int warp_q_pos0 = p.mask.q_pos0 + m0 + wg * 64 + w * 16;
    float s[64];         // logits of tile j, then their exponentials (fp32) until they are packed into pa
    uint32_t pa[8][4];   // P as the A fragment of O += P V, one 16-key slice per entry
    float alpha[2];      // rescale of o and l_run from tile j - 1's row max to tile j's

    // Ring item i: K of tile i / 2 (even i) or V of tile i / 2 (odd i), in slot i % kFwdStages.
    auto wait_full = [&](int i) { mbar_wait(&bars.kv_full[i % kFwdStages], (i / kFwdStages) & 1); };
    auto release = [&](int i) {
      if (lane == 0) mbar_arrive(&bars.kv_empty[i % kFwdStages]);
    };
    // The two warpgroups take turns issuing their GEMMs (named barrier 1 + wg: "warpgroup wg may issue"), so
    // that one warpgroup's softmax runs while the other's GEMMs are on the tensor cores. Warpgroup 0 goes first.
    // Each warpgroup passes the turn n_kv + 1 times; warpgroup 1 skips its last hand-over, which nobody waits for.
    auto turn_begin = [&]() { named_bar_sync(1 + wg, 256); };
    auto turn_end = [&](bool last) {
      if (!(last && wg == 1)) named_bar_arrive(2 - wg, 256);
    };
    if (wg == 1) named_bar_arrive(1, 256);
    // S = Q K_j^T, one commit group
    auto issue_s = [&](int j) {
      const uint64_t kd = desc_kmajor_sw128(kv_base + ((2 * j) % kFwdStages) * kFwdTileBytes);
#pragma unroll
      for (int ks = 0; ks < kHeadDim / 16; ++ks) {
        const uint32_t off = (ks >> 2) * (kFwdTileBytes / 2) + (ks & 3) * 32;
        wgmma_ss<128, kF16, 0, 0>(s, desc_advance(q_desc, off), desc_advance(kd, off), ks > 0);
      }
      wgmma_commit();
    };
    // O += P_j V_j, one commit group (P from registers, V read MN-major)
    auto issue_pv = [&](int j) {
      const uint64_t vd = desc_mnmajor_sw128(kv_base + ((2 * j + 1) % kFwdStages) * kFwdTileBytes, kFwdTileBytes / 2);
#pragma unroll
      for (int kk = 0; kk < kTile / 16; ++kk) wgmma_rs128<kF16, 1>(o, pa[kk], desc_advance(vd, kk * 2048), 1);
      wgmma_commit();
    };
    // online softmax of tile j on the fragment: row max, alpha, m_run / l_run update, s <- exp2(s * scale - m)
    auto softmax = [&](int j) {
      int k_tile_pos;
      bool need_mask;   // warp-uniform: does any row of this warp need a mask on this KV tile?
      bool mixed = true;  // kMap: the tile reads bias and segment ids
      if constexpr (kInfer) {
        const int e = list[j];
        k_tile_pos = (e >> 1) * kTile;
        need_mask = e & 1;
      } else if constexpr (kMap) {
        const int e = list[j];
        k_tile_pos = p.mask.k_pos0 + (e >> 1) * kTile;
        // clean tiles keep the rounding of the masked path (s * scale, then - m): bit-identical to the step without a map
        need_mask = true;
        mixed = e & 1;
      } else {
        k_tile_pos = p.mask.k_pos0 + j * kTile;
        need_mask = kDrop || has_bias || has_seg || (p.mask.causal && (k_tile_pos + kTile - 1 > warp_q_pos0));
      }
      float mx[2] = {-INFINITY, -INFINITY};
      if (!need_mask) {
#pragma unroll
        for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
        mx[0] = quad_max(mx[0]) * scale;
        mx[1] = quad_max(mx[1]) * scale;
      } else if constexpr (kInfer) {
        // this thread's two rows: 4 mask words each (the tile's 128 keys); padding rows read none (all visible)
        uint32_t mw[2][4];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = r0 + 8 * hh;
          uint4 w4 = make_uint4(~0u, ~0u, ~0u, ~0u);
          if (p.bits && row < p.Sq)
            w4 = *reinterpret_cast<const uint4*>(p.bits + ((long long)b * p.Sq + row) * (p.n_kt * 4) + k_tile_pos / 32);
          mw[hh][0] = w4.x; mw[hh][1] = w4.y; mw[hh][2] = w4.z; mw[hh][3] = w4.w;
        }
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int hh = (i >> 1) & 1;
          const int col = (i >> 2) * 8 + quad * 2 + (i & 1);   // col >> 5 == i >> 4
          float tv = s[i] * scale;
          if (!((mw[hh][i >> 4] >> (col & 31)) & 1u)) tv = kMaskedLogit;
          if (k_tile_pos + col >= p.Sk) tv = -INFINITY;       // past the cache: in no sum, not even a masked one
          s[i] = tv;
          mx[hh] = fmaxf(mx[hh], tv);
        }
        mx[0] = quad_max(mx[0]);
        mx[1] = quad_max(mx[1]);
      } else {
        // per-row mask inputs, reloaded per masked tile (L1 hits) rather than held in registers across the loop
        const bool use_bias = has_bias && mixed, use_seg = has_seg && mixed;
        const float* bias_row = use_bias ? p.mask.bias + (long long)b * p.mask.bias_stride : nullptr;
        const int* seg_row = use_seg ? p.mask.seg + (long long)b * p.mask.seg_stride : nullptr;
        int q_pos[2];
        int my_seg[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          q_pos[hh] = p.mask.q_pos0 + r0 + 8 * hh;
          my_seg[hh] = use_seg ? seg_row[q_pos[hh]] : 0;
        }
        // kDrop: bit i of dropped is the decision of fragment entry i (row hh = (i >> 1) & 1, key 8 g + 2 quad + e,
        // g = i >> 2, e = i & 1). Call t covers rows r0, r0 + 8 (q_pos[0] has bit 3 clear) and keys 16 t + 2 quad +
        // {0, 1, 8, 9} (k_tile_pos is a multiple of 128; both checked on the host): its 8 entries are i = 8 t .. 8 t + 7,
        // with the row picking the word pair, g & 1 the word and e the half.
        uint64_t dropped = 0u;
        if constexpr (kDrop) {
#pragma unroll 1   // one call at a time: unrolled (fully, or by 2), ptxas interleaves the calls and spills
          for (int t = 0; t < 8; ++t) {
            const uint4 r = drop_block(p.drop, q_pos[0], k_tile_pos + 16 * t + 2 * quad, h, b);
            uint32_t bits = 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j) bits |= uint32_t(drop_pick(r, (j >> 1) & 1, (j >> 2) & 1, j & 1, p.drop.thr)) << j;
            dropped |= uint64_t(bits) << (8 * t);
          }
        }
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int hh = (i >> 1) & 1;
          const int col = (i >> 2) * 8 + quad * 2 + (i & 1);
          float tv = s[i] * scale;
          if (use_bias) {
            const float bt = bias_row[k_tile_pos + col] * kLog2e;
            tv = (bt < kMaskedLogit) ? kMaskedLogit : tv + bt;
          }
          if (use_seg && seg_row[k_tile_pos + col] != my_seg[hh]) tv = kMaskedLogit;
          if (p.mask.causal && k_tile_pos + col > q_pos[hh]) tv = kMaskedLogit;
          if (kDrop && ((dropped >> i) & 1u)) tv = kMaskedLogit;
          s[i] = tv;
          mx[hh] = fmaxf(mx[hh], tv);
        }
        mx[0] = quad_max(mx[0]);
        mx[1] = quad_max(mx[1]);
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float m_new = fmaxf(m_run[hh], mx[hh]);
        alpha[hh] = (m_run[hh] == -INFINITY) ? 0.f : ex2f(m_run[hh] - m_new);
        m_run[hh] = m_new;
        // rounded on its own, never fused with the first += below: l_run keeps its multiply-then-add rounding
        l_run[hh] = __fmul_rn(l_run[hh], alpha[hh]);
      }
      // kF16: s <- p * 2^15 through the exponent (15 - m), and l_run adds the product s * 2^-15 (exact) in the FFMA
      // that would otherwise be an FADD. Where -m absorbs the 15 (m = kMaskedLogit), s stays p, so l_run gathers
      // p * 2^-15 and o the unboosted P; the 2^-15 that the epilogues fold into wb / wv then scales o the same way,
      // so o / l, every carry and every inference partial stay consistent (only such a row's lse, about -1e30 * ln 2,
      // loses 15 * ln 2, which it cannot show).
      const float neg_m[2] = {kF16 ? kPBoostLog2 - m_run[0] : -m_run[0], kF16 ? kPBoostLog2 - m_run[1] : -m_run[1]};
      // masked tiles hold s * scale already: fmaf(s, 1, -m) rounds exactly as s - m does
      const float mul = need_mask ? 1.0f : scale;
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int hh = (i >> 1) & 1;
        s[i] = ex2f(fmaf(s[i], mul, neg_m[hh]));
        if constexpr (kF16) l_run[hh] = fmaf(s[i], kPBoostInv, l_run[hh]);
        else l_run[hh] += s[i];
      }
    };
    auto pack_p = [&]() {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int i = 8 * kk + 2 * t;
          pa[kk][t] = kF16 ? pack_f16x2(s[i], s[i + 1]) : pack_bf16x2(s[i], s[i + 1]);
        }
    };

    // Software pipeline: iteration j issues S_j and O += P_{j-1} V_{j-1} back to back, then runs tile j's
    // softmax while the PV group is still on the tensor cores.
    // ---- prologue: S_0, softmax_0 (o is still zero: no rescale)
    wait_full(0);
    turn_begin();
    wgmma_fence();
    issue_s(0);
    turn_end(false);
    wgmma_wait<0>();
    reg_fence(s);
    release(0);
    softmax(0);
    pack_p();
    // ---- steady state
    for (int j = 1; j < n_kv; ++j) {
      wait_full(2 * j);
      wait_full(2 * j - 1);
      turn_begin();
      reg_fence(o);
      wgmma_fence();
      issue_s(j);
      issue_pv(j - 1);
      turn_end(false);
      wgmma_wait<1>();   // S_j done; PV_{j-1} may still run
      reg_fence(s);
      release(2 * j);
      softmax(j);
      // No rescale when no row of the warp raised its max (alpha == 1, and x * 1 is exact). The branch also ends the
      // basic block of the exponentials, which is why the PV wait sits in both arms: in one block with them, ptxas
      // hoists the wait above them, and they would run after PV_{j-1} instead of under it
      // (tests/test_attn_fwd_schedule_cpu.py checks the SASS).
      if (__any_sync(0xffffffffu, alpha[0] != 1.f || alpha[1] != 1.f)) {
        wgmma_wait<0>();
        reg_fence(o);
#pragma unroll
        for (int i = 0; i < 64; ++i) o[i] *= alpha[(i >> 1) & 1];
      } else {
        wgmma_wait<0>();
        reg_fence(o);
      }
      release(2 * j - 1);
      pack_p();
    }
    // ---- epilogue: the last O += P V
    wait_full(2 * n_kv - 1);
    turn_begin();
    reg_fence(o);
    wgmma_fence();
    issue_pv(n_kv - 1);
    turn_end(true);
    wgmma_wait<0>();
    reg_fence(o);
    release(2 * n_kv - 1);
  }

  if constexpr (kInfer) {
    // ---------------------------------------------------------------- epilogue: this CTA's partial
    const int split = blockIdx.x % p.splits;
    const float l_rows[2] = {quad_sum(l_run[0]), quad_sum(l_run[1])};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q_row = r0 + 8 * hh;
      const float l_run_row = l_rows[hh];
      if (q_row >= p.Sq) continue;
      const long long pidx = (((long long)b * p.Sq + q_row) * p.H + h) * p.splits + split;
      const float wv = *p.scale_v * kPBoostInv;   // V was stored as v16 * scale_v, P as p * 2^15
#pragma unroll
      for (int g = 0; g < kHeadDim / 8; ++g) {
        const int c = g * 8 + quad * 2;
        *reinterpret_cast<float2*>(p.o_part + pidx * kHeadDim + c) =
            make_float2(o[4 * g + 2 * hh] * wv, o[4 * g + 2 * hh + 1] * wv);
      }
      if (quad == 0) {
        p.ml_part[pidx * 2] = m_run[hh];
        p.ml_part[pidx * 2 + 1] = l_run_row;
      }
    }
  } else {
  // ---------------------------------------------------------------- epilogue: merge carry, write
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q_row = r0 + 8 * hh;
    const float l_run_row = quad_sum(l_run[hh]);
    const long long ml_idx = ((long long)b * p.H + h) * p.Sq + q_row;
    const long long o_idx = (((long long)b * p.Sq + q_row) * p.H + h) * kHeadDim;
    float m_c = -INFINITY, l_c = 0.f;
    if (!p.first) {
      m_c = p.acc_m[ml_idx];
      l_c = p.acc_l[ml_idx];
    }
    const float m_new = fmaxf(m_c, m_run[hh]);
    float wa = (m_c == -INFINITY) ? 0.f : ex2f(m_c - m_new);          // weight of the carry
    float wb = (m_run[hh] == -INFINITY) ? 0.f : ex2f(m_run[hh] - m_new);  // weight of this step
    const float l_new = wa * l_c + wb * l_run_row;
    // kDrop: no surviving key in the whole row (its max never left the masked level): out = 0, lse at the masked level
    const bool dead = kDrop && p.last && m_new <= kMaskedLogit;
    if (p.scale_v) wb *= *p.scale_v * (kF16 ? kPBoostInv : 1.f);   // V was stored as v16 * scale_v, P as p * 2^15
    if (p.last) {
      const float inv = l_new > 0.f ? 1.0f / l_new : 0.f;
      wa *= inv;
      wb *= inv;
    }
#pragma unroll
    for (int g = 0; g < kHeadDim / 8; ++g) {
      const int c = g * 8 + quad * 2;
      float2 f = make_float2(o[4 * g + 2 * hh] * wb, o[4 * g + 2 * hh + 1] * wb);
      if (!p.first) {
        const float2 a2 = *reinterpret_cast<const float2*>(p.acc_o + o_idx + c);
        f.x = fmaf(a2.x, wa, f.x);
        f.y = fmaf(a2.y, wa, f.y);
      }
      if (dead) f = make_float2(0.f, 0.f);
      if (p.last) {
        *reinterpret_cast<uint32_t*>(p.out + o_idx + c) = pack_bf16x2(f.x, f.y);
        if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + o_idx + c) = f;
      } else {
        *reinterpret_cast<float2*>(p.acc_o + o_idx + c) = f;
      }
    }
    if (quad == 0) {
      if (p.last) {
        p.lse[ml_idx] = dead ? kMaskedLogit * kLn2 : l_new > 0.f ? (m_new + log2f(l_new)) * kLn2 : -INFINITY;
      } else {
        p.acc_m[ml_idx] = m_new;
        p.acc_l[ml_idx] = l_new;
      }
    }
  }
  }
}

template <bool kF16, bool kInfer = false, bool kMap = false>
__global__ void __launch_bounds__(kFwdThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ FwdParams p) {
  attn_fwd_body<kF16, kInfer, kMap, false>(tmQ, tmK, tmV, p);
}

template <bool kF16, bool kMap>
__global__ void __launch_bounds__(kFwdThreads, 1)
attn_fwd_dropout_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ FwdParams p) {
  attn_fwd_body<kF16, false, kMap, true>(tmQ, tmK, tmV, p);
}

static bool make_qkv_tmap(CUtensorMap* tm, const void* ptr, int B, int S, int H) {
  // [B, S, H, 128] bf16 -> dims (d, h, s, b); one box = 64 d x 128 rows of one head (128B swizzle)
  uint64_t dims[4] = {uint64_t(kHeadDim), uint64_t(H), uint64_t(S), uint64_t(B)};
  uint64_t strides[3] = {uint64_t(kHeadDim) * 2, uint64_t(H) * kHeadDim * 2, uint64_t(S) * H * kHeadDim * 2};
  uint32_t box[4] = {64, 1, uint32_t(kTile), 1};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace lwm

using namespace lwm;

// One attn_fwd_kernel or attn_fwd_dropout_kernel instance; its dynamic shared-memory limit is raised once per device.
template <bool kF16, bool kInfer, bool kMap, bool kDrop>
static int launch_fwd(dim3 grid, cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                      const FwdParams& p) {
  static_assert(!(kInfer && (kMap || kDrop)), "the inference mode has no block-map or dropout instance");
  void (*kernel)(CUtensorMap, CUtensorMap, CUtensorMap, FwdParams);
  if constexpr (kDrop) kernel = attn_fwd_dropout_kernel<kF16, kMap>;
  else kernel = attn_fwd_kernel<kF16, kInfer, kMap>;
  static bool attr_set_dev[64] = {};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  bool& attr_set = attr_set_dev[cur_dev & 63];      // function attributes are per device
  if (!attr_set) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmemBytes) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "attn_fwd: cannot raise dynamic shared memory limit");
    attr_set = true;
  }
  kernel<<<grid, kFwdThreads, kFwdSmemBytes, st>>>(tq, tk, tv, p);
  return lwm_check_launch(kDrop ? "attn_fwd_dropout_kernel" : kInfer ? "attn_fwd_kernel (inference)" : "attn_fwd_kernel");
}

// One ring step (include/lwm_b200.h): the scales select the fp16-operand kernel, tiles / tile_count the block map,
// drop_threshold > 0 the dropout instances.
extern "C" int lwm_attn_fwd_step(const void* q, const void* k, const void* v, const float* scale_q,
                                 const float* scale_k, const float* scale_v, float* out_f32, void* out, float* lse,
                                 float* acc_o, float* acc_m, float* acc_l, int B, int H, int Sq, int Sk, int D,
                                 long long q_pos0, long long k_pos0, int causal, const float* bias,
                                 long long bias_stride, const int* segment_ids, long long seg_stride,
                                 float softmax_scale, int first, int last, const int* tiles, const int* tile_count,
                                 long long seed, unsigned drop_threshold, int batch0, void* stream) {
  if (!scale_k != !scale_q || !scale_v != !scale_q)
    return lwm_fail(LWM_ERR_ARG, "attn_fwd: scales are all given (fp16 operands) or all null (bf16)");
  if (out_f32 && !scale_q) return lwm_fail(LWM_ERR_ARG, "attn_fwd: out_f32 needs the fp16 operand scales");
  if (!tiles != !tile_count) return lwm_fail(LWM_ERR_ARG, "attn_fwd: tiles and tile_count are both given or both null");
  if (tiles && !bias && !segment_ids) return lwm_fail(LWM_ERR_ARG, "attn_fwd: a block map needs bias or segment_ids");
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_fwd: head_dim must be 128");
  if (B <= 0 || H <= 0 || Sq <= 0 || Sk <= 0 || Sq % kTile || Sk % kTile)
    return lwm_fail(LWM_ERR_SHAPE, "attn_fwd: Sq and Sk must be positive multiples of 128");
  if (!q || !k || !v) return lwm_fail(LWM_ERR_ARG, "attn_fwd: null q/k/v");
  if (last && (!out || !lse)) return lwm_fail(LWM_ERR_ARG, "attn_fwd: out/lse required on the last step");
  if (!(first && last) && (!acc_o || !acc_m || !acc_l))
    return lwm_fail(LWM_ERR_ARG, "attn_fwd: carry buffers required unless first && last");
  if (q_pos0 + Sq > 0x7fffffffLL || k_pos0 + Sk > 0x7fffffffLL)
    return lwm_fail(LWM_ERR_SHAPE, "attn_fwd: global positions must fit in int32");
  if (bias && bias_stride < k_pos0 + Sk)
    return lwm_fail(LWM_ERR_SHAPE, "attn_fwd: bias is indexed by GLOBAL key position: bias_stride < k_pos0 + Sk");
  if (segment_ids && (seg_stride < q_pos0 + Sq || seg_stride < k_pos0 + Sk))
    return lwm_fail(LWM_ERR_SHAPE, "attn_fwd: segment_ids is indexed by GLOBAL position: seg_stride < max(q_pos0 + Sq, k_pos0 + Sk)");
  DropParams drop;
  if (const int s = decode_drop_params(seed, drop_threshold, batch0, B, H, q_pos0, k_pos0, "attn_fwd", &drop)) return s;
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tq, tk, tv;
  if (!make_qkv_tmap(&tq, q, B, Sq, H) || !make_qkv_tmap(&tk, k, B, Sk, H) || !make_qkv_tmap(&tv, v, B, Sk, H))
    return lwm_fail(LWM_ERR_CUDA, "attn_fwd: cuTensorMapEncodeTiled failed (pointers must be 16B aligned)");
  FwdParams p{};
  p.B = B; p.H = H; p.Sq = Sq; p.Sk = Sk;
  p.scale_log2 = softmax_scale * kLog2e;
  p.mask.q_pos0 = int(q_pos0); p.mask.k_pos0 = int(k_pos0); p.mask.causal = causal;
  p.mask.bias = bias; p.mask.bias_stride = bias_stride;
  p.mask.seg = segment_ids; p.mask.seg_stride = seg_stride;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.lse = lse; p.acc_o = acc_o; p.acc_m = acc_m; p.acc_l = acc_l;
  p.first = first; p.last = last;
  p.scale_q = scale_q; p.scale_k = scale_k; p.scale_v = scale_v;
  p.out_f32 = out_f32;
  p.bits = nullptr; p.tiles = tiles; p.tile_count = tile_count;
  p.n_kt = Sk / kTile; p.splits = 1;
  p.drop = drop;
  const dim3 grid(Sq / kTile, H, B);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_flags([&](auto f16, auto map, auto dropout) {
    return launch_fwd<f16, false, map, dropout>(grid, st, tq, tk, tv, p);
  }, scale_q != nullptr, tiles != nullptr, drop.thr != 0);
}

// Inference mode (ringattention_inference with Q >= kInferMinQ rows): q16 [B,Q,H,128], k16/v16 [B,Sk,H,128] scaled fp16
// copies, any Q and Sk; bits / tiles / tile_count from lwm_attn_mask_pack + lwm_attn_infer_tilemap. Writes one
// partial per (b, q, h) row: o_part [B*Q*H,128], ml_part [B*Q*H,2] (the decode partial layout). splits > 1: CTAs per
// Q tile, each over a slice of its tile list; their partials go through workspace (splits * B*Q*H * 130 floats) and
// are merged here.
extern "C" int lwm_attn_infer_partial(const void* q16, const void* k16, const void* v16, const float* scale_q,
                                      const float* scale_k, const float* scale_v, const unsigned* bits,
                                      const int* tiles, const int* tile_count, float* o_part, float* ml_part,
                                      void* workspace, int B, int H, int Q, int Sk, int D, int splits,
                                      float softmax_scale, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_infer_partial: head_dim must be 128");
  if (!q16 || !k16 || !v16 || !scale_q || !scale_k || !scale_v || !tiles || !tile_count || !o_part || !ml_part)
    return lwm_fail(LWM_ERR_ARG, "attn_infer_partial: null pointer");
  if (splits > 1 && !workspace) return lwm_fail(LWM_ERR_ARG, "attn_infer_partial: workspace required when splits > 1");
  if (B <= 0 || H <= 0 || Q <= 0 || Sk <= 0 || B > 65535 || H > 65535 || splits <= 0 || splits > 1024)
    return lwm_fail(LWM_ERR_SHAPE, "attn_infer_partial: bad shape (B, H <= 65535; 1 <= splits <= 1024)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  CUtensorMap tq, tk, tv;
  if (!make_qkv_tmap(&tq, q16, B, Q, H) || !make_qkv_tmap(&tk, k16, B, Sk, H) || !make_qkv_tmap(&tv, v16, B, Sk, H))
    return lwm_fail(LWM_ERR_CUDA, "attn_infer_partial: cuTensorMapEncodeTiled failed (pointers must be 16B aligned)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long rows = (long long)B * Q * H;
  FwdParams p{};
  p.B = B; p.H = H; p.Sq = Q; p.Sk = Sk;
  p.scale_log2 = softmax_scale * kLog2e;
  p.first = 1; p.last = 0;
  p.scale_q = scale_q; p.scale_k = scale_k; p.scale_v = scale_v;
  p.bits = bits; p.tiles = tiles; p.tile_count = tile_count;
  p.n_kt = (Sk + kTile - 1) / kTile;
  p.splits = splits;
  p.o_part = splits > 1 ? reinterpret_cast<float*>(workspace) : o_part;
  p.ml_part = splits > 1 ? reinterpret_cast<float*>(workspace) + rows * splits * kHeadDim : ml_part;
  const dim3 grid(unsigned((Q + kTile - 1) / kTile * splits), H, B);
  const int s = launch_fwd<true, true, false, false>(grid, st, tq, tk, tv, p);
  if (s || splits == 1) return s;
  lwm_decode_merge_partials(p.o_part, p.ml_part, splits, o_part, ml_part, rows, st);
  return lwm_check_launch("decode_merge_kernel");
}
