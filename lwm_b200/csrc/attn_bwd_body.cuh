// The body of attn_bwd_kernel and attn_bwd_dropout_kernel (attn_bwd.cu), included inside both: with the body in a
// shared __device__ function instead, ptxas schedules the existing ordered instances differently.
// In scope: the kernel parameters tmQ, tmK, tmV, tmDO, tmDQ, p and the compile-time flags kF16, kMap, kBits, kOrdered,
// kDrop.
  // no static shared memory in this kernel: the dynamic window starts 1024-aligned (checked below)
  extern __shared__ __align__(1024) uint8_t smem[];
  float (*s_lse)[kBQ] = reinterpret_cast<float (*)[kBQ]>(smem + kOffLse);
  float (*s_delta)[kBQ] = reinterpret_cast<float (*)[kBQ]>(smem + kOffDelta);
  BwdBarriers& bars = *reinterpret_cast<BwdBarriers*>(smem + kOffBars);
  if (smem_u32(smem) & 1023u) __trap();

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // (n, h, b): blockIdx, or with kOrdered the ticket's, kept in shared memory. The consumer warpgroups re-read them
  // where they use them (as the other instances re-read blockIdx) rather than hold them in registers across their loop.
  volatile int* s_nhb = reinterpret_cast<volatile int*>(smem + kOffTicket);
  if constexpr (kOrdered) take_ticket(p.order_ws, p.H, p.B, s_nhb);
  auto cta_n = [&]() -> int { return kOrdered ? s_nhb[0] : int(blockIdx.x); };
  auto cta_h = [&]() -> int { return kOrdered ? s_nhb[1] : int(blockIdx.y); };
  auto cta_b = [&]() -> int { return kOrdered ? s_nhb[2] : int(blockIdx.z); };
  const int n = cta_n();  // kv tile (ascending = heaviest first under causal masking)
  const int h = cta_h(), b = cta_b();
  const int n_q_tiles = p.Sq / kBQ;
  // first Q tile with a row that can see key 0 of key tile kt
  auto first_q_tile = [&](int kt) {
    if (!p.mask.causal) return 0;
    const long long diff = (long long)p.mask.k_pos0 + (long long)kt * kTile - p.mask.q_pos0;
    return diff <= 0 ? 0 : int(min(diff / kBQ, (long long)n_q_tiles));
  };
  const int i_start = first_q_tile(n);
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
        int* sem = nullptr;
        if constexpr (kOrdered) {
          sem = p.order_ws + kOrderHeader + (b * p.H + h) * n_q_tiles + row0 / kBQ;
          dq_wait_turn(sem, kMap ? p.turns[list0 + it] : n, p.order_ws + 1);
        }
#pragma unroll
        for (int j = 0; j < kHeadDim / 32; ++j)
          tma_reduce_add_4d(&tmDQ, smem + kOffDQ + st * kDQB + j * kDQBox, 32 * j, h, row0, b);
        tma_commit_group();
        tma_wait_group_read<0>();
        mbar_arrive(&bars.dq_empty[st]);   // the staging tile is free once read, before the reductions complete
        if constexpr (kOrdered) dq_pass_turn(sem);
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
  // positions fit in int32 (checked on the host); int keeps the loop under the register budget. kOrdered recomputes it
  // (and i_start) from cta_n() where it is used.
  const int wg_k_last = p.mask.k_pos0 + n * kTile + wg * 64 + 63;
  auto k_last = [&]() { return kOrdered ? p.mask.k_pos0 + cta_n() * kTile + wg * 64 + 63 : wg_k_last; };

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
    const int q_tile_pos = p.mask.q_pos0 + (kMap ? entry >> 1 : (kOrdered ? first_q_tile(cta_n()) : i_start) + it) * kBQ;
    // kMap: clean tiles keep the masked path's rounding (fmaf(s, scale, 0)): bit-identical to the step without a map
    const bool need_mask =
        kBits ? bool(entry & 1) : (kDrop || kMap || has_bias || has_seg || (p.mask.causal && q_tile_pos < k_last()));
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
      const int key0 = cta_n() * kTile + kr0;
      const int sh = key0 & 31;
      const int kw = gridDim.x * 4;
      const uint32_t* wcol = p.bits ? p.bits + (long long)cta_b() * p.q_rows * kw + (key0 >> 5) : nullptr;
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
      const int bt = cta_b();
      const int* seg_row = use_seg ? p.mask.seg + (long long)bt * p.mask.seg_stride : nullptr;
      const int k_pos = p.mask.k_pos0 + cta_n() * kTile + kr0;   // this thread's keys: k_pos, k_pos + 8
      // kDrop: bit i of dropped is the decision of fragment entry i (query column 8 g + 2 quad + e, g = i >> 2,
      // e = i & 1; key k_pos + 8 hh, hh = (i >> 1) & 1). Call c covers columns 16 t + 2 quad + e and + 8 (t = c >> 1,
      // e = c & 1) against keys k_pos and k_pos + 8: kr0 & 15 < 8, and q_pos0, k_pos0 are multiples of 128 (checked on
      // the host), so the pairs differ in bit 3 only. The query's bit 3 picks the word pair, the key's the word.
      uint32_t dropped = 0u;
      if constexpr (kDrop) {
#pragma unroll 1   // one call at a time: unrolled, the 8 independent calls are interleaved and spill
        for (int c = 0; c < 8; ++c) {
          const int t = c >> 1, e = c & 1;
          const uint4 r = drop_block(p.drop, q_tile_pos + 16 * t + 2 * quad + e, k_pos, cta_h(), bt);
#pragma unroll
          for (int qb = 0; qb < 2; ++qb)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
              dropped |= uint32_t(drop_pick(r, qb, hh, k_pos & 1, p.drop.thr)) << (4 * (2 * t + qb) + 2 * hh + e);
        }
      }
      int my_seg[2];
      float bias_t[2] = {0.f, 0.f};
      bool key_masked[2] = {false, false};
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        my_seg[hh] = use_seg ? seg_row[k_pos + 8 * hh] : 0;
        if (use_bias) {
          bias_t[hh] = p.mask.bias[(long long)bt * p.mask.bias_stride + k_pos + 8 * hh] * kLog2e;
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
        if (kDrop && ((dropped >> i) & 1u)) tv = kMaskedLogit;
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
    if (kBits && cta_n() * kTile + kr0 + 8 * hh >= p.Sk) continue;   // key rows past the cache are not written
    const long long row =
        ((((long long)cta_b() * p.Sk + (long long)cta_n() * kTile + kr0 + 8 * hh) * p.H + cta_h()) * kHeadDim);
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
