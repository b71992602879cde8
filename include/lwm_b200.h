/* lwm_b200 — C ABI of the H100 (sm_90a) hot-path library: liblwm_b200.so
 *
 * This is the drop-in boundary for the two LWM hot paths (SURVEY.md §8b):
 *   - the blockwise `ringattention(q, k, v, attn_bias, segment_ids, ...)` call bound at
 *     the reference's lwm/llama.py:539-569 (forward) and its custom_vjp backward;
 *   - the VQGAN tokenizer ops of lwm/vqgan.py:105-351 (conv / GroupNorm / SiLU / resample /
 *     nearest-codebook lookup).
 * The reference has no native boundary of its own (it is pure Python/JAX); these entry points are
 * what a Python (ctypes / XLA-FFI custom call) binding on the reference side would bind — see
 * INTEGRATION.md for the stub.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless named host_*;
 *   - all tensor memory is caller-owned; calls are asynchronous on `stream` (a cudaStream_t);
 *   - return value: 0 on success, LWM_ERR_* otherwise; lwm_last_error() gives the message
 *     (thread-local). There is NO CPU fallback: on a non-sm_90 device every call fails with
 *     LWM_ERR_DEVICE;
 *   - one host thread per GPU/process (torchrun model); contexts are not thread-safe.
 */
#ifndef LWM_B200_H_
#define LWM_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define LWM_B200_ABI_VERSION 5

#define LWM_OK 0
#define LWM_ERR_DEVICE 1
#define LWM_ERR_SHAPE 2
#define LWM_ERR_ARG 3
#define LWM_ERR_CUDA 4

int lwm_abi_version(void);
const char* lwm_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * Ring attention, forward: ONE ring step (one held K/V block against the local query shard).
 * Replaces the body of the reference's per-step `_blockwise_attention_fwd` (un-vendored
 * `ringattention` package; call site lwm/llama.py:541-569; algorithm SURVEY.md Appendix A).
 *
 *   q            [B, Sq, H, D] bf16      local query shard (contiguous)
 *   k, v         [B, Sk, H, D] bf16      the K/V block currently held by this rank
 *   scale_q/k/v  all NULL (bf16 operands), or all given: fp16 operand mode (below), q/k/v are the scaled fp16 copies
 *                and these their device scales
 *   out_f32      fp16 operand mode only, else NULL: the un-rounded fp32 copy of `out`, written when `last`, so that
 *                delta = rowsum(dO o O) of the backward is not limited by the bf16 rounding of `out`
 *   out          [B, Sq, H, D] bf16      final output, written when `last`
 *   lse          [B, H, Sq]    fp32      log-sum-exp (natural log) of the scaled+biased logits,
 *                                        written when `last` (residual for the backward)
 *   acc_o/m/l    fp32 carries [B,Sq,H,D] / [B,H,Sq] / [B,H,Sq] (numerator, running max in the
 *                log2 domain, denominator) — the reference's (numerator, max_score, denominator)
 *                scan carry. Read unless `first`, written unless `last`. May be NULL when
 *                first && last (single-step, ring_size 1).
 *   q_pos0/k_pos0 global token position of local row 0 of q / of the held k block: causal,
 *                bias and segment masks are evaluated on GLOBAL positions as in the reference's
 *                _chunk_attention_bias.
 *   causal       1 <=> blockwise_kwargs.causal_block_size == 1 ; 0 <=> None
 *   bias         [B, bias_stride] fp32 additive per-key bias indexed by global key position
 *                (the [B,1,1,S_global] attn_bias of lwm/llama.py:533-537 squeezed), or NULL
 *   segment_ids  [B, seg_stride] int32 indexed by global position, or NULL
 *   softmax_scale 1/sqrt(D)
 *   tiles, tile_count  both NULL, or the forward block map of lwm_attn_step_tilemap built from the same arguments (bias
 *                or segment_ids required then): the kernel visits only the KV tiles in it. Results are bit-identical.
 *   seed, drop_threshold, batch0  attention dropout (below); drop_threshold 0: none, seed is ignored.
 * Constraints: D == 128; Sq, Sk multiples of 128. A partial set of scales, out_f32 without scales, or only one of
 * tiles / tile_count is LWM_ERR_ARG.
 *
 * Attention dropout (the reference's blockwise_kwargs deterministic=False, attn_pdrop=p, dropout_rng): a dropped (q, k)
 * entry is removed from the numerator and the denominator of the softmax (it takes the masked logit; no 1/(1-p)
 * rescale), so P = 0 and dS = 0 there in the backward. A row left without a surviving key (every visible key dropped,
 * or fully masked) writes out = 0 and an lse at the masked level (lwm_attn_bwd_lse turns it into -inf: zero gradients).
 * The mask is regenerated from (seed, drop_threshold, b, h, GLOBAL q, GLOBAL k) in the tile kernels, never stored
 * (lwm_b200/csrc/attn_dropout.cuh): Philox4x32-10, key (seed & 0xffffffff, seed >> 32), counter
 * (((k >> 4) << 2) | ((k >> 1) & 3), q & ~8, h, b), the 16-bit half k & 1 of word 2 ((q >> 3) & 1) + ((k >> 3) & 1);
 * dropped iff it is below drop_threshold = min(65535, round(p * 65536)). b is the GLOBAL batch row: batch0 >= 0 is the
 * global batch row of the call's batch row 0 (a caller that launches a slice of the batch passes its offset, so that
 * every batch row draws its own mask). The same for any ring layout, chunking, block map or executor.
 * drop_threshold > 65535 or batch0 < 0 is LWM_ERR_ARG. With dropout, q_pos0 and k_pos0 must be multiples of 128, B and
 * H <= 65535 and batch0 + B < 2^31 (LWM_ERR_SHAPE).
 * lwm_attn_dropout_mask: out [n_q, n_k] uint8 = the decisions (1 = dropped) of batch row b, head h, global queries
 *   q_pos0 .. q_pos0 + n_q - 1 and keys k_pos0 .. k_pos0 + n_k - 1 (drop_threshold in [1, 65535]), from the tile
 *   kernels' device function.
 */
int lwm_attn_fwd_step(const void* q, const void* k, const void* v, const float* scale_q, const float* scale_k,
                      const float* scale_v, float* out_f32, void* out, float* lse, float* acc_o, float* acc_m,
                      float* acc_l, int B, int H, int Sq, int Sk, int D, long long q_pos0, long long k_pos0, int causal,
                      const float* bias, long long bias_stride, const int* segment_ids, long long seg_stride,
                      float softmax_scale, int first, int last, const int* tiles, const int* tile_count, long long seed,
                      unsigned drop_threshold, int batch0, void* stream);
int lwm_attn_dropout_mask(long long seed, unsigned drop_threshold, int b, int h, long long q_pos0, long long k_pos0,
                          int n_q, int n_k, unsigned char* out, void* stream);

/* Ring attention, forward step of the fp8 mode (no gradient: the prefill under torch.no_grad()). S = Q K^T runs on the
 * FP8 tensor cores; P V, the softmax, the carries and the epilogue are those of the fp16 operand mode.
 *   q8, k8       [B, Sq, H, 128] / [B, Sk, H, 128] e4m3 copies x8 = e4m3(x / scale), scale = 2^(e-7) with e the
 *                exponent of the tensor's largest finite |x| (lwm_attn_e4m3_scale_from_absmax, lwm_attn_to_e4m3_scaled)
 *   v16          [B, Sk, H, 128] fp16 copy of v as in the fp16 operand mode (scale 2^(e-12), lwm_attn_to_f16_scaled)
 *   scale_q/k/v  their device scales, all required
 * The logits are (q8 . k8) * scale_q * scale_k in fp32. Every other argument, constraint and output is that of
 * lwm_attn_fwd_step in the fp16 operand mode (out_f32 optional); there is no dropout. */
int lwm_attn_fwd_e4m3_step(const void* q8, const void* k8, const void* v16, const float* scale_q, const float* scale_k,
                           const float* scale_v, float* out_f32, void* out, float* lse, float* acc_o, float* acc_m,
                           float* acc_l, int B, int H, int Sq, int Sk, int D, long long q_pos0, long long k_pos0,
                           int causal, const float* bias, long long bias_stride, const int* segment_ids,
                           long long seg_stride, float softmax_scale, int first, int last, const int* tiles,
                           const int* tile_count, void* stream);

/* Ring attention, backward.
 * lwm_attn_bwd_prep: delta[b,h,s] = sum_d dout[b,s,h,d] * out[b,s,h,d]  (fp32), once per backward. out fp32
 *                    (out_dtype 0) or bf16 (1); dout bf16 when scale_do is NULL, else its scaled fp16 copy with its
 *                    device scale.
 * lwm_attn_bwd_lse:  nlse2[i] = -lse[i]*log2(e) + offset_log2 (-inf for rows whose lse is at the masked level), once per
 *                    backward; lwm_attn_bwd_step takes THIS array as its `lse` argument (the per-tile kernel is
 *                    exp-bound). offset_log2 = 0 for bf16 operands and LWM_ATTN_F16_P_BOOST_LOG2 for the fp16 operand
 *                    mode: the fp16 kernel keeps P^T * 2^14 so that the normalised probabilities of a 128K .. 1M-key
 *                    row stay normal fp16 numbers.
 * lwm_attn_bwd_step: one ring step of the reference's custom_vjp bwd (SURVEY.md Appendix A `bwd`):
 *   recomputes P from (q, k, lse), accumulates
 *     dq_acc [B,Sq,H,D] fp32 += dS K / sqrt(D)        (atomic fp32 tile reductions; zero it first)
 *     dk_acc [B,Sk,H,D] fp32 += dS^T Q / sqrt(D)      (read-modify-write by the owning CTA)
 *     dv_acc [B,Sk,H,D] fp32 += P^T dO
 *   dk_acc/dv_acc travel with the K/V block around the ring exactly like the reference's dk, dv.
 *   dkv_init != 0: the dk_acc/dv_acc rows of the key tiles this launch visits are WRITTEN instead of accumulated
 *   (first visit of a block: saves zero-filling the accumulators); key tiles no query row can see are zero-filled.
 *   scale_q/k/v/do: all NULL (bf16 operands) or all given (fp16 operand mode, dout its scaled fp16 copy too);
 *   tiles, tile_count: both NULL, or the backward block map of lwm_attn_step_tilemap (bias or segment_ids required):
 *   dK and dV are bit-identical to the call without it, dQ differs only by the order of its fp32 reductions, which
 *   already varies from run to run;
 *   order_ws: NULL, or the workspace of the ordered dQ reduction (below);
 *   seed, drop_threshold, batch0: the forward's attention dropout. Other arguments as for lwm_attn_fwd_step.
 * Reproducible dQ (what torch.use_deterministic_algorithms(True) asks for): with an order_ws, every dQ element receives
 * its key tiles' fp32 contributions in ascending key-tile order, so dQ is the same bits on every run (dK and dV already
 * are); lwm_attn_infer_bwd (below) takes it the same way. order_ws is a caller-owned int32 workspace of
 *     2 + B * H * ceil(Sq/64)                    words without a block map,
 *     2 + B * H * ceil(Sq/64) + B * n_kt * ceil(Sq/64)   with one (n_kt = ceil(Sk/128); Sq = Q for the inference op),
 * used on the call's stream and zeroed there by the call; it must not be shared by calls that may run concurrently.
 * B, H <= 65535, and the workspace words and B * H * n_kt must fit in int32 (LWM_ERR_SHAPE).
 * Word 1 is an error flag: nonzero after the call if a dQ tile waited more than 4 s for its turn (a bug, never expected;
 * the reduction then went on unordered).
 */
#define LWM_ATTN_F16_P_BOOST_LOG2 14.0f
int lwm_attn_bwd_prep(const void* out, int out_dtype, const void* dout, const float* scale_do, float* delta, int B,
                      int H, int Sq, int D, void* stream);
int lwm_attn_bwd_lse(const float* lse, float* nlse2, long long n, float offset_log2, void* stream);
int lwm_attn_bwd_step(const void* q, const void* k, const void* v, const void* dout, const float* scale_q,
                      const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                      const float* delta, float* dq_acc, float* dk_acc, float* dv_acc, int B, int H, int Sq, int Sk,
                      int D, long long q_pos0, long long k_pos0, int causal, const float* bias, long long bias_stride,
                      const int* segment_ids, long long seg_stride, float softmax_scale, int dkv_init,
                      const int* tiles, const int* tile_count, int* order_ws, long long seed, unsigned drop_threshold,
                      int batch0, void* stream);

/* fp16-internal precision mode (optional): the tensor cores take bf16 x bf16 or fp16 x fp16 only, so the
 * higher-precision mode converts every operand once to an exact, power-of-two-scaled fp16 copy
 * (lwm_attn_to_f16: x16 = x / scale, scale = 2^(e-12) with e the exponent of the tensor's largest FINITE |x|,
 * clamped at -114; 1 when no element is finite and nonzero; NaN and +-inf stay what they are) and keeps the
 * probabilities P and dS at fp16's 11 significant bits instead of bf16's 8. The scales are DEVICE scalars written
 * by lwm_attn_to_f16; all scale factors are undone in fp32 inside the kernels. Same semantics otherwise. */
int lwm_attn_to_f16(const void* src_bf16, void* dst_f16, float* scale_out, void* workspace4, long long n, void* stream);

/* Block map of a training step with a padding bias and/or segment ids (packed or padded sequences): the tile kernels
 * then visit only the (Q tile, KV tile) pairs that hold a visible entry, and read the mask only where it varies.
 * lwm_attn_step_tilemap  bias / segment_ids as for lwm_attn_fwd_step (at least one non-null), the step's B, Sq, Sk,
 *                        q_pos0, k_pos0, causal -> forward map fwd_tiles [B][Sq/128][Sk/128] (per 128-row Q tile the
 *                        ascending KV tiles kt*2 + mixed), fwd_count [B][Sq/128], and backward map bwd_tiles
 *                        [B][Sk/128][Sq/64] (per 128-key K tile the ascending 64-row Q tiles qt*2 + mixed), bwd_count
 *                        [B][Sk/128]. Either map may be omitted (both of its pointers null). workspace >=
 *                        B * (Sq/64 + Sk/128) * 16 bytes. A pair is left out when every entry is masked (bias below the
 *                        masked level, or disjoint segment ids); in the forward only for Q tiles whose every row sees its
 *                        own key in this step. mixed = the pair reads bias / segment ids per element. */
int lwm_attn_step_tilemap(const float* bias, long long bias_stride, const int* segment_ids, long long seg_stride, int B,
                          int Sq, int Sk, long long q_pos0, long long k_pos0, int causal, int* fwd_tiles, int* fwd_count,
                          int* bwd_tiles, int* bwd_count, void* workspace, void* stream);

/* Sharded-tensor variant of the fp16 operand conversion (ring executor): every rank publishes the bit pattern of the
 * largest finite |x| of its shard (lwm_attn_absmax: atomicMax into *out_bits, caller zeroes it; NaN and +-inf are
 * skipped; dtype 0 = fp32, 1 = bf16), all ranks derive
 * the SAME power-of-two scale from the gathered patterns (lwm_attn_scale_from_absmax over bits[i*stride], i < n), and
 * convert with it (lwm_attn_to_f16_scaled: dst = fp16(x / *scale); an fp32 source — the dtype the reference's scripts
 * run with — is rounded ONCE to fp16's 11 significant bits instead of going through bf16's 8).
 * lwm_reduce_cast_f32: dst = cast(sum of n_src <= 16 fp32 arrays, fixed order) — folds the dK/dV partials that
 * landed in the owner's heap and writes the gradient in its final dtype (0 fp32, 1 bf16) in one pass. host_srcs is a
 * HOST array of device pointers. */
#define LWM_REDUCE_MAX_SRCS 16
int lwm_attn_absmax(const void* x, int dtype, long long n, unsigned* out_bits, void* stream);
/* largest finite |x| -> *scale_out = 2^(e-12) in one call (workspace: 4 bytes, zeroed here) */
int lwm_attn_absmax_scale(const void* x, int dtype, long long n, unsigned* workspace, float* scale_out, void* stream);
int lwm_attn_scale_from_absmax(const unsigned* bits, int n, int stride, float* scale_out, void* stream);
int lwm_attn_to_f16_scaled(const void* x, int dtype, void* dst_f16, const float* scale, long long n, void* stream);
/* e4m3 operand copies of the fp8 mode (lwm_attn_fwd_e4m3_step), same protocol with a smaller top exponent:
 * lwm_attn_e4m3_scale_from_absmax: *scale_out = 2^(e-7) from the gathered patterns (e clamped at -114; 1 when every
 *   pattern is 0), so the largest finite |x| / scale lies in [128, 256), below e4m3's 448: nothing saturates.
 * lwm_attn_to_e4m3_scaled: dst [n] bytes = e4m3(x / *scale), round to nearest even, bit for bit torch's
 *   x.div(scale).to(torch.float8_e4m3fn) for finite x. e4m3fn has no infinity: +-inf become the NaN bytes 0x7f / 0xff
 *   (as torch's cast) and a NaN a NaN byte of either sign, where the fp16 copies keep +-inf. dtype 0 = fp32, 1 = bf16;
 *   n % 8 == 0. */
int lwm_attn_e4m3_scale_from_absmax(const unsigned* bits, int n, int stride, float* scale_out, void* stream);
int lwm_attn_to_e4m3_scaled(const void* x, int dtype, void* dst_e4m3, const float* scale, long long n, void* stream);
int lwm_reduce_cast_f32(const float* const* host_srcs, int n_src, void* dst, int dst_dtype, long long n, void* stream);

/* Decode-time attention — the reference's `ringattention_inference(q, k, v, attn_mask, axis_name)` (call site
 * lwm/llama.py:601-614; SURVEY.md §8f next-row 1): a few query rows against this rank's KV-cache shard with an
 * explicit boolean mask [B,1,Q,K_global] (nonzero = attend; masked logits take finfo.min semantics).
 * lwm_attn_decode_partial reduces the local shard to one partial per (b, q, h): numerator o_part [B*Q*H,128] fp32 and
 * ml_part [B*Q*H,2] = (max in the log2 domain, denominator). q, k, v are all fp32 (dtype 0, read directly) or all bf16
 * (1), k_exp and v_exp NULL; or k_exp and v_exp are both given: k / v are then the 8-bit KV cache (below) with these
 * exponents, dtype is q's, and the partials are bit for bit those on the cache dequantized to q's dtype. position_ids int32 [B,Q] and inv_freq [64] as for lwm_attn_rope, or both NULL: q is UN-rotated and is rotated as
 * it is loaded, rounded to its dtype — bit for bit lwm_attn_rope (out_dtype = dtype) followed by the call without
 * them, without the rotated q in memory. workspace >= splits * B*Q*H * 130 floats. HBM-bound: K and V are streamed
 * exactly once.
 * lwm_attn_decode_merge folds n_part partials (the all-gathered per-rank partials, laid out [row][n_part]) into out
 * [B,Q,H,128], bf16 (out_dtype 1) or the un-rounded fp32 (0), and lse [B*Q*H]. */
int lwm_attn_decode_partial(const void* q, const void* k, const void* v, int dtype, const signed char* k_exp,
                            const signed char* v_exp, const unsigned char* mask, float* o_part, float* ml_part, void* workspace, int B, int H, int Q, int Sk, int D,
                            long long k_pos0, long long mask_stride_b, long long mask_stride_q, int splits,
                            float softmax_scale, const int* position_ids, const float* inv_freq, void* stream);
int lwm_attn_decode_merge(const float* o_parts, const float* ml_parts, int n_part, void* out, int out_dtype, float* lse,
                          long long rows, void* stream);

/* Tensor-core inference path (multi-row queries). The mask becomes bits and a per-(b, 128-row Q tile) list of KV tiles:
 * lwm_attn_mask_pack      mask element (b, q, k) at mask[b*stride_b + q*stride_q + k*stride_k] (uint8/bool, nonzero =
 *                         attend; stride_b = 0 broadcasts over the batch) -> bits [n_slabs][B][Q][ceil(ncols/128)*4]
 *                         uint32 for the key columns [col0 + s*ncols, col0 + (s+1)*ncols) of slab s (bit j of word w
 *                         <=> column 32w + j; zero padded), and row_any [B][Q] int32 = the row has a true entry.
 * lwm_attn_infer_tilemap  bits [B][Q][ceil(Sk/128)*4] (null: every key visible), row_any [B][Q] over ALL keys of the
 *                         ring (null: no row is fully masked) -> tiles [B][ceil(Q/128)][ceil(Sk/128)] (kt*2 + mixed)
 *                         and tile_count [B][ceil(Q/128)].
 * lwm_attn_infer_partial  q16 [B,Q,H,128], k16/v16 [B,Sk,H,128] power-of-two-scaled fp16 copies (lwm_attn_to_f16_scaled)
 *                         with their device scales; fp32 logits, softmax and accumulation on the tensor cores. Writes
 *                         the decode partial layout o_part [B*Q*H,128], ml_part [B*Q*H,2]; splits > 1 CTAs per Q tile
 *                         need workspace >= splits * B*Q*H * 130 floats. Keys >= Sk enter no sum. */
int lwm_attn_mask_pack(const unsigned char* mask, long long stride_b, long long stride_q, long long stride_k, int B,
                       int Q, long long col0, int ncols, int n_slabs, unsigned* bits, int* row_any, void* stream);
int lwm_attn_infer_tilemap(const unsigned* bits, const int* row_any, int B, int Q, int Sk, int* tiles, int* tile_count,
                           void* stream);
int lwm_attn_infer_partial(const void* q16, const void* k16, const void* v16, const float* scale_q,
                           const float* scale_k, const float* scale_v, const unsigned* bits, const int* tiles,
                           const int* tile_count, float* o_part, float* ml_part, void* workspace, int B, int H, int Q,
                           int Sk, int D, int splits, float softmax_scale, void* stream);

/* Backward of the inference op (the VJP of s = where(mask, q.k/sqrt(D), finfo.min), softmax(s) v):
 * lwm_attn_infer_bwd_tilemap  bits [B][Q][ceil(Sk/128)*4] (null: every key visible), row_any [B][Q] over ALL keys of the
 *                         ring (null: every row live) -> per (b, 128-key tile) the ascending list of 64-row Q tiles,
 *                         tiles [B][ceil(Sk/128)][ceil(Q/64)] (t*2 + mixed) and tile_count [B][ceil(Sk/128)]. A pair is
 *                         left out when no live row (row < Q, row_any set) has a true bit in it, and clean (no mask
 *                         read) when every live row's bits are all true and every key is < Sk.
 * lwm_attn_infer_bwd      q16 / dout16 [B,Q,H,128], k16 / v16 [B,Sk,H,128] scaled fp16 copies with their device scales,
 *                         any Q and Sk. lse: lwm_attn_bwd_lse of the forward's lse with offset LWM_ATTN_F16_P_BOOST_LOG2,
 *                         -inf for rows with no visible key, and delta = rowsum(dout o out), both [B,H,Qp] with
 *                         Qp = Q rounded up to 64 (rows >= Q: lse -inf). dq_acc [B,Q,H,128] fp32 is accumulated into;
 *                         dk_acc / dv_acc [B,Sk,H,128] fp32 are written. Masked entries and keys >= Sk contribute
 *                         nothing; nothing outside the tensors' rows is read or written. order_ws: NULL, or the
 *                         workspace of the ordered dQ reduction, as for lwm_attn_bwd_step with its block map. */
int lwm_attn_infer_bwd_tilemap(const unsigned* bits, const int* row_any, int B, int Q, int Sk, int* tiles,
                               int* tile_count, void* stream);
int lwm_attn_infer_bwd(const void* q16, const void* k16, const void* v16, const void* dout16, const float* scale_q,
                       const float* scale_k, const float* scale_v, const float* scale_do, const float* lse,
                       const float* delta, const unsigned* bits, const int* tiles, const int* tile_count,
                       float* dq_acc, float* dk_acc, float* dv_acc, int B, int H, int Q, int Sk, int D,
                       float softmax_scale, int* order_ws, void* stream);

/* Attention prologue: rotary position embedding (lwm/llama.py:344-375 precompute_freqs_cis / apply_rotary_emb, applied
 * at llama.py:517-519 on the head-split projections right before the ring-attention call; SURVEY.md §8f next-row 2).
 * xq [B,S,Hq,128], xk [B,S,Hk,128] (= the [B,S,H*128] projection outputs: the head split is a view), dtype codes
 * 0 = fp32, 1 = bf16; out_* same shapes in out_dtype (the reference's `dtype` argument). position_ids [B,S] int32
 * (global positions; llama.py:515 gathers the table by them); inv_freq [64] fp32 = 1/theta^(2j/128) as the table builder
 * computes it (host mirror: lwm_b200.rope.precompute_inv_freq). The complex64 table is not materialised: the angle
 * float32(float64(pos)*float64(inv_freq[j])) is rebuilt in-kernel, cos/sin correctly rounded from double.
 * conj != 0 multiplies by the conjugate (the VJP of the rotation: gradients w.r.t. the un-rotated q/k). Hk may be 0. */
int lwm_attn_rope(const void* xq, const void* xk, int in_dtype, void* out_q, void* out_k, int out_dtype,
                  const int* position_ids, const float* inv_freq, int B, int S, int Hq, int Hk, int D, int conj,
                  void* stream);

/* The KV-cache write of the generation path with the rotary embedding on the keys (`ShardedKVCache.concatenate(...,
 * freqs_cis, position_ids)`): rows [src0, src0+n) of the UN-rotated k_new and of v_new [B,n_src,H,128] go to rows
 * [dst0, dst0+n) of this rank's cache shards cache_k / cache_v [B,L,H,128], all of one dtype (0 = fp32, 1 = bf16).
 * k is rotated at position_ids [B,n_src] int32 (the positions of the source rows) and rounded to the cache dtype, v
 * is copied: bit for bit lwm_attn_rope (out_dtype = in_dtype) followed by two row copies, in one launch. */
int lwm_kv_cache_write_rope(const void* k_new, const void* v_new, int dtype, void* cache_k, void* cache_v,
                            const int* position_ids, const float* inv_freq, int B, int n_src, long long src0, int n,
                            int L, long long dst0, int H, int D, void* stream);

/* The 8-bit KV cache of the generation path (`ShardedKVCache(..., dtype=torch.int8)`; format in
 * lwm_b200/csrc/kv_q8.cuh and DESIGN.md §5). A cache tensor is data int8 [B,L,H,128] (codes) plus exp int8 [B,H,L,4]
 * (one power-of-two exponent per 32-element group, head-major), both 4-byte aligned. A row's value is code * 2^e, exact
 * in fp32 and bf16; code -128 is NaN.
 * lwm_kv_cache_write_q8     rows [src0, src0+n) of k_src / v_src [B,n_src,H,128] (src_dtype 0 = fp32, 1 = bf16)
 *                           quantized into rows [dst0, dst0+n) of the k and v caches [B,L,H,128]. position_ids [B,n_src]
 *                           int32 and inv_freq [64], or both NULL: k is first rotated and rounded to the source dtype,
 *                           bit for bit as lwm_kv_cache_write_rope stores it. One launch for k and v.
 * lwm_kv_dequant_q8         data / exp of [B,L,H,128] rows -> out [B,L,H,128] in out_dtype (0 = fp32, 1 = bf16), exact. */
int lwm_kv_cache_write_q8(const void* k_src, const void* v_src, int src_dtype, signed char* k_data, signed char* k_exp,
                          signed char* v_data, signed char* v_exp, const int* position_ids, const float* inv_freq,
                          int B, int n_src, long long src0, int n, int L, long long dst0, int H, int D, void* stream);
int lwm_kv_dequant_q8(const signed char* data, const signed char* exp, void* out, int out_dtype, int B, int L, int H,
                      int D, void* stream);
/* The operand passes of the tensor-core attention paths (lwm_attn_absmax, lwm_attn_to_f16_scaled,
 * lwm_attn_to_e4m3_scaled) read straight from the cache rows, with no dequantized copy in memory. Both give the bits the
 * plain pass gives on lwm_kv_dequant_q8's output (fp32 or bf16: the values are exact in both). B = 1 with data / exp at
 * batch row b (data + b*L*H*128, exp + b*H*L*4) passes one row of the batch.
 * lwm_kv_q8_absmax          atomicMax of the largest finite |code * 2^e| bit pattern into *out_bits (caller zeroes it;
 *                           the NaN code is skipped). Composes with lwm_attn_scale_from_absmax and
 *                           lwm_attn_e4m3_scale_from_absmax like lwm_attn_absmax.
 * lwm_kv_q8_stage           dst [B,L,H,128] = fp16(value / *scale) (dst_dtype 2, dst 8-byte aligned) or e4m3(value /
 *                           *scale) (dst_dtype 3, 4-byte aligned), the codes of lwm_attn_stage_rope. */
int lwm_kv_q8_absmax(const signed char* data, const signed char* exp, int B, int L, int H, int D, unsigned* out_bits,
                     void* stream);
int lwm_kv_q8_stage(const signed char* data, const signed char* exp, void* dst, int dst_dtype, const float* scale,
                    int B, int L, int H, int D, void* stream);

/* The decode step without host values that change from token to token, so that it can be captured once in a CUDA graph
 * and replayed (`ShardedKVCache` with torch.cuda.graph; INTEGRATION.md "Decode in a CUDA graph").
 * lwm_kv_cache_write_at     the decode write of k_new / v_new [B,1,H,128] (src_dtype 0 = fp32, 1 = bf16) into this
 *                           rank's shard [B,L,H,128] of a max_length-row cache, whose rows are [lo, lo + L), at the
 *                           global slot cursor[0]. cursor is int32 [2]: the slot, then an arrival counter that must be
 *                           zero and is zero again after the call; the call advances the slot by one, on every rank.
 *                           Only the owner of the slot writes. The cache is, like the existing writes store it:
 *                             k_exp, v_exp NULL, no positions: bf16 / fp32 of src_dtype, rows copied bit for bit;
 *                             k_exp, v_exp NULL, positions: as lwm_kv_cache_write_rope;
 *                             k_exp, v_exp given: the 8-bit cache (cache_k / cache_v its codes), as lwm_kv_cache_write_q8.
 *                           position_ids int32 [B] and inv_freq [64], or both NULL; max_position bounds the positions.
 *                           A slot >= max_length, or any position outside [0, max_position), writes nothing and ORs
 *                           LWM_DEVICE_ERR_SLOT / LWM_DEVICE_ERR_POSITION into *err, a sticky int32 the caller reads
 *                           and clears.
 * lwm_rope_check_positions  ORs LWM_DEVICE_ERR_POSITION into *err if any of position_ids [n] is outside
 *                           [0, max_position): the range check of a rotating op's positions without a device->host
 *                           copy. */
#define LWM_DEVICE_ERR_SLOT 1
#define LWM_DEVICE_ERR_POSITION 2
int lwm_kv_cache_write_at(const void* k_new, const void* v_new, int src_dtype, void* cache_k, void* cache_v,
                          signed char* k_exp, signed char* v_exp, const int* position_ids, const float* inv_freq,
                          int max_position, int* cursor, long long lo, int L, int max_length, int B, int H, int D,
                          int* err, void* stream);
int lwm_rope_check_positions(const int* position_ids, long long n, int max_position, int* err, void* stream);

/* The operand passes of the attention op with the rotary embedding folded in (`ringattention(..., freqs_cis,
 * position_ids)`): x [B,S,H,128] fp32 (0) or bf16 (1) holds UN-rotated q or k, position_ids int32 [B,S], inv_freq [64]
 * as for lwm_attn_rope. Every pass works on rope(x) rounded to x's dtype — bit for bit what lwm_attn_rope writes — so
 * each equals lwm_attn_rope followed by the plain pass, without the rotated tensor in memory.
 * lwm_attn_absmax_rope      atomicMax of the finite |rope(x)| bit patterns into *out_bits (caller zeroes it), as lwm_attn_absmax.
 * lwm_attn_stage_rope       dst_dtype 2: dst = fp16(rope(x) / *scale), as lwm_attn_to_f16_scaled; dst_dtype 1: dst =
 *                           bf16(rope(x)), the bf16 operand mode's copy (scale unused, may be null); dst_dtype 3:
 *                           dst = e4m3(rope(x) / *scale), as lwm_attn_to_e4m3_scaled (one byte per element).
 * lwm_reduce_cast_rope_f32  dst [B,S,H,128] = T(rope*(T(sum of n_src <= 16 fp32 arrays, fixed order))), T = fp32 (0) or
 *                           bf16 (1), rope* the conjugate rotation: lwm_reduce_cast_f32 followed by lwm_attn_rope(conj=1)
 *                           in one pass (the gradient w.r.t. the un-rotated q / k). host_srcs: HOST array of device
 *                           pointers; dst may be one of them (in place). */
int lwm_attn_absmax_rope(const void* x, int dtype, const int* position_ids, const float* inv_freq, int B, int S, int H,
                         unsigned* out_bits, void* stream);
int lwm_attn_stage_rope(const void* x, int dtype, void* dst, int dst_dtype, const float* scale, const int* position_ids,
                        const float* inv_freq, int B, int S, int H, void* stream);
int lwm_reduce_cast_rope_f32(const float* const* host_srcs, int n_src, void* dst, int dst_dtype,
                             const int* position_ids, const float* inv_freq, int B, int S, int H, void* stream);

/* Element-wise helpers used by the ring host loop. */
int lwm_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream);
/* dst[i] += src[i] (fp32, n % 4 == 0): folds a dK/dV partial received from a peer into the owner's accumulator. */
int lwm_add_f32(float* dst, const float* src, long long n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Peer-memory ring context — what replaces the reference's `lax.ppermute(k, v)` ring exchange (un-vendored
 * `ringattention` package, entered at lwm/llama.py:539-569; SURVEY.md §8b "Ring-attn C ABI", §8e).
 * On an NVSwitch box the ring is a schedule, not a topology: every rank owns one heap (cudaMalloc + cudaIpc handle)
 * that all peers map; K/V (and Q/dO) blocks are PULLED out of the owner's heap and dK/dV partials / O / dQ chunks are
 * PUT into landing slots of the owner's heap with copy-engine transfers (no SMs, no matching call on the peer), ordered
 * by 32-bit flags living in the heaps: lwm_ring_signal = remote flag write enqueued behind the payload on the same
 * stream, lwm_ring_wait = cuStreamWaitValue32(>=) on the local flag. No host synchronisation on the data path.
 *
 * Bootstrap (host side, once per process group): every rank calls lwm_ring_ctx_create, exchanges the
 * LWM_RING_HANDLE_BYTES-byte handle of lwm_ring_ctx_get_handle with all peers by any means (torch.distributed
 * all_gather here), then lwm_ring_ctx_open_peers(handles of all ranks, rank-major).
 * signal_mode: how the remote flag write is issued — 0 cuStreamWriteValue32 on the peer mapping (default),
 * 1 cuMemsetD32Async, 2 a 4-byte copy-engine transfer (values < 4096); tools/probe_ipc.cu exercises all three.
 * Ownership: the context owns the heap and the mappings; everything else stays caller-owned. Not thread-safe
 * (one host thread per rank). lwm_ring_ctx_heap(ctx, peer) is the address, valid in THIS process, of rank `peer`'s
 * heap payload (the layout inside it is the caller's: lwm_b200/ring_peer.py documents the one the op uses). */
typedef struct lwm_ring_ctx lwm_ring_ctx;
#define LWM_RING_HANDLE_BYTES 64
#define LWM_RING_MAX_WORLD 16
#define LWM_RING_FLAG_BYTES 65536
#define LWM_RING_NUM_FLAGS (LWM_RING_FLAG_BYTES / 4)
int lwm_ring_ctx_create(int rank, int world, long long heap_bytes, int signal_mode, lwm_ring_ctx** ctx);
int lwm_ring_ctx_get_handle(lwm_ring_ctx* ctx, void* handle64);
int lwm_ring_ctx_open_peers(lwm_ring_ctx* ctx, const void* handles /* world * LWM_RING_HANDLE_BYTES */);
void* lwm_ring_ctx_heap(lwm_ring_ctx* ctx, int peer);
long long lwm_ring_ctx_heap_bytes(lwm_ring_ctx* ctx);
int lwm_ring_copy(void* dst, const void* src, long long bytes, void* stream);
int lwm_ring_signal(lwm_ring_ctx* ctx, int peer, int flag, unsigned value, void* stream);
int lwm_ring_wait(lwm_ring_ctx* ctx, int flag, unsigned value, void* stream);
int lwm_ring_ctx_destroy(lwm_ring_ctx* ctx);

/* The schedule and the heap layout of the peer-memory ring as pure functions (host-only; no device is touched), so that
 * a host in any language can drive the lwm_ring_* primitives above. Same results as lwm_b200/ring_schedule.py::
 * make_peer_plan and lwm_b200/ring_peer.py::Layout (tests/test_ring_plan_native_cpu.py compares them field by field).
 * lwm_ring_plan: rank `rank` of `world`, per-rank shard lengths Sq / Sk, causal flag; zigzag = 1 selects the
 *   load-balanced work assignment (rank r computes query half-chunks r and 2P-1-r; needs Sq == Sk, Sq % 256 == 0), 0 the
 *   reference's (every rank its own rows). q[]: query chunks this rank computes (owner = rank whose shard holds the rows);
 *   q_sends[]: rows of MY shard that a peer computes (it pulls them from my stage and puts the results back);
 *   fwd/bwd groups: K/V chunks to have pulled before the group's launches (group g = chunks
 *   [first_chunk[g], first_chunk[g+1]), launches [first_launch[g], first_launch[g+1])); a launch = query chunk q_chunk
 *   against `rows` keys starting at global key row key_row0, all staged by `owner`; incoming[]: dK/dV partials that
 *   will land in my heap, slot = chunk_index * world + peer; own_computed[]: my chunk indices I compute on myself.
 * lwm_ring_layout: byte offsets of the regions inside one set (scales table [world][4] fp32, position-ordered K and V
 *   arrays [B, world*Sk, H, D], Q/dO stage [B,Sq,H,D], 4-byte and 2-byte landing areas for O/dQ rows, dK/dV landing
 *   slots: slot s = lp + (2*s + {0: dK, 1: dV}) * slot_bytes); set 1 starts at set_bytes. */
#define LWM_RING_MAX_CHUNKS 32
#define LWM_RING_MAX_LAUNCHES 128
typedef struct { int owner, index; long long start, length, pos0; } lwm_ring_chunk;
typedef struct { int q_chunk, owner; long long key_row0, rows; } lwm_ring_launch;
typedef struct {
  int world, rank, zigzag, chunks_per_rank;
  int n_q; lwm_ring_chunk q[2];
  int n_q_sends; struct { long long start, length; int peer; } q_sends[LWM_RING_MAX_CHUNKS];
  int n_fwd_groups, n_fwd_chunks, n_fwd_launches;
  int fwd_group_first_chunk[LWM_RING_MAX_CHUNKS + 1], fwd_group_first_launch[LWM_RING_MAX_CHUNKS + 1];
  lwm_ring_chunk fwd_chunks[LWM_RING_MAX_CHUNKS]; lwm_ring_launch fwd_launches[LWM_RING_MAX_LAUNCHES];
  int n_bwd_groups, n_bwd_chunks, n_bwd_launches;
  int bwd_group_first_chunk[LWM_RING_MAX_CHUNKS + 1], bwd_group_first_launch[LWM_RING_MAX_CHUNKS + 1];
  lwm_ring_chunk bwd_chunks[LWM_RING_MAX_CHUNKS]; lwm_ring_launch bwd_launches[LWM_RING_MAX_LAUNCHES];
  int n_incoming; struct { int chunk_index, peer; } incoming[LWM_RING_MAX_CHUNKS];
  int n_own; int own_computed[2];
} lwm_ring_plan_t;
typedef struct {
  long long scales, kg, vg, qs, lq4, lq2, lp, slot_bytes, set_bytes, total, chunk_rows;
  int n_slots;
} lwm_ring_layout_t;
int lwm_ring_plan(int world, int rank, long long Sq, long long Sk, int causal, int zigzag, int fwd_group_chunks,
                  lwm_ring_plan_t* out);
int lwm_ring_layout(int B, long long Sq, long long Sk, int H, int D, int world, int chunks_per_rank, int op_itemsize,
                    lwm_ring_layout_t* out);

/* ---------------------------------------------------------------------------------------------
 * VQGAN tokenizer (lwm/vqgan.py:105-351). Activations are NHWC fp32 (flax layout and dtype).
 *
 * lwm_vq_gn_stats  (sum, sum of squares) per (sample, group) for flax nn.GroupNorm()
 *                  (32 groups; vqgan.py:161,181,251,254); stats [N, groups, 2] float64, zeroed here.
 * lwm_vq_prep      turns an activation into the conv kernel's tensor-core operand planes:
 *                  y = silu(groupnorm(x)) when gn_stats != NULL (ResnetBlock, vqgan.py:251-256), else y = x;
 *                  optional nearest 2x upsampling (Upsample, vqgan.py:312-316);
 *                  hi = bf16(y) and, if lo != NULL, lo = bf16(y - hi); planes are [N,H',W',C_pad].
 * lwm_vq_conv2d    flax nn.Conv as an implicit GEMM on wgmma: ksize 1|3, stride 1 (SAME, pad=ksize/2) or
 *                  the Downsample conv (stride 2, pad 0 on top/left, implicit zero bottom/right,
 *                  vqgan.py:292-300). Weights pre-packed [taps][Cout_pad][C_pad] bf16 (hi / lo).
 *                  n_pass 1 = bf16 operands; 3 = split-bf16 (hi+lo) operands, fp32-class accuracy.
 *                  out = conv + bias (+ residual) (clamped to [-1,1] when clip, vqgan.py:141).
 * lwm_vq_conv_cin3 Encoder conv_in (3 -> Cout, 3x3 SAME, vqgan.py:155) on the CUDA cores; w is HWIO.
 * lwm_vq_argmin    VectorQuantizer (vqgan.py:207-215): idx = argmin_n (sum z^2 + sum e_n^2 - 2 z.e_n) with the
 *                  first index on ties, fp32 with a pinned operation order (bit-exact vs oracle/vqgan_ref.py);
 *                  zq_st (optional) = z + (e[idx] - z). workspace: 8 * N * 8 bytes. Non-finite distances follow
 *                  np.argmin: the first NaN wins and an all-+inf row gives index 0, so idx is always in [0, n_e).
 * lwm_vq_gather    out[i] = codebook[idx[i]] (decode path, vqgan.py:193-195).
 */
int lwm_vq_gn_stats(const float* x, double* stats, int N, int H, int W, int C, int groups, void* stream);
int lwm_vq_prep(const float* x, const double* gn_stats, const float* gamma, const float* beta, void* hi, void* lo,
                int N, int H, int W, int C, int C_pad, int groups, int upsample2x, float eps, void* stream);
int lwm_vq_conv2d(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                  const float* residual, float* out, int N, int Hin, int Win, int Cpad, int Ho, int Wo, int Cout,
                  int Cout_pad, int ksize, int stride, int pad, int n_pass, int clip, void* stream);
int lwm_vq_conv_cin3(const float* x, const float* w_hwio, const float* bias, float* y, int N, int H, int W, int Cout,
                     void* stream);
/* "fp16x2" precision mode of the conv stack (the default: <= 1e-3 vs the fp32 reference at 2x instead of 3x the
 * algorithmic tensor work and half the operand bytes):
 * lwm_vq_prep_f16    like lwm_vq_prep, but ONE fp16 operand plane [N,H',W',C_pad] holding y / s, with a power of two s
 *                    written to the device float *scale_out. Without GroupNorm s = 2^(e-12), e the exponent of the
 *                    largest finite |x|: x_absmax (required then) holds its bit pattern when x_absmax_given (lwm_vq_conv2d_f16's
 *                    absmax_out of the conv that produced x), else it is computed into it; with GroupNorm s brings a bound on
 *                    |y| derived from gn_stats, gamma and beta into [1, 2^13) (s = 1 for ordinary layers). The plane is
 *                    then never inf nor fp16-subnormal because of the activation's magnitude.
 * lwm_vq_conv2d_f16  activation = that plane, a_scale = its scale (device float; NULL = 1, multiplied back in fp32
 *                    in the epilogue); weights split w = hi + lo (two fp16, pre-multiplied by the power of two
 *                    1/w_scale_inv so that lo stays a normal fp16) and STACKED along Cout: w_stacked
 *                    [taps][Cout_pad/BN][2*BN][C_pad], BN = largest multiple of 16 <= 128 dividing Cout_pad, rows [0,BN) = hi, [BN,2BN) = lo. One
 *                    64 x 2BN wgmma per warpgroup yields A.hi | A.lo side by side; the epilogue adds them, applies w_scale_inv, bias,
 *                    residual, clip. gn_stats_out (optional; zeroed by the caller; [N, groups, 2] float64): the epilogue
 *                    also accumulates (sum, sum of squares) of the OUTPUT per (sample, group) — the statistics of the
 *                    GroupNorm that consumes this tensor (vqgan.py:251,254,161,181), so lwm_vq_gn_stats' extra pass
 *                    over the activation disappears. absmax_out (optional; zeroed by the caller): atomicMax of the
 *                    output's finite |value| bit patterns, the x_absmax of an lwm_vq_prep_f16 that reads this tensor. */
int lwm_vq_prep_f16(const float* x, const double* gn_stats, const float* gamma, const float* beta, void* out,
                    float* scale_out, unsigned* x_absmax, int x_absmax_given, int N, int H, int W, int C, int C_pad,
                    int groups, int upsample2x, float eps, void* stream);
int lwm_vq_conv2d_f16(const void* a, const float* a_scale, const void* w_stacked, const float* bias,
                      const float* residual, float* out, double* gn_stats_out, unsigned* absmax_out, int N, int Hin,
                      int Win, int Cpad, int Ho, int Wo, int Cout, int Cout_pad, int ksize, int stride, int pad,
                      float w_scale_inv, int groups, int clip, void* stream);
/* Reproducible, batch-invariant tokenizer (what torch.use_deterministic_algorithms(True) asks for): with these in
 * place of lwm_vq_gn_stats, lwm_vq_prep_f16 and lwm_vq_conv2d_f16, every sample's result is the same bits on every run
 * and whatever else shares its batch. No atomics feed a sum, and no scale spans the batch:
 * lwm_vq_gn_stats_ordered    the statistics of lwm_vq_gn_stats (same [N, groups, 2] float64 layout), from per-block
 *                            partials over fixed 128-pixel ranges of each image, summed in a fixed order in float64.
 *                            workspace: caller-owned, >= N * ceil(H*W/128) * groups * 2 floats (workspace_bytes).
 * lwm_vq_prep_f16_ordered    lwm_vq_prep_f16 with one power-of-two scale per sample: scale_out [N], x_absmax [N]
 *                            (uint32 bit patterns; computed into it per sample unless x_absmax_given), the GroupNorm
 *                            bound taken over the sample's own groups.
 * lwm_vq_conv2d_f16_ordered  lwm_vq_conv2d_f16 reading a_scale [N] (NULL = 1) and writing absmax_out [N] (zeroed by
 *                            the call). gn_stats_out (optional) is written, not accumulated: every (8x16-pixel tile,
 *                            warp) stores its per-group partials to workspace (>= N * Ho/8 * Wo/16 * 8 * groups * 2
 *                            floats), which are summed in a fixed order in float64. It needs Cout/groups == 4, or a
 *                            multiple of 8 that divides the N tile (every LWM layer that has a GroupNorm qualifies). */
int lwm_vq_gn_stats_ordered(const float* x, double* stats, float* workspace, long long workspace_bytes, int N, int H,
                            int W, int C, int groups, void* stream);
int lwm_vq_prep_f16_ordered(const float* x, const double* gn_stats, const float* gamma, const float* beta, void* out,
                            float* scale_out, unsigned* x_absmax, int x_absmax_given, int N, int H, int W, int C,
                            int C_pad, int groups, int upsample2x, float eps, void* stream);
int lwm_vq_conv2d_f16_ordered(const void* a, const float* a_scale, const void* w_stacked, const float* bias,
                              const float* residual, float* out, double* gn_stats_out, float* workspace,
                              long long workspace_bytes, unsigned* absmax_out, int N, int Hin, int Win, int Cpad,
                              int Ho, int Wo, int Cout, int Cout_pad, int ksize, int stride, int pad,
                              float w_scale_inv, int groups, int clip, void* stream);
int lwm_vq_argmin(const float* z, const float* codebook, int* idx, float* zq_st, void* workspace, int N, int n_e,
                  int e_dim, void* stream);
int lwm_vq_gather(const int* idx, const float* codebook, float* out, long long N, int n_e, int e_dim, void* stream);

/* Vision token framing (SURVEY.md §8f next-row 4). lwm_vq_frame_tokens: codes [n_clips, T_in, P] int32 -> tokens
 * [n_clips, T_out, P+1]: every kept frame's P codes followed by eof_token, or eov_token after the clip's last frame
 * (lwm/vision_chat.py:97-104; lwm/data.py:193-212, defaults P=256, eof=8192, eov=8193 at data.py:134-136).
 * frame_idx [T_out] (device, or NULL when T_out == T_in) selects source frames (data.py:196-202 uniform selection).
 * lwm_vq_unframe_tokens: tokens [n_frames, P+1] -> codes [n_frames, P] (lwm/vision_generation.py:160,221). */
int lwm_vq_frame_tokens(const int* codes, const int* frame_idx, int* tokens, int n_clips, int T_in, int T_out,
                        int tokens_per_frame, int eof_token, int eov_token, void* stream);
int lwm_vq_unframe_tokens(const int* tokens, int* codes, long long n_frames, int tokens_per_frame, void* stream);

/* Frame preprocessing in front of the encoder (lwm/vision_chat.py:59-74 `Sampler._process_frame`): PIL's default
 * bicubic resize of uint8 RGB frames, the crop, and x / 127.5 - 1 in fp32 — bit-identical to Pillow's 8-bit path.
 *   frames     [T, H, W, C] uint8, C == 3 (RGB)
 *   x_bounds   [out_w, 2] int32 (first input column, tap count) and x_coeffs [out_w, kx] int32: Pillow's fixed-point
 *              (2^22) coefficients of the horizontal pass W -> out_w; a pass that keeps the size is given as the
 *              identity (one tap of 2^22). y_bounds / y_coeffs [out_h, ky]: the vertical pass H -> out_h.
 *              The host builder is lwm_b200/vision_frames.py::pass_tables.
 *   left, top, crop_w, crop_h   the crop window inside the out_w x out_h resized frame (integer: after PIL's rounding)
 *   out        [T, crop_h, crop_w, 3] fp32 in [-1, 1]
 * Only the crop window is computed. One launch per call. */
int lwm_vq_frames_prep(const unsigned char* frames, int T, int H, int W, int C, const int* x_bounds, const int* x_coeffs,
                       int out_w, int kx, const int* y_bounds, const int* y_coeffs, int out_h, int ky, int left, int top,
                       int crop_w, int crop_h, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LWM_B200_H_ */
