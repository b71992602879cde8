// Decode-time attention (SURVEY.md §8f next-row 1): the reference's `ringattention_inference`
// (bound at lwm/llama.py:601-614; SURVEY.md Appendix A): a few query rows (q_len = 1 while generating)
// against the sequence-sharded KV cache with an explicit boolean mask [B,1,Q,K_global]:
//     s = where(mask, q.k / sqrt(D), finfo.min) ; online softmax ; out = num / den.
// This is a pure HBM stream (every K and V row is read exactly once, 2 x S_loc x H x 256 B), so
// instead of rotating K/V around a ring each rank reduces its own shard to a partial (o, lse) — split
// over the keys across many CTAs so that all SMs pull on HBM — and the P partials are merged
// (log-sum-exp weights) after one tiny all-gather. No tensor cores: the GEMV has 1 FLOP per byte.
//   decode_partial_kernel  grid (splits, H, B*Q): warp = one key at a time per lane-quad layout:
//                          lane l owns dims [4l, 4l+4) of q, k, v rows (one coalesced 256 B row per load)
//                          bf16 or fp32 rows (one uint2 / float4 per lane and row). Below INFER_MIN_Q query
//                          rows only; longer queries go to the tensor-core inference mode of attn_fwd_kernel.
//                          kRope: q is un-rotated and is rotated at its position as it is loaded (lane l's dims are
//                          the whole pairs 2l, 2l+1), rounded to q's dtype first: the value lwm_attn_rope would write.
//                          KV = signed char: the 8-bit cache of kv_q8.cuh (the q8 instances): lane l loads one
//                          32-bit code word per key row (128 B per warp) and the row's exponent word, dequantizes
//                          exactly into fp32 and runs the same arithmetic in the same key order, so its partials are
//                          bit for bit those of the T instance on the dequantized (to T) cache.
//   decode_merge_kernel    merges `n_part` partials per (b, q, h): used for the key splits (of both kernels) and,
//                          after the exchange, for the ranks; writes bf16 or fp32.
#include "attn_common.cuh"
#include "capi_internal.h"
#include "kv_q8.cuh"
#include "rope_common.cuh"

#include <type_traits>

namespace lwm {

constexpr int kDecWarps = 4;

template <typename T, bool kRope = false, typename KV = T>
__global__ void __launch_bounds__(kDecWarps * 32)
decode_partial_kernel(const T* __restrict__ q, const KV* __restrict__ k,
                      const KV* __restrict__ v, const unsigned char* __restrict__ mask,
                      float* __restrict__ o_part, float* __restrict__ ml_part, int B, int H, int Q, int Sk,
                      long long k_pos0, long long mask_stride_b, long long mask_stride_q, int splits,
                      float scale_log2, const int* __restrict__ position_ids = nullptr,
                      const float* __restrict__ inv_freq = nullptr, const unsigned* __restrict__ k_exp = nullptr,
                      const unsigned* __restrict__ v_exp = nullptr) {
  constexpr bool kF32 = std::is_same<T, float>::value;   // fp32 rows: one float4 per lane, bf16 rows: one uint2
  constexpr bool kQ8 = std::is_same<KV, signed char>::value;   // 8-bit rows: one code word per lane
  using Raw = typename std::conditional<kQ8, unsigned, typename std::conditional<kF32, float4, uint2>::type>::type;
  const int split = blockIdx.x, h = blockIdx.y;
  const int b = blockIdx.z / Q, qi = blockIdx.z % Q;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (Sk + splits - 1) / splits;
  const int k_begin = split * per, k_end = min(Sk, k_begin + per);

  float q0, q1, q2, q3;
  if constexpr (kF32) {
    const float4 qf = reinterpret_cast<const float4*>(q + (((size_t)b * Q + qi) * H + h) * kHeadDim)[lane];
    q0 = qf.x; q1 = qf.y; q2 = qf.z; q3 = qf.w;
  } else {
    const uint2 qraw = reinterpret_cast<const uint2*>(q + (((size_t)b * Q + qi) * H + h) * kHeadDim)[lane];
    const __nv_bfloat162 q01 = *reinterpret_cast<const __nv_bfloat162*>(&qraw.x);
    const __nv_bfloat162 q23 = *reinterpret_cast<const __nv_bfloat162*>(&qraw.y);
    q0 = __low2float(q01); q1 = __high2float(q01);
    q2 = __low2float(q23); q3 = __high2float(q23);
  }
  if constexpr (kRope) {
    // pairs (2*lane, 2*lane+1) at this row's position, with rope_rotate8's separately rounded products
    const long long tok = (long long)b * Q + qi;
    const float2 f0 = rope_cos_sin(position_ids, inv_freq, tok, 2 * lane, 1.0f);
    const float2 f1 = rope_cos_sin(position_ids, inv_freq, tok, 2 * lane + 1, 1.0f);
    float y0 = __fsub_rn(__fmul_rn(q0, f0.x), __fmul_rn(q1, f0.y));
    float y1 = __fadd_rn(__fmul_rn(q0, f0.y), __fmul_rn(q1, f0.x));
    float y2 = __fsub_rn(__fmul_rn(q2, f1.x), __fmul_rn(q3, f1.y));
    float y3 = __fadd_rn(__fmul_rn(q2, f1.y), __fmul_rn(q3, f1.x));
    if constexpr (!kF32) {
      y0 = __bfloat162float(__float2bfloat16_rn(y0)); y1 = __bfloat162float(__float2bfloat16_rn(y1));
      y2 = __bfloat162float(__float2bfloat16_rn(y2)); y3 = __bfloat162float(__float2bfloat16_rn(y3));
    }
    q0 = y0; q1 = y1; q2 = y2; q3 = y3;
  }
  q0 *= scale_log2; q1 *= scale_log2; q2 *= scale_log2; q3 *= scale_log2;
  const unsigned char* mrow = mask ? mask + (size_t)b * mask_stride_b + (size_t)qi * mask_stride_q + k_pos0 : nullptr;

  float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const size_t row_stride = (size_t)H * kHeadDim;   // elements between consecutive keys of one head
  const KV* kb = k + ((size_t)b * Sk) * row_stride + (size_t)h * kHeadDim;
  const KV* vb = v + ((size_t)b * Sk) * row_stride + (size_t)h * kHeadDim;
  const size_t exp0 = ((size_t)b * H + h) * Sk;     // the exponent words of this (b, h), one per key
  // each warp strides over the CTA's key range, 4 keys in flight per iteration
  for (int j0 = k_begin + warp * 4; j0 < k_end; j0 += kDecWarps * 4) {
    float s[4];
    Raw vr[4];
    unsigned ve[4];   // kQ8: the exponent words of the value rows
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      float part = 0.f;
      vr[u] = Raw{};
      if (j < k_end) {
        const Raw kr = reinterpret_cast<const Raw*>(kb + (size_t)j * row_stride)[lane];
        vr[u] = reinterpret_cast<const Raw*>(vb + (size_t)j * row_stride)[lane];
        if constexpr (kQ8) {
          ve[u] = v_exp[exp0 + j];
          const float4 kf = q8_dequant4(kr, k_exp[exp0 + j], lane);
          part = q0 * kf.x + q1 * kf.y + q2 * kf.z + q3 * kf.w;
        } else if constexpr (kF32) {
          part = q0 * kr.x + q1 * kr.y + q2 * kr.z + q3 * kr.w;
        } else {
          const __nv_bfloat162 k01 = *reinterpret_cast<const __nv_bfloat162*>(&kr.x);
          const __nv_bfloat162 k23 = *reinterpret_cast<const __nv_bfloat162*>(&kr.y);
          part = q0 * __low2float(k01) + q1 * __high2float(k01) + q2 * __low2float(k23) + q3 * __high2float(k23);
        }
      }
      s[u] = part;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      if (j < k_end) {   // warp-uniform
        float t = s[u];
        if (mrow && !mrow[j]) t = kMaskedLogit;
        const float m_new = fmaxf(m, t);
        const float c = ex2f(m - m_new), p = ex2f(t - m_new);
        float4 vf;
        if constexpr (kQ8) {
          vf = q8_dequant4(vr[u], ve[u], lane);
        } else if constexpr (kF32) {
          vf = vr[u];
        } else {
          const __nv_bfloat162 v01 = *reinterpret_cast<const __nv_bfloat162*>(&vr[u].x);
          const __nv_bfloat162 v23 = *reinterpret_cast<const __nv_bfloat162*>(&vr[u].y);
          vf = make_float4(__low2float(v01), __high2float(v01), __low2float(v23), __high2float(v23));
        }
        l = l * c + p;
        a0 = a0 * c + p * vf.x;
        a1 = a1 * c + p * vf.y;
        a2 = a2 * c + p * vf.z;
        a3 = a3 * c + p * vf.w;
        m = m_new;
      }
    }
  }
  // merge the 4 warps through shared memory
  __shared__ float s_o[kDecWarps][kHeadDim];
  __shared__ float s_m[kDecWarps], s_l[kDecWarps];
  *reinterpret_cast<float4*>(&s_o[warp][lane * 4]) = make_float4(a0, a1, a2, a3);
  if (lane == 0) {
    s_m[warp] = m;
    s_l[warp] = l;
  }
  __syncthreads();
  if (warp == 0) {
    float mm = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float ll = 0.f;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) {
      const float c = (s_m[w] == -INFINITY) ? 0.f : ex2f(s_m[w] - mm);
      const float4 o = *reinterpret_cast<const float4*>(&s_o[w][lane * 4]);
      acc.x += c * o.x; acc.y += c * o.y; acc.z += c * o.z; acc.w += c * o.w;
      ll += c * s_l[w];
    }
    const size_t pidx = (((size_t)(b * Q + qi) * H + h) * splits + split);
    *reinterpret_cast<float4*>(o_part + pidx * kHeadDim + lane * 4) = acc;
    if (lane == 0) {
      ml_part[pidx * 2] = mm;
      ml_part[pidx * 2 + 1] = ll;
    }
  }
}

// partials: o_part [rows][n_part][128] (un-normalised numerators), ml_part [rows][n_part][2] (max in log2 domain,
// denominator). out != null: write out = num/den (bf16, or fp32 when kF32Out) and lse (natural log); else write one
// merged partial. The layout is the one decode_partial_kernel's splits and attn_fwd_kernel's inference mode write.
template <bool kF32Out>
__global__ void decode_merge_kernel(const float* __restrict__ o_part, const float* __restrict__ ml_part, int n_part,
                                    void* __restrict__ out, float* __restrict__ lse,
                                    float* __restrict__ o_merged, float* __restrict__ ml_merged, long long rows) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float mm = -INFINITY;
  for (int p = 0; p < n_part; ++p) mm = fmaxf(mm, ml_part[(row * n_part + p) * 2]);
  float ll = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = 0; p < n_part; ++p) {
    const float mp = ml_part[(row * n_part + p) * 2];
    const float c = (mp == -INFINITY) ? 0.f : ex2f(mp - mm);
    const float4 o = *reinterpret_cast<const float4*>(o_part + (row * n_part + p) * kHeadDim + lane * 4);
    acc.x += c * o.x; acc.y += c * o.y; acc.z += c * o.z; acc.w += c * o.w;
    ll += c * ml_part[(row * n_part + p) * 2 + 1];
  }
  if (out) {
    const float inv = ll > 0.f ? 1.0f / ll : 0.f;
    if constexpr (kF32Out)
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + row * kHeadDim + lane * 4) =
          make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
    else
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + row * kHeadDim + lane * 4) =
          make_uint2(pack_bf16x2(acc.x * inv, acc.y * inv), pack_bf16x2(acc.z * inv, acc.w * inv));
    if (lse && lane == 0) lse[row] = ll > 0.f ? (mm + log2f(ll)) * kLn2 : -INFINITY;
  } else {
    *reinterpret_cast<float4*>(o_merged + row * kHeadDim + lane * 4) = acc;
    if (lane == 0) {
      ml_merged[row * 2] = mm;
      ml_merged[row * 2 + 1] = ll;
    }
  }
}

}  // namespace lwm

using namespace lwm;

// merge n_part partials per row into one partial (o_merged, ml_merged); shared with attn_fwd.cu's inference mode.
void lwm_decode_merge_partials(const float* o_parts, const float* ml_parts, int n_part, float* o_merged,
                               float* ml_merged, long long rows, cudaStream_t st) {
  decode_merge_kernel<false><<<unsigned((rows + 3) / 4), 128, 0, st>>>(o_parts, ml_parts, n_part, nullptr, nullptr,
                                                                       o_merged, ml_merged, rows);
}

template <typename T, bool kRope, typename KV = T>
static int decode_partial_launch(const void* q, const void* k, const void* v, const unsigned char* mask,
                                 float* o_part, float* ml_part, void* workspace, int B, int H, int Q, int Sk, int D,
                                 long long k_pos0, long long mask_stride_b, long long mask_stride_q, int splits,
                                 float softmax_scale, const int* position_ids, const float* inv_freq, void* stream,
                                 const void* k_exp, const void* v_exp) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_decode: head_dim must be 128");
  if (!q || !k || !v || !o_part || !ml_part || !workspace) return lwm_fail(LWM_ERR_ARG, "attn_decode: null pointer");
  if (B <= 0 || H <= 0 || Q <= 0 || Sk <= 0 || splits <= 0 || (long long)B * Q > 65535)
    return lwm_fail(LWM_ERR_SHAPE, "attn_decode: bad shape");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long rows = (long long)B * Q * H;
  float* ws_o = reinterpret_cast<float*>(workspace);
  float* ws_ml = ws_o + rows * splits * kHeadDim;
  dim3 grid(splits, H, B * Q);
  decode_partial_kernel<T, kRope, KV><<<grid, kDecWarps * 32, 0, st>>>(
      reinterpret_cast<const T*>(q), reinterpret_cast<const KV*>(k), reinterpret_cast<const KV*>(v), mask, ws_o, ws_ml,
      B, H, Q, Sk, k_pos0, mask_stride_b, mask_stride_q, splits, softmax_scale * kLog2e, position_ids, inv_freq,
      reinterpret_cast<const unsigned*>(k_exp), reinterpret_cast<const unsigned*>(v_exp));
  lwm_decode_merge_partials(ws_o, ws_ml, splits, o_part, ml_part, rows, st);
  return lwm_check_launch("attn_decode kernels");
}

// q [B,Q,H,128], k,v [B,Sk,H,128] (this rank's KV shard), all fp32 (dtype 0: read directly, one float4 per lane and
// row) or all bf16 (1); or, with k_exp / v_exp, k / v the 8-bit cache (kv_q8.cuh: data int8 [B,Sk,H,128], exp int8
// [B,H,Sk,4]) and dtype q's: the partials then equal, bit for bit, those on the cache dequantized to q's dtype
// (lwm_kv_dequant_q8). mask uint8 [B, ., Q, .] addressed as mask[b*mask_stride_b + q*mask_stride_q + k_pos0 + j]
// (nonzero = attend) or NULL; o_part [B*Q*H, 128] fp32 + ml_part [B*Q*H, 2] fp32 : this rank's partial (numerator,
// (max_log2, denominator)); workspace: splits * B*Q*H * (128 + 2) floats. position_ids int32 [B,Q] and inv_freq [64]
// (as for lwm_attn_rope), or both null: q is un-rotated and is rotated as it is loaded, so the result equals
// lwm_attn_rope (out_dtype = q's) followed by the call without them, bit for bit.
extern "C" int lwm_attn_decode_partial(const void* q, const void* k, const void* v, int dtype, const signed char* k_exp,
                                       const signed char* v_exp, const unsigned char* mask, float* o_part,
                                       float* ml_part, void* workspace, int B, int H, int Q, int Sk, int D,
                                       long long k_pos0, long long mask_stride_b, long long mask_stride_q, int splits,
                                       float softmax_scale, const int* position_ids, const float* inv_freq,
                                       void* stream) {
  if (dtype != 0 && dtype != 1) return lwm_fail(LWM_ERR_ARG, "attn_decode: dtype codes are 0 (fp32) or 1 (bf16)");
  if (!position_ids != !inv_freq) return lwm_fail(LWM_ERR_ARG, "attn_decode: null position_ids / inv_freq");
  if (!k_exp != !v_exp)
    return lwm_fail(LWM_ERR_ARG, "attn_decode: null pointer: k_exp and v_exp are both given (8-bit cache) or both null");
  const bool q8 = k_exp != nullptr;
  if (q8 && ((reinterpret_cast<size_t>(k) | reinterpret_cast<size_t>(v) | reinterpret_cast<size_t>(k_exp) |
              reinterpret_cast<size_t>(v_exp)) & 3) != 0)
    return lwm_fail(LWM_ERR_ARG, "attn_decode: the 8-bit cache's data and exp must be 4-byte aligned");
  return with_flags([&](auto bf16, auto rope, auto cache8) {
    using T = std::conditional_t<bf16, __nv_bfloat16, float>;
    using KV = std::conditional_t<cache8, signed char, T>;
    return decode_partial_launch<T, rope, KV>(q, k, v, mask, o_part, ml_part, workspace, B, H, Q, Sk, D, k_pos0,
                                              mask_stride_b, mask_stride_q, splits, softmax_scale, position_ids,
                                              inv_freq, stream, k_exp, v_exp);
  }, dtype == 1, position_ids != nullptr, q8);
}

// merge n_part partials per row (e.g. the all-gathered per-rank partials) into out, bf16 (out_dtype 1) or the
// un-rounded fp32 (0), and lse.
extern "C" int lwm_attn_decode_merge(const float* o_parts, const float* ml_parts, int n_part, void* out, int out_dtype,
                                     float* lse, long long rows, void* stream) {
  if (!o_parts || !ml_parts || !out || n_part <= 0 || rows <= 0) return lwm_fail(LWM_ERR_ARG, "attn_decode_merge: bad args");
  if (out_dtype != 0 && out_dtype != 1)
    return lwm_fail(LWM_ERR_ARG, "attn_decode_merge: out dtype codes are 0 (fp32) or 1 (bf16)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  auto* kernel = out_dtype == 0 ? decode_merge_kernel<true> : decode_merge_kernel<false>;
  kernel<<<unsigned((rows + 3) / 4), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(o_parts, ml_parts, n_part, out,
                                                                                       lse, nullptr, nullptr, rows);
  return lwm_check_launch("decode_merge_kernel");
}
