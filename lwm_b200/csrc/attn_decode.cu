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
//   decode_merge_kernel    merges `n_part` partials per (b, q, h): used for the key splits and, after the
//                          all-gather, for the ranks.
#include "attn_common.cuh"
#include "capi_internal.h"

namespace lwm {

constexpr int kDecWarps = 4;

__global__ void __launch_bounds__(kDecWarps * 32)
decode_partial_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                      const __nv_bfloat16* __restrict__ v, const unsigned char* __restrict__ mask,
                      float* __restrict__ o_part, float* __restrict__ ml_part, int B, int H, int Q, int Sk,
                      long long k_pos0, long long mask_stride_b, long long mask_stride_q, int splits,
                      float scale_log2) {
  const int split = blockIdx.x, h = blockIdx.y;
  const int b = blockIdx.z / Q, qi = blockIdx.z % Q;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (Sk + splits - 1) / splits;
  const int k_begin = split * per, k_end = min(Sk, k_begin + per);

  const uint2 qraw = reinterpret_cast<const uint2*>(q + (((size_t)b * Q + qi) * H + h) * kHeadDim)[lane];
  const __nv_bfloat162 q01 = *reinterpret_cast<const __nv_bfloat162*>(&qraw.x);
  const __nv_bfloat162 q23 = *reinterpret_cast<const __nv_bfloat162*>(&qraw.y);
  const float q0 = __low2float(q01) * scale_log2, q1 = __high2float(q01) * scale_log2;
  const float q2 = __low2float(q23) * scale_log2, q3 = __high2float(q23) * scale_log2;
  const unsigned char* mrow = mask ? mask + (size_t)b * mask_stride_b + (size_t)qi * mask_stride_q + k_pos0 : nullptr;

  float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const size_t row_stride = (size_t)H * kHeadDim;   // elements between consecutive keys of one head
  const __nv_bfloat16* kb = k + ((size_t)b * Sk) * row_stride + (size_t)h * kHeadDim;
  const __nv_bfloat16* vb = v + ((size_t)b * Sk) * row_stride + (size_t)h * kHeadDim;
  // each warp strides over the CTA's key range, 4 keys in flight per iteration
  for (int j0 = k_begin + warp * 4; j0 < k_end; j0 += kDecWarps * 4) {
    float s[4];
    uint2 vr[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      float part = 0.f;
      vr[u] = make_uint2(0, 0);
      if (j < k_end) {
        const uint2 kr = reinterpret_cast<const uint2*>(kb + (size_t)j * row_stride)[lane];
        vr[u] = reinterpret_cast<const uint2*>(vb + (size_t)j * row_stride)[lane];
        const __nv_bfloat162 k01 = *reinterpret_cast<const __nv_bfloat162*>(&kr.x);
        const __nv_bfloat162 k23 = *reinterpret_cast<const __nv_bfloat162*>(&kr.y);
        part = q0 * __low2float(k01) + q1 * __high2float(k01) + q2 * __low2float(k23) + q3 * __high2float(k23);
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
        const __nv_bfloat162 v01 = *reinterpret_cast<const __nv_bfloat162*>(&vr[u].x);
        const __nv_bfloat162 v23 = *reinterpret_cast<const __nv_bfloat162*>(&vr[u].y);
        l = l * c + p;
        a0 = a0 * c + p * __low2float(v01);
        a1 = a1 * c + p * __high2float(v01);
        a2 = a2 * c + p * __low2float(v23);
        a3 = a3 * c + p * __high2float(v23);
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
// denominator). normalise != 0: write out (bf16) = num/den and lse (natural log); else write one merged partial.
__global__ void decode_merge_kernel(const float* __restrict__ o_part, const float* __restrict__ ml_part, int n_part,
                                    __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
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
    *reinterpret_cast<uint2*>(out + row * kHeadDim + lane * 4) =
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

// q [B,Q,H,128] bf16 ; k,v [B,Sk,H,128] bf16 (this rank's KV shard) ; mask uint8 [B, ., Q, .] addressed as
// mask[b*mask_stride_b + q*mask_stride_q + k_pos0 + j] (nonzero = attend) or NULL ;
// o_part [B*Q*H, 128] fp32 + ml_part [B*Q*H, 2] fp32 : this rank's partial (numerator, (max_log2, denominator));
// workspace: splits * B*Q*H * (128 + 2) floats.
extern "C" int lwm_attn_decode_partial(const void* q, const void* k, const void* v, const unsigned char* mask,
                                       float* o_part, float* ml_part, void* workspace, int B, int H, int Q, int Sk,
                                       int D, long long k_pos0, long long mask_stride_b, long long mask_stride_q,
                                       int splits, float softmax_scale, void* stream) {
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
  decode_partial_kernel<<<grid, kDecWarps * 32, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), reinterpret_cast<const __nv_bfloat16*>(k),
      reinterpret_cast<const __nv_bfloat16*>(v), mask, ws_o, ws_ml, B, H, Q, Sk, k_pos0, mask_stride_b, mask_stride_q,
      splits, softmax_scale * kLog2e);
  decode_merge_kernel<<<unsigned((rows + 3) / 4), 128, 0, st>>>(ws_o, ws_ml, splits, nullptr, nullptr, o_part, ml_part,
                                                                rows);
  return lwm_check_launch("attn_decode kernels");
}

// merge n_part partials per row (e.g. the all-gathered per-rank partials) into out (bf16) and lse.
extern "C" int lwm_attn_decode_merge(const float* o_parts, const float* ml_parts, int n_part, void* out, float* lse,
                                     long long rows, void* stream) {
  if (!o_parts || !ml_parts || !out || n_part <= 0 || rows <= 0) return lwm_fail(LWM_ERR_ARG, "attn_decode_merge: bad args");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  decode_merge_kernel<<<unsigned((rows + 3) / 4), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      o_parts, ml_parts, n_part, reinterpret_cast<__nv_bfloat16*>(out), lse, nullptr, nullptr, rows);
  return lwm_check_launch("decode_merge_kernel");
}
