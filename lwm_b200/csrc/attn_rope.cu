// Rotary position embedding of the attention prologue (lwm/llama.py:344-375 `precompute_freqs_cis` /
// `apply_rotary_emb`, applied at llama.py:517-519 right before the ring-attention call) — SURVEY.md §8f next-row 2.
//
// The reference gathers rows of a host-built complex64 table [max_pos, D/2] (512 MB at 1 M positions) by
// position_ids and multiplies in fp32 complex arithmetic. Here the table is never materialised: the angle of
// (position, pair j) is rebuilt exactly as the table builder does — float32(float64(pos) * float64(inv_freq[j])),
// np.outer of an int64 and a float32 vector — and cos/sin of that float32 angle are taken in double precision and
// rounded once, i.e. within 0.5 ulp of the true value (numpy's float32 sin/cos are within 1 ulp of it). One CTA
// serves kPos token positions: 256 threads build the kPos*64 (cos, sin) pairs once in shared memory, then every
// thread rotates 8-element vectors of all heads of Q and K for those positions, so the transcendental cost is
// amortised over H heads and the kernel is a pure HBM stream: each element is read once and written once.
// The [B,S,H*D] projection output and the op's [B,S,H,D] input are the same memory: the head split is free.
#include "capi_internal.h"
#include "kv_write.cuh"
#include "rope_common.cuh"

namespace lwm {

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256, 3) rope_kernel(const TIn* __restrict__ xq, const TIn* __restrict__ xk,
                                                   TOut* __restrict__ oq, TOut* __restrict__ ok,
                                                   const int* __restrict__ position_ids,
                                                   const float* __restrict__ inv_freq, long long n_tok, int Hq,
                                                   int Hk, float sin_sign) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  const long long tok0 = (long long)blockIdx.x * kRopePos;
  rope_fill_table(cs, position_ids, inv_freq, tok0, n_tok, sin_sign);
  __syncthreads();
  const int vq = Hq * (kRopeDim / 8), vk = Hk * (kRopeDim / 8), vt = vq + vk;
  // batches of independent 16/32-byte loads per thread (8 / 4) before the first use: ~100 KB in flight per SM
  constexpr int kBatch = Raw8<TIn>::kBatch;
  const int total = kRopePos * vt;
  for (int base = threadIdx.x; base < total; base += kBatch * blockDim.x) {
    Raw8<TIn> raw[kBatch];
    int off[kBatch];   // element offset from this CTA's first token (q or k tensor)
    int cs_idx[kBatch];
    bool live[kBatch], is_q[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int v = base + u * blockDim.x;
      const int p = v / vt, r = v - p * vt;
      const long long tok = tok0 + p;
      live[u] = v < total && tok < n_tok;
      is_q[u] = r < vq;
      const int rr = is_q[u] ? r : r - vq;
      off[u] = (p * (is_q[u] ? Hq : Hk)) * kRopeDim + rr * 8;
      cs_idx[u] = p * kRopePairs + (rr & 15) * 4;
      if (live[u]) raw[u].load((is_q[u] ? xq + tok0 * Hq * kRopeDim : xk + tok0 * Hk * kRopeDim) + off[u]);
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (!live[u]) continue;
      float x[8], y[8];
      raw[u].unpack(x);
      rope_rotate8(x, y, &cs[0][0], cs_idx[u]);
      store8<TOut>((is_q[u] ? oq + tok0 * Hq * kRopeDim : ok + tok0 * Hk * kRopeDim) + off[u], y);
    }
  }
}

template <typename TIn, typename TOut>
static int launch_rope(const void* xq, const void* xk, void* oq, void* ok, const int* pos, const float* inv_freq,
                       long long n_tok, int Hq, int Hk, int conj, cudaStream_t stream) {
  const long long blocks = (n_tok + kRopePos - 1) / kRopePos;
  rope_kernel<TIn, TOut><<<unsigned(blocks), 256, 0, stream>>>(
      reinterpret_cast<const TIn*>(xq), reinterpret_cast<const TIn*>(xk), reinterpret_cast<TOut*>(oq),
      reinterpret_cast<TOut*>(ok), pos, inv_freq, n_tok, Hq, Hk, conj ? -1.0f : 1.0f);
  return lwm_check_launch("rope_kernel");
}

// KV-cache write of new rows with the rotary embedding on the keys (kv_write.cuh: kv_write_rows), one CTA per kRopePos
// tokens like rope_kernel.
template <typename T>
__global__ void __launch_bounds__(256) kv_write_rope_kernel(const T* __restrict__ k_new, const T* __restrict__ v_new,
                                                            T* __restrict__ cache_k, T* __restrict__ cache_v,
                                                            const int* __restrict__ position_ids,
                                                            const float* __restrict__ inv_freq, int n_src,
                                                            long long src0, int n, int L, long long dst0, int H,
                                                            long long n_tok) {
  kv_write_rows<T, true>(k_new, v_new, cache_k, cache_v, position_ids, inv_freq, n_src, src0, n, L, dst0, H, n_tok,
                         (long long)blockIdx.x * kRopePos);
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_kv_cache_write_rope(const void* k_new, const void* v_new, int dtype, void* cache_k, void* cache_v,
                                       const int* position_ids, const float* inv_freq, int B, int n_src,
                                       long long src0, int n, int L, long long dst0, int H, int D, void* stream) {
  if (D != kRopeDim) return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_rope: head_dim must be 128");
  if (B <= 0 || n <= 0 || H <= 0 || n_src <= 0 || L <= 0)
    return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_rope: bad sizes");
  if (src0 < 0 || src0 + n > n_src || dst0 < 0 || dst0 + n > L)
    return lwm_fail(LWM_ERR_SHAPE, "kv_cache_write_rope: rows out of range");
  if (!k_new || !v_new || !cache_k || !cache_v || !position_ids || !inv_freq)
    return lwm_fail(LWM_ERR_ARG, "kv_cache_write_rope: null pointer");
  if (dtype != 0 && dtype != 1) return lwm_fail(LWM_ERR_ARG, "kv_cache_write_rope: dtype codes are 0 (fp32) or 1 (bf16)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long n_tok = (long long)B * n;
  const unsigned blocks = unsigned((n_tok + kRopePos - 1) / kRopePos);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 0)
    kv_write_rope_kernel<float><<<blocks, 256, 0, st>>>(
        reinterpret_cast<const float*>(k_new), reinterpret_cast<const float*>(v_new), reinterpret_cast<float*>(cache_k),
        reinterpret_cast<float*>(cache_v), position_ids, inv_freq, n_src, src0, n, L, dst0, H, n_tok);
  else
    kv_write_rope_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(k_new), reinterpret_cast<const __nv_bfloat16*>(v_new),
        reinterpret_cast<__nv_bfloat16*>(cache_k), reinterpret_cast<__nv_bfloat16*>(cache_v), position_ids, inv_freq,
        n_src, src0, n, L, dst0, H, n_tok);
  return lwm_check_launch("kv_write_rope_kernel");
}

extern "C" int lwm_attn_rope(const void* xq, const void* xk, int in_dtype, void* out_q, void* out_k, int out_dtype,
                             const int* position_ids, const float* inv_freq, int B, int S, int Hq, int Hk, int D,
                             int conj, void* stream) {
  if (D != kRopeDim) return lwm_fail(LWM_ERR_SHAPE, "attn_rope: head_dim must be 128");
  if (B <= 0 || S <= 0 || Hq <= 0 || Hk < 0) return lwm_fail(LWM_ERR_SHAPE, "attn_rope: bad sizes");
  if (!xq || !out_q || !position_ids || !inv_freq || (Hk > 0 && (!xk || !out_k)))
    return lwm_fail(LWM_ERR_ARG, "attn_rope: null pointer");
  if ((in_dtype != 0 && in_dtype != 1) || (out_dtype != 0 && out_dtype != 1))
    return lwm_fail(LWM_ERR_ARG, "attn_rope: dtype codes are 0 (fp32) or 1 (bf16)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long n_tok = (long long)B * S;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (in_dtype == 0 && out_dtype == 0)
    return launch_rope<float, float>(xq, xk, out_q, out_k, position_ids, inv_freq, n_tok, Hq, Hk, conj, st);
  if (in_dtype == 0 && out_dtype == 1)
    return launch_rope<float, __nv_bfloat16>(xq, xk, out_q, out_k, position_ids, inv_freq, n_tok, Hq, Hk, conj, st);
  if (in_dtype == 1 && out_dtype == 0)
    return launch_rope<__nv_bfloat16, float>(xq, xk, out_q, out_k, position_ids, inv_freq, n_tok, Hq, Hk, conj, st);
  return launch_rope<__nv_bfloat16, __nv_bfloat16>(xq, xk, out_q, out_k, position_ids, inv_freq, n_tok, Hq, Hk, conj, st);
}
