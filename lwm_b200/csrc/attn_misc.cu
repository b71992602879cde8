// Small HBM-bound helpers around the attention tile kernels:
//   lwm_attn_bwd_prep     delta[b,h,s] = sum_d dout*out  (the rowsum(g∘out) term of the reference's
//                         custom_vjp bwd, SURVEY.md Appendix A `bwd`)
//   lwm_cast_f32_to_bf16  final cast of the fp32 gradient accumulators to the input dtype
//   lwm_attn_*_rope       the operand passes with the rotary embedding of q / k applied on the fly
#include "attn_common.cuh"
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cstdio>
#include <type_traits>
#include "capi_internal.h"
#include "e4m3.cuh"
#include "rope_common.cuh"
#include "../../include/lwm_b200.h"

namespace lwm {

// one warp per (b, s, h) row of 128 elements: 4 bf16 per lane from each tensor (8-byte loads)
__global__ void bwd_prep_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                                float* __restrict__ delta, int B, int H, int S) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // over B*S*H
  const long long n_rows = (long long)B * S * H;
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const uint2 a = reinterpret_cast<const uint2*>(out + row * kHeadDim)[lane];
  const uint2 g = reinterpret_cast<const uint2*>(dout + row * kHeadDim)[lane];
  const __nv_bfloat162 a0 = *reinterpret_cast<const __nv_bfloat162*>(&a.x);
  const __nv_bfloat162 a1 = *reinterpret_cast<const __nv_bfloat162*>(&a.y);
  const __nv_bfloat162 g0 = *reinterpret_cast<const __nv_bfloat162*>(&g.x);
  const __nv_bfloat162 g1 = *reinterpret_cast<const __nv_bfloat162*>(&g.y);
  float acc = __low2float(a0) * __low2float(g0) + __high2float(a0) * __high2float(g0) +
              __low2float(a1) * __low2float(g1) + __high2float(a1) * __high2float(g1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    const int h = int(row % H);
    const long long bs = row / H;
    const int s = int(bs % S);
    const int b = int(bs / S);
    delta[((long long)b * H + h) * S + s] = acc;
  }
}

// same with an fp32 `out` (fp16 precision mode keeps the un-rounded output as residual)
__global__ void bwd_prep_f32_kernel(const float* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                                    float* __restrict__ delta, int B, int H, int S) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long n_rows = (long long)B * S * H;
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float4 a = reinterpret_cast<const float4*>(out + row * kHeadDim)[lane];
  const uint2 g = reinterpret_cast<const uint2*>(dout + row * kHeadDim)[lane];
  const __nv_bfloat162 g0 = *reinterpret_cast<const __nv_bfloat162*>(&g.x);
  const __nv_bfloat162 g1 = *reinterpret_cast<const __nv_bfloat162*>(&g.y);
  float acc = a.x * __low2float(g0) + a.y * __high2float(g0) + a.z * __low2float(g1) + a.w * __high2float(g1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    const int h = int(row % H);
    const long long bs = row / H;
    delta[((long long)(bs / S) * H + h) * S + (bs % S)] = acc;
  }
}

// nlse2 = -lse * log2(e), with rows whose lse sits at the masked level (never saw an unmasked key: padded rows)
// mapped to -inf so that the backward gives them p = 0 — hoisted out of the tile kernel, where every key-tile CTA
// would redo it for every query column.
__global__ void lse_to_nlse2_kernel(const float* __restrict__ lse, float* __restrict__ nlse2, long long n, float offset) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float l = lse[i];
    nlse2[i] = (l < -1.0e29f) ? -INFINITY : fmaf(-l, kLog2e, offset);
  }
}

__global__ void cast_f32_bf16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 f = src[i];
    dst[i] = make_uint2(pack_bf16x2(f.x, f.y), pack_bf16x2(f.z, f.w));
  }
}

__global__ void add_f32_kernel(float4* __restrict__ dst, const float4* __restrict__ src, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 a = dst[i];
    const float4 b = src[i];
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    dst[i] = a;
  }
}

// largest finite |x| over a bf16 tensor as raw fp32 bits (NaN and +-inf are skipped: finite_abs_bits)
__global__ void absmax_bf16_kernel(const uint4* __restrict__ x, long long n8, unsigned* __restrict__ out_bits) {
  unsigned m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      m = max(m, finite_abs_bits(w[k] << 16));           // low bf16, as fp32 bits
      m = max(m, finite_abs_bits(w[k] & 0xffff0000u));   // high bf16
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_bits, m);
}

// x16 = fp16(x / scale) with scale = 2^(e-12), e = exponent of the tensor's largest finite |x| (scale 1 when no
// element is finite and nonzero): that magnitude lands in [2^12, 2^13), so anything down to 2^-26 of it stays a
// normal fp16 and the conversion of every such bf16 value (8 significant bits) is exact. NaN and +-inf stay what
// they are. e is clamped at -114 as in scale_from_absmax_kernel, so that 2^(e-12) and 2^(12-e) are normal floats.
__global__ void bf16_to_scaled_f16_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long n8,
                                          const unsigned* __restrict__ absmax_bits, float* __restrict__ scale_out) {
  const unsigned bits = *absmax_bits;
  const int e = max(int(bits >> 23) - 127, -114);
  const float inv = bits ? __uint_as_float(unsigned(127 - (e - 12)) << 23) : 1.0f;   // 2^(12-e)
  if (blockIdx.x == 0 && threadIdx.x == 0) *scale_out = bits ? __uint_as_float(unsigned(127 + (e - 12)) << 23) : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    unsigned o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float lo = __uint_as_float(w[k] << 16) * inv, hi = __uint_as_float(w[k] & 0xffff0000u) * inv;
      o[k] = pack_f16x2(lo, hi);
    }
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}


// largest finite |x| over an fp32 tensor as raw bits
__global__ void absmax_f32_kernel(const uint4* __restrict__ x, long long n4, unsigned* __restrict__ out_bits) {
  unsigned m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    m = max(max(m, finite_abs_bits(v.x)),
            max(finite_abs_bits(v.y), max(finite_abs_bits(v.z), finite_abs_bits(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_bits, m);
}

// scale = 2^(e-kTop), e = exponent of max_i bits[i*stride] (1.0 for all-zero): one thread. The ring executor feeds it
// the |max| bit patterns of every rank's shard, so that all ranks derive the SAME scale for a sharded tensor.
// kTop = 12: the fp16 operand copies (the maximum lands in [2^12, 2^13)); 7: the e4m3 ones ([2^7, 2^8), below 448).
template <int kTop>
__global__ void scale_from_absmax_kernel(const unsigned* __restrict__ bits, int n, int stride, float* __restrict__ scale_out) {
  unsigned m = 0;
  for (int i = 0; i < n; ++i) m = max(m, bits[(long long)i * stride]);
  const int e = max(int(m >> 23) - 127, -114);   // keeps 2^(e-kTop) and 2^(kTop-e) normal floats
  *scale_out = m ? __uint_as_float(unsigned(127 + (e - kTop)) << 23) : 1.0f;
}

// x16 = fp16(x / *scale) for a power-of-two scale held on the device; source bf16 (exact for every value above
// 2^-26 of the scale's tensor maximum) or fp32 (one rounding to fp16's 11 significant bits).
__global__ void bf16_to_f16_by_scale_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long n8,
                                            const float* __restrict__ scale) {
  const float inv = 1.0f / *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    unsigned o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = pack_f16x2(__uint_as_float(w[k] << 16) * inv, __uint_as_float(w[k] & 0xffff0000u) * inv);
    y[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
__global__ void f32_to_f16_by_scale_kernel(const float4* __restrict__ x, uint2* __restrict__ y, long long n4,
                                           const float* __restrict__ scale) {
  const float inv = 1.0f / *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    y[i] = make_uint2(pack_f16x2(v.x * inv, v.y * inv), pack_f16x2(v.z * inv, v.w * inv));
  }
}

// x8 = e4m3(x / *scale) for a power-of-two scale held on the device (lwm_attn_to_e4m3_scaled), 8 elements per item
__global__ void bf16_to_e4m3_by_scale_kernel(const uint4* __restrict__ x, uint2* __restrict__ y, long long n8,
                                             const float* __restrict__ scale) {
  const float inv = 1.0f / *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = x[i];
    y[i] = make_uint2(pack_e4m3x4(__uint_as_float(v.x << 16) * inv, __uint_as_float(v.x & 0xffff0000u) * inv,
                                  __uint_as_float(v.y << 16) * inv, __uint_as_float(v.y & 0xffff0000u) * inv),
                      pack_e4m3x4(__uint_as_float(v.z << 16) * inv, __uint_as_float(v.z & 0xffff0000u) * inv,
                                  __uint_as_float(v.w << 16) * inv, __uint_as_float(v.w & 0xffff0000u) * inv));
  }
}
__global__ void f32_to_e4m3_by_scale_kernel(const float4* __restrict__ x, uint2* __restrict__ y, long long n8,
                                            const float* __restrict__ scale) {
  const float inv = 1.0f / *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 a = x[2 * i], b = x[2 * i + 1];
    y[i] = make_uint2(pack_e4m3x4(a.x * inv, a.y * inv, a.z * inv, a.w * inv),
                      pack_e4m3x4(b.x * inv, b.y * inv, b.z * inv, b.w * inv));
  }
}

// delta = rowsum(out o dout) with dout given as the scaled fp16 operand copy (dout = dout16 * *scale_do) and out in
// fp32 (kOutF32) or bf16: the ring executor only ever holds the fp16 copy of a remote dO chunk.
template <bool kOutF32>
__global__ void bwd_prep_f16_kernel(const void* __restrict__ out, const __half* __restrict__ dout16,
                                    const float* __restrict__ scale_do, float* __restrict__ delta, int B, int H, int S) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long n_rows = (long long)B * S * H;
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  float a[4];
  if (kOutF32) {
    const float4 t = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(out) + row * kHeadDim)[lane];
    a[0] = t.x; a[1] = t.y; a[2] = t.z; a[3] = t.w;
  } else {
    const uint2 t = reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(out) + row * kHeadDim)[lane];
    a[0] = __uint_as_float(t.x << 16); a[1] = __uint_as_float(t.x & 0xffff0000u);
    a[2] = __uint_as_float(t.y << 16); a[3] = __uint_as_float(t.y & 0xffff0000u);
  }
  const uint2 g = reinterpret_cast<const uint2*>(dout16 + row * kHeadDim)[lane];
  const __half2 g0 = *reinterpret_cast<const __half2*>(&g.x);
  const __half2 g1 = *reinterpret_cast<const __half2*>(&g.y);
  float acc = a[0] * __low2float(g0) + a[1] * __high2float(g0) + a[2] * __low2float(g1) + a[3] * __high2float(g1);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    const int h = int(row % H);
    const long long bs = row / H;
    delta[((long long)(bs / S) * H + h) * S + (bs % S)] = acc * (*scale_do);
  }
}

// dst = cast(sum_i srcs[i]) : folds the dK/dV partials that landed in the owner's heap (plus the owner's own partial)
// and produces the gradient in its final dtype in ONE pass (fp32 sum in a fixed order -> run-to-run deterministic).
struct ReduceSrcs { const float4* p[LWM_REDUCE_MAX_SRCS]; };
template <bool kToBf16>
__global__ void reduce_cast_kernel(const ReduceSrcs srcs, int n_src, void* __restrict__ dst, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 a = srcs.p[0][i];
    for (int s = 1; s < n_src; ++s) {
      const float4 b = srcs.p[s][i];
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    if (kToBf16) reinterpret_cast<uint2*>(dst)[i] = make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w));
    else reinterpret_cast<float4*>(dst)[i] = a;
  }
}


// ---- the same passes over q / k with the rotary embedding applied on the fly (rope_common.cuh) ----
// x [n_tok, H, 128] with one position per token: the value every pass below works on is rope(x) rounded to x's
// dtype, bit for bit what lwm_attn_rope(x -> x's dtype) writes, so each pass equals "rotate, then the plain pass".
// A CTA of 256 threads walks token groups of kRopePos (grid stride); per group it builds the (cos, sin) table once,
// under the group's first loads, and then streams the group's H*16 vectors of 8 elements.

// One token group of the rotating passes: the group's first batch of loads is issued, then the (cos, sin) table of its
// kRopePos tokens is built (its double-precision sincos runs under those loads), and then f(element offset, y[8]) is
// called for every 8-element vector of the group, y = rope(x) rounded to TIn. Every thread of the CTA calls it.
template <typename TIn, typename F>
__device__ __forceinline__ void rope_group_apply(const TIn* __restrict__ x, const int* __restrict__ pos,
                                                 const float* __restrict__ inv_freq, long long tok0, long long n_tok,
                                                 int H, float2 (*cs)[kRopePairs], F&& f) {
  const int vt = H * (kRopeDim / 8);
  const long long left = n_tok - tok0;
  const int total = (left < kRopePos ? int(left) : kRopePos) * vt;
  const long long e0 = tok0 * H * kRopeDim;
  constexpr int kBatch = Raw8<TIn>::kBatch;
  Raw8<TIn> raw[kBatch];
  auto load = [&](int base) {
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int v = base + u * blockDim.x;
      if (v < total) raw[u].load(x + e0 + (long long)v * 8);
    }
  };
  auto use = [&](int base) {
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int v = base + u * blockDim.x;
      if (v >= total) continue;
      const int p = v / vt, r = v - p * vt;
      float xv[8], y[8];
      raw[u].unpack(xv);
      rope_rotate8(xv, y, &cs[0][0], p * kRopePairs + (r & 15) * 4);
      round8<TIn>(y);
      f(e0 + (long long)v * 8, y);
    }
  };
  load(threadIdx.x);
  __syncthreads();                      // the previous group's table is no longer read
  rope_fill_table(cs, pos, inv_freq, tok0, n_tok, 1.0f);
  __syncthreads();
  use(threadIdx.x);
  for (int base = threadIdx.x + kBatch * blockDim.x; base < total; base += kBatch * blockDim.x) {
    load(base);
    use(base);
  }
}

// absmax_*_kernel of rope(x): atomicMax of the finite |value| bit patterns into *out_bits
template <typename TIn>
__global__ void __launch_bounds__(256) absmax_rope_kernel(const TIn* __restrict__ x, const int* __restrict__ pos,
                                                          const float* __restrict__ inv_freq, long long n_tok, int H,
                                                          unsigned* __restrict__ out_bits) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  unsigned m = 0;
  for (long long tok0 = (long long)blockIdx.x * kRopePos; tok0 < n_tok; tok0 += (long long)gridDim.x * kRopePos) {
    rope_group_apply<TIn>(x, pos, inv_freq, tok0, n_tok, H, cs, [&](long long, const float (&y)[8]) {
#pragma unroll
      for (int i = 0; i < 8; ++i) m = max(m, finite_abs_bits(__float_as_uint(y[i])));
    });
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_bits, m);
}

// *_to_f16_by_scale_kernel of rope(x) (kDst 2: fp16(value / *scale)), the bf16 operand mode's copy (kDst 1:
// bf16(value)), or *_to_e4m3_by_scale_kernel of rope(x) (kDst 3: e4m3(value / *scale))
template <typename TIn, int kDst>
__global__ void __launch_bounds__(256) stage_rope_kernel(const TIn* __restrict__ x, void* __restrict__ dst,
                                                         const float* __restrict__ scale, const int* __restrict__ pos,
                                                         const float* __restrict__ inv_freq, long long n_tok, int H) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  const float inv = kDst != 1 ? 1.0f / *scale : 1.0f;
  for (long long tok0 = (long long)blockIdx.x * kRopePos; tok0 < n_tok; tok0 += (long long)gridDim.x * kRopePos) {
    rope_group_apply<TIn>(x, pos, inv_freq, tok0, n_tok, H, cs, [&](long long e, const float (&y)[8]) {
      if constexpr (kDst == 3) {
        reinterpret_cast<uint2*>(dst)[e / 8] = make_uint2(pack_e4m3x4(y[0] * inv, y[1] * inv, y[2] * inv, y[3] * inv),
                                                          pack_e4m3x4(y[4] * inv, y[5] * inv, y[6] * inv, y[7] * inv));
      } else {
        unsigned o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          o[k] = kDst == 2 ? pack_f16x2(y[2 * k] * inv, y[2 * k + 1] * inv) : pack_bf16x2(y[2 * k], y[2 * k + 1]);
        reinterpret_cast<uint4*>(dst)[e / 8] = make_uint4(o[0], o[1], o[2], o[3]);
      }
    });
  }
}

// reduce_cast_kernel followed by the conjugate rotation of the cast value, rounded again to the destination dtype:
// dst = T(rope*(T(sum_i srcs[i]))) with T = bf16 (kToBf16) or fp32, the sum in source order. dst may be a source
// (in place: every element is read by the thread that writes it, before it writes it), hence no __restrict__ on it.
template <bool kToBf16>
__global__ void __launch_bounds__(256) reduce_cast_rope_kernel(const ReduceSrcs srcs, int n_src, void* dst,
                                                               const int* __restrict__ pos,
                                                               const float* __restrict__ inv_freq, long long n_tok,
                                                               int H) {
  __shared__ float2 cs[kRopePos][kRopePairs];
  const int vt = H * (kRopeDim / 8);
  for (long long tok0 = (long long)blockIdx.x * kRopePos; tok0 < n_tok; tok0 += (long long)gridDim.x * kRopePos) {
    __syncthreads();
    rope_fill_table(cs, pos, inv_freq, tok0, n_tok, -1.0f);
    __syncthreads();
    const long long left = n_tok - tok0;
    const int total = (left < kRopePos ? int(left) : kRopePos) * vt;
    const long long q0 = tok0 * H * (kRopeDim / 4);     // in float4
    for (int v = threadIdx.x; v < total; v += blockDim.x) {
      const long long i = q0 + 2LL * v;
      float4 a = srcs.p[0][i], c = srcs.p[0][i + 1];
      for (int s = 1; s < n_src; ++s) {
        const float4 b = srcs.p[s][i], d = srcs.p[s][i + 1];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        c.x += d.x; c.y += d.y; c.z += d.z; c.w += d.w;
      }
      float xv[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w}, y[8];
      const int p = v / vt, r = v - p * vt;
      if (kToBf16) {
        round8<__nv_bfloat16>(xv);
        rope_rotate8(xv, y, &cs[0][0], p * kRopePairs + (r & 15) * 4);
        store8<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(dst) + 4 * i, y);
      } else {
        rope_rotate8(xv, y, &cs[0][0], p * kRopePairs + (r & 15) * 4);
        store8<float>(reinterpret_cast<float*>(dst) + 4 * i, y);
      }
    }
  }
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_attn_bwd_lse(const float* lse, float* nlse2, long long n, float offset_log2, void* stream) {
  if (!lse || !nlse2 || n <= 0) return lwm_fail(LWM_ERR_ARG, "attn_bwd_lse: bad args");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long want = (n + 255) / 256;
  lse_to_nlse2_kernel<<<unsigned(want < kNumSMs * 8 ? want : kNumSMs * 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      lse, nlse2, n, offset_log2);
  return lwm_check_launch("lse_to_nlse2_kernel");
}

extern "C" int lwm_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream) {
  if (n % 4) return lwm_fail(LWM_ERR_SHAPE, "cast_f32_to_bf16: n must be a multiple of 4");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (n == 0) return LWM_OK;
  const long long n4 = n / 4;
  const int threads = 256;
  const long long want = (n4 + threads - 1) / threads;
  const unsigned blocks = unsigned(want < kNumSMs * 16 ? want : kNumSMs * 16);
  cast_f32_bf16_kernel<<<blocks, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(src), reinterpret_cast<uint2*>(dst), n4);
  return lwm_check_launch("cast_f32_bf16_kernel");
}

extern "C" int lwm_add_f32(float* dst, const float* src, long long n, void* stream) {
  if (n % 4) return lwm_fail(LWM_ERR_SHAPE, "add_f32: n must be a multiple of 4");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (n == 0) return LWM_OK;
  const long long n4 = n / 4;
  const int threads = 256;
  const long long want = (n4 + threads - 1) / threads;
  const unsigned blocks = unsigned(want < kNumSMs * 16 ? want : kNumSMs * 16);
  add_f32_kernel<<<blocks, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float4*>(dst), reinterpret_cast<const float4*>(src), n4);
  return lwm_check_launch("add_f32_kernel");
}

// bf16 tensor -> exact scaled fp16 copy + its power-of-two scale (device float). workspace: 4 bytes.
extern "C" int lwm_attn_to_f16(const void* src_bf16, void* dst_f16, float* scale_out, void* workspace, long long n,
                               void* stream) {
  if (!src_bf16 || !dst_f16 || !scale_out || !workspace) return lwm_fail(LWM_ERR_ARG, "attn_to_f16: null pointer");
  if (n <= 0 || n % 8) return lwm_fail(LWM_ERR_SHAPE, "attn_to_f16: n must be a positive multiple of 8");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(workspace, 0, 4, st) != cudaSuccess) return lwm_fail(LWM_ERR_CUDA, "attn_to_f16: memset failed");
  const long long n8 = n / 8;
  const long long want = (n8 + 255) / 256;
  const unsigned blocks = unsigned(want < kNumSMs * 8 ? want : kNumSMs * 8);
  absmax_bf16_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(src_bf16), n8,
                                             reinterpret_cast<unsigned*>(workspace));
  bf16_to_scaled_f16_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(src_bf16),
                                                    reinterpret_cast<uint4*>(dst_f16), n8,
                                                    reinterpret_cast<const unsigned*>(workspace), scale_out);
  return lwm_check_launch("attn_to_f16 kernels");
}


static unsigned grid_for(long long items, int threads, int waves) {
  const long long want = (items + threads - 1) / threads;
  return unsigned(want < kNumSMs * waves ? (want > 0 ? want : 1) : kNumSMs * waves);
}

// atomicMax of the |x| bit patterns into *out_bits (the caller zeroes it); dtype 0 = fp32, 1 = bf16.
extern "C" int lwm_attn_absmax(const void* x, int dtype, long long n, unsigned* out_bits, void* stream) {
  if (!x || !out_bits || n <= 0 || n % 8 || (dtype != 0 && dtype != 1)) return lwm_fail(LWM_ERR_ARG, "attn_absmax: bad arguments (n % 8 == 0)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 1) absmax_bf16_kernel<<<grid_for(n / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 8, out_bits);
  else absmax_f32_kernel<<<grid_for(n / 4, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 4, out_bits);
  return lwm_check_launch("absmax kernel");
}

// |x|max -> power-of-two scale in one call: workspace (4 bytes) is zeroed, filled by the absmax kernel, and turned into
// *scale_out = 2^(e-12). What the ring executor runs per shard before staging (every operand carries its owner's scale).
extern "C" int lwm_attn_absmax_scale(const void* x, int dtype, long long n, unsigned* workspace, float* scale_out, void* stream) {
  if (!x || !workspace || !scale_out || n <= 0 || n % 8 || (dtype != 0 && dtype != 1))
    return lwm_fail(LWM_ERR_ARG, "attn_absmax_scale: bad arguments (n % 8 == 0)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(workspace, 0, 4, st) != cudaSuccess) return lwm_fail(LWM_ERR_CUDA, "attn_absmax_scale: memset failed");
  if (dtype == 1) absmax_bf16_kernel<<<grid_for(n / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 8, workspace);
  else absmax_f32_kernel<<<grid_for(n / 4, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), n / 4, workspace);
  scale_from_absmax_kernel<12><<<1, 1, 0, st>>>(workspace, 1, 1, scale_out);
  return lwm_check_launch("absmax_scale kernels");
}

extern "C" int lwm_attn_scale_from_absmax(const unsigned* bits, int n, int stride, float* scale_out, void* stream) {
  if (!bits || !scale_out || n <= 0 || stride <= 0) return lwm_fail(LWM_ERR_ARG, "attn_scale_from_absmax: bad arguments");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  scale_from_absmax_kernel<12><<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(bits, n, stride, scale_out);
  return lwm_check_launch("scale_from_absmax_kernel");
}

extern "C" int lwm_attn_to_f16_scaled(const void* x, int dtype, void* dst_f16, const float* scale, long long n, void* stream) {
  if (!x || !dst_f16 || !scale || n <= 0 || n % 8 || (dtype != 0 && dtype != 1)) return lwm_fail(LWM_ERR_ARG, "attn_to_f16_scaled: bad arguments (n % 8 == 0)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 1)
    bf16_to_f16_by_scale_kernel<<<grid_for(n / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(dst_f16), n / 8, scale);
  else
    f32_to_f16_by_scale_kernel<<<grid_for(n / 4, 256, 8), 256, 0, st>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(dst_f16), n / 4, scale);
  return lwm_check_launch("to_f16_by_scale kernel");
}

extern "C" int lwm_attn_e4m3_scale_from_absmax(const unsigned* bits, int n, int stride, float* scale_out, void* stream) {
  if (!bits || !scale_out || n <= 0 || stride <= 0) return lwm_fail(LWM_ERR_ARG, "attn_e4m3_scale_from_absmax: bad arguments");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  scale_from_absmax_kernel<7><<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(bits, n, stride, scale_out);
  return lwm_check_launch("scale_from_absmax_kernel");
}

extern "C" int lwm_attn_to_e4m3_scaled(const void* x, int dtype, void* dst_e4m3, const float* scale, long long n,
                                       void* stream) {
  if (!x || !dst_e4m3 || !scale || n <= 0 || n % 8 || (dtype != 0 && dtype != 1))
    return lwm_fail(LWM_ERR_ARG, "attn_to_e4m3_scaled: bad arguments (n % 8 == 0)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint2* y = reinterpret_cast<uint2*>(dst_e4m3);
  if (dtype == 1)
    bf16_to_e4m3_by_scale_kernel<<<grid_for(n / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), y, n / 8, scale);
  else
    f32_to_e4m3_by_scale_kernel<<<grid_for(n / 8, 256, 8), 256, 0, st>>>(reinterpret_cast<const float4*>(x), y, n / 8, scale);
  return lwm_check_launch("to_e4m3_by_scale kernel");
}

// delta = rowsum(out o dout); out fp32 (out_dtype 0) or bf16 (1); dout bf16, or its scaled fp16 copy when scale_do is
// given (the ring executor only ever holds the fp16 copy of a remote dO chunk).
extern "C" int lwm_attn_bwd_prep(const void* out, int out_dtype, const void* dout, const float* scale_do, float* delta,
                                 int B, int H, int Sq, int D, void* stream) {
  if (D != kHeadDim) return lwm_fail(LWM_ERR_SHAPE, "attn_bwd_prep: head_dim must be 128");
  if (!out || !dout || !delta) return lwm_fail(LWM_ERR_ARG, "attn_bwd_prep: null pointer");
  if (out_dtype != 0 && out_dtype != 1) return lwm_fail(LWM_ERR_ARG, "attn_bwd_prep: out dtype codes are 0 (fp32) or 1 (bf16)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long rows = (long long)B * Sq * H;
  const int warps = 8;
  const unsigned blocks = unsigned((rows + warps - 1) / warps);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const __nv_bfloat16* dout_bf16 = reinterpret_cast<const __nv_bfloat16*>(dout);
  const __half* dout16 = reinterpret_cast<const __half*>(dout);
  if (scale_do && out_dtype == 0) bwd_prep_f16_kernel<true><<<blocks, warps * 32, 0, st>>>(out, dout16, scale_do, delta, B, H, Sq);
  else if (scale_do) bwd_prep_f16_kernel<false><<<blocks, warps * 32, 0, st>>>(out, dout16, scale_do, delta, B, H, Sq);
  else if (out_dtype == 0) bwd_prep_f32_kernel<<<blocks, warps * 32, 0, st>>>(reinterpret_cast<const float*>(out), dout_bf16, delta, B, H, Sq);
  else bwd_prep_kernel<<<blocks, warps * 32, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(out), dout_bf16, delta, B, H, Sq);
  return lwm_check_launch("bwd_prep kernel");
}

// host_srcs: HOST array of n_src device pointers (fp32, n elements each); dst_dtype 0 = fp32, 1 = bf16.
extern "C" int lwm_reduce_cast_f32(const float* const* host_srcs, int n_src, void* dst, int dst_dtype, long long n, void* stream) {
  if (!host_srcs || !dst || n_src < 1 || n_src > LWM_REDUCE_MAX_SRCS || n <= 0 || n % 4 || (dst_dtype != 0 && dst_dtype != 1))
    return lwm_fail(LWM_ERR_ARG, "reduce_cast_f32: bad arguments (1..16 sources, n % 4 == 0)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  ReduceSrcs rs;
  for (int i = 0; i < LWM_REDUCE_MAX_SRCS; ++i) rs.p[i] = reinterpret_cast<const float4*>(host_srcs[i < n_src ? i : 0]);
  for (int i = 0; i < n_src; ++i)
    if (!host_srcs[i]) return lwm_fail(LWM_ERR_ARG, "reduce_cast_f32: null source");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dst_dtype == 1) reduce_cast_kernel<true><<<grid_for(n / 4, 256, 16), 256, 0, st>>>(rs, n_src, dst, n / 4);
  else reduce_cast_kernel<false><<<grid_for(n / 4, 256, 16), 256, 0, st>>>(rs, n_src, dst, n / 4);
  return lwm_check_launch("reduce_cast_kernel");
}

// ---- entry points of the rotating passes: x [B,S,H,128] (dtype 0 fp32, 1 bf16), position_ids int32 [B,S], inv_freq [64]

// LWM_ERR_ARG with the message "<fn>: <reason>"
static int rope_fail(const char* fn, const char* reason) {
  char msg[128];
  snprintf(msg, sizeof(msg), "%s: %s", fn, reason);
  return lwm_fail(LWM_ERR_ARG, msg);
}

// LWM_OK, or the failure status of the rotation arguments every rotating pass takes: positions, inv_freq, B, S, H
static int rope_table_args(const char* fn, const int* pos, const float* inv_freq, int B, int S, int H) {
  if (!pos || !inv_freq) return rope_fail(fn, "null pointer");
  if (B <= 0 || S <= 0 || H <= 0) return rope_fail(fn, "bad sizes");
  return LWM_OK;
}

// LWM_OK, or the failure status of an input x [B,S,H,128] of dtype code 0 (fp32) or 1 (bf16) and its rotation
static int rope_input_args(const char* fn, const void* x, int dtype, const int* pos, const float* inv_freq, int B, int S,
                           int H) {
  if (!x) return rope_fail(fn, "null pointer");
  if (dtype != 0 && dtype != 1) return rope_fail(fn, "dtype codes are 0 (fp32) or 1 (bf16)");
  return rope_table_args(fn, pos, inv_freq, B, S, H);
}

static unsigned rope_grid(long long n_tok) { return grid_for((n_tok + kRopePos - 1) / kRopePos, 1, 8); }

extern "C" int lwm_attn_absmax_rope(const void* x, int dtype, const int* position_ids, const float* inv_freq, int B,
                                    int S, int H, unsigned* out_bits, void* stream) {
  if (int e = rope_input_args("attn_absmax_rope", x, dtype, position_ids, inv_freq, B, S, H)) return e;
  if (!out_bits) return lwm_fail(LWM_ERR_ARG, "attn_absmax_rope: null pointer");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long n_tok = (long long)B * S;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 1)
    absmax_rope_kernel<__nv_bfloat16><<<rope_grid(n_tok), 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(x), position_ids, inv_freq, n_tok, H, out_bits);
  else
    absmax_rope_kernel<float><<<rope_grid(n_tok), 256, 0, st>>>(reinterpret_cast<const float*>(x), position_ids,
                                                                inv_freq, n_tok, H, out_bits);
  return lwm_check_launch("absmax_rope_kernel");
}

extern "C" int lwm_attn_stage_rope(const void* x, int dtype, void* dst, int dst_dtype, const float* scale,
                                   const int* position_ids, const float* inv_freq, int B, int S, int H, void* stream) {
  if (int e = rope_input_args("attn_stage_rope", x, dtype, position_ids, inv_freq, B, S, H)) return e;
  if (!dst) return lwm_fail(LWM_ERR_ARG, "attn_stage_rope: null pointer");
  if (dst_dtype != 1 && dst_dtype != 2 && dst_dtype != 3)
    return lwm_fail(LWM_ERR_ARG, "attn_stage_rope: dst dtype codes are 1 (bf16), 2 (scaled fp16) or 3 (scaled e4m3)");
  if (dst_dtype != 1 && !scale) return lwm_fail(LWM_ERR_ARG, "attn_stage_rope: scaled fp16 / e4m3 needs a scale");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const long long n_tok = (long long)B * S;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned g = rope_grid(n_tok);
  auto launch = [&](auto src, auto mode) {
    using TIn = std::remove_const_t<std::remove_pointer_t<decltype(src)>>;
    stage_rope_kernel<TIn, decltype(mode)::value><<<g, 256, 0, st>>>(src, dst, scale, position_ids, inv_freq, n_tok, H);
  };
  auto by_dst = [&](auto src) {
    if (dst_dtype == 3) launch(src, std::integral_constant<int, 3>{});
    else if (dst_dtype == 2) launch(src, std::integral_constant<int, 2>{});
    else launch(src, std::integral_constant<int, 1>{});
  };
  if (dtype == 1) by_dst(reinterpret_cast<const __nv_bfloat16*>(x));
  else by_dst(reinterpret_cast<const float*>(x));
  return lwm_check_launch("stage_rope_kernel");
}

extern "C" int lwm_reduce_cast_rope_f32(const float* const* host_srcs, int n_src, void* dst, int dst_dtype,
                                        const int* position_ids, const float* inv_freq, int B, int S, int H,
                                        void* stream) {
  if (!host_srcs || !dst || n_src < 1 || n_src > LWM_REDUCE_MAX_SRCS || (dst_dtype != 0 && dst_dtype != 1))
    return lwm_fail(LWM_ERR_ARG, "reduce_cast_rope_f32: bad arguments (1..16 sources, dst dtype 0 or 1)");
  if (int e = rope_table_args("reduce_cast_rope_f32", position_ids, inv_freq, B, S, H)) return e;
  for (int i = 0; i < n_src; ++i)
    if (!host_srcs[i]) return lwm_fail(LWM_ERR_ARG, "reduce_cast_rope_f32: null source");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  ReduceSrcs rs;
  for (int i = 0; i < LWM_REDUCE_MAX_SRCS; ++i) rs.p[i] = reinterpret_cast<const float4*>(host_srcs[i < n_src ? i : 0]);
  const long long n_tok = (long long)B * S;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dst_dtype == 1)
    reduce_cast_rope_kernel<true><<<rope_grid(n_tok), 256, 0, st>>>(rs, n_src, dst, position_ids, inv_freq, n_tok, H);
  else
    reduce_cast_rope_kernel<false><<<rope_grid(n_tok), 256, 0, st>>>(rs, n_src, dst, position_ids, inv_freq, n_tok, H);
  return lwm_check_launch("reduce_cast_rope_kernel");
}
