// HBM-bound pieces of the VQGAN tokenizer (lwm/vqgan.py), NHWC fp32 activations:
//   lwm_vq_gn_stats   per-(sample, group) sum and sum of squares for flax nn.GroupNorm() (32 groups,
//                     statistics over H,W,C/32 — vqgan.py:161,181,251,254); lwm_vq_gn_stats_ordered sums them in an
//                     order fixed by (H, W, C) alone (torch.use_deterministic_algorithms)
//   lwm_vq_prep       GroupNorm-apply + SiLU (vqgan.py:251-256) and/or nearest 2x upsampling
//                     (vqgan.py:312-316) fused with the conversion of the activation into the
//                     tensor-core operand planes (bf16 hi, bf16 lo = x - hi) the conv kernel reads by TMA
//   lwm_vq_conv_cin3  direct 3x3 SAME conv for the 3-channel input layer (Encoder conv_in,
//                     vqgan.py:155): 27 MACs per output, far too thin for the tensor pipe
//   lwm_vq_argmin     VectorQuantizer nearest-code search (vqgan.py:207-215), bit-exact fp32 order
//   lwm_vq_gather     codebook lookup for decode (vqgan.py:193-195)
#include "ptx.cuh"
#include "capi_internal.h"

namespace lwm {

// |x| max of an fp32 tensor as raw bits, atomicMax into *out_bits (attn_misc.cu)
__global__ void absmax_f32_kernel(const uint4* __restrict__ x, long long n4, unsigned* __restrict__ out_bits);

// ------------------------------------------------------------------------------------------------
// GroupNorm statistics: stats[n][g] = (sum, sumsq) in double (atomics; zeroed by the caller).
// Thread t owns channel quad (t % (C/4)) and strides over pixels, so a warp reads whole 128 B lines.
// ------------------------------------------------------------------------------------------------
__global__ void gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C,
                                int groups, int pix_per_block) {
  extern __shared__ float s_part[];  // [groups][2]
  const int n = blockIdx.y;
  const int quads = C / 4;
  const int cpg = C / groups;
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) s_part[i] = 0.f;
  __syncthreads();
  const int q = threadIdx.x % quads;
  const int prow = threadIdx.x / quads;
  const int prows = blockDim.x / quads;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  float s = 0.f, ss = 0.f;
  if (prow < prows) {
    const float4* base = reinterpret_cast<const float4*>(x + (size_t)n * HW * C) + q;
    for (int p = p0 + prow; p < p1; p += prows) {
      const float4 v = base[(size_t)p * quads];
      s += (v.x + v.y) + (v.z + v.w);
      ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
    }
  }
  const int g = (q * 4) / cpg;
  atomicAdd(&s_part[2 * g], s);
  atomicAdd(&s_part[2 * g + 1], ss);
  __syncthreads();
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x)
    atomicAdd(&stats[((size_t)n * groups) * 2 + i], (double)s_part[i]);
}

// Ordered variant: block = kGnOrderedPix pixels of one image (a partition fixed by H, W and the block size, which depends
// on C only); the per-thread sums are added in a fixed order per group and written to part[n][block][group][2].
constexpr int kGnOrderedPix = 128;

__global__ void gn_stats_partial_kernel(const float* __restrict__ x, float* __restrict__ part, int HW, int C,
                                        int groups) {
  extern __shared__ float2 s_red[];   // [blockDim.x] (sum, sumsq) of each thread
  const int n = blockIdx.y;
  const int quads = C / 4;
  const int q = threadIdx.x % quads;
  const int prow = threadIdx.x / quads;
  const int prows = blockDim.x / quads;
  const int p0 = blockIdx.x * kGnOrderedPix;
  const int p1 = min(HW, p0 + kGnOrderedPix);
  float s = 0.f, ss = 0.f;
  const float4* base = reinterpret_cast<const float4*>(x + (size_t)n * HW * C) + q;
  for (int p = p0 + prow; p < p1; p += prows) {
    const float4 v = base[(size_t)p * quads];
    s += (v.x + v.y) + (v.z + v.w);
    ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  s_red[threadIdx.x] = make_float2(s, ss);
  __syncthreads();
  const int qpg = C / groups / 4;   // channel quads per group
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < prows; ++r)
      for (int qq = g * qpg; qq < (g + 1) * qpg; ++qq) {
        const float2 t = s_red[r * quads + qq];
        a += t.x;
        b += t.y;
      }
    reinterpret_cast<float2*>(part)[((size_t)n * gridDim.x + blockIdx.x) * groups + g] = make_float2(a, b);
  }
}

// stats[n][j] = sum over p of part[n][p][j] in double (j = 2 * group + {0: sum, 1: sumsq}), in a fixed order: thread
// (r, j) adds rows r, r + 16, ... in ascending order, then thread (0, j) adds the 16 row sums in ascending r.
__global__ void __launch_bounds__(512) gn_finalize_kernel(const float* __restrict__ part, double* __restrict__ stats,
                                                          int P, int cols) {
  __shared__ double s_row[16][32];
  const int n = blockIdx.y, lane = threadIdx.x & 31, r = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  double t = 0.0;
  if (j < cols)
    for (int i = r; i < P; i += 16) t += (double)part[((size_t)n * P + i) * cols + j];
  s_row[r][lane] = t;
  __syncthreads();
  if (r == 0 && j < cols) {
    double sum = 0.0;
#pragma unroll
    for (int i = 0; i < 16; ++i) sum += s_row[i][lane];
    stats[(size_t)n * cols + j] = sum;
  }
}

// |x| max of each image's finite elements (n4 float4s per image) as raw bits: atomicMax into out_bits[n]
__global__ void absmax_per_image_kernel(const uint4* __restrict__ x, long long n4, unsigned* __restrict__ out_bits) {
  const uint4* xi = x + (size_t)blockIdx.y * n4;
  unsigned m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = xi[i];
    m = max(max(m, finite_abs_bits(v.x)), max(finite_abs_bits(v.y), max(finite_abs_bits(v.z), finite_abs_bits(v.w))));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_bits + blockIdx.y, m);
}

// ------------------------------------------------------------------------------------------------
// prep: y = [silu(gn(x))] at (h>>up, w>>up); hi = bf16(y); lo = bf16(y - hi). Output planes have
// C_pad >= C channels (multiple of 64 for the conv's 128-byte TMA rows); padding channels are zero.
// ------------------------------------------------------------------------------------------------
// kF16: ONE fp16 plane (the fp16x2 conv mode: 11 significant bits, half the bytes of the hi+lo pair) instead, written
// as y / s with a power-of-two scale s (block 0 stores s to *scale_out; the conv multiplies it back in fp32), so that
// the plane is neither inf nor fp16-subnormal whatever the activation's magnitude:
//   no GroupNorm  s = 2^(e-12), e the exponent of the largest finite |x| (*absmax_bits: from the producing conv's epilogue, or from
//                 an absmax pass over x): the largest element lands in [2^12, 2^13), as for the attention operands.
//                 Scaling x by 2^k gives the same plane.
//   GroupNorm     |silu(t)| <= |t| <= max|gamma| * (sqrt(n_g * E[x^2]) + |mean|) * rstd + max|beta| over every
//                 (sample, group), n_g the group's element count (|x - mean| <= |x| + |mean| and x^2 <= n_g E[x^2]).
//                 Every block derives the same bound B from the statistics; s = 1 while B lies in [1, 2^13), which
//                 is every ordinary layer, and otherwise the power of two that brings B into that range.
// kPerImage (with kF16): one scale per sample, scale_out[n], from sample n's own |x|max (absmax_bits[n]) or its own
// groups' bound, so that no sample's plane depends on the others in the batch.
__device__ __forceinline__ int gn_plane_shift(float bound) {   // s = 2^shift brings bound into [1, 2^13)
  const unsigned bits = __float_as_uint(bound);
  const int e = max(int((bits >> 23) & 0xffu) - 127, -114);
  return bits ? min(e, 0) + max(e - 12, 0) : 0;
}
__device__ __forceinline__ int absmax_plane_shift(unsigned bits) {   // the largest |x| lands in [2^12, 2^13)
  return bits ? max(int((bits >> 23) & 0xffu) - 127, -114) - 12 : 0;
}

template <bool kF16, bool kPerImage>
__global__ void prep_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                            const float* __restrict__ gamma, const float* __restrict__ beta,
                            __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int N, int H, int W,
                            int C, int C_pad, int groups, int up, float eps, int write_lo,
                            const unsigned* __restrict__ absmax_bits, float* __restrict__ scale_out) {
  // one thread = 8 channels of one output pixel: 2 x 16 B loads, 16 B stores per plane.
  // (mean, rstd) of every (sample, group) are derived once per block from the float64 sums into shared memory: the
  // element loop is then pure fp32 (FFMA + 2 MUFU per element), no float64 arithmetic per quad.
  extern __shared__ float s_mr[];    // [N*groups][2] (with GroupNorm), then kPerImage: s_inv [N], s_bnd [N]
  float* s_inv = s_mr + (stats ? 2 * N * groups : 0);   // kPerImage: 1 / scale of each sample
  unsigned* s_bnd = reinterpret_cast<unsigned*>(s_inv + N);   // kPerImage: bit pattern of each sample's group bound
  const int Ho = H << up, Wo = W << up;
  const int octs = C_pad / 8;
  const size_t total = (size_t)N * Ho * Wo * octs;
  const int cpg = stats ? C / groups : 1;
  __shared__ unsigned s_bound[3];    // kF16 with GroupNorm: bit patterns of max over (sample, group) of
                                     // (sqrt(n_g E[x^2]) + |mean|) * rstd, of max|gamma| and of max|beta|
  if (stats) {
    if (kF16 && threadIdx.x < 3) s_bound[threadIdx.x] = 0u;
    if constexpr (kPerImage)
      for (int i = threadIdx.x; i < N; i += blockDim.x) s_bnd[i] = 0u;
    if (kF16) __syncthreads();
    const double inv_cnt = 1.0 / ((double)H * W * cpg);
    const float n_g = float((double)H * W * cpg);
    float dev_max = 0.f;
    for (int i = threadIdx.x; i < N * groups; i += blockDim.x) {
      const float mean = float(stats[2 * i] * inv_cnt);
      const float msq = float(stats[2 * i + 1] * inv_cnt);
      float var = msq - mean * mean;   // flax fast variance, clamped at 0
      var = fmaxf(var, 0.f);
      s_mr[2 * i] = mean;
      s_mr[2 * i + 1] = rsqrtf(var + eps);
      // finite terms only: a (sample, group) with non-finite statistics has a non-finite plane at any scale, and must
      // not flush the planes of the other samples to zero
      if constexpr (kPerImage)
        atomicMax(s_bnd + i / groups, __float_as_uint(finite_absf((sqrtf(n_g * msq) + fabsf(mean)) * s_mr[2 * i + 1])));
      else if (kF16)
        dev_max = fmaxf(dev_max, finite_absf((sqrtf(n_g * msq) + fabsf(mean)) * s_mr[2 * i + 1]));
    }
    if (kF16) {
      float g_max = 0.f, b_max = 0.f;
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        g_max = fmaxf(g_max, finite_absf(gamma[c]));
        b_max = fmaxf(b_max, finite_absf(beta[c]));
      }
      // non-negative floats order like their bit patterns
      const unsigned m0 = __reduce_max_sync(0xffffffffu, __float_as_uint(dev_max));
      const unsigned m1 = __reduce_max_sync(0xffffffffu, __float_as_uint(g_max));
      const unsigned m2 = __reduce_max_sync(0xffffffffu, __float_as_uint(b_max));
      if ((threadIdx.x & 31) == 0) {
        atomicMax(&s_bound[0], m0);
        atomicMax(&s_bound[1], m1);
        atomicMax(&s_bound[2], m2);
      }
    }
    __syncthreads();
  }
  float inv_scale = 1.f;   // kF16: 1 / s
  if constexpr (kPerImage) {
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      const int shift = stats ? gn_plane_shift(__uint_as_float(s_bound[1]) * __uint_as_float(s_bnd[i]) +
                                               __uint_as_float(s_bound[2]))
                              : absmax_plane_shift(absmax_bits[i]);
      s_inv[i] = __uint_as_float(unsigned(127 - shift) << 23);
      if (blockIdx.x == 0) scale_out[i] = __uint_as_float(unsigned(127 + shift) << 23);
    }
    __syncthreads();
  } else if constexpr (kF16) {
    const int shift =      // s = 2^shift
        stats ? gn_plane_shift(__uint_as_float(s_bound[1]) * __uint_as_float(s_bound[0]) + __uint_as_float(s_bound[2]))
              : absmax_plane_shift(*absmax_bits);
    inv_scale = __uint_as_float(unsigned(127 - shift) << 23);
    if (blockIdx.x == 0 && threadIdx.x == 0) *scale_out = __uint_as_float(unsigned(127 + shift) << 23);
  }
#pragma unroll 2
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int o8 = int(i % octs);
    size_t pix = i / octs;
    const int wo = int(pix % Wo);
    pix /= Wo;
    const int ho = int(pix % Ho);
    const int n = int(pix / Ho);
    const int c0 = o8 * 8;
    float y[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float* src = x + (((size_t)n * H + (ho >> up)) * W + (wo >> up)) * C + c0;
#pragma unroll
    for (int hq = 0; hq < 2; ++hq) {
      const int c = c0 + hq * 4;
      if (c < C) {
        const float4 v = *reinterpret_cast<const float4*>(src + hq * 4);
        float* yy = y + hq * 4;
        yy[0] = v.x; yy[1] = v.y; yy[2] = v.z; yy[3] = v.w;
        if (stats) {
          const int g = c / cpg;
          const float mean = s_mr[2 * (n * groups + g)], rstd = s_mr[2 * (n * groups + g) + 1];
          const float4 g4 = *reinterpret_cast<const float4*>(gamma + c);
          const float4 b4 = *reinterpret_cast<const float4*>(beta + c);
          const float gg[4] = {g4.x, g4.y, g4.z, g4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float t = (yy[e] - mean) * rstd * gg[e] + bb[e];
            yy[e] = __fdividef(t, 1.0f + __expf(-t));   // silu = t * sigmoid(t)
          }
        }
      }
    }
    uint32_t h4[4], l4[4];
    const size_t o = (((size_t)n * Ho + ho) * Wo + wo) * C_pad + c0;
    if constexpr (kF16) {
      const float inv = kPerImage ? s_inv[n] : inv_scale;
#pragma unroll
      for (int e = 0; e < 4; ++e) h4[e] = pack_f16x2(y[2 * e] * inv, y[2 * e + 1] * inv);
      *reinterpret_cast<uint4*>(hi + o) = make_uint4(h4[0], h4[1], h4[2], h4[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(y[2 * e]), h1 = __float2bfloat16_rn(y[2 * e + 1]);
        h4[e] = uint32_t(__bfloat16_as_ushort(h0)) | (uint32_t(__bfloat16_as_ushort(h1)) << 16);
        l4[e] = pack_bf16x2(y[2 * e] - __bfloat162float(h0), y[2 * e + 1] - __bfloat162float(h1));
      }
      *reinterpret_cast<uint4*>(hi + o) = make_uint4(h4[0], h4[1], h4[2], h4[3]);
      if (write_lo) *reinterpret_cast<uint4*>(lo + o) = make_uint4(l4[0], l4[1], l4[2], l4[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// direct conv, Cin = 3, 3x3 SAME, Cout = 128: block = 8 rows x 16 cols of output pixels x all 128 channels,
// 128 threads; thread = 8 consecutive pixels of one row x 16 output channels (a 128-register tile: 12 shared-
// memory loads feed 128 FMAs per tap — the first version did one load per FMA and was LSU-bound at 1.8 ms).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
conv_cin3_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                 float* __restrict__ y, int N, int H, int W) {
  constexpr int Cout = 128;
  __shared__ __align__(16) float s_w[27 * Cout];   // HWIO order: [(kh*3+kw)*3+c][cout]
  __shared__ float s_in[10 * 18 * 3];               // input patch with a 1-pixel halo
  const int tiles_w = W / 16;
  const int tw = blockIdx.x % tiles_w, th = blockIdx.x / tiles_w, n = blockIdx.y;
  for (int i = threadIdx.x; i < 27 * Cout / 4; i += blockDim.x)
    reinterpret_cast<float4*>(s_w)[i] = reinterpret_cast<const float4*>(w)[i];
  for (int i = threadIdx.x; i < 10 * 18 * 3; i += blockDim.x) {
    const int c = i % 3, px = (i / 3) % 18, py = i / 54;
    const int gy = th * 8 + py - 1, gx = tw * 16 + px - 1;
    s_in[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? x[(((size_t)n * H + gy) * W + gx) * 3 + c] : 0.f;
  }
  __syncthreads();
  const int cg = threadIdx.x & 7;        // 16 output channels [16*cg, 16*cg+16)
  const int pg = threadIdx.x >> 3;       // 16 pixel groups: row pg>>1, columns 8*(pg&1) .. +8
  const int row = pg >> 1, x0 = (pg & 1) * 8;
  float acc[8][16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float b = bias[cg * 16 + j];
#pragma unroll
    for (int p2 = 0; p2 < 8; ++p2) acc[p2][j] = b;
  }
#pragma unroll
  for (int t = 0; t < 27; ++t) {
    const int kh = t / 9, kw = (t / 3) % 3, c = t % 3;
    float a[8], wv[16];
#pragma unroll
    for (int p2 = 0; p2 < 8; ++p2) a[p2] = s_in[((row + kh) * 18 + (x0 + p2 + kw)) * 3 + c];
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) {
      const float4 w4 = *reinterpret_cast<const float4*>(&s_w[t * Cout + cg * 16 + 4 * j4]);
      wv[4 * j4] = w4.x; wv[4 * j4 + 1] = w4.y; wv[4 * j4 + 2] = w4.z; wv[4 * j4 + 3] = w4.w;
    }
#pragma unroll
    for (int p2 = 0; p2 < 8; ++p2)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[p2][j] = fmaf(a[p2], wv[j], acc[p2][j]);
  }
#pragma unroll
  for (int p2 = 0; p2 < 8; ++p2) {
    float* dst = y + (((size_t)n * H + th * 8 + row) * W + tw * 16 + x0 + p2) * Cout + cg * 16;
#pragma unroll
    for (int j = 0; j < 16; j += 4)
      *reinterpret_cast<float4*>(dst + j) = make_float4(acc[p2][j], acc[p2][j + 1], acc[p2][j + 2], acc[p2][j + 3]);
  }
}

// ------------------------------------------------------------------------------------------------
// VectorQuantizer: idx[b] = argmin_n ((sum z^2 + sum e_n^2) - 2 z.e_n), first index on ties.
// Arithmetic order pinned to oracle/vqgan_ref.py::vq_distances_f32: sequential over d, multiply and
// add rounded separately (__fmul_rn/__fadd_rn forbid FMA contraction) => bit-exact indices.
// Block = 128 threads, 16 rows of z; the codebook streams through in tiles of 128 codes
// (thread = one code held in registers), rows broadcast from shared memory.
// ------------------------------------------------------------------------------------------------
constexpr int kVqDim = 64;
constexpr int kVqSplits = 8;   // the codebook is scanned in 8 slices so that 4096 rows still fill the GPU

// thread = one row of z (held in registers); the block's codebook slice streams through shared memory
// in tiles of 128 codes (broadcast reads). Every thread visits codes in ascending order, so a strict
// '<' keeps the first minimal index. Partial (distance, index) per slice go to `part_*`; an empty slice
// (n_e < 8) reports index -1.
// Non-finite distances follow np.argmin over the oracle's float32 distances: the first NaN wins, and a row whose
// distances are all +inf keeps its first code (|z| >~ 1.8e19 overflows sum z^2; a NaN pixel makes every distance
// NaN). The first code of a slice is therefore always taken, whatever its distance.
__device__ __forceinline__ bool vq_better(float d, float best_d, int best_i) {
  return best_i < 0 || (!isnan(best_d) && (isnan(d) || d < best_d));
}

__global__ void __launch_bounds__(128)
vq_argmin_partial_kernel(const float* __restrict__ z, const float* __restrict__ emb, float* __restrict__ part_d,
                         int* __restrict__ part_i, int N, int n_e) {
  __shared__ __align__(16) float s_e[128][kVqDim];
  __shared__ float s_ee[128];
  const int row = blockIdx.x * 128 + threadIdx.x;
  const int per = (n_e + kVqSplits - 1) / kVqSplits;
  const int c_begin = blockIdx.y * per, c_end = min(n_e, c_begin + per);
  float zr[kVqDim];
#pragma unroll
  for (int d4 = 0; d4 < kVqDim / 4; ++d4) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < N) v = reinterpret_cast<const float4*>(z + (size_t)row * kVqDim)[d4];
    zr[4 * d4] = v.x; zr[4 * d4 + 1] = v.y; zr[4 * d4 + 2] = v.z; zr[4 * d4 + 3] = v.w;
  }
  float zz = 0.f;
#pragma unroll
  for (int d = 0; d < kVqDim; ++d) zz = __fadd_rn(zz, __fmul_rn(zr[d], zr[d]));
  float best_d = INFINITY;
  int best_i = -1;
  for (int c0 = c_begin; c0 < c_end; c0 += 128) {
    __syncthreads();
    {
      const int code = c0 + threadIdx.x;
      float ee = 0.f;
      if (code < c_end) {
        const float4* src = reinterpret_cast<const float4*>(emb + (size_t)code * kVqDim);
#pragma unroll
        for (int d4 = 0; d4 < kVqDim / 4; ++d4) {
          const float4 v = src[d4];
          *reinterpret_cast<float4*>(&s_e[threadIdx.x][4 * d4]) = v;
          ee = __fadd_rn(ee, __fmul_rn(v.x, v.x));
          ee = __fadd_rn(ee, __fmul_rn(v.y, v.y));
          ee = __fadd_rn(ee, __fmul_rn(v.z, v.z));
          ee = __fadd_rn(ee, __fmul_rn(v.w, v.w));
        }
      }
      s_ee[threadIdx.x] = ee;
    }
    __syncthreads();
    const int cnt = min(128, c_end - c0);
    for (int j = 0; j < cnt; ++j) {
      float dot = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < kVqDim / 4; ++d4) {
        const float4 e4 = *reinterpret_cast<const float4*>(&s_e[j][4 * d4]);
        dot = __fadd_rn(dot, __fmul_rn(zr[4 * d4], e4.x));
        dot = __fadd_rn(dot, __fmul_rn(zr[4 * d4 + 1], e4.y));
        dot = __fadd_rn(dot, __fmul_rn(zr[4 * d4 + 2], e4.z));
        dot = __fadd_rn(dot, __fmul_rn(zr[4 * d4 + 3], e4.w));
      }
      const float dist = __fadd_rn(__fadd_rn(zz, s_ee[j]), -__fmul_rn(2.0f, dot));
      if (vq_better(dist, best_d, best_i)) {
        best_d = dist;
        best_i = c0 + j;
      }
    }
  }
  if (row < N) {
    part_d[(size_t)blockIdx.y * N + row] = best_d;
    part_i[(size_t)blockIdx.y * N + row] = best_i;
  }
}

// merge the slices in ascending order (same rule as within a slice => first index), emit idx and the
// straight-through value. idx is always in [0, n_e): at least slice 0 is non-empty.
__global__ void vq_argmin_final_kernel(const float* __restrict__ z, const float* __restrict__ emb,
                                       const float* __restrict__ part_d, const int* __restrict__ part_i,
                                       int* __restrict__ idx, float* __restrict__ zq_st, int N) {
  const int row = blockIdx.x * (blockDim.x / 16) + threadIdx.x / 16;
  const int q = threadIdx.x % 16;
  if (row >= N) return;
  float bd = INFINITY;
  int bi = -1;
  for (int s = 0; s < kVqSplits; ++s) {
    const int i = part_i[(size_t)s * N + row];
    const float d = part_d[(size_t)s * N + row];
    if (i >= 0 && vq_better(d, bd, bi)) {
      bd = d;
      bi = i;
    }
  }
  if (q == 0) idx[row] = bi;
  if (zq_st) {  // z + (e[idx] - z), rounded like the reference (vqgan.py:215)
    const float4 zv = reinterpret_cast<const float4*>(z + (size_t)row * kVqDim)[q];
    const float4 ev = reinterpret_cast<const float4*>(emb + (size_t)bi * kVqDim)[q];
    float4 o;
    o.x = __fadd_rn(zv.x, __fadd_rn(ev.x, -zv.x));
    o.y = __fadd_rn(zv.y, __fadd_rn(ev.y, -zv.y));
    o.z = __fadd_rn(zv.z, __fadd_rn(ev.z, -zv.z));
    o.w = __fadd_rn(zv.w, __fadd_rn(ev.w, -zv.w));
    reinterpret_cast<float4*>(zq_st + (size_t)row * kVqDim)[q] = o;
  }
}

__global__ void vq_gather_kernel(const int* __restrict__ idx, const float4* __restrict__ emb, float4* __restrict__ out,
                                 long long N, int quads, int n_e) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < N * quads;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / quads;
    int c = idx[r];
    c = min(max(c, 0), n_e - 1);
    out[i] = emb[(long long)c * quads + (i % quads)];
  }
}

}  // namespace lwm

using namespace lwm;

extern "C" int lwm_vq_gn_stats(const float* x, double* stats, int N, int H, int W, int C, int groups, void* stream) {
  if (!x || !stats) return lwm_fail(LWM_ERR_ARG, "vq_gn_stats: null pointer");
  if (C % groups || (C / groups) % 4 || C % 4) return lwm_fail(LWM_ERR_SHAPE, "vq_gn_stats: C/groups must be a multiple of 4");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(stats, 0, sizeof(double) * 2 * N * groups, st) != cudaSuccess)
    return lwm_fail(LWM_ERR_CUDA, "vq_gn_stats: memset failed");
  const int quads = C / 4;
  int threads = ((512 / quads) > 0 ? (512 / quads) : 1) * quads;   // whole pixel rows per block
  if (threads > 1024) threads = quads;
  const int HW = H * W;
  int ppb = 256;
  while ((HW + ppb - 1) / ppb * N < 296 && ppb > 16) ppb /= 2;   // >= 2 blocks per SM
  dim3 grid((HW + ppb - 1) / ppb, N);
  gn_stats_kernel<<<grid, threads, groups * 2 * sizeof(float), st>>>(x, stats, HW, C, groups, ppb);
  return lwm_check_launch("gn_stats_kernel");
}

// the statistics [N, cols / 2, 2] of per-image partials part [N][P][cols] (lwm_vq_gn_stats_ordered, and
// lwm_vq_conv2d_f16_ordered's epilogue)
int lwm_vq_gn_finalize(const float* part, double* stats, int N, int P, int cols, cudaStream_t st) {
  gn_finalize_kernel<<<dim3((cols + 31) / 32, N), 512, 0, st>>>(part, stats, P, cols);
  return lwm_check_launch("gn_finalize_kernel");
}

extern "C" int lwm_vq_gn_stats_ordered(const float* x, double* stats, float* workspace, long long workspace_bytes,
                                       int N, int H, int W, int C, int groups, void* stream) {
  if (!x || !stats || !workspace) return lwm_fail(LWM_ERR_ARG, "vq_gn_stats_ordered: null pointer");
  if (N <= 0 || H <= 0 || W <= 0 || groups <= 0 || C % groups || (C / groups) % 4 || C > 4096)
    return lwm_fail(LWM_ERR_SHAPE, "vq_gn_stats_ordered: C/groups must be a multiple of 4, C <= 4096, non-empty");
  const long long HW = (long long)H * W;
  const long long P = (HW + kGnOrderedPix - 1) / kGnOrderedPix;
  if (HW > (1ll << 31) - 1) return lwm_fail(LWM_ERR_SHAPE, "vq_gn_stats_ordered: H * W exceeds int32");
  if (workspace_bytes < (long long)N * P * groups * 2 * (long long)sizeof(float))
    return lwm_fail(LWM_ERR_SHAPE, "vq_gn_stats_ordered: workspace too small (N * ceil(H*W/128) * groups * 2 floats)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int quads = C / 4;
  int threads = ((512 / quads) > 0 ? (512 / quads) : 1) * quads;   // whole pixel rows per block: a function of C
  if (threads > 1024) threads = quads;
  gn_stats_partial_kernel<<<dim3(unsigned(P), N), threads, threads * sizeof(float2), st>>>(x, workspace, int(HW), C,
                                                                                            groups);
  const int status = lwm_check_launch("gn_stats_partial_kernel");
  return status != LWM_OK ? status : lwm_vq_gn_finalize(workspace, stats, N, int(P), groups * 2, st);
}

extern "C" int lwm_vq_prep(const float* x, const double* gn_stats, const float* gamma, const float* beta, void* hi,
                           void* lo, int N, int H, int W, int C, int C_pad, int groups, int upsample2x, float eps,
                           void* stream) {
  if (!x || !hi) return lwm_fail(LWM_ERR_ARG, "vq_prep: null pointer");
  if (C % 4 || C_pad % 8 || C_pad < C) return lwm_fail(LWM_ERR_SHAPE, "vq_prep: C % 4 and C_pad % 8 required");
  if (gn_stats && (!gamma || !beta || C % groups || (C / groups) % 4))
    return lwm_fail(LWM_ERR_SHAPE, "vq_prep: GroupNorm needs gamma/beta and C/groups % 4 == 0");
  if (gn_stats && (size_t)N * groups * 8 > 40 * 1024) return lwm_fail(LWM_ERR_SHAPE, "vq_prep: N * groups too large (<= 5120)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  const size_t total = (size_t)N * (H << upsample2x) * (W << upsample2x) * (C_pad / 8);
  const int threads = 256;
  const size_t want = (total + threads - 1) / threads;
  const unsigned blocks = unsigned(want < kNumSMs * 32 ? want : kNumSMs * 32);
  prep_kernel<false, false><<<blocks, threads, gn_stats ? size_t(N) * groups * 8 : 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, gn_stats, gamma, beta, reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo), N, H, W,
      C, C_pad, groups, upsample2x ? 1 : 0, eps, lo != nullptr, nullptr, nullptr);
  return lwm_check_launch("prep_kernel");
}

// fp16x2 conv mode: y = [silu(groupnorm(x))] (optionally nearest-2x upsampled) as ONE fp16 plane [N,H',W',C_pad]
// holding y / *scale_out (prep_kernel). Without GroupNorm the scale comes from x_absmax (|x|max bits): read as given
// (x_absmax_given, e.g. from lwm_vq_conv2d_f16's absmax_out), or computed into it here.
extern "C" int lwm_vq_prep_f16(const float* x, const double* gn_stats, const float* gamma, const float* beta, void* out,
                               float* scale_out, unsigned* x_absmax, int x_absmax_given, int N, int H, int W, int C,
                               int C_pad, int groups, int upsample2x, float eps, void* stream) {
  if (!x || !out || !scale_out) return lwm_fail(LWM_ERR_ARG, "vq_prep_f16: null pointer");
  if (!gn_stats && !x_absmax) return lwm_fail(LWM_ERR_ARG, "vq_prep_f16: the plane without GroupNorm needs x_absmax");
  if (C % 4 || C_pad % 8 || C_pad < C) return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16: C % 4 and C_pad % 8 required");
  if (gn_stats && (!gamma || !beta || C % groups || (C / groups) % 4))
    return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16: GroupNorm needs gamma/beta and C/groups % 4 == 0");
  if (gn_stats && (size_t)N * groups * 8 > 40 * 1024) return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16: N * groups too large (<= 5120)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!gn_stats && !x_absmax_given) {
    if (cudaMemsetAsync(x_absmax, 0, 4, st) != cudaSuccess) return lwm_fail(LWM_ERR_CUDA, "vq_prep_f16: memset failed");
    const long long n4 = (long long)N * H * W * C / 4;
    const long long want4 = (n4 + 255) / 256;
    absmax_f32_kernel<<<unsigned(want4 < kNumSMs * 8 ? (want4 > 0 ? want4 : 1) : kNumSMs * 8), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(x), n4, x_absmax);
  }
  const size_t total = (size_t)N * (H << upsample2x) * (W << upsample2x) * (C_pad / 8);
  const int threads = 256;
  const size_t want = (total + threads - 1) / threads;
  const unsigned blocks = unsigned(want < kNumSMs * 32 ? want : kNumSMs * 32);
  prep_kernel<true, false><<<blocks, threads, gn_stats ? size_t(N) * groups * 8 : 0, st>>>(
      x, gn_stats, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out), nullptr, N, H, W, C, C_pad, groups,
      upsample2x ? 1 : 0, eps, 0, x_absmax, scale_out);
  return lwm_check_launch("prep_kernel<f16>");
}

// lwm_vq_prep_f16 with one scale per sample: scale_out [N], x_absmax [N] (each sample's |x|max bits; computed here into
// it unless x_absmax_given, e.g. lwm_vq_conv2d_f16_ordered's absmax_out).
extern "C" int lwm_vq_prep_f16_ordered(const float* x, const double* gn_stats, const float* gamma, const float* beta,
                                       void* out, float* scale_out, unsigned* x_absmax, int x_absmax_given, int N, int H,
                                       int W, int C, int C_pad, int groups, int upsample2x, float eps, void* stream) {
  if (!x || !out || !scale_out) return lwm_fail(LWM_ERR_ARG, "vq_prep_f16_ordered: null pointer");
  if (!gn_stats && !x_absmax) return lwm_fail(LWM_ERR_ARG, "vq_prep_f16_ordered: the plane without GroupNorm needs x_absmax");
  if (N <= 0 || H <= 0 || W <= 0) return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16_ordered: empty tensor");
  if (C % 4 || C_pad % 8 || C_pad < C) return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16_ordered: C % 4 and C_pad % 8 required");
  if (gn_stats && (!gamma || !beta || groups <= 0 || C % groups || (C / groups) % 4))
    return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16_ordered: GroupNorm needs gamma/beta and C/groups % 4 == 0");
  const size_t smem = (gn_stats ? size_t(N) * groups * 8 : 0) + size_t(N) * 8;
  if (smem > 40 * 1024) return lwm_fail(LWM_ERR_SHAPE, "vq_prep_f16_ordered: N (* groups) too large for the block's tables");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!gn_stats && !x_absmax_given) {
    if (cudaMemsetAsync(x_absmax, 0, sizeof(unsigned) * N, st) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "vq_prep_f16_ordered: memset failed");
    const long long n4 = (long long)H * W * C / 4;
    const long long want4 = (n4 + 255) / 256, cap = kNumSMs * 8 / N;   // atomicMax: any grid gives the same bits
    const long long per_image = want4 < cap ? want4 : cap;
    absmax_per_image_kernel<<<dim3(unsigned(per_image > 0 ? per_image : 1), N), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(x), n4, x_absmax);
  }
  const size_t total = (size_t)N * (H << upsample2x) * (W << upsample2x) * (C_pad / 8);
  const int threads = 256;
  const size_t want = (total + threads - 1) / threads;
  const unsigned blocks = unsigned(want < kNumSMs * 32 ? want : kNumSMs * 32);
  prep_kernel<true, true><<<blocks, threads, smem, st>>>(
      x, gn_stats, gamma, beta, reinterpret_cast<__nv_bfloat16*>(out), nullptr, N, H, W, C, C_pad, groups,
      upsample2x ? 1 : 0, eps, 0, x_absmax, scale_out);
  return lwm_check_launch("prep_kernel<f16, per image>");
}

extern "C" int lwm_vq_conv_cin3(const float* x, const float* w_hwio, const float* bias, float* y, int N, int H, int W,
                                int Cout, void* stream) {
  if (!x || !w_hwio || !bias || !y) return lwm_fail(LWM_ERR_ARG, "vq_conv_cin3: null pointer");
  if (H % 8 || W % 16 || Cout != 128)
    return lwm_fail(LWM_ERR_SHAPE, "vq_conv_cin3: H % 8, W % 16 and Cout == 128 (hidden_channels, vqgan.py:64)");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  dim3 grid((H / 8) * (W / 16), N);
  conv_cin3_kernel<<<grid, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, w_hwio, bias, y, N, H, W);
  return lwm_check_launch("conv_cin3_kernel");
}

extern "C" int lwm_vq_argmin(const float* z, const float* codebook, int* idx, float* zq_st, void* workspace,
                             int N, int n_e, int e_dim, void* stream) {
  if (!z || !codebook || !idx || !workspace) return lwm_fail(LWM_ERR_ARG, "vq_argmin: null pointer");
  if (e_dim != kVqDim) return lwm_fail(LWM_ERR_SHAPE, "vq_argmin: e_dim must be 64 (quantized_embed_dim, vqgan.py:72)");
  if (N <= 0 || n_e <= 0) return lwm_fail(LWM_ERR_SHAPE, "vq_argmin: empty input");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* part_d = reinterpret_cast<float*>(workspace);            // workspace: 8 * N * (4 + 4) bytes
  int* part_i = reinterpret_cast<int*>(part_d + (size_t)kVqSplits * N);
  dim3 grid((N + 127) / 128, kVqSplits);
  vq_argmin_partial_kernel<<<grid, 128, 0, st>>>(z, codebook, part_d, part_i, N, n_e);
  vq_argmin_final_kernel<<<(N + 15) / 16, 256, 0, st>>>(z, codebook, part_d, part_i, idx, zq_st, N);
  return lwm_check_launch("vq_argmin kernels");
}

extern "C" int lwm_vq_gather(const int* idx, const float* codebook, float* out, long long N, int n_e, int e_dim,
                             void* stream) {
  if (!idx || !codebook || !out) return lwm_fail(LWM_ERR_ARG, "vq_gather: null pointer");
  if (e_dim % 4) return lwm_fail(LWM_ERR_SHAPE, "vq_gather: e_dim % 4");
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  if (N == 0) return LWM_OK;
  const int quads = e_dim / 4;
  const long long total = N * quads;
  const unsigned blocks = unsigned((total + 255) / 256 < kNumSMs * 16 ? (total + 255) / 256 : kNumSMs * 16);
  vq_gather_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      idx, reinterpret_cast<const float4*>(codebook), reinterpret_cast<float4*>(out), N, quads, n_e);
  return lwm_check_launch("vq_gather_kernel");
}
