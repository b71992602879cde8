// VQGAN convolutions (flax nn.Conv of lwm/vqgan.py: ResnetBlock 3x3, 1x1 shortcuts, Downsample
// stride-2, Upsample conv, conv_out, quant/post_quant 1x1) as a persistent implicit GEMM on the
// Hopper tensor cores (wgmma).
//
//   GEMM view  M = N*Ho*Wo output pixels, N = Cout, K = taps * Cin.
//   A operand  the activation plane [N,Hin,Win,Cpad] (bf16, written by lwm_vq_prep) is never
//              im2col'ed in memory: for tap (kh,kw) and a 64-channel slice, ONE 4-D TMA box
//              (64 ch x 16 px x 8 rows) lands as a 128-row x 128-byte K-major swizzled tile; the
//              tap shift is just a coordinate offset and out-of-image pixels are zero-filled by
//              the TMA unit (SAME padding / the bottom-right pad of Downsample for free). Stride-2
//              convs use the tensor map's element strides.
//   B operand  weights pre-packed [tap][Cout_pad][Cpad] bf16 (K-major), 3-D TMA box (64, BN, 1).
//   precision  n_pass = 1: bf16 x bf16 (fast). n_pass = 3: both operands split x = hi + lo (two bf16)
//              and D += A_hi B_hi + A_lo B_hi + A_hi B_lo — fp32-class accuracy (2^-16 products,
//              fp32 accumulation), which is what the reference's fp32 convs need.
//              n_pass = 2 ("fp16x2"): the activation is ONE fp16 plane and the weights are split w = hi + lo (two fp16,
//              pre-scaled by a power of two); both halves are stacked along N ([BN hi rows | BN lo rows]) so a single
//              64 x 2BN x 16 wgmma per warpgroup produces A.hi and A.lo side by side and the epilogue adds the two
//              halves: 2x the algorithmic MMA work instead of 3x and one operand plane to write and read instead of two.
//              The plane holds x / a_scale (a power of two, lwm_vq_prep_f16), restored with w_scale_inv in fp32.
//   GN stats   optional epilogue: per-(sample, group) sum / sum of squares of the conv OUTPUT (bias and residual
//              included) — the statistics the next GroupNorm needs — so no separate pass re-reads the activation;
//              likewise |output|max, the scale of a raw fp16 plane of the output (Downsample, 1x1 shortcut).
//   ordered    kOrdered instances (torch.use_deterministic_algorithms): no atomics and no sums carried across tiles. Each
//              (tile, consumer warp) writes its per-group (sum, sumsq) to its own slot of a workspace indexed by (image,
//              M tile within the image, warp), so the reduction order depends on the image's own pixels only, never on N,
//              the grid or the SM count; gn_finalize_kernel adds the slots in a fixed order. The fp16 plane has one scale
//              per image (a_scale[n]) and the |output|max goes to absmax[n].
//   pipeline   warp 8: TMA producer through a ring of `stages` slots; warpgroups 0 / 1: pixels [0,64) / [64,128)
//              of the 8x16 tile, fp32 accumulators in registers, epilogue (+ bias (+ residual) -> fp32 NHWC)
//              straight from the accumulator fragment. Grid = #SMs, tiles strided.
#include "ptx.cuh"
#include "tmap.h"
#include "capi_internal.h"

namespace lwm {

constexpr int kConvThreads = 384;
constexpr int kConvConsumerWarps = 8;
constexpr int kATile = 128 * 128;  // 16 KB: 128 pixels x 64 bf16

struct ConvParams {
  int N, Ho, Wo, Cout, Cpad;      // output geometry, real Cout, padded Cin
  int taps_w, taps;               // 3 (or 1), 9 (or 1)
  int stride, pad;                // input coordinate = out*stride + tap - pad
  int BN, n_tiles;                // N-tile width (<= 256, multiple of 16) and count
  int n_pass;                     // 1 (bf16), 3 (bf16x3) or 2 (fp16 activation x stacked fp16 hi|lo weights)
  float w_scale_inv;              // n_pass 2: the weights were packed multiplied by 1/w_scale_inv (a power of two)
  const float* a_scale;           // n_pass 2, optional: the activation plane holds x / *a_scale (a power of two)
  double* stats;                  // optional [N, groups, 2] (sum, sumsq) of the output, accumulated with atomics
  unsigned* absmax;               // n_pass 2, optional: atomicMax of the output's |value| bit patterns (the next
                                  // fp16 plane's scale, without another pass over the tensor)
  int groups;
  int stages;
  int clip;                       // 1: clamp the result to [-1, 1] (VQGANModel.decode, vqgan.py:141)
  const float* bias;              // [Cout]
  const float* residual;          // [N,Ho,Wo,Cout] or null
  float* out;                     // [N,Ho,Wo,Cout]
  float* part;                    // kOrdered, optional: [N][Ho/8 * Wo/16][8 warps][groups][2] (sum, sumsq) per (tile, warp)
};

// NI: the wgmma N (BN, or 2*BN for the stacked fp16x2 weights); kF16: fp16 operands (n_pass 2), else bf16;
// kOrdered (kF16 only): per-image a_scale / absmax, and the statistics as per-(tile, warp) partials in p.part.
template <int NI, bool kF16, bool kOrdered>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
                  const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo,
                  const ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if (smem_u32(smem) & 1023u) __trap();
  const int b_bytes = (p.n_pass == 2 ? 2 : 1) * p.BN * 128;
  const int stage_bytes = (p.n_pass == 3 ? 2 : 1) * (kATile + b_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* empty = full + 8;
  float* s_stats = reinterpret_cast<float*>(empty + 8);   // [64][2] per-group partials of the current tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_w = p.Wo / 16, tiles_h = p.Ho / 8;
  const int m_tiles = p.N * tiles_h * tiles_w;
  const int total_tiles = m_tiles * p.n_tiles;
  const int k_chunks = p.Cpad / 64;
  const int k_iters = p.taps * k_chunks;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConvConsumerWarps);
    }
    fence_mbar_init();
    for (int i = 0; i < 128; ++i) s_stats[i] = 0.f;
  }
  __syncthreads();

  // every CTA owns a CONTIGUOUS range of tiles, ordered N-tile-major then image-major: consecutive tiles share the
  // activation halo in L2, and (image, N tile) — the key of the GroupNorm-statistics accumulators — changes at most a
  // few times per CTA
  const int tile_begin = int((long long)total_tiles * blockIdx.x / gridDim.x);
  const int tile_end = int((long long)total_tiles * (blockIdx.x + 1) / gridDim.x);
  auto decode_tile = [&](int tile, int& n, int& oh0, int& ow0, int& nt) {
    nt = tile / m_tiles;
    int m = tile % m_tiles;
    ow0 = (m % tiles_w) * 16;
    m /= tiles_w;
    oh0 = (m % tiles_h) * 8;
    n = m / tiles_h;
  };

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      tma_prefetch_desc(&tmAhi);
      tma_prefetch_desc(&tmBhi);
      if (p.n_pass == 3) {
        tma_prefetch_desc(&tmAlo);
        tma_prefetch_desc(&tmBlo);
      }
      int it = 0;
      for (int tile = tile_begin; tile < tile_end; ++tile) {
        int n, oh0, ow0, nt;
        decode_tile(tile, n, oh0, ow0, nt);
        for (int ki = 0; ki < k_iters; ++ki, ++it) {
          const int s = it % p.stages;
          const uint32_t ph = (it / p.stages) & 1;
          mbar_wait(&empty[s], ph ^ 1);
          const int tap = ki / k_chunks, c0 = (ki % k_chunks) * 64;
          const int kh = tap / p.taps_w, kw = tap % p.taps_w;
          const int ix = ow0 * p.stride + kw - p.pad, iy = oh0 * p.stride + kh - p.pad;
          uint8_t* st = smem + s * stage_bytes;
          mbar_arrive_expect_tx(&full[s], stage_bytes);
          tma_load_4d(st, &tmAhi, &full[s], c0, ix, iy, n);
          tma_load_3d(st + kATile, &tmBhi, &full[s], c0, nt * (p.n_pass == 2 ? 2 : 1) * p.BN, tap);
          if (p.n_pass == 3) {
            tma_load_4d(st + kATile + b_bytes, &tmAlo, &full[s], c0, ix, iy, n);
            tma_load_3d(st + 2 * kATile + b_bytes, &tmBlo, &full[s], c0, nt * p.BN, tap);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, quad = lane & 3;
  const int ncols = kF16 ? NI / 2 : NI;   // output channels per tile (hi | lo halves are summed for fp16x2)
  // GroupNorm statistics of the output: per-thread running sums for every 8-channel group of the current N tile, kept
  // in registers across tiles and folded (warp shuffle -> shared -> double atomics) only when the (image, N tile) pair
  // changes — a handful of times per CTA thanks to the contiguous tile ranges.
  constexpr int kStatG = kF16 ? NI / 16 : 1;
  float st1[kStatG], st2[kStatG];
#pragma unroll
  for (int i = 0; i < kStatG; ++i) st1[i] = st2[i] = 0.f;
  int st_n = -1, st_nt = -1;
  const bool want_stats = kOrdered ? p.part != nullptr : p.stats != nullptr;
  const int cpg = want_stats ? p.Cout / p.groups : 1;
  // fp16x2: accumulator units -> output units, w_scale_inv * a_scale (a product of powers of two: exact)
  const float out_scale = (kF16 && p.a_scale) ? p.w_scale_inv * *p.a_scale : p.w_scale_inv;
  float amax = 0.f;     // largest finite |output|: a NaN or inf output stays one in the next plane, whatever its scale
  auto flush_stats = [&]() {
    if (st_n < 0) return;
#pragma unroll
    for (int g = 0; g < kStatG; ++g) {
      float s1 = st1[g], s2 = st2[g];
#pragma unroll
      for (int sh = 4; sh < 32; sh <<= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, sh);
        s2 += __shfl_xor_sync(0xffffffffu, s2, sh);
      }
      const int c = st_nt * p.BN + g * 8 + lane * 2;   // lanes 0..3: a channel pair, never straddling a group
      if (lane < 4 && g * 8 < ncols && c < p.Cout) {
        atomicAdd(&s_stats[2 * (c / cpg)], s1);
        atomicAdd(&s_stats[2 * (c / cpg) + 1], s2);
      }
      st1[g] = st2[g] = 0.f;
    }
    named_bar_sync(1, 256);
    if (threadIdx.x < 2 * p.groups) {
      const float t = s_stats[threadIdx.x];
      if (t != 0.f) atomicAdd(&p.stats[(size_t)st_n * p.groups * 2 + threadIdx.x], (double)t);
      s_stats[threadIdx.x] = 0.f;
    }
    named_bar_sync(1, 256);
  };

  int it = 0;
  for (int tile = tile_begin; tile < tile_end; ++tile) {
    int n, oh0, ow0, nt;
    decode_tile(tile, n, oh0, ow0, nt);
    if (!kOrdered && p.stats && (n != st_n || nt != st_nt)) {
      flush_stats();
      st_n = n;
      st_nt = nt;
    }
    float acc[NI / 2];
    int prev_s = -1;
    for (int ki = 0; ki < k_iters; ++ki, ++it) {
      const int s = it % p.stages;
      mbar_wait(&full[s], (it / p.stages) & 1);
      const uint32_t a_hi = smem_u32(smem + s * stage_bytes);
      const uint64_t dAh = desc_kmajor_sw128(a_hi + wg * 64 * 128), dBh = desc_kmajor_sw128(a_hi + kATile);
      const uint64_t dAl = desc_kmajor_sw128(a_hi + kATile + b_bytes + wg * 64 * 128);
      const uint64_t dBl = desc_kmajor_sw128(a_hi + 2 * kATile + b_bytes);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t o = ks * 32;
        wgmma_ss<NI, kF16, 0, 0>(acc, desc_advance(dAh, o), desc_advance(dBh, o), (ki | ks) != 0);
        if (!kF16 && p.n_pass == 3) {
          wgmma_ss<NI, kF16, 0, 0>(acc, desc_advance(dAl, o), desc_advance(dBh, o), 1);
          wgmma_ss<NI, kF16, 0, 0>(acc, desc_advance(dAh, o), desc_advance(dBl, o), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-step's wgmmas are done: its slot may be refilled
      if (prev_s >= 0 && lane == 0) mbar_arrive(&empty[prev_s]);
      prev_s = s;
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (lane == 0) mbar_arrive(&empty[prev_s]);

    // ---- epilogue: this thread's pixels are rows r and r + 8 of its warp's 16 (one image row of the 8x16 tile)
    const int c_base = nt * p.BN;
    float tile_scale = out_scale;
    if constexpr (kOrdered) tile_scale = p.a_scale ? p.w_scale_inv * p.a_scale[n] : p.w_scale_inv;
    const bool vec = (p.Cout & 1) == 0;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const size_t pix = ((size_t)n * p.Ho + oh0 + wg * 4 + w) * p.Wo + ow0 + (lane >> 2) + 8 * hh;
      float* dst = p.out + pix * p.Cout;
      const float* res = p.residual ? p.residual + pix * p.Cout : nullptr;
#pragma unroll
      for (int g = 0; g < NI / 8; ++g) {
        if (g * 8 >= ncols) break;
        const int c = c_base + g * 8 + quad * 2;
        float v0 = acc[4 * g + 2 * hh], v1 = acc[4 * g + 2 * hh + 1];
        if (kF16) {
          v0 = (v0 + acc[4 * g + 2 * hh + NI / 4]) * tile_scale;
          v1 = (v1 + acc[4 * g + 2 * hh + 1 + NI / 4]) * tile_scale;
        }
        if (vec && c + 1 < p.Cout) {
          const float2 b2 = *reinterpret_cast<const float2*>(p.bias + c);
          float2 o2 = make_float2(v0 + b2.x, v1 + b2.y);
          if (res) {
            const float2 r2 = *reinterpret_cast<const float2*>(res + c);
            o2.x += r2.x;
            o2.y += r2.y;
          }
          if (p.clip) {
            o2.x = fminf(fmaxf(o2.x, -1.f), 1.f);
            o2.y = fminf(fmaxf(o2.y, -1.f), 1.f);
          }
          *reinterpret_cast<float2*>(dst + c) = o2;
          if (kF16 && p.absmax) amax = fmaxf(amax, fmaxf(finite_absf(o2.x), finite_absf(o2.y)));
          if (kF16 && want_stats) {   // stats need Cout % 16 == 0 (checked on the host): always this path
            st1[g < kStatG ? g : 0] += o2.x + o2.y;
            st2[g < kStatG ? g : 0] += o2.x * o2.x + o2.y * o2.y;
          }
        } else {
          const float vv[2] = {v0, v1};
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (c + e < p.Cout) {
              float o = vv[e] + p.bias[c + e];
              if (res) o += res[c + e];
              if (p.clip) o = fminf(fmaxf(o, -1.f), 1.f);
              dst[c + e] = o;
              if (kF16 && p.absmax) amax = fmaxf(amax, finite_absf(o));
            }
        }
      }
    }
    if constexpr (kOrdered) {
      if (want_stats) {
        // this warp's 16 pixels: add the 8 row lanes of each channel pair, then the pairs of a group, then (cpg > 8) the
        // 8-channel chunks of a group in ascending order — a fixed shuffle tree, no atomics
        float* slot = p.part + (((size_t)n * tiles_h * tiles_w + (oh0 / 8) * tiles_w + ow0 / 16) * 8 + warp) * p.groups * 2;
        float g1 = 0.f, g2 = 0.f;
#pragma unroll
        for (int g = 0; g < kStatG; ++g) {
          float s1 = st1[g], s2 = st2[g];
          st1[g] = st2[g] = 0.f;
#pragma unroll
          for (int sh = 4; sh < 32; sh <<= 1) {
            s1 += __shfl_xor_sync(0xffffffffu, s1, sh);
            s2 += __shfl_xor_sync(0xffffffffu, s2, sh);
          }
          s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
          s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
          if (cpg >= 8) {
            s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
            s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
          }
          const int c = c_base + g * 8;   // first channel of the chunk (warp-uniform)
          if (g * 8 >= ncols || c >= p.Cout) continue;
          if (cpg <= 8) {       // lanes 0 (and 2 when cpg == 4) hold the chunk's whole groups
            if (lane == 0 || (cpg == 4 && lane == 2))
              *reinterpret_cast<float2*>(slot + 2 * ((c + 2 * lane) / cpg)) = make_float2(s1, s2);
          } else {
            g1 = c % cpg ? g1 + s1 : s1;
            g2 = c % cpg ? g2 + s2 : s2;
            if ((c + 8) % cpg == 0 && lane == 0) *reinterpret_cast<float2*>(slot + 2 * (c / cpg)) = make_float2(g1, g2);
          }
        }
      }
      if (p.absmax) {   // atomicMax: the result does not depend on the order
        const unsigned m = __reduce_max_sync(0xffffffffu, __float_as_uint(amax));
        if (lane == 0 && m) atomicMax(p.absmax + n, m);
        amax = 0.f;
      }
    }
  }
  if (!kOrdered && p.stats) flush_stats();
  if (!kOrdered && kF16 && p.absmax) {
    // non-negative floats order like their bit patterns
    const unsigned m = __reduce_max_sync(0xffffffffu, __float_as_uint(amax));
    if (lane == 0 && m) atomicMax(p.absmax, m);
  }
}

typedef void (*ConvKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const ConvParams);

// the instantiated wgmma widths: bf16 (n_pass 1 / 3) BN in {16, 32, 64, 128, 256}; fp16x2 2*BN in {32, 64, ..., 256}
// the ordered instances: fp16x2 only
static ConvKernel conv_kernel_for(int NI, bool f16, bool ordered, int* variant) {
#define LWM_CONV_CASE(n, f, o, idx)             \
  if (NI == n && f16 == f && ordered == o) {    \
    *variant = idx;                             \
    return conv_wgmma_kernel<n, f, o>;          \
  }
  LWM_CONV_CASE(16, false, false, 0) LWM_CONV_CASE(32, false, false, 1) LWM_CONV_CASE(64, false, false, 2)
  LWM_CONV_CASE(128, false, false, 3) LWM_CONV_CASE(256, false, false, 4)
  LWM_CONV_CASE(32, true, false, 5) LWM_CONV_CASE(64, true, false, 6) LWM_CONV_CASE(96, true, false, 7)
  LWM_CONV_CASE(128, true, false, 8) LWM_CONV_CASE(160, true, false, 9) LWM_CONV_CASE(192, true, false, 10)
  LWM_CONV_CASE(224, true, false, 11) LWM_CONV_CASE(256, true, false, 12)
  LWM_CONV_CASE(32, true, true, 13) LWM_CONV_CASE(64, true, true, 14) LWM_CONV_CASE(96, true, true, 15)
  LWM_CONV_CASE(128, true, true, 16) LWM_CONV_CASE(160, true, true, 17) LWM_CONV_CASE(192, true, true, 18)
  LWM_CONV_CASE(224, true, true, 19) LWM_CONV_CASE(256, true, true, 20)
#undef LWM_CONV_CASE
  return nullptr;
}
constexpr int kConvVariants = 21;

}  // namespace lwm

using namespace lwm;

int lwm_vq_gn_finalize(const float* part, double* stats, int N, int P, int cols, cudaStream_t st);   // vq_elementwise.cu

// fp16x2 stacks hi|lo: the wgmma is 2*BN wide -> BN = largest multiple of 16 <= 128 dividing Cout_pad
static int f16_tile_n(int Cout_pad) {
  int BN;
  for (BN = 128; BN >= 16; BN -= 16)
    if (Cout_pad % BN == 0) break;
  return BN;
}

static int conv_launch(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                       const float* residual, float* out, int N, int Hin, int Win, int Cpad, int Ho, int Wo, int Cout,
                       int Cout_pad, int ksize, int stride, int pad, int n_pass, int clip, float w_scale_inv,
                       const float* a_scale, double* stats, unsigned* absmax, int groups, void* stream,
                       bool ordered = false, float* part = nullptr, long long part_bytes = 0) {
  if (!a_hi || !w_hi || !bias || !out) return lwm_fail(LWM_ERR_ARG, "vq_conv2d: null pointer");
  if (n_pass < 1 || n_pass > 3) return lwm_fail(LWM_ERR_ARG, "vq_conv2d: n_pass must be 1 (bf16), 2 (fp16x2) or 3 (bf16x3)");
  if (n_pass == 3 && (!a_lo || !w_lo)) return lwm_fail(LWM_ERR_ARG, "vq_conv2d: n_pass=3 needs the lo planes");
  if (Cpad % 64 || Cout_pad % 16 || Cout > Cout_pad) return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: Cpad % 64, Cout_pad % 16");
  if (Ho % 8 || Wo % 16) return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: output must tile by 8 x 16 pixels");
  if ((ksize != 1 && ksize != 3) || (stride != 1 && stride != 2)) return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: ksize 1|3, stride 1|2");
  if (stats && (groups <= 0 || groups > 64 || Cout % groups || (Cout / groups) % 4 || Cout % 16))
    return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: output statistics need Cout % 16 == 0 and (Cout/groups) % 4 == 0, groups <= 64");
  if (stats && n_pass != 2)
    return lwm_fail(LWM_ERR_ARG, "vq_conv2d: output statistics are an epilogue of the fp16x2 scheme (N tile <= 128)");
  const long long m_tiles = (long long)N * (Ho / 8) * (Wo / 16);
  if (ordered && stats) {
    // a group's channels lie in one 8-channel chunk (cpg 4) or in whole chunks of one N tile
    const int cpg = Cout / groups, bn = f16_tile_n(Cout_pad);
    if (cpg != 4 && (cpg % 8 || bn % cpg))
      return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d_f16_ordered: ordered statistics need Cout/groups == 4, or a multiple of 8 "
                                     "that divides the N tile");
    if (!part) return lwm_fail(LWM_ERR_ARG, "vq_conv2d_f16_ordered: output statistics need the workspace");
    if (part_bytes < m_tiles * 8 * groups * 2 * (long long)sizeof(float))
      return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d_f16_ordered: workspace too small (N * Ho/8 * Wo/16 * 8 * groups * 2 floats)");
  }
  if (!lwm_check_device()) return LWM_ERR_DEVICE;
  int BN = Cout_pad;
  if (n_pass == 2) {
    BN = f16_tile_n(Cout_pad);
  } else {
    if (Cout_pad > 256 && Cout_pad % 128)
      return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: Cout_pad > 256 must be a multiple of 128");
    for (BN = 256; BN > 16; BN >>= 1)      // the widest instantiated wgmma N that divides Cout_pad
      if (Cout_pad % BN == 0) break;
  }
  int variant = 0;
  const ConvKernel kern = conv_kernel_for(n_pass == 2 ? 2 * BN : BN, n_pass == 2, ordered, &variant);
  if (!kern) return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: no kernel for this N tile");
  const int taps = ksize * ksize;
  const CUtensorMapDataType dt = n_pass == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const int wrows = (n_pass == 2 ? 2 : 1);
  CUtensorMap tAh, tAl, tBh, tBl;
  {
    uint64_t dims[4] = {uint64_t(Cpad), uint64_t(Win), uint64_t(Hin), uint64_t(N)};
    uint64_t strides[3] = {uint64_t(Cpad) * 2, uint64_t(Win) * Cpad * 2, uint64_t(Hin) * Win * Cpad * 2};
    uint32_t box[4] = {64, uint32_t(16 * stride), uint32_t(8 * stride), 1};
    uint32_t es[4] = {1, uint32_t(stride), uint32_t(stride), 1};
    if (!encode_tmap(&tAh, dt, 4, a_hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, es))
      return lwm_fail(LWM_ERR_CUDA, "vq_conv2d: activation tensor map failed");
    if (n_pass == 3 &&
        !encode_tmap(&tAl, dt, 4, a_lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, es))
      return lwm_fail(LWM_ERR_CUDA, "vq_conv2d: activation (lo) tensor map failed");
  }
  {
    uint64_t dims[3] = {uint64_t(Cpad), uint64_t(Cout_pad) * wrows, uint64_t(taps)};
    uint64_t strides[2] = {uint64_t(Cpad) * 2, uint64_t(Cout_pad) * wrows * Cpad * 2};
    uint32_t box[3] = {64, uint32_t(BN * wrows), 1};
    if (!encode_tmap(&tBh, dt, 3, w_hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return lwm_fail(LWM_ERR_CUDA, "vq_conv2d: weight tensor map failed");
    if (n_pass == 3 &&
        !encode_tmap(&tBl, dt, 3, w_lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return lwm_fail(LWM_ERR_CUDA, "vq_conv2d: weight (lo) tensor map failed");
  }
  if (n_pass != 3) { tAl = tAh; tBl = tBh; }
  ConvParams p;
  p.N = N; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout; p.Cpad = Cpad;
  p.taps_w = ksize; p.taps = taps; p.stride = stride; p.pad = pad;
  p.BN = BN; p.n_tiles = Cout_pad / BN; p.n_pass = n_pass;
  p.bias = bias; p.residual = residual; p.out = out; p.clip = clip;
  p.w_scale_inv = w_scale_inv; p.a_scale = a_scale; p.stats = ordered ? nullptr : stats; p.absmax = absmax;
  p.groups = groups; p.part = ordered && stats ? part : nullptr;
  const int stage_bytes = (n_pass == 3 ? 2 : 1) * (kATile + wrows * BN * 128);
  int stages = (227 * 1024 - 2048) / stage_bytes;
  if (stages > 6) stages = 6;
  if (stages < 2) return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d: tile does not fit in shared memory");
  p.stages = stages;
  const int smem_bytes = stages * stage_bytes + 1024;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  static bool attr_set_dev[64][kConvVariants] = {};      // function attributes are per device
  if (!attr_set_dev[dev & 63][variant]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
      return lwm_fail(LWM_ERR_CUDA, "vq_conv2d: cannot raise dynamic shared memory limit");
    attr_set_dev[dev & 63][variant] = true;
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int total_tiles = N * (Ho / 8) * (Wo / 16) * p.n_tiles;
  const int grid = total_tiles < sms ? total_tiles : sms;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ordered && absmax && cudaMemsetAsync(absmax, 0, sizeof(unsigned) * N, st) != cudaSuccess)
    return lwm_fail(LWM_ERR_CUDA, "vq_conv2d_f16_ordered: memset failed");
  kern<<<grid, kConvThreads, smem_bytes, st>>>(tAh, tAl, tBh, tBl, p);
  const int status = lwm_check_launch("conv_wgmma_kernel");
  if (status != LWM_OK || !p.part) return status;
  return lwm_vq_gn_finalize(p.part, stats, N, int(m_tiles / N) * 8, groups * 2, st);
}

// a_hi/a_lo: [N,Hin,Win,Cpad] bf16 planes; w_hi/w_lo: [taps][Cout_pad][Cpad] bf16; out/residual fp32 NHWC.
extern "C" int lwm_vq_conv2d(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo,
                             const float* bias, const float* residual, float* out, int N, int Hin, int Win,
                             int Cpad, int Ho, int Wo, int Cout, int Cout_pad, int ksize, int stride, int pad,
                             int n_pass, int clip, void* stream) {
  if (n_pass != 1 && n_pass != 3) return lwm_fail(LWM_ERR_ARG, "vq_conv2d: n_pass must be 1 (bf16) or 3 (bf16x3)");
  return conv_launch(a_hi, a_lo, w_hi, w_lo, bias, residual, out, N, Hin, Win, Cpad, Ho, Wo, Cout, Cout_pad, ksize,
                     stride, pad, n_pass, clip, 1.0f, nullptr, nullptr, nullptr, 0, stream);
}

// fp16x2 mode: a [N,Hin,Win,Cpad] fp16 plane (lwm_vq_prep_f16) holding x / *a_scale (a device float; NULL = 1);
// w_stacked [taps][Cout_pad/BN][2*BN][Cpad] fp16 with
// BN = the largest multiple of 16 <= 128 that divides Cout_pad: rows [0,BN) = fp16(w / w_scale_inv), rows [BN,2BN) = fp16(w / w_scale_inv - hi).
// gn_stats_out (optional, zeroed by the caller): [N, groups, 2] double (sum, sumsq) of the OUTPUT tensor.
// absmax_out (optional, zeroed by the caller): atomicMax of the output's |value| bit patterns.
extern "C" int lwm_vq_conv2d_f16(const void* a, const float* a_scale, const void* w_stacked, const float* bias,
                                 const float* residual, float* out, double* gn_stats_out, unsigned* absmax_out,
                                 int N, int Hin, int Win, int Cpad, int Ho, int Wo, int Cout, int Cout_pad, int ksize,
                                 int stride, int pad, float w_scale_inv, int groups, int clip, void* stream) {
  if (!(w_scale_inv > 0.f)) return lwm_fail(LWM_ERR_ARG, "vq_conv2d_f16: w_scale_inv must be positive");
  return conv_launch(a, nullptr, w_stacked, nullptr, bias, residual, out, N, Hin, Win, Cpad, Ho, Wo, Cout, Cout_pad,
                     ksize, stride, pad, 2, clip, w_scale_inv, a_scale, gn_stats_out, absmax_out, groups, stream);
}

// lwm_vq_conv2d_f16 whose result does not depend on the batch or the run: a_scale [N] (one scale per image, NULL = 1),
// absmax_out [N] (zeroed here), and gn_stats_out [N, groups, 2] double summed in a fixed order from per-(tile, warp)
// partials in `workspace` (N * Ho/8 * Wo/16 * 8 * groups * 2 floats).
extern "C" int lwm_vq_conv2d_f16_ordered(const void* a, const float* a_scale, const void* w_stacked, const float* bias,
                                         const float* residual, float* out, double* gn_stats_out, float* workspace,
                                         long long workspace_bytes, unsigned* absmax_out, int N, int Hin, int Win,
                                         int Cpad, int Ho, int Wo, int Cout, int Cout_pad, int ksize, int stride,
                                         int pad, float w_scale_inv, int groups, int clip, void* stream) {
  if (!(w_scale_inv > 0.f)) return lwm_fail(LWM_ERR_ARG, "vq_conv2d_f16_ordered: w_scale_inv must be positive");
  if (N <= 0 || Hin <= 0 || Win <= 0 || Ho <= 0 || Wo <= 0 || Cout <= 0)
    return lwm_fail(LWM_ERR_SHAPE, "vq_conv2d_f16_ordered: empty tensor");
  return conv_launch(a, nullptr, w_stacked, nullptr, bias, residual, out, N, Hin, Win, Cpad, Ho, Wo, Cout, Cout_pad,
                     ksize, stride, pad, 2, clip, w_scale_inv, a_scale, gn_stats_out, absmax_out, groups, stream, true,
                     workspace, workspace_bytes);
}
