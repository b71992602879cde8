// Shared definitions for the ring-attention tile kernels (forward and backward).
#pragma once
#include "ptx.cuh"

namespace lwm {

constexpr int kHeadDim = 128;   // LWM-7B: hidden 4096 / 32 heads (lwm/llama.py:70-81)
constexpr int kTile = 128;      // rows per Q tile (forward) and keys per KV tile
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
// Logit (log2 domain) given to a masked position. The reference adds finfo(dtype).min, which
// absorbs the logit entirely in fp32, so every masked position carries the same value: a row
// whose visited keys are all masked averages them uniformly instead of producing NaN
// (SURVEY.md 8a "edge-case semantics"). A large finite constant reproduces exactly that.
constexpr float kMaskedLogit = -1.0e30f;

// Position-dependent inputs of one (q shard, kv block) step; everything is indexed by GLOBAL
// token position, as in the reference's _chunk_attention_bias (SURVEY.md Appendix A).
struct MaskParams {
  int q_pos0;            // global position of local query row 0
  int k_pos0;            // global position of local key row 0
  int causal;            // 1 <=> causal_block_size == 1 ; 0 <=> causal_block_size is None
  const float* bias;     // [B, bias_stride] additive per-key bias at global key position, or null
  long long bias_stride;
  const int* seg;        // [B, seg_stride] segment ids at global position, or null
  long long seg_stride;
};

}  // namespace lwm
