// The 8-bit KV cache format: the one place that knows how K/V rows are quantized and laid out.
//
// Layout of an 8-bit pool of `planes` (layer, k/v, row, kv head) planes, `cap` positions each:
//   codes   uint8 [planes][cap][hd]          one byte per element; read as uint32 words, element 4i+j
//                                            sits in bits 8j of word i (mx.quantize's packing, bits=8)
//   scales  bf16  [planes][cap][hd / gs]     one per group of gs consecutive elements along head_dim
//   biases  bf16  [planes][cap][hd / gs]
//
// Arithmetic (mx.quantize / mx.dequantize with bits = 8, affine mode), per group, in fp32:
//   w_max, w_min; mask = |w_min| > |w_max|
//   scale = max((w_max - w_min) / 255, 1e-7), negated unless mask
//   edge  = mask ? w_min : w_max; q0 = rint(edge / scale)
//   q0 != 0: scale = edge / q0, bias = edge;  otherwise bias = 0
//   code  = clamp(rint((w - bias) / scale), 0, 255)
//   scale and bias are rounded to bf16 only when stored (codes use the fp32 values)
// The dequantized element is bf16(scale * code + bias) with the STORED scale and bias: scale * code is
// exact in fp32 (8 + 8 significant bits), so this is one fp32 rounding of the sum, then one to bf16.  This
// rounding is this project's choice and is unpinned at the mlx boundary: MLX dequantizes in the storage dtype
// and may round scale * code to bf16 before adding the bias; its quantized_matmul folds scale and bias into
// the dot product instead.  The size of either difference is not measured.
// Divisions are IEEE (__fdiv_rn) and rint is round-half-even; the build uses no fast-math.
#pragma once
#include "common.cuh"
#include "decode.cuh"

namespace b200 {

struct KvqPlanes {
  uint8_t* codes;
  bf16* scales;
  bf16* biases;
  int gs;   // group size: 32, 64 or 128
};

// One group of gs = 32 * E elements held by one warp, E consecutive elements per lane (E <= 4).
// Returns the codes of the lane's elements and the group's fp32 scale / bias (before storage rounding).
__device__ __forceinline__ void kvq_quantize_group(const float* w, int E, uint32_t* code, float* scale_out,
                                                   float* bias_out) {
  float mx = -INFINITY, mn = INFINITY;
  #pragma unroll
  for (int e = 0; e < 4; ++e) if (e < E) {
    mx = fmaxf(mx, w[e]);
    mn = fminf(mn, w[e]);
  }
  mx = warp_max(mx);
  mn = -warp_max(-mn);
  const bool mask = fabsf(mn) > fabsf(mx);
  float scale = fmaxf(__fdiv_rn(mx - mn, 255.f), 1e-7f);
  scale = mask ? scale : -scale;
  const float edge = mask ? mn : mx;
  const float q0 = rintf(__fdiv_rn(edge, scale));
  float bias = 0.f;
  if (q0 != 0.f) {
    scale = __fdiv_rn(edge, q0);
    bias = edge;
  }
  #pragma unroll
  for (int e = 0; e < 4; ++e) if (e < E) {
    const float q = rintf(__fdiv_rn(w[e] - bias, scale));
    code[e] = (uint32_t)fminf(fmaxf(q, 0.f), 255.f);
  }
  *scale_out = scale;
  *bias_out = bias;
}

// dequantized element (fp32 value of the bf16 result) from the stored bf16 scale / bias
__device__ __forceinline__ float kvq_dequant(uint32_t code, float scale, float bias) {
  return rbf(fmaf(scale, (float)code, bias));
}

// decode attention over an 8-bit pool (kvq.cu).  kc8 / vc8: K / V planes of the bound row of this layer
// (kv head stride cap * hd codes, cap * hd / gs scales); stage_k / stage_v: bf16 planes [n_kv][cap][hd] where
// the QKV kernel left the new row at position ctx.  Quantizes the new row, appends it to the pool and attends
// over positions 0..ctx, the new one in its quantized form.
int kvq_decode_prepare(const DecodeDims& d, int cluster);
// quantize positions [pos0, pos0 + n) of `planes` bf16 planes (capacity cap) into dst (capacity dst_cap); writeback:
// replace those bf16 rows by their dequantized values
int kvq_quantize_rows(bf16* src, int cap, const KvqPlanes& dst, int dst_cap, long planes, int pos0, int n, int hd,
                      bool writeback, cudaStream_t s);
int launch_attn_q8(const DecodeDims& d, const bf16* qbuf, const KvqPlanes& kc8, const KvqPlanes& vc8,
                   const bf16* stage_k, const bf16* stage_v, bf16* out, const DecState* st, int cluster,
                   cudaStream_t s);

}  // namespace b200
