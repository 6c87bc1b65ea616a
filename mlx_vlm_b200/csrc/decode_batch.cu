// Lock-step batched decode (continuous batching, SURVEY §8 a15 / config C5): B <= 16 independent
// requests advance one token per step and share ONE stream of the weights.
//
// The reference batches rows by left-padding them to a common length inside a BatchKVCache
// (generate/ar.py:929-1390, models/cache.py:972-1201).  Here every row keeps its own length:
// the KV pool is (layer, k/v, row, kv head, capacity, head_dim), the per-row state (next token,
// cache length, rope position) lives in device arrays, and one captured CUDA graph per step
// replays unchanged while rows join and leave:
//   per layer   qkv      gemm_wt (weight-major wgmma GEMM, token tile 16, split-K partials)
//               bd_attn  finishes q/k/v from the partials (+bias, M-RoPE at the row's position,
//                        KV append at the row's length) and attends over the row's keys; on a layer
//                        whose pool is 8-bit (kv_bits=8, format kvq.cuh) the same kernel quantizes the
//                        new row, appends its codes / scales / biases and attends over the dequantized
//                        keys and values, the new row included
//               o_proj   gemm_wt partials -> finish_rows (+residual, RMSNorm)
//               gate/up  gemm_wt with the SwiGLU epilogue
//               down     gemm_wt partials -> finish_rows (+residual, next RMSNorm)
//   then        head     gemm_wt over all rows,  bd_sample: bf16 logprobs, lowest-index argmax,
//                        state update, embedding + first RMSNorm of the next step
// The weight bytes are read once per step whatever B is: B = 8 costs ~the step of B = 1.
// Rounding points: identical to the batch-1 kernels (oracle/qwen2vl.py::lm_layers_forward).
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "kvq.cuh"

namespace b200 {

namespace {

constexpr int BD_AG_MAX = 4;  // q heads per attention CTA: 4, 2 or 1 — the smallest that keeps the grid within one wave

// h[b] = embed[tok[b]];  xn[b] = RMSNorm(h[b]) * w   (the first norm of the next step)
__device__ __forceinline__ void bd_embed_norm_row(const bf16* __restrict__ embed, int tok, int H,
                                                  const bf16* __restrict__ lnw, float eps, bf16* h,
                                                  bf16* xn, float* red) {
  const int nv = H >> 3;
  float ss = 0.f;
  for (int c = threadIdx.x; c < nv; c += blockDim.x) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(embed + (long)tok * H + c * 8));
    *reinterpret_cast<uint4*>(h + c * 8) = v;
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
  }
  const float tot = block_sum(ss, red, blockDim.x >> 5);
  const float rs = 1.0f / sqrtf(tot / (float)H + eps);
  for (int c = threadIdx.x; c < nv; c += blockDim.x) {
    float f[8], w[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(embed + (long)tok * H + c * 8)), f);
    unpack8(__ldg(reinterpret_cast<const uint4*>(lnw + c * 8)), w);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = rbf(rbf(f[j] * rs) * w[j]);
    uint4 o;
    o.x = pack2(f[0], f[1]); o.y = pack2(f[2], f[3]); o.z = pack2(f[4], f[5]); o.w = pack2(f[6], f[7]);
    *reinterpret_cast<uint4*>(xn + c * 8) = o;
  }
}

__global__ void __launch_bounds__(256) bd_begin_kernel(const int* __restrict__ tok, const bf16* __restrict__ embed,
                                                       int H, const bf16* __restrict__ lnw, float eps,
                                                       bf16* __restrict__ h, bf16* __restrict__ xn) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  bd_embed_norm_row(embed, tok[b], H, lnw, eps, h + (long)b * H, xn + (long)b * H, red);
}

// ---- attention of one (row, kv head, q-head part): finishes q/k/v from the qkv partials ----------
struct BdAttnP {
  const float* P;     // [S][B][QKV] fp32 split-K partials of the qkv GEMM
  int S, B, QKV;
  const bf16* bias;   // [QKV]
  const float* inv_freq;
  const int *ctx, *pos;
  bf16* kv;           // layer's K plane of row 0
  long v_off;         // elements from the K plane to the V plane
  long row_stride;    // elements between rows
  bf16* out;          // [B][n_heads*hd]
  int n_heads, n_kv, cap, hsplit;
  float scale_bf;
  const bf16 *qn, *kn;  // Qwen3-VL q_norm / k_norm weights of the layer (nullptr: no q/k norm)
  float eps;
  // 8-bit layer (Q8 variant): the layer's K codes / scales / biases of row 0.  Codes sit at the same element
  // offsets as the bf16 planes (row_stride, v_off); scales and biases at those offsets / gs.
  uint8_t* q8c;
  bf16 *q8s, *q8b;
  int gs;
};

// 8 codes -> their dequantized values (bf16 exactly: kvq_dequant rounds), packed as 8 bf16
__device__ __forceinline__ uint4 bd_q8_unpack8(uint2 w, float s, float b) {
  float f[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    f[e] = kvq_dequant((w.x >> (8 * e)) & 0xffu, s, b);
    f[4 + e] = kvq_dequant((w.y >> (8 * e)) & 0xffu, s, b);
  }
  uint4 o;
  o.x = pack2(f[0], f[1]); o.y = pack2(f[2], f[3]); o.z = pack2(f[4], f[5]); o.w = pack2(f[6], f[7]);
  return o;
}

// key j of an 8-bit K plane (HD codes, HD / gs scales per position), dequantized into the bf16 layout of a key row
template <int HD>
__device__ __forceinline__ void bd_q8_key(const uint8_t* codes, const bf16* sc, const bf16* bi, int gs, long j,
                                          uint4 (&kv)[HD / 8]) {
  constexpr int NG = HD / 32;   // most groups per position (gs = 32)
  const int ng = HD / gs;
  float s[NG], b[NG];
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    s[g] = g < ng ? bf2f(__ldcg(sc + j * ng + g)) : 0.f;
    b[g] = g < ng ? bf2f(__ldcg(bi + j * ng + g)) : 0.f;
  }
  const uint2* c = reinterpret_cast<const uint2*>(codes + j * HD);
#pragma unroll
  for (int ch = 0; ch < HD / 8; ++ch) {
    const int g = ch * 8 / gs;
    float sg = s[0], bg = b[0];
#pragma unroll
    for (int t = 1; t < NG; ++t)
      if (g == t) { sg = s[t]; bg = b[t]; }
    kv[ch] = bd_q8_unpack8(__ldcg(c + ch), sg, bg);
  }
}

// the 8 * NV codes of dims [d0, d0 + 8 * NV) of value j of an 8-bit V plane (NV = 1: in .x / .y) and the scale / bias
// of their quantization group (8 * NV divides gs); dequantized where they are used
template <int HD, int NV>
__device__ __forceinline__ void bd_q8_val(const uint8_t* codes, const bf16* sc, const bf16* bi, int gs, long j, int d0,
                                          uint4& c, float& s, float& b) {
  const long si = j * (HD / gs) + d0 / gs;
  s = bf2f(__ldcg(sc + si));
  b = bf2f(__ldcg(bi + si));
  if constexpr (NV == 2) {
    c = __ldcg(reinterpret_cast<const uint4*>(codes + j * HD + d0));
  } else {
    const uint2 w = __ldcg(reinterpret_cast<const uint2*>(codes + j * HD + d0));
    c = make_uint4(w.x, w.y, 0u, 0u);
  }
}

template <int HD, int AG, bool Q8>
__global__ void __launch_bounds__(256) bd_attn_kernel(const BdAttnP p) {
  pdl_launch_dependents();
  extern __shared__ __align__(16) uint8_t bd_sm[];
  constexpr int NCH = HD / 8, half = HD / 2;
  constexpr int SEG = HD / 8;   // dims per lane in the P.V phase (lane = key sub-index x dim segment)
  constexpr int NV = SEG / 8;   // 16-byte vectors per lane and key
  constexpr int VU = 8;         // key trips in flight per warp in the P.V phase (32 keys)
  constexpr int PMAX = 12;      // split-K partials summed with all loads in flight
  float* qs = reinterpret_cast<float*>(bd_sm);  // [AG][HD] q * scale (rotated)
  float* kn = qs + AG * HD;                     // [HD] new key (rotated)
  float* vn = kn + HD;                          // [HD] new value
  float* sc = vn + HD;                          // [AG][cap]
  float* red = sc + (long)AG * p.cap;           // [8][AG*HD]
  __shared__ float s_m[8][AG], s_l[8][AG];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.y;
  const int Gall = p.n_heads / p.n_kv;
  const int Gc = (Gall + p.hsplit - 1) / p.hsplit;
  const int kvh = blockIdx.x / p.hsplit, part = blockIdx.x % p.hsplit;
  const int G = min(Gc, Gall - part * Gc);
  const int h0 = kvh * Gall + part * Gc;
  const long plane0 = (long)row * p.row_stride + (long)kvh * p.cap * HD;   // element offset of this row's K plane
  bf16* kb = Q8 ? nullptr : p.kv + plane0;
  bf16* vb = Q8 ? nullptr : kb + p.v_off;
  // Q8: codes at the same element offsets, scales / biases at offsets / gs
  const uint8_t* kq = Q8 ? p.q8c + plane0 : nullptr;
  const uint8_t* vq = Q8 ? kq + p.v_off : nullptr;
  const bf16* kqs = Q8 ? p.q8s + plane0 / p.gs : nullptr;
  const bf16* kqb = Q8 ? p.q8b + plane0 / p.gs : nullptr;
  const bf16* vqs = Q8 ? kqs + p.v_off / p.gs : nullptr;
  const bf16* vqb = Q8 ? kqb + p.v_off / p.gs : nullptr;
  pdl_wait();
  const int ctx = p.ctx[row], pos = p.pos[row];
  const int nkeys = ctx + 1;
  // Every dependent global round trip costs ~1 us here, so the requests are issued as early as their
  // addresses are known: the first block of cached keys (one row per lane) goes out BEFORE the
  // split-K partials of q/k/v are summed, the first block of values before the softmax.
  uint4 kfirst[NCH];
  {
    // (the 8-bit variant loads its first keys in the score loop: holding them dequantized across the sums spills)
    if constexpr (!Q8) {
      const int j = warp * 32 + lane;
      const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * HD);
#pragma unroll
      for (int c = 0; c < NCH; ++c) kfirst[c] = (j < ctx) ? __ldcg(kr + c) : make_uint4(0, 0, 0, 0);
    }
  }
  // ---- finish q (G heads), k, v of this step: sum of the split-K partials + bias, one rounding ----
  for (int i = threadIdx.x; i < (G + 2) * HD; i += 256) {
    const int slot = i / HD, j = i % HD;
    const int n = (slot < G ? (h0 + slot) : (slot == G ? p.n_heads + kvh : p.n_heads + p.n_kv + kvh)) * HD + j;
    float a = 0.f;
    for (int s0 = 0; s0 < p.S; s0 += PMAX) {
      float v[PMAX];
#pragma unroll
      for (int u = 0; u < PMAX; ++u)
        v[u] = (s0 + u < p.S) ? __ldcg(p.P + ((long)(s0 + u) * p.B + row) * p.QKV + n) : 0.f;
#pragma unroll
      for (int u = 0; u < PMAX; ++u) a += v[u];
    }
    a = rbf(a + bf2f(p.bias[n]));
    (slot < G ? qs + slot * HD : (slot == G ? kn : vn))[j] = a;
  }
  __syncthreads();
  if (p.qn) {  // q_norm / k_norm (qwen3_vl/language.py:84-89) before the rotary, one warp per head
    for (int slot = warp; slot <= G; slot += 8) {
      float* v = slot < G ? qs + slot * HD : kn;
      float x[HD / 32];
#pragma unroll
      for (int u = 0; u < HD / 32; ++u) x[u] = v[lane + 32 * u];
      warp_head_rms<HD / 32>(x, slot < G ? p.qn : p.kn, p.eps);
#pragma unroll
      for (int u = 0; u < HD / 32; ++u) v[lane + 32 * u] = x[u];
    }
    __syncthreads();
  }
  // M-RoPE at a decode position: the three axes carry the same position (language.py:476-509)
  for (int i = threadIdx.x; i < (G + 1) * half; i += 256) {
    const int slot = i / half, j = i % half;
    float* v = slot < G ? qs + slot * HD : kn;
    const float y1 = v[j], y2 = v[j + half];
    const float ang = (float)pos * p.inv_freq[j];
    const float c = rbf(cosf(ang)), sn = rbf(sinf(ang));
    float o1 = rbf(rbf(y1 * c) + rbf((-y2) * sn));
    float o2 = rbf(rbf(y2 * c) + rbf(y1 * sn));
    if (slot < G) {
      o1 = rbf(o1 * p.scale_bf);
      o2 = rbf(o2 * p.scale_bf);
    }
    v[j] = o1;
    v[j + half] = o2;
  }
  for (int i = threadIdx.x + G * HD; i < AG * HD; i += 256) qs[i] = 0.f;
  __syncthreads();
  if constexpr (Q8) {
    // quantize the new K and V row (warp w < 2 * ng: group w % ng of K, then of V) with the format's own
    // arithmetic, append it (one CTA per kv head), and attend to its dequantized values from here on
    const int ng = HD / p.gs, E = p.gs >> 5;
    if (warp < 2 * ng) {
      const int side = warp / ng, g = warp % ng;
      float* src = (side ? vn : kn) + g * p.gs + lane * E;
      float w[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) w[e] = e < E ? src[e] : 0.f;
      uint32_t code[4];
      float scale, bias;
      kvq_quantize_group(w, E, code, &scale, &bias);
      const float sb = rbf(scale), bb = rbf(bias);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (e < E) src[e] = kvq_dequant(code[e], sb, bb);
      if (part == 0) {
        const long at = plane0 + (side ? p.v_off : 0) + (long)ctx * HD;
        uint8_t* c = p.q8c + at + g * p.gs + lane * E;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (e < E) c[e] = (uint8_t)code[e];
        if (lane == 0) {
          p.q8s[at / p.gs + g] = f2bf(scale);
          p.q8b[at / p.gs + g] = f2bf(bias);
        }
      }
    }
    __syncthreads();
  } else if (part == 0) {  // append the new position to the row's cache (one CTA per kv head)
    for (int i = threadIdx.x; i < HD; i += 256) {
      kb[(long)ctx * HD + i] = f2bf(kn[i]);
      vb[(long)ctx * HD + i] = f2bf(vn[i]);
    }
  }
  // ---- scores: lane <-> key; cached keys from global, the new key from shared memory ----
  float lm[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) lm[g] = -INFINITY;
  for (int j0 = warp * 32; j0 < nkeys; j0 += 256) {
    const int j = j0 + lane;
    uint4 kv[NCH];
    if (!Q8 && j0 == warp * 32) {
#pragma unroll
      for (int c = 0; c < NCH; ++c) kv[c] = kfirst[c];
    } else if (j < ctx) {
      if constexpr (Q8) {
        bd_q8_key<HD>(kq, kqs, kqb, p.gs, j, kv);
      } else {
        const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * HD);
#pragma unroll
        for (int c = 0; c < NCH; ++c) kv[c] = __ldcg(kr + c);
      }
    }
    if (j < nkeys) {
      if (j == ctx) {
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          kv[c].x = pack2(kn[c * 8 + 0], kn[c * 8 + 1]); kv[c].y = pack2(kn[c * 8 + 2], kn[c * 8 + 3]);
          kv[c].z = pack2(kn[c * 8 + 4], kn[c * 8 + 5]); kv[c].w = pack2(kn[c * 8 + 6], kn[c * 8 + 7]);
        }
      }
      float s[AG][2];
#pragma unroll
      for (int g = 0; g < AG; ++g) s[g][0] = s[g][1] = 0.f;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        float kf[8];
        unpack8(kv[c], kf);
#pragma unroll
        for (int g = 0; g < AG; ++g) {
          const float4 a = *reinterpret_cast<const float4*>(qs + g * HD + c * 8);
          const float4 b = *reinterpret_cast<const float4*>(qs + g * HD + c * 8 + 4);
          s[g][0] = fmaf(a.x, kf[0], fmaf(a.y, kf[1], fmaf(a.z, kf[2], fmaf(a.w, kf[3], s[g][0]))));
          s[g][1] = fmaf(b.x, kf[4], fmaf(b.y, kf[5], fmaf(b.z, kf[6], fmaf(b.w, kf[7], s[g][1]))));
        }
      }
#pragma unroll
      for (int g = 0; g < AG; ++g) {
        const float r = rbf(s[g][0] + s[g][1]);
        sc[(long)g * p.cap + j] = r;
        lm[g] = fmaxf(lm[g], r);
      }
    }
  }
  // first block of values: warp w, trip q, key = 32 * w + 4 * q + ksub; lane = (ksub, dim segment)
  const int seg = lane & 7, ksub = lane >> 3;
  static_assert(NV <= 2, "one 16-byte code word per lane and key");
  uint4 vfirst[VU][NV];
  uint4 vfc[VU];            // 8-bit variant: codes and group scale / bias of the first block of values
  float vfs[VU], vfb[VU];
#pragma unroll
  for (int q = 0; q < VU; ++q) {
    const int j = warp * 32 + q * 4 + ksub;
    if constexpr (Q8) {
      if (j < ctx) bd_q8_val<HD, NV>(vq, vqs, vqb, p.gs, j, seg * SEG, vfc[q], vfs[q], vfb[q]);
    } else {
#pragma unroll
      for (int v = 0; v < NV; ++v)
        vfirst[q][v] = (j < ctx) ? __ldcg(reinterpret_cast<const uint4*>(vb + (long)j * HD + seg * SEG + v * 8))
                                 : make_uint4(0, 0, 0, 0);
    }
  }
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    lm[g] = warp_max(lm[g]);
    if (lane == 0) s_m[warp][g] = lm[g];
  }
  __syncthreads();
  float M[AG], ls[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    float m = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) m = fmaxf(m, s_m[w][g]);
    M[g] = m;
    ls[g] = 0.f;
  }
  for (int j = threadIdx.x; j < nkeys; j += 256) {
#pragma unroll
    for (int g = 0; g < AG; ++g) {
      const float e = expf(sc[(long)g * p.cap + j] - M[g]);
      sc[(long)g * p.cap + j] = e;
      ls[g] += e;
    }
  }
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    ls[g] = warp_sum(ls[g]);
    if (lane == 0) s_l[warp][g] = ls[g];
  }
  __syncthreads();
  float L[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    float l = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) l += s_l[w][g];
    L[g] = l;
  }
  for (int j = threadIdx.x; j < nkeys; j += 256) {
#pragma unroll
    for (int g = 0; g < AG; ++g) sc[(long)g * p.cap + j] = rbf(sc[(long)g * p.cap + j] / L[g]);
  }
  __syncthreads();
  // ---- P.V: 256 keys per CTA iteration, 8 x NV 16-byte loads in flight per lane ----
  float acc[AG][SEG];
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int e = 0; e < SEG; ++e) acc[g][e] = 0.f;
  for (int j0 = 0; j0 < nkeys; j0 += 256) {
    uint4 vv[VU][NV];
    uint4 vc[VU];
    float vs[VU], vbi[VU];
#pragma unroll
    for (int q = 0; q < VU; ++q) {
      const int j = j0 + warp * 32 + q * 4 + ksub;
      if constexpr (Q8) {
        if (j0 == 0) {
          vc[q] = vfc[q]; vs[q] = vfs[q]; vbi[q] = vfb[q];
        } else if (j < ctx) {
          bd_q8_val<HD, NV>(vq, vqs, vqb, p.gs, j, seg * SEG, vc[q], vs[q], vbi[q]);
        }
      } else {
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          if (j0 == 0) vv[q][v] = vfirst[q][v];
          else vv[q][v] = (j < ctx) ? __ldcg(reinterpret_cast<const uint4*>(vb + (long)j * HD + seg * SEG + v * 8))
                                    : make_uint4(0, 0, 0, 0);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < VU; ++q) {
      const int j = j0 + warp * 32 + q * 4 + ksub;
      if (j < nkeys) {
        float pj[AG];
#pragma unroll
        for (int g = 0; g < AG; ++g) pj[g] = sc[(long)g * p.cap + j];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          float vf[8];
          if (j == ctx) {
#pragma unroll
            for (int e = 0; e < 8; ++e) vf[e] = rbf(vn[seg * SEG + v * 8 + e]);
          } else if constexpr (Q8) {
            const uint32_t w0 = v ? vc[q].z : vc[q].x, w1 = v ? vc[q].w : vc[q].y;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              vf[e] = kvq_dequant((w0 >> (8 * e)) & 0xffu, vs[q], vbi[q]);
              vf[4 + e] = kvq_dequant((w1 >> (8 * e)) & 0xffu, vs[q], vbi[q]);
            }
          } else {
            unpack8(vv[q][v], vf);
          }
#pragma unroll
          for (int g = 0; g < AG; ++g)
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[g][v * 8 + e] = fmaf(pj[g], vf[e], acc[g][v * 8 + e]);
        }
      }
    }
  }
  // sum over the 4 key sub-indices of the warp, then over the 8 warps through shared memory
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int e = 0; e < SEG; ++e) {
      float a = acc[g][e];
      a += __shfl_xor_sync(0xffffffffu, a, 8);
      a += __shfl_xor_sync(0xffffffffu, a, 16);
      if (ksub == 0) red[((long)warp * AG + g) * HD + seg * SEG + e] = a;
    }
  __syncthreads();
  bf16* orow = p.out + (long)row * p.n_heads * HD + (long)h0 * HD;
  for (int i = threadIdx.x; i < G * HD; i += 256) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[(long)w * AG * HD + i];
    orow[i] = f2bf(s);
  }
}

// ---- sampler + state update + next embedding, one CTA per row ------------------------------------
struct BdSampleP {
  const bf16* logits;  // [B][ldv]
  bf16* logprobs;      // [B][ldv] or nullptr
  int V, ldv, H;
  int *tok, *ctx, *pos, *n_out;
  const int* active;
  int* token_log;      // [log_cap][max_b]
  float* lp_log;       // [log_cap][max_b]
  int log_cap, max_b;
  const bf16* embed;
  const bf16* ln0;     // first RMSNorm weight
  float eps;
  bf16 *h, *xn;
};

__global__ void __launch_bounds__(1024) bd_sample_kernel(const BdSampleP p) {
  pdl_launch_dependents();
  __shared__ float red[32];
  __shared__ float2 stat[32];
  __shared__ unsigned long long keys[32];
  __shared__ float s_lse;
  __shared__ int s_tok;
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  // rows are ldv = round8(V) apart; the tail [V, ldv) holds -inf (preset once, never written)
  const bf16* lg = p.logits + (long)b * p.ldv;
  const int nv = p.ldv >> 3;
  // logsumexp over the bf16 logits (fp32), then logprobs = bf16(logit - bf16(lse)) (ar.py:368)
  float m = -INFINITY, l = 0.f;
  for (int c = threadIdx.x; c < nv; c += 1024) {
    float f[8];
    unpack8(__ldcg(reinterpret_cast<const uint4*>(lg + c * 8)), f);
    float cm = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) cm = fmaxf(cm, f[j]);
    const float mn = fmaxf(m, cm);
    float add = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) add += expf(f[j] - mn);
    l = l * expf(m - mn) + add;
    m = mn;
  }
  {
    const float wm = warp_max(m);
    const float wl = warp_sum(l > 0.f ? l * expf(m - wm) : 0.f);
    if (lane == 0) stat[warp] = make_float2(wm, wl);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = -INFINITY;
    for (int w = 0; w < 32; ++w) M = fmaxf(M, stat[w].x);
    float L = 0.f;
    for (int w = 0; w < 32; ++w)
      if (stat[w].y > 0.f) L += stat[w].y * expf(stat[w].x - M);
    s_lse = rbf(M + logf(L));
  }
  __syncthreads();
  const float lse = s_lse;
  unsigned long long best = 0ull;
  for (int c = threadIdx.x; c < nv; c += 1024) {
    float f[8], o[8];
    unpack8(__ldcg(reinterpret_cast<const uint4*>(lg + c * 8)), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] = rbf(f[j] - lse);
      const unsigned long long key =
          ((unsigned long long)orderable(o[j]) << 32) | (0xFFFFFFFFu - (uint32_t)(c * 8 + j));
      best = key > best ? key : best;
    }
    if (p.logprobs) {
      uint4 ov;
      ov.x = pack2(o[0], o[1]); ov.y = pack2(o[2], o[3]); ov.z = pack2(o[4], o[5]); ov.w = pack2(o[6], o[7]);
      *reinterpret_cast<uint4*>(p.logprobs + (long)b * p.ldv + c * 8) = ov;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if (lane == 0) keys[warp] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long k = 0ull;
    for (int w = 0; w < 32; ++w) k = keys[w] > k ? keys[w] : k;
    const int tok = (int)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull));
    const uint32_t ob = (uint32_t)(k >> 32);
    const uint32_t fb = (ob & 0x80000000u) ? (ob & 0x7FFFFFFFu) : ~ob;
    const int n = p.n_out[b];
    p.token_log[(long)(n % p.log_cap) * p.max_b + b] = tok;
    p.lp_log[(long)(n % p.log_cap) * p.max_b + b] = __uint_as_float(fb);
    p.n_out[b] = n + 1;
    if (p.active[b]) {  // a finished row keeps recomputing its last position (its slot is dead)
      p.tok[b] = tok;
      p.ctx[b] += 1;
      p.pos[b] += 1;
    }
    s_tok = p.active[b] ? tok : p.tok[b];
  }
  __syncthreads();
  bd_embed_norm_row(p.embed, s_tok, p.H, p.ln0, p.eps, p.h + (long)b * p.H, p.xn + (long)b * p.H, red);
}

// ---- per-row logits processors (sample_utils.make_logits_processors), one CTA per row -------------------------------
// Runs between the head and bd_sample, in place on the step's bf16 logits, only when some row has processors.  First
// the step's input token joins the row's history (ar.py:1070-1074), then in the order make_logits_processors returns
// them: logit bias, repetition, presence, frequency.  Each is a gather of the current values, then a scatter; a
// token that occurs several times in a window writes the same value several times (penalised once).  Rounding
// points are those of the torch ops: bias bf16(x + v); repetition bf16(x * p) for x < 0 else bf16(x * fp32(1 / p))
// (the reciprocal of a division by a scalar); presence bf16(x - p); frequency bf16(x - sum) with sum the fp32
// accumulation of p once per occurrence.
struct BdProcsP {
  bf16* logits;
  int ldv, V;   // ids outside [0, V) in a history or a bias list are skipped
  const int *tok, *active;
  BdProcs pr;
};

__global__ void __launch_bounds__(1024) bd_procs_kernel(const BdProcsP p) {
  __shared__ int win[BD_HIST_MAX];
  const int b = blockIdx.x, t = threadIdx.x;
  pdl_wait();
  const int* par = p.pr.params + b * BD_PROC_PARAMS;
  const int flags = par[0];
  if (flags == 0) return;
  const float* pen = p.pr.penalties + b * BD_PROC_PARAMS;
  bf16* lg = p.logits + (long)b * p.ldv;
  int* hist = p.pr.hist + (long)b * p.pr.hist_cap;
  const int cap = p.pr.hist_cap;
  int len = p.pr.hist_len[b];
  if (p.active[b]) {
    if (t == 0) {
      hist[len % cap] = p.tok[b];
      p.pr.hist_len[b] = len + 1;
    }
    len += 1;
  }
  __syncthreads();
  // the last W tokens of the history (W = the widest window in use), oldest first
  int W = 0;
  if (flags & BD_PROC_REP) W = max(W, par[1]);
  if (flags & BD_PROC_PRES) W = max(W, par[2]);
  if (flags & BD_PROC_FREQ) W = max(W, par[3]);
  W = min(W, min(len, cap));
  if (t < W) {
    const int id = hist[(len - W + t) % cap];
    win[t] = (id >= 0 && id < p.V) ? id : -1;
  }
  if (flags & BD_PROC_BIAS) {
    const int nb = par[4];
    const int* ids = p.pr.bias_ids + (long)b * p.pr.bias_cap;
    const float* vals = p.pr.bias_vals + (long)b * p.pr.bias_cap;
    for (int i = t; i < nb; i += blockDim.x)
      if (ids[i] >= 0 && ids[i] < p.V) lg[ids[i]] = f2bf(bf2f(lg[ids[i]]) + vals[i]);
  }
  __syncthreads();
  if (flags & BD_PROC_REP) {
    const int w0 = W - min(par[1], W);
    const int id = (t >= w0 && t < W) ? win[t] : -1;
    const float x = id >= 0 ? bf2f(lg[id]) : 0.f;
    __syncthreads();
    if (id >= 0) lg[id] = f2bf(x < 0.f ? x * pen[0] : x * pen[1]);
    __syncthreads();
  }
  if (flags & BD_PROC_PRES) {
    const int w0 = W - min(par[2], W);
    const int id = (t >= w0 && t < W) ? win[t] : -1;
    const float x = id >= 0 ? bf2f(lg[id]) : 0.f;
    __syncthreads();
    if (id >= 0) lg[id] = f2bf(x - pen[2]);
    __syncthreads();
  }
  if (flags & BD_PROC_FREQ) {
    const int w0 = W - min(par[3], W);
    const int id = (t >= w0 && t < W) ? win[t] : -1;
    float x = 0.f, sub = 0.f;
    if (id >= 0) {
      x = bf2f(lg[id]);
      for (int j = w0; j < W; ++j)
        if (win[j] == id) sub += pen[3];
    }
    __syncthreads();
    if (id >= 0) lg[id] = f2bf(x - sub);
  }
}

// ---- top-k logprobs: lower token id first among equal logprobs ------------------------------------------------------
// Keys (orderable logprob << 32 | ~id) are unique per token, so "largest key" is the order asked for.  Part kernel: one
// CTA per (slice of BD_TOPK_SLICE tokens, row) picks its k largest keys in k rounds over shared memory; merge kernel:
// one CTA per row ranks the slices' candidates.
__global__ void __launch_bounds__(256) bd_topk_part_kernel(const bf16* __restrict__ lp, int ldv, int V, int k,
                                                           unsigned long long* __restrict__ cand) {
  __shared__ uint32_t key[BD_TOPK_SLICE];
  __shared__ unsigned long long red[8];
  const int s = blockIdx.x, b = blockIdx.y, S = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  const int base = s * BD_TOPK_SLICE, n = min(BD_TOPK_SLICE, V - base);
  for (int i = threadIdx.x; i < n; i += 256) key[i] = orderable(bf2f(lp[(long)b * ldv + base + i]));
  __syncthreads();
  unsigned long long prev = ~0ull;
  for (int r = 0; r < k; ++r) {
    unsigned long long best = 0ull;
    for (int i = threadIdx.x; i < n; i += 256) {
      const unsigned long long kk = ((unsigned long long)key[i] << 32) | (0xFFFFFFFFu - (uint32_t)(base + i));
      if (kk < prev && kk > best) best = kk;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if (lane == 0) red[warp] = best;
    __syncthreads();
    best = 0ull;
#pragma unroll
    for (int w = 0; w < 8; ++w) best = red[w] > best ? red[w] : best;
    __syncthreads();
    if (threadIdx.x == 0) cand[((long)b * S + s) * k + r] = best;
    prev = best;
  }
}

__global__ void __launch_bounds__(256) bd_topk_merge_kernel(const unsigned long long* __restrict__ cand, int S, int k,
                                                            const int* __restrict__ n_out, int log_cap, int max_b,
                                                            int* __restrict__ ids_log, float* __restrict__ lp_log) {
  __shared__ unsigned long long c[BD_TOPK_CAND_MAX];
  const int b = blockIdx.x, n = S * k;
  pdl_wait();
  for (int i = threadIdx.x; i < n; i += 256) c[i] = cand[(long)b * n + i];
  __syncthreads();
  const long at = ((long)(n_out ? (n_out[b] - 1) % log_cap : 0) * max_b + b) * BD_TOPK_MAX;   // no log: [B][20]
  for (int i = threadIdx.x; i < n; i += 256) {
    const unsigned long long kk = c[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += c[j] > kk;
    if (rank < k) {
      const uint32_t ob = (uint32_t)(kk >> 32);
      ids_log[at + rank] = (int)(0xFFFFFFFFu - (uint32_t)(kk & 0xFFFFFFFFull));
      lp_log[at + rank] = __uint_as_float((ob & 0x80000000u) ? (ob & 0x7FFFFFFFu) : ~ob);
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
struct BatchDecoder {
  int max_b = 0, B = 0;
  int log_cap = 4096;
  int ldv = 0;  // row stride of logits / logprobs: vocab rounded up to 8
  int *tok = nullptr, *ctx = nullptr, *pos = nullptr, *active = nullptr, *n_out = nullptr;
  int* token_log = nullptr;
  float* lp_log = nullptr;
  bf16 *h = nullptr, *xn = nullptr, *qkv_dummy = nullptr, *att = nullptr, *act = nullptr, *logits = nullptr,
       *logprobs = nullptr;
  float* partial = nullptr;
  long partial_bytes = 0;
  int* stage_host = nullptr;  // pinned [4][max_b]
  cudaGraphExec_t gexec = nullptr;
  const void* graph_kv = nullptr;
  const void* graph_q8 = nullptr;
  int graph_q8_layers = 0, graph_gs = 0;
  int graph_B = 0, graph_cap = 0, graph_lp = 0;
  long steps_done = 0;
  bool want_logprobs = false;
  BdProcs procs = {}, graph_procs = {};
  unsigned long long* topk_cand = nullptr;  // [max_b][slices][k] keys of the top-k part kernel
  int* topk_ids = nullptr;                  // [log_cap][max_b][BD_TOPK_MAX]
  float* topk_lp = nullptr;
};

static bool bd_same_procs(const BdProcs& a, const BdProcs& b) {
  return a.params == b.params && a.penalties == b.penalties && a.bias_ids == b.bias_ids &&
         a.bias_vals == b.bias_vals && a.bias_cap == b.bias_cap && a.hist == b.hist && a.hist_len == b.hist_len &&
         a.hist_cap == b.hist_cap && a.top_k == b.top_k;
}

static void bd_free(BatchDecoder* d) {
  if (!d) return;
  if (d->gexec) cudaGraphExecDestroy(d->gexec);
  for (void* p : {(void*)d->tok, (void*)d->ctx, (void*)d->pos, (void*)d->active, (void*)d->n_out, (void*)d->token_log,
                  (void*)d->lp_log, (void*)d->h, (void*)d->xn, (void*)d->att, (void*)d->act, (void*)d->logits,
                  (void*)d->logprobs, (void*)d->partial, (void*)d->topk_cand, (void*)d->topk_ids, (void*)d->topk_lp})
    if (p) cudaFree(p);
  if (d->stage_host) cudaFreeHost(d->stage_host);
  delete d;
}

void batch_decoder_destroy(void* d) { bd_free(reinterpret_cast<BatchDecoder*>(d)); }

static int bd_alloc(BatchDecoder* d, const BdModel& m, int max_b) {
  const DecodeDims& dd = m.d;
  const long QH = (long)dd.n_heads * dd.hd;
  d->max_b = max_b;
  B200_CUDA(cudaMalloc(&d->tok, max_b * 4)); B200_CUDA(cudaMalloc(&d->ctx, max_b * 4));
  B200_CUDA(cudaMalloc(&d->pos, max_b * 4)); B200_CUDA(cudaMalloc(&d->active, max_b * 4));
  B200_CUDA(cudaMalloc(&d->n_out, max_b * 4));
  B200_CUDA(cudaMemset(d->n_out, 0, max_b * 4));
  B200_CUDA(cudaMalloc(&d->token_log, (size_t)d->log_cap * max_b * 4));
  B200_CUDA(cudaMalloc(&d->lp_log, (size_t)d->log_cap * max_b * 4));
  B200_CUDA(cudaMalloc(&d->h, (size_t)max_b * dd.hidden * 2)); B200_CUDA(cudaMalloc(&d->xn, (size_t)max_b * dd.hidden * 2));
  B200_CUDA(cudaMalloc(&d->att, (size_t)max_b * QH * 2)); B200_CUDA(cudaMalloc(&d->act, (size_t)max_b * dd.inter * 2));
  d->ldv = (dd.vocab + 7) & ~7;
  B200_CUDA(cudaMalloc(&d->logits, (size_t)max_b * d->ldv * 2));
  B200_CUDA(cudaMalloc(&d->logprobs, (size_t)max_b * d->ldv * 2));
  {
    std::vector<uint16_t> ninf((size_t)max_b * d->ldv, (uint16_t)0xFF80);  // bf16 -inf
    B200_CUDA(cudaMemcpy(d->logits, ninf.data(), ninf.size() * 2, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemcpy(d->logprobs, ninf.data(), ninf.size() * 2, cudaMemcpyHostToDevice));
  }
  // split-K partials: at most ~sm_count CTAs x 128 rows x 16 tokens of fp32 per GEMM, x2 margin
  d->partial_bytes = 64L << 20;
  B200_CUDA(cudaMalloc(&d->partial, d->partial_bytes));
  B200_CUDA(cudaMallocHost(&d->stage_host, (size_t)4 * max_b * 4));
  return B200_OK;
}

static size_t bd_attn_smem(const DecodeDims& d, int ag) {
  return ((size_t)(ag + 2) * d.hd + (size_t)ag * d.cap + (size_t)8 * ag * d.hd) * 4;
}

// q heads per attention CTA: the latency chain of a CTA (partials -> rope -> keys -> softmax -> values) does not
// shrink with fewer heads, its arithmetic does; so use as many CTAs as fit one wave of the SMs
static int bd_attn_heads_per_cta(const DecodeDims& d, int B, int sm_count) {
  const int Gall = d.n_heads / d.n_kv;
  for (int ag : {1, 2, 4})
    if ((long)d.n_kv * ((Gall + ag - 1) / ag) * B <= sm_count) return ag;
  return BD_AG_MAX;
}

template <int HD, bool Q8>
static int bd_attn_launch(int ag, dim3 grid, size_t smem, cudaStream_t s, const BdAttnP& ap) {
  B200_CUDA(launch(ag == 1 ? bd_attn_kernel<HD, 1, Q8> : ag == 2 ? bd_attn_kernel<HD, 2, Q8> : bd_attn_kernel<HD, 4, Q8>,
                   grid, dim3(256), smem, s, PDL_LAUNCH, ap));
  return B200_OK;
}

static int bd_attn_dispatch(const DecodeDims& d, int ag, dim3 grid, cudaStream_t s, const BdAttnP& ap, bool q8) {
  const size_t smem = bd_attn_smem(d, ag);
  if (d.hd == 128) return q8 ? bd_attn_launch<128, true>(ag, grid, smem, s, ap) : bd_attn_launch<128, false>(ag, grid, smem, s, ap);
  return q8 ? bd_attn_launch<64, true>(ag, grid, smem, s, ap) : bd_attn_launch<64, false>(ag, grid, smem, s, ap);
}

static int bd_set_smem_attrs() {
  const void* ks[] = {(const void*)bd_attn_kernel<128, 1, false>, (const void*)bd_attn_kernel<128, 2, false>,
                      (const void*)bd_attn_kernel<128, 4, false>, (const void*)bd_attn_kernel<64, 1, false>,
                      (const void*)bd_attn_kernel<64, 2, false>,  (const void*)bd_attn_kernel<64, 4, false>,
                      (const void*)bd_attn_kernel<128, 1, true>,  (const void*)bd_attn_kernel<128, 2, true>,
                      (const void*)bd_attn_kernel<128, 4, true>,  (const void*)bd_attn_kernel<64, 1, true>,
                      (const void*)bd_attn_kernel<64, 2, true>,   (const void*)bd_attn_kernel<64, 4, true>};
  for (const void* k : ks)
    if (int rc = kernel_opt_in(k, 200 * 1024, false)) return rc;
  return B200_OK;
}

// one lock-step step as plain launches on `s` (also what gets captured)
static int bd_enqueue_step(BatchDecoder* d, const BdModel& m, cudaStream_t s, long* launches) {
  const DecodeDims& dd = m.d;
  const int B = d->B, H = dd.hidden, I = dd.inter;
  const int QH = dd.n_heads * dd.hd, QKV = (dd.n_heads + 2 * dd.n_kv) * dd.hd;
  int rc;
  const int Gall = dd.n_heads / dd.n_kv;
  const int ag_heads = bd_attn_heads_per_cta(dd, B, m.sm_count);
  const int hs = (Gall + ag_heads - 1) / ag_heads;
  for (int l = 0; l < m.n_layers; ++l) {
    const LayerW& lw = m.layers[l];
    int split = 1;
    if ((rc = gemm_wt_tuned(d->xn, H, lw.wqkv, nullptr, nullptr, 0, nullptr, 0, d->partial, d->partial_bytes, B, QKV,
                            H, B200_EPI_NONE, B200_WT_PARTIAL, 0, true, m.sm_count, &split, s)))
      return rc;
    BdAttnP ap;
    ap.P = d->partial; ap.S = split; ap.B = B; ap.QKV = QKV; ap.bias = lw.bqkv; ap.inv_freq = m.inv_freq;
    const bool q8 = l < m.q8_layers;
    ap.ctx = d->ctx; ap.pos = d->pos; ap.v_off = m.v_off;
    ap.kv = q8 ? nullptr : m.kv + (long)(l - m.q8_layers) * m.layer_stride;
    ap.q8c = q8 ? m.q8_codes + (long)l * m.layer_stride : nullptr;
    ap.q8s = q8 ? m.q8_scales + (long)l * m.layer_stride / m.q8_gs : nullptr;
    ap.q8b = q8 ? m.q8_biases + (long)l * m.layer_stride / m.q8_gs : nullptr;
    ap.gs = q8 ? m.q8_gs : 0;
    ap.row_stride = m.row_stride; ap.out = d->att; ap.n_heads = dd.n_heads; ap.n_kv = dd.n_kv; ap.cap = dd.cap;
    ap.hsplit = hs; ap.scale_bf = dd.scale_bf;
    ap.qn = m.qn ? m.qn[l] : nullptr; ap.kn = m.kn ? m.kn[l] : nullptr; ap.eps = dd.eps;
    if ((rc = bd_attn_dispatch(dd, ag_heads, dim3(dd.n_kv * hs, B), s, ap, q8))) return rc;
    if ((rc = gemm_wt_tuned(d->att, QH, lw.wo, nullptr, nullptr, 0, nullptr, 0, d->partial, d->partial_bytes, B, H, QH,
                            B200_EPI_NONE, B200_WT_PARTIAL, 0, true, m.sm_count, &split, s)))
      return rc;
    if ((rc = finish_rows(d->partial, split, nullptr, d->h, H, d->h, H, B200_NORM_RMS, lw.ln2, nullptr, dd.eps, d->xn,
                          H, B, H, s)))
      return rc;
    if ((rc = gemm_wt_tuned(d->xn, H, lw.wgu, nullptr, nullptr, 0, d->act, I, nullptr, 0, B, 2 * I, H, B200_EPI_NONE,
                            B200_WT_SWIGLU, I, false, m.sm_count, nullptr, s)))
      return rc;
    if ((rc = gemm_wt_tuned(d->act, I, lw.wd, nullptr, nullptr, 0, nullptr, 0, d->partial, d->partial_bytes, B, H, I,
                            B200_EPI_NONE, B200_WT_PARTIAL, 0, true, m.sm_count, &split, s)))
      return rc;
    const bf16* nw = (l + 1 == m.n_layers) ? m.final_norm : m.layers[l + 1].ln1;
    if ((rc = finish_rows(d->partial, split, nullptr, d->h, H, d->h, H, B200_NORM_RMS, nw, nullptr, dd.eps, d->xn, H, B,
                          H, s)))
      return rc;
    *launches += 7;
  }
  if ((rc = gemm_wt_tuned(d->xn, H, m.head, nullptr, nullptr, 0, d->logits, d->ldv, nullptr, 0, B, dd.vocab, H,
                          B200_EPI_NONE, B200_WT_BF16, 0, false, m.sm_count, nullptr, s)))
    return rc;
  if (d->procs.params) {
    BdProcsP pp;
    pp.logits = d->logits; pp.ldv = d->ldv; pp.V = dd.vocab; pp.tok = d->tok; pp.active = d->active; pp.pr = d->procs;
    B200_CUDA(launch(bd_procs_kernel, dim3(B), dim3(1024), 0, s, PDL_LAUNCH, pp));
    *launches += 1;
  }
  BdSampleP sp;
  sp.logits = d->logits; sp.logprobs = d->want_logprobs ? d->logprobs : nullptr; sp.V = dd.vocab; sp.ldv = d->ldv; sp.H = H;
  sp.tok = d->tok; sp.ctx = d->ctx; sp.pos = d->pos; sp.n_out = d->n_out; sp.active = d->active;
  sp.token_log = d->token_log; sp.lp_log = d->lp_log; sp.log_cap = d->log_cap; sp.max_b = d->max_b;
  sp.embed = m.embed; sp.ln0 = m.layers[0].ln1; sp.eps = dd.eps; sp.h = d->h; sp.xn = d->xn;
  B200_CUDA(launch(bd_sample_kernel, dim3(B), dim3(1024), 0, s, PDL_LAUNCH, sp));
  *launches += 2;
  if (d->procs.top_k > 0) {  // over the logprob rows bd_sample wrote (want_logprobs is forced on)
    const int S = (dd.vocab + BD_TOPK_SLICE - 1) / BD_TOPK_SLICE, k = d->procs.top_k;
    B200_CUDA(launch(bd_topk_part_kernel, dim3(S, B), dim3(256), 0, s, PDL_LAUNCH, (const bf16*)d->logprobs, d->ldv, dd.vocab,
                        k, d->topk_cand));
    B200_CUDA(launch(bd_topk_merge_kernel, dim3(B), dim3(256), 0, s, PDL_LAUNCH, (const unsigned long long*)d->topk_cand, S, k,
                        (const int*)d->n_out, d->log_cap, d->max_b, d->topk_ids, d->topk_lp));
    *launches += 2;
  }
  return B200_OK;
}

int batch_decoder_begin(void** handle, const BdModel& m, int B, const int* tok, const int* ctx, const int* pos,
                        const int* active, cudaStream_t s) {
  B200_REQUIRE(B >= 1 && B <= 16, "batch decode: B=%d (1..16)", B);
  B200_REQUIRE(m.d.hd == 64 || m.d.hd == 128, "batch decode: head_dim %d (64|128)", m.d.hd);
  B200_REQUIRE(B <= m.kv_batch, "batch decode: B=%d > KV pool rows %d", B, m.kv_batch);
  B200_REQUIRE(bd_attn_smem(m.d, BD_AG_MAX) <= 200 * 1024, "batch decode: cache capacity %d too large for the attention kernel", m.d.cap);
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(*handle);
  if (!d) {
    d = new BatchDecoder();
    int rc = bd_alloc(d, m, 16);
    if (rc) {
      bd_free(d);
      return rc;
    }
    *handle = d;
    if ((rc = bd_set_smem_attrs())) return rc;
  }
  d->B = B;
  d->procs = BdProcs{};
  for (int b = 0; b < B; ++b) {
    B200_REQUIRE(ctx[b] >= 0 && ctx[b] < m.d.cap, "batch decode: row %d holds %d tokens, capacity %d", b, ctx[b], m.d.cap);
    d->stage_host[b] = tok[b];
    d->stage_host[d->max_b + b] = ctx[b];
    d->stage_host[2 * d->max_b + b] = pos[b];
    d->stage_host[3 * d->max_b + b] = active[b];
  }
  B200_CUDA(cudaStreamSynchronize(s));  // the staging buffer may still feed an earlier copy
  B200_CUDA(cudaMemcpyAsync(d->tok, d->stage_host, B * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d->ctx, d->stage_host + d->max_b, B * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d->pos, d->stage_host + 2 * d->max_b, B * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d->active, d->stage_host + 3 * d->max_b, B * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemsetAsync(d->n_out, 0, d->max_b * 4, s));
  d->steps_done = 0;
  bd_begin_kernel<<<B, 256, 0, s>>>(d->tok, m.embed, m.d.hidden, m.layers[0].ln1, m.d.eps, d->h, d->xn);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int batch_decoder_step(void* handle, const BdModel& m, int n_steps, bool want_logprobs, cudaStream_t s,
                       cudaStream_t cap_stream, long* launches) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  B200_REQUIRE(d && d->B > 0 && n_steps > 0, "batch decode: begin() first");
  B200_REQUIRE(d->steps_done + n_steps <= d->log_cap, "batch decode: fetch the tokens before step %d", d->log_cap);
  want_logprobs = want_logprobs || d->procs.top_k > 0;
  d->want_logprobs = want_logprobs;
  int rc;
  int done = 0;
  const bool stale = !d->gexec || d->graph_kv != m.kv || d->graph_B != d->B || d->graph_cap != m.d.cap ||
                     d->graph_lp != (int)want_logprobs || d->graph_q8 != m.q8_codes ||
                     d->graph_q8_layers != m.q8_layers || d->graph_gs != m.q8_gs ||
                     !bd_same_procs(d->graph_procs, d->procs);
  if (stale) {
    if (d->gexec) {
      cudaGraphExecDestroy(d->gexec);
      d->gexec = nullptr;
    }
    // first step eagerly: the GEMM configurations are measured on first use (not under capture)
    if ((rc = bd_enqueue_step(d, m, s, launches))) return rc;
    done = 1;
    if (n_steps > 1) {
      cudaGraph_t graph = nullptr;
      long dummy = 0;
      B200_CUDA(cudaStreamBeginCapture(cap_stream, cudaStreamCaptureModeThreadLocal));
      rc = bd_enqueue_step(d, m, cap_stream, &dummy);
      cudaError_t ce = cudaStreamEndCapture(cap_stream, &graph);
      if (rc) {
        if (graph) cudaGraphDestroy(graph);
        return rc;
      }
      if (ce != cudaSuccess) return cuda_fail(ce, "cudaStreamEndCapture(batch step)", __FILE__, __LINE__);
      ce = cudaGraphInstantiate(&d->gexec, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) return cuda_fail(ce, "cudaGraphInstantiate(batch step)", __FILE__, __LINE__);
      d->graph_kv = m.kv; d->graph_B = d->B; d->graph_cap = m.d.cap; d->graph_lp = (int)want_logprobs;
      d->graph_q8 = m.q8_codes; d->graph_q8_layers = m.q8_layers; d->graph_gs = m.q8_gs;
      d->graph_procs = d->procs;
    }
  }
  for (int i = done; i < n_steps; ++i) B200_CUDA(cudaGraphLaunch(d->gexec, s));
  *launches += (long)(n_steps - done) *
               (m.n_layers * 7 + 2 + (d->procs.params ? 1 : 0) + (d->procs.top_k > 0 ? 2 : 0));
  d->steps_done += n_steps;
  return B200_OK;
}

int batch_decoder_fetch(void* handle, long first_step, int n_steps, int* tok_host, float* lp_host, cudaStream_t s) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  B200_REQUIRE(d && first_step >= 0 && n_steps > 0 && first_step + n_steps <= d->log_cap, "batch fetch: bad range");
  // rows of the log are [max_b] wide; the host buffer is [n_steps][B]
  B200_CUDA(cudaMemcpy2DAsync(tok_host, (size_t)d->B * 4, d->token_log + first_step * d->max_b, (size_t)d->max_b * 4,
                              (size_t)d->B * 4, n_steps, cudaMemcpyDeviceToHost, s));
  if (lp_host)
    B200_CUDA(cudaMemcpy2DAsync(lp_host, (size_t)d->B * 4, d->lp_log + first_step * d->max_b, (size_t)d->max_b * 4,
                                (size_t)d->B * 4, n_steps, cudaMemcpyDeviceToHost, s));
  return B200_OK;
}

int batch_decoder_set_procs(void* handle, const BdProcs& pr, int vocab) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  B200_REQUIRE(d && d->B > 0, "batch procs: begin() first");
  B200_REQUIRE(pr.top_k >= 0 && pr.top_k <= BD_TOPK_MAX, "batch procs: top_k %d (0..%d)", pr.top_k, BD_TOPK_MAX);
  B200_REQUIRE(!pr.params || (pr.penalties && pr.hist && pr.hist_len && pr.hist_cap >= 1 && pr.hist_cap <= BD_HIST_MAX &&
                              (pr.bias_cap == 0 || (pr.bias_ids && pr.bias_vals && pr.bias_cap > 0))),
               "batch procs: bad arguments (history capacity 1..%d)", BD_HIST_MAX);
  const int S = (vocab + BD_TOPK_SLICE - 1) / BD_TOPK_SLICE;
  B200_REQUIRE(pr.top_k == 0 || S * pr.top_k <= BD_TOPK_CAND_MAX, "batch procs: vocabulary %d too large for top-k", vocab);
  if (pr.top_k > 0 && !d->topk_ids) {
    B200_CUDA(cudaMalloc(&d->topk_cand, (size_t)d->max_b * BD_TOPK_CAND_MAX * 8));
    B200_CUDA(cudaMalloc(&d->topk_ids, (size_t)d->log_cap * d->max_b * BD_TOPK_MAX * 4));
    B200_CUDA(cudaMalloc(&d->topk_lp, (size_t)d->log_cap * d->max_b * BD_TOPK_MAX * 4));
  }
  d->procs = pr;
  return B200_OK;
}

int batch_decoder_fetch_topk(void* handle, long first_step, int n_steps, int* ids_host, float* lp_host, cudaStream_t s) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  B200_REQUIRE(d && d->topk_ids && first_step >= 0 && n_steps > 0 && first_step + n_steps <= d->log_cap,
               "batch fetch top-k: bad range, or top-k never enabled");
  const size_t w = (size_t)BD_TOPK_MAX * 4;
  B200_CUDA(cudaMemcpy2DAsync(ids_host, d->B * w, d->topk_ids + first_step * d->max_b * BD_TOPK_MAX, d->max_b * w,
                              d->B * w, n_steps, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpy2DAsync(lp_host, d->B * w, d->topk_lp + first_step * d->max_b * BD_TOPK_MAX, d->max_b * w,
                              d->B * w, n_steps, cudaMemcpyDeviceToHost, s));
  return B200_OK;
}

int batch_procs_apply(bf16* logits, const bf16* logprobs, int B, int V, int ldv, const int* tok, const int* active,
                      const BdProcs& pr, int* top_ids, float* top_lp, cudaStream_t s) {
  B200_REQUIRE(B >= 1 && B <= 16 && V > 0 && ldv >= V, "batch procs apply: bad arguments");
  B200_REQUIRE(pr.top_k >= 0 && pr.top_k <= BD_TOPK_MAX, "batch procs apply: top_k %d", pr.top_k);
  if (pr.params) {
    B200_REQUIRE(logits && tok && active && pr.penalties && pr.hist && pr.hist_len && pr.hist_cap >= 1 &&
                 pr.hist_cap <= BD_HIST_MAX, "batch procs apply: bad processor arguments");
    BdProcsP pp;
    pp.logits = logits; pp.ldv = ldv; pp.V = V; pp.tok = tok; pp.active = active; pp.pr = pr;
    B200_CUDA(launch(bd_procs_kernel, dim3(B), dim3(1024), 0, s, PDL_LAUNCH, pp));
  }
  if (pr.top_k > 0) {
    const int S = (V + BD_TOPK_SLICE - 1) / BD_TOPK_SLICE;
    B200_REQUIRE(logprobs && top_ids && top_lp && S * pr.top_k <= BD_TOPK_CAND_MAX, "batch procs apply: bad top-k arguments");
    unsigned long long* cand = nullptr;
    B200_CUDA(cudaMallocAsync(&cand, (size_t)B * S * pr.top_k * 8, s));
    cudaError_t e = launch(bd_topk_part_kernel, dim3(S, B), dim3(256), 0, s, PDL_LAUNCH, logprobs, ldv, V, pr.top_k, cand);
    if (e == cudaSuccess)
      e = launch(bd_topk_merge_kernel, dim3(B), dim3(256), 0, s, PDL_LAUNCH, (const unsigned long long*)cand, S, pr.top_k,
                 (const int*)nullptr, 1, B, top_ids, top_lp);
    B200_CUDA(cudaFreeAsync(cand, s));
    B200_CUDA(e);
  }
  return B200_OK;
}

int batch_kvq_attention(const float* qkv, const bf16* bias, const float* inv_freq, const int* ctx, const int* pos,
                        uint8_t* codes, bf16* scales, bf16* biases, int gs, int pool_rows, int cap, bf16* out, int B,
                        int n_heads, int n_kv, int hd, const bf16* qn, const bf16* kn, float eps, int sm_count,
                        cudaStream_t s) {
  B200_REQUIRE(hd == 64 || hd == 128, "batch kvq attention: head_dim %d (64|128)", hd);
  B200_REQUIRE((gs == 32 || gs == 64 || gs == 128) && hd % gs == 0, "batch kvq attention: group size %d", gs);
  B200_REQUIRE(B >= 1 && B <= pool_rows && n_kv > 0 && n_heads % n_kv == 0, "batch kvq attention: bad arguments");
  DecodeDims d = {};
  d.n_heads = n_heads; d.n_kv = n_kv; d.hd = hd; d.cap = cap; d.eps = eps;
  d.scale_bf = __bfloat162float(__float2bfloat16_rn(1.0f / sqrtf((float)hd)));
  B200_REQUIRE(bd_attn_smem(d, BD_AG_MAX) <= 200 * 1024, "batch kvq attention: capacity %d too large", cap);
  int rc = bd_set_smem_attrs();
  if (rc) return rc;
  const int ag_heads = bd_attn_heads_per_cta(d, B, sm_count);
  const int hs = (n_heads / n_kv + ag_heads - 1) / ag_heads;
  BdAttnP ap = {};
  ap.P = qkv; ap.S = 1; ap.B = B; ap.QKV = (n_heads + 2 * n_kv) * hd; ap.bias = bias; ap.inv_freq = inv_freq;
  ap.ctx = ctx; ap.pos = pos; ap.row_stride = (long)n_kv * cap * hd; ap.v_off = (long)pool_rows * ap.row_stride;
  ap.out = out; ap.n_heads = n_heads; ap.n_kv = n_kv; ap.cap = cap; ap.hsplit = hs; ap.scale_bf = d.scale_bf;
  ap.qn = qn; ap.kn = kn; ap.eps = eps;
  ap.q8c = codes; ap.q8s = scales; ap.q8b = biases; ap.gs = gs;
  return bd_attn_dispatch(d, ag_heads, dim3(n_kv * hs, B), s, ap, true);
}

const void* batch_decoder_buffer(void* handle, int which) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  if (!d) return nullptr;
  return which == 0 ? (const void*)d->logits : (which == 1 ? (const void*)d->logprobs : (const void*)d->token_log);
}

}  // namespace b200
