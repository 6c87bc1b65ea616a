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
//                        KV append at the row's length) and attends over the row's keys
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

namespace b200 {

namespace {

constexpr int BD_AG_MAX = 4;  // q heads per attention CTA: 4, 2 or 1 — the smallest that keeps the grid within one wave

__device__ __forceinline__ void bd_pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void bd_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ float bd_block_sum(float v, float* red, int nwarps) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < nwarps; ++w) t += red[w];
  return t;
}

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
  const float tot = bd_block_sum(ss, red, blockDim.x >> 5);
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
  // weights of the GEMMs that follow (o_proj, gate/up, down): this kernel is a chain of dependent round trips that
  // leaves HBM idle, so its CTAs ask the L2 for them up front (l2_prefetch_span; weights are static during a step)
  const void* pf[3];
  long pf_bytes[3];
};

template <int HD, int AG>
__global__ void __launch_bounds__(256) bd_attn_kernel(const BdAttnP p) {
  bd_pdl_launch();
  if (threadIdx.x == 0) {
    const int n = gridDim.x * gridDim.y, id = blockIdx.y * gridDim.x + blockIdx.x;
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (p.pf_bytes[i] > 0) l2_prefetch_span(p.pf[i], p.pf_bytes[i], id, n);
  }
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
  bf16* kb = p.kv + (long)row * p.row_stride + (long)kvh * p.cap * HD;
  bf16* vb = kb + p.v_off;
  bd_pdl_wait();
  const int ctx = p.ctx[row], pos = p.pos[row];
  const int nkeys = ctx + 1;
  // Every dependent global round trip costs ~1 us here, so the requests are issued as early as their
  // addresses are known: the first block of cached keys (one row per lane) goes out BEFORE the
  // split-K partials of q/k/v are summed, the first block of values before the softmax.
  uint4 kfirst[NCH];
  {
    const int j = warp * 32 + lane;
    const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * HD);
#pragma unroll
    for (int c = 0; c < NCH; ++c) kfirst[c] = (j < ctx) ? __ldcg(kr + c) : make_uint4(0, 0, 0, 0);
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
  if (part == 0) {  // append the new position to the row's cache (one CTA per kv head)
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
    if (j0 == warp * 32) {
#pragma unroll
      for (int c = 0; c < NCH; ++c) kv[c] = kfirst[c];
    } else if (j < ctx) {
      const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * HD);
#pragma unroll
      for (int c = 0; c < NCH; ++c) kv[c] = __ldcg(kr + c);
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
  uint4 vfirst[VU][NV];
#pragma unroll
  for (int q = 0; q < VU; ++q) {
    const int j = warp * 32 + q * 4 + ksub;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      vfirst[q][v] = (j < ctx) ? __ldcg(reinterpret_cast<const uint4*>(vb + (long)j * HD + seg * SEG + v * 8))
                               : make_uint4(0, 0, 0, 0);
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
#pragma unroll
    for (int q = 0; q < VU; ++q) {
      const int j = j0 + warp * 32 + q * 4 + ksub;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        if (j0 == 0) vv[q][v] = vfirst[q][v];
        else vv[q][v] = (j < ctx) ? __ldcg(reinterpret_cast<const uint4*>(vb + (long)j * HD + seg * SEG + v * 8))
                                  : make_uint4(0, 0, 0, 0);
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
__device__ __forceinline__ uint32_t bd_orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

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
  bd_pdl_launch();
  __shared__ float red[32];
  __shared__ float2 stat[32];
  __shared__ unsigned long long keys[32];
  __shared__ float s_lse;
  __shared__ int s_tok;
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  bd_pdl_wait();
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
          ((unsigned long long)bd_orderable(o[j]) << 32) | (0xFFFFFFFFu - (uint32_t)(c * 8 + j));
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
  int graph_B = 0, graph_cap = 0, graph_lp = 0;
  long steps_done = 0;
  bool want_logprobs = false;
};

static void bd_free(BatchDecoder* d) {
  if (!d) return;
  if (d->gexec) cudaGraphExecDestroy(d->gexec);
  for (void* p : {(void*)d->tok, (void*)d->ctx, (void*)d->pos, (void*)d->active, (void*)d->n_out, (void*)d->token_log,
                  (void*)d->lp_log, (void*)d->h, (void*)d->xn, (void*)d->att, (void*)d->act, (void*)d->logits,
                  (void*)d->logprobs, (void*)d->partial})
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

template <typename... KArgs, typename... Args>
static int bd_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  B200_CUDA(cudaLaunchKernelEx(&cfg, kern, KArgs(args)...));
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

template <int HD>
static int bd_attn_launch(int ag, dim3 grid, size_t smem, cudaStream_t s, const BdAttnP& ap) {
  switch (ag) {
    case 1: return bd_launch(bd_attn_kernel<HD, 1>, grid, dim3(256), smem, s, ap);
    case 2: return bd_launch(bd_attn_kernel<HD, 2>, grid, dim3(256), smem, s, ap);
    default: return bd_launch(bd_attn_kernel<HD, 4>, grid, dim3(256), smem, s, ap);
  }
}

// L2 prefetch budget of the latency-bound kernels of a step, in bytes (B200_BD_PREFETCH_MB).  DEFAULT 0 = off: the
// prefetch traffic can lengthen the attention kernel's dependent round trips by more than the L2-resident weights save
// the GEMMs (not measured on the H100, whose L2 is 50 MB).  Kept as a tuning knob.
static long bd_prefetch_budget() {
  static long v = -1;
  if (v < 0) {
    const char* e = getenv("B200_BD_PREFETCH_MB");
    long mb = e ? atol(e) : 0;
    if (mb < 0) mb = 0;
    if (mb > 120) mb = 120;
    v = mb << 20;
  }
  return v;
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
    ap.ctx = d->ctx; ap.pos = d->pos; ap.kv = m.kv + (long)l * m.layer_stride; ap.v_off = m.v_off;
    ap.row_stride = m.row_stride; ap.out = d->att; ap.n_heads = dd.n_heads; ap.n_kv = dd.n_kv; ap.cap = dd.cap;
    ap.hsplit = hs; ap.scale_bf = dd.scale_bf;
    ap.qn = m.qn ? m.qn[l] : nullptr; ap.kn = m.kn ? m.kn[l] : nullptr; ap.eps = dd.eps;
    {  // o_proj, then gate/up, then down, as far as the budget goes
      long left = bd_prefetch_budget();
      const void* w[3] = {lw.wo, lw.wgu, lw.wd};
      const long bytes[3] = {(long)H * QH * 2, 2L * I * H * 2, (long)H * I * 2};
      for (int i = 0; i < 3; ++i) {
        ap.pf[i] = w[i];
        ap.pf_bytes[i] = bytes[i] < left ? bytes[i] : left;
        left -= ap.pf_bytes[i];
      }
    }
    const dim3 ag(dd.n_kv * hs, B);
    if (dd.hd == 128) rc = bd_attn_launch<128>(ag_heads, ag, bd_attn_smem(dd, ag_heads), s, ap);
    else rc = bd_attn_launch<64>(ag_heads, ag, bd_attn_smem(dd, ag_heads), s, ap);
    if (rc) return rc;
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
    // the finish of `down` is the other HBM-idle spot: it asks for the next layer's qkv weights
    const void* nq = (l + 1 == m.n_layers) ? nullptr : (const void*)m.layers[l + 1].wqkv;
    const long nq_bytes = nq ? ((long)QKV * H * 2 < bd_prefetch_budget() ? (long)QKV * H * 2 : bd_prefetch_budget()) : 0;
    if ((rc = finish_rows(d->partial, split, nullptr, d->h, H, d->h, H, B200_NORM_RMS, nw, nullptr, dd.eps, d->xn, H, B,
                          H, s, nq, nq_bytes)))
      return rc;
    *launches += 7;
  }
  if ((rc = gemm_wt_tuned(d->xn, H, m.head, nullptr, nullptr, 0, d->logits, d->ldv, nullptr, 0, B, dd.vocab, H,
                          B200_EPI_NONE, B200_WT_BF16, 0, false, m.sm_count, nullptr, s)))
    return rc;
  BdSampleP sp;
  sp.logits = d->logits; sp.logprobs = d->want_logprobs ? d->logprobs : nullptr; sp.V = dd.vocab; sp.ldv = d->ldv; sp.H = H;
  sp.tok = d->tok; sp.ctx = d->ctx; sp.pos = d->pos; sp.n_out = d->n_out; sp.active = d->active;
  sp.token_log = d->token_log; sp.lp_log = d->lp_log; sp.log_cap = d->log_cap; sp.max_b = d->max_b;
  sp.embed = m.embed; sp.ln0 = m.layers[0].ln1; sp.eps = dd.eps; sp.h = d->h; sp.xn = d->xn;
  if ((rc = bd_launch(bd_sample_kernel, dim3(B), dim3(1024), 0, s, sp))) return rc;
  *launches += 2;
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
    static unsigned long long attr_mask = 0ull;
    if (first_use_on_device(&attr_mask)) {
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<128, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(bd_attn_kernel<64, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
  }
  d->B = B;
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
  d->want_logprobs = want_logprobs;
  int rc;
  int done = 0;
  const bool stale = !d->gexec || d->graph_kv != m.kv || d->graph_B != d->B || d->graph_cap != m.d.cap ||
                     d->graph_lp != (int)want_logprobs;
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
    }
  }
  for (int i = done; i < n_steps; ++i) B200_CUDA(cudaGraphLaunch(d->gexec, s));
  *launches += (long)(n_steps - done) * (m.n_layers * 7 + 2);
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

const void* batch_decoder_buffer(void* handle, int which) {
  BatchDecoder* d = reinterpret_cast<BatchDecoder*>(handle);
  if (!d) return nullptr;
  return which == 0 ? (const void*)d->logits : (which == 1 ? (const void*)d->logprobs : (const void*)d->token_log);
}

}  // namespace b200
