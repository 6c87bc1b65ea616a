// The autoregressive decode step (reference generate/ar.py:496-515 -> _step
// :334-389 -> models/qwen2_vl/language.py:404-518 with L == 1), batch 1.
//
// The step is HBM-bound (3.09 GB of weights per token) and latency-chained
// (norm -> qkv -> attention -> o_proj -> norm -> gate/up -> down, 28 times), so the
// design goal is: the weight stream never stops.
//
//   * k_stream<MODE>: persistent weight-streaming GEMV.  One producer thread per
//     CTA issues `cp.async.bulk` (TMA engine, mbarrier complete_tx) copies of whole
//     row tiles into a shared-memory ring; 8 consumer warps dot the tiles with the
//     activation vector held in registers.  The producer does not depend on the
//     previous kernel, so with programmatic dependent launch (PDL) the NEXT
//     kernel's ring fills while the current kernel is still finishing: ~100 KB per
//     CTA, two CTAs of consecutive kernels co-resident per SM.
//     MODES: QKV    RMSNorm + [Wq;Wk;Wv] + bias + M-RoPE + KV append
//            ORES   o_proj + residual          (row per warp)
//            GATEUP RMSNorm + gate/up + SwiGLU
//            DRES   down + residual            (split-K across warps)
//            HEAD   final RMSNorm + tied-embedding GEMV + logsumexp partials
//   * k_attn1: single-CTA GQA attention per (kv head, q-head group), lane-per-key
//     scores (no shuffles), for contexts up to ATT1_MAX_CAP keys; k_attn (cluster
//     of CTAs, DSMEM push) beyond that.
//   * k_sample: logprobs (bf16), greedy argmax (lowest index on ties), token log,
//     state advance, next-token embedding.
// Rounding points follow oracle/qwen2vl.py::lm_layers_forward.
#include <cooperative_groups.h>

#include "common.cuh"
#include "decode.cuh"

namespace cg = cooperative_groups;

namespace b200 {

// ---------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint4 ldg16(const void* p) {
  return *reinterpret_cast<const uint4*>(p);
}
__device__ __forceinline__ uint32_t s_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mb_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mb_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ void mb_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  const uint32_t addr = s_u32(bar);
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// 1-D bulk copy global -> shared through the TMA engine, evict-first in L2
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1], %2, [%3], %4;" ::"r"(s_u32(dst)),
      "l"(src), "r"(bytes), "r"(s_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ---------------------------------------------------------------------------
// k_stream: persistent weight-streaming GEMV
// ---------------------------------------------------------------------------
enum { SM_QKV = 0, SM_ORES = 1, SM_GATEUP = 2, SM_DRES = 3, SM_HEAD = 4 };

struct StreamP {
  const bf16* W;     // rows of matrix 1 (qkv / wo / gate / wd / embedding)
  const bf16* W2;    // GATEUP: up rows
  const bf16* bias;  // QKV
  const bf16* x;     // activation vector (K)
  const bf16* lnw;   // RMSNorm weight (NORM modes)
  bf16* out;         // ORES/DRES: h (in place); GATEUP: act; HEAD: logits; QKV: qbuf
  bf16* kc;          // QKV
  bf16* vc;          // QKV
  const DecState* st;
  const float* inv_freq;
  float2* partials;  // HEAD
  int N;             // output rows (QKV: unused)
  int K;
  int R;             // row(-pair)s per tile
  int S;             // K slices per row (R * S == 8 consumer warps)
  int tiles;
  int n_stages;
  int stage_bytes;
  // QKV geometry
  int n_heads, n_kv, hd, cap;
  float eps;
  int raw_qk;        // QKV: q / k rows left unrotated (Qwen3-VL: k_qk_norm_rope normalises and rotates them)
};

constexpr int STREAM_CONSUMERS = 256;            // 8 warps
constexpr int STREAM_THREADS = STREAM_CONSUMERS + 32;  // + producer warp
constexpr int STREAM_SMEM_BUDGET = 100 * 1024;   // two CTAs (consecutive kernels) per SM

template <int MODE>
struct StreamTraits {
  static constexpr bool PAIR = (MODE == SM_QKV || MODE == SM_GATEUP);
  static constexpr bool NORM = (MODE == SM_QKV || MODE == SM_GATEUP || MODE == SM_HEAD);
  static constexpr int NRW = PAIR ? 2 : 1;
};

// global row index of (tile t, local row r, which matrix m) and its source pointer
template <int MODE>
__device__ __forceinline__ const bf16* tile_src(const StreamP& p, int t, int m) {
  if (MODE == SM_QKV) {
    const int half = p.hd >> 1;
    const int per_slot = half / p.R;  // tiles per head slot
    const int slot = t / per_slot, jb = t % per_slot;
    return p.W + ((long)slot * p.hd + (long)m * half + (long)jb * p.R) * p.K;
  }
  if (MODE == SM_GATEUP) return (m == 0 ? p.W : p.W2) + (long)t * p.R * p.K;
  return p.W + (long)t * p.R * p.K;
}

template <int MODE, int CHX>
__global__ void __launch_bounds__(STREAM_THREADS, 2) k_stream(const StreamP p) {
  using T = StreamTraits<MODE>;
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ uint64_t full_bar[8], empty_bar[8];
  __shared__ float red[2][8][2];
  __shared__ float2 wstat[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mb_init(&full_bar[s], 1);
      mb_init(&empty_bar[s], 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  const int my_tiles = (p.tiles > (int)blockIdx.x)
                           ? (p.tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int rows_unit = p.K * 2;  // bytes per weight row

  if (warp == 8) {
    // ===== producer: independent of the previous kernel -> runs ahead under PDL =====
    if (lane == 0) {
      const uint64_t pol = policy_evict_first();
      for (int it = 0; it < my_tiles; ++it) {
        const int t = blockIdx.x + it * gridDim.x;
        const int s = it % p.n_stages;
        const uint32_t ph = (it / p.n_stages) & 1;
        mb_wait(&empty_bar[s], ph ^ 1);
        int rows = p.R;
        if (MODE != SM_QKV) rows = min(p.R, p.N - t * p.R);
        const uint32_t bytes = (uint32_t)rows * rows_unit;
        mb_expect_tx(&full_bar[s], bytes * T::NRW);
        uint8_t* dst = sm + (long)s * p.stage_bytes;
        bulk_g2s(dst, tile_src<MODE>(p, t, 0), bytes, &full_bar[s], pol);
        if (T::PAIR) bulk_g2s(dst + (long)p.R * rows_unit, tile_src<MODE>(p, t, 1), bytes,
                              &full_bar[s], pol);
      }
    }
    return;
  }

  // ===== consumers =====
  const int rloc = warp % p.R;   // row (pair) within the tile
  const int sub = warp / p.R;    // K slice
  const int nvec = p.K >> 3;
  const int cb = (int)((long)nvec * sub / p.S), ce = (int)((long)nvec * (sub + 1) / p.S);
  pdl_wait();  // the activation vector / state of the previous kernel is now visible
  // activation slice of this warp, in registers (packed bf16)
  uint4 xv[CHX];
#pragma unroll
  for (int u = 0; u < CHX; ++u) {
    const int c = cb + lane + 32 * u;
    xv[u] = (c < ce) ? ldg16(p.x + (long)c * 8) : make_uint4(0, 0, 0, 0);
  }
  if (T::NORM) {
    uint4 lw4[CHX];
#pragma unroll
    for (int u = 0; u < CHX; ++u) {
      const int c = cb + lane + 32 * u;
      lw4[u] = (c < ce) ? ldg16(p.lnw + (long)c * 8) : make_uint4(0, 0, 0, 0);
    }
    float ss = 0.f;
    if (p.S == 1) {  // the slice is the whole vector: reuse the registers
#pragma unroll
      for (int u = 0; u < CHX; ++u) {
        float f[8];
        unpack8(xv[u], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
      }
    } else {
      for (int c = lane; c < nvec; c += 32) {
        float f[8];
        unpack8(ldg16(p.x + (long)c * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
      }
    }
    ss = warp_sum(ss);
    const float rs = 1.0f / sqrtf(ss / (float)p.K + p.eps);
#pragma unroll
    for (int u = 0; u < CHX; ++u) {
      float f[8], lf[8];
      unpack8(xv[u], f);
      unpack8(lw4[u], lf);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = rbf(rbf(f[j] * rs) * lf[j]);
      xv[u].x = pack2(f[0], f[1]);
      xv[u].y = pack2(f[2], f[3]);
      xv[u].z = pack2(f[4], f[5]);
      xv[u].w = pack2(f[6], f[7]);
    }
  }
  float run_m = -INFINITY, run_l = 0.f;  // HEAD: running logsumexp (lane 0 of slice-0 warps)
  int ctx = 0, pos = 0;
  if (MODE == SM_QKV) {
    ctx = p.st->ctx;
    pos = p.st->pos;
  }

  for (int it = 0; it < my_tiles; ++it) {
    const int t = blockIdx.x + it * gridDim.x;
    const int s = it % p.n_stages;
    const uint32_t ph = (it / p.n_stages) & 1;
    int rows = p.R;
    if (MODE != SM_QKV) rows = min(p.R, p.N - t * p.R);
    mb_wait(&full_bar[s], ph);
    const uint8_t* base = sm + (long)s * p.stage_bytes + (long)rloc * rows_unit;
    float acc[T::NRW];
    {
      // 8 independent partial sums per row: the FMAs of a chunk do not chain
      float a8[T::NRW][8];
#pragma unroll
      for (int m = 0; m < T::NRW; ++m)
#pragma unroll
        for (int j = 0; j < 8; ++j) a8[m][j] = 0.f;
      if (rloc < rows) {
#pragma unroll
        for (int u0 = 0; u0 < CHX; u0 += 2) {  // two chunks (LDS.128) in flight per row
          uint4 w4[T::NRW][2];
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int c = cb + lane + 32 * (u0 + q);
#pragma unroll
            for (int m = 0; m < T::NRW; ++m)
              w4[m][q] = (u0 + q < CHX && c < ce)
                             ? *reinterpret_cast<const uint4*>(base + (long)m * p.R * rows_unit +
                                                               (long)c * 16)
                             : make_uint4(0, 0, 0, 0);
          }
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            if (u0 + q < CHX) {
              float xf[8];
              unpack8(xv[u0 + q], xf);
#pragma unroll
              for (int m = 0; m < T::NRW; ++m) {
                float wf[8];
                unpack8(w4[m][q], wf);
#pragma unroll
                for (int j = 0; j < 8; ++j) a8[m][j] = fmaf(wf[j], xf[j], a8[m][j]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int m = 0; m < T::NRW; ++m)
        acc[m] = ((a8[m][0] + a8[m][1]) + (a8[m][2] + a8[m][3])) +
                 ((a8[m][4] + a8[m][5]) + (a8[m][6] + a8[m][7]));
    }
#pragma unroll
    for (int m = 0; m < T::NRW; ++m) acc[m] = warp_sum(acc[m]);
    __syncwarp();
    if (lane == 0) mb_arrive(&empty_bar[s]);  // this warp is done reading the stage
    if (p.S > 1) {  // split-K: combine the slices of a row through shared memory
      if (lane == 0) {
#pragma unroll
        for (int m = 0; m < T::NRW; ++m) red[it & 1][warp][m] = acc[m];
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (sub == 0) {
#pragma unroll
        for (int m = 0; m < T::NRW; ++m) {
          float a = 0.f;
          for (int q = 0; q < p.S; ++q) a += red[it & 1][rloc + q * p.R][m];
          acc[m] = a;
        }
      }
    }
    if (sub == 0 && lane == 0 && rloc < rows) {
      if (MODE == SM_QKV) {
        const int half = p.hd >> 1;
        const int per_slot = half / p.R;
        const int slot = t / per_slot, j = (t % per_slot) * p.R + rloc;
        const int r1 = slot * p.hd + j, r2 = r1 + half;
        const float y1 = rbf(acc[0] + bf2f(p.bias[r1]));
        const float y2 = rbf(acc[T::NRW - 1] + bf2f(p.bias[r2]));
        if (slot >= p.n_heads + p.n_kv) {
          bf16* dst = p.vc + ((long)(slot - p.n_heads - p.n_kv) * p.cap + ctx) * p.hd;
          dst[j] = f2bf(y1);
          dst[j + half] = f2bf(y2);
        } else if (p.raw_qk) {
          bf16* dst = (slot < p.n_heads) ? p.out + (long)slot * p.hd
                                         : p.kc + ((long)(slot - p.n_heads) * p.cap + ctx) * p.hd;
          dst[j] = f2bf(y1);
          dst[j + half] = f2bf(y2);
        } else {
          // M-RoPE, identical t/h/w position on decode (language.py:476-509)
          const float ang = (float)pos * p.inv_freq[j];
          const float c = rbf(cosf(ang)), sn = rbf(sinf(ang));
          const float o1 = rbf(rbf(y1 * c) + rbf((-y2) * sn));
          const float o2 = rbf(rbf(y2 * c) + rbf(y1 * sn));
          bf16* dst = (slot < p.n_heads) ? p.out + (long)slot * p.hd
                                         : p.kc + ((long)(slot - p.n_heads) * p.cap + ctx) * p.hd;
          dst[j] = f2bf(o1);
          dst[j + half] = f2bf(o2);
        }
      } else if (MODE == SM_GATEUP) {
        const int i = t * p.R + rloc;
        p.out[i] = f2bf(swiglu_bf(rbf(acc[0]), rbf(acc[T::NRW - 1])));
      } else if (MODE == SM_ORES || MODE == SM_DRES) {
        const int r = t * p.R + rloc;
        p.out[r] = f2bf(rbf(bf2f(p.out[r]) + rbf(acc[0])));
      } else {  // HEAD
        const int v = t * p.R + rloc;
        const float a = rbf(acc[0]);
        p.out[v] = f2bf(a);
        const float mn = fmaxf(run_m, a);
        run_l = run_l * expf(run_m - mn) + expf(a - mn);
        run_m = mn;
      }
    }
  }
  if (MODE == SM_HEAD) {
    if (lane == 0) wstat[warp] = make_float2(run_m, run_l);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (threadIdx.x == 0) {
      float M = -INFINITY;
      for (int i = 0; i < 8; ++i) M = fmaxf(M, wstat[i].x);
      float L = 0.f;
      for (int i = 0; i < 8; ++i)
        if (wstat[i].y > 0.f) L += wstat[i].y * expf(wstat[i].x - M);
      p.partials[blockIdx.x] = make_float2(M, L);
    }
  }
}

// ---------------------------------------------------------------------------
// k_qk_norm_rope (Qwen3-VL, language.py:84-89 then the M-RoPE of :113-119): after a raw_qk QKV kernel, q_norm /
// k_norm and the rotary of one decode position on the q heads (qbuf, in place) and the new K row (the cache at
// ctx, in place).  One warp per head.
template <int NU>
__global__ void __launch_bounds__(256) k_qk_norm_rope(const DecodeDims d, bf16* __restrict__ qbuf,
                                                      bf16* __restrict__ kc, const DecState* __restrict__ st,
                                                      const float* __restrict__ inv_freq,
                                                      const bf16* __restrict__ qn, const bf16* __restrict__ kn) {
  pdl_launch_dependents();
  pdl_wait();
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (slot >= d.n_heads + d.n_kv) return;
  const int ctx = st->ctx, pos = st->pos;
  bf16* base = slot < d.n_heads ? qbuf + (long)slot * d.hd : kc + ((long)(slot - d.n_heads) * d.cap + ctx) * d.hd;
  float x[NU];
#pragma unroll
  for (int u = 0; u < NU; ++u) x[u] = bf2f(base[lane + 32 * u]);
  warp_head_rms<NU>(x, slot < d.n_heads ? qn : kn, d.eps);
  warp_head_rope<NU>(x, pos, inv_freq);
#pragma unroll
  for (int u = 0; u < NU; ++u) base[lane + 32 * u] = f2bf(x[u]);
}

// ---------------------------------------------------------------------------
// k_attn1: one CTA per (kv head, q-head group), all keys.  Scores: one key per
// lane (no shuffles), q broadcast from shared memory.  Rounding points as in
// oracle/mlx_semantics.py::sdpa.
// ---------------------------------------------------------------------------
constexpr int ATT_MAXG = 8;   // q heads handled by one CTA (cluster kernel)
constexpr int ATT_MAXCL = 8;  // cluster size
constexpr int ATT1_G = 4;     // q heads per CTA (single-CTA kernel)

template <int HD>
__global__ void __launch_bounds__(256) k_attn1(const DecodeDims d, const bf16* __restrict__ qbuf,
                                               const bf16* __restrict__ kc,
                                               const bf16* __restrict__ vc,
                                               bf16* __restrict__ out,
                                               const DecState* __restrict__ st, int hsplit) {
  pdl_launch_dependents();
  extern __shared__ __align__(16) uint8_t sm[];
  constexpr int EPL = HD / 32;   // dims per lane in the P.V phase
  constexpr int NCH = HD / 8;    // 16-byte chunks per key row
  const int Gall = d.n_heads / d.n_kv;
  const int G = Gall / hsplit;
  float* qs = reinterpret_cast<float*>(sm);   // [ATT1_G][HD]
  float* sc = qs + ATT1_G * HD;               // [ATT1_G][cap]
  float* red = sc + (long)ATT1_G * d.cap;     // [8][ATT1_G*HD]
  __shared__ float s_m[8][ATT1_G], s_l[8][ATT1_G];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kvh = blockIdx.x / hsplit;
  const int h0 = kvh * Gall + (blockIdx.x % hsplit) * G;
  const bf16* kb = kc + (long)kvh * d.cap * HD;
  const bf16* vb = vc + (long)kvh * d.cap * HD;
  pdl_wait();
  const int nkeys = st->ctx + 1;
  for (int i = threadIdx.x; i < ATT1_G * HD; i += blockDim.x)
    qs[i] = (i < G * HD) ? rbf(bf2f(qbuf[(long)h0 * HD + i]) * d.scale_bf) : 0.f;
  __syncthreads();
  // ---- scores: lane <-> key; the whole key row is fetched with NCH loads in flight ----
  float lm[ATT1_G];
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g) lm[g] = -INFINITY;
  for (int j0 = warp * 32; j0 < nkeys; j0 += 256) {
    const int j = j0 + lane;
    if (j < nkeys) {
      const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * HD);
      uint4 kv[NCH];
#pragma unroll
      for (int c = 0; c < NCH; ++c) kv[c] = kr[c];
      float s[ATT1_G][2];
#pragma unroll
      for (int g = 0; g < ATT1_G; ++g) s[g][0] = s[g][1] = 0.f;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        float kf[8];
        unpack8(kv[c], kf);
#pragma unroll
        for (int g = 0; g < ATT1_G; ++g) {
          const float4 a = *reinterpret_cast<const float4*>(qs + g * HD + c * 8);
          const float4 b = *reinterpret_cast<const float4*>(qs + g * HD + c * 8 + 4);
          s[g][0] = fmaf(a.x, kf[0], fmaf(a.y, kf[1], fmaf(a.z, kf[2], fmaf(a.w, kf[3], s[g][0]))));
          s[g][1] = fmaf(b.x, kf[4], fmaf(b.y, kf[5], fmaf(b.z, kf[6], fmaf(b.w, kf[7], s[g][1]))));
        }
      }
#pragma unroll
      for (int g = 0; g < ATT1_G; ++g) {
        const float r = rbf(s[g][0] + s[g][1]);
        sc[(long)g * d.cap + j] = r;
        lm[g] = fmaxf(lm[g], r);
      }
    }
  }
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g) {
    lm[g] = warp_max(lm[g]);
    if (lane == 0) s_m[warp][g] = lm[g];
  }
  __syncthreads();
  // ---- softmax numerators exp(s - M) (kept in sc), row sums via warp partials ----
  float M[ATT1_G], ls[ATT1_G];
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g) {
    float m = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) m = fmaxf(m, s_m[w][g]);
    M[g] = m;
    ls[g] = 0.f;
  }
  for (int j = threadIdx.x; j < nkeys; j += 256) {
#pragma unroll
    for (int g = 0; g < ATT1_G; ++g) {
      const float e = expf(sc[(long)g * d.cap + j] - M[g]);
      sc[(long)g * d.cap + j] = e;
      ls[g] += e;
    }
  }
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g) {
    ls[g] = warp_sum(ls[g]);
    if (lane == 0) s_l[warp][g] = ls[g];
  }
  __syncthreads();
  float L[ATT1_G];
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g) {
    float l = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) l += s_l[w][g];
    L[g] = l;
  }
  // p = bf16(exp / L), in place, one key per thread
  for (int j = threadIdx.x; j < nkeys; j += 256) {
#pragma unroll
    for (int g = 0; g < ATT1_G; ++g) sc[(long)g * d.cap + j] = rbf(sc[(long)g * d.cap + j] / L[g]);
  }
  __syncthreads();
  // ---- partial out: warp w takes keys w, w+8, ...; 4 keys in flight ----
  float acc[ATT1_G][EPL];
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g)
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[g][e] = 0.f;
  for (int j0 = warp; j0 < nkeys; j0 += 32) {
    float vf[4][EPL];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + 8 * q;
#pragma unroll
      for (int e = 0; e < EPL; ++e) vf[q][e] = 0.f;
      if (j < nkeys) {
        const bf16* vr = vb + (long)j * HD + lane * EPL;
        if (EPL == 4) {
          float t4[4];
          unpack4(*reinterpret_cast<const uint2*>(vr), t4);
#pragma unroll
          for (int e = 0; e < EPL; ++e) vf[q][e] = t4[e];
        } else {
          const uint32_t w = *reinterpret_cast<const uint32_t*>(vr);
          vf[q][0] = __uint_as_float(w << 16);
          vf[q][EPL - 1] = __uint_as_float(w & 0xffff0000u);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + 8 * q;
      if (j < nkeys) {
#pragma unroll
        for (int g = 0; g < ATT1_G; ++g) {
          const float pj = sc[(long)g * d.cap + j];
#pragma unroll
          for (int e = 0; e < EPL; ++e) acc[g][e] = fmaf(pj, vf[q][e], acc[g][e]);
        }
      }
    }
  }
#pragma unroll
  for (int g = 0; g < ATT1_G; ++g)
#pragma unroll
    for (int e = 0; e < EPL; ++e) red[((long)warp * ATT1_G + g) * HD + lane * EPL + e] = acc[g][e];
  __syncthreads();
  for (int i = threadIdx.x; i < G * HD; i += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[(long)w * ATT1_G * HD + i];
    out[(long)h0 * HD + i] = f2bf(s);
  }
}

// ---------------------------------------------------------------------------
// k_attn: long contexts — a cluster of CL CTAs per (kv head, q-head group); rank r
// owns keys [r*chunk, (r+1)*chunk).  Softmax statistics and partial outputs are
// PUSHED to the peers' shared memory (st.shared::cluster): two cluster barriers.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_attn(const DecodeDims d, const bf16* __restrict__ qbuf,
                                              const bf16* __restrict__ kc,
                                              const bf16* __restrict__ vc, bf16* __restrict__ out,
                                              const DecState* __restrict__ st, int chunk_cap,
                                              int hsplit) {
  pdl_launch_dependents();
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) uint8_t sm[];
  const int Gall = d.n_heads / d.n_kv;
  const int G = Gall / hsplit;  // q heads of this CTA
  const int hd = d.hd;
  const int EPL = hd >> 5;  // elements per lane (hd = 64 -> 2, 128 -> 4)
  float* sc = reinterpret_cast<float*>(sm);            // [G][chunk_cap]
  float* stats = sc + (long)ATT_MAXG * chunk_cap;      // [CL][G][2]   (filled by the peers)
  float* part = stats + ATT_MAXCL * ATT_MAXG * 2;      // [CL][G*hd]   (rank 0 only is read)
  float* red = part + (long)ATT_MAXCL * ATT_MAXG * hd; // [8][G*hd]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kvh = blockIdx.y / hsplit;
  const int h0 = kvh * Gall + (blockIdx.y % hsplit) * G;  // first q head of this CTA
  const bf16* kb = kc + (long)kvh * d.cap * hd;
  const bf16* vb = vc + (long)kvh * d.cap * hd;
  pdl_wait();
  const int nkeys = st->ctx + 1;
  const int chunk = (nkeys + CL - 1) / CL;
  const int k0 = min(nkeys, rank * chunk), k1 = min(nkeys, k0 + chunk);
  const int nloc = k1 - k0;

  float qs[ATT_MAXG][4];
#pragma unroll
  for (int g = 0; g < ATT_MAXG; ++g) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      qs[g][e] = 0.f;
      if (g < G && e < EPL)
        qs[g][e] = rbf(bf2f(qbuf[(long)(h0 + g) * hd + lane * EPL + e]) * d.scale_bf);
    }
  }
  // ---- scores (rounded to bf16) ----
  for (int j = warp; j < nloc; j += 8) {
    const bf16* kr = kb + (long)(k0 + j) * hd + lane * EPL;
    float kf[4] = {0.f, 0.f, 0.f, 0.f};
    if (EPL == 4) {
      unpack4(*reinterpret_cast<const uint2*>(kr), kf);
    } else {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(kr);
      kf[0] = __uint_as_float(w << 16);
      kf[1] = __uint_as_float(w & 0xffff0000u);
    }
    float s[ATT_MAXG];
#pragma unroll
    for (int g = 0; g < ATT_MAXG; ++g)
      s[g] = (g < G) ? qs[g][0] * kf[0] + qs[g][1] * kf[1] + qs[g][2] * kf[2] + qs[g][3] * kf[3] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int g = 0; g < ATT_MAXG; ++g)
        if (g < G) s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
    if (lane == 0) {
#pragma unroll
      for (int g = 0; g < ATT_MAXG; ++g)
        if (g < G) sc[(long)g * chunk_cap + j] = rbf(s[g]);
    }
  }
  __syncthreads();
  // ---- local max / sum(exp) per head (warp g), pushed to every rank ----
  if (warp < G) {
    float m = -INFINITY;
    for (int j = lane; j < nloc; j += 32) m = fmaxf(m, sc[(long)warp * chunk_cap + j]);
    m = warp_max(m);
    float l = 0.f;
    for (int j = lane; j < nloc; j += 32) l += expf(sc[(long)warp * chunk_cap + j] - m);
    l = warp_sum(l);
    if (nloc == 0) l = 0.f;
    if (lane < CL) {
      float* dst = cluster.map_shared_rank(stats, lane) + ((long)rank * ATT_MAXG + warp) * 2;
      dst[0] = m;
      dst[1] = l;
    }
  }
  cluster.sync();
  // ---- global statistics from LOCAL shared memory; p = bf16(exp(s - M) / L) ----
  if (warp < G) {
    float M = -INFINITY;
    for (int r = 0; r < CL; ++r) M = fmaxf(M, stats[((long)r * ATT_MAXG + warp) * 2]);
    float Ltot = 0.f;
    for (int r = 0; r < CL; ++r) {
      const float mr = stats[((long)r * ATT_MAXG + warp) * 2];
      const float lr = stats[((long)r * ATT_MAXG + warp) * 2 + 1];
      if (lr > 0.f) Ltot += lr * expf(mr - M);
    }
    for (int j = lane; j < nloc; j += 32) {
      float* p = &sc[(long)warp * chunk_cap + j];
      *p = rbf(expf(*p - M) / Ltot);
    }
  }
  __syncthreads();
  // ---- partial output: warp w takes keys w, w+8, ... ; lane owns EPL dims ----
  float acc[ATT_MAXG][4];
#pragma unroll
  for (int g = 0; g < ATT_MAXG; ++g)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[g][e] = 0.f;
  for (int j = warp; j < nloc; j += 8) {
    const bf16* vr = vb + (long)(k0 + j) * hd + lane * EPL;
    float vf[4] = {0.f, 0.f, 0.f, 0.f};
    if (EPL == 4) {
      unpack4(*reinterpret_cast<const uint2*>(vr), vf);
    } else {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(vr);
      vf[0] = __uint_as_float(w << 16);
      vf[1] = __uint_as_float(w & 0xffff0000u);
    }
#pragma unroll
    for (int g = 0; g < ATT_MAXG; ++g) {
      if (g < G) {
        const float p = sc[(long)g * chunk_cap + j];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[g][e] = fmaf(p, vf[e], acc[g][e]);
      }
    }
  }
#pragma unroll
  for (int g = 0; g < ATT_MAXG; ++g)
    if (g < G)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (e < EPL) red[((long)warp * G + g) * hd + lane * EPL + e] = acc[g][e];
  __syncthreads();
  float* part0 = cluster.map_shared_rank(part, 0) + (long)rank * ATT_MAXG * hd;
  for (int i = threadIdx.x; i < G * hd; i += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[(long)w * G * hd + i];
    part0[i] = s;  // push to rank 0
  }
  cluster.sync();
  if (rank == 0) {
    for (int i = threadIdx.x; i < G * hd; i += blockDim.x) {
      float s = 0.f;
      for (int r = 0; r < CL; ++r) s += part[(long)r * ATT_MAXG * hd + i];
      out[(long)h0 * hd + i] = f2bf(s);
    }
  }
}

// ---------------------------------------------------------------------------
// k_sample: logprobs = bf16(logits - bf16(logsumexp)), greedy argmax with the
// lowest index on ties (packed 64-bit atomicMax), last CTA finalises the step.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(256) k_sample(const DecodeDims d,
                                                const bf16* __restrict__ logits,
                                                const float2* __restrict__ partials, int n_part,
                                                bf16* __restrict__ logprobs,
                                                const bf16* __restrict__ E, bf16* __restrict__ h,
                                                DecState* __restrict__ st,
                                                int* __restrict__ token_log, int log_cap,
                                                const int* __restrict__ force_tokens,
                                                int advance) {
  __shared__ float s_lse;
  __shared__ unsigned long long s_best;
  __shared__ int s_last, s_feed;
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    float M = -INFINITY;
    for (int i = lane; i < n_part; i += 32) M = fmaxf(M, partials[i].x);
    M = warp_max(M);
    float L = 0.f;
    for (int i = lane; i < n_part; i += 32)
      if (partials[i].y > 0.f) L += partials[i].y * expf(partials[i].x - M);
    L = warp_sum(L);
    if (lane == 0) {
      s_lse = rbf(M + logf(L));
      s_best = 0ull;
    }
  }
  __syncthreads();
  const float lse = s_lse;
  unsigned long long best = 0ull;
  const int nvec = (d.vocab + 7) >> 3;  // the tail of an odd vocabulary holds -inf (preset at creation)
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < nvec; c += gridDim.x * blockDim.x) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(logits + (long)c * 8), f);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] = rbf(f[j] - lse);
      const unsigned long long key =
          ((unsigned long long)orderable(o[j]) << 32) | (0xFFFFFFFFu - (uint32_t)(c * 8 + j));
      best = key > best ? key : best;
    }
    uint4 ov;
    ov.x = pack2(o[0], o[1]);
    ov.y = pack2(o[2], o[3]);
    ov.z = pack2(o[4], o[5]);
    ov.w = pack2(o[6], o[7]);
    *reinterpret_cast<uint4*>(logprobs + (long)c * 8) = ov;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) atomicMax(&s_best, best);
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicMax(&st->best_key, s_best);
    __threadfence();
    const unsigned int done = atomicAdd(&st->blocks_done, 1u);
    s_last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  // ---- last CTA: finalise the step ----
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned long long key = atomicMax(&st->best_key, 0ull);  // read
    const int tok = (int)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
    const int n = st->n_out;
    token_log[n % log_cap] = tok;
    int feed = tok;
    if (st->use_force) feed = force_tokens[n % log_cap];
    s_feed = feed;
    st->tok = feed;
    st->n_out = n + 1;
    st->ctx += advance;  // 1 for a decode step, 0 for the prefill call (state pre-armed)
    st->pos += advance;
    st->best_key = 0ull;
    st->blocks_done = 0u;
  }
  __syncthreads();
  const int feed = s_feed;
  const int nv = d.hidden >> 3;
  for (int c = threadIdx.x; c < nv; c += blockDim.x)
    *reinterpret_cast<uint4*>(h + c * 8) =
        *reinterpret_cast<const uint4*>(E + (long)feed * d.hidden + c * 8);
}

// small kernel: arm / overwrite the decode state (after prefill, or explicitly)
__global__ void k_set_state(DecState* st, int tok, int ctx, int pos, int use_force, int set_tok,
                            const bf16* __restrict__ E, bf16* __restrict__ h, int hidden) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (set_tok) st->tok = tok;
    st->ctx = ctx;
    st->pos = pos;
    st->use_force = use_force;
  }
  if (set_tok) {
    const int nv = hidden >> 3;
    for (int c = threadIdx.x; c < nv; c += blockDim.x)
      *reinterpret_cast<uint4*>(h + c * 8) =
          *reinterpret_cast<const uint4*>(E + (long)tok * hidden + c * 8);
  }
}

// ---------------------------------------------------------------------------
// host-side launchers
// ---------------------------------------------------------------------------
static int g_sm_count = 132;
static bool g_pdl = false;  // off by default; programmatic dependent launch for this kernel mix: not measured on the H100
void decode_set_sm_count(int n) { g_sm_count = n > 0 ? n : 132; }
void decode_set_pdl(bool on) { g_pdl = on; }

template <typename... KArgs, typename... Args>
static int launch_ex(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                     int cluster_x, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (g_pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  B200_CUDA(cudaLaunchKernelEx(&cfg, kern, KArgs(args)...));
  return B200_OK;
}

// tile geometry: R row(-pair)s per tile (R*S == 8 consumer warps), stage <= ~50 KB
static int stream_geometry(StreamP& p, bool pair, int units /*rows or pairs available*/) {
  const long unit = (long)p.K * 2 * (pair ? 2 : 1);
  int R = 8;
  while (R > 1 && (R * unit > 50 * 1024 || R > units)) R >>= 1;
  // fewer rows per tile -> more K slices: keep the activation slice within the 10 chunks per lane of the largest
  // k_stream instantiation (e.g. K = 6144: 4 rows would need 12)
  while (R > 1 && cdiv(cdiv(p.K >> 3, 8 / R), 32) > 10) R >>= 1;
  B200_REQUIRE(R * unit <= STREAM_SMEM_BUDGET / 2, "decode: K=%d too large for the weight ring", p.K);
  p.R = R;
  p.S = 8 / R;
  p.stage_bytes = (int)(R * unit);
  int ns = STREAM_SMEM_BUDGET / p.stage_bytes;
  p.n_stages = ns > 8 ? 8 : ns;
  return B200_OK;
}

template <int MODE>
static int launch_stream(const StreamP& p, int max_ctas, cudaStream_t s) {
  const int nvec = p.K >> 3;
  const int chx = cdiv(cdiv(nvec, p.S), 32);
  const int grid = p.tiles < max_ctas ? p.tiles : max_ctas;
  const size_t smem = (size_t)p.n_stages * p.stage_bytes;
  if (chx <= 2) return launch_ex(k_stream<MODE, 2>, dim3(grid), dim3(STREAM_THREADS), smem, s, 1, p);
  if (chx <= 6) return launch_ex(k_stream<MODE, 6>, dim3(grid), dim3(STREAM_THREADS), smem, s, 1, p);
  if (chx <= 10) return launch_ex(k_stream<MODE, 10>, dim3(grid), dim3(STREAM_THREADS), smem, s, 1, p);
  set_error("decode: K=%d needs %d activation chunks per lane (max 10)", p.K, chx);
  return B200_ERR_INVALID;
}

// every kernel of the decode step asks for the SAME (maximum) shared-memory carve-out:
// a carve-out change between kernels needs an idle SM and would forbid the
// co-residency of consecutive kernels that PDL relies on.
template <typename F>
static int set_carveout(F kern, int dyn_smem) {
  if (dyn_smem > 0)
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_smem));
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
  return B200_OK;
}
template <int MODE, int CHX>
static int set_stream_attr() {
  return set_carveout(k_stream<MODE, CHX>, STREAM_SMEM_BUDGET);
}

static int attn_hsplit(const DecodeDims& d, int gmax) {
  const int G = d.n_heads / d.n_kv;
  int hs = 1;
  while (G / hs > gmax || (G % hs) != 0) ++hs;
  if (hs == 1 && G % 2 == 0 && G >= 4) hs = 2;
  return hs;
}

constexpr int ATT1_MAX_CAP = 4096;
static size_t attn1_smem(const DecodeDims& d) {
  return ((size_t)ATT1_G * d.hd + (size_t)ATT1_G * d.cap + (size_t)8 * ATT1_G * d.hd) * 4;
}
size_t attn_smem_bytes(const DecodeDims& d, int chunk_cap) {
  return ((size_t)ATT_MAXG * chunk_cap + (size_t)ATT_MAXCL * ATT_MAXG * 2 +
          (size_t)ATT_MAXCL * ATT_MAXG * d.hd + (size_t)8 * ATT_MAXG * d.hd) * 4;
}

int decode_prepare(const DecodeDims& d, int cluster) {
  int rc;
  if ((rc = set_stream_attr<SM_QKV, 2>()) || (rc = set_stream_attr<SM_QKV, 6>()) ||
      (rc = set_stream_attr<SM_QKV, 10>()) || (rc = set_stream_attr<SM_ORES, 2>()) ||
      (rc = set_stream_attr<SM_ORES, 6>()) || (rc = set_stream_attr<SM_ORES, 10>()) ||
      (rc = set_stream_attr<SM_GATEUP, 2>()) || (rc = set_stream_attr<SM_GATEUP, 6>()) ||
      (rc = set_stream_attr<SM_GATEUP, 10>()) || (rc = set_stream_attr<SM_DRES, 2>()) ||
      (rc = set_stream_attr<SM_DRES, 6>()) || (rc = set_stream_attr<SM_DRES, 10>()) ||
      (rc = set_stream_attr<SM_HEAD, 2>()) || (rc = set_stream_attr<SM_HEAD, 6>()) ||
      (rc = set_stream_attr<SM_HEAD, 10>()))
    return rc;
  if (d.cap <= ATT1_MAX_CAP) {
    const size_t smem = attn1_smem(d);
    B200_REQUIRE(smem <= 220 * 1024, "decode attention: cache capacity %d too large", d.cap);
    if ((rc = set_carveout(k_attn1<128>, (int)smem)) || (rc = set_carveout(k_attn1<64>, (int)smem)))
      return rc;
  } else {
    const size_t smem = attn_smem_bytes(d, cdiv(d.cap, cluster));
    B200_REQUIRE(smem <= 220 * 1024, "decode attention: cache capacity %d too large", d.cap);
    if ((rc = set_carveout(k_attn, (int)smem))) return rc;
  }
  if ((rc = set_carveout(k_sample, 0)) || (rc = set_carveout(k_set_state, 0)) ||
      (rc = set_carveout(k_qk_norm_rope<4>, 0)) || (rc = set_carveout(k_qk_norm_rope<2>, 0)))
    return rc;
  return B200_OK;
}

int launch_qkv(const DecodeDims& d, const LayerW& lw, const bf16* h, bf16* qbuf, bf16* kc,
               bf16* vc, const DecState* st, const float* inv_freq, cudaStream_t s, const bf16* qn,
               const bf16* kn) {
  StreamP p = {};
  p.W = lw.wqkv; p.bias = lw.bqkv; p.x = h; p.lnw = lw.ln1; p.out = qbuf; p.kc = kc; p.vc = vc;
  p.st = st; p.inv_freq = inv_freq; p.K = d.hidden; p.N = 0;
  p.n_heads = d.n_heads; p.n_kv = d.n_kv; p.hd = d.hd; p.cap = d.cap; p.eps = d.eps;
  p.raw_qk = qn != nullptr;
  const int half = d.hd / 2;
  int rc = stream_geometry(p, true, half);
  if (rc) return rc;
  B200_REQUIRE(half % p.R == 0, "decode qkv: head_dim/2=%d not a multiple of tile rows %d", half, p.R);
  p.tiles = (d.n_heads + 2 * d.n_kv) * (half / p.R);
  if ((rc = launch_stream<SM_QKV>(p, g_sm_count, s)) || !qn) return rc;
  B200_REQUIRE(kn && (d.hd == 64 || d.hd == 128), "decode q/k norm: head_dim=%d (64 | 128)", d.hd);
  const dim3 grid(cdiv(d.n_heads + d.n_kv, 8));
  if (d.hd == 128) return launch_ex(k_qk_norm_rope<4>, grid, dim3(256), 0, s, 1, d, qbuf, kc, st, inv_freq, qn, kn);
  return launch_ex(k_qk_norm_rope<2>, grid, dim3(256), 0, s, 1, d, qbuf, kc, st, inv_freq, qn, kn);
}

int launch_attn(const DecodeDims& d, const bf16* qbuf, const bf16* kc, const bf16* vc, bf16* out,
                const DecState* st, int cluster, cudaStream_t s) {
  B200_REQUIRE(d.hd == 64 || d.hd == 128, "decode attention: head_dim=%d (64|128)", d.hd);
  if (d.cap <= ATT1_MAX_CAP) {
    const int hs = attn_hsplit(d, ATT1_G);
    if (d.hd == 128)
      return launch_ex(k_attn1<128>, dim3(d.n_kv * hs), dim3(256), attn1_smem(d), s, 1, d, qbuf, kc,
                       vc, out, st, hs);
    return launch_ex(k_attn1<64>, dim3(d.n_kv * hs), dim3(256), attn1_smem(d), s, 1, d, qbuf, kc, vc,
                     out, st, hs);
  }
  const int hs = attn_hsplit(d, ATT_MAXG);
  B200_REQUIRE(cluster <= ATT_MAXCL, "decode attention: cluster %d > %d", cluster, ATT_MAXCL);
  const int chunk_cap = cdiv(d.cap, cluster);
  return launch_ex(k_attn, dim3(cluster, d.n_kv * hs, 1), dim3(256), attn_smem_bytes(d, chunk_cap),
                   s, cluster, d, qbuf, kc, vc, out, st, chunk_cap, hs);
}

int launch_res(const bf16* W, const bf16* x, bf16* h, int N, int K, cudaStream_t s) {
  StreamP p = {};
  p.W = W; p.x = x; p.out = h; p.N = N; p.K = K;
  int rc = stream_geometry(p, false, N);
  if (rc) return rc;
  p.tiles = cdiv(N, p.R);
  return p.S == 1 ? launch_stream<SM_ORES>(p, g_sm_count, s) : launch_stream<SM_DRES>(p, g_sm_count, s);
}

int launch_gateup(const DecodeDims& d, const LayerW& lw, const bf16* h, bf16* act,
                  cudaStream_t s) {
  StreamP p = {};
  p.W = lw.wgu; p.W2 = lw.wgu + (long)d.inter * d.hidden; p.x = h; p.lnw = lw.ln2; p.out = act;
  p.N = d.inter; p.K = d.hidden; p.eps = d.eps;
  int rc = stream_geometry(p, true, d.inter);
  if (rc) return rc;
  p.tiles = cdiv(d.inter, p.R);
  return launch_stream<SM_GATEUP>(p, g_sm_count, s);
}

// CTAs of the head kernel (== number of logsumexp partials k_sample reduces)
static int head_ctas(const DecodeDims& d) {
  StreamP p = {};
  p.K = d.hidden;
  if (stream_geometry(p, false, d.vocab)) return 1;
  const int tiles = cdiv(d.vocab, p.R);
  return tiles < g_sm_count * 2 ? tiles : g_sm_count * 2;
}
int head_grid() { return g_sm_count * 2; }

int launch_head(const DecodeDims& d, const bf16* norm_w, const bf16* E, const bf16* h,
                bf16* logits, float2* partials, cudaStream_t s) {
  StreamP p = {};
  p.W = E; p.x = h; p.lnw = norm_w; p.out = logits; p.partials = partials; p.N = d.vocab;
  p.K = d.hidden; p.eps = d.eps;
  int rc = stream_geometry(p, false, d.vocab);
  if (rc) return rc;
  p.tiles = cdiv(d.vocab, p.R);
  return launch_stream<SM_HEAD>(p, head_ctas(d), s);
}

int launch_sample(const DecodeDims& d, const bf16* logits, const float2* partials, bf16* logprobs,
                  const bf16* E, bf16* h, DecState* st, int* token_log, int log_cap,
                  const int* force_tokens, int advance, cudaStream_t s) {
  return launch_ex(k_sample, dim3(g_sm_count), dim3(256), 0, s, 1, d, logits, partials,
                   head_ctas(d), logprobs, E, h, st, token_log, log_cap, force_tokens, advance);
}

int launch_set_state(DecState* st, int tok, int ctx, int pos, int use_force, int set_tok,
                     const bf16* E, bf16* h, int hidden, cudaStream_t s) {
  k_set_state<<<1, 256, 0, s>>>(st, tok, ctx, pos, use_force, set_tok, E, h, hidden);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200
