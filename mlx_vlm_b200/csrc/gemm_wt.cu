// gemm_wt: the Linear layers of the prefill / vision / batched-decode paths as a WEIGHT-MAJOR
// wgmma GEMM:   D[n, t] = sum_k W[n, k] * X[t, k]      (C[t, n] = D[n, t])
//
// Why weight-major ("swap AB"): the token count of this path is small and awkward for a 64- or
// 128-row M side, while the weight rows are many and regular.  So the weight rows take the M side
// (128 rows per CTA, 64 per consumer warpgroup, streamed exactly once per token tile) and the
// tokens the N side, whose width TN is any multiple of 16 up to 256 and is chosen per problem.
//
//   * TMA (cp.async.bulk.tensor, 128B swizzle) feeds a shared-memory ring of `n_stages` stages
//     of KS k-blocks (64 columns each); warpgroup 0 is the producer, warpgroups 1 and 2 issue
//     wgmma m64n16k16 per 16 tokens (fp32 accumulators in registers);
//   * programmatic dependent launch: the weight tiles of the first stages do not depend on the
//     previous kernel and are requested BEFORE griddepcontrol.wait, so the cold-HBM latency of a
//     layer's weights overlaps the previous kernel's tail;
//   * split-K over gridDim.z for the GEMMs with few weight rows and long K (o_proj, down, fc2):
//     fp32 partial tiles, summed in a FIXED order by the row-op kernel that follows
//     (finish_rows: bias + residual + RMSNorm / LayerNorm of the next block, fused);
//   * epilogue: registers -> transposed through shared memory -> coalesced 16-byte rows of C
//     (bias / GELU / residual), or SwiGLU of interleaved gate/up row blocks (64 + 64 rows per
//     tile, two TMA boxes), or fp32 partial tiles.
//
// Replaces nn.Linear of the reference (models/qwen2_vl/vision.py:83-102,108-119,132-133,168-169;
// language.py:52-55; mlp.py:9-15; activations.py:8-10).  Rounding points follow
// oracle/mlx_semantics.py::linear (+ activations, residual add).
#include <array>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int WT_ROWS = 128;        // weight rows per CTA (the wgmma M side)
constexpr int WT_BK = 64;           // one k-block: 64 bf16 = 128 B = one swizzle row
constexpr int WT_WBLK = WT_ROWS * 128;  // bytes of one weight k-block tile
constexpr int WT_MAX_STAGES = 16;
constexpr int WT_EPI_TOK = 64;      // tokens staged per epilogue pass
constexpr int WT_THREADS = 384;    // producer warpgroup + 2 consumer warpgroups
constexpr int WT_TN_AUTO = 128;    // widest token tile the automatic / measured choice uses

struct WtParams {
  const bf16* bias;
  const bf16* residual;
  bf16* C;
  float* partial;
  long ldc, ldr;
  int T, N, K;
  int TN, KS, n_stages;
  int kb_per_split;
  int epilogue, mode;
  int inter;
  unsigned flags;  // debug: 1 = no MMA (loads only), 2 = no loads (MMA on stale smem), 4 = no epilogue stores
  // fp32-accurate towers (LLaVA / Idefics2: the reference runs them in fp32 with bf16-valued weights):
  // X is a SPLIT operand [x_hi | x_lo] (n parts of K_w columns, each padded to 64) multiplied by the SAME
  // weight k-blocks (kb_w of them): D = W.x_hi + W.x_lo in fp32 — exact to ~2^-17 relative.
  int kb_w;          // > 0: weight k-block = k-block % kb_w
  float* C32;        // B200_WT_F32: fp32 output (bias, activation, fp32 residual)
  const float* res32;
  long ldc32, ldr32;
  bf16* Csplit;      // B200_WT_SPLIT: output written as [hi | lo] bf16 halves, n_pad columns apart
  long ld_split;
  int n_pad;
};

__device__ __forceinline__ void w_ebar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // the 2 consumer warpgroups

// accumulator -> bf16 staging element: + bias, one rounding, activation
template <int EPI>
__device__ __forceinline__ bf16 wt_stage_bf16(float acc, float bias_v) {
  float v = rbf(acc + bias_v);
  if constexpr (EPI == B200_EPI_GELU_FAST) v = gelu_fast_bf(v);
  if constexpr (EPI == B200_EPI_GELU_EXACT) v = gelu_exact_bf(v);
  return f2bf(v);
}

// the fp32-accurate paths: no rounding anywhere
template <int EPI>
__device__ __forceinline__ float wt_stage_f32(float acc, float bias_v) {
  float v = acc + bias_v;
  if constexpr (EPI == B200_EPI_GELU_FAST) v = v * sigmoid_f(1.702f * v);
  if constexpr (EPI == B200_EPI_GELU_EXACT) v = v * (1.0f + erff(v / 1.41421356237309515f)) * 0.5f;
  if constexpr (EPI == B200_EPI_GELU_TANH) {
    const float u = 0.7978845608028654f * (v + 0.044715f * v * v * v);
    v = 0.5f * v * (1.0f + tanhf(u));
  }
  return v;
}

// Accumulator chunks (16 tokens each) of pass c0 -> staging tile [token][weight row].  KIND: 0 = raw fp32
// (partial tiles), 1 = bf16 with the epilogue EPI, 2 = fp32 with the epilogue EPI.
template <int KIND, int EPI, int WT_MAX_CH>
__device__ __forceinline__ void wt_stage(const float (&acc)[WT_MAX_CH][8], int n_ch, int c0, int row_lo,
                                         const float (&bias_v)[2], uint8_t* stg) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < WT_MAX_CH; ++c) {
    if (c >= n_ch || c * 16 < c0 || c * 16 >= c0 + WT_EPI_TOK) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int hr = (i >> 1) & 1;
      const int row = row_lo + 8 * hr;
      const int tl = c * 16 - c0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      if constexpr (KIND == 0) reinterpret_cast<float*>(stg)[tl * WT_ROWS + row] = acc[c][i];
      else if constexpr (KIND == 1) reinterpret_cast<bf16*>(stg)[tl * WT_ROWS + row] = wt_stage_bf16<EPI>(acc[c][i], bias_v[hr]);
      else reinterpret_cast<float*>(stg)[tl * WT_ROWS + row] = wt_stage_f32<EPI>(acc[c][i], bias_v[hr]);
    }
  }
}

// TOWER = false: the bf16 paths (B200_WT_BF16 / PARTIAL / SWIGLU); TOWER = true: the fp32-accurate paths
// (B200_WT_F32 / SPLIT).  Two instantiations keep each one's code small (tools/wt_ab_probe.py A/B-times builds).
// WT_MAX_CH: 16-token accumulator chunks per thread, 8 (TN <= 128) or 16 (TN <= 256).  The 16-chunk
// instantiation spills (168 registers per thread at 384 threads); it serves explicit configurations
// only, the automatic and measured choices stay at TN <= WT_TN_AUTO.
template <bool TOWER, int WT_MAX_CH>
__global__ void __launch_bounds__(WT_THREADS, 1)
gemm_wt_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
               const WtParams p) {
  extern __shared__ uint8_t wt_smem_raw[];
  __shared__ uint64_t full_bar[WT_MAX_STAGES], empty_bar[WT_MAX_STAGES];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wt_smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const bool swiglu = !TOWER && (p.mode == B200_WT_SWIGLU);
  const int rb = blockIdx.x;
  const int n0 = rb * (swiglu ? 64 : WT_ROWS);  // first output feature (SwiGLU: channel) of the tile
  const int t0 = blockIdx.y * p.TN;
  const int split = blockIdx.z;
  const int kb_total = (p.K + WT_BK - 1) / WT_BK;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(kb_total, kb0 + p.kb_per_split);
  const int n_it = (kb1 - kb0 + p.KS - 1) / p.KS;
  const int xblk = p.TN * 128;                      // bytes of one token k-block tile
  const int stage_bytes = p.KS * (WT_WBLK + xblk);
  const int NS = p.n_stages;

  pdl_launch_dependents();  // the next kernel may start its prologue / weight prefetch as SM resources free up

  auto issue_w = [&](int it, int s) {
    uint8_t* sW = ring + (long)s * stage_bytes;
    const int cnt = min(p.KS, kb1 - kb0 - it * p.KS);
    if (p.flags & 2u) {  // debug: no loads at all, the MMAs run on whatever the ring holds
      mbar_arrive(&full_bar[s]);
      return;
    }
    mbar_expect_tx(&full_bar[s], (uint32_t)cnt * (WT_WBLK + xblk));
    for (int j = 0; j < cnt; ++j) {
      int kbw = kb0 + it * p.KS + j;
      if (p.kb_w > 0) kbw %= p.kb_w;
      const int kc = kbw * WT_BK;
      if (swiglu) {
        tma_2d(sW + j * WT_WBLK, &tmW, &full_bar[s], kc, n0);
        tma_2d(sW + j * WT_WBLK + 64 * 128, &tmW, &full_bar[s], kc, p.inter + n0);
      } else {
        tma_2d(sW + j * WT_WBLK, &tmW, &full_bar[s], kc, n0);
      }
    }
  };
  auto issue_x = [&](int it, int s) {
    if (p.flags & 2u) return;
    uint8_t* sX = ring + (long)s * stage_bytes + p.KS * WT_WBLK;
    const int cnt = min(p.KS, kb1 - kb0 - it * p.KS);
    for (int j = 0; j < cnt; ++j)
      tma_2d(sX + j * xblk, &tmX, &full_bar[s], (kb0 + it * p.KS + j) * WT_BK, t0);
  };

  const int pre = n_it < NS ? n_it : NS;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmX)) : "memory");
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
    // weights never depend on the previous kernel: request them before waiting for it
    for (int it = 0; it < pre; ++it) issue_w(it, it);
  }
  __syncthreads();
  pdl_wait();  // everything the previous kernels wrote (X, residual) is visible from here on

  if (wg == 0) {
    if (threadIdx.x == 0) {  // ===== TMA producer =====
      for (int it = 0; it < pre; ++it) issue_x(it, it);
      for (int it = pre; it < n_it; ++it) {
        const int s = it % NS;
        mbar_wait(&empty_bar[s], ((it / NS) & 1) ^ 1);
        issue_w(it, s);
        issue_x(it, s);
      }
    }
    return;
  }

  // ===== consumers: warpgroup c = wg - 1 multiplies weight rows [64 c, 64 c + 64) by the TN tokens,
  // 16 tokens per wgmma (accumulator chunk ch = tokens [16 ch, 16 ch + 16)) =====
  const int c = wg - 1;
  const int n_ch = p.TN >> 4;
  float acc[WT_MAX_CH][8];
#pragma unroll
  for (int ch = 0; ch < WT_MAX_CH; ++ch)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[ch][i] = 0.f;
  for (int it = 0; it < n_it; ++it) {
    const int s = it % NS;
    mbar_wait(&full_bar[s], (it / NS) & 1);
    if (!(p.flags & 1u)) {
      const uint32_t w_a = smem_u32(ring + (long)s * stage_bytes) + c * 64 * 128;
      const uint32_t x_a = smem_u32(ring + (long)s * stage_bytes + p.KS * WT_WBLK);
      const int cnt = min(p.KS, kb1 - kb0 - it * p.KS);
#pragma unroll
      for (int ch = 0; ch < WT_MAX_CH; ++ch) wg_fence_acc(acc[ch]);
      wg_arrive();
      for (int j = 0; j < cnt; ++j) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t dw = wg_desc(w_a + j * WT_WBLK + kk * 32);
#pragma unroll
          for (int ch = 0; ch < WT_MAX_CH; ++ch)
            if (ch < n_ch) wgmma_n16_ss(acc[ch], dw, wg_desc(x_a + j * xblk + ch * 2048 + kk * 32), 1u);
        }
      }
      wg_commit();
      wg_wait<0>();
#pragma unroll
      for (int ch = 0; ch < WT_MAX_CH; ++ch) wg_fence_acc(acc[ch]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);  // this warp's MMAs have read the ring slot
  }

  // ===== epilogue (the 256 consumer threads) =====
  const int tid = threadIdx.x - 128;
  const int row_lo = c * 64 + ((tid >> 5) & 3) * 16 + (lane >> 2);  // weight rows row_lo and row_lo + 8
  float bias_v[2] = {0.f, 0.f};
  if ((TOWER || p.mode == B200_WT_BF16) && p.bias) {
    if (n0 + row_lo < p.N) bias_v[0] = bf2f(p.bias[n0 + row_lo]);
    if (n0 + row_lo + 8 < p.N) bias_v[1] = bf2f(p.bias[n0 + row_lo + 8]);
  }
  uint8_t* stg = ring;  // reused once both warpgroups have finished reading the ring
  w_ebar();
  for (int c0 = 0; c0 < p.TN; c0 += WT_EPI_TOK) {
    if (!(p.flags & 1u)) {
      if (!TOWER && p.mode == B200_WT_PARTIAL) {
        wt_stage<0, B200_EPI_NONE, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
      } else if constexpr (TOWER) {
        if (p.epilogue == B200_EPI_GELU_FAST) wt_stage<2, B200_EPI_GELU_FAST, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
        else if (p.epilogue == B200_EPI_GELU_EXACT) wt_stage<2, B200_EPI_GELU_EXACT, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
        else if (p.epilogue == B200_EPI_GELU_TANH) wt_stage<2, B200_EPI_GELU_TANH, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
        else wt_stage<2, B200_EPI_NONE, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
      } else {
        // one unrolled loop per epilogue kind, chosen OUTSIDE the loop: left to itself the compiler merges the
        // three kinds into one predicated body per element
        if (p.epilogue == B200_EPI_GELU_FAST) wt_stage<1, B200_EPI_GELU_FAST, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
        else if (p.epilogue == B200_EPI_GELU_EXACT) wt_stage<1, B200_EPI_GELU_EXACT, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
        else wt_stage<1, B200_EPI_NONE, WT_MAX_CH>(acc, n_ch, c0, row_lo, bias_v, stg);
      }
    }
    w_ebar();
    if (!(p.flags & 4u)) {
      if (!TOWER && p.mode == B200_WT_BF16) {
        const bool vec_all = ((p.ldc & 7) == 0) && (!p.residual || (p.ldr & 7) == 0) &&
                            ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) &&
                            (!p.residual || (reinterpret_cast<uintptr_t>(p.residual) & 15) == 0);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int idx = tid + 256 * u;
          const int tl = idx >> 4, ch = idx & 15;
          const int t = t0 + c0 + tl, n = n0 + ch * 8;
          if (c0 + tl >= p.TN || t >= p.T || n >= p.N) continue;
          const uint4 sv = *reinterpret_cast<const uint4*>(stg + (tl * WT_ROWS + ch * 8) * 2);
          const bool vec_ok = vec_all && n + 8 <= p.N;  // only the last chunk of an odd N goes element-wise
          if (vec_ok) {
            uint4 o = sv;
            if (p.residual) {
              float r[8], v[8];
              unpack8(*reinterpret_cast<const uint4*>(p.residual + (long)t * p.ldr + n), r);
              unpack8(sv, v);
#pragma unroll
              for (int e = 0; e < 8; ++e) v[e] = rbf(r[e] + v[e]);
              o.x = pack2(v[0], v[1]); o.y = pack2(v[2], v[3]); o.z = pack2(v[4], v[5]); o.w = pack2(v[6], v[7]);
            }
            *reinterpret_cast<uint4*>(p.C + (long)t * p.ldc + n) = o;
          } else {
            float v[8];
            unpack8(sv, v);
            for (int e = 0; e < 8 && n + e < p.N; ++e) {
              float o = v[e];
              if (p.residual) o = rbf(bf2f(p.residual[(long)t * p.ldr + n + e]) + o);
              p.C[(long)t * p.ldc + n + e] = f2bf(o);
            }
          }
        }
      } else if (!TOWER && p.mode == B200_WT_SWIGLU) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int idx = tid + 256 * u;
          const int tl = idx >> 3, ch = idx & 7;
          const int t = t0 + c0 + tl, i = n0 + ch * 8;
          if (c0 + tl >= p.TN || t >= p.T || i >= p.inter) continue;
          float g[8], uu[8], o[8];
          unpack8(*reinterpret_cast<const uint4*>(stg + (tl * WT_ROWS + ch * 8) * 2), g);
          unpack8(*reinterpret_cast<const uint4*>(stg + (tl * WT_ROWS + 64 + ch * 8) * 2), uu);
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = swiglu_bf(g[e], uu[e]);
          uint4 ov;
          ov.x = pack2(o[0], o[1]); ov.y = pack2(o[2], o[3]); ov.z = pack2(o[4], o[5]); ov.w = pack2(o[6], o[7]);
          *reinterpret_cast<uint4*>(p.C + (long)t * p.ldc + i) = ov;
        }
      } else if constexpr (TOWER) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int idx = tid + 256 * u;
          const int tl = idx >> 5, ch = idx & 31;
          const int t = t0 + c0 + tl, n = n0 + ch * 4;
          if (c0 + tl >= p.TN || t >= p.T || n >= p.N) continue;
          float4 v = *reinterpret_cast<const float4*>(stg + (tl * WT_ROWS + ch * 4) * 4);
          if (p.mode == B200_WT_F32) {
            float* dst = p.C32 + (long)t * p.ldc32 + n;
            if (n + 4 <= p.N && (p.ldc32 & 3) == 0) {
              if (p.res32) {
                const float4 r = *reinterpret_cast<const float4*>(p.res32 + (long)t * p.ldr32 + n);
                v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
              }
              *reinterpret_cast<float4*>(dst) = v;
            } else {
              const float vv[4] = {v.x, v.y, v.z, v.w};
              for (int e = 0; e < 4 && n + e < p.N; ++e)
                dst[e] = vv[e] + (p.res32 ? p.res32[(long)t * p.ldr32 + n + e] : 0.f);
            }
          } else {  // [hi | lo]: hi = bf16(v), lo = bf16(v - hi)
            const float vv[4] = {v.x, v.y, v.z, v.w};
            float hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              hi[e] = rbf(vv[e]);
              lo[e] = vv[e] - hi[e];
            }
            bf16* dh = p.Csplit + (long)t * p.ld_split + n;
            if (n + 4 <= p.N) {
              *reinterpret_cast<uint2*>(dh) = make_uint2(pack2(hi[0], hi[1]), pack2(hi[2], hi[3]));
              *reinterpret_cast<uint2*>(dh + p.n_pad) = make_uint2(pack2(lo[0], lo[1]), pack2(lo[2], lo[3]));
            } else {
              for (int e = 0; e < 4 && n + e < p.N; ++e) {
                dh[e] = f2bf(hi[e]);
                dh[p.n_pad + e] = f2bf(lo[e]);
              }
            }
          }
        }
      } else {  // fp32 partial tile -> P[split][t][n]
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int idx = tid + 256 * u;
          const int tl = idx >> 5, ch = idx & 31;
          const int t = t0 + c0 + tl, n = n0 + ch * 4;
          if (c0 + tl >= p.TN || t >= p.T || n >= p.N) continue;
          const float4 v = *reinterpret_cast<const float4*>(stg + (tl * WT_ROWS + ch * 4) * 4);
          float* dst = p.partial + ((long)split * p.T + t) * p.N + n;
          if (n + 4 <= p.N && (p.N & 3) == 0) {
            *reinterpret_cast<float4*>(dst) = v;
          } else {
            const float vv[4] = {v.x, v.y, v.z, v.w};
            for (int e = 0; e < 4 && n + e < p.N; ++e) dst[e] = vv[e];
          }
        }
      }
    }
    w_ebar();
  }
}

// ---------------------------------------------------------------------------------------------
// finish_rows: h[t] = r(resid[t] + r(sum_s P[s][t] + bias)) and, fused, the normalisation that
// the NEXT block applies to h (RMSNorm / LayerNorm with the oracle's rounding points).  One CTA
// per token row; the split-K partials are added in split order (deterministic).
// ---------------------------------------------------------------------------------------------
// <256 threads, 8 vectors> for sequences (one CTA per row, many rows) and <1024, 2> for the few rows of a batched
// decode step: there the kernel is a chain of L2 round trips, and 1024 threads issue every load of a row at once
constexpr int FIN_N_MAX = 8192;  // N <= FIN_THREADS * 4 * FIN_MAXV in both shapes

template <int FIN_THREADS, int FIN_MAXV>
__global__ void __launch_bounds__(FIN_THREADS)
finish_rows_kernel(const float* __restrict__ P, int S, const bf16* __restrict__ bias,
                   const bf16* __restrict__ resid, long ldr, bf16* __restrict__ h_out, long ldh,
                   int norm_kind, const bf16* __restrict__ nw, const bf16* __restrict__ nb, float eps,
                   bf16* __restrict__ xn, long ldx, int T, int N) {
  __shared__ float red[FIN_THREADS / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const int nv = N >> 2;
  float4 h[FIN_MAXV];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int u = 0; u < FIN_MAXV; ++u) {
    const int c = threadIdx.x + FIN_THREADS * u;
    h[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nv) {
      // the split-K partials of this chunk: up to 8 loads in flight, added in split order
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = 0; s0 < S; s0 += 8) {
        float4 v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
          v[i] = (s0 + i < S) ? __ldcg(reinterpret_cast<const float4*>(P + ((long)(s0 + i) * T + t) * N + c * 4))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          a.x += v[i].x; a.y += v[i].y; a.z += v[i].z; a.w += v[i].w;
        }
      }
      if (bias) {
        float bb[4];
        unpack4(*reinterpret_cast<const uint2*>(bias + c * 4), bb);
        a.x += bb[0]; a.y += bb[1]; a.z += bb[2]; a.w += bb[3];
      }
      a.x = rbf(a.x); a.y = rbf(a.y); a.z = rbf(a.z); a.w = rbf(a.w);
      if (resid) {
        float rr[4];
        unpack4(*reinterpret_cast<const uint2*>(resid + (long)t * ldr + c * 4), rr);
        a.x = rbf(rr[0] + a.x); a.y = rbf(rr[1] + a.y); a.z = rbf(rr[2] + a.z); a.w = rbf(rr[3] + a.w);
      }
      h[u] = a;
      if (h_out)
        *reinterpret_cast<uint2*>(h_out + (long)t * ldh + c * 4) = make_uint2(pack2(a.x, a.y), pack2(a.z, a.w));
      s1 += (a.x + a.y) + (a.z + a.w);
      s2 += (a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w);
    }
  }
  if (norm_kind == B200_NORM_NONE) return;
  if (norm_kind == B200_NORM_RMS) {
    const float tot = block_sum<FIN_THREADS / 32>(s2, red);
    const float rs = 1.0f / sqrtf(tot / (float)N + eps);
#pragma unroll
    for (int u = 0; u < FIN_MAXV; ++u) {
      const int c = threadIdx.x + FIN_THREADS * u;
      if (c < nv) {
        float w[4];
        unpack4(*reinterpret_cast<const uint2*>(nw + c * 4), w);
        const float4 a = h[u];
        *reinterpret_cast<uint2*>(xn + (long)t * ldx + c * 4) =
            make_uint2(pack2(rbf(rbf(a.x * rs) * w[0]), rbf(rbf(a.y * rs) * w[1])),
                       pack2(rbf(rbf(a.z * rs) * w[2]), rbf(rbf(a.w * rs) * w[3])));
      }
    }
    return;
  }
  // LayerNorm: fp32 mean / variance (two passes over the registers), cast, * w, + b
  const float mu = block_sum<FIN_THREADS / 32>(s1, red) / (float)N;
  float v = 0.f;
#pragma unroll
  for (int u = 0; u < FIN_MAXV; ++u) {
    const int c = threadIdx.x + FIN_THREADS * u;
    if (c < nv) {
      const float4 a = h[u];
      const float d0 = a.x - mu, d1 = a.y - mu, d2 = a.z - mu, d3 = a.w - mu;
      v += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
  }
  const float var = block_sum<FIN_THREADS / 32>(v, red) / (float)N;
  const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
  for (int u = 0; u < FIN_MAXV; ++u) {
    const int c = threadIdx.x + FIN_THREADS * u;
    if (c < nv) {
      const float4 a = h[u];
      float o[4] = {rbf((a.x - mu) * rstd), rbf((a.y - mu) * rstd), rbf((a.z - mu) * rstd),
                    rbf((a.w - mu) * rstd)};
      if (nw) {
        float w[4];
        unpack4(*reinterpret_cast<const uint2*>(nw + c * 4), w);
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = rbf(o[e] * w[e]);
      }
      if (nb) {
        float b[4];
        unpack4(*reinterpret_cast<const uint2*>(nb + c * 4), b);
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = rbf(o[e] + b[e]);
      }
      *reinterpret_cast<uint2*>(xn + (long)t * ldx + c * 4) = make_uint2(pack2(o[0], o[1]), pack2(o[2], o[3]));
    }
  }
}

// 2-D K-major bf16 operand (rows x K, row pitch ld elements), box = box_rows x 64
int wt_tmap(const void* ptr, long ld, int rows, int k, int box_rows, CUtensorMap* out) {
  const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)WT_BK, (cuuint32_t)box_rows};
  return bf16_tmap(2, ptr, dims, strides, box, out);
}

// (ptr, rank, dims[3], strides[2], box[3]) of a tensor map, unused entries 0
typedef std::array<cuuint64_t, 10> TmapKey;
struct TmapHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = 0;
    for (cuuint64_t v : k) h = h * 1000003u ^ std::hash<cuuint64_t>()(v);
    return h;
  }
};

}  // namespace

// ---- host: tensor maps (declared in wgmma.cuh; gemm_wt and attention_fa) ---------------------
int bf16_tmap(int rank, const void* ptr, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
              CUtensorMap* out) {
  B200_REQUIRE(rank == 2 || rank == 3, "bf16_tmap: rank %d", rank);
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeTiledFn enc = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
                    qres == cudaDriverEntryPointSuccess;
    return ok ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
  }();
  static std::unordered_map<TmapKey, CUtensorMap, TmapHash> cache;
  static std::mutex mu;
  TmapKey key{};
  key[0] = (cuuint64_t)(uintptr_t)ptr;
  key[1] = (cuuint64_t)rank;
  for (int i = 0; i < rank; ++i) {
    key[2 + i] = dims[i];
    key[7 + i] = box[i];
    if (i > 0) key[4 + i] = strides[i - 1];
  }
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return B200_OK;
    }
  }
  if (!enc) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return B200_ERR_CUDA;
  }
  const cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap tm;
  CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rank=%d ptr=%p dims=(%llu,%llu,%llu) strides=(%llu,%llu) "
              "box=(%llu,%llu,%llu)", (int)r, rank, ptr, (unsigned long long)key[2], (unsigned long long)key[3],
              (unsigned long long)key[4], (unsigned long long)key[5], (unsigned long long)key[6],
              (unsigned long long)key[7], (unsigned long long)key[8], (unsigned long long)key[9]);
    return B200_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 16384) cache.clear();
    cache[key] = tm;
  }
  *out = tm;
  return B200_OK;
}

static int round16(int x) { return (x + 15) & ~15; }

// Tile / pipeline configuration for (T, row blocks, K) from a small cost model.  Its rates are H100
// SXM estimates, not measurements: gemm_wt_tuned times candidate configurations on the device by
// default and uses this model only where it cannot measure (stream capture, B200_WT_TUNE=0).
//   * one CTA per SM (384 threads at 168 registers fill the register file);
//   * a CTA costs a few us of fixed latency (launch, barrier set-up, first TMA round trip, epilogue)
//     + per k-block max(MMA time at the data-sheet 989 TFLOP/s spread over 132 SMs, shared-memory
//     fill time at ~130 GB/s per SM);
//   * token tiles are at most WT_TN_AUTO = 128 wide: wider tiles need the 16-chunk accumulator
//     instantiation, which spills;
//   * split-K buys parallelism for the GEMMs with few weight rows at the price of fp32 partial
//     traffic (written here, read by finish_rows);
//   * the weights are streamed from HBM once: nothing is faster than bytes / 3.35 TB/s.
void gemm_wt_auto(int T, int row_blocks, int K, bool allow_split, WtConfig* best, int sm_count) {
  const int kb_total = cdiv(K, WT_BK);
  const int t16 = round16(T);
  int tn_c[12];
  int n_tn = 0;
  auto add_tn = [&](int tn) {
    if (tn < 16) tn = 16;
    if (tn > WT_TN_AUTO) tn = WT_TN_AUTO;
    if (tn > t16) tn = t16;
    for (int i = 0; i < n_tn; ++i)
      if (tn_c[i] == tn) return;
    tn_c[n_tn++] = tn;
  };
  for (int k = 1; k <= 3; ++k) add_tn(round16(cdiv(T, k)));
  if (T > WT_TN_AUTO) {
    const int nt = cdiv(T, WT_TN_AUTO);
    for (int k = 0; k < 3; ++k) add_tn(round16(cdiv(T, nt + k)));
  }
  add_tn(64); add_tn(96); add_tn(112); add_tn(128);
  double best_t = 1e30;
  best->TN = tn_c[0]; best->KS = 1; best->stages = 2; best->split = 1;
  for (int it = 0; it < n_tn; ++it) {
    const int TN = tn_c[it];
    const int tt = cdiv(T, TN);
    const long base = (long)row_blocks * tt;
    for (int KS = 1; KS <= 4; KS *= 2) {
      const int stage = KS * (WT_WBLK + TN * 128);
      {
        int st = 208 * 1024 / stage;
        if (st > 8) st = 8;
        if (st < 2 || st * KS < 3 || (long)st * stage < (long)WT_EPI_TOK * WT_ROWS * 4) continue;
        int cand[6] = {1, 0, 0, 0, 0, 0};
        int n_sp = 1;
        if (allow_split) {
          for (int target : {sm_count, 2 * sm_count, 3 * sm_count}) {
            int sp = (int)(target / base);
            if (sp > kb_total / 4) sp = kb_total / 4;
            if (sp < 1) sp = 1;
            sp = cdiv(kb_total, cdiv(kb_total, sp));
            bool dup = false;
            for (int i = 0; i < n_sp; ++i) dup |= cand[i] == sp;
            if (!dup) cand[n_sp++] = sp;
          }
        }
        for (int is = 0; is < n_sp; ++is) {
          const int split = cand[is];
          if (split > 1 && (long)split * T * row_blocks * 128 * 4 > (40L << 20)) continue;  // partial-tile budget
          const long ctas = base * split;
          const int kbs = cdiv(kb_total, split);
          const double t_mma = 2.0 * WT_ROWS * TN * WT_BK / (989e6 / 132);   // us per k-block
          const double t_fill = (WT_WBLK + TN * 128) / 130e3 * (KS == 1 ? 1.15 : 1.0);
          const double t_kb = t_mma > t_fill ? t_mma : t_fill;
          const double t_fix = 5.2;                                  // first wave, prologue hidden by PDL
          const long per_sm = (ctas + sm_count - 1) / sm_count;      // CTAs an SM has to run
          double t = t_fix + kbs * t_kb + (per_sm - 1) * (9.5 + kbs * t_kb);  // serialised waves pay the full CTA latency
          if (st * KS < 4) t *= 1.08;
          const double fill_total = (double)ctas * kbs * (WT_WBLK + TN * 128);
          if (t < t_fix + fill_total / 12e6) t = t_fix + fill_total / 12e6;   // chip-wide L2 -> SM fill rate
          const double hbm = (double)row_blocks * 128 * K * 2 / 3.35e6 + 3.0;   // weights stream from HBM once
          if (t < hbm) t = hbm + 0.01 * kbs * t_kb;
          if (split > 1) t += (double)split * T * row_blocks * 128 * 4 / 3.35e6 + 0.2 * split;
          if (t < best_t) {
            best_t = t;
            best->TN = TN; best->KS = KS; best->stages = st; best->split = split;
          }
        }
      }
    }
  }
}

int gemm_wt(const void* X, long ldx, const void* W, const void* bias, const void* residual, long ldr,
            void* C, long ldc, float* partial, int T, int N, int K, int epilogue, int mode, int inter,
            const WtConfig& cfg, unsigned flags, cudaStream_t st, const WtExt* ext) {
  B200_REQUIRE(T > 0 && N > 0 && K > 0, "gemm_wt: empty problem T=%d N=%d K=%d", T, N, K);
  B200_REQUIRE((ldx % 8) == 0 && (K % 8) == 0, "gemm_wt: ldx (%ld) and K (%d) must be multiples of 8", ldx, K);
  B200_REQUIRE(((uintptr_t)X & 15) == 0 && ((uintptr_t)W & 15) == 0, "gemm_wt: X and W must be 16-byte aligned");
  B200_REQUIRE(cfg.TN >= 16 && cfg.TN <= 256 && (cfg.TN % 16) == 0, "gemm_wt: TN=%d", cfg.TN);
  B200_REQUIRE(cfg.KS >= 1 && cfg.stages >= 2 && cfg.stages <= WT_MAX_STAGES && cfg.split >= 1,
               "gemm_wt: bad config KS=%d stages=%d split=%d", cfg.KS, cfg.stages, cfg.split);
  B200_REQUIRE(mode >= B200_WT_BF16 && mode <= B200_WT_SPLIT, "gemm_wt: mode %d", mode);
  B200_REQUIRE((mode != B200_WT_F32 && mode != B200_WT_SPLIT) || ext, "gemm_wt: fp32 / split output needs WtExt");
  B200_REQUIRE(mode != B200_WT_F32 || (ext->C32 && ((uintptr_t)ext->C32 & 15) == 0), "gemm_wt: fp32 output missing / misaligned");
  B200_REQUIRE(mode != B200_WT_SPLIT || (ext->Csplit && (ext->n_pad % 8) == 0 && (ext->ld_split % 8) == 0 &&
                                         ((uintptr_t)ext->Csplit & 15) == 0),
               "gemm_wt: split output missing / misaligned");
  B200_REQUIRE(mode != B200_WT_PARTIAL || partial, "gemm_wt: partial buffer missing");
  B200_REQUIRE(mode == B200_WT_PARTIAL || cfg.split == 1, "gemm_wt: split-K needs the partial mode");
  B200_REQUIRE(mode != B200_WT_SWIGLU || (inter > 0 && (inter % 8) == 0 && N == 2 * inter),
               "gemm_wt: SwiGLU needs N == 2 * inter (inter %% 8 == 0)");
  const int kb_total = cdiv(K, WT_BK);
  WtParams p;
  memset(&p, 0, sizeof(p));
  p.bias = (const bf16*)bias; p.residual = (const bf16*)residual; p.C = (bf16*)C; p.partial = partial;
  p.ldc = ldc; p.ldr = ldr; p.T = T; p.N = N; p.K = K;
  p.TN = cfg.TN; p.KS = cfg.KS; p.n_stages = cfg.stages;
  p.kb_per_split = cdiv(kb_total, cfg.split);
  const int splits = cdiv(kb_total, p.kb_per_split);
  B200_REQUIRE(splits == cfg.split, "gemm_wt: split %d leaves empty splits (%d k-blocks)", cfg.split, kb_total);
  p.epilogue = epilogue; p.mode = mode; p.inter = inter; p.flags = flags;
  int k_w = K;  // columns of W (the split operand repeats the weight k-blocks)
  if (ext) {
    p.kb_w = ext->kb_w; p.C32 = ext->C32; p.res32 = ext->res32; p.ldc32 = ext->ldc32; p.ldr32 = ext->ldr32;
    p.Csplit = ext->Csplit; p.ld_split = ext->ld_split; p.n_pad = ext->n_pad;
    if (ext->kb_w > 0) k_w = ext->k_w;
  }
  const int stage = cfg.KS * (WT_WBLK + cfg.TN * 128);
  const size_t smem = (size_t)cfg.stages * stage + 1024;
  B200_REQUIRE(smem <= 227 * 1024 - 1024, "gemm_wt: %zu B of shared memory", smem);
  B200_REQUIRE((size_t)cfg.stages * stage >= (size_t)WT_EPI_TOK * WT_ROWS * 4, "gemm_wt: ring smaller than the epilogue staging tile");
  CUtensorMap tw, tx;
  int rc = wt_tmap(W, (long)(ext && ext->ldw > 0 ? ext->ldw : k_w), N, k_w, mode == B200_WT_SWIGLU ? 64 : WT_ROWS, &tw);
  if (rc) return rc;
  if ((rc = wt_tmap(X, ldx, T, K, cfg.TN, &tx))) return rc;
  const int row_blocks = mode == B200_WT_SWIGLU ? cdiv(inter, 64) : cdiv(N, WT_ROWS);
  const bool tower = mode == B200_WT_F32 || mode == B200_WT_SPLIT, wide = cfg.TN > 128;
  auto* kern = !tower ? (!wide ? gemm_wt_kernel<false, 8> : gemm_wt_kernel<false, 16>)
                      : (!wide ? gemm_wt_kernel<true, 8> : gemm_wt_kernel<true, 16>);
  if ((rc = kernel_opt_in((const void*)kern, 227 * 1024 - 1024, true))) return rc;
  B200_CUDA(launch(kern, dim3(row_blocks, cdiv(T, cfg.TN), splits), dim3(WT_THREADS), smem, st, PDL_LAUNCH, tw, tx,
                   p));
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Measured configuration choice ("measure, don't guess"): the first call for a problem class
// (tokens rounded up to 64, N, K, mode) times a short list of candidate configurations on the
// caller's stream with the call's own operands (CUDA events, one warm-up + two timed launches
// each) and caches the winner; later calls cost one hash lookup.  Candidates: token tile
// {64,96,112,128}, 2 k-blocks per stage with a deep ring vs 1 with a short one, and split-K to one
// or two waves.  The list is ordered and
// the first candidate within 3 % of the best wins, so the choice is stable run to run.
// B200_WT_TUNE=0 uses the cost model (gemm_wt_auto) instead.
// ---------------------------------------------------------------------------------------------
struct TuneKey {
  int tb, N, K, mode, split_ok, dev;
  bool operator==(const TuneKey& o) const {
    return tb == o.tb && N == o.N && K == o.K && mode == o.mode && split_ok == o.split_ok && dev == o.dev;
  }
};
struct TuneHash {
  size_t operator()(const TuneKey& k) const {
    size_t h = (size_t)k.tb;
    for (int v : {k.N, k.K, k.mode, k.split_ok, k.dev}) h = h * 1000003u ^ (size_t)v;
    return h;
  }
};

// B200_WT_TUNE_FILE=<path>: measured choices are appended to the file and read back at the first call of a
// later process, so a service does not re-measure at every start and a profiler run (whose serialised
// replays distort the measurement) uses exactly the production configurations.
static const char* tune_file() {
  static const char* f = getenv("B200_WT_TUNE_FILE");
  return (f && *f) ? f : nullptr;
}

static int tune_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200_WT_TUNE");
    v = (e && atoi(e) == 0) ? 0 : 1;
  }
  return v;
}

// whether a configuration's fp32 partial tiles fit the caller's partial buffer
static bool wt_fits(const WtConfig& c, int mode, int T, int N, long partial_bytes) {
  return !(mode == B200_WT_PARTIAL && (long)c.split * T * N * 4 > partial_bytes);
}

// The ordered list of configurations gemm_wt_tuned times for a problem class, the cost model's choice first; empty
// when not even one unsplit set of partial tiles fits `partial_bytes`.  Pure host code (no CUDA call).
static std::vector<WtConfig> gemm_wt_candidates(int T, int N, int K, int mode, int inter, bool allow_split,
                                                int sm_count, long partial_bytes) {
  const int row_blocks = mode == B200_WT_SWIGLU ? cdiv(inter, 64) : cdiv(N, WT_ROWS);
  const int kb_total = cdiv(K, WT_BK);
  auto fits = [&](const WtConfig& c) { return wt_fits(c, mode, T, N, partial_bytes); };
  std::vector<WtConfig> cand;
  auto add = [&](int tn, int ks, int budget, int split) {
    if (tn > round16(T)) tn = round16(T);
    if (tn > WT_TN_AUTO) tn = WT_TN_AUTO;
    const int stage = ks * (WT_WBLK + tn * 128);
    int stg = budget / stage;
    if (stg > 6) stg = 6;
    if (stg < 2 || (long)stg * stage < (long)WT_EPI_TOK * WT_ROWS * 4) return;
    split = cdiv(kb_total, cdiv(kb_total, split < 1 ? 1 : split));
    WtConfig c{tn, ks, stg, split};
    if (!fits(c)) return;
    for (const auto& o : cand)
      if (o.TN == c.TN && o.KS == c.KS && o.stages == c.stages && o.split == c.split) return;
    cand.push_back(c);
  };
  WtConfig model;
  gemm_wt_auto(T, row_blocks, K, allow_split, &model, sm_count);
  if (fits(model)) cand.push_back(model);
  int tns[8], n_tn = 0;
  if (T <= 96) {
    tns[n_tn++] = round16(T);
    if (T > 48) tns[n_tn++] = round16(cdiv(T, 2));
  } else {
    for (int tn : {128, 96, 112, 64}) tns[n_tn++] = tn;
  }
  for (int i = 0; i < n_tn; ++i) {
    const int tn = tns[i];
    const long base = (long)row_blocks * cdiv(T, tn);
    int sps[3] = {1, 1, 1};
    if (allow_split) {
      int a = (int)(sm_count / base), b = (int)(2L * sm_count / base);
      const int cap_k = kb_total / 4 > 0 ? kb_total / 4 : 1;
      sps[1] = a < 1 ? 1 : (a > cap_k ? cap_k : a);
      sps[2] = b < 1 ? 1 : (b > cap_k ? cap_k : b);
    }
    // (measured and discarded: restricting the list to <= 110 KB configurations so that the NEXT kernel's prologue
    // can always co-reside under PDL made the C2 prefill 2-5 % slower)
    for (int sp : sps) {
      add(tn, 2, 208 * 1024, sp);  // 256-byte weight-row bursts
      add(tn, 1, 110 * 1024, sp);  // one k-block per stage, shorter ring
    }
  }
  if (cand.empty()) {
    gemm_wt_auto(T, row_blocks, K, false, &model, sm_count);
    if (fits(model)) cand.push_back(model);
  }
  return cand;
}

int gemm_wt_tuned(const void* X, long ldx, const void* W, const void* bias, const void* residual, long ldr,
                  void* C, long ldc, float* partial, long partial_bytes, int T, int N, int K, int epilogue,
                  int mode, int inter, bool allow_split, int sm_count, int* split_out, cudaStream_t st,
                  const WtExt* ext, WtConfig* cfg_out) {
  static std::unordered_map<TuneKey, WtConfig, TuneHash> cache;
  static std::mutex mu;
  const int row_blocks = mode == B200_WT_SWIGLU ? cdiv(inter, 64) : cdiv(N, WT_ROWS);
  const int kb_total = cdiv(K, WT_BK);
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  const TuneKey key{(T + 63) / 64, N, K, mode, allow_split ? 1 : 0, dev};
  WtConfig cfg;
  bool have = false;
  {
    std::lock_guard<std::mutex> g(mu);
    static bool file_read = false;
    if (!file_read) {
      file_read = true;
      if (const char* path = tune_file()) {
        if (FILE* fp = fopen(path, "r")) {
          int tb, n, k, md, so, tn, ks, stg, sp;
          while (fscanf(fp, "%d %d %d %d %d %d %d %d %d", &tb, &n, &k, &md, &so, &tn, &ks, &stg, &sp) == 9)
            if (tn >= 16 && tn <= 256 && tn % 16 == 0 && ks >= 1 && stg >= 2 && stg <= WT_MAX_STAGES && sp >= 1)
              cache[TuneKey{tb, n, k, md, so, dev}] = WtConfig{tn, ks, stg, sp};
          fclose(fp);
        }
      }
    }
    auto it = cache.find(key);
    if (it != cache.end()) {
      cfg = it->second;
      have = true;
    }
  }
  auto fits = [&](const WtConfig& c) { return wt_fits(c, mode, T, N, partial_bytes); };
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  if (!have && (!tune_enabled() || cap != cudaStreamCaptureStatusNone)) {
    gemm_wt_auto(T, row_blocks, K, allow_split, &cfg, sm_count);
    while (cfg.split > 1 && !fits(cfg)) cfg.split = cdiv(kb_total, cdiv(kb_total, cfg.split - 1));
    have = true;  // not cached: a later un-captured call may still tune
  } else if (!have) {
    const std::vector<WtConfig> cand =
        gemm_wt_candidates(T, N, K, mode, inter, allow_split, sm_count, partial_bytes);
    B200_REQUIRE(!cand.empty(), "gemm_wt: the partial-tile buffer (%ld B) is too small for T=%d N=%d", partial_bytes,
                 T, N);
    // ---- time them (the tuning launches never add a residual: the output stays idempotent) ----
    // An output that is also its own residual (h += W.x in place, bf16 or fp32) must not be overwritten by the
    // measurement: whenever a residual is given, those launches write a scratch buffer from the stream-ordered
    // allocator instead of the caller's output.
    WtExt ext_copy;
    const WtExt* ext_t = nullptr;
    float* scratch32 = nullptr;
    void* C_t = C;
    if (residual && C) {
      B200_CUDA(cudaMallocAsync(&C_t, (size_t)T * (size_t)ldc * sizeof(bf16), st));
    }
    if (ext) {
      ext_copy = *ext;
      if (mode == B200_WT_F32 && ext->res32 && ext->C32) {
        B200_CUDA(cudaMallocAsync((void**)&scratch32, (size_t)T * (size_t)ext->ldc32 * sizeof(float), st));
        ext_copy.C32 = scratch32;
      }
      ext_copy.res32 = nullptr;
      ext_t = &ext_copy;
    }
    // each candidate is replayed from a small captured graph (6 launches): the measurement sees the
    // kernel back to back with its programmatic dependent launch, not the host's launch overhead
    cudaEvent_t e0, e1;
    B200_CUDA(cudaEventCreate(&e0));
    B200_CUDA(cudaEventCreate(&e1));
    std::vector<float> ms(cand.size(), 1e30f);
    int rc = B200_OK;
    constexpr int REP = 16;
    for (size_t i = 0; i < cand.size() && rc == B200_OK; ++i) {
      cudaGraph_t graph = nullptr;
      cudaGraphExec_t gx = nullptr;
      if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
        rc = B200_ERR_CUDA;
        break;
      }
      for (int r = 0; r < REP && rc == B200_OK; ++r)
        rc = gemm_wt(X, ldx, W, bias, nullptr, 0, C_t, ldc, partial, T, N, K, epilogue, mode, inter, cand[i], 0, st, ext_t);
      cudaError_t ce = cudaStreamEndCapture(st, &graph);
      if (rc != B200_OK || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        if (rc == B200_OK) rc = B200_ERR_CUDA;
        break;
      }
      ce = cudaGraphInstantiate(&gx, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) {
        rc = B200_ERR_CUDA;
        break;
      }
      cudaGraphLaunch(gx, st);  // warm-up
      cudaEventRecord(e0, st);
      cudaGraphLaunch(gx, st);
      cudaGraphLaunch(gx, st);
      cudaEventRecord(e1, st);
      if (cudaEventSynchronize(e1) != cudaSuccess) rc = B200_ERR_CUDA;
      float t = 0.f;
      cudaEventElapsedTime(&t, e0, e1);
      ms[i] = t / (2.f * REP);
      cudaGraphExecDestroy(gx);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (scratch32) cudaFreeAsync(scratch32, st);
    if (C_t != C) cudaFreeAsync(C_t, st);
    if (rc) {
      set_error("gemm_wt: configuration measurement failed (T=%d N=%d K=%d mode=%d)", T, N, K, mode);
      return rc;
    }
    float best = 1e30f;
    for (float t : ms) best = t < best ? t : best;
    size_t pick = 0;
    for (size_t i = 0; i < cand.size(); ++i)
      if (ms[i] <= best * 1.03f) {
        pick = i;
        break;
      }
    cfg = cand[pick];
    if (getenv("B200_WT_TUNE_LOG"))
      fprintf(stderr, "[gemm_wt tune] T=%d N=%d K=%d mode=%d -> TN=%d KS=%d stages=%d split=%d (%.1f us, %zu candidates)\n",
              T, N, K, mode, cfg.TN, cfg.KS, cfg.stages, cfg.split, ms[pick] * 1000.f, cand.size());
    std::lock_guard<std::mutex> g(mu);
    cache[key] = cfg;
    if (const char* path = tune_file()) {
      if (FILE* fp = fopen(path, "a")) {
        fprintf(fp, "%d %d %d %d %d %d %d %d %d\n", key.tb, key.N, key.K, key.mode, key.split_ok, cfg.TN, cfg.KS,
                cfg.stages, cfg.split);
        fclose(fp);
      }
    }
  }
  // a cached configuration was tuned for a token count in the same 64-bucket: re-check the bounds
  if (cfg.TN > round16(T)) cfg.TN = round16(T);
  while (cfg.split > 1 && !fits(cfg)) cfg.split = cdiv(kb_total, cdiv(kb_total, cfg.split - 1));
  B200_REQUIRE(fits(cfg), "gemm_wt: the partial-tile buffer (%ld B) is too small for T=%d N=%d", partial_bytes, T, N);
  if (split_out) *split_out = cfg.split;
  if (cfg_out) *cfg_out = cfg;
  return gemm_wt(X, ldx, W, bias, residual, ldr, C, ldc, partial, T, N, K, epilogue, mode, inter, cfg, 0, st, ext);
}

int finish_rows(const float* P, int S, const void* bias, const void* resid, long ldr, void* h_out,
                long ldh, int norm_kind, const void* nw, const void* nb, float eps, void* xn, long ldx,
                int T, int N, cudaStream_t st) {
  B200_REQUIRE(P && S >= 1 && T > 0 && N > 0 && (N % 4) == 0 && N <= FIN_N_MAX,
               "finish_rows: T=%d N=%d S=%d", T, N, S);
  B200_REQUIRE(norm_kind == B200_NORM_NONE || (xn && (norm_kind != B200_NORM_RMS || nw)),
               "finish_rows: norm output / weight missing");
  B200_REQUIRE((ldr % 4) == 0 && (ldh % 4) == 0 && (ldx % 4) == 0, "finish_rows: strides must be multiples of 4");
  const bool few_rows = T <= 32;
  B200_CUDA(launch(few_rows ? finish_rows_kernel<1024, 2> : finish_rows_kernel<256, 8>, dim3(T),
                   dim3(few_rows ? 1024 : 256), 0, st, PDL_LAUNCH, P, S, (const bf16*)bias, (const bf16*)resid, ldr,
                   (bf16*)h_out, ldh, norm_kind, (const bf16*)nw, (const bf16*)nb, eps, (bf16*)xn, ldx, T, N));
  return B200_OK;
}

}  // namespace b200

// ---- C ABI ------------------------------------------------------------------
using namespace b200;
extern "C" {

/* explicit-configuration entry (benchmark sweeps, tests): cfg = {TN, KS, stages, split}; a 0 in
 * cfg[0] asks for the automatic choice.  partial: fp32 [split][T][N] (mode B200_WT_PARTIAL). */
int b200_gemm_wt(const void* X, long ldx, const void* W, const void* bias, const void* residual,
                 long ldr, void* C, long ldc, float* partial, int T, int N, int K, int epilogue,
                 int mode, int inter, const int* cfg4, unsigned flags, void* stream) {
  WtConfig c;
  if (cfg4 && cfg4[0] > 0) {
    c.TN = cfg4[0]; c.KS = cfg4[1]; c.stages = cfg4[2]; c.split = cfg4[3];
  } else {
    const int rbs = mode == B200_WT_SWIGLU ? cdiv(inter, 64) : cdiv(N, 128);
    gemm_wt_auto(T, rbs, K, mode == B200_WT_PARTIAL, &c, 132);
  }
  return gemm_wt(X, ldx, W, bias, residual, ldr, C, ldc, partial, T, N, K, epilogue, mode, inter, c,
                 flags, (cudaStream_t)stream);
}

int b200_finish_rows(const float* P, int S, const void* bias, const void* resid, long ldr, void* h_out,
                     long ldh, int norm_kind, const void* nw, const void* nb, float eps, void* xn,
                     long ldx, int T, int N, void* stream) {
  return finish_rows(P, S, bias, resid, ldr, h_out, ldh, norm_kind, nw, nb, eps, xn, ldx, T, N,
                     (cudaStream_t)stream);
}

int b200_gemm_wt_auto_config(int T, int N, int K, int mode, int inter, int* cfg4_out) {
  WtConfig c;
  const int rbs = mode == B200_WT_SWIGLU ? cdiv(inter, 64) : cdiv(N, 128);
  gemm_wt_auto(T, rbs, K, mode == B200_WT_PARTIAL, &c, 132);
  cfg4_out[0] = c.TN; cfg4_out[1] = c.KS; cfg4_out[2] = c.stages; cfg4_out[3] = c.split;
  return B200_OK;
}

int b200_gemm_wt_candidates(int T, int N, int K, int mode, int inter, int allow_split, int sm_count,
                            long partial_bytes, int* cfg_out, int max_n, int* n_out) {
  B200_REQUIRE(T > 0 && N > 0 && K > 0 && sm_count > 0 && n_out && (max_n <= 0 || cfg_out),
               "gemm_wt_candidates: T=%d N=%d K=%d sm_count=%d", T, N, K, sm_count);
  const std::vector<WtConfig> cand =
      gemm_wt_candidates(T, N, K, mode, inter, allow_split != 0, sm_count, partial_bytes);
  *n_out = (int)cand.size();
  for (int i = 0; i < (int)cand.size() && i < max_n; ++i) {
    cfg_out[4 * i] = cand[i].TN; cfg_out[4 * i + 1] = cand[i].KS;
    cfg_out[4 * i + 2] = cand[i].stages; cfg_out[4 * i + 3] = cand[i].split;
  }
  return B200_OK;
}

int b200_gemm_wt_tuned(const void* X, long ldx, const void* W, const void* bias, const void* residual, long ldr,
                       void* C, long ldc, float* partial, long partial_bytes, int T, int N, int K, int epilogue,
                       int mode, int inter, int allow_split, int sm_count, int* cfg4_out, void* stream) {
  WtConfig c{0, 0, 0, 0};
  const int rc = gemm_wt_tuned(X, ldx, W, bias, residual, ldr, C, ldc, partial, partial_bytes, T, N, K, epilogue,
                               mode, inter, allow_split != 0, sm_count, nullptr, (cudaStream_t)stream, nullptr, &c);
  if (cfg4_out) {
    cfg4_out[0] = c.TN; cfg4_out[1] = c.KS; cfg4_out[2] = c.stages; cfg4_out[3] = c.split;
  }
  return rc;
}
}
