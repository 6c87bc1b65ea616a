// k_mega_tc: the decode step as one persistent kernel whose GEMV phases run on the tensor
// cores (wgmma.mma_async, fp32 accumulators in the registers of warpgroup 0).
//
// Why: in k_mega (decode_mega.cu) the 8 consumer warps spend CUDA-core instructions on every
// weight element; here a weight tile is consumed by a few wgmma instructions, so the stream is
// bounded by HBM and by the phase boundaries only.
//
//   * weights are re-packed once at load into TILE IMAGES: row block (128 rows) x K block
//     (64 columns) = 16 KB in the 128-byte-swizzled K-major layout wgmma reads, K blocks of
//     a row block contiguous -> the producer's plain 1-D cp.async.bulk lands a ready A operand;
//   * the activation vector is the B operand: 8 rows x K, row 0 = x (m64n8k16, two per 128 rows);
//   * warps 0..3 issue the MMAs of a unit, exchange column 0 through shared memory and run the
//     per-row epilogue (thread = row);
//   * phases with few rows (qkv, o_proj, down) are split along K over the SMs; their fp32
//     partial sums are reduced, in a fixed order, by the prologue of the NEXT phase, which
//     also carries the residual stream in shared memory (no global round trip for h).
// Rounding points: oracle/qwen2vl.py::lm_layers_forward (fp32 accumulation, one bf16 rounding
// per Linear, RMSNorm 2 roundings, residual add 1).
#include "mega_common.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int TC_SUB = 16 * 1024;   // one tile image: 128 rows x 64 bf16, 128B swizzle

struct TcShared {
  MegaShared m;
  float vrow[128];      // column 0 of a unit's accumulator: one value per row of the row block
  float xch[64];        // gate/up exchange between the lane halves of a row block
  float redf[8];
  float2 lse_w[4];
};

__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void ebar() { asm volatile("bar.sync 2, 128;" ::: "memory"); }

// unit u of a phase -> (row block, K split) and its K-block range
struct TcUnit {
  int rb, ks, kb0, kb1;
};
__device__ __forceinline__ TcUnit tc_unit(const MegaTcPhase& g, int u) {
  TcUnit t;
  t.rb = u / g.S;
  t.ks = u - t.rb * g.S;
  t.kb0 = (int)((long)g.KB * t.ks / g.S);
  t.kb1 = (int)((long)g.KB * (t.ks + 1) / g.S);
  return t;
}

// ---- producer ----------------------------------------------------------------------
// In-flight throttle: the bandwidth-delay product of one SM's HBM share (~44 GB/s x ~1 us) is
// about ONE 48 KB tile; more requests in flight add no throughput but queue ahead of the
// consumers' small latency-critical loads (measured: with 4 tiles in flight a 1.5 KB L2-hit
// load at a phase start took 3.6 us).  So tile i is requested only after tile i - max_inflight
// has landed; the ring still fills up completely while the consumers are stalled.
struct Producer {
  Ring rg, lag;
  int issued;
};
__device__ __forceinline__ void tc_produce(const MegaTcP& P, const MegaTcPhase& g,
                                           const uint8_t* Wt, uint8_t* ring, TcShared* sh,
                                           Producer& pr, uint64_t pol) {
  Ring& rg = pr.rg;
  for (int u = blockIdx.x; u < g.units; u += gridDim.x) {
    const TcUnit t = tc_unit(g, u);
    for (int kb = t.kb0; kb < t.kb1; kb += P.sps) {
      const int n = min(P.sps, t.kb1 - kb);
      const int s = rg.slot();
      if (pr.issued >= P.max_inflight) {
        mb_wait(&sh->m.full_bar[pr.lag.slot()], pr.lag.parity(), &sh->m.err);
        pr.lag.advance();
      }
      ++pr.issued;
      mb_wait(&sh->m.empty_bar[s], rg.parity() ^ 1u, &sh->m.err);
      const uint32_t bytes = (uint32_t)n * TC_SUB;
      mb_expect_tx(&sh->m.full_bar[s], bytes);
      bulk_g2s(ring + (long)s * P.base.stage_bytes, Wt + ((long)t.rb * g.KB + kb) * TC_SUB, bytes,
               &sh->m.full_bar[s], pol);
      rg.advance();
    }
  }
}

// L2 prefetch of this CTA's tiles of a phase (fire and forget): issued at the start of a layer
// for the MLP weights, so that the ring refills from L2 while the qkv / attention / o_proj
// chain (latency-bound, ~12 % of the layer's bytes) would otherwise leave HBM idle
__device__ __forceinline__ void tc_l2_prefetch(const MegaTcP& P, const MegaTcPhase& g,
                                               const uint8_t* Wt) {
  for (int u = blockIdx.x; u < g.units; u += gridDim.x) {
    const TcUnit t = tc_unit(g, u);
    for (int kb = t.kb0; kb < t.kb1; kb += P.sps) {
      const int n = min(P.sps, t.kb1 - kb);
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(Wt + ((long)t.rb * g.KB + kb) * TC_SUB),
                   "r"((uint32_t)n * TC_SUB)
                   : "memory");
    }
  }
}

// ---- prologue helpers (256 consumer threads) -------------------------------------------
// chunk c (8 elements) of the operand row 0; local K block = c / 8
__device__ __forceinline__ uint4* xop_chunk(uint8_t* xop, int kstride, int c) {
  return reinterpret_cast<uint4*>(xop + (long)(c >> 3) * kstride + (c & 7) * 16);
}
__device__ __forceinline__ void xop_zero_rows(uint8_t* xop, int kstride, int nkb) {
  const int per = (kstride - 128) / 16;  // uint4 slots of rows 1.. of one K block
  for (int i = threadIdx.x; i < nkb * per; i += 256) {
    const int kb = i / per, o = i - kb * per;
    *reinterpret_cast<uint4*>(xop + (long)kb * kstride + 128 + o * 16) = make_uint4(0, 0, 0, 0);
  }
}
// sum of the ATT_UN partial attention outputs of 4 consecutive channels: all loads in flight at
// once (one L2 round trip), added in unit order (deterministic)
__device__ __forceinline__ float4 sum_parts4(const float* base, long stride, int S) {
  float4 v[ATT_UN];
#pragma unroll
  for (int ks = 0; ks < ATT_UN; ++ks)
    v[ks] = (ks < S) ? __ldcg(reinterpret_cast<const float4*>(base + (long)ks * stride))
                     : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 a = v[0];
#pragma unroll
  for (int ks = 1; ks < ATT_UN; ++ks) {
    a.x += v[ks].x; a.y += v[ks].y; a.z += v[ks].z; a.w += v[ks].w;
  }
  return a;
}

// residual update + RMSNorm -> operand.  h_new = first ? h_global : bf16(hres + bf16(sum parts))
__device__ __forceinline__ void zero_acc(long long* acc, int n) {
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) acc[i] = 0ll;
}

__device__ __forceinline__ void pro_norm(const MegaTcP& P, uint8_t* xop, uint16_t* hres,
                                         TcShared* sh, const long long* acc, bool first,
                                         const bf16* lnw, long long* tdbg = nullptr) {
  int tn = 0;
#define PRO_STAMP() do { if (tdbg && threadIdx.x == 128) tdbg[tn++] = gtimer(); } while (0)
  PRO_STAMP();
  const DecodeDims& d = P.base.d;
  const int nvec = d.hidden >> 3;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // RMSNorm weights are requested together with the partial sums (one round trip, not two)
  constexpr int NW = 4;
  uint4 lw8[NW];
#pragma unroll
  for (int u = 0; u < NW; ++u) {
    const int c = threadIdx.x + 256 * u;
    lw8[u] = (c < nvec) ? __ldg(reinterpret_cast<const uint4*>(lnw + (long)c * 8)) : make_uint4(0, 0, 0, 0);
  }
  xop_zero_rows(xop, P.x_kstride, (d.hidden + 63) >> 6);
  float ss = 0.f;
  for (int c = threadIdx.x; c < 2 * nvec; c += 256) {  // 4 elements per thread and trip
    float f[4];
    if (first) {
      unpack4(__ldcg(reinterpret_cast<const uint2*>(P.base.h + (long)c * 4)), f);
    } else {
      const longlong2 q0 = __ldcg(reinterpret_cast<const longlong2*>(acc + (long)c * 4));
      const longlong2 q1 = __ldcg(reinterpret_cast<const longlong2*>(acc + (long)c * 4 + 2));
      float hv[4];
      unpack4(*reinterpret_cast<const uint2*>(hres + c * 4), hv);
      f[0] = rbf(hv[0] + rbf(__ll2float_rn(q0.x) * TC_FIX_INV));
      f[1] = rbf(hv[1] + rbf(__ll2float_rn(q0.y) * TC_FIX_INV));
      f[2] = rbf(hv[2] + rbf(__ll2float_rn(q1.x) * TC_FIX_INV));
      f[3] = rbf(hv[3] + rbf(__ll2float_rn(q1.y) * TC_FIX_INV));
    }
    *reinterpret_cast<uint2*>(hres + c * 4) = make_uint2(pack2(f[0], f[1]), pack2(f[2], f[3]));
#pragma unroll
    for (int j = 0; j < 4; ++j) ss = fmaf(f[j], f[j], ss);
  }
  PRO_STAMP();  // partial sums loaded, residual updated
  ss = warp_sum(ss);
  if (lane == 0) sh->redf[warp] = ss;
  cbar();
  PRO_STAMP();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += sh->redf[w];
  const float rs = 1.0f / sqrtf(tot / (float)d.hidden + d.eps);
#pragma unroll
  for (int u = 0; u < NW; ++u) {
    const int c = threadIdx.x + 256 * u;
    if (c >= nvec) break;
    float f[8], lf[8];
    unpack8(*reinterpret_cast<const uint4*>(hres + c * 8), f);
    unpack8(lw8[u], lf);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = rbf(rbf(f[j] * rs) * lf[j]);
    uint4 o;
    o.x = pack2(f[0], f[1]); o.y = pack2(f[2], f[3]); o.z = pack2(f[4], f[5]); o.w = pack2(f[6], f[7]);
    *xop_chunk(xop, P.x_kstride, c) = o;
  }
  // K padding (hidden not a multiple of 64): the tail chunks of the last block are zero
  for (int c = nvec + threadIdx.x; c < ((d.hidden + 63) >> 6) * 8; c += 256)
    *xop_chunk(xop, P.x_kstride, c) = make_uint4(0, 0, 0, 0);
  PRO_STAMP();  // normalised operand written
  fence_async_smem();
  PRO_STAMP();
  cbar();
  PRO_STAMP();
}

// K slice of the attention output: x = bf16(sum over the ATT_UN key ranges of the partials)
__device__ __forceinline__ void pro_attn_slice(const MegaTcP& P, uint8_t* xop, const MegaTcPhase& g) {
  const MegaP& p = P.base;
  const DecodeDims& d = p.d;
  if ((int)blockIdx.x < g.units) {
    const TcUnit t = tc_unit(g, blockIdx.x);
    xop_zero_rows(xop, P.x_kstride, t.kb1 - t.kb0);
    const int c0 = t.kb0 * 8, c1 = min(t.kb1 * 8, g.K >> 3);
    for (int c = c0 + threadIdx.x; c < c1; c += 256) {
      const int d0 = c * 8, h = d0 / d.hd, Gall = d.n_heads / d.n_kv, G = (Gall + p.hsplit - 1) / p.hsplit;
      const int grp = (h / Gall) * p.hsplit + (h % Gall) / G, gi = (h % Gall) % G;
      const float* src = p.att_part + (long)grp * ATT_UN * MEGA_ATT_G * d.hd + (long)gi * d.hd + (d0 % d.hd);
      const float4 sa = sum_parts4(src, (long)MEGA_ATT_G * d.hd, ATT_UN);
      const float4 sb = sum_parts4(src + 4, (long)MEGA_ATT_G * d.hd, ATT_UN);
      uint4 o;
      o.x = pack2(sa.x, sa.y); o.y = pack2(sa.z, sa.w); o.z = pack2(sb.x, sb.y); o.w = pack2(sb.z, sb.w);
      *xop_chunk(xop, P.x_kstride, c - c0) = o;
    }
    // K padding (K not a multiple of 64): the tail chunks of the last block stay zero
    for (int c = max(c1, c0) + threadIdx.x; c < t.kb1 * 8; c += 256)
      *xop_chunk(xop, P.x_kstride, c - c0) = make_uint4(0, 0, 0, 0);
  }
  fence_async_smem();
  cbar();
}

// K slice of a bf16 activation vector in global memory (down projection input)
__device__ __forceinline__ void pro_slice(const MegaTcP& P, uint8_t* xop, const MegaTcPhase& g,
                                          const bf16* x, long long* tdbg = nullptr) {
  int tn = 0;
  PRO_STAMP();
  if ((int)blockIdx.x < g.units) {
    const TcUnit t = tc_unit(g, blockIdx.x);
    xop_zero_rows(xop, P.x_kstride, t.kb1 - t.kb0);
    const int c0 = t.kb0 * 8, c1 = min(t.kb1 * 8, g.K >> 3);
    for (int c = c0 + threadIdx.x; c < t.kb1 * 8; c += 256)
      *xop_chunk(xop, P.x_kstride, c - c0) = (c < c1) ? ldcg16(x + (long)c * 8) : make_uint4(0, 0, 0, 0);
  }
  PRO_STAMP();
  fence_async_smem();
  PRO_STAMP();
  cbar();
  PRO_STAMP();
}

// ---- consumers (warpgroup 0 = warps 0..3): the MMAs of a unit, then its per-row epilogue ----------
// D[128 rows x 8] = W tile . X^T as two m64n8k16 halves per 16-wide K step; only column 0 (operand
// row 0 = the activation vector) is used.  Thread r of the warpgroup then owns row r of the block.
template <int MODE>
__device__ __forceinline__ void tc_consume(const MegaTcP& P, const MegaTcPhase& g, uint8_t* ring,
                                           const uint8_t* xop, TcShared* sh, Ring& rg, bool xfull,
                                           long long* acc_out, bf16* out, long long* tdbg) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = warp * 32 + lane;
  int tn = 0;
  if (tdbg && r == 0) tdbg[tn++] = gtimer();
  const uint32_t xop_a = wg_smem(xop), ring_a = wg_smem(ring);
  float run_m = -INFINITY, run_l = 0.f;
  for (int u = blockIdx.x; u < g.units; u += gridDim.x) {
    const TcUnit t = tc_unit(g, u);
    float acc[2][4];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[hf][i] = 0.f;
    for (int kb = t.kb0; kb < t.kb1; kb += P.sps) {
      const int n = min(P.sps, t.kb1 - kb);
      const int s = rg.slot();
      mb_wait(&sh->m.full_bar[s], rg.parity(), &sh->m.err);
      if (tdbg && r == 0 && tn < 27) tdbg[tn++] = gtimer();
      const uint32_t a0 = ring_a + (uint32_t)s * (uint32_t)P.base.stage_bytes;
      // the operand holds either the whole vector (norm phases) or this unit's K slice
      const uint32_t b0 = xop_a + (uint32_t)(kb - (xfull ? 0 : t.kb0)) * (uint32_t)P.x_kstride;
      wg_fence_acc(acc[0]);
      wg_fence_acc(acc[1]);
      wg_arrive();
#pragma unroll
      for (int sb = 0; sb < 3; ++sb) {
        if (sb < n) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint64_t db = wg_desc(b0 + sb * P.x_kstride + kk * 32);
            wgmma_n8_ss(acc[0], wg_desc(a0 + sb * TC_SUB + kk * 32), db, 1u);
            wgmma_n8_ss(acc[1], wg_desc(a0 + sb * TC_SUB + 64 * 128 + kk * 32), db, 1u);
          }
        }
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc[0]);
      wg_fence_acc(acc[1]);
      __syncwarp();
      if (lane == 0) mb_arrive(&sh->m.empty_bar[s]);  // this warp's MMAs have read the ring slot
      if (tdbg && r == 0 && tn < 27) tdbg[tn++] = gtimer();
      rg.advance();
    }
    if ((lane & 3) == 0) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        sh->vrow[hf * 64 + warp * 16 + (lane >> 2)] = acc[hf][0];
        sh->vrow[hf * 64 + warp * 16 + (lane >> 2) + 8] = acc[hf][2];
      }
    }
    ebar();
    const float v = sh->vrow[r];
    ebar();
    if (MODE == PH_GATEUP) {
      // rows 0..63 = gate, 64..127 = up of the same 64 intermediate channels
      if (r >= 64) sh->xch[r - 64] = v;
      ebar();
      if (r < 64) {
        const int ch = t.rb * 64 + r;
        if (ch < g.N) out[ch] = f2bf(swiglu_bf(rbf(v), rbf(sh->xch[r])));
      }
      ebar();
    } else if (MODE == PH_HEAD) {
      const int row = t.rb * 128 + r;
      float a = -INFINITY;
      if (row < g.N) {
        a = rbf(v);
        out[row] = f2bf(a);
        const float mn = fmaxf(run_m, a);
        run_l = run_l * expf(run_m - mn) + expf(a - mn);
        run_m = mn;
      }
    } else {
      const int row = t.rb * 128 + r;
      if (row < g.N) fix_add(acc_out + row, v);
    }
  }
  if (MODE == PH_HEAD) {
    const float m = warp_max(run_m);
    float l = (run_l > 0.f) ? run_l * expf(run_m - m) : 0.f;
    l = warp_sum(l);
    if (lane == 0) sh->lse_w[warp] = make_float2(m, l);
    ebar();
    if (threadIdx.x == 0) {
      float M = -INFINITY;
      for (int i = 0; i < 4; ++i) M = fmaxf(M, sh->lse_w[i].x);
      float L = 0.f;
      for (int i = 0; i < 4; ++i)
        if (sh->lse_w[i].y > 0.f) L += sh->lse_w[i].y * expf(sh->lse_w[i].x - M);
      P.base.partials[blockIdx.x] = make_float2(M, L);
    }
  }
}

template <int MODE>
__device__ __forceinline__ void tc_run(const MegaTcP& P, const MegaTcPhase& g, uint8_t* ring,
                                       const uint8_t* xop, TcShared* sh, Ring& rg, long long* acc_out, bf16* out,
                                       long long* tdbg = nullptr) {
  if ((threadIdx.x >> 5) < 4) {
    tc_consume<MODE>(P, g, ring, xop, sh, rg, MODE == PH_QKV || MODE == PH_GATEUP || MODE == PH_HEAD, acc_out, out,
                     tdbg);
    if (tdbg && threadIdx.x == 0) tdbg[28] = gtimer();
  }
}

}  // namespace

__global__ void __launch_bounds__(MEGA_THREADS, 1) k_mega_tc(const __grid_constant__ MegaTcP P) {
  extern __shared__ uint8_t sm_raw[];
  __shared__ TcShared sh;
  const MegaP& p = P.base;
  const DecodeDims& d = p.d;
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sm_raw) + 1023) &
                                           ~static_cast<uintptr_t>(1023));
  uint8_t* ring = sm;
  uint8_t* xop = sm + (long)p.n_stages * p.stage_bytes;          // B operand / attention scratch
  uint16_t* hres = reinterpret_cast<uint16_t*>(xop + P.region_bytes);  // residual stream (bf16)
  float* scratch = reinterpret_cast<float*>(xop);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (p.st->error) return;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mb_init(&sh.m.full_bar[s], 1);
      mb_init(&sh.m.empty_bar[s], 4);  // one arrival per consumer warp
    }
    sh.m.err = 0;
    for (int i = 0; i < d.hd / 2; ++i) sh.m.invf[i] = p.inv_freq[i];
    sh.m.bar_base = p.st->bar_base;
    sh.m.att_base = p.st->att_base;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  Ring rg;
  rg.cur = 0;
  rg.ph = 0;
  rg.n_stages = p.n_stages;

  if (warp == 8) {
    // ===== producer: the whole step's weight stream =====
    if (lane == 0) {
      const uint64_t pol = policy_evict_first();
      Producer pr;
      pr.rg = rg;
      pr.lag = rg;
      pr.issued = 0;
      for (int l = 0; l < p.n_layers; ++l) {
        const LayerWT& lt = P.lt[l];
        if (p.l2_prefetch >= 1) tc_l2_prefetch(P, P.ph[PH_GATEUP], lt.wgu);
        if (p.l2_prefetch >= 2) tc_l2_prefetch(P, P.ph[PH_DRES], lt.wd);
        tc_produce(P, P.ph[PH_QKV], lt.wqkv, ring, &sh, pr, pol);
        tc_produce(P, P.ph[PH_ORES], lt.wo, ring, &sh, pr, pol);
        tc_produce(P, P.ph[PH_GATEUP], lt.wgu, ring, &sh, pr, pol);
        tc_produce(P, P.ph[PH_DRES], lt.wd, ring, &sh, pr, pol);
      }
      tc_produce(P, P.ph[PH_HEAD], P.head_t, ring, &sh, pr, pol);
    }
    return;
  }

  // ===== consumers =====
  unsigned bidx = 0;
  const int ctx = p.st->ctx, pos = p.st->pos;
  for (int l = 0; l < p.n_layers; ++l) {
    const LayerW& lw = p.layers[l];
    bf16* kc = p.kv + (long)l * p.kv_layer_stride;
    bf16* vc = kc + p.kv_v_offset;
    // ---- qkv: h (+ previous layer's down partials) -> norm -> split-K partials ----
    pro_norm(P, xop, hres, &sh, P.d_acc, l == 0, lw.ln1);
    tc_run<PH_QKV>(P, P.ph[PH_QKV], ring, xop, &sh, rg, P.qkv_acc, nullptr);
    grid_barrier(p, &sh.m, bidx);
    // ---- attention (finishes q/k/v from the partials) ----
    if ((int)blockIdx.x < p.attn_ctas) {
      const AttnParts ap = {P.qkv_acc, lw.bqkv, pos, nullptr, 0u};
      if (d.hd == 128) attn_phase<128, ATT_PARTS>(p, kc, vc, scratch, &sh.m, ctx + 1, l, ap);
      else attn_phase<64, ATT_PARTS>(p, kc, vc, scratch, &sh.m, ctx + 1, l, ap);
    }
    grid_barrier(p, &sh.m, bidx);
    // ---- o_proj: split-K partials ----
    zero_acc(P.d_acc, d.hidden);  // last read by this layer's qkv prologue, next written by down
    pro_attn_slice(P, xop, P.ph[PH_ORES]);
    tc_run<PH_ORES>(P, P.ph[PH_ORES], ring, xop, &sh, rg, P.o_acc, nullptr);
    grid_barrier(p, &sh.m, bidx);
    // ---- gate/up: h += o ; norm ; SwiGLU ----
    long long* td = (p.dbg && l == 5 && blockIdx.x == 0) ? p.dbg + 4096 : nullptr;
    if (td && threadIdx.x == 128) td[0] = gtimer();
    zero_acc(P.qkv_acc, P.ph[PH_QKV].N);  // read by this layer's attention, next written by qkv
    pro_norm(P, xop, hres, &sh, P.o_acc, false, lw.ln2, td ? p.dbg + 4096 + 160 : nullptr);
    tc_run<PH_GATEUP>(P, P.ph[PH_GATEUP], ring, xop, &sh, rg, nullptr, p.act,
                      td ? td + 1 : nullptr);
    grid_barrier(p, &sh.m, bidx);
    // ---- down: split-K partials ----
    td = (p.dbg && l == 5 && blockIdx.x == 0) ? p.dbg + 4096 + 64 : nullptr;
    if (td && threadIdx.x == 128) td[0] = gtimer();
    zero_acc(P.o_acc, d.hidden);  // read by this layer's gate/up prologue, next written by o_proj
    pro_slice(P, xop, P.ph[PH_DRES], p.act, td ? p.dbg + 4096 + 176 : nullptr);
    tc_run<PH_DRES>(P, P.ph[PH_DRES], ring, xop, &sh, rg, P.d_acc, nullptr,
                    td ? td + 1 : nullptr);
    grid_barrier(p, &sh.m, bidx);
  }
  pro_norm(P, xop, hres, &sh, P.d_acc, p.n_layers == 0, p.final_norm);
  tc_run<PH_HEAD>(P, P.ph[PH_HEAD], ring, xop, &sh, rg, nullptr, p.logits);
  grid_barrier(p, &sh.m, bidx);
  mega_sample_finalize(p, sh.m, bidx);
}

// ---------------------------------------------------------------------------
// weight packing: [N, K] row-major bf16 -> tile images
// ---------------------------------------------------------------------------
// dst 16-byte chunk index i = ((rb * KB + kb) * 128 + r) * 8 + pc, pc = physical chunk in the
// 128-byte row; logical chunk = pc ^ (r & 7) (the 128B swizzle TMA would have applied).
// interleave != 0 (gate/up): row block rb = 64 rows of src followed by 64 rows of src2.
__global__ void k_pack_tiles(const bf16* __restrict__ src, const bf16* __restrict__ src2, int N,
                             int K, int RB, int KB, int interleave, uint4* __restrict__ dst) {
  const long total = (long)RB * KB * 128 * 8;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    const int pc = (int)(i & 7);
    const int r = (int)((i >> 3) & 127);
    const long blk = i >> 10;
    const int kb = (int)(blk % KB), rb = (int)(blk / KB);
    const int lc = pc ^ (r & 7);
    const int col = kb * 64 + lc * 8;
    const bf16* row_ptr = nullptr;
    if (interleave) {
      const int ch = rb * 64 + (r & 63);
      if (ch < N) row_ptr = (r < 64 ? src : src2) + (long)ch * K;
    } else {
      const int row = rb * 128 + r;
      if (row < N) row_ptr = src + (long)row * K;
    }
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row_ptr) {
      if (col + 8 <= K) {
        v = *reinterpret_cast<const uint4*>(row_ptr + col);
      } else if (col < K) {
        unsigned short tmp[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int j = 0; j < K - col; ++j) tmp[j] = reinterpret_cast<const unsigned short*>(row_ptr)[col + j];
        v = *reinterpret_cast<const uint4*>(tmp);
      }
    }
    dst[i] = v;
  }
}

size_t mega_tc_packed_bytes(int N, int K, bool interleave) {
  const long RB = interleave ? cdiv(N, 64) : cdiv(N, 128);
  return (size_t)RB * cdiv(K, 64) * TC_SUB;
}

int mega_tc_pack(const bf16* src, const bf16* src2, int N, int K, bool interleave, void* dst,
                 cudaStream_t s) {
  B200_REQUIRE((K % 8) == 0, "pack: K %d %% 8 != 0", K);
  const int RB = interleave ? cdiv(N, 64) : cdiv(N, 128), KB = cdiv(K, 64);
  k_pack_tiles<<<1184, 256, 0, s>>>(src, src2, N, K, RB, KB, interleave ? 1 : 0,
                                   reinterpret_cast<uint4*>(dst));
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------
// host: geometry + launch
// ---------------------------------------------------------------------------
static void tc_geometry(MegaTcPhase& g, int K, int N, int rows_per_block, int grid, int sps,
                        bool allow_split) {
  g.K = K;
  g.N = N;
  g.KB = cdiv(K, 64);
  g.RB = cdiv(N, rows_per_block);
  int S = 1;
  if (allow_split && g.RB < grid) {
    S = grid / g.RB;
    const int by_tile = cdiv(g.KB, sps);  // no point in splitting below one ring stage
    if (S > by_tile) S = by_tile;
    if (S < 1) S = 1;
  }
  g.S = S;
  g.units = g.RB * S;
}

int mega_tc_fill(MegaTcP& P, int sm_count) {
  MegaP& p = P.base;
  const DecodeDims& d = p.d;
  const int grid = sm_count;
  P.sps = 3;  // K blocks per ring stage (tc_mma unrolls 3)
  p.stage_bytes = P.sps * TC_SUB;
  const int qkv_rows = (d.n_heads + 2 * d.n_kv) * d.hd;
  tc_geometry(P.ph[PH_QKV], d.hidden, qkv_rows, 128, grid, P.sps, true);
  tc_geometry(P.ph[PH_ORES], d.n_heads * d.hd, d.hidden, 128, grid, P.sps, true);
  tc_geometry(P.ph[PH_GATEUP], d.hidden, d.inter, 64, grid, P.sps, false);
  tc_geometry(P.ph[PH_DRES], d.inter, d.hidden, 128, grid, P.sps, true);
  tc_geometry(P.ph[PH_HEAD], d.hidden, d.vocab, 128, grid, P.sps, false);
  for (int i : {PH_QKV, PH_ORES, PH_DRES})
    B200_REQUIRE(P.ph[i].units <= grid, "mega_tc: split phase %d has %d units > %d CTAs", i,
                 P.ph[i].units, grid);
  B200_REQUIRE((d.hidden % 8) == 0 && (d.inter % 8) == 0 && ((d.n_heads * d.hd) % 8) == 0,
               "mega_tc: dims must be multiples of 8");
  // attention geometry (same rules as k_mega)
  const int G = d.n_heads / d.n_kv;
  int hs = (G + MEGA_ATT_G - 1) / MEGA_ATT_G;  // <= MEGA_ATT_G q heads per CTA, uneven split allowed
  if (hs == 1 && G % 2 == 0 && G >= 4) hs = 2;
  p.hsplit = hs;
  p.attn_ctas = d.n_kv * hs * ATT_UN;
  B200_REQUIRE(p.attn_ctas <= grid, "mega_tc: %d attention CTAs > %d SMs", p.attn_ctas, grid);
  B200_REQUIRE(d.hd == 64 || d.hd == 128, "mega_tc: head_dim %d (64|128)", d.hd);
  B200_REQUIRE(d.hidden <= 8192, "mega_tc: hidden %d > 8192", d.hidden);
  // operand region: the largest K range any CTA multiplies in one phase
  int max_kb = 0;
  for (int i = 0; i < 5; ++i) {
    const MegaTcPhase& g = P.ph[i];
    const int kb = cdiv(g.KB, g.S) + (g.S > 1 ? 1 : 0);
    if (kb > max_kb) max_kb = kb;
  }
  const size_t xop_bytes = (size_t)max_kb * P.x_kstride;
  const size_t att = ((size_t)MEGA_ATT_G * cdiv(d.cap, ATT_UN) + (size_t)8 * MEGA_ATT_G * d.hd +
                      (size_t)(MEGA_ATT_G + 2) * d.hd) * 4;
  size_t region = xop_bytes > att ? xop_bytes : att;
  region = (region + 1023) & ~(size_t)1023;
  P.region_bytes = (int)region;
  const size_t hres_bytes = ((size_t)d.hidden * 2 + 127) & ~(size_t)127;
  const long budget = 227 * 1024 - 2048 - 1024 /*alignment slack*/ - (long)region - (long)hres_bytes;
  int ns = (int)(budget / p.stage_bytes);
  B200_REQUIRE(ns >= 2, "mega_tc: no room for the weight ring (region %zu B)", region);
  p.n_stages = ns > 8 ? 8 : ns;
  P.smem_bytes = (size_t)p.n_stages * p.stage_bytes + region + hres_bytes + 1024;
  return B200_OK;
}

int mega_tc_launch(const MegaTcP& P, int sm_count, cudaStream_t s) {
  static unsigned long long set_mask = 0ull;  // per device
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (!(set_mask >> (dev & 63) & 1ull)) {
    B200_CUDA(cudaFuncSetAttribute(k_mega_tc, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   227 * 1024 - 2048));
    B200_CUDA(cudaFuncSetAttribute(k_mega_tc, cudaFuncAttributePreferredSharedMemoryCarveout,
                                   cudaSharedmemCarveoutMaxShared));
    set_mask |= 1ull << (dev & 63);
  }
  // cooperative launch: see decode_mega.cu::mega_launch_f
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(sm_count);
  cfg.blockDim = dim3(MEGA_THREADS);
  cfg.dynamicSmemBytes = P.smem_bytes;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  B200_CUDA(cudaLaunchKernelEx(&cfg, k_mega_tc, P));
  return B200_OK;
}

}  // namespace b200
