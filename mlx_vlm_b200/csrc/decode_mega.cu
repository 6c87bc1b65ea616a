// k_mega: the WHOLE decode step (28 x {qkv, attention, o_proj, gate/up, down} + head
// + sampler) as ONE persistent kernel, one CTA per SM.
//
// Why: the step is a chain of ~140 small dependent phases.  As separate kernels
// each boundary costs several microseconds during which HBM idles (measured: the
// 4.7 MB o_proj kernel takes 5.9 us, 0.7 us of it streaming).  Here
//   * warp 8 of every CTA is a PRODUCER that walks the static tile schedule of the
//     whole step and streams weight tiles (cp.async.bulk -> shared-memory ring,
//     mbarrier complete_tx) without ever waiting for a phase boundary: the ring
//     (up to 4 x 48 KB per SM, ~28 MB chip-wide) runs ahead across phases and layers;
//   * warps 0..7 are CONSUMERS that execute the phases in order, separated by a
//     software grid barrier (one atomic + acquire spin, ~1 us) instead of a kernel
//     boundary; activations cross CTAs through L2 (ld.global.cg).
// Rounding points follow oracle/qwen2vl.py::lm_layers_forward (same device
// functions as the multi-kernel path in decode.cu).
#include "mega_common.cuh"

namespace b200 {

namespace {

template <int MODE>
__device__ __forceinline__ const bf16* mega_tile_src(const MegaPhase& g, const bf16* W,
                                                     const bf16* W2, int hd, int t, int m) {
  if (MODE == PH_QKV) {
    const int half = hd >> 1;
    const int per_slot = half / g.R;
    const int slot = t / per_slot, jb = t % per_slot;
    return W + ((long)slot * hd + (long)m * half + (long)jb * g.R) * g.K;
  }
  if (MODE == PH_GATEUP) return (m == 0 ? W : W2) + (long)t * g.R * g.K;
  return W + (long)t * g.R * g.K;
}

// ---- producer: stream the tiles of one phase --------------------------------
template <int MODE>
__device__ __forceinline__ void produce_phase(const MegaPhase& g, const bf16* W, const bf16* W2,
                                              int hd, uint8_t* ring, MegaShared* sh, Ring& rg,
                                              uint64_t pol, long long* tdbg = nullptr) {
  using T = PhTraits<MODE>;
  const int rows_unit = g.K * 2;
  int tn = 0;
  for (int t = blockIdx.x; t < g.tiles; t += gridDim.x) {
    const int s = rg.slot();
    mbar_wait_bounded(&sh->empty_bar[s], rg.parity() ^ 1u, &sh->err);
    if (tdbg && tn < 30) tdbg[tn++] = gtimer();
    int rows = g.R;
    if (MODE != PH_QKV) rows = min(g.R, g.N - t * g.R);
    const uint32_t bytes = (uint32_t)rows * rows_unit;
    mbar_expect_tx(&sh->full_bar[s], bytes * T::NRW);
    uint8_t* dst = ring + (long)s * MEGA_STAGE;
    bulk_g2s(dst, mega_tile_src<MODE>(g, W, W2, hd, t, 0), bytes, &sh->full_bar[s], pol);
    if (T::PAIR)
      bulk_g2s(dst + (long)g.R * rows_unit, mega_tile_src<MODE>(g, W, W2, hd, t, 1), bytes,
               &sh->full_bar[s], pol);
    rg.advance();
  }
}

// ---- q/k-norm phase (Qwen3-VL, language.py:84-89 then the rotary): one consumer warp per q head / new K row,
// in place in qbuf and the cache at ctx.  Loads and stores bypass L1 (the rows were written by other CTAs in the
// QKV phase, and the attention phase of other CTAs reads them after the next grid barrier).
template <int NU>
__device__ __forceinline__ void qk_norm_phase(const MegaP& p, int l, bf16* qbuf, bf16* kc, int ctx, int pos) {
  const DecodeDims& d = p.d;
  const int lane = threadIdx.x & 31;
  for (int slot = blockIdx.x * 8 + (threadIdx.x >> 5); slot < d.n_heads + d.n_kv; slot += gridDim.x * 8) {
    bf16* base = slot < d.n_heads ? qbuf + (long)slot * d.hd : kc + ((long)(slot - d.n_heads) * d.cap + ctx) * d.hd;
    float x[NU];
#pragma unroll
    for (int u = 0; u < NU; ++u) x[u] = bf2f(__ldcg(base + lane + 32 * u));
    warp_head_rms<NU>(x, slot < d.n_heads ? p.qn[l] : p.kn[l], d.eps);
    warp_head_rope<NU>(x, pos, p.inv_freq);
#pragma unroll
    for (int u = 0; u < NU; ++u) __stcg(base + lane + 32 * u, f2bf(x[u]));
  }
}

// ---- consumers: one GEMV phase ----------------------------------------------
struct PhaseIO {
  const bf16* x;     // activation vector (cross-CTA: read with ld.cg)
  const bf16* lnw;   // RMSNorm weight
  const bf16* bias;  // QKV
  bf16* out;         // h / act / logits / qbuf
  bf16 *kc, *vc;     // QKV
  float2* partials;  // HEAD
  const float* xpart;  // ORES: partial attention outputs to be summed (instead of x)
};

template <int MODE, int CHX>
__device__ __forceinline__ void consume_phase(const MegaP& p, const MegaPhase& g, const PhaseIO& io,
                                              uint8_t* ring, uint8_t* xs_raw, MegaShared* sh,
                                              Ring& rg, int ctx, int pos,
                                              long long* tdbg = nullptr) {
  using T = PhTraits<MODE>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int tn = 0;
  if (tdbg && threadIdx.x == 0) tdbg[tn++] = gtimer();
  const int rloc = warp % g.R, sub = warp / g.R;
  const int nvec = g.K >> 3;
  const int cb = (int)((long)nvec * sub / g.S), ce = (int)((long)nvec * (sub + 1) / g.S);
  const int rows_unit = g.K * 2;
  // ---- prologue: the 256 consumer threads load / RMS-normalise the activation vector ONCE
  // per CTA into shared memory (one global round trip, two block barriers); each warp then
  // takes its register slice from there.  (Per-warp redundant normalisation cost 2.4 us of
  // every NORM phase in the round-1 timeline; this costs 0.8-1.0 us.)
  uint4* xs = reinterpret_cast<uint4*>(xs_raw);
  {
    float ss = 0.f;
    for (int c = threadIdx.x; c < nvec; c += 256) {
      uint4 v;
      if ((MODE == PH_ORES || MODE == PH_DRES) && io.xpart) {
        // x = bf16( sum over the ATT_UN key ranges of the partial attention outputs )
        const DecodeDims& d = p.d;
        const int d0 = c * 8, h = d0 / d.hd, Gall = d.n_heads / d.n_kv, G = (Gall + p.hsplit - 1) / p.hsplit;
        const int grp = (h / Gall) * p.hsplit + (h % Gall) / G, gi = (h % Gall) % G;
        const float* src = io.xpart + (long)grp * ATT_UN * MEGA_ATT_G * d.hd + (long)gi * d.hd + (d0 % d.hd);
        float4 a[ATT_UN], b[ATT_UN];
#pragma unroll
        for (int u = 0; u < ATT_UN; ++u) {
          a[u] = __ldcg(reinterpret_cast<const float4*>(src + (long)u * MEGA_ATT_G * d.hd));
          b[u] = __ldcg(reinterpret_cast<const float4*>(src + (long)u * MEGA_ATT_G * d.hd + 4));
        }
        float4 sa = a[0], sb = b[0];
#pragma unroll
        for (int u = 1; u < ATT_UN; ++u) {
          sa.x += a[u].x; sa.y += a[u].y; sa.z += a[u].z; sa.w += a[u].w;
          sb.x += b[u].x; sb.y += b[u].y; sb.z += b[u].z; sb.w += b[u].w;
        }
        v.x = pack2(sa.x, sa.y);
        v.y = pack2(sa.z, sa.w);
        v.z = pack2(sb.x, sb.y);
        v.w = pack2(sb.z, sb.w);
      } else {
        v = ldcg16(io.x + (long)c * 8);
      }
      xs[c] = v;
      if (T::NORM) {
        float f[8];
        unpack8(v, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
      }
    }
    if (T::NORM) {
      ss = warp_sum(ss);
      if (lane == 0) sh->s_l[warp][0] = ss;
      cbar();
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) tot += sh->s_l[w][0];
      const float rs = 1.0f / sqrtf(tot / (float)g.K + p.d.eps);
      for (int c = threadIdx.x; c < nvec; c += 256) {
        float f[8], lf[8];
        unpack8(xs[c], f);
        unpack8(__ldg(reinterpret_cast<const uint4*>(io.lnw + (long)c * 8)), lf);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = rbf(rbf(f[j] * rs) * lf[j]);
        uint4 o;
        o.x = pack2(f[0], f[1]);
        o.y = pack2(f[2], f[3]);
        o.z = pack2(f[4], f[5]);
        o.w = pack2(f[6], f[7]);
        xs[c] = o;
      }
    }
    cbar();
  }
  uint4 xv[CHX];
#pragma unroll
  for (int u = 0; u < CHX; ++u) {
    const int c = cb + lane + 32 * u;
    xv[u] = (c < ce) ? xs[c] : make_uint4(0, 0, 0, 0);
  }
  if (tdbg && threadIdx.x == 0) tdbg[tn++] = gtimer();
  float run_m = -INFINITY, run_l = 0.f;
  // epilogue operands fetched BEFORE the tiles are waited for (off the critical path)
  float hpre = 0.f;  // ORES/DRES: lane i holds the residual value of this warp's i-th tile
  if ((MODE == PH_ORES || MODE == PH_DRES) && sub == 0) {
    const int t = blockIdx.x + lane * gridDim.x;
    const int r = t * g.R + rloc;
    if (t < g.tiles && r < g.N) hpre = ldcg_bf(io.out + r);
  }
  float pb1 = 0.f, pb2 = 0.f, pc = 1.f;  // QKV, first tile: bias + inverse frequency
  if (MODE == PH_QKV && (int)blockIdx.x < g.tiles) {
    const int hd = p.d.hd, half = hd >> 1;
    const int per_slot = half / g.R;
    const int slot = blockIdx.x / per_slot, j = (blockIdx.x % per_slot) * g.R + rloc;
    pb1 = bf2f(io.bias[slot * hd + j]);
    pb2 = bf2f(io.bias[slot * hd + j + half]);
    pc = p.inv_freq[j];  // raw inverse frequency; cos/sin are taken in the epilogue so that
                         // this load does not stall the warp before its tile
  }
  float keep0 = 0.f, keep1 = 0.f;
  // epilogue of tiles [it0, it0+cnt): lane i owns tile it0+i (only the slice-0 warps hold sums)
  auto flush = [&](int it0, int cnt) {
    const int ti = it0 + lane;
    const int t = blockIdx.x + ti * gridDim.x;
    const bool mine = (sub == 0) && (lane < cnt) && (t < g.tiles) &&
                      (MODE == PH_QKV || t * g.R + rloc < g.N);
    if (MODE == PH_QKV) {
      if (mine) {
        const int hd = p.d.hd, half = hd >> 1;
        const int per_slot = half / g.R;
        const int slot = t / per_slot, j = (t % per_slot) * g.R + rloc;
        const int r1 = slot * hd + j, r2 = r1 + half;
        const float y1 = rbf(keep0 + (ti == 0 ? pb1 : bf2f(io.bias[r1])));
        const float y2 = rbf(keep1 + (ti == 0 ? pb2 : bf2f(io.bias[r2])));
        if (slot >= p.d.n_heads + p.d.n_kv) {
          bf16* dst = io.vc + ((long)(slot - p.d.n_heads - p.d.n_kv) * p.d.cap + ctx) * hd;
          dst[j] = f2bf(y1);
          dst[j + half] = f2bf(y2);
        } else if (p.qk_norm) {  // raw q / k: the q/k-norm phase normalises and rotates them
          bf16* dst = (slot < p.d.n_heads) ? io.out + (long)slot * hd
                                           : io.kc + ((long)(slot - p.d.n_heads) * p.d.cap + ctx) * hd;
          dst[j] = f2bf(y1);
          dst[j + half] = f2bf(y2);
        } else {
          const float ang = (float)pos * (ti == 0 ? pc : p.inv_freq[j]);
          const float c = rbf(cosf(ang)), sn = rbf(sinf(ang));
          const float o1 = rbf(rbf(y1 * c) + rbf((-y2) * sn));
          const float o2 = rbf(rbf(y2 * c) + rbf(y1 * sn));
          bf16* dst = (slot < p.d.n_heads)
                          ? io.out + (long)slot * hd
                          : io.kc + ((long)(slot - p.d.n_heads) * p.d.cap + ctx) * hd;
          dst[j] = f2bf(o1);
          dst[j + half] = f2bf(o2);
        }
      }
    } else if (MODE == PH_GATEUP) {
      if (mine) io.out[t * g.R + rloc] = f2bf(swiglu_bf(rbf(keep0), rbf(keep1)));
    } else if (MODE == PH_ORES || MODE == PH_DRES) {
      if (mine) {
        const int r = t * g.R + rloc;
        const float hv = (it0 == 0) ? hpre : ldcg_bf(io.out + r);  // lane i prefetched tile i
        io.out[r] = f2bf(rbf(hv + rbf(keep0)));
      }
    } else {  // HEAD: logits + running logsumexp (warp-parallel over the 32 tiles)
      const float a = mine ? rbf(keep0) : -INFINITY;
      if (mine) io.out[t * g.R + rloc] = f2bf(a);
      const float m = warp_max(a);
      if (m > -INFINITY) {
        const float e = mine ? expf(a - m) : 0.f;
        const float l = warp_sum(e);
        const float mn = fmaxf(run_m, m);
        run_l = run_l * expf(run_m - mn) + l * expf(m - mn);
        run_m = mn;
      }
    }
  };
  int it = 0;
  for (int t = blockIdx.x; t < g.tiles; t += gridDim.x, ++it) {
    const int s = rg.slot();
    int rows = g.R;
    if (MODE != PH_QKV) rows = min(g.R, g.N - t * g.R);
    mbar_wait_bounded(&sh->full_bar[s], rg.parity(), &sh->err);
    if (tdbg && threadIdx.x == 0 && tn < 30) tdbg[tn++] = gtimer();
    rg.advance();
    const uint8_t* base = ring + (long)s * MEGA_STAGE + (long)rloc * rows_unit;
    float acc[T::NRW];
    {
      float a8[T::NRW][8];
#pragma unroll
      for (int m = 0; m < T::NRW; ++m)
#pragma unroll
        for (int j = 0; j < 8; ++j) a8[m][j] = 0.f;
      if (rloc < rows) {
        // the whole tile slice of this warp -> registers first (one LDS latency per tile),
        // then NRW*8 independent FMA chains
        uint4 w4[T::NRW][CHX];
#pragma unroll
        for (int u = 0; u < CHX; ++u) {
          const int c = cb + lane + 32 * u;
#pragma unroll
          for (int m = 0; m < T::NRW; ++m)
            w4[m][u] = (c < ce) ? *reinterpret_cast<const uint4*>(base + (long)m * g.R * rows_unit +
                                                                  (long)c * 16)
                                : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < CHX; ++u) {
          float xf[8];
          unpack8(xv[u], xf);
#pragma unroll
          for (int m = 0; m < T::NRW; ++m) {
            float wf[8];
            unpack8(w4[m][u], wf);
#pragma unroll
            for (int j = 0; j < 8; j += 2)
              ffma2(a8[m][j], a8[m][j + 1], wf[j], wf[j + 1], xf[j], xf[j + 1]);
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
    if (lane == 0) mbar_arrive(&sh->empty_bar[s]);
    if (tdbg && threadIdx.x == 0 && tn < 30) tdbg[tn++] = gtimer();
    if (g.S > 1) {
      if (lane == 0) {
#pragma unroll
        for (int m = 0; m < T::NRW; ++m) sh->red[it & 1][warp][m] = acc[m];
      }
      cbar();
      if (sub == 0) {
#pragma unroll
        for (int m = 0; m < T::NRW; ++m) {
          float a = 0.f;
          for (int q = 0; q < g.S; ++q) a += sh->red[it & 1][rloc + q * g.R][m];
          acc[m] = a;
        }
      }
    }
    // ---- deferred epilogue: lane (it % 32) keeps this tile's sums; the per-row math
    // (SwiGLU / rotary / residual / logsumexp) runs once per 32 tiles, one tile per lane,
    // instead of once per tile on lane 0 (measured: 0.38 us of a 1.02 us tile period)
    if (lane == (it & 31)) {
      keep0 = acc[0];
      keep1 = acc[T::NRW - 1];
    }
    if ((it & 31) == 31) flush(it - 31, 32);
  }
  if (it & 31) flush(it & ~31, it & 31);
  if (MODE == PH_HEAD) {
    if (lane == 0) sh->wstat[warp] = make_float2(run_m, run_l);
    cbar();
    if (threadIdx.x == 0) {
      float M = -INFINITY;
      for (int i = 0; i < 8; ++i) M = fmaxf(M, sh->wstat[i].x);
      float L = 0.f;
      for (int i = 0; i < 8; ++i)
        if (sh->wstat[i].y > 0.f) L += sh->wstat[i].y * expf(sh->wstat[i].x - M);
      io.partials[blockIdx.x] = make_float2(M, L);
    }
  }
}

}  // namespace

template <int CHH, int CHI>
__global__ void __launch_bounds__(MEGA_THREADS, 1) k_mega(const MegaP p) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ MegaShared sh;
  uint8_t* ring = sm;
  uint8_t* xs = sm + (long)p.n_stages * MEGA_STAGE;  // activation vector (GEMV phases) /
  float* scratch = reinterpret_cast<float*>(xs);     // attention scratch (attention phase)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (p.st->error) return;  // a previous step gave up: do not spin again
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(&sh.full_bar[s], 1);
      mbar_init(&sh.empty_bar[s], 8);
    }
    sh.err = 0;
    sh.bar_base = p.st->bar_base;
    sh.att_base = p.st->att_base;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
  }
  __syncthreads();
  Ring rg;
  rg.cur = 0;
  rg.ph = 0;
  rg.n_stages = p.n_stages;
  const DecodeDims& d = p.d;

  if (warp == 8) {
    // ===== producer: the whole step's weight stream, never blocked by a phase =====
    if (lane == 0) {
      const uint64_t pol = policy_evict_first();
      for (int l = 0; l < p.n_layers; ++l) {
        const LayerW& lw = p.layers[l];
        produce_phase<PH_QKV>(p.ph[PH_QKV], lw.wqkv, nullptr, d.hd, ring, &sh, rg, pol);
        produce_phase<PH_ORES>(p.ph[PH_ORES], lw.wo, nullptr, d.hd, ring, &sh, rg, pol);
        produce_phase<PH_GATEUP>(p.ph[PH_GATEUP], lw.wgu, lw.wgu + (long)d.inter * d.hidden, d.hd, ring, &sh, rg,
                                 pol, (p.dbg && l == 5 && blockIdx.x == 0) ? p.dbg + 4096 + 96 : nullptr);
        produce_phase<PH_DRES>(p.ph[PH_DRES], lw.wd, nullptr, d.hd, ring, &sh, rg, pol);
      }
      produce_phase<PH_HEAD>(p.ph[PH_HEAD], p.head, nullptr, d.hd, ring, &sh, rg, pol);
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
    {
      PhaseIO io = {p.h, lw.ln1, lw.bqkv, p.qbuf, kc, vc, nullptr, nullptr};
      consume_phase<PH_QKV, CHH>(p, p.ph[PH_QKV], io, ring, xs, &sh, rg, ctx, pos);
    }
    grid_barrier(p, &sh, bidx);
    if (p.qk_norm) {
      if (d.hd == 128) qk_norm_phase<4>(p, l, p.qbuf, kc, ctx, pos);
      else qk_norm_phase<2>(p, l, p.qbuf, kc, ctx, pos);
      grid_barrier(p, &sh, bidx);
    }
    if ((int)blockIdx.x < p.attn_ctas) {
      if (d.hd == 128) attn_phase<128>(p, kc, vc, scratch, &sh, ctx + 1, l,
                                       (p.dbg && l == 5 && blockIdx.x < 2) ? p.dbg + 4096 + 128 + 32 * blockIdx.x : nullptr);
      else attn_phase<64>(p, kc, vc, scratch, &sh, ctx + 1, l);
    }
    grid_barrier(p, &sh, bidx);
    {
      PhaseIO io = {p.attn, nullptr, nullptr, p.h, nullptr, nullptr, nullptr, p.att_part};
      if (p.ph[PH_ORES].S == 1) consume_phase<PH_ORES, CHH>(p, p.ph[PH_ORES], io, ring, xs, &sh, rg, 0, 0);
      else consume_phase<PH_DRES, CHH>(p, p.ph[PH_ORES], io, ring, xs, &sh, rg, 0, 0);
    }
    grid_barrier(p, &sh, bidx);
    {
      PhaseIO io = {p.h, lw.ln2, nullptr, p.act, nullptr, nullptr, nullptr, nullptr};
      long long* td = (p.dbg && l == 5 && (blockIdx.x == 0 || blockIdx.x == 77))
                          ? p.dbg + 4096 + (blockIdx.x ? 32 : 0) : nullptr;
      consume_phase<PH_GATEUP, CHH>(p, p.ph[PH_GATEUP], io, ring, xs, &sh, rg, 0, 0, td);
    }
    grid_barrier(p, &sh, bidx);
    {
      PhaseIO io = {p.act, nullptr, nullptr, p.h, nullptr, nullptr, nullptr, nullptr};
      long long* td = (p.dbg && l == 5 && blockIdx.x == 0) ? p.dbg + 4096 + 64 : nullptr;
      consume_phase<PH_DRES, CHI>(p, p.ph[PH_DRES], io, ring, xs, &sh, rg, 0, 0, td);
    }
    grid_barrier(p, &sh, bidx);
  }
  {
    PhaseIO io = {p.h, p.final_norm, nullptr, p.logits, nullptr, nullptr, p.partials, nullptr};
    consume_phase<PH_HEAD, CHH>(p, p.ph[PH_HEAD], io, ring, xs, &sh, rg, 0, 0);
  }
  grid_barrier(p, &sh, bidx);
  mega_sample_finalize(p, sh, bidx);
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static int mega_geometry(MegaPhase& g, int K, int N, bool pair, int units) {
  g.K = K;
  g.N = N;
  const long unit = (long)K * 2 * (pair ? 2 : 1);
  int R = 8;
  while (R > 1 && (R * unit > MEGA_STAGE || R > units)) R >>= 1;
  // as decode.cu::stream_geometry: more K slices when a slice would exceed the 10 chunks per lane of the largest
  // instantiation (K = 6144, Qwen3-VL-2B's down projection)
  while (R > 1 && cdiv(cdiv(K >> 3, 8 / R), 32) > 10) R >>= 1;
  B200_REQUIRE(R * unit <= MEGA_STAGE, "mega: K=%d does not fit a %d-byte ring stage", K, MEGA_STAGE);
  g.R = R;
  g.S = 8 / R;
  return B200_OK;
}

// region after the ring: attention scratch, or the activation vector of a GEMV phase.
// The scratch holds (MEGA_ATT_G + 2) * head_dim floats that attn_phase does not use, and
// mega_spare_bytes() follows it unused: together they keep the ring depth and the cache capacity
// at which decode gives way to the per-phase kernels where they were measured.
static size_t mega_attn_scratch(const DecodeDims& d) {
  const size_t att = ((size_t)MEGA_ATT_G * cdiv(d.cap, ATT_UN) + (size_t)8 * MEGA_ATT_G * d.hd +
                      (size_t)(MEGA_ATT_G + 2) * d.hd) * 4;
  const size_t xs = (size_t)max(max(d.inter, d.hidden), d.n_heads * d.hd) * 2;
  return ((att > xs ? att : xs) + 127) & ~(size_t)127;
}
static size_t mega_spare_bytes(const DecodeDims& d) { return ((size_t)d.hidden * 2 + 127) & ~(size_t)127; }

int mega_fill(MegaP& p, int sm_count) {
  const DecodeDims& d = p.d;
  int rc;
  const int half = d.hd / 2;
  if ((rc = mega_geometry(p.ph[PH_QKV], d.hidden, 0, true, half))) return rc;
  B200_REQUIRE(half % p.ph[PH_QKV].R == 0, "mega: head_dim/2 %% tile rows != 0");
  p.ph[PH_QKV].tiles = (d.n_heads + 2 * d.n_kv) * (half / p.ph[PH_QKV].R);
  if ((rc = mega_geometry(p.ph[PH_ORES], d.n_heads * d.hd, d.hidden, false, d.hidden))) return rc;
  p.ph[PH_ORES].tiles = cdiv(d.hidden, p.ph[PH_ORES].R);
  if ((rc = mega_geometry(p.ph[PH_GATEUP], d.hidden, d.inter, true, d.inter))) return rc;
  p.ph[PH_GATEUP].tiles = cdiv(d.inter, p.ph[PH_GATEUP].R);
  if ((rc = mega_geometry(p.ph[PH_DRES], d.inter, d.hidden, false, d.hidden))) return rc;
  p.ph[PH_DRES].tiles = cdiv(d.hidden, p.ph[PH_DRES].R);
  if ((rc = mega_geometry(p.ph[PH_HEAD], d.hidden, d.vocab, false, d.vocab))) return rc;
  p.ph[PH_HEAD].tiles = cdiv(d.vocab, p.ph[PH_HEAD].R);
  const int G = d.n_heads / d.n_kv;
  int hs = (G + MEGA_ATT_G - 1) / MEGA_ATT_G;  // <= MEGA_ATT_G q heads per CTA, uneven split allowed
  if (hs == 1 && G % 2 == 0 && G >= 4) hs = 2;
  p.hsplit = hs;
  p.attn_ctas = d.n_kv * hs * ATT_UN;
  B200_REQUIRE(p.attn_ctas <= sm_count, "mega: %d attention CTAs > %d SMs", p.attn_ctas, sm_count);
  B200_REQUIRE(d.hd == 64 || d.hd == 128, "mega: head_dim %d (64|128)", d.hd);
  const size_t scratch = mega_attn_scratch(d);
  p.scratch_bytes = (int)scratch;
  const long budget = 227 * 1024 - 2048 - (long)scratch - (long)mega_spare_bytes(d);
  int ns = (int)(budget / MEGA_STAGE);
  B200_REQUIRE(ns >= 2, "mega: cache capacity %d leaves no room for the weight ring", d.cap);
  p.n_stages = ns > 8 ? 8 : ns;
  p.stage_bytes = MEGA_STAGE;
  return B200_OK;
}

static int mega_chx(const MegaPhase& g) { return cdiv(cdiv(g.K >> 3, g.S), 32); }

template <int CHH, int CHI>
static int launch_k_mega(const MegaP& p, int grid, size_t smem, cudaStream_t s) {
  int rc;
  if ((rc = kernel_opt_in((const void*)k_mega<CHH, CHI>, 227 * 1024 - 2048, true))) return rc;
  // COOPERATIVE launch: the software grid barrier needs every CTA resident at once; the driver
  // refuses the launch (instead of letting it deadlock) if the grid cannot be co-resident, and
  // never schedules it partially next to another kernel.
  B200_CUDA(launch(k_mega<CHH, CHI>, dim3(grid), dim3(MEGA_THREADS), smem, s, LaunchOpts{false, 0, true}, p));
  return B200_OK;
}

int mega_launch(const MegaP& p, int sm_count, cudaStream_t s) {
  const size_t smem = (size_t)p.n_stages * MEGA_STAGE + mega_attn_scratch(p.d) + mega_spare_bytes(p.d);
  int chh = mega_chx(p.ph[PH_QKV]);
  chh = max(chh, mega_chx(p.ph[PH_ORES]));
  chh = max(chh, mega_chx(p.ph[PH_GATEUP]));
  chh = max(chh, mega_chx(p.ph[PH_HEAD]));
  const int chi = mega_chx(p.ph[PH_DRES]);
  // every CTA must be resident at once (software grid barrier): one CTA per SM
  const int grid = sm_count;
  if (chh <= 2 && chi <= 2) return launch_k_mega<2, 2>(p, grid, smem, s);
  if (chh <= 6 && chi <= 10) return launch_k_mega<6, 10>(p, grid, smem, s);
  if (chh <= 8 && chi <= 10) return launch_k_mega<8, 10>(p, grid, smem, s);  // Qwen2-VL-7B widths
  if (chh <= 10 && chi <= 10) return launch_k_mega<10, 10>(p, grid, smem, s);
  set_error("mega: unsupported widths (hidden chunks %d, inter chunks %d per lane)", chh, chi);
  return B200_ERR_INVALID;
}

}  // namespace b200
