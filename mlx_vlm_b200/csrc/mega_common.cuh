// Device pieces of the persistent decode kernel k_mega (decode_mega.cu): the software grid barrier,
// the distributed attention phase and the sampler.
#pragma once
#include "common.cuh"
#include "decode.cuh"

namespace b200 {

namespace {

// activations written by other CTAs in an earlier phase: read through L2
__device__ __forceinline__ uint4 ldcg16(const void* p) {
  return __ldcg(reinterpret_cast<const uint4*>(p));
}
__device__ __forceinline__ float ldcg_bf(const bf16* p) {
  return __uint_as_float((uint32_t)__ldcg(reinterpret_cast<const unsigned short*>(p)) << 16);
}
// (d0,d1) += (a0,a1) * (b0,b1): two IEEE fp32 FMAs (Hopper has no packed fp32 FMA)
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = __fmaf_rn(a0, b0, d0);
  d1 = __fmaf_rn(a1, b1, d1);
}
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

enum { PH_QKV = 0, PH_ORES = 1, PH_GATEUP = 2, PH_DRES = 3, PH_HEAD = 4 };

__device__ __forceinline__ long long gtimer() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

template <int MODE>
struct PhTraits {
  static constexpr bool PAIR = (MODE == PH_QKV || MODE == PH_GATEUP);
  static constexpr bool NORM = (MODE == PH_QKV || MODE == PH_GATEUP || MODE == PH_HEAD);
  static constexpr int NRW = PAIR ? 2 : 1;
};

}  // namespace

constexpr int MEGA_THREADS = 288;
constexpr int MEGA_STAGE = 48 * 1024;
constexpr int MEGA_ATT_G = 4;
constexpr int ATT_UN = 8;  // key ranges per (kv head, q-head group) in the attention phase

struct MegaShared {
  uint64_t full_bar[8], empty_bar[8];
  float red[2][8][2];
  float2 wstat[8];
  float s_m[8][MEGA_ATT_G], s_l[8][MEGA_ATT_G];
  unsigned long long bar_base;
  unsigned long long att_base;
  float lse;
  unsigned long long best;
  int feed;
  int err;
};

// ring position shared by producer and consumers (each keeps its own copy)
struct Ring {
  int cur;        // ring slot of the next tile
  uint32_t ph;    // its phase parity
  int n_stages;
  __device__ __forceinline__ int slot() const { return cur; }
  __device__ __forceinline__ uint32_t parity() const { return ph; }
  __device__ __forceinline__ void advance() {  // no integer division on the per-tile path
    if (++cur == n_stages) {
      cur = 0;
      ph ^= 1u;
    }
  }
};


namespace {

// ---- consumers: attention ------------------------------------------------------
// Under the weight stream every dependent global round trip costs ~1 us, so the phase
// is built around the NUMBER of such trips.  CTA (grp, unit): grp = (kv head, q-head
// group), unit = one of ATT_UN key ranges.
//   1. all q / K / V requests of the CTA are issued up front; scores of the OWN key range
//      (coalesced: 8 lanes per key, 4 keys per warp instruction, software-pipelined trips),
//      local (max, sum exp) per head;
//   2. the ATT_UN x heads statistics are exchanged as self-validating {value, epoch} words
//      polled by one warp (no counter, no separate load): global (M, L) by a butterfly;
//   3. p = bf16(exp(s - M) / L) precomputed cooperatively, partial P.V -> global fp32;
//   4. the partial outputs are summed, in a fixed order, by the o_proj prologue.
// Measured history of this phase (tools/mega_timeline.py, ctx ~470): one CTA per (kv head,
// group) 15.9 us; one CTA per q head 17.1 us; every unit recomputing all scores 11.1 us;
// counter barrier + last-arriver combine 10.6 us; one-warp statistics read, no combine 5.4 us;
// polled statistics words 4.7 us.
template <int HD>
__device__ __forceinline__ void attn_phase(const MegaP& p, const bf16* kc, const bf16* vc,
                                           float* scratch, MegaShared* sh, int nkeys, int layer,
                                           long long* tdbg = nullptr) {
  int tn = 0;
#define ATT_STAMP() do { if (tdbg && threadIdx.x == 0 && tn < 30) tdbg[tn++] = gtimer(); } while (0)
  ATT_STAMP();
  constexpr int EPL = HD / 32, SEG = HD / 8, AG = MEGA_ATT_G, NV = SEG / 8, UNR = 2;
  const DecodeDims& d = p.d;
  const int Gall = d.n_heads / d.n_kv;
  // q heads of a kv head are split over p.hsplit CTAs, Gc per CTA; the last part may hold fewer
  // (Qwen2-VL-7B: 7 q heads per kv head -> 4 + 3)
  const int Gc = (Gall + p.hsplit - 1) / p.hsplit;
  const int ucap = (d.cap + ATT_UN - 1) / ATT_UN;
  float* sc = scratch;                       // [AG][ucap]
  float* red = sc + (long)AG * ucap;         // [8][AG*HD]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = blockIdx.x / ATT_UN, unit = blockIdx.x % ATT_UN;
  const int kvh = grp / p.hsplit, part = grp % p.hsplit;
  const int G = min(Gc, Gall - part * Gc);
  const int h0 = kvh * Gall + part * Gc;
  const bf16* kb = kc + (long)kvh * d.cap * HD;
  const bf16* vb = vc + (long)kvh * d.cap * HD;
  const int per = (nkeys + ATT_UN - 1) / ATT_UN;
  const int u0 = min(nkeys, unit * per), u1 = min(nkeys, u0 + per);
  const int seg = lane & 7, ksub = lane >> 3;
  // ---- all global requests of the phase are issued before the first use: q, the first
  // 2 x 4 keys of this warp, and the V rows of its first VPRE keys (one round trip) ----
  constexpr int VPRE = 8;
  uint4 qraw[AG][NV];
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int v = 0; v < NV; ++v)
      qraw[g][v] = (g < G) ? ldcg16(p.qbuf + (long)(h0 + g) * HD + seg * SEG + v * 8)
                           : make_uint4(0, 0, 0, 0);
  uint4 kvn[UNR][NV];
  {
    const int j0 = u0 + warp * 4;
#pragma unroll
    for (int q = 0; q < UNR; ++q) {
      const int j = j0 + 32 * q + ksub;
#pragma unroll
      for (int v = 0; v < NV; ++v)
        kvn[q][v] = (j < u1) ? ldcg16(kb + (long)j * HD + seg * SEG + v * 8) : make_uint4(0, 0, 0, 0);
    }
  }
  uint2 vraw[VPRE];
#pragma unroll
  for (int q = 0; q < VPRE; ++q) {
    const int j = u0 + warp + 8 * q;
    vraw[q] = make_uint2(0, 0);
    if (j < u1) {
      const bf16* vr = vb + (long)j * HD + lane * EPL;
      if (EPL == 4) vraw[q] = __ldcg(reinterpret_cast<const uint2*>(vr));
      else vraw[q].x = __ldcg(reinterpret_cast<const uint32_t*>(vr));
    }
  }
  float qr[AG][SEG];
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      float f[8];
      unpack8(qraw[g][v], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) qr[g][v * 8 + i] = rbf(f[i] * d.scale_bf);
    }
  ATT_STAMP();  // q loaded
  // ---- 1. scores of the own range (software-pipelined over trips of 2 x 4 keys) ----
  float lm[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) lm[g] = -INFINITY;
  for (int j0 = u0 + warp * 4; j0 < u1; j0 += 32 * UNR) {
    uint4 kv[UNR][NV];
#pragma unroll
    for (int q = 0; q < UNR; ++q)
#pragma unroll
      for (int v = 0; v < NV; ++v) kv[q][v] = kvn[q][v];
    if (j0 + 32 * UNR < u1) {
#pragma unroll
      for (int q = 0; q < UNR; ++q) {
        const int j = j0 + 32 * UNR + 32 * q + ksub;
#pragma unroll
        for (int v = 0; v < NV; ++v)
          kvn[q][v] = (j < u1) ? ldcg16(kb + (long)j * HD + seg * SEG + v * 8)
                                : make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int q = 0; q < UNR; ++q) {
      const int j = j0 + 32 * q + ksub;
      float s[AG];
#pragma unroll
      for (int g = 0; g < AG; ++g) s[g] = 0.f;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        float kf[8];
        unpack8(kv[q][v], kf);
#pragma unroll
        for (int g = 0; g < AG; ++g)
#pragma unroll
          for (int i = 0; i < 8; ++i) s[g] = fmaf(qr[g][v * 8 + i], kf[i], s[g]);
      }
#pragma unroll
      for (int o = 1; o < 8; o <<= 1)
#pragma unroll
        for (int g = 0; g < AG; ++g) s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
      if (j < u1 && seg == 0) {
#pragma unroll
        for (int g = 0; g < AG; ++g) {
          const float r = rbf(s[g]);
          sc[(long)g * ucap + (j - u0)] = r;
          lm[g] = fmaxf(lm[g], r);
        }
      }
    }
  }
  ATT_STAMP();  // scores done
  float vpre[VPRE][EPL];
#pragma unroll
  for (int q = 0; q < VPRE; ++q) {
    if (EPL == 4) {
      float t4[4];
      unpack4(vraw[q], t4);
#pragma unroll
      for (int e = 0; e < EPL; ++e) vpre[q][e] = t4[e];
    } else {
      vpre[q][0] = __uint_as_float(vraw[q].x << 16);
      vpre[q][EPL - 1] = __uint_as_float(vraw[q].x & 0xffff0000u);
    }
  }
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    lm[g] = warp_max(lm[g]);
    if (lane == 0) sh->s_m[warp][g] = lm[g];
  }
  cbar();
  float ml[AG], ls[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    float m = -INFINITY;
#pragma unroll
    for (int w = 0; w < 8; ++w) m = fmaxf(m, sh->s_m[w][g]);
    ml[g] = m;
    ls[g] = 0.f;
  }
  for (int j = threadIdx.x; j < u1 - u0; j += 256) {
#pragma unroll
    for (int g = 0; g < AG; ++g) ls[g] += expf(sc[(long)g * ucap + j] - ml[g]);
  }
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    ls[g] = warp_sum(ls[g]);
    if (lane == 0) sh->s_l[warp][g] = ls[g];
  }
  cbar();
  ATT_STAMP();  // local stats done
  // ---- 2 + 3. exchange the softmax statistics inside the group WITHOUT a counter: every
  // (unit, head) pair is published as two self-validating 8-byte words {float bits, epoch}
  // (8-byte accesses are single-copy atomic; the epoch changes every attention phase), and
  // ONE warp (lane = u*AG + g) polls the 32 pairs directly.  This replaces
  // store + atomic arrive + counter poll + stats load (3 dependent L2 round trips) by
  // store + poll (round 1: 750 -> 897 tok/s came from shortening this chain).
  {
    static_assert(ATT_UN * MEGA_ATT_G == 32, "one lane per (unit, head)");
    unsigned long long* gw = reinterpret_cast<unsigned long long*>(p.att_stats) + (long)grp * ATT_UN * AG * 2;
    const uint32_t epoch = (uint32_t)(sh->att_base + (unsigned long long)layer + 1ull);
    if (warp == 0) {
      if (lane < AG) {
        float l = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) l += sh->s_l[w][lane];
        const float lv = (u1 > u0) ? l : 0.f;
        const unsigned long long wm = ((unsigned long long)__float_as_uint(ml[lane]) << 32) | epoch;
        const unsigned long long wl = ((unsigned long long)__float_as_uint(lv) << 32) | epoch;
        asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(gw + (long)(unit * AG + lane) * 2),
                     "l"(wm), "l"(wl)
                     : "memory");
      }
      unsigned long long a, b;
      unsigned spins = 0;
      do {
        asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(gw + (long)lane * 2) : "memory");
        if (++spins > (1u << 22)) {
          sh->err = 3;
          break;
        }
      } while ((uint32_t)a != epoch || (uint32_t)b != epoch);
      const float sx = __uint_as_float((uint32_t)(a >> 32)), sy = __uint_as_float((uint32_t)(b >> 32));
      // max / rescaled sum over the units of head g = lane % AG: butterfly over the unit bits
      float m = sx;
#pragma unroll
      for (int o = AG; o < 32; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      float l = (sy > 0.f) ? sy * expf(sx - m) : 0.f;
#pragma unroll
      for (int o = AG; o < 32; o <<= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
      if (lane < AG) {
        sh->s_m[0][lane] = m;
        sh->s_l[0][lane] = l;
      }
    }
  }
  cbar();
  ATT_STAMP();  // statistics exchanged
  float M[AG], L[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) {
    M[g] = sh->s_m[0][g];
    L[g] = sh->s_l[0][g];
  }
  // p = bf16(exp(s - M) / L) for the own keys, one key per thread, in place
  for (int j = threadIdx.x; j < u1 - u0; j += 256) {
#pragma unroll
    for (int g = 0; g < AG; ++g)
      sc[(long)g * ucap + j] = rbf(expf(sc[(long)g * ucap + j] - M[g]) / L[g]);
  }
  cbar();
  ATT_STAMP();  // global stats read
  float acc[AG][EPL];
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[g][e] = 0.f;
#pragma unroll
  for (int q = 0; q < VPRE; ++q) {
    const int j = u0 + warp + 8 * q;
    if (j < u1) {
#pragma unroll
      for (int g = 0; g < AG; ++g) {
        const float pj = sc[(long)g * ucap + (j - u0)];
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[g][e] = fmaf(pj, vpre[q][e], acc[g][e]);
      }
    }
  }
  for (int j0 = u0 + warp + 8 * VPRE; j0 < u1; j0 += 32) {  // 4 keys per trip, loads first
    float vf[4][EPL];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + 8 * q;
#pragma unroll
      for (int e = 0; e < EPL; ++e) vf[q][e] = 0.f;
      if (j < u1) {
        const bf16* vr = vb + (long)j * HD + lane * EPL;
        if (EPL == 4) {
          float t4[4];
          unpack4(__ldcg(reinterpret_cast<const uint2*>(vr)), t4);
#pragma unroll
          for (int e = 0; e < EPL; ++e) vf[q][e] = t4[e];
        } else {
          const uint32_t w = __ldcg(reinterpret_cast<const uint32_t*>(vr));
          vf[q][0] = __uint_as_float(w << 16);
          vf[q][EPL - 1] = __uint_as_float(w & 0xffff0000u);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + 8 * q;
      if (j < u1) {
#pragma unroll
        for (int g = 0; g < AG; ++g) {
          const float pj = sc[(long)g * ucap + (j - u0)];
#pragma unroll
          for (int e = 0; e < EPL; ++e) acc[g][e] = fmaf(pj, vf[q][e], acc[g][e]);
        }
      }
    }
  }
#pragma unroll
  for (int g = 0; g < AG; ++g)
#pragma unroll
    for (int e = 0; e < EPL; ++e) red[((long)warp * AG + g) * HD + lane * EPL + e] = acc[g][e];
  ATT_STAMP();  // PV done
  cbar();
  float* mypart = p.att_part + ((long)grp * ATT_UN + unit) * AG * HD;
  for (int i = threadIdx.x; i < G * HD; i += 256) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[(long)w * AG * HD + i];
    mypart[i] = s;
  }
  cbar();
  // (the ATT_UN partial outputs are summed, in a fixed order, by the o_proj prologue)
  ATT_STAMP();  // end
#undef ATT_STAMP
}

// software grid barrier among the consumer threads of all CTAs
__device__ __forceinline__ void grid_barrier(const MegaP& p, MegaShared* sh, unsigned& idx) {
  cbar();
  if (threadIdx.x == 0) {
    if (p.dbg && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1))
      p.dbg[((blockIdx.x ? 1 : 0) * 1024 + idx) * 2] = gtimer();
    const unsigned long long target = sh->bar_base + (unsigned long long)(idx + 1) * gridDim.x;
    // release: the CTA's writes (ordered before by bar.sync) become visible before the count
    asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(p.bar), "l"(1ull) : "memory");
    unsigned spins = 0;
    while (ld_acquire_u64(p.bar) < target) {
      if (++spins > (1u << 22)) {
        sh->err = 1;
        break;
      }
    }
    if (p.dbg && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1))
      p.dbg[((blockIdx.x ? 1 : 0) * 1024 + idx) * 2 + 1] = gtimer();
  }
  ++idx;
  cbar();
}

// ---- sampler + end-of-step bookkeeping (all consumer threads of all CTAs) -----------
__device__ __forceinline__ void mega_sample_finalize(const MegaP& p, MegaShared& sh, unsigned& bidx) {
  const DecodeDims& d = p.d;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // ---- sampler: logprobs = bf16(logits - bf16(lse)), argmax with lowest index ----
  if (warp == 0) {
    float M = -INFINITY;
    for (int i = lane; i < (int)gridDim.x; i += 32) M = fmaxf(M, __ldcg(&p.partials[i]).x);
    M = warp_max(M);
    float L = 0.f;
    for (int i = lane; i < (int)gridDim.x; i += 32) {
      const float2 pr = __ldcg(&p.partials[i]);
      if (pr.y > 0.f) L += pr.y * expf(pr.x - M);
    }
    L = warp_sum(L);
    if (lane == 0) {
      sh.lse = rbf(M + logf(L));
      sh.best = 0ull;
    }
  }
  cbar();
  {
    const float lse = sh.lse;
    unsigned long long best = 0ull;
    const int nvec = (d.vocab + 7) >> 3;  // the tail of an odd vocabulary holds -inf (preset at creation)
    for (int c = blockIdx.x * 256 + threadIdx.x; c < nvec; c += gridDim.x * 256) {
      float f[8], o[8];
      unpack8(ldcg16(p.logits + (long)c * 8), f);
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
      *reinterpret_cast<uint4*>(p.logprobs + (long)c * 8) = ov;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if (lane == 0) atomicMax(&sh.best, best);
    cbar();
    if (threadIdx.x == 0) atomicMax(&p.st->best_key, sh.best);
  }
  grid_barrier(p, &sh, bidx);
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) {
      const unsigned long long key = ld_acquire_u64(&p.st->best_key);
      const int tok = (int)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
      const int n = p.st->n_out;
      p.token_log[n % p.log_cap] = tok;
      int feed = tok;
      if (p.st->use_force) feed = p.force[n % p.log_cap];
      sh.feed = feed;
      p.st->tok = feed;
      p.st->n_out = n + 1;
      p.st->ctx += p.advance;
      p.st->pos += p.advance;
      p.st->best_key = 0ull;
      p.st->bar_base = sh.bar_base + (unsigned long long)bidx * gridDim.x;
      p.st->att_base = sh.att_base + (unsigned long long)p.n_layers;
      if (sh.err) p.st->error = sh.err;
    }
    cbar();
    const int feed = sh.feed;
    const int nv = d.hidden >> 3;
    for (int c = threadIdx.x; c < nv; c += 256)
      *reinterpret_cast<uint4*>(p.h + c * 8) =
          __ldg(reinterpret_cast<const uint4*>(p.embed + (long)feed * d.hidden + c * 8));
  } else if (threadIdx.x == 0 && sh.err) {
    p.st->error = sh.err;
  }
}

}  // namespace

}  // namespace b200
