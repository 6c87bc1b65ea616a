// Device pieces shared by the two persistent decode kernels (k_mega: CUDA-core consumers,
// decode_mega.cu; k_mega_tc: wgmma consumers, decode_mega_tc.cu): mbarrier / bulk-copy
// wrappers, the software grid barrier, the distributed attention phase and the sampler.
#pragma once
#include "common.cuh"
#include "decode.cuh"

namespace b200 {

namespace {

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
// bounded wait: a scheduling bug must not hang the GPU (sets *err and falls through)
__device__ __forceinline__ void mb_wait(uint64_t* bar, uint32_t parity, int* err) {
  uint32_t done;
  const uint32_t addr = s_u32(bar);
  unsigned spins = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (!done && ++spins > (1u << 20)) {
      *err = 2;
      break;
    }
  } while (!done);
}
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
// activations written by other CTAs in an earlier phase: read through L2
__device__ __forceinline__ uint4 ldcg16(const void* p) {
  return __ldcg(reinterpret_cast<const uint4*>(p));
}
// ---- self-validating activation words (dataflow mode of k_mega) -------------------------
// A value that crosses CTAs inside a layer is published as an 8-byte word {payload << 32 |
// epoch}; 8-byte accesses are single-copy atomic, the epoch is unique per (step, layer), so a
// reader simply re-loads until the tag matches: barrier + load (3 dependent L2 round trips)
// become one polled load.
__device__ __forceinline__ void st_word(unsigned long long* p, uint32_t payload, uint32_t epoch) {
  const unsigned long long w = ((unsigned long long)payload << 32) | epoch;
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ void ld_word2(const unsigned long long* p, unsigned long long& a,
                                         unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
// 8 consecutive per-element words (payload = bf16 bits) -> one 16-byte vector of 8 bf16
__device__ __forceinline__ uint4 poll8(const unsigned long long* w, uint32_t epoch, int* err) {
  unsigned long long a[8];
  unsigned spins = 0;
  bool ok;
  do {
#pragma unroll
    for (int i = 0; i < 4; ++i) ld_word2(w + 2 * i, a[2 * i], a[2 * i + 1]);
    ok = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) ok = ok && ((uint32_t)a[i] == epoch);
    if (!ok) {
      __nanosleep(200);  // back off: ~28k threads poll the same few KB of L2
      if (++spins > (1u << 20)) {
        *err = 4;
        break;
      }
    }
  } while (!ok);
  uint4 v;
  v.x = ((uint32_t)(a[0] >> 32) & 0xffffu) | ((uint32_t)(a[1] >> 32) << 16);
  v.y = ((uint32_t)(a[2] >> 32) & 0xffffu) | ((uint32_t)(a[3] >> 32) << 16);
  v.z = ((uint32_t)(a[4] >> 32) & 0xffffu) | ((uint32_t)(a[5] >> 32) << 16);
  v.w = ((uint32_t)(a[6] >> 32) & 0xffffu) | ((uint32_t)(a[7] >> 32) << 16);
  return v;
}
__device__ __forceinline__ uint32_t bf_bits(float x) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x));
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
// k_mega_tc: split-K partial sums are accumulated EXACTLY in 64-bit fixed point (2^-32 units)
// with red.global.add.u64: the sum is independent of the arrival order (deterministic) and the
// reader needs ONE load per row instead of one per split.  fp32 -> fixed is exact for
// |v| >= 2^-9 and within 2^-33 absolute below; |v| < 2^31.
constexpr float TC_FIX_SCALE = 4294967296.0f;
constexpr float TC_FIX_INV = 1.0f / 4294967296.0f;
__device__ __forceinline__ void fix_add(long long* acc, float v) {
  const long long q = __float2ll_rn(v * TC_FIX_SCALE);
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc), "l"(q) : "memory");
}
__device__ __forceinline__ float fix_get(const long long* acc) {
  return __ll2float_rn(__ldcg(acc)) * TC_FIX_INV;
}

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
  float invf[64];  // rotary inverse frequencies (k_mega_tc: no global round trip in the prologue)
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
// PARTS (k_mega_tc): q / k / v of this step arrive as fixed-point split-K sums of the qkv
// GEMV; the phase prologue finishes them (+ bias, round, rotary, q * scale) in shared
// memory, the unit that owns the new key scores it from there and one CTA per kv head
// appends it to the cache.
struct AttnParts {
  const long long* acc;  // PARTS: [qkv rows] fixed-point sums
  const bf16* bias;
  int pos;
  // FLOW (k_mega dataflow mode): q / k / v of this step as finished, rotated bf16 PAIRS (dims j and
  // j + hd/2 of a head) in self-validating words [head slot][hd/2]
  const unsigned long long* qkvw;
  uint32_t epoch;
};

enum { ATT_PLAIN = 0, ATT_PARTS = 1, ATT_FLOW = 2 };
template <int HD, int AMODE>
__device__ __forceinline__ void attn_phase(const MegaP& p, const bf16* kc, const bf16* vc,
                                           float* scratch, MegaShared* sh, int nkeys, int layer,
                                           const AttnParts& ap, long long* tdbg = nullptr) {
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
  constexpr bool PARTS = (AMODE != ATT_PLAIN);  // q / new k / new v come through shared memory
  const bool owner = PARTS && (u1 == nkeys) && (u1 > u0);  // holds the new key (index nkeys-1)
  const int u1g = u1 - (owner ? 1 : 0);                    // keys that are read from the cache
  float* qs = red + (long)8 * AG * HD;                     // PARTS: [AG][HD] q * scale
  float* kn = qs + (long)AG * HD;                          //        [HD] new key
  float* vn = kn + HD;                                     //        [HD] new value
  const int seg = lane & 7, ksub = lane >> 3;
  // ---- all global requests of the phase are issued before the first use: q, the first
  // 2 x 4 keys of this warp, and the V rows of its first VPRE keys (one round trip) ----
  constexpr int VPRE = 8;
  uint4 qraw[AG][NV];
  if (!PARTS) {
#pragma unroll
    for (int g = 0; g < AG; ++g)
#pragma unroll
      for (int v = 0; v < NV; ++v)
        qraw[g][v] = (g < G) ? ldcg16(p.qbuf + (long)(h0 + g) * HD + seg * SEG + v * 8)
                             : make_uint4(0, 0, 0, 0);
  }
  uint4 kvn[UNR][NV];
  {
    const int j0 = u0 + warp * 4;
#pragma unroll
    for (int q = 0; q < UNR; ++q) {
      const int j = j0 + 32 * q + ksub;
#pragma unroll
      for (int v = 0; v < NV; ++v)
        kvn[q][v] = (j < u1g) ? ldcg16(kb + (long)j * HD + seg * SEG + v * 8) : make_uint4(0, 0, 0, 0);
    }
  }
  uint2 vraw[VPRE];
#pragma unroll
  for (int q = 0; q < VPRE; ++q) {
    const int j = u0 + warp + 8 * q;
    vraw[q] = make_uint2(0, 0);
    if (j < u1g) {
      const bf16* vr = vb + (long)j * HD + lane * EPL;
      if (EPL == 4) vraw[q] = __ldcg(reinterpret_cast<const uint2*>(vr));
      else vraw[q].x = __ldcg(reinterpret_cast<const uint32_t*>(vr));
    }
  }
  float qr[AG][SEG];
  if (AMODE == ATT_FLOW) {
    // poll the finished q (x scale) / new k / new v pairs published by the qkv phase
    const int half = HD / 2;
    const int nslot = G + (owner ? 2 : 0);
    for (int i = threadIdx.x; i < nslot * half; i += 256) {
      const int slot = i / half, j = i % half;
      const int hs = (slot < G) ? (h0 + slot) : (slot == G ? d.n_heads + kvh : d.n_heads + d.n_kv + kvh);
      const unsigned long long* wp = ap.qkvw + (long)hs * half + j;
      unsigned long long w;
      unsigned spins = 0;
      do {
        asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(wp) : "memory");
        if ((uint32_t)w != ap.epoch) {
          __nanosleep(200);
          if (++spins > (1u << 20)) {
            sh->err = 4;
            break;
          }
        }
      } while ((uint32_t)w != ap.epoch);
      const uint32_t pr = (uint32_t)(w >> 32);
      float lo = __uint_as_float(pr << 16), hi = __uint_as_float(pr & 0xffff0000u);
      float* dst = (slot < G) ? qs + (long)slot * HD : (slot == G ? kn : vn);
      if (slot < G) {
        lo = rbf(lo * d.scale_bf);
        hi = rbf(hi * d.scale_bf);
      }
      dst[j] = lo;
      dst[j + half] = hi;
    }
    cbar();
#pragma unroll
    for (int g = 0; g < AG; ++g)
#pragma unroll
      for (int i = 0; i < SEG; ++i) qr[g][i] = (g < G) ? qs[(long)g * HD + seg * SEG + i] : 0.f;
  } else if (PARTS) {
    const int half = HD / 2;
    const int nslot = G + (owner ? 2 : 0);
    for (int i = threadIdx.x; i < nslot * HD; i += 256) {
      const int slot = i / HD, j = i % HD;
      const int row = (slot < G) ? (h0 + slot) * HD + j
                                 : ((slot == G ? d.n_heads + kvh : d.n_heads + d.n_kv + kvh) * HD + j);
      const float s = fix_get(ap.acc + row);
      (slot < G ? qs + (long)slot * HD : (slot == G ? kn : vn))[j] = rbf(s + bf2f(ap.bias[row]));
    }
    cbar();
    const int nrot = G + (owner ? 1 : 0);
    for (int i = threadIdx.x; i < nrot * half; i += 256) {
      const int slot = i / half, j = i % half;
      float* v = (slot < G) ? qs + (long)slot * HD : kn;
      const float y1 = v[j], y2 = v[j + half];
      const float ang = (float)ap.pos * sh->invf[j];
      const float c = rbf(cosf(ang)), sn = rbf(sinf(ang));
      float o1 = rbf(rbf(y1 * c) + rbf((-y2) * sn));
      float o2 = rbf(rbf(y2 * c) + rbf(y1 * sn));
      if (slot < G) {
        o1 = rbf(o1 * d.scale_bf);
        o2 = rbf(o2 * d.scale_bf);
      }
      v[j] = o1;
      v[j + half] = o2;
    }
    cbar();
    if (owner && part == 0) {  // append the new position to the cache (one CTA per kv head)
      bf16* kw = const_cast<bf16*>(kb) + (long)(nkeys - 1) * HD;
      bf16* vw = const_cast<bf16*>(vb) + (long)(nkeys - 1) * HD;
      for (int i = threadIdx.x; i < HD; i += 256) {
        kw[i] = f2bf(kn[i]);
        vw[i] = f2bf(vn[i]);
      }
    }
#pragma unroll
    for (int g = 0; g < AG; ++g)
#pragma unroll
      for (int i = 0; i < SEG; ++i) qr[g][i] = (g < G) ? qs[(long)g * HD + seg * SEG + i] : 0.f;
  } else {
#pragma unroll
    for (int g = 0; g < AG; ++g)
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        float f[8];
        unpack8(qraw[g][v], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) qr[g][v * 8 + i] = rbf(f[i] * d.scale_bf);
      }
  }
  ATT_STAMP();  // q loaded
  // ---- 1. scores of the own range (software-pipelined over trips of 2 x 4 keys) ----
  float lm[AG];
#pragma unroll
  for (int g = 0; g < AG; ++g) lm[g] = -INFINITY;
  for (int j0 = u0 + warp * 4; j0 < u1g; j0 += 32 * UNR) {
    uint4 kv[UNR][NV];
#pragma unroll
    for (int q = 0; q < UNR; ++q)
#pragma unroll
      for (int v = 0; v < NV; ++v) kv[q][v] = kvn[q][v];
    if (j0 + 32 * UNR < u1g) {
#pragma unroll
      for (int q = 0; q < UNR; ++q) {
        const int j = j0 + 32 * UNR + 32 * q + ksub;
#pragma unroll
        for (int v = 0; v < NV; ++v)
          kvn[q][v] = (j < u1g) ? ldcg16(kb + (long)j * HD + seg * SEG + v * 8)
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
      if (j < u1g && seg == 0) {
#pragma unroll
        for (int g = 0; g < AG; ++g) {
          const float r = rbf(s[g]);
          sc[(long)g * ucap + (j - u0)] = r;
          lm[g] = fmaxf(lm[g], r);
        }
      }
    }
  }
  if (PARTS && owner && warp == 0) {  // the new key: q . k from shared memory
#pragma unroll
    for (int g = 0; g < AG; ++g) {
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < EPL; ++e)
        s = fmaf((g < G) ? qs[(long)g * HD + lane * EPL + e] : 0.f, kn[lane * EPL + e], s);
      s = warp_sum(s);
      const float r = rbf(s);
      if (lane == 0) sc[(long)g * ucap + (nkeys - 1 - u0)] = r;
      lm[g] = fmaxf(lm[g], r);
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
    if (j < u1g) {
#pragma unroll
      for (int g = 0; g < AG; ++g) {
        const float pj = sc[(long)g * ucap + (j - u0)];
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[g][e] = fmaf(pj, vpre[q][e], acc[g][e]);
      }
    }
  }
  if (PARTS && owner && warp == 0) {  // the new value row comes from shared memory
#pragma unroll
    for (int g = 0; g < AG; ++g) {
      const float pj = sc[(long)g * ucap + (nkeys - 1 - u0)];
#pragma unroll
      for (int e = 0; e < EPL; ++e) acc[g][e] = fmaf(pj, vn[lane * EPL + e], acc[g][e]);
    }
  }
  for (int j0 = u0 + warp + 8 * VPRE; j0 < u1g; j0 += 32) {  // 4 keys per trip, loads first
    float vf[4][EPL];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + 8 * q;
#pragma unroll
      for (int e = 0; e < EPL; ++e) vf[q][e] = 0.f;
      if (j < u1g) {
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
      if (j < u1g) {
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

__device__ __forceinline__ uint32_t orderable_u(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
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
            ((unsigned long long)orderable_u(o[j]) << 32) | (0xFFFFFFFFu - (uint32_t)(c * 8 + j));
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
