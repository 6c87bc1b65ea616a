// Prefill / vision attention: TMA-fed, warp-specialised, wgmma (Hopper) with the scores and the
// output in registers.  The loads are pipelined (a producer warpgroup fills double-buffered K and
// V^T slots ahead of the consumers); the MMAs of a consumer are not: Q.K^T, softmax and P.V of a
// tile run one after another.  Same arithmetic and rounding points as attention_tc.cu (the
// reference's mlx-CPU SDPA: oracle/mlx_semantics.py::sdpa; models/base.py:305-373, qwen2_vl/vision.py:154):
//     qs = bf16(q * bf16(scale))       -- done by the rotary kernels that already touch q
//     s  = bf16(qs . k^T);  p = bf16(softmax_fp32(s));  o = bf16(p . v)
// p is rounded AFTER normalisation with the final row max / sum, so the kernel is two-pass over
// the keys and the second pass recomputes the score tile on the tensor cores.
// Per CTA = 128 query rows of one head:
//   warpgroup 0     TMA producer: Q once, K tiles for both passes, V^T tiles for pass 2 (3-D tensor
//                   maps over the packed qkv buffer / the KV cache, 128B swizzle, zero-filled tails)
//   warpgroups 1,2  64 query rows each: S = Qs . K^T (m64n128), softmax in registers (a row is held
//                   by the 4 threads of a quad), O += P . V with P as the register A operand
// V is consumed as V^T ([head][dim][key], keys contiguous): a K-major B operand that TMA can
// load directly; the rotary kernels emit it (rowops.cu: *_qkv_post).
#include "common.cuh"
#include "decode.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int FA_TQ = 128, FA_TK = 128;
constexpr int FA_BLK = 16 * 1024;       // one 128-row x 64-column bf16 operand block
constexpr int FA_THREADS = 384;         // producer warpgroup, 2 consumer warpgroups

struct FaParams {
  bf16* out;
  long o_ts;
  int n_heads, n_kv, hd, hdp, Lq, S, causal;
  int q0, k0;  // token offsets of this segment inside the tensors the maps describe
  const int4* segs;  // optional [gridDim.z]: (q0, Lq, k0, S) of segment blockIdx.z — several independent sequences of one
                     // concatenated batch in ONE launch (the tail wave of a 160-CTA launch per sequence idles half the SMs)
};

struct FaBars {
  uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2];
};

// 2^x on the SFU (one MUFU instruction, rel. error 2^-22: far below the bf16 rounding of p that follows)
__device__ __forceinline__ float f_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(FA_THREADS, 1)
attention_fa_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const FaParams p_in) {
  FaParams p = p_in;
  if (p_in.segs) {   // static table (written before the producing kernels ran): safe to read ahead of griddepcontrol.wait
    const int4 sg = __ldg(p_in.segs + blockIdx.z);
    p.q0 = sg.x; p.Lq = sg.y; p.k0 = sg.z; p.S = sg.w;
    if ((int)blockIdx.x * FA_TQ >= p.Lq) return;   // the grid is sized for the longest segment
  }
  extern __shared__ uint8_t fa_smem_raw[];
  __shared__ FaBars bars;
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fa_smem_raw) + 1023) &
                                           ~static_cast<uintptr_t>(1023));
  uint8_t* Qs = sm;                          // [128 q][128 d]            2 k-blocks
  uint8_t* Ks = sm + 2 * FA_BLK;             // 2 slots x [128 keys][128 d]
  uint8_t* Vs = sm + 6 * FA_BLK;             // 2 slots x 2 key-blocks x [hdp d][64 keys]
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int h = blockIdx.y, kvh = h / (p.n_heads / p.n_kv);
  const int row0 = blockIdx.x * FA_TQ;
  const int S = p.S;
  const int q_last = min(row0 + FA_TQ, p.Lq) - 1;
  const int vis_tile = p.causal ? min(S, S - p.Lq + q_last + 1) : S;
  const int n_tiles = (vis_tile + FA_TK - 1) / FA_TK;
  const int kbq = (p.hdp + 63) >> 6;         // 64-column blocks of the head dimension
  const int vblk = p.hdp * 128;              // bytes of one 64-key block of a V^T tile

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmQ)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmK)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmV)) : "memory");
    mbar_init(&bars.q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bars.k_full[i], 1);
      mbar_init(&bars.k_empty[i], 8);   // one arrival per consumer warp
      mbar_init(&bars.v_full[i], 1);
      mbar_init(&bars.v_empty[i], 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    if (threadIdx.x == 0) {  // ===== TMA producer =====
      mbar_expect_tx(&bars.q_full, (uint32_t)kbq * FA_BLK);
      for (int c = 0; c < kbq; ++c) tma_3d(Qs + c * FA_BLK, &tmQ, &bars.q_full, c * 64, h, p.q0 + row0);
      for (int i = 0; i < 2 * n_tiles; ++i) {
        const int j = i % n_tiles, s = i & 1;
        mbar_wait(&bars.k_empty[s], ((i >> 1) & 1) ^ 1);
        mbar_expect_tx(&bars.k_full[s], (uint32_t)kbq * FA_BLK);
        for (int c = 0; c < kbq; ++c)
          tma_3d(Ks + s * 2 * FA_BLK + c * FA_BLK, &tmK, &bars.k_full[s], c * 64, kvh, p.k0 + j * FA_TK);
        if (i >= n_tiles) {
          const int sv = j & 1;
          mbar_wait(&bars.v_empty[sv], ((j >> 1) & 1) ^ 1);
          mbar_expect_tx(&bars.v_full[sv], 2u * (uint32_t)vblk);
          for (int c = 0; c < 2; ++c)
            tma_3d(Vs + sv * 2 * FA_BLK + c * vblk, &tmV, &bars.v_full[sv], p.k0 + j * FA_TK + c * 64, 0, kvh);
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup c = wg - 1 owns query rows [64 c, 64 c + 64) of the tile; its thread holds
  // rows r0 and r0 + 8 of the score / output accumulators (wgmma.cuh) =====
  const int c = wg - 1;
  const int r0 = c * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  int vis[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int qi = row0 + r0 + 8 * hr;
    vis[hr] = (qi < p.Lq) ? (p.causal ? min(S, S - p.Lq + qi + 1) : S) : S;
  }
  const int col0 = 2 * (lane & 3);
  constexpr float LOG2E = 1.4426950408889634f;
  const uint32_t q_a = smem_u32(Qs) + c * 64 * 128;
  const int ksteps = p.hdp >> 4;
  float sacc[64];
  // S = Qs . K^T of the tile in ring slot s (M64 x N128 per warpgroup), then the slot is released
  auto scores = [&](int s, uint32_t par) {
    mbar_wait(&bars.k_full[s], par);
    const uint32_t k_a = smem_u32(Ks + s * 2 * FA_BLK);
    wg_fence_acc(sacc);
    wg_arrive();
    for (int ks = 0; ks < ksteps; ++ks) {
      const uint32_t off = (uint32_t)((ks >> 2) * FA_BLK + (ks & 3) * 32);
      wgmma_n128_ss(sacc, wg_desc(q_a + off), wg_desc(k_a + off), ks > 0 ? 1u : 0u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars.k_empty[s]);
  };
  mbar_wait(&bars.q_full, 0);
  // The softmax is the instruction-bound part: the inner loops are kept to a few instructions per element
  // (bf16 rounding, one FMA into the exponent, ex2 on the SFU, multiplication by 1/l).
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int i = 0; i < n_tiles; ++i) {  // ---- pass 1: row max and sum of exp over bf16 scores ----
    scores(i & 1, (i >> 1) & 1);
    const int jbase = i * FA_TK + col0;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float cm = -INFINITY;
#pragma unroll
      for (int e = 0; e < 64; e += 4) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int idx = e + 2 * hr + u;
          const float v = (jbase + 8 * (e >> 2) + u < vis[hr]) ? rbf(sacc[idx]) : -INFINITY;
          sacc[idx] = v;
          cm = fmaxf(cm, v);
        }
      }
      cm = quad_max(cm);
      if (cm > -INFINITY) {
        const float mn = fmaxf(m[hr], cm);
        const float nb = -mn * LOG2E;
        float add = 0.f;
#pragma unroll
        for (int e = 0; e < 64; e += 4) add += f_ex2(fmaf(sacc[e + 2 * hr], LOG2E, nb)) + f_ex2(fmaf(sacc[e + 2 * hr + 1], LOG2E, nb));
        l[hr] = l[hr] * f_ex2((m[hr] - mn) * LOG2E) + add;
        m[hr] = mn;
      }
    }
  }
  float inv_l[2], nbm[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    inv_l[hr] = 1.0f / quad_sum(l[hr]);
    nbm[hr] = -m[hr] * LOG2E;
  }
  float oacc[8][8];
#pragma unroll
  for (int ch = 0; ch < 8; ++ch)
#pragma unroll
    for (int e = 0; e < 8; ++e) oacc[ch][e] = 0.f;
  const int n_och = p.hdp >> 4;
  for (int j = 0; j < n_tiles; ++j) {  // ---- pass 2: p = bf16(exp(s - m) / l), O += P . V ----
    const int i = n_tiles + j;
    scores(i & 1, (i >> 1) & 1);
    const int jbase = j * FA_TK + col0;
    uint32_t pa[8][4];  // P as the A operand of 8 k-steps of 16 keys
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // q: (row half, column group) of the A fragment
        const int hr = q & 1, g = 2 * ks + (q >> 1);
        float pv[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float pe = f_ex2(fmaf(rbf(sacc[4 * g + 2 * hr + u]), LOG2E, nbm[hr])) * inv_l[hr];
          pv[u] = (jbase + 8 * g + u < vis[hr]) ? pe : 0.f;
        }
        pa[ks][q] = pack2(pv[0], pv[1]);
      }
    }
    const int sv = j & 1;
    mbar_wait(&bars.v_full[sv], (j >> 1) & 1);
    const uint32_t v_a = smem_u32(Vs + sv * 2 * FA_BLK);
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) wg_fence_acc(oacc[ch]);
    wg_arrive();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t koff = (uint32_t)((ks >> 2) * vblk + (ks & 3) * 32);
#pragma unroll
      for (int ch = 0; ch < 8; ++ch)
        if (ch < n_och) wgmma_n16_rs(oacc[ch], pa[ks], wg_desc(v_a + koff + ch * 2048), 1u);
    }
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) wg_fence_acc(oacc[ch]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars.v_empty[sv]);
  }
  // ---- epilogue: O -> bf16 -> global, two columns per store ----
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int qi = row0 + r0 + 8 * hr;
    if (qi >= p.Lq) continue;
    bf16* orow = p.out + (long)(p.q0 + qi) * p.o_ts + (long)h * p.hd;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const int col = ch * 16 + g * 8 + col0;
        if (col < p.hd)
          *reinterpret_cast<uint32_t*>(orow + col) = pack2(oacc[ch][4 * g + 2 * hr], oacc[ch][4 * g + 2 * hr + 1]);
      }
    }
  }
}

// ---- host: 3-D tensor maps ----------------------------------------------------------------
// bf16 tensor: dims (d0 contiguous, d1 with stride s1 elements, d2 with stride s2), box (b0, b1, b2)
int fa_tmap3(const void* ptr, int d0, int d1, long s1, int d2, long s2, int b0, int b1, int b2, CUtensorMap* out) {
  const cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
  const cuuint64_t strides[2] = {(cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
  const cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, (cuuint32_t)b2};
  return bf16_tmap(3, ptr, dims, strides, box, out);
}

}  // namespace

bool attention_fa_supported(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                            const void* vt, long vt_hs, long vt_ds, const void* out, long o_ts, int hd) {
  auto al = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  return hd % 8 == 0 && hd >= 16 && hd <= 128 && al(q) && al(k) && al(vt) && al(out) && (q_ts % 8) == 0 &&
         (q_hs % 8) == 0 && (k_ts % 8) == 0 && (k_hs % 8) == 0 && (vt_hs % 8) == 0 && (vt_ds % 8) == 0 &&
         (o_ts % 8) == 0;
}

// q: PRE-SCALED queries (bf16(q * bf16(scale))), element (t, h, d) at q + t*q_ts + h*q_hs + d
// k: keys, element (s, kvh, d) at k + s*k_ts + kvh*k_hs + d
// vt: values transposed, element (kvh, d, s) at vt + kvh*vt_hs + d*vt_ds + s   (keys contiguous)
// The tensors hold q_tot query tokens / k_tot keys; this call attends queries [q0, q0+Lq) to keys
// [k0, k0+S) (one vision segment, or the whole prompt); out row t is written at out + t*o_ts.
int attention_fa(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs, const void* vt,
                 long vt_hs, long vt_ds, void* out, long o_ts, int n_heads, int n_kv, int hd, int Lq, int S,
                 int causal, cudaStream_t st, int q0, int q_tot, int k0, int k_tot, const void* segs, int n_seg) {
  if (q_tot <= 0) q_tot = q0 + Lq;
  if (k_tot <= 0) k_tot = k0 + S;
  B200_REQUIRE(!segs || n_seg > 0, "attention_fa: segment table without segments");
  B200_REQUIRE(attention_fa_supported(q, q_ts, q_hs, k, k_ts, k_hs, vt, vt_hs, vt_ds, out, o_ts, hd),
               "attention_fa: unsupported layout (hd=%d)", hd);
  B200_REQUIRE(Lq > 0 && S > 0 && n_heads % n_kv == 0, "attention_fa: bad shape");
  const int hdp = (hd + 15) & ~15;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = fa_tmap3(q, hd, n_heads, q_hs, q_tot, q_ts, 64, 1, FA_TQ, &tq))) return rc;
  if ((rc = fa_tmap3(k, hd, n_kv, k_hs, k_tot, k_ts, 64, 1, FA_TK, &tk))) return rc;
  if ((rc = fa_tmap3(vt, k_tot, hd, vt_ds, n_kv, vt_hs, 64, hdp, 1, &tv))) return rc;
  const size_t smem = 10 * FA_BLK + 1024;
  if ((rc = kernel_opt_in((const void*)attention_fa_kernel, (int)smem, false))) return rc;
  FaParams p;
  p.out = (bf16*)out; p.o_ts = o_ts; p.n_heads = n_heads; p.n_kv = n_kv; p.hd = hd; p.hdp = hdp;
  p.Lq = Lq; p.S = S; p.causal = causal; p.q0 = q0; p.k0 = k0;
  p.segs = (const int4*)segs;
  B200_CUDA(launch(attention_fa_kernel, dim3(cdiv(Lq, FA_TQ), n_heads, segs ? n_seg : 1), dim3(FA_THREADS), smem, st,
                   PDL_LAUNCH, tq, tk, tv, p));
  return B200_OK;
}

}  // namespace b200

extern "C" int b200_attention_fa(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                                 const void* vt, long vt_hs, long vt_ds, void* out, long o_ts, int n_heads,
                                 int n_kv, int hd, int Lq, int S, int causal, void* stream) {
  return b200::attention_fa(q, q_ts, q_hs, k, k_ts, k_hs, vt, vt_hs, vt_ds, out, o_ts, n_heads, n_kv, hd, Lq, S,
                            causal, (cudaStream_t)stream, 0, Lq, 0, S, nullptr, 0);
}

extern "C" int b200_attention_fa_seg(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                                     const void* vt, long vt_hs, long vt_ds, void* out, long o_ts, int n_heads,
                                     int n_kv, int hd, int Lq, int S, int causal, int q0, int q_tot, int k0, int k_tot,
                                     const void* segs, int n_seg, void* stream) {
  return b200::attention_fa(q, q_ts, q_hs, k, k_ts, k_hs, vt, vt_hs, vt_ds, out, o_ts, n_heads, n_kv, hd, Lq, S,
                            causal, (cudaStream_t)stream, q0, q_tot, k0, k_tot, segs, n_seg);
}
