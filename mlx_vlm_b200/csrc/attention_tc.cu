// Prefill / vision attention on the Hopper tensor cores (wgmma), with the reference's mlx-CPU
// rounding points (oracle/mlx_semantics.py::sdpa; models/base.py:305-373,
// qwen2_vl/vision.py:154):   qs = bf16(q*bf16(scale)); s = bf16(qs.k^T);
// p = bf16(softmax_fp32(s)); o = bf16(p.v).
//
// p must be rounded AFTER normalisation with the final row max / sum, so the kernel is
// two-pass over the keys, and the second pass RECOMPUTES the score tile on the tensor
// cores instead of keeping [rows x S] scores around (v1, attention.cu, kept them in shared
// memory and ran on CUDA cores).
//
// One CTA = 128 query rows of one head, two warpgroups of 64 rows each:
//   S[64 x 128 keys] = Qs . K^T      wgmma m64n128k16, A = Qs, B = K tile, both K-major in
//                                    128B-swizzled shared memory, fp32 in registers
//   O[64 x hd]      += P . V         A = P (bf16 in registers), B = V^T tile
//                                    (transposed on the way into shared memory)
// Tiles are staged by the threads themselves (16-byte loads, swizzled stores): the head
// dimension (80 for the ViT) is zero-padded to 128 on the fly, q is scaled while staged.
#include "common.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int TQ = 128;          // query rows per CTA
constexpr int TK = 128;          // keys per tile
constexpr int KBLK = 16 * 1024;  // one 128-row x 64-column bf16 operand block

struct AttnTcParams {
  const bf16 *q, *k, *v;
  bf16* out;
  long q_ts, q_hs, k_ts, k_hs, v_ts, v_hs, o_ts;
  int n_heads, n_kv, hd, Lq, S, causal;
  float scale_bf;
};

// byte offset of element (row r, column c) of a [128 x 128] bf16 operand stored as two
// 64-column blocks, each 128 rows x 128 B with the 128-byte swizzle
__device__ __forceinline__ uint32_t sw_off(int r, int c) {
  const int blk = c >> 6, cc = c & 63;
  return (uint32_t)(blk * KBLK + r * 128 + ((((cc >> 3) ^ (r & 7))) << 4) + ((cc & 7) << 1));
}

constexpr int ATC_THREADS = 256;  // two warpgroups, 64 query rows each

// stage `rows` x hd (zero-padded to 128 x 128) of a row-major source into an operand tile.
// All loads of a thread are issued before its first store (one memory latency per tile; the
// first version interleaved load/store and paid it 16 times).
template <bool SCALE>
__device__ __forceinline__ void stage_rows(uint8_t* dst, const bf16* src, long row_stride, int row0,
                                           int row_end, int hd, float scale_bf) {
  constexpr int NU = 128 * 16 / ATC_THREADS;
  uint4 v[NU];
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int idx = threadIdx.x + ATC_THREADS * u;
    const int r = idx >> 4, ch = idx & 15;
    const int gr = row0 + r;
    v[u] = (gr < row_end && ch * 8 < hd)
               ? __ldg(reinterpret_cast<const uint4*>(src + (long)gr * row_stride + ch * 8))
               : make_uint4(0, 0, 0, 0);
  }
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int idx = threadIdx.x + ATC_THREADS * u;
    const int r = idx >> 4, ch = idx & 15;
    if (SCALE) {
      float f[8];
      unpack8(v[u], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = rbf(f[i] * scale_bf);
      v[u].x = pack2(f[0], f[1]); v[u].y = pack2(f[2], f[3]);
      v[u].z = pack2(f[4], f[5]); v[u].w = pack2(f[6], f[7]);
    }
    *reinterpret_cast<uint4*>(dst + sw_off(r, ch * 8)) = v[u];
  }
}

// stage V[key0 .. key0+128)[0..hd) TRANSPOSED: tile rows = head dims, columns = keys.
// A thread takes two adjacent keys and 8 dims: 8 four-byte stores per step.
__device__ __forceinline__ void stage_vt(uint8_t* dst, const bf16* v, long row_stride, int key0,
                                         int key_end, int hd) {
  constexpr int NU = 64 * 16 / ATC_THREADS;
  uint4 va[NU], vb8[NU];
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int idx = threadIdx.x + ATC_THREADS * u;
    const int kp = idx & 63, ch = idx >> 6;  // key pair, dim chunk
    const int ka = key0 + 2 * kp, kb = ka + 1;
    const bool dim_ok = ch * 8 < hd;         // dims beyond hd are never read (N = hd)
    va[u] = (dim_ok && ka < key_end) ? __ldg(reinterpret_cast<const uint4*>(v + (long)ka * row_stride + ch * 8))
                                     : make_uint4(0, 0, 0, 0);
    vb8[u] = (dim_ok && kb < key_end) ? __ldg(reinterpret_cast<const uint4*>(v + (long)kb * row_stride + ch * 8))
                                      : make_uint4(0, 0, 0, 0);
  }
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int idx = threadIdx.x + ATC_THREADS * u;
    const int kp = idx & 63, ch = idx >> 6;
    if (ch * 8 >= hd) continue;
    const uint4 a = va[u], b = vb8[u];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t lo = (aw[i] & 0xffffu) | (bw[i] << 16);          // dim 2i   of keys (ka, kb)
      const uint32_t hi = (aw[i] >> 16) | (bw[i] & 0xffff0000u);      // dim 2i+1
      *reinterpret_cast<uint32_t*>(dst + sw_off(ch * 8 + 2 * i, 2 * kp)) = lo;
      *reinterpret_cast<uint32_t*>(dst + sw_off(ch * 8 + 2 * i + 1, 2 * kp)) = hi;
    }
  }
}

__global__ void __launch_bounds__(ATC_THREADS, 1) attention_tc_kernel(const AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                           ~static_cast<uintptr_t>(1023));
  uint8_t* Qs = sm;                 // [128 q][128 d]
  uint8_t* Ks = sm + 2 * KBLK;      // [128 keys][128 d]
  uint8_t* Vt = sm + 4 * KBLK;      // [128 d][128 keys]
  const int t = threadIdx.x, lane = t & 31;
  const int wg = t >> 7;            // warpgroup wg owns query rows [64 wg, 64 wg + 64)
  const int h = blockIdx.y, kvh = h / (p.n_heads / p.n_kv);
  const int row0 = blockIdx.x * TQ;
  const int hd = p.hd, S = p.S;

  stage_rows<true>(Qs, p.q + (long)h * p.q_hs, p.q_ts, row0, p.Lq, hd, p.scale_bf);

  const bf16* kb = p.k + (long)kvh * p.k_hs;
  const bf16* vb = p.v + (long)kvh * p.v_hs;
  // this thread holds accumulator rows r0 and r0 + 8 (wgmma.cuh); visible keys per row (bottom-right
  // aligned causal mask); rows past Lq compute on finite garbage and are never stored
  const int r0 = wg * 64 + ((t >> 5) & 3) * 16 + (lane >> 2);
  const int col0 = 2 * (lane & 3);
  int vis[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int qi = row0 + r0 + 8 * hr;
    vis[hr] = (qi < p.Lq) ? (p.causal ? min(S, S - p.Lq + qi + 1) : S) : S;
  }
  const int q_last = min(row0 + TQ, p.Lq) - 1;
  const int vis_tile = p.causal ? min(S, S - p.Lq + q_last + 1) : S;
  const int n_tiles = (vis_tile + TK - 1) / TK;

  const uint32_t q_a = smem_u32(Qs) + wg * 64 * 128, k_a = smem_u32(Ks), v_a = smem_u32(Vt);
  const int ksteps = hd >> 4;  // 16 dims per MMA
  float sacc[64];
  auto scores = [&]() {
    wg_fence_acc(sacc);
    wg_arrive();
    for (int ks = 0; ks < ksteps; ++ks) {
      const uint32_t off = (uint32_t)((ks >> 2) * KBLK + (ks & 3) * 32);
      wgmma_n128_ss(sacc, wg_desc(q_a + off), wg_desc(k_a + off), ks > 0 ? 1u : 0u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(sacc);
  };
  constexpr float LOG2E = 1.4426950408889634f;

  // ---------------- pass 1: row max and sum of exp over the bf16-rounded scores ----------------
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int jt = 0; jt < n_tiles; ++jt) {
    if (jt > 0) __syncthreads();  // every warpgroup's MMAs have read the previous K tile
    stage_rows<false>(Ks, kb, p.k_ts, jt * TK, S, hd, 0.f);
    fence_proxy_async();
    __syncthreads();
    scores();
    const int jbase = jt * TK + col0;
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
        float add = 0.f;
#pragma unroll
        for (int e = 0; e < 64; e += 4)
          add += exp2f((sacc[e + 2 * hr] - mn) * LOG2E) + exp2f((sacc[e + 2 * hr + 1] - mn) * LOG2E);
        l[hr] = l[hr] * exp2f((m[hr] - mn) * LOG2E) + add;
        m[hr] = mn;
      }
    }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) l[hr] = quad_sum(l[hr]);

  // ---------------- pass 2: p = bf16(exp(s - m) / l), O += P . V ----------------
  float oacc[8][8];
#pragma unroll
  for (int ch = 0; ch < 8; ++ch)
#pragma unroll
    for (int e = 0; e < 8; ++e) oacc[ch][e] = 0.f;
  const int n_och = hd >> 4;
  for (int jt = 0; jt < n_tiles; ++jt) {
    __syncthreads();  // the previous tile's MMAs have read Ks / Vt
    stage_rows<false>(Ks, kb, p.k_ts, jt * TK, S, hd, 0.f);
    stage_vt(Vt, vb, p.v_ts, jt * TK, S, hd);
    fence_proxy_async();
    __syncthreads();
    scores();
    const int jbase = jt * TK + col0;
    uint32_t pa[8][4];  // P as the A operand of 8 k-steps of 16 keys
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int hr = q & 1, g = 2 * ks + (q >> 1);
        float pv[2];
#pragma unroll
        for (int u = 0; u < 2; ++u)
          pv[u] = (jbase + 8 * g + u < vis[hr]) ? exp2f((rbf(sacc[4 * g + 2 * hr + u]) - m[hr]) * LOG2E) / l[hr] : 0.f;
        pa[ks][q] = pack2(pv[0], pv[1]);
      }
    }
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) wg_fence_acc(oacc[ch]);
    wg_arrive();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t koff = (uint32_t)((ks >> 2) * KBLK + (ks & 3) * 32);
#pragma unroll
      for (int ch = 0; ch < 8; ++ch)
        if (ch < n_och) wgmma_n16_rs(oacc[ch], pa[ks], wg_desc(v_a + koff + ch * 2048), 1u);
    }
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) wg_fence_acc(oacc[ch]);
  }
  // ---------------- epilogue: O -> bf16 -> global, two columns per store ----------------
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int qi = row0 + r0 + 8 * hr;
    if (qi >= p.Lq) continue;
    bf16* orow = p.out + (long)qi * p.o_ts + (long)h * hd;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const int col = ch * 16 + g * 8 + col0;
        if (col < hd)
          *reinterpret_cast<uint32_t*>(orow + col) = pack2(oacc[ch][4 * g + 2 * hr], oacc[ch][4 * g + 2 * hr + 1]);
      }
    }
  }
}

}  // namespace

bool attention_tc_supported(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                            const void* v, long v_ts, long v_hs, const void* out, long o_ts, int hd) {
  auto al = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  return hd % 16 == 0 && hd >= 16 && hd <= 128 && al(q) && al(k) && al(v) && al(out) &&
         (q_ts % 8) == 0 && (q_hs % 8) == 0 && (k_ts % 8) == 0 && (k_hs % 8) == 0 &&
         (v_ts % 8) == 0 && (v_hs % 8) == 0 && (o_ts % 8) == 0;
}

int attention_tc(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                 const void* v, long v_ts, long v_hs, void* out, long o_ts, int n_heads, int n_kv,
                 int hd, int Lq, int S, int causal, float scale, cudaStream_t st) {
  const size_t smem = 6 * KBLK + 1024;
  if (int rc = kernel_opt_in((const void*)attention_tc_kernel, (int)smem, false)) return rc;
  AttnTcParams p;
  p.q = (const bf16*)q; p.k = (const bf16*)k; p.v = (const bf16*)v; p.out = (bf16*)out;
  p.q_ts = q_ts; p.q_hs = q_hs; p.k_ts = k_ts; p.k_hs = k_hs; p.v_ts = v_ts; p.v_hs = v_hs;
  p.o_ts = o_ts; p.n_heads = n_heads; p.n_kv = n_kv; p.hd = hd; p.Lq = Lq; p.S = S;
  p.causal = causal;
  p.scale_bf = __bfloat162float(__float2bfloat16_rn(scale));
  dim3 grid(cdiv(Lq, TQ), n_heads);
  attention_tc_kernel<<<grid, ATC_THREADS, smem, st>>>(p);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200
