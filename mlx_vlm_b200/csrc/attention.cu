// Prefill / vision attention with the reference's mlx-CPU rounding points
// (mx.fast.scaled_dot_product_attention fallback graph, see
// oracle/mlx_semantics.py::sdpa):   qs = bf16(q*bf16(scale)); s = bf16(qs.k^T);
// p = bf16(softmax_fp32(s)); o = bf16(p.v).
// Because p must be rounded AFTER normalisation with the final row max / sum, the
// kernel is two-pass over the keys (scores kept in shared memory as bf16, which
// is lossless since they are already rounded), not an online-softmax.
//
// v1: CUDA-core FMA, one CTA per (16 query rows, head); K/V tiles are re-read
// through L1 by the 8 warps of the CTA.  The tensor-core version is attention_tc.cu.
#include <stdlib.h>

#include "common.cuh"

namespace b200 {

constexpr int ATT_QT = 16;       // query rows per CTA
constexpr int ATT_THREADS = 256; // 8 warps, 2 rows each

struct AttnParams {
  const bf16 *q, *k, *v;
  bf16* out;
  long q_ts, q_hs, k_ts, k_hs, v_ts, v_hs, o_ts;
  int n_heads, n_kv, hd, Lq, S, causal;
  float scale_bf;  // scale rounded to bf16
};

__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(const AttnParams p) {
  extern __shared__ __align__(16) uint8_t smem_att[];
  float* qs = reinterpret_cast<float*>(smem_att);                      // [QT][hd]
  bf16* sc = reinterpret_cast<bf16*>(smem_att + ATT_QT * p.hd * 4);     // [QT][S]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y;
  const int kvh = h / (p.n_heads / p.n_kv);
  const int row0 = blockIdx.x * ATT_QT;
  const int hd = p.hd, S = p.S;
  const int nvec = hd >> 3;

  // stage the scaled, rounded query tile
  for (int i = threadIdx.x; i < ATT_QT * hd; i += ATT_THREADS) {
    const int r = i / hd, d = i % hd;
    const int qi = row0 + r;
    qs[i] = (qi < p.Lq) ? rbf(bf2f(p.q[(long)qi * p.q_ts + (long)h * p.q_hs + d]) * p.scale_bf) : 0.f;
  }
  __syncthreads();

  const bf16* kb = p.k + (long)kvh * p.k_hs;
  const bf16* vb = p.v + (long)kvh * p.v_hs;
  const int r_a = warp * 2, r_b = warp * 2 + 1;
  const int qa = row0 + r_a, qb = row0 + r_b;
  // number of visible keys per row (bottom-right aligned causal mask)
  const int vis_a = p.causal ? min(S, S - p.Lq + qa + 1) : S;
  const int vis_b = p.causal ? min(S, S - p.Lq + qb + 1) : S;
  const int vis_max = max(vis_a, vis_b);

  // ---- pass 1: scores (rounded to bf16), running max ----
  float m_a = -INFINITY, m_b = -INFINITY;
  const float* qra = qs + r_a * hd;
  const float* qrb = qs + r_b * hd;
  for (int j = lane; j < vis_max; j += 32) {
    const uint4* kr = reinterpret_cast<const uint4*>(kb + (long)j * p.k_ts);
    float da = 0.f, db = 0.f;
    for (int c = 0; c < nvec; ++c) {
      float kf[8];
      unpack8(__ldg(kr + c), kf);
      const float4 a0 = *reinterpret_cast<const float4*>(qra + c * 8);
      const float4 a1 = *reinterpret_cast<const float4*>(qra + c * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(qrb + c * 8);
      const float4 b1 = *reinterpret_cast<const float4*>(qrb + c * 8 + 4);
      da += a0.x * kf[0] + a0.y * kf[1] + a0.z * kf[2] + a0.w * kf[3] + a1.x * kf[4] +
            a1.y * kf[5] + a1.z * kf[6] + a1.w * kf[7];
      db += b0.x * kf[0] + b0.y * kf[1] + b0.z * kf[2] + b0.w * kf[3] + b1.x * kf[4] +
            b1.y * kf[5] + b1.z * kf[6] + b1.w * kf[7];
    }
    const float sa = (j < vis_a) ? rbf(da) : -INFINITY;
    const float sb = (j < vis_b) ? rbf(db) : -INFINITY;
    sc[(long)r_a * S + j] = f2bf(sa);
    sc[(long)r_b * S + j] = f2bf(sb);
    m_a = fmaxf(m_a, sa);
    m_b = fmaxf(m_b, sb);
  }
  m_a = warp_max(m_a);
  m_b = warp_max(m_b);
  __syncwarp();
  // ---- softmax in fp32, p rounded to bf16 (in place) ----
  float l_a = 0.f, l_b = 0.f;
  for (int j = lane; j < vis_max; j += 32) {
    const float sa = bf2f(sc[(long)r_a * S + j]), sb = bf2f(sc[(long)r_b * S + j]);
    l_a += (j < vis_a) ? expf(sa - m_a) : 0.f;
    l_b += (j < vis_b) ? expf(sb - m_b) : 0.f;
  }
  l_a = warp_sum(l_a);
  l_b = warp_sum(l_b);
  for (int j = lane; j < vis_max; j += 32) {
    const float sa = bf2f(sc[(long)r_a * S + j]), sb = bf2f(sc[(long)r_b * S + j]);
    const float pa = (j < vis_a) ? expf(sa - m_a) / l_a : 0.f;
    const float pb = (j < vis_b) ? expf(sb - m_b) / l_b : 0.f;
    sc[(long)r_a * S + j] = f2bf(pa);
    sc[(long)r_b * S + j] = f2bf(pb);
  }
  __syncwarp();
  // ---- pass 2: out = p . v ; lane owns dims {2*lane, 2*lane+1} + 64*i ----
  float oa[4] = {0.f, 0.f, 0.f, 0.f}, ob[4] = {0.f, 0.f, 0.f, 0.f};
  const int d0 = lane * 2, d1 = 64 + lane * 2;
  const bool has0 = d0 < hd, has1 = d1 < hd;
  for (int j = 0; j < vis_max; ++j) {
    const float pa = bf2f(sc[(long)r_a * S + j]), pb = bf2f(sc[(long)r_b * S + j]);
    const bf16* vr = vb + (long)j * p.v_ts;
    if (has0) {
      const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(vr + d0));
      const float v0 = __uint_as_float(w << 16), v1 = __uint_as_float(w & 0xffff0000u);
      oa[0] += pa * v0; oa[1] += pa * v1;
      ob[0] += pb * v0; ob[1] += pb * v1;
    }
    if (has1) {
      const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(vr + d1));
      const float v0 = __uint_as_float(w << 16), v1 = __uint_as_float(w & 0xffff0000u);
      oa[2] += pa * v0; oa[3] += pa * v1;
      ob[2] += pb * v0; ob[3] += pb * v1;
    }
  }
  if (qa < p.Lq) {
    bf16* o = p.out + (long)qa * p.o_ts + (long)h * hd;
    if (has0) *reinterpret_cast<uint32_t*>(o + d0) = pack2(oa[0], oa[1]);
    if (has1) *reinterpret_cast<uint32_t*>(o + d1) = pack2(oa[2], oa[3]);
  }
  if (qb < p.Lq) {
    bf16* o = p.out + (long)qb * p.o_ts + (long)h * hd;
    if (has0) *reinterpret_cast<uint32_t*>(o + d0) = pack2(ob[0], ob[1]);
    if (has1) *reinterpret_cast<uint32_t*>(o + d1) = pack2(ob[2], ob[3]);
  }
}

// attention_tc.cu: the tensor-core kernel (default whenever the layout allows 16-byte tiles)
bool attention_tc_supported(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                            const void* v, long v_ts, long v_hs, const void* out, long o_ts, int hd);
int attention_tc(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                 const void* v, long v_ts, long v_hs, void* out, long o_ts, int n_heads, int n_kv,
                 int hd, int Lq, int S, int causal, float scale, cudaStream_t st);

static int g_attn_impl = -1;  // -1: read B200_ATTN_V1 once; 0: tensor cores; 1: CUDA-core v1
void attention_set_impl(int v1) { g_attn_impl = v1 ? 1 : 0; }

int attention(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
              const void* v, long v_ts, long v_hs, void* out, long o_ts, int n_heads, int n_kv,
              int hd, int Lq, int S, int causal, float scale, cudaStream_t st) {
  B200_REQUIRE(Lq > 0 && S > 0 && n_heads > 0 && n_kv > 0 && n_heads % n_kv == 0,
               "attention: bad shape Lq=%d S=%d heads=%d kv=%d", Lq, S, n_heads, n_kv);
  B200_REQUIRE(!causal || S >= Lq, "attention: causal needs S >= Lq");
  if (g_attn_impl < 0) {
    const char* e = getenv("B200_ATTN_V1");
    g_attn_impl = (e && e[0] == '1') ? 1 : 0;
  }
  if (g_attn_impl == 0 &&
      attention_tc_supported(q, q_ts, q_hs, k, k_ts, k_hs, v, v_ts, v_hs, out, o_ts, hd))
    return attention_tc(q, q_ts, q_hs, k, k_ts, k_hs, v, v_ts, v_hs, out, o_ts, n_heads, n_kv, hd,
                        Lq, S, causal, scale, st);
  B200_REQUIRE(hd % 8 == 0 && hd <= 128, "attention: head_dim %d unsupported (need %%8, <=128)", hd);
  B200_REQUIRE((k_ts % 8) == 0 && (k_hs % 8) == 0 && (v_ts % 2) == 0 && (v_hs % 2) == 0 &&
                   (o_ts % 2) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 3) == 0,
               "attention: strides/pointers must keep 16-byte key rows");
  B200_REQUIRE(!causal || S >= Lq, "attention: causal needs S >= Lq");
  const size_t smem = (size_t)ATT_QT * hd * 4 + (size_t)ATT_QT * S * 2;
  B200_REQUIRE(smem <= 220 * 1024, "attention: S=%d too long for the two-pass kernel", S);
  static size_t max_set = 48 * 1024;
  if (smem > max_set) {
    B200_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(220 * 1024)));
    max_set = 220 * 1024;
  }
  AttnParams p;
  p.q = (const bf16*)q; p.k = (const bf16*)k; p.v = (const bf16*)v; p.out = (bf16*)out;
  p.q_ts = q_ts; p.q_hs = q_hs; p.k_ts = k_ts; p.k_hs = k_hs; p.v_ts = v_ts; p.v_hs = v_hs;
  p.o_ts = o_ts; p.n_heads = n_heads; p.n_kv = n_kv; p.hd = hd; p.Lq = Lq; p.S = S;
  p.causal = causal;
  p.scale_bf = __bfloat162float(__float2bfloat16_rn(scale));
  dim3 grid(cdiv(Lq, ATT_QT), n_heads);
  attention_kernel<<<grid, ATT_THREADS, smem, st>>>(p);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200

extern "C" int b200_attention(const void* q, long q_ts, long q_hs, const void* k, long k_ts,
                              long k_hs, const void* v, long v_ts, long v_hs, void* out,
                              long o_ts, int n_heads, int n_kv, int hd, int Lq, int S, int causal,
                              float scale, void* stream) {
  return b200::attention(q, q_ts, q_hs, k, k_ts, k_hs, v, v_ts, v_hs, out, o_ts, n_heads, n_kv,
                         hd, Lq, S, causal, scale, (cudaStream_t)stream);
}
