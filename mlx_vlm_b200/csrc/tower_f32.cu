// fp32-accurate vision towers (LLaVA-1.5 CLIP-L/14, Idefics2 SigLIP + perceiver).
//
// The reference never casts `pixel_values` for these models (utils.py:2091 builds a float32 array,
// llava.py:61-63 / idefics2.py:212-251 feed it straight in), so mlx type promotion makes every op
// of the tower an fp32 computation with bf16-VALUED weights; the features are rounded to bf16
// only at the merge (llava.py:101-104).  A bf16 tower is 1.4e-2 away from that (87 % of the
// feature elements differ, tools/tower_precision_study.py), so it is not a drop-in.
//
// How the tensor cores still do the work: an fp32 activation x is carried as TWO bf16 halves
// x_hi = bf16(x), x_lo = bf16(x - x_hi) ("split operand", 16 mantissa bits); because the weights are
// exactly bf16, W.x = W.x_hi + W.x_lo needs two kind::f16 MMAs with fp32 accumulation — the GEMM
// (gemm_wt.cu) simply sees a K twice as long whose weight k-blocks repeat.  Everything between the
// GEMMs is fp32 here: LayerNorm, residual stream, GELU, softmax, attention.
#include "common.cuh"
#include "decode.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ void split_store4(bf16* dst, int n_pad, float a, float b, float c, float d) {
  const float h0 = rbf(a), h1 = rbf(b), h2 = rbf(c), h3 = rbf(d);
  *reinterpret_cast<uint2*>(dst) = make_uint2(pack2(h0, h1), pack2(h2, h3));
  *reinterpret_cast<uint2*>(dst + n_pad) = make_uint2(pack2(a - h0, b - h1), pack2(c - h2, d - h3));
}

__device__ __forceinline__ void split_store2(bf16* dst, int n_pad, float a, float b) {
  const float h0 = rbf(a), h1 = rbf(b);
  *reinterpret_cast<uint32_t*>(dst) = pack2(h0, h1);
  *reinterpret_cast<uint32_t*>(dst + n_pad) = pack2(a - h0, b - h1);
}

// LayerNorm in fp32 (nn.LayerNorm on an fp32 array: fp32 statistics, fp32 affine); output as fp32
// and / or as the split operand of the next GEMM.  One CTA per row, N % 4 == 0, N <= 8192.
__global__ void __launch_bounds__(256) f32_layer_norm_kernel(const float* __restrict__ x, long ldx,
                                                             const bf16* __restrict__ w,
                                                             const bf16* __restrict__ b, float eps,
                                                             float* __restrict__ out32, long ld32,
                                                             bf16* __restrict__ out_split, long ld_split,
                                                             int n_pad, int N) {
  __shared__ float red[8];
  const int t = blockIdx.x;
  const int nv = N >> 2;
  float4 h[8];
  float s1 = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int c = threadIdx.x + 256 * u;
    h[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nv) {
      h[u] = *reinterpret_cast<const float4*>(x + (long)t * ldx + c * 4);
      s1 += (h[u].x + h[u].y) + (h[u].z + h[u].w);
    }
  }
  const float mu = block_sum<8>(s1, red) / (float)N;
  float v = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int c = threadIdx.x + 256 * u;
    if (c < nv) {
      const float d0 = h[u].x - mu, d1 = h[u].y - mu, d2 = h[u].z - mu, d3 = h[u].w - mu;
      v += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
  }
  const float rstd = rsqrtf(block_sum<8>(v, red) / (float)N + eps);
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int c = threadIdx.x + 256 * u;
    if (c < nv) {
      float wf[4] = {1.f, 1.f, 1.f, 1.f}, bb[4] = {0.f, 0.f, 0.f, 0.f};
      if (w) unpack4(*reinterpret_cast<const uint2*>(w + c * 4), wf);
      if (b) unpack4(*reinterpret_cast<const uint2*>(b + c * 4), bb);
      const float o0 = (h[u].x - mu) * rstd * wf[0] + bb[0], o1 = (h[u].y - mu) * rstd * wf[1] + bb[1];
      const float o2 = (h[u].z - mu) * rstd * wf[2] + bb[2], o3 = (h[u].w - mu) * rstd * wf[3] + bb[3];
      if (out32) *reinterpret_cast<float4*>(out32 + (long)t * ld32 + c * 4) = make_float4(o0, o1, o2, o3);
      if (out_split) split_store4(out_split + (long)t * ld_split + c * 4, n_pad, o0, o1, o2, o3);
    }
  }
}

// RMSNorm in fp32 (nn.RMSNorm on fp32 rows, bf16-valued weight) -> fp32 and / or split output.  Input row
// t is written to output row (t / seg_in) * seg_out + seg_off + t % seg_in: the Idefics2 perceiver
// normalises the context and the latents separately and attends over their concatenation
// (idefics2.py:60-90), so both norms write into ONE [context; latents] buffer per image.
__global__ void __launch_bounds__(256) f32_rms_norm_kernel(const float* __restrict__ x, long ldx,
                                                           const bf16* __restrict__ w, float eps,
                                                           float* __restrict__ out32, long ld32,
                                                           bf16* __restrict__ out_split, long ld_split, int n_pad,
                                                           int N, int seg_in, int seg_out, int seg_off) {
  __shared__ float red[8];
  const int t = blockIdx.x;
  const long ot = seg_in > 0 ? (long)(t / seg_in) * seg_out + seg_off + t % seg_in : t;
  const int nv = N >> 2;
  float4 h[8];
  float s2 = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int c = threadIdx.x + 256 * u;
    h[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nv) {
      h[u] = *reinterpret_cast<const float4*>(x + (long)t * ldx + c * 4);
      s2 += (h[u].x * h[u].x + h[u].y * h[u].y) + (h[u].z * h[u].z + h[u].w * h[u].w);
    }
  }
  const float rs = rsqrtf(block_sum<8>(s2, red) / (float)N + eps);
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int c = threadIdx.x + 256 * u;
    if (c < nv) {
      float wf[4];
      unpack4(*reinterpret_cast<const uint2*>(w + c * 4), wf);
      const float o0 = h[u].x * rs * wf[0], o1 = h[u].y * rs * wf[1], o2 = h[u].z * rs * wf[2], o3 = h[u].w * rs * wf[3];
      if (out32) *reinterpret_cast<float4*>(out32 + ot * ld32 + c * 4) = make_float4(o0, o1, o2, o3);
      if (out_split) split_store4(out_split + ot * ld_split + c * 4, n_pad, o0, o1, o2, o3);
    }
  }
}

// SwiGLU in fp32: gu [T, 2I] = [gate | up] -> split operand of silu(gate) * up (idefics2.py:146-171, mlp)
__global__ void f32_swiglu_split_kernel(const float* __restrict__ gu, long ldg, bf16* __restrict__ out, long ld_split,
                                        int n_pad, int T, int I) {
  const int nv = I >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (long)T * nv; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i / nv), c = (int)(i % nv);
    const float4 g = *reinterpret_cast<const float4*>(gu + (long)t * ldg + c * 4);
    const float4 u = *reinterpret_cast<const float4*>(gu + (long)t * ldg + I + c * 4);
    split_store4(out + (long)t * ld_split + c * 4, n_pad, g.x * sigmoid_f(g.x) * u.x, g.y * sigmoid_f(g.y) * u.y,
                 g.z * sigmoid_f(g.z) * u.z, g.w * sigmoid_f(g.w) * u.w);
  }
}

// fp32 [T, N] -> split operand [T, hi | lo] (zero padding columns are the caller's: buffers are zeroed once)
__global__ void f32_split_kernel(const float* __restrict__ x, long ldx, bf16* __restrict__ out, long ld_split,
                                 int n_pad, int T, int N) {
  const int nv = N >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (long)T * nv; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i / nv), c = (int)(i % nv);
    const float4 v = *reinterpret_cast<const float4*>(x + (long)t * ldx + c * 4);
    split_store4(out + (long)t * ld_split + c * 4, n_pad, v.x, v.y, v.z, v.w);
  }
}

// Idefics3 / SmolVLM pixel shuffle (reference idefics3.py:47-62) fused with the operand split of the connector's
// Linear: x fp32 [n_img, side, side, E] -> split operand [n_img * (side / s)^2, E s^2]; output row (yg, xg), column
// (dy s + dx) E + e = x[yg s + dy, xg s + dx, e].  round_in: the values are rounded to bf16 first (the reference's
// tower output is bf16), which makes the lo half zero.
__global__ void pixel_shuffle_split_kernel(const float* __restrict__ x, int n_img, int side, int E, int s, int round_in,
                                           bf16* __restrict__ out, long ld_split, int n_pad) {
  const int g = side / s, ev = E >> 2, cols = s * s * ev;
  const long total = (long)n_img * g * g * cols;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const long r = i / cols;
    const int e4 = c % ev, d = c / ev, dx = d % s, dy = d / s;
    const int xg = (int)(r % g), yg = (int)((r / g) % g), b = (int)(r / ((long)g * g));
    float4 v = *reinterpret_cast<const float4*>(x + (((long)b * side + yg * s + dy) * side + xg * s + dx) * E + e4 * 4);
    if (round_in) v = make_float4(rbf(v.x), rbf(v.y), rbf(v.z), rbf(v.w));
    split_store4(out + r * ld_split + (long)d * E + e4 * 4, n_pad, v.x, v.y, v.z, v.w);
  }
}

// 2-D rotary embedding of the Qwen2-VL / Qwen2.5-VL vision towers on fp32 q and k in place (reference
// qwen2_5_vl/vision.py:35-50: x * cos + rotate_half(x) * sin in fp32 with cos / sin tiled twice along the head):
// qkv [T, 3 * n_heads * hd] fp32 (q | k | v), pos_hw [T][2] the (row, column) of each patch, inv_freq [hd / 4];
// pair j < hd / 2 turns by pos[j < hd / 4 ? row : column] * inv_freq[j mod hd / 4].
__global__ void f32_vision_rope_kernel(float* __restrict__ qkv, long ld, const int* __restrict__ pos_hw,
                                       const float* __restrict__ inv_freq, int T, int n_heads, int hd) {
  const int half = hd >> 1, quarter = hd >> 2;
  const long total = (long)T * 2 * n_heads * half;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int j = (int)(i % half);
    long r = i / half;
    const int h = (int)(r % n_heads);
    r /= n_heads;
    const int which = (int)(r & 1), t = (int)(r >> 1);
    const int axis = j < quarter ? 0 : 1;
    const float ang = (float)pos_hw[t * 2 + axis] * inv_freq[j - axis * quarter];
    const float c = cosf(ang), sn = sinf(ang);
    float* base = qkv + (long)t * ld + ((long)which * n_heads + h) * hd;
    const float x1 = base[j], x2 = base[j + half];
    base[j] = __fadd_rn(__fmul_rn(x1, c), __fmul_rn(-x2, sn));
    base[j + half] = __fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, sn));
  }
}

// out[(i * unit + u), :] = in[(idx[i] * unit + u), :]  — the window permutation of Qwen2.5-VL's merge units and its
// inverse (qwen2_5_vl/vision.py:343-347,386-388); rows of n fp32 values (n % 4 == 0)
__global__ void f32_gather_rows_kernel(const float* __restrict__ in, long ld_in, const int* __restrict__ idx, int n_idx,
                                       int unit, int n, float* __restrict__ out, long ld_out) {
  const int nv = n >> 2;
  const long total = (long)n_idx * unit * nv;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % nv);
    const long r = i / nv;
    const int u = (int)(r % unit);
    const long g = r / unit;
    *reinterpret_cast<float4*>(out + r * ld_out + c * 4) =
        *reinterpret_cast<const float4*>(in + ((long)idx[g] * unit + u) * ld_in + c * 4);
  }
}

// Conv2d(kernel == stride) as a Linear: NHWC fp32 pixels -> rows of (kh, kw, c)-ordered patches, written
// as a split operand [B * gh * gw, Kp | Kp] (K = ps * ps * C, zero padded to Kp).  (llava/vision.py:108-127)
__global__ void clip_patchify_kernel(const float* __restrict__ pix, int B, int H, int W, int C, int ps,
                                     bf16* __restrict__ out, int Kp) {
  const int gh = H / ps, gw = W / ps, K = ps * ps * C;
  const long total = (long)B * gh * gw * Kp;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kp);
    const long r = i / Kp;
    float v = 0.f;
    if (k < K) {
      const int c = k % C, kw = (k / C) % ps, kh = k / (C * ps);
      const int gx = (int)(r % gw), gy = (int)((r / gw) % gh), b = (int)(r / ((long)gw * gh));
      v = pix[(((long)b * H + gy * ps + kh) * W + gx * ps + kw) * C + c];
    }
    const float hi = rbf(v);
    out[r * 2 * Kp + k] = f2bf(hi);
    out[r * 2 * Kp + Kp + k] = f2bf(v - hi);
  }
}

// emb[b][0] = cls + pos[0];  emb[b][1 + p] = patch[b][p] + pos[1 + p]   (fp32; cls == nullptr: no class
// token, emb[b][p] = patch[b][p] + pos[pos_ids[b][p]] — the SigLIP form with bucketed position ids)
__global__ void tower_embed_kernel(const float* __restrict__ patch, const bf16* __restrict__ cls,
                                   const bf16* __restrict__ pos, const int* __restrict__ pos_ids,
                                   float* __restrict__ emb, int B, int P, int E, int n_pos) {
  const int L = P + (cls ? 1 : 0);
  const long total = (long)B * L * (E >> 2);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (E >> 2));
    const long r = i / (E >> 2);
    const int l = (int)(r % L), b = (int)(r / L);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    float pe[4];
    int pid = l;
    if (cls) {
      if (l == 0) {
        float cf[4];
        unpack4(*reinterpret_cast<const uint2*>(cls + c * 4), cf);
        v = make_float4(cf[0], cf[1], cf[2], cf[3]);
      } else {
        v = *reinterpret_cast<const float4*>(patch + ((long)b * P + l - 1) * E + c * 4);
      }
    } else {
      v = *reinterpret_cast<const float4*>(patch + ((long)b * P + l) * E + c * 4);
      if (pos_ids) {
        pid = pos_ids[(long)b * P + l];
        if (pid < 0) pid += n_pos;  // numpy-style negative index (the reference's digitize(...) - 1 quirk)
      }
    }
    unpack4(*reinterpret_cast<const uint2*>(pos + (long)pid * E + c * 4), pe);
    *reinterpret_cast<float4*>(emb + r * E + c * 4) = make_float4(v.x + pe[0], v.y + pe[1], v.z + pe[2], v.w + pe[3]);
  }
}

// ---- fp32 attention on the CUDA cores (exact fp32 softmax; flash-style running max / sum) -----------
// Register-tiled: CTA = 64 query rows of one head of one segment, 128 threads as 8 (query groups of 8 rows) x
// 16 (key groups of 4 keys / dim lanes); 65 KB of shared memory -> three CTAs per SM, and CLIP's 8 x 16 x 10 = 1280
// CTAs fill 2.9 of 3 waves (128-row CTAs at two per SM wasted 28 % of the third wave).  Per 64-key tile:
//   S[8 x 4] per thread = Q^T . K^T out of shared memory (both stored dim-major so that a thread's 8 queries /
//   4 keys are one or two 16-byte loads and the 16 lanes of a key group read 256 contiguous bytes: 32 FMAs per
//   3 shared loads), running max over the 16 lanes of a query group (4 shuffles per row), p = exp(s - m) written
//   as P^T[key][query] (only the half-warp that owns the rows reads it back: __syncwarp), then
//   O[8 x HDP/16] += P . V with the thread's dims interleaved (dim = e * 16 + lane: conflict-free, coalesced stores).
// The round-1 version of this kernel (4 threads per row, 1 FMA per shared load) ran at ~6 TFLOP/s and was 88 % of the
// CLIP tower's time; this one is bounded by the FMA pipe.
struct AttnF32P {
  const float *q, *k, *v;
  long q_ts, q_hs, k_ts, k_hs, v_ts, v_hs;  // element strides: token, head
  float* out32;
  long o_ts;
  bf16* out_split;
  long os_ts;
  int n_pad;
  int n_heads, n_kv, Lq, S, hd;
  long q_seg, k_seg;   // tokens between consecutive segments (blockIdx.z)
  const unsigned char* key_mask;  // optional [segments][S]: 0 = key masked out
  const int* cu;                  // optional [segments + 1]: segment z = tokens [cu[z], cu[z+1]) of q, k and v (self-attention
                                  // over ragged segments, e.g. Qwen2.5-VL's windows); Lq is then the longest segment
  float scale;
};

constexpr int AF_BQ = 64, AF_BK = 64, AF_THREADS = AF_BQ * 2;
constexpr int AF_PP = AF_BQ + 4;  // P^T row pitch: +4 floats; with rows stored as (key % 4) * 16 + key / 4 the 16 lanes of
                                  // a key group write consecutive rows -> conflict-free 16-byte stores

template <int HDP>
static constexpr size_t attn_f32_smem() {
  return ((size_t)HDP * AF_BQ + (size_t)HDP * AF_BK + (size_t)AF_BK * HDP + (size_t)AF_BK * AF_PP) * 4 + AF_BK;
}

template <int HDP>
__global__ void __launch_bounds__(AF_THREADS) attention_f32_kernel(const AttnF32P p) {
  constexpr int BQ = AF_BQ, BK = AF_BK, PP = AF_PP, DPT = HDP / 16, NT = AF_THREADS;
  extern __shared__ __align__(16) float af_sm[];
  float* Qt = af_sm;               // [HDP][BQ]  q * scale, dim-major
  float* Kt = Qt + HDP * BQ;       // [HDP][BK]
  float* Vs = Kt + HDP * BK;       // [BK][HDP]
  float* Pt = Vs + BK * HDP;       // [BK][PP]
  unsigned char* Ms = reinterpret_cast<unsigned char*>(Pt + BK * PP);  // [BK] 1 = key takes part
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int h = blockIdx.y, kvh = h / (p.n_heads / p.n_kv), seg = blockIdx.z;
  const int q0 = blockIdx.x * BQ;
  const int hd = p.hd, hd4 = hd >> 2;
  long q_first = (long)seg * p.q_seg, k_first = (long)seg * p.k_seg;
  int Lq = p.Lq, S = p.S;
  if (p.cu) {
    q_first = k_first = p.cu[seg];
    Lq = S = p.cu[seg + 1] - p.cu[seg];
    if (q0 >= Lq) return;   // uniform per CTA
  }
  const float* qb = p.q + q_first * p.q_ts + (long)h * p.q_hs;
  const float* kb = p.k + k_first * p.k_ts + (long)kvh * p.k_hs;
  const float* vb = p.v + k_first * p.v_ts + (long)kvh * p.v_hs;
  // Q^T: lane <-> query row (conflict-free transposed stores)
  for (int i = tid; i < BQ * (HDP / 4); i += NT) {
    const int r = i % BQ, c = i / BQ;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < Lq && c < hd4) v = *reinterpret_cast<const float4*>(qb + (long)(q0 + r) * p.q_ts + c * 4);
    Qt[(c * 4 + 0) * BQ + r] = v.x * p.scale;
    Qt[(c * 4 + 1) * BQ + r] = v.y * p.scale;
    Qt[(c * 4 + 2) * BQ + r] = v.z * p.scale;
    Qt[(c * 4 + 3) * BQ + r] = v.w * p.scale;
  }
  float o[8][DPT], m[8], l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    m[i] = -INFINITY;
    l[i] = 0.f;
#pragma unroll
    for (int e = 0; e < DPT; ++e) o[i][e] = 0.f;
  }
  for (int j0 = 0; j0 < S; j0 += BK) {
    __syncthreads();
    for (int i = tid; i < BK * (HDP / 4); i += NT) {   // K^T: lane <-> key
      const int r = i % BK, c = i / BK;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + r < S && c < hd4) v = *reinterpret_cast<const float4*>(kb + (long)(j0 + r) * p.k_ts + c * 4);
      Kt[(c * 4 + 0) * BK + r] = v.x;
      Kt[(c * 4 + 1) * BK + r] = v.y;
      Kt[(c * 4 + 2) * BK + r] = v.z;
      Kt[(c * 4 + 3) * BK + r] = v.w;
    }
    for (int i = tid; i < BK * (HDP / 4); i += NT) {   // V: row-major
      const int r = i / (HDP / 4), c = i % (HDP / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + r < S && c < hd4) v = *reinterpret_cast<const float4*>(vb + (long)(j0 + r) * p.v_ts + c * 4);
      *reinterpret_cast<float4*>(Vs + r * HDP + c * 4) = v;
    }
    if (tid < BK) Ms[tid] = (j0 + tid < S) && (!p.key_mask || p.key_mask[(long)seg * S + j0 + tid]);
    __syncthreads();
    // ---- S = Q . K^T for this thread's 8 rows x 4 keys ----
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 4
    for (int d = 0; d < HDP; ++d) {
      const float4 qa = *reinterpret_cast<const float4*>(Qt + d * BQ + ty * 8);
      const float4 qc = *reinterpret_cast<const float4*>(Qt + d * BQ + ty * 8 + 4);
      const float4 kk = *reinterpret_cast<const float4*>(Kt + d * BK + tx * 4);
      const float qv[8] = {qa.x, qa.y, qa.z, qa.w, qc.x, qc.y, qc.z, qc.w};
      const float kv[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    bool on[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) on[j] = Ms[tx * 4 + j] != 0;
    // ---- running max / sum, p -> P^T ----
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) mx = on[j] ? fmaxf(mx, s[i][j]) : mx;
#pragma unroll
      for (int w = 1; w < 16; w <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, w));
      const float mn = fmaxf(m[i], mx);
      const float f = (mn == -INFINITY) ? 1.f : __expf(m[i] - mn);   // nothing seen yet: keep zeros
      m[i] = mn;
      l[i] *= f;
#pragma unroll
      for (int e = 0; e < DPT; ++e) o[i][e] *= f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float pj = on[j] ? __expf(s[i][j] - mn) : 0.f;
        s[i][j] = pj;
        l[i] += pj;   // this thread's share of the row sum (reduced over the 16 lanes at the end)
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // key tx * 4 + j lives in P^T row j * 16 + tx
      float* dst = Pt + (j * 16 + tx) * PP + ty * 8;
      *reinterpret_cast<float4*>(dst) = make_float4(s[0][j], s[1][j], s[2][j], s[3][j]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(s[4][j], s[5][j], s[6][j], s[7][j]);
    }
    __syncwarp();   // rows ty*8.. of P^T are written and read by the same half-warp only
    // ---- O += P . V ----
#pragma unroll 4
    for (int r = 0; r < BK; ++r) {
      const int j = (r & 15) * 4 + (r >> 4);   // the key stored in P^T row r
      const float4 pa = *reinterpret_cast<const float4*>(Pt + r * PP + ty * 8);
      const float4 pc = *reinterpret_cast<const float4*>(Pt + r * PP + ty * 8 + 4);
      const float pv[8] = {pa.x, pa.y, pa.z, pa.w, pc.x, pc.y, pc.z, pc.w};
      float vv[DPT];
#pragma unroll
      for (int e = 0; e < DPT; ++e) vv[e] = Vs[j * HDP + e * 16 + tx];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < DPT; ++e) o[i][e] = fmaf(pv[i], vv[e], o[i][e]);
    }
    __syncwarp();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float ls = l[i];
#pragma unroll
    for (int w = 1; w < 16; w <<= 1) ls += __shfl_xor_sync(0xffffffffu, ls, w);
    const int qi = q0 + ty * 8 + i;
    if (qi >= Lq) continue;
    const float inv = 1.0f / ls;
    const long t = q_first + qi;
#pragma unroll
    for (int e = 0; e < DPT; ++e) {
      const int d = e * 16 + tx;
      if (d >= hd) continue;
      const float a = o[i][e] * inv;
      const long col = (long)h * hd + d;
      if (p.out32) p.out32[t * p.o_ts + col] = a;
      if (p.out_split) {
        const float hi = rbf(a);
        p.out_split[t * p.os_ts + col] = f2bf(hi);
        p.out_split[t * p.os_ts + col + p.n_pad] = f2bf(a - hi);
      }
    }
  }
}

template <int HDP>
static int attn_f32_launch(const AttnF32P& p, dim3 grid, cudaStream_t st) {
  if (int rc = kernel_opt_in((const void*)attention_f32_kernel<HDP>, (int)attn_f32_smem<HDP>(), false)) return rc;
  attention_f32_kernel<HDP><<<grid, AF_THREADS, attn_f32_smem<HDP>(), st>>>(p);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace

int f32_layer_norm(const float* x, long ldx, const void* w, const void* b, float eps, float* out32, long ld32,
                   void* out_split, long ld_split, int n_pad, int T, int N, cudaStream_t st) {
  B200_REQUIRE(x && T > 0 && N > 0 && (N % 4) == 0 && N <= 8192 && (ldx % 4) == 0, "f32_layer_norm: T=%d N=%d", T, N);
  B200_REQUIRE(out32 || out_split, "f32_layer_norm: no output");
  B200_REQUIRE(!out_split || ((ld_split % 4) == 0 && (n_pad % 4) == 0), "f32_layer_norm: split pitch");
  f32_layer_norm_kernel<<<T, 256, 0, st>>>(x, ldx, (const bf16*)w, (const bf16*)b, eps, out32, ld32,
                                           (bf16*)out_split, ld_split, n_pad, N);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int f32_rms_norm(const float* x, long ldx, const void* w, float eps, float* out32, long ld32, void* out_split,
                 long ld_split, int n_pad, int T, int N, int seg_in, int seg_out, int seg_off, cudaStream_t st) {
  B200_REQUIRE(x && w && T > 0 && N > 0 && (N % 4) == 0 && N <= 8192 && (ldx % 4) == 0 && (out32 || out_split),
               "f32_rms_norm: T=%d N=%d", T, N);
  f32_rms_norm_kernel<<<T, 256, 0, st>>>(x, ldx, (const bf16*)w, eps, out32, ld32, (bf16*)out_split, ld_split, n_pad, N,
                                         seg_in, seg_out, seg_off);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int f32_swiglu_split(const float* gu, long ldg, void* out, long ld_split, int n_pad, int T, int I, cudaStream_t st) {
  B200_REQUIRE(gu && out && T > 0 && I > 0 && (I % 4) == 0 && (ldg % 4) == 0 && (ld_split % 4) == 0, "f32_swiglu: bad shape");
  f32_swiglu_split_kernel<<<grid_for((long)T * (I / 4), 256), 256, 0, st>>>(gu, ldg, (bf16*)out, ld_split, n_pad, T, I);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int f32_split(const float* x, long ldx, void* out, long ld_split, int n_pad, int T, int N, cudaStream_t st) {
  B200_REQUIRE(x && out && T > 0 && N > 0 && (N % 4) == 0 && (ldx % 4) == 0 && (ld_split % 4) == 0 && (n_pad % 4) == 0,
               "f32_split: bad shape");
  f32_split_kernel<<<grid_for((long)T * (N / 4), 256), 256, 0, st>>>(x, ldx, (bf16*)out, ld_split, n_pad, T, N);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int pixel_shuffle_split(const float* x, int n_img, int side, int E, int s, int round_in, void* out, long ld_split,
                        int n_pad, cudaStream_t st) {
  B200_REQUIRE(x && out && n_img > 0 && s > 0 && side > 0 && side % s == 0 && (E % 4) == 0 && n_pad >= E * s * s &&
                   (ld_split % 4) == 0 && (n_pad % 4) == 0, "pixel_shuffle_split: bad shape");
  const long total = (long)n_img * (side / s) * (side / s) * s * s * (E / 4);
  pixel_shuffle_split_kernel<<<grid_for(total, 256), 256, 0, st>>>(x, n_img, side, E, s, round_in, (bf16*)out, ld_split,
                                                                 n_pad);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int clip_patchify(const float* pix, int B, int H, int W, int C, int ps, void* out, int Kp, cudaStream_t st) {
  B200_REQUIRE(pix && out && B > 0 && H % ps == 0 && W % ps == 0 && Kp >= ps * ps * C && (Kp % 8) == 0,
               "clip_patchify: bad shape");
  const long total = (long)B * (H / ps) * (W / ps) * Kp;
  clip_patchify_kernel<<<grid_for(total, 256), 256, 0, st>>>(pix, B, H, W, C, ps, (bf16*)out, Kp);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int tower_embed(const float* patch, const void* cls, const void* pos, const int* pos_ids, float* emb, int B, int P,
                int E, int n_pos, cudaStream_t st) {
  B200_REQUIRE(patch && pos && emb && B > 0 && P > 0 && (E % 4) == 0, "tower_embed: bad shape");
  const long total = (long)B * (P + (cls ? 1 : 0)) * (E / 4);
  tower_embed_kernel<<<grid_for(total, 256), 256, 0, st>>>(patch, (const bf16*)cls, (const bf16*)pos, pos_ids, emb, B, P,
                                                         E, n_pos);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int f32_vision_rope(float* qkv, long ld, const int* pos_hw, const float* inv_freq, int T, int n_heads, int hd,
                    cudaStream_t st) {
  B200_REQUIRE(qkv && pos_hw && inv_freq && T > 0 && n_heads > 0 && (hd % 4) == 0 && ld >= 3L * n_heads * hd,
               "f32_vision_rope: bad shape");
  f32_vision_rope_kernel<<<grid_for((long)T * n_heads * hd, 256), 256, 0, st>>>(qkv, ld, pos_hw, inv_freq, T, n_heads, hd);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int f32_gather_rows(const float* in, long ld_in, const int* idx, int n_idx, int unit, int n, float* out, long ld_out,
                    cudaStream_t st) {
  B200_REQUIRE(in && idx && out && n_idx > 0 && unit > 0 && n > 0 && (n % 4) == 0 && (ld_in % 4) == 0 && (ld_out % 4) == 0,
               "f32_gather_rows: bad shape");
  f32_gather_rows_kernel<<<grid_for((long)n_idx * unit * (n / 4), 256), 256, 0, st>>>(in, ld_in, idx, n_idx, unit, n, out,
                                                                                   ld_out);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int attention_f32(const float* q, long q_ts, long q_hs, const float* k, long k_ts, long k_hs, const float* v,
                  long v_ts, long v_hs, float* out32, long o_ts, void* out_split, long os_ts, int n_pad,
                  int n_heads, int n_kv, int hd, int Lq, int S, int n_seg, long q_seg, long k_seg,
                  const unsigned char* key_mask, float scale, cudaStream_t st, const int* cu = nullptr) {
  B200_REQUIRE(q && k && v && (out32 || out_split) && Lq > 0 && S > 0 && n_seg > 0 && n_heads % n_kv == 0,
               "attention_f32: bad arguments");
  B200_REQUIRE(!cu || !key_mask, "attention_f32: ragged segments take no key mask");
  B200_REQUIRE((q_ts % 4) == 0 && (k_ts % 4) == 0 && (v_ts % 4) == 0 && (q_hs % 4) == 0 && (k_hs % 4) == 0 &&
                   (v_hs % 4) == 0 && (o_ts % 4) == 0 && (os_ts % 4) == 0 && (n_pad % 4) == 0,
               "attention_f32: strides must be multiples of 4 elements");
  AttnF32P p;
  p.q = q; p.k = k; p.v = v; p.q_ts = q_ts; p.q_hs = q_hs; p.k_ts = k_ts; p.k_hs = k_hs; p.v_ts = v_ts; p.v_hs = v_hs;
  p.out32 = out32; p.o_ts = o_ts; p.out_split = (bf16*)out_split; p.os_ts = os_ts; p.n_pad = n_pad;
  p.n_heads = n_heads; p.n_kv = n_kv; p.Lq = Lq; p.S = S; p.q_seg = q_seg; p.k_seg = k_seg; p.key_mask = key_mask;
  p.scale = scale;
  p.cu = cu;
  p.hd = hd;
  B200_REQUIRE((hd % 4) == 0 && hd <= 96, "attention_f32: head_dim %d (multiple of 4, <= 96)", hd);
  const dim3 grid(cdiv(Lq, AF_BQ), n_heads, n_seg);
  if (hd <= 16) return attn_f32_launch<16>(p, grid, st);
  if (hd <= 32) return attn_f32_launch<32>(p, grid, st);
  if (hd <= 64) return attn_f32_launch<64>(p, grid, st);   // CLIP-L
  if (hd <= 80) return attn_f32_launch<80>(p, grid, st);   // SigLIP-SO400M: 72 dims, padded with zeros
  return attn_f32_launch<96>(p, grid, st);                 // Idefics2 perceiver
}

}  // namespace b200

using namespace b200;
extern "C" {
int b200_f32_layer_norm(const float* x, long ldx, const void* w, const void* b, float eps, float* out32, long ld32,
                        void* out_split, long ld_split, int n_pad, int T, int N, void* st) {
  return f32_layer_norm(x, ldx, w, b, eps, out32, ld32, out_split, ld_split, n_pad, T, N, (cudaStream_t)st);
}
int b200_f32_rms_norm(const float* x, long ldx, const void* w, float eps, float* out32, long ld32, void* out_split,
                      long ld_split, int n_pad, int T, int N, int seg_in, int seg_out, int seg_off, void* st) {
  return f32_rms_norm(x, ldx, w, eps, out32, ld32, out_split, ld_split, n_pad, T, N, seg_in, seg_out, seg_off,
                      (cudaStream_t)st);
}
int b200_f32_swiglu_split(const float* gu, long ldg, void* out, long ld_split, int n_pad, int T, int I, void* st) {
  return f32_swiglu_split(gu, ldg, out, ld_split, n_pad, T, I, (cudaStream_t)st);
}
int b200_f32_split(const float* x, long ldx, void* out, long ld_split, int n_pad, int T, int N, void* st) {
  return f32_split(x, ldx, out, ld_split, n_pad, T, N, (cudaStream_t)st);
}
int b200_pixel_shuffle_split(const float* x, int n_img, int side, int E, int s, int round_in, void* out_split,
                             long ld_split, int n_pad, void* st) {
  return pixel_shuffle_split(x, n_img, side, E, s, round_in, out_split, ld_split, n_pad, (cudaStream_t)st);
}
int b200_clip_patchify(const float* pix, int B, int H, int W, int C, int ps, void* out, int Kp, void* st) {
  return clip_patchify(pix, B, H, W, C, ps, out, Kp, (cudaStream_t)st);
}
int b200_tower_embed(const float* patch, const void* cls, const void* pos, const int* pos_ids, float* emb, int B,
                     int P, int E, int n_pos, void* st) {
  return tower_embed(patch, cls, pos, pos_ids, emb, B, P, E, n_pos, (cudaStream_t)st);
}
int b200_attention_f32(const float* q, long q_ts, long q_hs, const float* k, long k_ts, long k_hs, const float* v,
                       long v_ts, long v_hs, float* out32, long o_ts, void* out_split, long os_ts, int n_pad,
                       int n_heads, int n_kv, int hd, int Lq, int S, int n_seg, long q_seg, long k_seg,
                       const unsigned char* key_mask, float scale, void* st) {
  return attention_f32(q, q_ts, q_hs, k, k_ts, k_hs, v, v_ts, v_hs, out32, o_ts, out_split, os_ts, n_pad, n_heads,
                       n_kv, hd, Lq, S, n_seg, q_seg, k_seg, key_mask, scale, (cudaStream_t)st);
}
int b200_attention_f32_varlen(const float* q, long q_ts, long q_hs, const float* k, long k_ts, long k_hs, const float* v,
                              long v_ts, long v_hs, float* out32, long o_ts, void* out_split, long os_ts, int n_pad,
                              int n_heads, int n_kv, int hd, const int* cu_seqlens, int n_seg, int max_len, float scale,
                              void* st) {
  B200_REQUIRE(cu_seqlens && max_len > 0, "attention_f32_varlen: needs cu_seqlens and the longest segment");
  return attention_f32(q, q_ts, q_hs, k, k_ts, k_hs, v, v_ts, v_hs, out32, o_ts, out_split, os_ts, n_pad, n_heads,
                       n_kv, hd, max_len, max_len, n_seg, 0, 0, nullptr, scale, (cudaStream_t)st, cu_seqlens);
}
int b200_f32_vision_rope(float* qkv, long ld, const int* pos_hw, const float* inv_freq, int T, int n_heads, int hd,
                         void* st) {
  return f32_vision_rope(qkv, ld, pos_hw, inv_freq, T, n_heads, hd, (cudaStream_t)st);
}
int b200_f32_gather_rows(const float* in, long ld_in, const int* idx, int n_idx, int unit, int n, float* out,
                         long ld_out, void* st) {
  return f32_gather_rows(in, ld_in, idx, n_idx, unit, n, out, ld_out, (cudaStream_t)st);
}
/* fp32-accurate Linear on the tensor cores: X = split operand [T, n_parts x Kp] (Kp = K_w rounded up to 64),
 * W [N, K_w] bf16; mode B200_WT_F32 (C32 = act(acc + bias) + res32) or B200_WT_SPLIT (Csplit = [hi | lo]).
 * cfg4 = {TN, KS, stages, 1} runs that configuration; NULL keeps the measured choice. */
int b200_gemm_wt_f32(const void* X, long ldx, const void* W, long ldw, const void* bias, const float* res32,
                     long ldr32, float* C32, long ldc32, void* Csplit, long ld_split, int n_pad, int T, int N,
                     int K_w, int n_parts, int epilogue, int mode, const int* cfg4, void* stream) {
  const int kbw = cdiv(K_w, 64);
  WtExt ext;
  ext.kb_w = kbw; ext.k_w = K_w; ext.ldw = ldw; ext.C32 = C32; ext.res32 = res32; ext.ldc32 = ldc32;
  ext.ldr32 = ldr32; ext.Csplit = (bf16*)Csplit; ext.ld_split = ld_split; ext.n_pad = n_pad;
  if (cfg4 && cfg4[0] > 0)
    return gemm_wt(X, ldx, W, bias, nullptr, 0, nullptr, 0, nullptr, T, N, n_parts * kbw * 64, epilogue, mode, 0,
                   WtConfig{cfg4[0], cfg4[1], cfg4[2], cfg4[3]}, 0, (cudaStream_t)stream, &ext);
  return gemm_wt_tuned(X, ldx, W, bias, nullptr, 0, nullptr, 0, nullptr, 0, T, N, n_parts * kbw * 64, epilogue, mode, 0,
                       false, 132, nullptr, (cudaStream_t)stream, &ext);
}
}
