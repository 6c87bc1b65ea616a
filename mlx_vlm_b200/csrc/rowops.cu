// Row-wise memory-bound kernels of the prefill / vision path: dtype cast, LayerNorm,
// RMSNorm, vision 2-D rotary, M-RoPE + KV append, SwiGLU, embed + image-feature
// merge.  All are HBM-bound: 16-byte vector accesses, one warp per row where a
// reduction is needed.  Rounding points follow oracle/mlx_semantics.py.
#include "common.cuh"
#include "decode.cuh"

namespace b200 {

// ---------------------------------------------------------------------------
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long n) {
  pdl_prologue();
  long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long stride = (long)gridDim.x * blockDim.x * 4;
  for (; i + 3 < n; i += stride) {
    float4 v = *reinterpret_cast<const float4*>(src + i);
    uint2 o;
    o.x = pack2(v.x, v.y);
    o.y = pack2(v.z, v.w);
    *reinterpret_cast<uint2*>(dst + i) = o;
  }
  if (i < n && i + 3 >= n) {
    for (long j = i; j < n; ++j) dst[j] = f2bf(src[j]);
  }
}

// ---------------------------------------------------------------------------
// mx.fast.layer_norm CPU fallback: fp32 stats, cast, *w (round), +b (round).
// One warp per row; dim % 8 == 0.
__global__ void layer_norm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                  const bf16* __restrict__ b, bf16* __restrict__ y, int rows,
                                  int dim, float eps) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const bf16* xr = x + (long)warp * dim;
  bf16* yr = y + (long)warp * dim;
  const int nvec = dim >> 3;
  float s = 0.f;
  for (int c = lane; c < nvec; c += 32) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j];
  }
  const float mu = warp_sum(s) / (float)dim;
  float v = 0.f;
  for (int c = lane; c < nvec; c += 32) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = f[j] - mu;
      v += d * d;
    }
  }
  const float var = warp_sum(v) / (float)dim;
  const float rstd = 1.0f / sqrtf(var + eps);
  for (int c = lane; c < nvec; c += 32) {
    float f[8], wf[8], bfv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), f);
    if (w) unpack8(*reinterpret_cast<const uint4*>(w + c * 8), wf);
    if (b) unpack8(*reinterpret_cast<const uint4*>(b + c * 8), bfv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float t = rbf((f[j] - mu) * rstd);
      if (w) t = rbf(t * wf[j]);
      if (b) t = rbf(t + bfv[j]);
      o[j] = t;
    }
    uint4 ov;
    ov.x = pack2(o[0], o[1]);
    ov.y = pack2(o[2], o[3]);
    ov.z = pack2(o[4], o[5]);
    ov.w = pack2(o[6], o[7]);
    *reinterpret_cast<uint4*>(yr + c * 8) = ov;
  }
}

// mx.fast.rms_norm CPU fallback: bf16(x * rsqrt(mean(x^2)+eps)) then * w (round).
__global__ void rms_norm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                bf16* __restrict__ y, int rows, int dim, float eps) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const bf16* xr = x + (long)warp * dim;
  bf16* yr = y + (long)warp * dim;
  const int nvec = dim >> 3;
  float s = 0.f;
  for (int c = lane; c < nvec; c += 32) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j] * f[j];
  }
  const float rs = 1.0f / sqrtf(warp_sum(s) / (float)dim + eps);
  for (int c = lane; c < nvec; c += 32) {
    float f[8], wf[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), f);
    unpack8(*reinterpret_cast<const uint4*>(w + c * 8), wf);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = rbf(rbf(f[j] * rs) * wf[j]);
    uint4 ov;
    ov.x = pack2(o[0], o[1]);
    ov.y = pack2(o[2], o[3]);
    ov.z = pack2(o[4], o[5]);
    ov.w = pack2(o[6], o[7]);
    *reinterpret_cast<uint4*>(yr + c * 8) = ov;
  }
}

// ---------------------------------------------------------------------------
// apply_rotary_pos_emb_vision (vision.py:35-50): fp32 cos/sin, ONE rounding.
// freqs for dim j of head_dim: half = hd/2; jj = j % half; jj < half/2 uses the
// h position with inv_freq[jj], else the w position with inv_freq[jj - half/2].
// One thread per (token, which in {q,k}, head, pair j<half).
__global__ void vision_rope_kernel(bf16* __restrict__ qkv, const int* __restrict__ pos_hw,
                                   const float* __restrict__ inv_freq, int n_tok, int n_heads,
                                   int hd) {
  const int half = hd >> 1, quarter = hd >> 2;
  const long total = (long)n_tok * 2 * n_heads * half;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % half);
    long r = idx / half;
    const int h = (int)(r % n_heads);
    r /= n_heads;
    const int which = (int)(r % 2);
    const int t = (int)(r / 2);
    const int axis = (j < quarter) ? 0 : 1;
    const float ang = (float)pos_hw[t * 2 + axis] * inv_freq[j - axis * quarter];
    const float c = cosf(ang), s = sinf(ang);
    bf16* base = qkv + ((long)t * 3 + which) * n_heads * hd + (long)h * hd;
    const float x1 = bf2f(base[j]), x2 = bf2f(base[j + half]);
    // out[j] = x1*cos + (-x2)*sin ; out[j+half] = x2*cos + x1*sin   (fp32, one cast)
    // separate fp32 mul / add like the reference's three array ops (no FMA contraction)
    base[j] = f2bf(__fadd_rn(__fmul_rn(x1, c), __fmul_rn(-x2, s)));
    base[j + half] = f2bf(__fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, s)));
  }
}

// ---------------------------------------------------------------------------
// M-RoPE (rope_utils.py:1227-1241 cos/sin cast to bf16; :1301-1334 three roundings)
// + KV append.  One thread per (t, head-slot, pair j < hd/2); head-slot covers
// n_heads q heads, n_kv k heads, n_kv v heads (v: plain copy).
__global__ void mrope_kv_write_kernel(bf16* __restrict__ qkv, const int* __restrict__ pos3,
                                      const float* __restrict__ inv_freq,
                                      const int* __restrict__ axis_sel, bf16* __restrict__ kc,
                                      bf16* __restrict__ vc, int T, int ctx0, int cap, int n_heads,
                                      int n_kv, int hd, float q_scale, bf16* __restrict__ vt,
                                      int t_ld, const KvRef* __restrict__ ref, int layer,
                                      bf16* __restrict__ kws, const int2* __restrict__ tok_loc,
                                      long row_stride) {
  // tok_loc (batched prefill of several sequences in one pass): token t belongs to pool row tok_loc[t].x and
  // lands at cache position tok_loc[t].y; kc / vc then point at row 0 and rows are row_stride elements apart
  pdl_prologue();
  if (ref) {  // cache location read from device memory: a captured graph stays valid when the pool moves
    kc = ref->k0 + (long)layer * ref->layer_stride;
    vc = kc + ref->v_off;
    cap = ref->cap;
  }
  const int half = hd >> 1;
  const int slots = n_heads + 2 * n_kv;
  const long total = (long)T * slots * half;
  const long row_elems = (long)slots * hd;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % half);
    long r = idx / half;
    const int slot = (int)(r % slots);
    const int t = (int)(r / slots);
    bf16* base = qkv + (long)t * row_elems + (long)slot * hd;
    const float x1 = bf2f(base[j]), x2 = bf2f(base[j + half]);
    if (slot >= n_heads + n_kv) {  // V: copy into the cache
      const int kvh = slot - n_heads - n_kv;
      const int2 loc = tok_loc ? tok_loc[t] : make_int2(0, ctx0 + t);
      if (loc.x >= 0) {   // (row -1: a padding token of a batched prefill)
        bf16* dst = vc + (long)loc.x * row_stride + ((long)kvh * cap + loc.y) * hd;
        dst[j] = base[j];
        dst[j + half] = base[j + half];
      }
      if (vt) {  // V^T [kv head][dim][token] for the pipelined attention kernel (attention_fa.cu)
        vt[((long)kvh * hd + j) * t_ld + t] = base[j];
        vt[((long)kvh * hd + j + half) * t_ld + t] = base[j + half];
      }
      continue;
    }
    const float ang = (float)pos3[axis_sel[j] * T + t] * inv_freq[j];
    const float c = rbf(cosf(ang)), s = rbf(sinf(ang));
    const float o1 = rbf(rbf(x1 * c) + rbf((-x2) * s));
    const float o2 = rbf(rbf(x2 * c) + rbf(x1 * s));
    if (slot < n_heads) {
      // q_scale != 0: qs = bf16(q * bf16(scale)) of the SDPA is applied here (base.py:305-373)
      base[j] = f2bf(q_scale != 0.f ? o1 * q_scale : o1);
      base[j + half] = f2bf(q_scale != 0.f ? o2 * q_scale : o2);
    } else {
      const int kvh = slot - n_heads;
      const int2 loc = tok_loc ? tok_loc[t] : make_int2(0, ctx0 + t);
      if (loc.x >= 0) {
        bf16* dst = kc + (long)loc.x * row_stride + ((long)kvh * cap + loc.y) * hd;
        dst[j] = f2bf(o1);
        dst[j + half] = f2bf(o2);
      }
      if (kws) {  // the prompt chunk's rotated keys [kv head][token][dim] for the pipelined attention
        bf16* d2 = kws + ((long)kvh * T + t) * hd;
        d2[j] = f2bf(o1);
        d2[j + half] = f2bf(o2);
      }
    }
  }
}

// The same operation, tiled (head_dim a multiple of 16): a CTA takes 32 tokens x a group of head slots; thread (token,
// chunk of 8 rotary pairs) computes its 8 cos / sin ONCE and re-uses them for every head of the group, all loads and
// stores are 16-byte vectors, and V^T goes through a shared-memory tile so that its stores are contiguous along the
// token axis.  Identical arithmetic, element for element, to the scalar kernel above (which evaluated cosf / sinf per
// element and wrote V^T with 2-byte stores a row apart).  grid (ceil(T / 32), slot groups), 256 threads.
__global__ void __launch_bounds__(256)
mrope_kv_write_tiled_kernel(bf16* __restrict__ qkv, const int* __restrict__ pos3, const float* __restrict__ inv_freq,
                            const int* __restrict__ axis_sel, bf16* __restrict__ kc, bf16* __restrict__ vc, int T, int ctx0,
                            int cap, int n_heads, int n_kv, int hd, float q_scale, bf16* __restrict__ vt, int t_ld,
                            const KvRef* __restrict__ ref, int layer, bf16* __restrict__ kws,
                            const int2* __restrict__ tok_loc, long row_stride, int slots_per_cta) {
  pdl_prologue();
  if (ref) {
    kc = ref->k0 + (long)layer * ref->layer_stride;
    vc = kc + ref->v_off;
    cap = ref->cap;
  }
  __shared__ bf16 tile[32][136];
  const int half = hd >> 1, nc = half >> 3, nv = hd >> 3;
  const int slots = n_heads + 2 * n_kv;
  const long row_elems = (long)slots * hd;
  const int t0 = blockIdx.x * 32;
  const int tl = threadIdx.x / nc, c = threadIdx.x % nc;
  const int t = t0 + tl;
  const bool act = threadIdx.x < 32 * nc && t < T;
  float cs[8], sn[8];
  int2 loc = make_int2(-1, 0);
  if (act) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = c * 8 + u;
      const float ang = (float)pos3[axis_sel[j] * T + t] * inv_freq[j];
      cs[u] = rbf(cosf(ang));
      sn[u] = rbf(sinf(ang));
    }
    loc = tok_loc ? tok_loc[t] : make_int2(0, ctx0 + t);
  }
  const int s_begin = blockIdx.y * slots_per_cta;
  const int s_end = min(slots, s_begin + slots_per_cta);
  for (int slot = s_begin; slot < s_end; ++slot) {
    if (slot < n_heads + n_kv) {   // q or k head: rotate
      if (!act) continue;
      bf16* base = qkv + (long)t * row_elems + (long)slot * hd;
      float x1[8], x2[8], o1[8], o2[8];
      unpack8(*reinterpret_cast<const uint4*>(base + c * 8), x1);
      unpack8(*reinterpret_cast<const uint4*>(base + half + c * 8), x2);
      const bool is_q = slot < n_heads;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        o1[u] = rbf(rbf(x1[u] * cs[u]) + rbf((-x2[u]) * sn[u]));
        o2[u] = rbf(rbf(x2[u] * cs[u]) + rbf(x1[u] * sn[u]));
        if (is_q && q_scale != 0.f) {   // qs = bf16(q * bf16(scale)) of the SDPA (base.py:305-373)
          o1[u] *= q_scale;
          o2[u] *= q_scale;
        }
      }
      uint4 w1, w2;
      w1.x = pack2(o1[0], o1[1]); w1.y = pack2(o1[2], o1[3]); w1.z = pack2(o1[4], o1[5]); w1.w = pack2(o1[6], o1[7]);
      w2.x = pack2(o2[0], o2[1]); w2.y = pack2(o2[2], o2[3]); w2.z = pack2(o2[4], o2[5]); w2.w = pack2(o2[6], o2[7]);
      if (is_q) {
        *reinterpret_cast<uint4*>(base + c * 8) = w1;
        *reinterpret_cast<uint4*>(base + half + c * 8) = w2;
      } else {
        const int kvh = slot - n_heads;
        if (loc.x >= 0) {   // (row -1: a padding token of a batched prefill)
          bf16* dst = kc + (long)loc.x * row_stride + ((long)kvh * cap + loc.y) * hd;
          *reinterpret_cast<uint4*>(dst + c * 8) = w1;
          *reinterpret_cast<uint4*>(dst + half + c * 8) = w2;
        }
        if (kws) {
          bf16* d2 = kws + ((long)kvh * T + t) * hd;
          *reinterpret_cast<uint4*>(d2 + c * 8) = w1;
          *reinterpret_cast<uint4*>(d2 + half + c * 8) = w2;
        }
      }
    } else {   // V head: copy into the cache, and transposed into V^T [kv head][dim][token]
      const int kvh = slot - n_heads - n_kv;
      for (int idx = threadIdx.x; idx < 32 * nv; idx += blockDim.x) {
        const int tl2 = idx / nv, c2 = idx % nv;
        const int t2 = t0 + tl2;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (t2 < T) {
          v = *reinterpret_cast<const uint4*>(qkv + (long)t2 * row_elems + (long)slot * hd + c2 * 8);
          const int2 l2 = tok_loc ? tok_loc[t2] : make_int2(0, ctx0 + t2);
          if (l2.x >= 0)
            *reinterpret_cast<uint4*>(vc + (long)l2.x * row_stride + ((long)kvh * cap + l2.y) * hd + c2 * 8) = v;
        }
        *reinterpret_cast<uint4*>(&tile[tl2][c2 * 8]) = v;
      }
      __syncthreads();
      if (vt) {
        for (int idx = threadIdx.x; idx < hd * 4; idx += blockDim.x) {
          const int d = idx >> 2, ch = idx & 3;
          if (t0 + ch * 8 >= t_ld) continue;
          unsigned short e[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) e[u] = __bfloat16_as_ushort(tile[ch * 8 + u][d]);
          uint4 o;
          o.x = e[0] | ((uint32_t)e[1] << 16); o.y = e[2] | ((uint32_t)e[3] << 16);
          o.z = e[4] | ((uint32_t)e[5] << 16); o.w = e[6] | ((uint32_t)e[7] << 16);
          *reinterpret_cast<uint4*>(vt + ((long)kvh * hd + d) * t_ld + t0 + ch * 8) = o;
        }
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------
// Qwen3-VL q_norm / k_norm (language.py:84-89) in place on the q and k heads of qkv (T, (n_heads + 2 n_kv) * hd),
// before mrope_kv_write rotates and appends them.  One warp per (token, q or k head).
template <int NU>
__global__ void __launch_bounds__(256) qk_norm_kernel(bf16* __restrict__ qkv, int T, int n_heads, int n_kv,
                                                      const bf16* __restrict__ qn, const bf16* __restrict__ kn,
                                                      float eps) {
  pdl_prologue();
  const int hd = 32 * NU, lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int qk = n_heads + n_kv;
  if (warp >= (long)T * qk) return;
  const int t = (int)(warp / qk), slot = (int)(warp % qk);
  bf16* base = qkv + (long)t * (qk + n_kv) * hd + (long)slot * hd;
  float x[NU];
#pragma unroll
  for (int u = 0; u < NU; ++u) x[u] = bf2f(base[lane + 32 * u]);
  warp_head_rms<NU>(x, slot < n_heads ? qn : kn, eps);
#pragma unroll
  for (int u = 0; u < NU; ++u) base[lane + 32 * u] = f2bf(x[u]);
}

int qk_norm(void* qkv, int T, int n_heads, int n_kv, int hd, const void* qn, const void* kn, float eps,
            cudaStream_t st) {
  B200_REQUIRE(T > 0 && qn && kn && (hd == 64 || hd == 128), "qk_norm: T=%d head_dim=%d (64 | 128)", T, hd);
  const long warps = (long)T * (n_heads + n_kv);
  const dim3 grid(cdiv(warps, 8));
  if (hd == 128)
    B200_CUDA(launch(qk_norm_kernel<4>, grid, dim3(256), 0, st, PDL_LAUNCH, (bf16*)qkv, T, n_heads, n_kv, (const bf16*)qn,
                         (const bf16*)kn, eps));
  else
    B200_CUDA(launch(qk_norm_kernel<2>, grid, dim3(256), 0, st, PDL_LAUNCH, (bf16*)qkv, T, n_heads, n_kv, (const bf16*)qn,
                         (const bf16*)kn, eps));
  return B200_OK;
}

// ---------------------------------------------------------------------------
__global__ void swiglu_kernel(const bf16* __restrict__ gu, bf16* __restrict__ out, int rows,
                              int inter) {
  const int nvec = inter >> 3;
  const long total = (long)rows * nvec;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % nvec);
    const long r = idx / nvec;
    float g[8], u[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(gu + r * 2 * inter + c * 8), g);
    unpack8(*reinterpret_cast<const uint4*>(gu + r * 2 * inter + inter + c * 8), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = swiglu_bf(g[j], u[j]);
    uint4 ov;
    ov.x = pack2(o[0], o[1]);
    ov.y = pack2(o[2], o[3]);
    ov.z = pack2(o[4], o[5]);
    ov.w = pack2(o[6], o[7]);
    *reinterpret_cast<uint4*>(out + r * inter + c * 8) = ov;
  }
}

// ---------------------------------------------------------------------------
// embed + merge (qwen2_vl.py:48,78-148).  grid = (CTAs per row, B).  Every CTA of a batch row computes
// the prefix count of image positions of that row with a block scan (each thread owns a contiguous chunk
// of ids, chunk totals are scanned with warp shuffles: integer, order-independent), then copies ITS share
// of the row's positions (16-byte vectors).  feature_start of row b = number of image positions in rows
// < b (counted redundantly by each CTA; B * T ids are a few KB).
__global__ void __launch_bounds__(512) embed_merge_kernel(const int* __restrict__ ids, int B, int T,
                                   const bf16* __restrict__ table, int hidden,
                                   const bf16* __restrict__ feats, int n_feats, int image_token,
                                   int video_token, bf16* __restrict__ out,
                                   int* __restrict__ src_out) {
  extern __shared__ int sh[];  // [T] src index per position
  __shared__ int s_any_image, s_start, s_warp[16];
  const int b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    s_any_image = 0;
    s_start = 0;
  }
  __syncthreads();
  // any image token anywhere? (reference: mx.sum(image_positions) == 0 -> video ids)
  int local = 0;
  for (int i = tid; i < B * T; i += blockDim.x) local |= (ids[i] == image_token);
  if (local) atomicOr(&s_any_image, 1);
  __syncthreads();
  const int tok = s_any_image ? image_token : video_token;
  // features consumed by earlier rows
  int cnt = 0;
  for (int i = tid; i < b * T; i += blockDim.x) cnt += (ids[i] == tok);
  if (cnt) atomicAdd(&s_start, cnt);
  // block scan of this row: thread i owns ids [i * per, (i + 1) * per)
  const int per = (T + blockDim.x - 1) / blockDim.x;
  const int t0 = min(tid * per, T), t1 = min(t0 + per, T);
  int mine = 0;
  for (int t = t0; t < t1; ++t) mine += (ids[b * T + t] == tok);
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int before = incl - mine;
  for (int w = 0; w < warp; ++w) before += s_warp[w];
  int run = s_start + before;
  for (int t = t0; t < t1; ++t) {
    const bool m = ids[b * T + t] == tok;
    sh[t] = m ? run : -1;
    run += m;
  }
  __syncthreads();
  const int nvec = hidden >> 3;
  const int rows_per = (T + gridDim.x - 1) / gridDim.x;
  const int r0 = min((int)blockIdx.x * rows_per, T), r1 = min(r0 + rows_per, T);
  for (long idx = tid; idx < (long)(r1 - r0) * nvec; idx += blockDim.x) {
    const int t = r0 + (int)(idx / nvec), c = (int)(idx % nvec);
    const int src = sh[t];
    const bf16* row;
    if (src >= 0) {
      row = feats + (long)min(src, max(n_feats - 1, 0)) * hidden;
    } else {
      row = table + (long)ids[b * T + t] * hidden;
    }
    *reinterpret_cast<uint4*>(out + ((long)b * T + t) * hidden + c * 8) =
        *reinterpret_cast<const uint4*>(row + c * 8);
  }
  if (src_out && blockIdx.x == 0)
    for (int t = tid; t < T; t += blockDim.x) src_out[b * T + t] = sh[t];
}

// ---------------------------------------------------------------------------
int cast_f32_bf16(const float* src, void* dst, long n, cudaStream_t st) {
  B200_REQUIRE(n >= 0, "cast: n<0");
  if (n == 0) return B200_OK;
  B200_REQUIRE(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 7) == 0, "cast: misaligned");
  B200_CUDA(launch(cast_f32_bf16_kernel, dim3(grid_for((n + 3) / 4, 256)), dim3(256), 0, st, PDL_LAUNCH, src, (bf16*)dst, n));
  return B200_OK;
}

int layer_norm(const void* x, const void* w, const void* b, void* y, int rows, int dim, float eps,
               cudaStream_t st) {
  B200_REQUIRE(rows > 0 && dim > 0 && (dim % 8) == 0, "layer_norm: rows=%d dim=%d", rows, dim);
  B200_CUDA(launch(layer_norm_kernel, dim3(cdiv(rows, 8)), dim3(256), 0, st, PDL_LAUNCH, (const bf16*)x, (const bf16*)w,
                       (const bf16*)b, (bf16*)y, rows, dim, eps));
  return B200_OK;
}

int rms_norm(const void* x, const void* w, void* y, int rows, int dim, float eps,
             cudaStream_t st) {
  B200_REQUIRE(rows > 0 && dim > 0 && (dim % 8) == 0 && w, "rms_norm: rows=%d dim=%d", rows, dim);
  B200_CUDA(launch(rms_norm_kernel, dim3(cdiv(rows, 8)), dim3(256), 0, st, PDL_LAUNCH, (const bf16*)x, (const bf16*)w,
                       (bf16*)y, rows, dim, eps));
  return B200_OK;
}

int vision_rope(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads,
                int hd, cudaStream_t st) {
  B200_REQUIRE(n_tok > 0 && n_heads > 0 && (hd % 4) == 0, "vision_rope: bad shape");
  const long total = (long)n_tok * 2 * n_heads * (hd / 2);
  vision_rope_kernel<<<grid_for(total, 256), 256, 0, st>>>((bf16*)qkv, pos_hw, inv_freq, n_tok,
                                                          n_heads, hd);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int mrope_kv_write(void* qkv, const int* pos3, const float* inv_freq, const int* axis_sel,
                   void* kc, void* vc, int T, int ctx0, int cap, int n_heads, int n_kv, int hd,
                   cudaStream_t st, float q_scale, void* vt, int t_ld, const KvRef* ref, int layer, void* kws,
                   const void* tok_loc, long row_stride) {
  B200_REQUIRE(T > 0 && ctx0 >= 0 && (ref || tok_loc || ctx0 + T <= cap), "mrope_kv_write: T=%d ctx0=%d cap=%d", T,
               ctx0, cap);
  B200_REQUIRE(!vt || t_ld >= T, "mrope_kv_write: V^T pitch %d < T %d", t_ld, T);
  if ((hd % 16) == 0 && hd <= 128 && (!vt || (t_ld % 8) == 0)) {
    const int slots = n_heads + 2 * n_kv, tiles = (T + 31) / 32;
    int groups = (4 * 132 + tiles - 1) / tiles;          // about four waves of CTAs
    if (groups > slots) groups = slots;
    if (groups < 1) groups = 1;
    const int per = (slots + groups - 1) / groups;
    B200_CUDA(launch(mrope_kv_write_tiled_kernel, dim3(tiles, (slots + per - 1) / per), dim3(256), 0, st, PDL_LAUNCH, (bf16*)qkv,
                         pos3, inv_freq, axis_sel, (bf16*)kc, (bf16*)vc, T, ctx0, cap, n_heads, n_kv, hd, q_scale, (bf16*)vt,
                         t_ld, ref, layer, (bf16*)kws, (const int2*)tok_loc, row_stride, per));
    return B200_OK;
  }
  const long total = (long)T * (n_heads + 2 * n_kv) * (hd / 2);
  B200_CUDA(launch(mrope_kv_write_kernel, dim3(grid_for(total, 256)), dim3(256), 0, st, PDL_LAUNCH, (bf16*)qkv, pos3, inv_freq,
                       axis_sel, (bf16*)kc, (bf16*)vc, T, ctx0, cap, n_heads, n_kv, hd, q_scale, (bf16*)vt, t_ld, ref,
                       layer, (bf16*)kws, (const int2*)tok_loc, row_stride));
  return B200_OK;
}

// ---------------------------------------------------------------------------
// Vision tower, after the qkv GEMM: 2-D rotary on q and k in place (same arithmetic as
// vision_rope_kernel), q pre-scaled for the SDPA (qs = bf16(q * bf16(scale))), and V written
// TRANSPOSED ([head][dim][token], tokens contiguous) through a shared-memory tile: the
// pipelined attention kernel loads Q, K and V^T with TMA and touches no operand with a thread.
// grid (ceil(T / 32), heads), 256 threads.
__global__ void vision_rope_table_kernel(const int* __restrict__ pos_hw, const float* __restrict__ inv_freq, int T,
                                        int half, float2* __restrict__ cs) {
  pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= T * half) return;
  const int t = idx / half, j = idx % half, quarter = half >> 1;
  const int axis = (j < quarter) ? 0 : 1;
  const float ang = (float)pos_hw[t * 2 + axis] * inv_freq[j - axis * quarter];
  cs[idx] = make_float2(cosf(ang), sinf(ang));
}

// `cs` (optional): cos / sin of every (token, rotary pair), computed once per tower call by
// vision_rope_table_kernel — the angles are the same for all heads and all 32 blocks.
__global__ void vision_qkv_post_kernel(bf16* __restrict__ qkv, const int* __restrict__ pos_hw,
                                       const float* __restrict__ inv_freq, int T, int n_heads, int hd,
                                       float scale_bf, bf16* __restrict__ vt, int t_ld,
                                       const float2* __restrict__ cs) {
  pdl_prologue();
  __shared__ bf16 tile[32][136];
  const int t0 = blockIdx.x * 32, h = blockIdx.y;
  const int half = hd >> 1, quarter = hd >> 2;
  const long row = 3L * n_heads * hd;
  if ((half & 7) == 0) {   // 8 rotary pairs per thread: two 16-byte loads, two 16-byte stores
    const int nc = half >> 3;
    for (int idx = threadIdx.x; idx < 32 * 2 * nc; idx += blockDim.x) {
      const int c = idx % nc, r = idx / nc;
      const int which = r & 1, t = t0 + (r >> 1);
      if (t >= T) continue;
      bf16* base = qkv + (long)t * row + ((long)which * n_heads + h) * hd;
      float x1[8], x2[8], o1[8], o2[8];
      unpack8(*reinterpret_cast<const uint4*>(base + c * 8), x1);
      unpack8(*reinterpret_cast<const uint4*>(base + half + c * 8), x2);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = c * 8 + u;
        float cv, sv;
        if (cs) {
          const float2 f = __ldg(cs + (long)t * half + j);
          cv = f.x;
          sv = f.y;
        } else {
          const int axis = (j < quarter) ? 0 : 1;
          const float ang = (float)pos_hw[t * 2 + axis] * inv_freq[j - axis * quarter];
          cv = cosf(ang);
          sv = sinf(ang);
        }
        o1[u] = rbf(__fadd_rn(__fmul_rn(x1[u], cv), __fmul_rn(-x2[u], sv)));
        o2[u] = rbf(__fadd_rn(__fmul_rn(x2[u], cv), __fmul_rn(x1[u], sv)));
        if (which == 0) {
          o1[u] *= scale_bf;
          o2[u] *= scale_bf;
        }
      }
      uint4 w1, w2;
      w1.x = pack2(o1[0], o1[1]); w1.y = pack2(o1[2], o1[3]); w1.z = pack2(o1[4], o1[5]); w1.w = pack2(o1[6], o1[7]);
      w2.x = pack2(o2[0], o2[1]); w2.y = pack2(o2[2], o2[3]); w2.z = pack2(o2[4], o2[5]); w2.w = pack2(o2[6], o2[7]);
      *reinterpret_cast<uint4*>(base + c * 8) = w1;
      *reinterpret_cast<uint4*>(base + half + c * 8) = w2;
    }
  } else {
    for (int idx = threadIdx.x; idx < 32 * 2 * half; idx += blockDim.x) {
      const int j = idx % half;
      const int r = idx / half;
      const int which = r & 1, t = t0 + (r >> 1);
      if (t >= T) continue;
      const int axis = (j < quarter) ? 0 : 1;
      const float ang = (float)pos_hw[t * 2 + axis] * inv_freq[j - axis * quarter];
      const float c = cosf(ang), sn = sinf(ang);
      bf16* base = qkv + (long)t * row + ((long)which * n_heads + h) * hd;
      const float x1 = bf2f(base[j]), x2 = bf2f(base[j + half]);
      float o1 = rbf(__fadd_rn(__fmul_rn(x1, c), __fmul_rn(-x2, sn)));
      float o2 = rbf(__fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, sn)));
      if (which == 0) {
        o1 *= scale_bf;
        o2 *= scale_bf;
      }
      base[j] = f2bf(o1);
      base[j + half] = f2bf(o2);
    }
  }
  const int nv = hd >> 3;
  for (int idx = threadIdx.x; idx < 32 * nv; idx += blockDim.x) {
    const int tl = idx / nv, c = idx % nv;
    const int t = t0 + tl;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (t < T) v = *reinterpret_cast<const uint4*>(qkv + (long)t * row + ((long)2 * n_heads + h) * hd + c * 8);
    *reinterpret_cast<uint4*>(&tile[tl][c * 8]) = v;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < hd * 4; idx += blockDim.x) {
    const int d = idx >> 2, ch = idx & 3;
    if (t0 + ch * 8 >= t_ld) continue;
    unsigned short e[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) e[u] = __bfloat16_as_ushort(tile[ch * 8 + u][d]);
    uint4 o;
    o.x = e[0] | ((uint32_t)e[1] << 16); o.y = e[2] | ((uint32_t)e[3] << 16);
    o.z = e[4] | ((uint32_t)e[5] << 16); o.w = e[6] | ((uint32_t)e[7] << 16);
    *reinterpret_cast<uint4*>(vt + ((long)h * hd + d) * t_ld + t0 + ch * 8) = o;
  }
}

int vision_rope_table(const int* pos_hw, const float* inv_freq, int n_tok, int hd, void* cs, cudaStream_t st) {
  B200_REQUIRE(n_tok > 0 && (hd % 4) == 0 && cs, "vision_rope_table: bad shape");
  const int total = n_tok * (hd / 2);
  B200_CUDA(launch(vision_rope_table_kernel, dim3(cdiv(total, 256)), dim3(256), 0, st, PDL_LAUNCH, pos_hw, inv_freq, n_tok, hd / 2,
                       (float2*)cs));
  return B200_OK;
}

int vision_qkv_post(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads, int hd,
                    float scale, void* vt, int t_ld, cudaStream_t st, const void* cs) {
  B200_REQUIRE(n_tok > 0 && n_heads > 0 && (hd % 8) == 0 && hd <= 128 && (t_ld % 8) == 0 && t_ld >= n_tok,
               "vision_qkv_post: bad shape (hd=%d t_ld=%d)", hd, t_ld);
  const float scale_bf = __bfloat162float(__float2bfloat16_rn(scale));
  B200_CUDA(launch(vision_qkv_post_kernel, dim3(cdiv(n_tok, 32), n_heads), dim3(256), 0, st, PDL_LAUNCH, (bf16*)qkv, pos_hw,
                       inv_freq, n_tok, n_heads, hd, scale_bf, (bf16*)vt, t_ld, (const float2*)cs));
  return B200_OK;
}

int swiglu(const void* gu, void* out, int rows, int inter, cudaStream_t st) {
  B200_REQUIRE(rows > 0 && inter > 0 && (inter % 8) == 0, "swiglu: bad shape");
  swiglu_kernel<<<grid_for((long)rows * (inter / 8), 256), 256, 0, st>>>((const bf16*)gu,
                                                                        (bf16*)out, rows, inter);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int embed_merge(const int* ids, int B, int T, const void* table, int hidden, const void* feats,
                int n_feats, int image_token, int video_token, void* out, int* src_out,
                cudaStream_t st) {
  B200_REQUIRE(B > 0 && T > 0 && (hidden % 8) == 0, "embed_merge: bad shape");
  B200_REQUIRE((long)T * 4 <= 200 * 1024, "embed_merge: T=%d too long", T);
  if ((size_t)T * 4 > 48 * 1024) {
    if (int rc = kernel_opt_in((const void*)embed_merge_kernel, T * 4, false)) return rc;
  }
  int per_row = (T + 7) / 8;  // >= 8 positions per CTA
  const int cap_ctas = (2 * 132 + B - 1) / B;
  if (per_row > cap_ctas) per_row = cap_ctas;
  embed_merge_kernel<<<dim3(per_row, B), 512, (size_t)T * 4, st>>>(ids, B, T, (const bf16*)table, hidden,
                                                   (const bf16*)feats, n_feats, image_token,
                                                   video_token, (bf16*)out, src_out);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200

using namespace b200;
extern "C" {
int b200_cast_f32_bf16(const float* s, void* d, long n, void* st) {
  return cast_f32_bf16(s, d, n, (cudaStream_t)st);
}
int b200_layer_norm(const void* x, const void* w, const void* b, void* y, int rows, int dim,
                    float eps, void* st) {
  return layer_norm(x, w, b, y, rows, dim, eps, (cudaStream_t)st);
}
int b200_rms_norm(const void* x, const void* w, void* y, int rows, int dim, float eps, void* st) {
  return rms_norm(x, w, y, rows, dim, eps, (cudaStream_t)st);
}
int b200_vision_rope(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads,
                     int hd, void* st) {
  return vision_rope(qkv, pos_hw, inv_freq, n_tok, n_heads, hd, (cudaStream_t)st);
}
int b200_mrope_kv_write(void* qkv, const int* pos3, const float* inv_freq, const int* axis_sel,
                        void* kc, void* vc, int T, int ctx0, int cap, int n_heads, int n_kv,
                        int hd, void* st) {
  return mrope_kv_write(qkv, pos3, inv_freq, axis_sel, kc, vc, T, ctx0, cap, n_heads, n_kv, hd,
                        (cudaStream_t)st, 0.f, nullptr, 0, nullptr, 0, nullptr, nullptr, 0);
}
int b200_qk_norm(void* qkv, int T, int n_heads, int n_kv, int hd, const void* q_norm_w, const void* k_norm_w,
                 float eps, void* st) {
  return qk_norm(qkv, T, n_heads, n_kv, hd, q_norm_w, k_norm_w, eps, (cudaStream_t)st);
}
int b200_vision_qkv_post(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads,
                         int hd, float scale, void* vt, int t_ld, void* st) {
  return vision_qkv_post(qkv, pos_hw, inv_freq, n_tok, n_heads, hd, scale, vt, t_ld, (cudaStream_t)st, nullptr);
}
int b200_swiglu(const void* gu, void* out, int rows, int inter, void* st) {
  return swiglu(gu, out, rows, inter, (cudaStream_t)st);
}
int b200_embed_merge(const int* ids, int B, int T, const void* table, int hidden,
                     const void* feats, int n_feats, int image_token, int video_token, void* out,
                     int* src_out, void* st) {
  return embed_merge(ids, B, T, table, hidden, feats, n_feats, image_token, video_token, out,
                     src_out, (cudaStream_t)st);
}
}
