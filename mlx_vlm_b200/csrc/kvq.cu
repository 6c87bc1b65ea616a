// 8-bit KV cache kernels (format: kvq.cuh).
//
//   * k_kvq_quantize / k_kvq_dequantize: bulk conversion between a bf16 pool and an 8-bit pool over the
//     first n positions of every plane (KVCache.to_quantized, QuantizedKVCache.state).
//   * k_attn_q8: the batch-1 decode attention of the per-phase step over an 8-bit pool.  Same cluster
//     structure and rounding points as k_attn (decode.cu); K/V rows are dequantized on load, and the new
//     row, which the QKV kernel left in a bf16 staging plane, is quantized first so that the current token
//     attends to its own key and value in their quantized form (QuantizedKVCache.update_and_fetch
//     quantizes before it returns).
#include <cooperative_groups.h>

#include "kvq.cuh"

namespace cg = cooperative_groups;

namespace b200 {

// one warp per group; 8 groups per CTA.  Positions [pos0, pos0 + n) of every plane.  `back` (may alias src):
// the dequantized values are written there too (prefill over an 8-bit prefix attends to what the pool holds)
__global__ void __launch_bounds__(256) k_kvq_quantize(const bf16* src, int src_cap, KvqPlanes dst, int dst_cap,
                                                      long planes, int n, int hd, int pos0, bf16* back) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ng = hd / dst.gs, E = dst.gs >> 5;
  const long grp = (long)blockIdx.x * 8 + warp;
  if (grp >= planes * n * ng) return;
  const int g = (int)(grp % ng);
  const long pn = grp / ng;
  const int pos = pos0 + (int)(pn % n);
  const long plane = pn / n;
  const bf16* s = src + ((long)plane * src_cap + pos) * hd + g * dst.gs + lane * E;
  float w[4];
  #pragma unroll
  for (int e = 0; e < 4; ++e) if (e < E) w[e] = bf2f(s[e]);
  uint32_t code[4];
  float scale, bias;
  kvq_quantize_group(w, E, code, &scale, &bias);
  uint8_t* c = dst.codes + ((long)plane * dst_cap + pos) * hd + g * dst.gs + lane * E;
  #pragma unroll
  for (int e = 0; e < 4; ++e) if (e < E) c[e] = (uint8_t)code[e];
  if (lane == 0) {
    const long si = ((long)plane * dst_cap + pos) * ng + g;
    dst.scales[si] = f2bf(scale);
    dst.biases[si] = f2bf(bias);
  }
  if (back) {
    const float sb = rbf(scale), bb = rbf(bias);
    bf16* o = back + ((long)plane * src_cap + pos) * hd + g * dst.gs + lane * E;
#pragma unroll
    for (int e = 0; e < 4; ++e) if (e < E) o[e] = f2bf(kvq_dequant(code[e], sb, bb));
  }
}

int kvq_quantize_rows(bf16* src, int cap, const KvqPlanes& dst, int dst_cap, long planes, int pos0, int n, int hd,
                      bool writeback, cudaStream_t s) {
  const long groups = planes * n * (hd / dst.gs);
  if (groups == 0) return B200_OK;
  k_kvq_quantize<<<(unsigned)((groups + 7) / 8), 256, 0, s>>>(src, cap, dst, dst_cap, planes, n, hd, pos0,
                                                                writeback ? src : nullptr);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// one thread per 4 elements (one code word)
__global__ void __launch_bounds__(256) k_kvq_dequantize(KvqPlanes src, int src_cap, bf16* __restrict__ dst,
                                                        int dst_cap, long planes, int n, int hd) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int w4 = hd >> 2;
  if (i >= planes * n * w4) return;
  const int c4 = (int)(i % w4);
  const long pn = i / w4;
  const int pos = (int)(pn % n);
  const long plane = pn / n;
  const int ng = hd / src.gs;
  const uint32_t code = *reinterpret_cast<const uint32_t*>(src.codes + ((long)plane * src_cap + pos) * hd + c4 * 4);
  const long si = ((long)plane * src_cap + pos) * ng + (c4 * 4) / src.gs;
  const float sc = bf2f(src.scales[si]), bi = bf2f(src.biases[si]);
  bf16* o = dst + ((long)plane * dst_cap + pos) * hd + c4 * 4;
  for (int j = 0; j < 4; ++j) o[j] = f2bf(kvq_dequant((code >> (8 * j)) & 0xffu, sc, bi));
}

constexpr int AQ_MAXG = 8;   // q heads per CTA
constexpr int AQ_MAXCL = 8;  // cluster size

static size_t attn_q8_smem(const DecodeDims& d, int chunk_cap) {
  return ((size_t)AQ_MAXG * chunk_cap + (size_t)AQ_MAXCL * AQ_MAXG * 2 + (size_t)AQ_MAXCL * AQ_MAXG * d.hd +
          (size_t)8 * AQ_MAXG * d.hd + 2 * (size_t)d.hd) * 4;
}

// EPL (2 or 4) dequantized elements of position `pos` of one kv head plane, dims [lane*EPL, lane*EPL+EPL)
__device__ __forceinline__ void kvq_load_row(const KvqPlanes& P, long row, int ng, int lane, int EPL, float* f) {
  const uint8_t* c = P.codes + row * (long)(ng * P.gs) + lane * EPL;
  const uint32_t code = (EPL == 4) ? *reinterpret_cast<const uint32_t*>(c)
                                   : (uint32_t)*reinterpret_cast<const uint16_t*>(c);
  const long si = row * ng + (lane * EPL) / P.gs;
  const float sc = bf2f(P.scales[si]), bi = bf2f(P.biases[si]);
#pragma unroll
  for (int e = 0; e < 4; ++e) f[e] = (e < EPL) ? kvq_dequant((code >> (8 * e)) & 0xffu, sc, bi) : 0.f;
}

__global__ void __launch_bounds__(256) k_attn_q8(const DecodeDims d, const bf16* __restrict__ qbuf, const KvqPlanes K,
                                                 const KvqPlanes V, const bf16* __restrict__ stage_k,
                                                 const bf16* __restrict__ stage_v, bf16* __restrict__ out,
                                                 const DecState* __restrict__ st, int chunk_cap, int hsplit) {
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) uint8_t sm[];
  const int Gall = d.n_heads / d.n_kv;
  const int G = Gall / hsplit;
  const int hd = d.hd;
  const int EPL = hd >> 5;
  const int ng = hd / K.gs;
  float* sc = reinterpret_cast<float*>(sm);               // [G][chunk_cap]
  float* stats = sc + (long)AQ_MAXG * chunk_cap;          // [CL][G][2]
  float* part = stats + AQ_MAXCL * AQ_MAXG * 2;           // [CL][G*hd]
  float* red = part + (long)AQ_MAXCL * AQ_MAXG * hd;      // [8][G*hd]
  float* newrow = red + (long)8 * AQ_MAXG * hd;           // [2][hd]: the new K and V row, dequantized
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kvh = blockIdx.y / hsplit;
  const int h0 = kvh * Gall + (blockIdx.y % hsplit) * G;
  const int ctx = st->ctx;
  const int nkeys = ctx + 1;
  const long row0 = (long)kvh * d.cap;   // position 0 of this kv head

  // ---- the new row: warp w < 2 * ng quantizes group w % ng of K (w < ng) or V; one CTA stores it ----
  if (warp < 2 * ng) {
    const int side = warp / ng, g = warp % ng, E = K.gs >> 5;
    const bf16* s = (side ? stage_v : stage_k) + (row0 + ctx) * hd + g * K.gs + lane * E;
    float w[4];
    #pragma unroll
    for (int e = 0; e < 4; ++e) if (e < E) w[e] = bf2f(s[e]);
    uint32_t code[4];
    float scale, bias;
    kvq_quantize_group(w, E, code, &scale, &bias);
    const float sb = rbf(scale), bb = rbf(bias);
    #pragma unroll
    for (int e = 0; e < 4; ++e) if (e < E)
        newrow[side * hd + g * K.gs + lane * E + e] = kvq_dequant(code[e], sb, bb);
    if (rank == 0 && (blockIdx.y % hsplit) == 0) {
      const KvqPlanes& P = side ? V : K;
      uint8_t* c = P.codes + (row0 + ctx) * hd + g * K.gs + lane * E;
      #pragma unroll
      for (int e = 0; e < 4; ++e) if (e < E) c[e] = (uint8_t)code[e];
      if (lane == 0) {
        P.scales[(row0 + ctx) * ng + g] = f2bf(scale);
        P.biases[(row0 + ctx) * ng + g] = f2bf(bias);
      }
    }
  }
  __syncthreads();

  const int chunk = (nkeys + CL - 1) / CL;
  const int k0 = min(nkeys, rank * chunk), k1 = min(nkeys, k0 + chunk);
  const int nloc = k1 - k0;
  float qs[AQ_MAXG][4];
#pragma unroll
  for (int g = 0; g < AQ_MAXG; ++g) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      qs[g][e] = 0.f;
      if (g < G && e < EPL) qs[g][e] = rbf(bf2f(qbuf[(long)(h0 + g) * hd + lane * EPL + e]) * d.scale_bf);
    }
  }
  // ---- scores (rounded to bf16) ----
  for (int j = warp; j < nloc; j += 8) {
    const int pos = k0 + j;
    float kf[4];
    if (pos == ctx) {
#pragma unroll
      for (int e = 0; e < 4; ++e) kf[e] = (e < EPL) ? newrow[lane * EPL + e] : 0.f;
    } else {
      kvq_load_row(K, row0 + pos, ng, lane, EPL, kf);
    }
    float s[AQ_MAXG];
#pragma unroll
    for (int g = 0; g < AQ_MAXG; ++g)
      s[g] = (g < G) ? qs[g][0] * kf[0] + qs[g][1] * kf[1] + qs[g][2] * kf[2] + qs[g][3] * kf[3] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int g = 0; g < AQ_MAXG; ++g)
        if (g < G) s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
    if (lane == 0) {
#pragma unroll
      for (int g = 0; g < AQ_MAXG; ++g)
        if (g < G) sc[(long)g * chunk_cap + j] = rbf(s[g]);
    }
  }
  __syncthreads();
  // ---- local max / sum(exp) per head (warp g), pushed to every rank ----
  if (warp < G) {
    float m = -INFINITY;
    for (int j = lane; j < nloc; j += 32) m = fmaxf(m, sc[(long)warp * chunk_cap + j]);
    m = warp_max(m);
    float l = 0.f;
    for (int j = lane; j < nloc; j += 32) l += expf(sc[(long)warp * chunk_cap + j] - m);
    l = warp_sum(l);
    if (nloc == 0) l = 0.f;
    if (lane < CL) {
      float* dst = cluster.map_shared_rank(stats, lane) + ((long)rank * AQ_MAXG + warp) * 2;
      dst[0] = m;
      dst[1] = l;
    }
  }
  cluster.sync();
  // ---- p = bf16(exp(s - M) / L) ----
  if (warp < G) {
    float M = -INFINITY;
    for (int r = 0; r < CL; ++r) M = fmaxf(M, stats[((long)r * AQ_MAXG + warp) * 2]);
    float Ltot = 0.f;
    for (int r = 0; r < CL; ++r) {
      const float mr = stats[((long)r * AQ_MAXG + warp) * 2];
      const float lr = stats[((long)r * AQ_MAXG + warp) * 2 + 1];
      if (lr > 0.f) Ltot += lr * expf(mr - M);
    }
    for (int j = lane; j < nloc; j += 32) {
      float* p = &sc[(long)warp * chunk_cap + j];
      *p = rbf(expf(*p - M) / Ltot);
    }
  }
  __syncthreads();
  // ---- partial output: warp w takes keys w, w+8, ... ; lane owns EPL dims ----
  float acc[AQ_MAXG][4];
#pragma unroll
  for (int g = 0; g < AQ_MAXG; ++g)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[g][e] = 0.f;
  for (int j = warp; j < nloc; j += 8) {
    const int pos = k0 + j;
    float vf[4];
    if (pos == ctx) {
#pragma unroll
      for (int e = 0; e < 4; ++e) vf[e] = (e < EPL) ? newrow[hd + lane * EPL + e] : 0.f;
    } else {
      kvq_load_row(V, row0 + pos, ng, lane, EPL, vf);
    }
#pragma unroll
    for (int g = 0; g < AQ_MAXG; ++g) {
      if (g < G) {
        const float p = sc[(long)g * chunk_cap + j];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[g][e] = fmaf(p, vf[e], acc[g][e]);
      }
    }
  }
#pragma unroll
  for (int g = 0; g < AQ_MAXG; ++g)
    if (g < G)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (e < EPL) red[((long)warp * G + g) * hd + lane * EPL + e] = acc[g][e];
  __syncthreads();
  float* part0 = cluster.map_shared_rank(part, 0) + (long)rank * AQ_MAXG * hd;
  for (int i = threadIdx.x; i < G * hd; i += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[(long)w * G * hd + i];
    part0[i] = s;
  }
  cluster.sync();
  if (rank == 0) {
    for (int i = threadIdx.x; i < G * hd; i += blockDim.x) {
      float s = 0.f;
      for (int r = 0; r < CL; ++r) s += part[(long)r * AQ_MAXG * hd + i];
      out[(long)h0 * hd + i] = f2bf(s);
    }
  }
}

static int attn_q8_hsplit(const DecodeDims& d) {
  const int G = d.n_heads / d.n_kv;
  int hs = 1;
  while (G / hs > AQ_MAXG || (G % hs) != 0) ++hs;
  if (hs == 1 && G % 2 == 0 && G >= 4) hs = 2;
  return hs;
}

int kvq_decode_prepare(const DecodeDims& d, int cluster) {
  const size_t smem = attn_q8_smem(d, cdiv(d.cap, cluster));
  B200_REQUIRE(smem <= 220 * 1024, "8-bit decode attention: cache capacity %d too large", d.cap);
  B200_CUDA(cudaFuncSetAttribute(k_attn_q8, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B200_CUDA(cudaFuncSetAttribute(k_attn_q8, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 cudaSharedmemCarveoutMaxShared));
  return B200_OK;
}

int launch_attn_q8(const DecodeDims& d, const bf16* qbuf, const KvqPlanes& kc8, const KvqPlanes& vc8,
                   const bf16* stage_k, const bf16* stage_v, bf16* out, const DecState* st, int cluster,
                   cudaStream_t s) {
  B200_REQUIRE(d.hd == 64 || d.hd == 128, "8-bit decode attention: head_dim=%d (64|128)", d.hd);
  B200_REQUIRE(kc8.gs == 32 || kc8.gs == 64 || kc8.gs == 128, "8-bit decode attention: group size %d", kc8.gs);
  B200_REQUIRE(d.hd % kc8.gs == 0, "8-bit decode attention: group size %d does not divide head_dim %d", kc8.gs,
               d.hd);
  B200_REQUIRE(cluster >= 1 && cluster <= AQ_MAXCL, "8-bit decode attention: cluster %d", cluster);
  const int hs = attn_q8_hsplit(d);
  const int chunk_cap = cdiv(d.cap, cluster);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cluster, d.n_kv * hs, 1);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = attn_q8_smem(d, chunk_cap);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  B200_CUDA(cudaLaunchKernelEx(&cfg, k_attn_q8, d, qbuf, kc8, vc8, stage_k, stage_v, out, st, chunk_cap, hs));
  return B200_OK;
}

}  // namespace b200

using namespace b200;

static int kvq_check(int hd, int gs) {
  B200_REQUIRE((gs == 32 || gs == 64 || gs == 128) && hd > 0 && hd % gs == 0,
               "kvq: group size %d must be 32, 64 or 128 and divide head_dim %d", gs, hd);
  return B200_OK;
}

int b200_kvq_quantize(const void* src, int src_cap, void* codes, void* scales, void* biases, int dst_cap,
                      long planes, int n_tokens, int hd, int group_size, void* stream) {
  B200_REQUIRE(src && codes && scales && biases && planes >= 0 && n_tokens >= 0 && n_tokens <= src_cap &&
                   n_tokens <= dst_cap,
               "kvq_quantize: bad arguments");
  int rc = kvq_check(hd, group_size);
  if (rc) return rc;
  const long groups = planes * n_tokens * (hd / group_size);
  if (groups == 0) return B200_OK;
  const KvqPlanes dst{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  k_kvq_quantize<<<(unsigned)((groups + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const bf16*)src, src_cap, dst,
                                                                                   dst_cap, planes, n_tokens, hd, 0,
                                                                                   nullptr);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_kvq_dequantize(const void* codes, const void* scales, const void* biases, int src_cap, void* dst,
                        int dst_cap, long planes, int n_tokens, int hd, int group_size, void* stream) {
  B200_REQUIRE(dst && codes && scales && biases && planes >= 0 && n_tokens >= 0 && n_tokens <= src_cap &&
                   n_tokens <= dst_cap && ((uintptr_t)codes & 3) == 0,
               "kvq_dequantize: bad arguments");
  int rc = kvq_check(hd, group_size);
  if (rc) return rc;
  const long words = planes * n_tokens * (hd / 4);
  if (words == 0) return B200_OK;
  const KvqPlanes src{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  k_kvq_dequantize<<<(unsigned)((words + 255) / 256), 256, 0, (cudaStream_t)stream>>>(src, src_cap, (bf16*)dst,
                                                                                      dst_cap, planes, n_tokens, hd);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

/* one 8-bit decode attention step outside the engine (tests): st->ctx = ctx */
int b200_kvq_decode_attention(const void* qbuf, void* k_codes, void* k_scales, void* k_biases, void* v_codes,
                              void* v_scales, void* v_biases, const void* stage_k, const void* stage_v, void* out,
                              int n_heads, int n_kv, int head_dim, int cap, int ctx, int group_size, int cluster,
                              void* stream) {
  B200_REQUIRE(qbuf && k_codes && k_scales && k_biases && v_codes && v_scales && v_biases && stage_k && stage_v && out &&
                   n_kv > 0 && n_heads % n_kv == 0 && ctx >= 0 && ctx < cap,
               "kvq_decode_attention: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  DecodeDims d = {};
  d.n_heads = n_heads; d.n_kv = n_kv; d.hd = head_dim; d.cap = cap;
  d.scale_bf = __bfloat162float(__float2bfloat16_rn(1.0f / sqrtf((float)head_dim)));
  int rc = kvq_decode_prepare(d, cluster);
  if (rc) return rc;
  DecState h = {};
  h.ctx = ctx;
  DecState* st = nullptr;
  B200_CUDA(cudaMallocAsync((void**)&st, sizeof(DecState), s));
  B200_CUDA(cudaMemcpyAsync(st, &h, sizeof(DecState), cudaMemcpyHostToDevice, s));
  const KvqPlanes K{(uint8_t*)k_codes, (bf16*)k_scales, (bf16*)k_biases, group_size};
  const KvqPlanes V{(uint8_t*)v_codes, (bf16*)v_scales, (bf16*)v_biases, group_size};
  rc = launch_attn_q8(d, (const bf16*)qbuf, K, V, (const bf16*)stage_k, (const bf16*)stage_v, (bf16*)out, st,
                      cluster, s);
  B200_CUDA(cudaFreeAsync(st, s));
  if (rc) return rc;
  return cudaStreamSynchronize(s) == cudaSuccess ? B200_OK : cuda_fail(cudaGetLastError(), "kvq_decode_attention",
                                                                         __FILE__, __LINE__);
}

/* one 8-bit lock-step attention (the Q8 variant of bd_attn_kernel) on caller buffers; see include/b200vlm.h */
int b200_batch_kvq_attention(const float* qkv, const void* bias, const float* inv_freq, const int* ctx, const int* pos,
                             void* codes, void* scales, void* biases, int group_size, int pool_rows, int cap, void* out,
                             int B, int n_heads, int n_kv, int head_dim, const void* q_norm, const void* k_norm, float eps,
                             void* stream) {
  B200_REQUIRE(qkv && bias && inv_freq && ctx && pos && codes && scales && biases && out && ((uintptr_t)codes & 15) == 0,
               "batch_kvq_attention: bad arguments");
  int dev = 0, sms = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return batch_kvq_attention(qkv, (const bf16*)bias, inv_freq, ctx, pos, (uint8_t*)codes, (bf16*)scales, (bf16*)biases,
                             group_size, pool_rows, cap, (bf16*)out, B, n_heads, n_kv, head_dim, (const bf16*)q_norm,
                             (const bf16*)k_norm, eps, sms, (cudaStream_t)stream);
}

/* row copy of any per-position plane set (bf16 K/V, 8-bit codes, scales or biases): byte-exact */
int b200_pool_copy_row(void* dst_pool, int dst_batch, int dst_cap, int dst_row, const void* src_pool, int src_batch,
                       int src_cap, int src_row, int n_layers, int n_kv, int bytes_per_position, int n_tokens,
                       void* stream) {
  B200_REQUIRE(dst_pool && src_pool && dst_row >= 0 && dst_row < dst_batch && src_row >= 0 && src_row < src_batch &&
                   n_tokens >= 0 && n_tokens <= dst_cap && n_tokens <= src_cap && bytes_per_position > 0,
               "pool_copy_row: bad arguments");
  if (n_tokens == 0) return B200_OK;
  const size_t bp = (size_t)bytes_per_position, w = (size_t)n_tokens * bp;
  for (int l = 0; l < n_layers; ++l)
    for (int kv = 0; kv < 2; ++kv) {
      const char* sp = (const char*)src_pool + ((((size_t)l * 2 + kv) * src_batch + src_row) * n_kv) * (size_t)src_cap * bp;
      char* dp = (char*)dst_pool + ((((size_t)l * 2 + kv) * dst_batch + dst_row) * n_kv) * (size_t)dst_cap * bp;
      B200_CUDA(cudaMemcpy2DAsync(dp, (size_t)dst_cap * bp, sp, (size_t)src_cap * bp, w, n_kv, cudaMemcpyDeviceToDevice,
                                  (cudaStream_t)stream));
    }
  return B200_OK;
}
