// 8-bit KV cache kernels (format: kvq.cuh): k_kvq_quantize / k_kvq_dequantize, the bulk conversion between a
// bf16 pool and an 8-bit pool over the first n positions of every plane (KVCache.to_quantized,
// QuantizedKVCache.state).  The per-phase decode attention over an 8-bit pool is k_attn<AttnQ8> (decode.cu).
#include "decode.cuh"

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
  int rc = attn_prepare(d, cluster, true);
  if (rc) return rc;
  DecState h = {};
  h.ctx = ctx;
  DecState* st = nullptr;
  B200_CUDA(cudaMallocAsync((void**)&st, sizeof(DecState), s));
  B200_CUDA(cudaMemcpyAsync(st, &h, sizeof(DecState), cudaMemcpyHostToDevice, s));
  const AttnKv kv{(const bf16*)stage_k, (const bf16*)stage_v,
                  KvqPlanes{(uint8_t*)k_codes, (bf16*)k_scales, (bf16*)k_biases, group_size},
                  KvqPlanes{(uint8_t*)v_codes, (bf16*)v_scales, (bf16*)v_biases, group_size}};
  rc = launch_attn(d, (const bf16*)qbuf, kv, (bf16*)out, st, cluster, s);
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
