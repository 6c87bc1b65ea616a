/*
 * b200vlm — C ABI of the H100-native generate path (libb200vlm.so).
 *
 * The reference (Blaizzy/mlx-vlm) has NO FFI: its hot path is Python calling the
 * third-party `mlx` array library.  This header is the boundary a maintainer
 * would bind instead of `mlx`: every entry point names the reference call site
 * (file:line under /root/reference/mlx_vlm) whose arithmetic it replaces.
 *
 * Conventions
 *   - plain pointers + sizes only; all data pointers are DEVICE pointers unless
 *     the name ends in `_host`.  Activations / weights are bf16 (uint16 storage),
 *     indices are int32, pixel values float32.
 *   - every call enqueues on the caller-supplied `stream` (a cudaStream_t cast to
 *     void*; NULL = legacy default stream) and returns without synchronising
 *     unless stated otherwise.
 *   - return value: B200_OK or an error code; b200_last_error() returns a
 *     thread-local message.  Nothing throws across the boundary.
 *   - an engine is not thread-safe (mirrors the reference's single GPU thread,
 *     server/generation.py:1044-1051); the caller owns every buffer it passes in
 *     (weights, workspace, KV pool stay referenced until engine destroy).
 */
#ifndef B200VLM_H
#define B200VLM_H

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID 1     /* bad argument / unsupported shape            */
#define B200_ERR_CUDA 2        /* a CUDA runtime / driver call failed         */
#define B200_ERR_UNSUPPORTED 3 /* device is not sm_90 (Hopper)                */
#define B200_ERR_STATE 4       /* engine used before weights / cache bound    */

#define B200_ABI_VERSION 2

const char* b200_last_error(void);
int b200_abi_version(void);
/* Fails with B200_ERR_UNSUPPORTED unless `device` is compute capability 10.x. */
int b200_device_check(int device, int* sm_count);

/* ------------------------------------------------------------------------- */
/* Op level (each is one kernel launch; used directly by the kernel tests)    */
/* ------------------------------------------------------------------------- */

/* qwen2_vl.py:44-45  pixel_values.astype(weight dtype) */
int b200_cast_f32_bf16(const float* src, void* dst, long n, void* stream);

/* gemm_wt output modes / finish_rows normalisation kinds */
#define B200_WT_BF16 0    /* C[t][n] = epi(bf16(acc + bias)) (+ residual), bf16            */
#define B200_WT_PARTIAL 1 /* fp32 split-K partial tiles P[split][t][n] (finish_rows adds them) */
#define B200_WT_SWIGLU 2  /* W = [gate rows; up rows]: C[t][i] = silu(gate) * up, bf16     */
#define B200_WT_F32 3     /* fp32 output (bias, fp32 activation, fp32 residual): fp32 towers  */
#define B200_WT_SPLIT 4   /* fp32 result written as [hi | lo] bf16 halves (next GEMM's operand) */
#define B200_NORM_NONE 0
#define B200_NORM_RMS 1   /* mx.fast.rms_norm   (language.py:139-140)                      */
#define B200_NORM_LN 2    /* mx.fast.layer_norm (vision.py:180-181)                        */

/* epilogues of b200_gemm_wt */
#define B200_EPI_NONE 0
#define B200_EPI_GELU_FAST 1  /* nn.GELU(approx="fast")  vision.py:167          */
#define B200_EPI_GELU_EXACT 2 /* nn.GELU()               vision.py:112          */
#define B200_EPI_GELU_TANH 3  /* nn.GELU(approx="precise") (fp32 towers only)   */

/* nn.Linear / nn.Conv3d(kernel==stride) / Embedding.as_linear, weight-major (gemm_wt.cu): Hopper tensor
 * cores (wgmma), TMA-fed, fp32 accumulate in registers; weight rows on the wgmma M side, TN tokens (16..256)
 * on the N side, optional split-K.  Replaces every nn.Linear in models/qwen2_vl/{vision,language}.py and
 * PatchEmbed.proj (vision.py:83-102).  mode B200_WT_BF16: C[T,N] = epi( bf16( X[T,K] . W[N,K]^T + bias[N] ) )
 * then, if residual, C = bf16(residual + C); row pitches ldx / ldc / ldr in elements (K and ldx multiples of 8).
 * B200_WT_PARTIAL: fp32 tiles partial[split][T][N] (bias / residual applied by
 * b200_finish_rows); B200_WT_SWIGLU: W = [gate; up] (N == 2*inter), C[T][inter] =
 * swiglu (mlp.py:9-15, activations.py:8-10).  cfg4 = {TN, k-blocks per stage, stages,
 * splits} or NULL / {0} for the automatic choice.  flags: debugging aids, pass 0. */
int b200_gemm_wt(const void* X, long ldx, const void* W, const void* bias, const void* residual,
                 long ldr, void* C, long ldc, float* partial, int T, int N, int K, int epilogue,
                 int mode, int inter, const int* cfg4, unsigned flags, void* stream);
int b200_gemm_wt_auto_config(int T, int N, int K, int mode, int inter, int* cfg4_out);
/* h[t] = bf16(resid[t] + bf16(sum_s partial[s][t] + bias)), and xn[t] = the RMSNorm /
 * LayerNorm of h[t] that the next block applies (language.py:139-148, vision.py:177-194):
 * the split-K reduction, the residual add and the norm in ONE pass over the row. */
int b200_finish_rows(const float* partial, int splits, const void* bias, const void* resid, long ldr,
                     void* h_out, long ldh, int norm_kind, const void* norm_w, const void* norm_b,
                     float eps, void* xn, long ldx, int T, int N, void* stream);

/* mx.fast.layer_norm (vision.py:180-181,108) / mx.fast.rms_norm (language.py:128-131) */
int b200_layer_norm(const void* x, const void* w, const void* b, void* y,
                    int rows, int dim, float eps, void* stream);
int b200_rms_norm(const void* x, const void* w, void* y, int rows, int dim,
                  float eps, void* stream);

/* apply_rotary_pos_emb_vision (vision.py:35-50) in place on the q and k thirds of
 * qkv (n_tok, 3, n_heads, head_dim).  pos_hw (n_tok,2) int32 = rot_pos_emb ids
 * (vision.py:219-249); inv_freq (head_dim/4) fp32. */
int b200_vision_rope(void* qkv, const int* pos_hw, const float* inv_freq,
                     int n_tok, int n_heads, int head_dim, void* stream);

/* apply_multimodal_rotary_pos_emb(style="chunked") (rope_utils.py:1456-1504,
 * 1227-1241) on q (in place) and k, then KVCache.update_and_fetch's append
 * (cache.py:345-367): k (rotated) and v rows go to kcache/vcache
 * [(n_kv, cap, head_dim)] at token index ctx0 + t.
 * qkv: (T, (n_heads + 2 n_kv) * head_dim); pos3: (3, T) int32;
 * inv_freq (head_dim/2) fp32; axis_sel (head_dim/2) int32 in {0,1,2}. */
int b200_mrope_kv_write(void* qkv, const int* pos3, const float* inv_freq,
                        const int* axis_sel, void* kcache, void* vcache,
                        int T, int ctx0, int cap, int n_heads, int n_kv,
                        int head_dim, void* stream);

/* Qwen3-VL Attention.q_norm / k_norm (qwen3_vl/language.py:59-60,84-89): mx.fast.rms_norm over each q and k head of
 * qkv (T, (n_heads + 2 n_kv) * head_dim) in place, weights (head_dim) bf16; the v heads are left alone.  Runs
 * before b200_mrope_kv_write.  head_dim 64 or 128. */
int b200_qk_norm(void* qkv, int T, int n_heads, int n_kv, int head_dim, const void* q_norm_w, const void* k_norm_w,
                 float eps, void* stream);

/* mx.fast.scaled_dot_product_attention as executed on the mlx CPU device
 * (fallback graph; base.py:366-373, vision.py:154): q*scale, scores, softmax and
 * output each rounded to bf16.  Strides in elements.  causal!=0: bottom-right
 * aligned (key j visible to query i iff j <= S - Lq + i).  scale is rounded to
 * bf16 inside. */
int b200_attention(const void* q, long q_tok_stride, long q_head_stride,
                   const void* k, long k_tok_stride, long k_head_stride,
                   const void* v, long v_tok_stride, long v_head_stride,
                   void* out, long out_tok_stride,
                   int n_heads, int n_kv, int head_dim, int Lq, int S,
                   int causal, float scale, void* stream);

/* swiglu (activations.py:8-10): out[r,i] = silu(gu[r,i]) * gu[r,I+i] */
/* Pipelined SDPA (attention_fa.cu): same arithmetic as b200_attention, operands TMA-loaded.
 * q must be PRE-SCALED (bf16(q * bf16(scale)): b200_vision_qkv_post / the engine's M-RoPE
 * kernel do it); vt = V transposed, element (kv head, dim, key) at vt + kvh*vt_hs + d*vt_ds + key. */
int b200_attention_fa(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                      const void* vt, long vt_hs, long vt_ds, void* out, long o_ts, int n_heads,
                      int n_kv, int hd, int Lq, int S, int causal, void* stream);
/* vision tower after the qkv GEMM: 2-D rotary on q,k in place (vision.py:35-50), q pre-scaled
 * by bf16(scale), V^T written to vt[head][dim][t_ld] (t_ld % 8 == 0, >= n_tok) */
int b200_vision_qkv_post(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads,
                         int hd, float scale, void* vt, int t_ld, void* stream);

int b200_swiglu(const void* gate_up, void* out, int rows, int inter, void* stream);

/* embed_tokens + merge_input_ids_with_image_features (qwen2_vl.py:48,78-148) for
 * B rows of T ids: out[b,t] = feats[start_b + cumsum(mask_b)[t]-1] where
 * ids==image_token (or ==video_token when no image token is present anywhere),
 * else table[ids[b,t]].  src_index_out (B*T int32, may be NULL) receives the
 * feature row used (or -1).  Count validation is done by the host caller. */
int b200_embed_merge(const int* ids, int B, int T, const void* table, int hidden,
                     const void* feats, int n_feats, int image_token, int video_token,
                     void* out, int* src_index_out, void* stream);

/* ------------------------------------------------------------------------- */
/* Engine level (Qwen2-VL): whole-tower / whole-step calls                     */
/* ------------------------------------------------------------------------- */
typedef struct b200_engine b200_engine;

typedef struct {
  /* text (language.py TextConfig) */
  int hidden, n_layers, inter, n_heads, n_kv_heads, head_dim, vocab;
  float rms_eps, rope_theta;
  int mrope_section[3];
  int tie_embeddings;
  /* vision (config.py:9-23) */
  int v_depth, v_embed, v_heads, v_mlp, v_patch_dim, v_merge, v_out;
  float v_ln_eps;
  int external_vision; /* 1: the engine holds the language model only (LLaVA / Idefics2: their fp32 towers
                          run through the tower ops); no v.* weights are required */
} b200_qwen2vl_config;

int b200_engine_create(const b200_qwen2vl_config* cfg, int device, b200_engine** out);
int b200_engine_destroy(b200_engine* e);

/* Weight registration by name (packed names, see DESIGN.md §layout):
 *   v.patch_embed.w | v.blk.<i>.{ln1.w,ln1.b,ln2.w,ln2.b,qkv.w,qkv.b,proj.w,proj.b,
 *   fc1.w,fc1.b,fc2.w,fc2.b} | v.merger.{ln.w,ln.b,fc1.w,fc1.b,fc2.w,fc2.b} |
 *   lm.embed | lm.head (untied only) | lm.norm | lm.<i>.{ln1,ln2,wqkv,bqkv,wo,wgu,wd}
 *   | lm.<i>.{qn,kn} (head_dim each: Qwen3-VL's q_norm / k_norm, qwen3_vl/language.py:59-60; set for every
 *   layer or for none.  With them every path that writes K normalises q and k per head before the rotary,
 *   the persistent k_mega kernel included) */
int b200_engine_set_weight(b200_engine* e, const char* name, const void* ptr, long n_elems);
/* scratch for activations; must be >= b200_engine_workspace_bytes(max tokens) */
long b200_engine_workspace_bytes(const b200_engine* e, int max_tokens, int max_patches);
int b200_engine_set_workspace(b200_engine* e, void* ptr, long bytes);
/* KV pool laid out (n_layers, 2, batch, n_kv, cap, head_dim) bf16 — per layer the
 * reference KVCache layout (B, n_kv_heads, S, head_dim), cache.py:345-367.
 * Every bind (this one, b200_engine_bind_kvq, b200_engine_bind_batch_kvq) replaces the previous binding, switches
 * a prefill write-through off and, when the new pool has no row b200_engine_set_kv_row selected, selects row 0. */
int b200_engine_bind_kv(b200_engine* e, void* pool, int batch, int cap);
/* 8-bit KV pool (kv_bits=8; format in csrc/kvq.cuh): codes (n_layers, 2, batch, n_kv, cap, head_dim) uint8,
 * scales and biases (n_layers, 2, batch, n_kv, cap, head_dim / group_size) bf16, group_size 32 | 64 | 128.
 * Replaces the bf16 binding: decode steps quantize the new K/V row, append it and attend over the dequantized
 * cache with the per-phase kernels (the persistent k_mega kernel reads bf16 pools only).  Prefill calls need a
 * bf16 pool (b200_engine_bind_kv) again. */
int b200_engine_bind_kvq(b200_engine* e, void* codes, void* scales, void* biases, int batch, int cap,
                         int group_size);
/* Prefill over an 8-bit cache: with the bf16 pool bound (its rows [0, ctx0) holding the dequantized prefix),
 * every prefill layer quantizes the chunk's new K/V rows into this 8-bit pool (same batch and capacity as the
 * bf16 one) and replaces them in the bf16 pool by their dequantized values before attending, so the chunk
 * attends to its prefix and to itself in quantized form.  The target is the row selected now, in every layer.
 * codes == NULL switches the write-through off; every bind and a change of the selected row switch it off too. */
int b200_engine_set_prefill_kvq(b200_engine* e, void* codes, void* scales, void* biases, int group_size);
/* Lock-step batch pool of kv_bits=8, the reference's batch rule (generate/ar.py:751-859 `_make_cache`: a
 * BatchQuantizedKVCache for every layer where models/cache.py:8-21 `should_quantize_kv_layer` holds, a BatchKVCache
 * for the others).  Layers 0 .. n_q8_layers-1 live in the 8-bit pool (n_q8_layers, 2, batch, n_kv, cap, ...) of the
 * b200_engine_bind_kvq format, layers n_q8_layers .. n_layers-1 in the bf16 pool (n_layers - n_q8_layers, 2, batch,
 * n_kv, cap, head_dim) — NULL when every layer is 8-bit.  Both share batch and cap.  b200_batch_begin /
 * b200_batch_decode then quantize each row's new K/V on the 8-bit layers before they are attended
 * (BatchQuantizedKVCache.update_and_fetch, models/cache.py:1747-1960).  Such a binding serves the batched decoder
 * only: prefill and single-row decode calls refuse it. */
int b200_engine_bind_batch_kvq(b200_engine* e, void* codes, void* scales, void* biases, int group_size, int n_q8_layers,
                               void* bf16_pool, int batch, int cap);
/* b200_engine_set_prefill_kvq into ROW `row` of an 8-bit batch pool of `rows` rows and capacity `cap` holding layers
 * 0 .. n_q8_layers-1 (the layout of b200_engine_bind_batch_kvq): the prefill of one admitted row writes its K/V rows
 * of those layers through to the batch pool (quantized before they are attended, BatchQuantizedKVCache.update_and_fetch
 * on a prefill chunk); the other layers stay bf16 in the bound pool.  Needs a bf16 pool bound; switched off like
 * b200_engine_set_prefill_kvq. */
int b200_engine_set_prefill_kvq_row(b200_engine* e, void* codes, void* scales, void* biases, int group_size, int rows,
                                    int cap, int row, int n_q8_layers);
/* One 8-bit decode attention step (the kernel of the per-phase decode step) on caller buffers, synchronous:
 * qbuf (n_heads, head_dim) bf16; K / V planes of one row and layer (n_kv, cap, ...); stage_k / stage_v bf16
 * (n_kv, cap, head_dim) holding the new row at position ctx; out (n_heads, head_dim) bf16. */
int b200_kvq_decode_attention(const void* qbuf, void* k_codes, void* k_scales, void* k_biases, void* v_codes,
                              void* v_scales, void* v_biases, const void* stage_k, const void* stage_v, void* out,
                              int n_heads, int n_kv, int head_dim, int cap, int ctx, int group_size, int cluster,
                              void* stream);
/* Bulk conversion between a bf16 pool and an 8-bit pool: the first n_tokens positions of `planes` planes
 * (plane = one (layer, k/v, row, kv head) of cap positions x head_dim elements), each side with its own
 * capacity.  Stream-ordered. */
int b200_kvq_quantize(const void* src, int src_cap, void* codes, void* scales, void* biases, int dst_cap,
                      long planes, int n_tokens, int head_dim, int group_size, void* stream);
int b200_kvq_dequantize(const void* codes, const void* scales, const void* biases, int src_cap, void* dst,
                        int dst_cap, long planes, int n_tokens, int head_dim, int group_size, void* stream);
/* rotary inverse-frequency tables, HOST fp32: lm (head_dim/2) =
 * compute_inv_freq (rope_utils.py:1042-1044), vision (v_head_dim/4) =
 * VisionRotaryEmbedding (vision.py:53-65).  Either may be NULL (keep default).
 * The Python host passes the values it computed with the reference's formula so
 * that host and device use bit-identical tables. */
int b200_engine_set_rope_tables(b200_engine* e, const float* lm_inv_freq_host,
                                const float* v_inv_freq_host);
/* M-RoPE frequency-to-axis table, HOST int32 (head_dim/2 entries in {0,1,2}: which of the t / h / w position ids
 * rotates frequency i).  The default is Qwen2-VL's chunked table (_chunked_position_selector, rope_utils.py:519-526);
 * Qwen3-VL passes _interleaved_position_selector's (rope_utils.py:511-516).  Prefill reads it; decode positions
 * are equal on all three axes. */
int b200_engine_set_axis_sel(b200_engine* e, const int* axis_sel_host);

/* VisionModel.__call__ (vision.py:257-290): pixel_values (n_patches, v_patch_dim)
 * f32, grid_thw_host (n_images,3) -> feats (n_patches / merge^2, v_out) bf16. */
int b200_engine_vision(b200_engine* e, const float* pixel_values,
                       const int* grid_thw_host, int n_images, void* feats_out,
                       void* stream);

/* LanguageModel.__call__ for L>1 (language.py:404-518; Qwen2Model :170-200):
 * embeds (T, hidden) bf16, pos3 (3,T) int32 device, cache row `row` holds ctx0
 * tokens already.  Appends T tokens of K/V.  If all_logits_out != NULL it
 * receives bf16 logits of every row (the reference computes them, ar.py:358),
 * rows round8(vocab) elements apart (= vocab for every vocabulary that is a
 * multiple of 8; 16-byte aligned rows otherwise); the last row always goes through the fused head+sampler:
 * logits / logprobs (ar.py:368) / greedy token (sample_utils.py:63-64) land in
 * the engine's step buffers and the decode state is armed with
 * position = ctx0 + T + rope_delta. */
int b200_engine_prefill(b200_engine* e, const void* embeds, const int* pos3,
                        int T, int ctx0, int rope_delta, void* all_logits_out,
                        void* stream);

/* PromptProcessingBatch (ar.py:1581-2175): n_seq FRESH prompts prefilled in one pass over the weights.
 * embeds (sum round8(T_g), hidden) bf16 = the sequences concatenated along the token axis, each padded to a
 * multiple of 8 tokens (finite values in the padding rows), pos3 (3, sum round8(T_g)) int32 device laid out the
 * same way; sequence g (seq_len[g] tokens, host array) fills KV pool row rows[g] (host array) from position 0; every GEMM
 * runs once over all tokens, attention is block-diagonal causal.  The first token of every sequence goes through
 * the fused head + sampler, in order: n_seq new entries in the token log. */
int b200_engine_prefill_batch(b200_engine* e, const void* embeds, const int* pos3, int n_seq,
                              const int* seq_len, const int* rows, void* stream);

/* generate_step's decode loop body (ar.py:496-515, _step :334-389) for greedy
 * sampling, n_steps times: embed(last token) -> 28 x decoder layer (L=1) -> norm
 * -> tied head -> logprobs -> argmax.  Launch-only; tokens accumulate in the
 * device token log.  force_token_host (may be NULL): teacher-forced input ids
 * for each step (testing). */
int b200_engine_decode(b200_engine* e, int n_steps, const int* force_tokens_host,
                       void* stream);
/* arm the decode state explicitly (used when the caller sampled the token itself) */
int b200_engine_set_next(b200_engine* e, int token, int ctx, int position, void* stream);

/* device pointers of the step buffers (valid until the next step is launched) */
const void* b200_engine_logits(const b200_engine* e);    /* (vocab) bf16 */
const void* b200_engine_logprobs(const b200_engine* e);  /* (vocab) bf16 */
const int* b200_engine_token_log(const b200_engine* e);  /* int32 ring of generated ids */
int b200_engine_token_log_capacity(const b200_engine* e);
/* number of tokens written so far (host mirror; launches counted, not completed) */
long b200_engine_tokens_launched(const b200_engine* e);
/* kernels launched by this engine since creation (bench `gpu_launches`) */
long b200_engine_launch_count(const b200_engine* e);
/* 0: decode via plain launches, 1: CUDA-graph replay (default) */
int b200_engine_set_graph(b200_engine* e, int enabled);
/* decode-step implementation.  0: one kernel per phase (28 x 5 + 2 launches);
 * 1 (default): ONE persistent kernel, CUDA-core GEMV consumers (k_mega: weight ring + software
 * grid barrier); a geometry it cannot hold runs the per-phase kernels.  Any other value is
 * B200_ERR_INVALID and leaves the mode unchanged. */
int b200_engine_set_mega(b200_engine* e, int enabled);
/* debugging / test aid: device pointer and size of an internal buffer.  names: "h", "act". */
int b200_engine_debug_buffer(b200_engine* e, const char* name, void** ptr, long* bytes);
/* synchronous: reads the device-side error flag (0 = none; a bounded wait gave up) */
int b200_engine_device_error(b200_engine* e, int* out);
/* debugging aid (k_mega): first call enables per-barrier globaltimer stamps, later
 * calls copy them out: out_host[2][1024][2] int64 = (arrive, release) per grid barrier
 * for CTA 0 and the last CTA of the most recent step. */
int b200_engine_mega_timeline(b200_engine* e, long long* out_host);
/* programmatic dependent launch between the decode-step kernels (default on) */
int b200_engine_set_pdl(b200_engine* e, int enabled);
/* CTAs per kv head in the decode attention cluster (1, 2, 4 or 8; default 8) */
int b200_engine_set_attn_cluster(b200_engine* e, int cluster);

/* stream-ordered helpers so the Python host needs no torch op on the hot path:
 * copy n generated ids [start, start+n) of the token log to HOST (pinned) memory;
 * copy the current logits/logprobs vector into a caller buffer (device). */
int b200_engine_fetch_tokens(b200_engine* e, long start, int n, int* host_out, void* stream);
/* ------------------------------------------------------------------------- */
/* fp32-accurate vision towers (LLaVA-1.5 CLIP, Idefics2 SigLIP + perceiver):    */
/* the reference runs them in fp32 with bf16-valued weights (llava.py:61-63,     */
/* idefics2.py:212-251).  Activations travel as split operands [hi | lo] (two    */
/* bf16 halves of an fp32 value, n_pad columns apart); the GEMMs run on the      */
/* tensor cores (W.x = W.x_hi + W.x_lo, fp32 accumulate), the rest in fp32.      */
/* ------------------------------------------------------------------------- */
/* nn.LayerNorm on fp32 rows -> fp32 and / or split output (llava/vision.py:84-104, idefics2/vision.py:94-121) */
int b200_f32_layer_norm(const float* x, long ldx, const void* w, const void* b, float eps, float* out32,
                        long ld32, void* out_split, long ld_split, int n_pad, int T, int N, void* stream);
int b200_f32_split(const float* x, long ldx, void* out_split, long ld_split, int n_pad, int T, int N, void* stream);
/* nn.RMSNorm on fp32 rows (idefics2.py:60-90,118-143); input row t goes to output row
 * (t / seg_in) * seg_out + seg_off + t % seg_in (seg_in == 0: row t) */
int b200_f32_rms_norm(const float* x, long ldx, const void* w, float eps, float* out32, long ld32, void* out_split,
                      long ld_split, int n_pad, int T, int N, int seg_in, int seg_out, int seg_off, void* stream);
/* fp32 SwiGLU of gu = [gate | up] ([T, 2I]) -> split operand (idefics2.py:146-171) */
int b200_f32_swiglu_split(const float* gu, long ldg, void* out_split, long ld_split, int n_pad, int T, int I,
                          void* stream);
/* Idefics3 / SmolVLM pixel shuffle (idefics3.py:47-62) written as the split operand of the connector's Linear:
 * x fp32 [n_img, side, side, E] -> [n_img (side/s)^2, E s^2], row (yg, xg), column (dy s + dx) E + e =
 * x[yg s + dy, xg s + dx, e]; round_in rounds the values to bf16 first (the reference's bf16 tower output) */
int b200_pixel_shuffle_split(const float* x, int n_img, int side, int E, int s, int round_in, void* out_split,
                             long ld_split, int n_pad, void* stream);
/* Conv2d(kernel == stride) patch rows, (kh, kw, c) order, from NHWC fp32 pixels, as a split operand
 * [B*gh*gw, Kp | Kp] (llava/vision.py:108-127, idefics2/vision.py:123-148) */
int b200_clip_patchify(const float* pixels_nhwc, int B, int H, int W, int C, int patch, void* out_split, int Kp,
                       void* stream);
/* class token + learned positions (CLIP), or positions gathered by pos_ids (SigLIP, idefics2/vision.py:150-173;
 * negative ids index from the end like numpy) */
int b200_tower_embed(const float* patch, const void* cls, const void* pos, const int* pos_ids, float* emb, int B,
                     int P, int E, int n_pos, void* stream);
/* fp32 SDPA (mx.fast.scaled_dot_product_attention on fp32 arrays), n_seg independent segments of Lq queries /
 * S keys q_seg / k_seg tokens apart; optional key mask [n_seg][S]; output fp32 and / or split */
int b200_attention_f32(const float* q, long q_ts, long q_hs, const float* k, long k_ts, long k_hs, const float* v,
                       long v_ts, long v_hs, float* out32, long o_ts, void* out_split, long os_ts, int n_pad,
                       int n_heads, int n_kv, int hd, int Lq, int S, int n_seg, long q_seg, long k_seg,
                       const unsigned char* key_mask, float scale, void* stream);
/* the same attention over RAGGED self-attention segments: segment z = tokens [cu_seqlens[z], cu_seqlens[z+1]) of q, k and
 * v (device int array of n_seg + 1 entries); max_len = the longest segment.  Qwen2.5-VL's windowed blocks
 * (qwen2_5_vl/vision.py:147-160: one SDPA per split of cu_seqlens). */
int b200_attention_f32_varlen(const float* q, long q_ts, long q_hs, const float* k, long k_ts, long k_hs, const float* v,
                              long v_ts, long v_hs, float* out32, long o_ts, void* out_split, long os_ts, int n_pad,
                              int n_heads, int n_kv, int hd, const int* cu_seqlens, int n_seg, int max_len, float scale,
                              void* stream);
/* 2-D rotary embedding on fp32 q and k in place (qwen2_5_vl/vision.py:35-50; qwen2_vl/vision.py:35-50): qkv [T, >= 3 *
 * n_heads * hd] = (q | k | v), pos_hw [T][2] (row, column) per patch, inv_freq [hd / 4] */
int b200_f32_vision_rope(float* qkv, long ld, const int* pos_hw, const float* inv_freq, int T, int n_heads, int hd,
                         void* stream);
/* out[i * unit + u] = in[idx[i] * unit + u] for rows of n fp32 values: the window permutation of merge units and its
 * inverse (qwen2_5_vl/vision.py:343-347,386-388) */
int b200_f32_gather_rows(const float* in, long ld_in, const int* idx, int n_idx, int unit, int n, float* out,
                         long ld_out, void* stream);
/* nn.Linear on fp32 activations: X split operand [T, n_parts x Kp], W [N, K_w] bf16 (row pitch ldw);
 * mode B200_WT_F32: C32 = act(acc + bias) + res32; mode B200_WT_SPLIT: Csplit = [hi | lo] of act(acc + bias) */
int b200_gemm_wt_f32(const void* X, long ldx, const void* W, long ldw, const void* bias, const float* res32,
                     long ldr32, float* C32, long ldc32, void* Csplit, long ld_split, int n_pad, int T, int N,
                     int K_w, int n_parts, int epilogue, int mode, void* stream);

/* ------------------------------------------------------------------------- */
/* Lock-step batched decode (continuous batching; generate/ar.py:929-1390        */
/* GenerationBatch, models/cache.py:972-1201 BatchKVCache)                       */
/* ------------------------------------------------------------------------- */
/* The bound KV pool is (layers, 2, rows, kv heads, capacity, head_dim); every row keeps its own
 * length (no left padding).  b200_engine_set_kv_row selects the row that b200_engine_prefill /
 * b200_engine_decode read and write (admission of a request = a batch-1 prefill into a free row).  A bind resets it
 * to 0 when the new pool has fewer rows; selecting another row switches a prefill write-through off. */
int b200_engine_set_kv_row(b200_engine* e, int row);
/* (Re)arm rows 0..B-1: next input token, cached length, rope position (length + M-RoPE delta) and
 * an active flag per row (host arrays).  B <= 16. */
int b200_batch_begin(b200_engine* e, int B, const int* tok, const int* ctx, const int* pos,
                     const int* active, void* stream);
/* n lock-step steps (one captured graph per step: ~7 kernels per layer, the weights are streamed
 * ONCE per step for all rows): greedy tokens + their bf16 logprobs go to a device log; the full
 * logprob rows are written only when want_logprobs != 0.  This is what
 * LanguageModel.fused_greedy_decode(inputs (B,1), cache=, rope_deltas=) runs (ar.py:1015-1042). */
int b200_batch_decode(b200_engine* e, int n_steps, int want_logprobs, void* stream);
/* tokens (and token logprobs) of steps [first_step, first_step+n) since the last begin:
 * host arrays [n_steps][B] */
int b200_batch_fetch(b200_engine* e, long first_step, int n_steps, int* tok_host, float* lp_host,
                     void* stream);
/* Per-row logits processors and top-k logprobs of the armed rows (sample_utils.make_logits_processors applied row by
 * row, GenerationBatch._step ar.py:1060-1121), until the next b200_batch_begin (which turns them off).  Each step,
 * between the head and the sampler, a row with processors appends its input token to its history and then applies,
 * in place on its bf16 logits: logit bias, repetition, presence and frequency penalty over the last context-size
 * tokens of the history, with the rounding points of the torch ops.  Device arrays owned by the caller, row b of
 * each at b * its row width:
 *   params int32 [rows][8]: flags (1 bias, 2 repetition, 4 presence, 8 frequency; 0 = none), repetition, presence
 *     and frequency context sizes, number of bias entries; penalties fp32 [rows][8]: repetition penalty,
 *     fp32(1 / repetition penalty), presence, frequency;
 *   bias_ids int32 / bias_vals fp32 (bf16-exact) [rows][bias_cap], ids in [0, vocab);
 *   hist int32 [rows][hist_cap] (hist_cap <= 1024) ring of each row's tokens, hist_len int32 [rows] tokens so far;
 *     ids outside [0, vocab) in it are skipped.
 * params NULL: no processors (no launch).  top_k 1..20: the k largest logprobs of every row and step go to a device
 * log (ties: lower token id first); 0: none. */
int b200_batch_set_procs(b200_engine* e, const int* params, const float* penalties, const int* bias_ids,
                         const float* bias_vals, int bias_cap, int* hist, int* hist_len, int hist_cap, int top_k);
/* top-k ids and logprobs of steps [first_step, first_step+n) since the last begin: host arrays [n_steps][B][20],
 * the first top_k of each row valid */
int b200_batch_fetch_topk(b200_engine* e, long first_step, int n_steps, int* ids_host, float* lp_host, void* stream);
/* The kernels of b200_batch_set_procs on caller buffers, stream-ordered (one step of B <= 16 rows, device arrays):
 * with params non-NULL the processors run in place on logits (B, ldv) bf16, appending tok[b] to row b's history
 * where active[b]; with top_k > 0 the top-k of logprobs (B, ldv) bf16 over [0, vocab) go to top_ids / top_lp
 * (B, 20).  History and bias ids outside [0, vocab) are skipped. */
int b200_batch_procs_apply(void* logits, const void* logprobs, int B, int vocab, int ldv, const int* tok,
                           const int* active, const int* params, const float* penalties, const int* bias_ids,
                           const float* bias_vals, int bias_cap, int* hist, int* hist_len, int hist_cap, int top_k,
                           int* top_ids, float* top_lp, void* stream);
/* device bf16 [B][round8(vocab)] of the last step; columns >= vocab hold -inf */
const void* b200_batch_logits(b200_engine* e);
const void* b200_batch_logprobs(b200_engine* e); /* same layout (want_logprobs) */
const int* b200_batch_token_log(b200_engine* e); /* device int32 [4096 steps][16 rows]        */
/* One lock-step attention of an 8-bit layer (the kv_bits=8 variant of the batched decoder's attention kernel) on
 * caller buffers, stream-ordered.  Replaces, for one decode step of a batch, BatchQuantizedKVCache.update_and_fetch
 * (models/cache.py:1805-1857) followed by quantized_scaled_dot_product_attention (models/base.py:260-356, the
 * quantized branch of scaled_dot_product_attention).  Arguments: qkv (B, (n_heads + 2 n_kv) head_dim) fp32 rows before bias; bias (n_heads + 2 n_kv)
 * head_dim bf16; inv_freq (head_dim / 2) fp32; ctx / pos (B) int32 device; codes / scales / biases the layer's planes
 * (2, pool_rows, n_kv, cap, ...) in the b200_engine_bind_kvq format; q_norm / k_norm (head_dim) bf16 or NULL.  Row b
 * quantizes its new K/V row, appends it at ctx[b] and attends over positions 0 .. ctx[b]; out (B, n_heads, head_dim). */
int b200_batch_kvq_attention(const float* qkv, const void* bias, const float* inv_freq, const int* ctx, const int* pos,
                             void* codes, void* scales, void* biases, int group_size, int pool_rows, int cap, void* out,
                             int B, int n_heads, int n_kv, int head_dim, const void* q_norm, const void* k_norm, float eps,
                             void* stream);
/* BatchKVCache / BatchQuantizedKVCache.filter / extend / extract (models/cache.py:1077-1201, 1747-1960) on device
 * pools: copy the first n_tokens positions of one row of a plane set (n_layers, 2, rows, n_kv, cap,
 * bytes_per_position) into a row of another (or the same) one.  A bf16 pool is bytes_per_position = 2 * head_dim;
 * the planes of an 8-bit pool are head_dim (codes) and 2 * head_dim / group_size (scales, biases).  The bytes move
 * unchanged. */
int b200_pool_copy_row(void* dst_pool, int dst_batch, int dst_cap, int dst_row, const void* src_pool, int src_batch,
                       int src_cap, int src_row, int n_layers, int n_kv, int bytes_per_position, int n_tokens,
                       void* stream);

int b200_memcpy_d2d(void* dst, const void* src, long bytes, void* stream);

/* timing helper for bench.py: average device duration (ms) of the decode-step
 * graph over the last b200_engine_decode call, measured with CUDA events on the
 * launching stream. */
float b200_engine_last_decode_ms(const b200_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* B200VLM_H */
