// Shared declarations of the decode-step kernels (decode.cu) and the engine.
#pragma once
#include "common.cuh"
#include "kvq.cuh"

namespace b200 {

struct DecodeDims {
  int hidden, inter, n_heads, n_kv, hd, vocab, cap;
  float eps;
  float scale_bf;  // head_dim^-0.5 rounded to bf16 (mlx fallback: array(scale, q.dtype))
};

struct LayerW {
  const bf16 *ln1, *ln2;   // RMSNorm weights
  const bf16 *wqkv, *bqkv; // [(n_heads+2n_kv)*hd, hidden], bias
  const bf16* wo;          // [hidden, hidden]
  const bf16* wgu;         // [2*inter, hidden]  (gate rows then up rows)
  const bf16* wd;          // [hidden, inter]
};

// device-resident decode state: lets a captured CUDA graph replay unchanged
struct DecState {
  unsigned long long best_key;  // packed (orderable logprob, ~index) of the running argmax
  unsigned int blocks_done;
  int tok;        // token fed to the next step
  int ctx;        // tokens in the cache == write index of the next step
  int pos;        // rope position of the next step (ctx + rope_delta)
  int n_out;      // tokens written to the token log
  int use_force;  // teacher forcing (tests)
  int error;      // set by a bounded wait that gave up (1: grid barrier, 2: mbarrier)
  unsigned long long bar_base;  // k_mega: value of the grid-barrier counter at step start
  unsigned long long att_base;  // k_mega: attention phases executed before this step
};

// ---- k_mega (decode_mega.cu): the whole step as one persistent kernel ----------
constexpr int MEGA_MAX_LAYERS = 64;
struct MegaPhase {
  int K, N;    // reduction length, output rows
  int R, S;    // row(-pair)s per tile, K slices per row (R*S == 8 consumer warps)
  int tiles;
};
struct MegaP {
  DecodeDims d;
  int n_layers;
  LayerW layers[MEGA_MAX_LAYERS];  // in kernel-parameter (constant) space
  const bf16 *final_norm, *head, *embed;
  bf16 *h, *qbuf, *attn, *act, *logits, *logprobs;
  bf16* kv;              // layer 0 K plane of cache row 0
  long kv_layer_stride;  // elements between layers
  long kv_v_offset;      // elements from a layer's K plane to its V plane
  float2* partials;
  DecState* st;
  int* token_log;
  int log_cap;
  const int* force;
  const float* inv_freq;
  MegaPhase ph[5];  // QKV, ORES, GATEUP, DRES, HEAD
  int n_stages, stage_bytes;
  int attn_ctas, hsplit;
  unsigned long long* bar;  // monotonic grid-barrier counter
  int advance;
  int scratch_bytes;  // attention scratch / activation vector region after the ring
  float* att_part;  // [groups][8 units][4*hd] fp32 partial attention outputs
  float* att_stats; // [groups][8 units][4 heads] x 2 words {float bits << 32 | epoch}: (max, sum exp)
  long long* dbg;  // optional [2][1024][2] globaltimer stamps (arrive, release) per barrier
  // Qwen3-VL q_norm / k_norm (qk_norm != 0): the QKV phase leaves q / k unrotated and a q/k-norm phase between two
  // grid barriers normalises and rotates them (the per-phase step's arithmetic, common.cuh::warp_head_rms / _rope)
  int qk_norm;
  const bf16* qn[MEGA_MAX_LAYERS];
  const bf16* kn[MEGA_MAX_LAYERS];
};
int mega_fill(MegaP& p, int sm_count);
int mega_launch(const MegaP& p, int sm_count, cudaStream_t s);

// lock-step batched decode (decode_batch.cu)
struct BdModel {
  DecodeDims d;
  int n_layers;
  const LayerW* layers;
  const bf16 *embed, *head, *final_norm;
  const float* inv_freq;
  bf16* kv;            // K plane of row 0 of the first bf16 layer (layer q8_layers), or nullptr
  long layer_stride, v_off, row_stride;
  int kv_batch, sm_count;
  const bf16* const* qn;  // per layer q_norm / k_norm weights (Qwen3-VL), or nullptr
  const bf16* const* kn;
  // kv_bits=8 (b200_engine_bind_batch_kvq): layers 0 .. q8_layers-1 live in an 8-bit pool (format kvq.cuh) of the
  // same rows and capacity, layers q8_layers .. n_layers-1 in the bf16 pool `kv`.  q8_layers = 0: all bf16.
  uint8_t* q8_codes;
  bf16 *q8_scales, *q8_biases;
  int q8_gs, q8_layers;
};
// one 8-bit lock-step attention on caller buffers (b200_batch_kvq_attention): qkv (B, (n_heads + 2 n_kv) hd) fp32
// finished-but-unbiased rows, the layer's 8-bit planes (2, pool_rows, n_kv, cap, ...) and per-row ctx / pos (device)
int batch_kvq_attention(const float* qkv, const bf16* bias, const float* inv_freq, const int* ctx, const int* pos,
                        uint8_t* codes, bf16* scales, bf16* biases, int gs, int pool_rows, int cap, bf16* out, int B,
                        int n_heads, int n_kv, int hd, const bf16* qn, const bf16* kn, float eps, int sm_count,
                        cudaStream_t s);
int batch_decoder_begin(void** handle, const BdModel& m, int B, const int* tok, const int* ctx, const int* pos,
                        const int* active, cudaStream_t s);
int batch_decoder_step(void* handle, const BdModel& m, int n_steps, bool want_logprobs, cudaStream_t s,
                       cudaStream_t cap_stream, long* launches);
int batch_decoder_fetch(void* handle, long first_step, int n_steps, int* tok_host, float* lp_host, cudaStream_t s);

// Per-row logits processors and top-k logprobs of the lock-step batch (b200_batch_set_procs).  Device arrays owned
// by the caller, row b at b * stride:
//   params    int32 [rows][BD_PROC_PARAMS]: flags (BD_PROC_*; 0 = none), repetition / presence / frequency context
//             sizes, number of bias entries
//   penalties fp32  [rows][BD_PROC_PARAMS]: repetition penalty, fp32(1 / repetition penalty), presence, frequency
//   bias_ids / bias_vals  [rows][bias_cap]: token ids and bf16-exact values of logit_bias
//   hist [rows][hist_cap] ring of each row's token history, hist_len [rows] tokens appended so far
constexpr int BD_PROC_PARAMS = 8, BD_HIST_MAX = 1024, BD_TOPK_MAX = 20;
constexpr int BD_TOPK_SLICE = 8192, BD_TOPK_CAND_MAX = 1024;
constexpr int BD_PROC_BIAS = 1, BD_PROC_REP = 2, BD_PROC_PRES = 4, BD_PROC_FREQ = 8;
struct BdProcs {
  const int* params;      // nullptr: no row has processors (no launch)
  const float* penalties;
  const int* bias_ids;
  const float* bias_vals;
  int bias_cap;
  int* hist;
  int* hist_len;
  int hist_cap;
  int top_k;              // 0 .. BD_TOPK_MAX (0: none)
};
// replaces the processors until the next batch_decoder_begin (which turns them off)
int batch_decoder_set_procs(void* handle, const BdProcs& pr, int vocab);
// top-k ids / logprobs of steps [first, first + n): host arrays [n][B][BD_TOPK_MAX]
int batch_decoder_fetch_topk(void* handle, long first_step, int n_steps, int* ids_host, float* lp_host, cudaStream_t s);
// the processors and the top-k of one step on caller buffers (b200_batch_procs_apply)
int batch_procs_apply(bf16* logits, const bf16* logprobs, int B, int V, int ldv, const int* tok, const int* active,
                      const BdProcs& pr, int* top_ids, float* top_lp, cudaStream_t s);
const void* batch_decoder_buffer(void* handle, int which);
void batch_decoder_destroy(void* handle);

void decode_set_sm_count(int n);
void decode_set_pdl(bool on);
// kernel attributes of the decode step that do not depend on the cache (once per engine)
int decode_prepare();
// the per-phase attention: bf16 pool, k_attn1 up to 4096 positions, else k_attn on clusters of `cluster` CTAs; 8-bit
// pool (q8), k_attn at every capacity.  Refuses a capacity its shared memory cannot hold; run before the steps it serves
int attn_prepare(const DecodeDims& d, int cluster, bool q8);
int head_grid();
// qn / kn (Qwen3-VL q_norm / k_norm weights, both or neither): the QKV kernel leaves q / k unrotated and a second
// kernel (k_qk_norm_rope) normalises and rotates the q heads and the new K row
int launch_qkv(const DecodeDims& d, const LayerW& lw, const bf16* h, bf16* qbuf, bf16* kc,
               bf16* vc, const DecState* st, const float* inv_freq, cudaStream_t s, const bf16* qn = nullptr,
               const bf16* kn = nullptr);
// The K / V rows of one layer (bound row, kv head stride cap positions) the per-phase attention reads.
//   bf16 pool:  k / v are its planes and k8.codes is null.
//   8-bit pool: k8 / v8 are its planes, and k / v the bf16 staging planes where the QKV kernel left the new row at
//               position ctx.  The attention quantizes that row, appends it to k8 / v8 and attends over positions
//               0..ctx, the new one in its quantized form.
struct AttnKv {
  const bf16 *k, *v;
  KvqPlanes k8, v8;
};
int launch_attn(const DecodeDims& d, const bf16* qbuf, const AttnKv& kv, bf16* out, const DecState* st, int cluster,
                cudaStream_t s);
int launch_res(const bf16* W, const bf16* x, bf16* h, int N, int K, cudaStream_t s);
int launch_gateup(const DecodeDims& d, const LayerW& lw, const bf16* h, bf16* act, cudaStream_t s);
int launch_head(const DecodeDims& d, const bf16* norm_w, const bf16* E, const bf16* h,
                bf16* logits, float2* partials, cudaStream_t s);
int launch_sample(const DecodeDims& d, const bf16* logits, const float2* partials, bf16* logprobs,
                  const bf16* E, bf16* h, DecState* st, int* token_log, int log_cap,
                  const int* force_tokens, int advance, cudaStream_t s);
int launch_set_state(DecState* st, int tok, int ctx, int pos, int use_force, int set_tok,
                     const bf16* E, bf16* h, int hidden, cudaStream_t s);

// where the bound KV pool lives (device copy: kernels of captured graphs read it instead of baked pointers)
struct KvRef {
  bf16* k0;            // K plane of layer 0, bound row
  long layer_stride;   // elements between layers
  long v_off;          // elements from a K plane to its V plane
  int cap;
};

// row ops / gemm / attention (other translation units)
int cast_f32_bf16(const float* src, void* dst, long n, cudaStream_t st);
int layer_norm(const void* x, const void* w, const void* b, void* y, int rows, int dim, float eps,
               cudaStream_t st);
int rms_norm(const void* x, const void* w, void* y, int rows, int dim, float eps, cudaStream_t st);
int vision_rope(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads,
                int hd, cudaStream_t st);
int mrope_kv_write(void* qkv, const int* pos3, const float* inv_freq, const int* axis_sel,
                   void* kc, void* vc, int T, int ctx0, int cap, int n_heads, int n_kv, int hd,
                   cudaStream_t st, float q_scale = 0.f, void* vt = nullptr, int t_ld = 0,
                   const KvRef* ref = nullptr, int layer = 0, void* kws = nullptr, const void* tok_loc = nullptr,
                   long row_stride = 0);
// Qwen3-VL q/k RMSNorm per head, in place on the q and k heads of qkv (before mrope_kv_write)
int qk_norm(void* qkv, int T, int n_heads, int n_kv, int hd, const void* qn, const void* kn, float eps,
            cudaStream_t st);
int vision_qkv_post(void* qkv, const int* pos_hw, const float* inv_freq, int n_tok, int n_heads, int hd,
                    float scale, void* vt, int t_ld, cudaStream_t st, const void* cs = nullptr);
// cos / sin table [n_tok][hd / 2] float2 for vision_qkv_post (computed once per tower call)
int vision_rope_table(const int* pos_hw, const float* inv_freq, int n_tok, int hd, void* cs, cudaStream_t st);
bool attention_fa_supported(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
                            const void* vt, long vt_hs, long vt_ds, const void* out, long o_ts, int hd);
int attention_fa(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs, const void* vt,
                 long vt_hs, long vt_ds, void* out, long o_ts, int n_heads, int n_kv, int hd, int Lq, int S,
                 int causal, cudaStream_t st, int q0 = 0, int q_tot = 0, int k0 = 0, int k_tot = 0,
                 const void* segs = nullptr, int n_seg = 0);   // segs: device int4 (q0, Lq, k0, S) per segment; Lq / S = the longest
int swiglu(const void* gu, void* out, int rows, int inter, cudaStream_t st);
int embed_merge(const int* ids, int B, int T, const void* table, int hidden, const void* feats,
                int n_feats, int image_token, int video_token, void* out, int* src_out,
                cudaStream_t st);
// weight-major wgmma GEMM (gemm_wt.cu) + the row op that finishes its split-K partials
struct WtConfig {
  int TN, KS, stages, split;
};
// extension for the fp32-accurate (split bf16) GEMMs of the LLaVA / Idefics2 towers
struct WtExt {
  int kb_w;          // > 0: X holds n parts [x_hi | x_lo | ..] of kb_w k-blocks each; W k-block = k-block % kb_w
  int k_w;           // columns of W (kb_w > 0)
  long ldw;          // row pitch of W in elements (0: k_w)
  float* C32;        // B200_WT_F32 output
  const float* res32;
  long ldc32, ldr32;
  bf16* Csplit;      // B200_WT_SPLIT output [hi | lo]
  long ld_split;
  int n_pad;         // columns between the hi and the lo half
};
void gemm_wt_auto(int T, int row_blocks, int K, bool allow_split, WtConfig* c, int sm_count);
int gemm_wt(const void* X, long ldx, const void* W, const void* bias, const void* residual, long ldr,
            void* C, long ldc, float* partial, int T, int N, int K, int epilogue, int mode, int inter,
            const WtConfig& cfg, unsigned flags, cudaStream_t st, const WtExt* ext = nullptr);
int gemm_wt_tuned(const void* X, long ldx, const void* W, const void* bias, const void* residual, long ldr,
                  void* C, long ldc, float* partial, long partial_bytes, int T, int N, int K, int epilogue,
                  int mode, int inter, bool allow_split, int sm_count, int* split_out, cudaStream_t st,
                  const WtExt* ext = nullptr, WtConfig* cfg_out = nullptr);
int finish_rows(const float* P, int S, const void* bias, const void* resid, long ldr, void* h_out,
                long ldh, int norm_kind, const void* nw, const void* nb, float eps, void* xn, long ldx,
                int T, int N, cudaStream_t st);
int attention(const void* q, long q_ts, long q_hs, const void* k, long k_ts, long k_hs,
              const void* v, long v_ts, long v_hs, void* out, long o_ts, int n_heads, int n_kv,
              int hd, int Lq, int S, int causal, float scale, cudaStream_t st);

}  // namespace b200
