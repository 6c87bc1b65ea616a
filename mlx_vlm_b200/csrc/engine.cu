// Engine: whole-tower / whole-step entry points of the C ABI (include/b200vlm.h).
// Owns the weight table, the decode state, the step buffers and the captured
// CUDA graph of one decode step.  The caller (Python, via ctypes) owns weights,
// workspace and the KV pool (torch-allocated device memory).
#include <stdarg.h>

#include <array>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "decode.cuh"
#include "kvq.cuh"

namespace b200 {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d in %s", (int)e, cudaGetErrorString(e), file, line, what);
  return B200_ERR_CUDA;
}

int kernel_opt_in(const void* kern, int max_dyn_smem, bool max_carveout) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, std::array<int, 2>> set;  // (kernel, device) -> values set, 0 = none
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  const cudaFuncAttribute attr[2] = {cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     cudaFuncAttributePreferredSharedMemoryCarveout};
  const int want[2] = {max_dyn_smem, max_carveout ? (int)cudaSharedmemCarveoutMaxShared : 0};
  std::lock_guard<std::mutex> g(mu);
  std::array<int, 2>& have = set[{kern, dev}];
  for (int i = 0; i < 2; ++i) {
    if (want[i] <= 0 || have[i] == want[i]) continue;
    B200_CUDA(cudaFuncSetAttribute(kern, attr[i], want[i]));
    have[i] = want[i];
  }
  return B200_OK;
}

struct VBlk {
  const bf16 *ln1w, *ln1b, *ln2w, *ln2b, *qkvw, *qkvb, *projw, *projb, *fc1w, *fc1b, *fc2w, *fc2b;
};

// Offset, in head rows (one position of one kv head), of the (layer, side, row) plane of a pool laid out
// (layers, 2, rows, n_kv, cap, ...).  Times head_dim: the element offset of a bf16 pool or of 8-bit codes; times
// head_dim / group_size: that of 8-bit scales and biases.
static long plane_off(int layer, int side, int row, int rows, int n_kv, int cap) {
  return (((long)layer * 2 + side) * rows + row) * n_kv * (long)cap;
}

// The reference's BatchKVCache.filter / extend / extract (models/cache.py:1077-1201) move rows between arrays: copy the
// first n_tokens positions of one row of a plane set (layers, 2, rows, n_kv, cap, bytes_per_position) into a row of
// another (or the same) one, byte for byte.  A bf16 pool is bytes_per_position = 2 * head_dim; the planes of an 8-bit
// pool are head_dim (codes) and 2 * head_dim / group_size (scales, biases).
extern "C" int b200_pool_copy_row(void* dst_pool, int dst_batch, int dst_cap, int dst_row, const void* src_pool,
                                  int src_batch, int src_cap, int src_row, int n_layers, int n_kv, int bytes_per_position,
                                  int n_tokens, void* stream) {
  B200_REQUIRE(dst_pool && src_pool && dst_row >= 0 && dst_row < dst_batch && src_row >= 0 && src_row < src_batch &&
                   n_tokens >= 0 && n_tokens <= dst_cap && n_tokens <= src_cap && bytes_per_position > 0,
               "pool_copy_row: bad arguments");
  if (n_tokens == 0) return B200_OK;
  const size_t bp = (size_t)bytes_per_position;
  for (int l = 0; l < n_layers; ++l)
    for (int kv = 0; kv < 2; ++kv) {
      const char* sp = (const char*)src_pool + plane_off(l, kv, src_row, src_batch, n_kv, src_cap) * bp;
      char* dp = (char*)dst_pool + plane_off(l, kv, dst_row, dst_batch, n_kv, dst_cap) * bp;
      B200_CUDA(cudaMemcpy2DAsync(dp, (size_t)dst_cap * bp, sp, (size_t)src_cap * bp, (size_t)n_tokens * bp, n_kv,
                                  cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    }
  return B200_OK;
}

// The KV cache the engine is bound to (caller-owned).  The kind decides which calls may use it: prefill needs bf16,
// single-request decode bf16 or q8, the lock-step batch decoder bf16 or q8_batch.
enum class KvKind { none, bf16, q8, q8_batch };
struct KvBinding {
  KvKind kind = KvKind::none;
  bf16* kv = nullptr;  // bf16 pool; q8_batch: layers n_q8 .. n_layers-1 (nullptr when every layer is 8-bit)
  KvqPlanes q8 = {};   // 8-bit pool of layers 0 .. n_q8-1
  int n_q8 = 0, rows = 0, cap = 0;  // rows and capacity of both pools
  bool operator==(const KvBinding& o) const {
    return kind == o.kind && kv == o.kv && q8.codes == o.q8.codes && q8.scales == o.q8.scales &&
           q8.biases == o.q8.biases && q8.gs == o.q8.gs && n_q8 == o.n_q8 && rows == o.rows && cap == o.cap;
  }
};
// Prefill write-through: every prefill layer below n_layers quantizes its chunk's K/V rows into row `row` of an
// 8-bit pool of `rows` rows and capacity `cap` (the b200_engine_bind_kvq layout) before they are attended
struct KvWriteThrough {
  KvqPlanes q8;
  int rows, cap, row, n_layers;
};

}  // namespace b200

using namespace b200;

struct b200_engine {
  b200_qwen2vl_config cfg;
  int device = 0, sm_count = 132;
  std::unordered_map<std::string, const bf16*> w;
  std::unordered_map<std::string, long> wn;
  bool resolved = false;
  // resolved weights
  const bf16* v_patch = nullptr;
  std::vector<VBlk> vblk;
  const bf16 *m_lnw = nullptr, *m_lnb = nullptr, *m_fc1w = nullptr, *m_fc1b = nullptr,
             *m_fc2w = nullptr, *m_fc2b = nullptr;
  const bf16 *embed = nullptr, *head = nullptr, *norm = nullptr;
  std::vector<LayerW> layers;
  // Qwen3-VL q_norm / k_norm weights per layer (lm.<i>.qn / lm.<i>.kn): registered for every layer or for none
  bool qk_norm = false;
  std::vector<const bf16*> qn, kn;
  // workspace (caller-owned)
  uint8_t* ws = nullptr;
  long ws_bytes = 0;
  // KV binding (set by bind() only) and the row of it that prefill / single-row decode read and write
  KvBinding kvb;
  int kv_row = 0;
  std::optional<KvWriteThrough> wt;  // cleared by every bind and by a change of kv_row
  // q8 kind: engine-owned bf16 staging planes [2][n_kv][cap][hd] where the decode QKV kernel leaves the new K/V row
  // before it is quantized
  bf16* q8_stage = nullptr;
  long q8_stage_elems = 0;
  void* batch = nullptr; // lock-step batched decoder (decode_batch.cu)
  std::vector<int> b_ctx, b_active;  // host mirrors of the batched rows' lengths
  // engine-owned small device buffers
  DecState* st = nullptr;
  bf16 *h = nullptr, *qbuf = nullptr, *attn = nullptr, *act = nullptr, *logits = nullptr,
       *logprobs = nullptr;
  float2* partials = nullptr;
  int *token_log = nullptr, *force = nullptr;
  float *lm_inv_freq = nullptr, *v_inv_freq = nullptr;
  int* axis_sel = nullptr;
  int* pos_hw = nullptr;
  long pos_hw_cap = 0;
  int* pos_hw_host = nullptr;   // pinned staging of the rot_pos_emb ids (no stream sync per call)
  long pos_hw_host_cap = 0;
  cudaEvent_t pos_ev = nullptr;
  // (row, position) of every token of a batched prefill: grow-only device buffer + pinned staging, like pos_hw (a
  // stream-ordered allocation per call made the driver trim / re-map its pool around every call: prefill calls of 85 ms
  // intermittently took 400-600 ms)
  int* loc_dev = nullptr;
  long loc_cap = 0;
  int* loc_host = nullptr;
  long loc_host_cap = 0;
  cudaEvent_t loc_ev = nullptr;
  // captured CUDA graphs of the vision tower / the prefill layers, keyed by everything that is baked
  // into their nodes (shapes, workspace, KV binding): the sequences are ~500 small launches, which
  // the host cannot enqueue as fast as the GPU executes them
  struct SeqGraph {
    std::vector<long> key;
    cudaGraphExec_t exec = nullptr;
    int seen = 0;
    long n_launch = 0;
  };
  std::vector<SeqGraph> vis_graphs, pre_graphs;
  KvRef* kvref = nullptr;       // device: where the bound pool row lives (read by the captured prefill)
  KvRef* kvref_host = nullptr;  // pinned staging
  cudaEvent_t kvref_ev = nullptr;
  int log_cap = 1 << 16;
  // host mirrors of the decode state
  int ctx_host = 0, pos_host = 0;
  long tokens_launched = 0, launches = 0;
  // graph
  bool use_graph = true;
  cudaGraphExec_t gexec = nullptr;
  cudaStream_t cap_stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int last_steps = 0;
  bool timing_valid = false;
  int attn_cluster = 8;
  // megakernel
  int use_mega = 1;  // 0: one kernel per phase, 1: k_mega
  bool mega_fits = true;  // false: this shape / cache capacity does not fit the persistent kernel
  bool active_mega() const { return mega_fits && use_mega; }
  float* att_part = nullptr;
  float* att_stats = nullptr;
  unsigned long long* bar = nullptr;
  bool mega_ready = false;
  MegaP mp;
  long long* dbg = nullptr;

  DecodeDims dims() const {
    DecodeDims d;
    d.hidden = cfg.hidden; d.inter = cfg.inter; d.n_heads = cfg.n_heads; d.n_kv = cfg.n_kv_heads;
    d.hd = cfg.head_dim; d.vocab = cfg.vocab; d.cap = kvb.cap; d.eps = cfg.rms_eps;
    d.scale_bf = __bfloat162float(__float2bfloat16_rn(1.0f / sqrtf((float)cfg.head_dim)));
    return d;
  }
  // element offset of the (layer, side, row) plane of a pool of the bound geometry (bf16 or 8-bit codes)
  long kv_off(int layer, int side, int row) const {
    return plane_off(layer, side, row, kvb.rows, cfg.n_kv_heads, kvb.cap) * cfg.head_dim;
  }
  bf16* kptr(int layer, int row) const { return kvb.kv + kv_off(layer, 0, row); }
  bf16* vptr(int layer, int row) const { return kvb.kv + kv_off(layer, 1, row); }
  KvqPlanes q8_plane(const KvqPlanes& pool, int layer, int side, int row, int rows, int cap) const {
    const long off = plane_off(layer, side, row, rows, cfg.n_kv_heads, cap);
    return KvqPlanes{pool.codes + off * cfg.head_dim, pool.scales + off * (cfg.head_dim / pool.gs),
                     pool.biases + off * (cfg.head_dim / pool.gs), pool.gs};
  }
};

static const bf16* need(b200_engine* e, const std::string& name, long n_expected, bool* ok) {
  auto it = e->w.find(name);
  if (it == e->w.end()) {
    set_error("engine: weight '%s' not set", name.c_str());
    *ok = false;
    return nullptr;
  }
  if (n_expected > 0 && e->wn[name] != n_expected) {
    set_error("engine: weight '%s' has %ld elements, expected %ld", name.c_str(), e->wn[name],
              n_expected);
    *ok = false;
    return nullptr;
  }
  return it->second;
}

static int resolve(b200_engine* e) {
  if (e->resolved) return B200_OK;
  const auto& c = e->cfg;
  bool ok = true;
  const long E = c.v_embed, Em = c.v_mlp, mg = (long)c.v_merge * c.v_merge * E;
  const bool vis = !c.external_vision;
  if (vis) e->v_patch = need(e, "v.patch_embed.w", E * c.v_patch_dim, &ok);
  e->vblk.resize(vis ? c.v_depth : 0);
  for (int i = 0; vis && i < c.v_depth && ok; ++i) {
    const std::string p = "v.blk." + std::to_string(i) + ".";
    VBlk& b = e->vblk[i];
    b.ln1w = need(e, p + "ln1.w", E, &ok); b.ln1b = need(e, p + "ln1.b", E, &ok);
    b.ln2w = need(e, p + "ln2.w", E, &ok); b.ln2b = need(e, p + "ln2.b", E, &ok);
    b.qkvw = need(e, p + "qkv.w", 3 * E * E, &ok); b.qkvb = need(e, p + "qkv.b", 3 * E, &ok);
    b.projw = need(e, p + "proj.w", E * E, &ok); b.projb = need(e, p + "proj.b", E, &ok);
    b.fc1w = need(e, p + "fc1.w", Em * E, &ok); b.fc1b = need(e, p + "fc1.b", Em, &ok);
    b.fc2w = need(e, p + "fc2.w", E * Em, &ok); b.fc2b = need(e, p + "fc2.b", E, &ok);
  }
  if (ok && vis) {
    e->m_lnw = need(e, "v.merger.ln.w", E, &ok); e->m_lnb = need(e, "v.merger.ln.b", E, &ok);
    e->m_fc1w = need(e, "v.merger.fc1.w", mg * mg, &ok); e->m_fc1b = need(e, "v.merger.fc1.b", mg, &ok);
    e->m_fc2w = need(e, "v.merger.fc2.w", (long)c.v_out * mg, &ok);
    e->m_fc2b = need(e, "v.merger.fc2.b", c.v_out, &ok);
  }
  const long H = c.hidden, I = c.inter, QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  if (ok) {
    e->embed = need(e, "lm.embed", (long)c.vocab * H, &ok);
    e->norm = need(e, "lm.norm", H, &ok);
    e->head = c.tie_embeddings ? e->embed : need(e, "lm.head", (long)c.vocab * H, &ok);
  }
  e->layers.resize(c.n_layers);
  for (int i = 0; i < c.n_layers && ok; ++i) {
    const std::string p = "lm." + std::to_string(i) + ".";
    LayerW& l = e->layers[i];
    l.ln1 = need(e, p + "ln1", H, &ok); l.ln2 = need(e, p + "ln2", H, &ok);
    l.wqkv = need(e, p + "wqkv", QKV * H, &ok); l.bqkv = need(e, p + "bqkv", QKV, &ok);
    l.wo = need(e, p + "wo", H * (long)c.n_heads * c.head_dim, &ok);
    l.wgu = need(e, p + "wgu", 2 * I * H, &ok); l.wd = need(e, p + "wd", H * I, &ok);
  }
  e->qk_norm = ok && c.n_layers > 0 && e->w.count("lm.0.qn");
  e->qn.assign(e->qk_norm ? c.n_layers : 0, nullptr);
  e->kn.assign(e->qk_norm ? c.n_layers : 0, nullptr);
  for (int i = 0; e->qk_norm && i < c.n_layers && ok; ++i) {
    const std::string p = "lm." + std::to_string(i) + ".";
    e->qn[i] = need(e, p + "qn", c.head_dim, &ok);
    e->kn[i] = need(e, p + "kn", c.head_dim, &ok);
  }
  if (!ok) return B200_ERR_STATE;
  e->resolved = true;
  return B200_OK;
}

static void drop_seq_graphs(b200_engine* e) {
  for (auto* v : {&e->vis_graphs, &e->pre_graphs}) {
    for (auto& g : *v)
      if (g.exec) cudaGraphExecDestroy(g.exec);
    v->clear();
  }
}

static void invalidate_graph(b200_engine* e) {
  e->mega_ready = false;
  e->mega_fits = true;
  if (e->gexec) {
    cudaGraphExecDestroy(e->gexec);
    e->gexec = nullptr;
  }
}

static int mega_prepare(b200_engine* e, cudaStream_t s) {
  const auto& c = e->cfg;
  B200_REQUIRE(c.n_layers <= MEGA_MAX_LAYERS, "mega: %d layers > %d", c.n_layers, MEGA_MAX_LAYERS);
  B200_REQUIRE(e->kvb.kind == KvKind::bf16,
               "mega: the persistent kernel reads a bf16 KV pool; an 8-bit pool runs the per-phase kernels");
  if (!e->bar) {
    B200_CUDA(cudaMalloc(&e->bar, sizeof(unsigned long long)));
    B200_CUDA(cudaMemset(e->bar, 0, sizeof(unsigned long long)));
    const size_t part = (size_t)64 * 8 * 4 * c.head_dim * sizeof(float);
    B200_CUDA(cudaMalloc(&e->att_part, part));
    B200_CUDA(cudaMalloc(&e->att_stats, (size_t)64 * 8 * 4 * 16));  // {value, epoch} word pairs
    B200_CUDA(cudaMemset(e->att_stats, 0, (size_t)64 * 8 * 4 * 16));
  }
  MegaP& p = e->mp;
  memset(&p, 0, sizeof(p));
  p.d = e->dims();
  p.n_layers = c.n_layers;
  for (int l = 0; l < c.n_layers; ++l) p.layers[l] = e->layers[l];
  p.att_part = e->att_part;
  p.att_stats = e->att_stats;
  p.final_norm = e->norm; p.head = e->head; p.embed = e->embed;
  p.h = e->h; p.qbuf = e->qbuf; p.attn = e->attn; p.act = e->act;
  p.logits = e->logits; p.logprobs = e->logprobs;
  p.kv = e->kptr(0, e->kv_row);
  p.kv_layer_stride = e->kv_off(1, 0, 0);
  p.kv_v_offset = e->kv_off(0, 1, 0);
  p.partials = e->partials; p.st = e->st; p.token_log = e->token_log; p.log_cap = e->log_cap;
  p.force = e->force; p.inv_freq = e->lm_inv_freq; p.bar = e->bar; p.advance = 1;
  p.dbg = e->dbg;
  p.qk_norm = e->qk_norm;
  for (int l = 0; e->qk_norm && l < c.n_layers; ++l) {
    p.qn[l] = e->qn[l];
    p.kn[l] = e->kn[l];
  }
  int rc;
  if ((rc = mega_fill(p, e->sm_count))) return rc;
  e->mega_ready = true;
  return B200_OK;
}

// one decode step as plain launches on stream s (also what gets captured)
static int enqueue_step(b200_engine* e, cudaStream_t s) {
  const DecodeDims d = e->dims();
  const auto& c = e->cfg;
  int rc;
  if (e->active_mega()) return mega_launch(e->mp, e->sm_count, s);
  // the 8-bit kind: the QKV kernel leaves the new K / V row in the staging planes, and the attention appends it to the
  // 8-bit pool
  const KvBinding& b = e->kvb;
  const bool q8 = b.kind == KvKind::q8;
  const long stage_v = (long)c.n_kv_heads * b.cap * c.head_dim;  // the V staging plane follows the K one
  for (int l = 0; l < c.n_layers; ++l) {
    const LayerW& lw = e->layers[l];
    bf16* kc = q8 ? e->q8_stage : e->kptr(l, e->kv_row);
    bf16* vc = q8 ? e->q8_stage + stage_v : e->vptr(l, e->kv_row);
    if ((rc = launch_qkv(d, lw, e->h, e->qbuf, kc, vc, e->st, e->lm_inv_freq, s, e->qk_norm ? e->qn[l] : nullptr,
                         e->qk_norm ? e->kn[l] : nullptr)))
      return rc;
    AttnKv kv{kc, vc};
    if (q8) {
      kv.k8 = e->q8_plane(b.q8, l, 0, e->kv_row, b.rows, b.cap);
      kv.v8 = e->q8_plane(b.q8, l, 1, e->kv_row, b.rows, b.cap);
    }
    if ((rc = launch_attn(d, e->qbuf, kv, e->attn, e->st, e->attn_cluster, s))) return rc;
    if ((rc = launch_res(lw.wo, e->attn, e->h, c.hidden, c.n_heads * c.head_dim, s))) return rc;
    if ((rc = launch_gateup(d, lw, e->h, e->act, s))) return rc;
    if ((rc = launch_res(lw.wd, e->act, e->h, c.hidden, c.inter, s))) return rc;
  }
  if ((rc = launch_head(d, e->norm, e->head, e->h, e->logits, e->partials, s))) return rc;
  if ((rc = launch_sample(d, e->logits, e->partials, e->logprobs, e->embed, e->h, e->st,
                          e->token_log, e->log_cap, e->force, 1, s)))
    return rc;
  return B200_OK;
}

static int kernels_per_step(const b200_engine* e) {
  return e->active_mega() ? 1 : e->cfg.n_layers * (e->qk_norm ? 6 : 5) + 2;
}


// ---------------------------------------------------------------------------------------------
// prefill / vision path: weight-major GEMMs (gemm_wt.cu), split-K partials finished by
// finish_rows (bias + residual + the NEXT norm fused), pipelined attention (attention_fa.cu)
// ---------------------------------------------------------------------------------------------
static long align256(long x) { return (x + 255) & ~255L; }
static const long WT_PARTIAL_BYTES = 48L << 20;  // fp32 split-K partial tiles (bounded: see gemm_wt_auto)
static long round8(long x) { return (x + 7) & ~7L; }

// Workspace layout, the one place that knows it: byte offsets of the buffers of an LM prefill of T tokens
// and of a vision tower call of N patches.  Both start at the workspace base; the fp32 split-K partials
// (ws_partial) sit at its end.
struct WsCarver {
  long end = 0;
  long take(long bytes) {
    const long at = end;
    end += align256(bytes);
    return at;
  }
};
struct LmWs {
  long h, xn, qkv, att, act, pos, vt, kws, end;
};
static LmWs lm_ws(const b200_qwen2vl_config& c, long T) {
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim, QH = (long)c.n_heads * c.head_dim;
  WsCarver w;
  LmWs o;
  o.h = w.take(T * c.hidden * 2);    // residual stream (graph input: the embeddings)
  o.xn = w.take(T * c.hidden * 2);   // normalised rows
  o.qkv = w.take(T * QKV * 2);
  o.att = w.take(T * QH * 2);
  // T x 2 x inter bf16 that no kernel addresses.  Without it the batched prefill of
  // test_qwen3_vl_gpu::test_lock_step_rows_equal_single_requests[tiny] samples a wrong first token (the same
  // bytes placed after `kws` also pass): kept until that dependency is found.  No kernel of a one-layer prefill
  // touches these bytes: with the workspace filled with NaN before each call, single prefills (fresh prompt, later
  // chunk, a 3600-token prompt) and batched prefills (Qwen2-VL-2B / 7B and Qwen3-VL head geometries) leave them NaN,
  // and no NaN reaches their outputs (tests/test_prefill_attention_gpu.py checks both).  Without the pad that test
  // still samples token 0, for a sequence of its second batched prefill (two layers, head_dim 64).
  w.take(T * 2L * c.inter * 2);
  o.act = w.take(T * c.inter * 2);   // SwiGLU output
  o.pos = w.take(3L * T * 4);        // position ids (graph input)
  o.vt = w.take((long)c.n_kv_heads * c.head_dim * round8(T) * 2);  // V^T of the prompt chunk
  o.kws = w.take((long)c.n_kv_heads * c.head_dim * T * 2);         // rotated K of the prompt chunk
  o.end = w.end;
  return o;
}
struct TowerWs {
  long x, h, y, qkv, mlp, att, vt, xin, fout, end;
};
static TowerWs tower_ws(const b200_qwen2vl_config& c, long N) {
  const long E = c.v_embed;
  WsCarver w;
  TowerWs o;
  o.x = w.take(N * c.v_patch_dim * 2);  // bf16 patches, then the rotary cos / sin table
  o.h = w.take(N * E * 2);
  o.y = w.take(N * E * 2);
  o.qkv = w.take(N * 3 * E * 2);
  o.mlp = w.take(N * (long)c.v_mlp * 2);
  o.att = w.take(N * E * 2);
  o.vt = w.take(E * round8(N) * 2);                // V^T of the tower
  o.xin = w.take(N * c.v_patch_dim * 4);           // staged fp32 pixel_values (graph input)
  o.fout = w.take((N / ((long)c.v_merge * c.v_merge) + 1) * c.v_out * 2);  // staged features (graph output)
  o.end = w.end;
  return o;
}
// creation-time helper: a bf16 buffer of -inf (the padding of logits rows beyond an odd vocabulary)
static int fill_bf16_neg_inf(void* dst, long n) {
  std::vector<uint16_t> host((size_t)n, (uint16_t)0xFF80);
  B200_CUDA(cudaMemcpy(dst, host.data(), (size_t)n * 2, cudaMemcpyHostToDevice));
  return B200_OK;
}
static float* ws_partial(b200_engine* e) {
  return reinterpret_cast<float*>(e->ws + ((e->ws_bytes - WT_PARTIAL_BYTES - 2048) & ~255L));
}

// y = epi(bf16(x . W^T + b))
static int linear(b200_engine* e, const bf16* x, long ldx, const bf16* W, const bf16* b, bf16* y, long ldy,
                  int T, int N, int K, int epi, cudaStream_t s) {
  e->launches += 1;
  return gemm_wt_tuned(x, ldx, W, b, nullptr, 0, y, ldy, nullptr, 0, T, N, K, epi, B200_WT_BF16, 0, false,
                       e->sm_count, nullptr, s);
}

// h = bf16(h + bf16(x . W^T + b)); xn = norm(h)   (split-K GEMM + one finishing row op)
static int linear_residual_norm(b200_engine* e, const bf16* x, long ldx, const bf16* W, const bf16* b,
                                bf16* h, long ldh, int norm_kind, const bf16* nw, const bf16* nb, float eps,
                                bf16* xn, long ldxn, int T, int N, int K, cudaStream_t s) {
  float* P = ws_partial(e);
  int split = 1;
  int rc;
  e->launches += 2;
  if ((long)T * N * 4 > WT_PARTIAL_BYTES) {
    // many tokens (a long chunk or a batched prefill): even one fp32 partial tile set does not fit the partial
    // region, and with this many token tiles split-K is not needed to fill the SMs either: bias + residual fused in
    // the bf16 epilogue (same rounding points as finish_rows), then the norm as its own row op
    if ((rc = gemm_wt_tuned(x, ldx, W, b, h, ldh, h, ldh, nullptr, 0, T, N, K, B200_EPI_NONE, B200_WT_BF16, 0, false,
                            e->sm_count, nullptr, s)))
      return rc;
    if (norm_kind == B200_NORM_RMS) return rms_norm(h, nw, xn, T, N, eps, s);
    if (norm_kind == B200_NORM_LN) return layer_norm(h, nw, nb, xn, T, N, eps, s);
    return B200_OK;
  }
  rc = gemm_wt_tuned(x, ldx, W, nullptr, nullptr, 0, nullptr, 0, P, WT_PARTIAL_BYTES, T, N, K, B200_EPI_NONE,
                     B200_WT_PARTIAL, 0, true, e->sm_count, &split, s);
  if (rc) return rc;
  return finish_rows(P, split, b, h, ldh, h, ldh, norm_kind, nw, nb, eps, xn, ldxn, T, N, s);
}

static int upload_pos(b200_engine* e, const std::vector<int>& pos, cudaStream_t s) {
  const long n = (long)pos.size();
  if (n > e->pos_hw_cap) {
    if (e->pos_hw) B200_CUDA(cudaFree(e->pos_hw));
    B200_CUDA(cudaMalloc(&e->pos_hw, n * 4));
    e->pos_hw_cap = n;
  }
  if (!e->pos_ev) B200_CUDA(cudaEventCreateWithFlags(&e->pos_ev, cudaEventDisableTiming));
  else B200_CUDA(cudaEventSynchronize(e->pos_ev));  // the previous call's copy has long finished
  if (n > e->pos_hw_host_cap) {
    if (e->pos_hw_host) B200_CUDA(cudaFreeHost(e->pos_hw_host));
    B200_CUDA(cudaMallocHost(&e->pos_hw_host, n * 4));
    e->pos_hw_host_cap = n;
  }
  memcpy(e->pos_hw_host, pos.data(), n * 4);
  B200_CUDA(cudaMemcpyAsync(e->pos_hw, e->pos_hw_host, n * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaEventRecord(e->pos_ev, s));
  return B200_OK;
}

static int upload_loc(b200_engine* e, const std::vector<int>& loc, cudaStream_t s) {
  const long n = (long)loc.size();
  if (!e->loc_ev) B200_CUDA(cudaEventCreateWithFlags(&e->loc_ev, cudaEventDisableTiming));
  else B200_CUDA(cudaEventSynchronize(e->loc_ev));  // the previous prefill that read the table has finished
  if (n > e->loc_cap) {
    if (e->loc_dev) B200_CUDA(cudaFree(e->loc_dev));
    B200_CUDA(cudaMalloc(&e->loc_dev, n * 4));
    e->loc_cap = n;
  }
  if (n > e->loc_host_cap) {
    if (e->loc_host) B200_CUDA(cudaFreeHost(e->loc_host));
    B200_CUDA(cudaMallocHost(&e->loc_host, n * 4));
    e->loc_host_cap = n;
  }
  memcpy(e->loc_host, loc.data(), n * 4);
  B200_CUDA(cudaMemcpyAsync(e->loc_dev, e->loc_host, n * 4, cudaMemcpyHostToDevice, s));
  return B200_OK;
}

// rot_pos_emb ids (vision.py:219-249), host side, merge-group-major order
static void build_pos_hw(const int* grid, int n_img, int ms, std::vector<int>* out) {
  out->clear();
  for (int i = 0; i < n_img; ++i) {
    const int t = grid[i * 3], h = grid[i * 3 + 1], w = grid[i * 3 + 2];
    for (int tt = 0; tt < t; ++tt)
      for (int bh = 0; bh < h / ms; ++bh)
        for (int bw = 0; bw < w / ms; ++bw)
          for (int ih = 0; ih < ms; ++ih)
            for (int iw = 0; iw < ms; ++iw) {
              out->push_back(bh * ms + ih);
              out->push_back(bw * ms + iw);
            }
  }
}


// Run `body` (a fixed sequence of launches on stream s) eagerly the first time a key is seen (the GEMM
// configurations are measured then), capture + instantiate it the second time, replay it afterwards.
template <class F>
static int seq_run(b200_engine* e, std::vector<b200_engine::SeqGraph>& cache, const std::vector<long>& key,
                   cudaStream_t s, F body) {
  b200_engine::SeqGraph* g = nullptr;
  for (auto& c : cache)
    if (c.key == key) g = &c;
  if (!g) {
    if (cache.size() >= 8) {
      if (cache.front().exec) cudaGraphExecDestroy(cache.front().exec);
      cache.erase(cache.begin());
    }
    cache.emplace_back();
    g = &cache.back();
    g->key = key;
  }
  if (g->exec) {
    B200_CUDA(cudaGraphLaunch(g->exec, s));
    e->launches += g->n_launch;
    return B200_OK;
  }
  if (g->seen++ == 0) return body();
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  if (cap != cudaStreamCaptureStatusNone) return body();  // already inside somebody else's capture
  const long l0 = e->launches;
  cudaGraph_t graph = nullptr;
  B200_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  const int rc = body();
  const cudaError_t ce = cudaStreamEndCapture(s, &graph);
  if (rc) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (ce != cudaSuccess) return cuda_fail(ce, "cudaStreamEndCapture(sequence)", __FILE__, __LINE__);
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ci = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ci != cudaSuccess) return cuda_fail(ci, "cudaGraphInstantiate(sequence)", __FILE__, __LINE__);
  g->exec = exec;
  g->n_launch = e->launches - l0;
  B200_CUDA(cudaGraphLaunch(exec, s));
  return B200_OK;
}

static int vision_body(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                       void* feats_out, cudaStream_t s);

static int vision(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                  void* feats_out, cudaStream_t s) {
  const auto& c = e->cfg;
  // graph input / output live at fixed workspace addresses: stage them around the captured body
  const TowerWs w = tower_ws(c, N);
  float* xin = (float*)(e->ws + w.xin);
  bf16* fout = (bf16*)(e->ws + w.fout);
  const long Nm = N / ((long)c.v_merge * c.v_merge);
  int rc;
  std::vector<int> pos;
  build_pos_hw(grid, n_images, c.v_merge, &pos);
  if ((rc = upload_pos(e, pos, s))) return rc;
  B200_CUDA(cudaMemcpyAsync(xin, pixel_values, (size_t)N * c.v_patch_dim * 4, cudaMemcpyDeviceToDevice, s));
  std::vector<long> key = {(long)(uintptr_t)e->ws, (long)e->ws_bytes, N, (long)n_images, (long)(uintptr_t)e->pos_hw};
  for (int i = 0; i < n_images * 3; ++i) key.push_back(grid[i]);
  rc = seq_run(e, e->vis_graphs, key, s, [&]() { return vision_body(e, xin, grid, n_images, N, fout, s); });
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(feats_out, fout, (size_t)Nm * c.v_out * 2, cudaMemcpyDeviceToDevice, s));
  return B200_OK;
}

static int vision_body(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                       void* feats_out, cudaStream_t s) {
  const auto& c = e->cfg;
  const long E = c.v_embed, Em = c.v_mlp;
  const int nh = c.v_heads, hd = c.v_embed / c.v_heads;
  const int t_ld = (int)round8(N);
  const TowerWs w = tower_ws(c, N);
  bf16* x = (bf16*)(e->ws + w.x);
  bf16* h = (bf16*)(e->ws + w.h);
  bf16* y = (bf16*)(e->ws + w.y);
  bf16* qkv = (bf16*)(e->ws + w.qkv);
  bf16* mlp = (bf16*)(e->ws + w.mlp);
  bf16* att = (bf16*)(e->ws + w.att);
  bf16* vt = (bf16*)(e->ws + w.vt);
  int rc;
  if ((rc = cast_f32_bf16(pixel_values, x, N * c.v_patch_dim, s))) return rc;
  if ((rc = linear(e, x, c.v_patch_dim, e->v_patch, nullptr, h, E, (int)N, (int)E, c.v_patch_dim, B200_EPI_NONE, s)))
    return rc;
  if ((rc = layer_norm(h, e->vblk[0].ln1w, e->vblk[0].ln1b, y, (int)N, (int)E, c.v_ln_eps, s))) return rc;
  e->launches += 2;
  const float scale = 1.0f / sqrtf((float)hd);
  // the patch input `x` is dead after the patch-embed GEMM: its workspace holds the rotary cos / sin table
  void* rope_cs = nullptr;
  if ((long)N * (hd / 2) * 8 <= N * (long)c.v_patch_dim * 2) {
    rope_cs = x;
    if ((rc = vision_rope_table(e->pos_hw, e->v_inv_freq, (int)N, hd, rope_cs, s))) return rc;
    e->launches += 1;
  }
  bool fa = attention_fa_supported(qkv, 3 * E, hd, qkv + E, 3 * E, hd, vt, (long)hd * t_ld, t_ld, att, E, hd);
  {  // the pipelined kernel loads V^T tiles with tokens innermost: a segment must start on a 16-byte boundary
     // (8 tokens); frames with other offsets (e.g. a 6 x 6-patch image followed by another) take `attention()`
    long o = 0;
    for (int im = 0; im < n_images && fa; ++im)
      for (int tt = 0; tt < grid[im * 3]; ++tt) {
        if (o % 8) fa = false;
        o += (long)grid[im * 3 + 1] * grid[im * 3 + 2];
      }
  }
  for (int i = 0; i < c.v_depth; ++i) {
    const VBlk& b = e->vblk[i];
    if ((rc = linear(e, y, E, b.qkvw, b.qkvb, qkv, 3 * E, (int)N, (int)(3 * E), (int)E, B200_EPI_NONE, s))) return rc;
    if (fa) {
      if ((rc = vision_qkv_post(qkv, e->pos_hw, e->v_inv_freq, (int)N, nh, hd, scale, vt, t_ld, s, rope_cs))) return rc;
    } else {
      if ((rc = vision_rope(qkv, e->pos_hw, e->v_inv_freq, (int)N, nh, hd, s))) return rc;
    }
    e->launches += 1;
    long off = 0;
    for (int im = 0; im < n_images; ++im) {
      const int t = grid[im * 3];
      const int seg = grid[im * 3 + 1] * grid[im * 3 + 2];
      for (int tt = 0; tt < t; ++tt) {  // one attention segment per frame (vision.py:270-281)
        if (fa) {
          rc = attention_fa(qkv, 3 * E, hd, qkv + E, 3 * E, hd, vt, (long)hd * t_ld, t_ld, att, E, nh, nh, hd, seg,
                            seg, 0, s, (int)off, (int)N, (int)off, (int)N);
        } else {
          const bf16* qb = qkv + off * 3 * E;
          rc = attention(qb, 3 * E, hd, qb + E, 3 * E, hd, qb + 2 * E, 3 * E, hd, att + off * E, E, nh, nh, hd,
                         seg, seg, 0, scale, s);
        }
        if (rc) return rc;
        off += seg;
        e->launches += 1;
      }
    }
    if ((rc = linear_residual_norm(e, att, E, b.projw, b.projb, h, E, B200_NORM_LN, b.ln2w, b.ln2b, c.v_ln_eps,
                                   y, E, (int)N, (int)E, (int)E, s)))
      return rc;
    if ((rc = linear(e, y, E, b.fc1w, b.fc1b, mlp, Em, (int)N, (int)Em, (int)E, B200_EPI_GELU_FAST, s))) return rc;
    const bool last = (i + 1 == c.v_depth);
    const bf16* nw = last ? e->m_lnw : e->vblk[i + 1].ln1w;
    const bf16* nb = last ? e->m_lnb : e->vblk[i + 1].ln1b;
    if ((rc = linear_residual_norm(e, mlp, Em, b.fc2w, b.fc2b, h, E, B200_NORM_LN, nw, nb,
                                   last ? 1e-6f : c.v_ln_eps, y, E, (int)N, (int)E, (int)Em, s)))
      return rc;
  }
  // PatchMerger (vision.py:105-120): y already holds LayerNorm(h) of the last block
  const long mg = (long)c.v_merge * c.v_merge * E;
  const long Nm = N / ((long)c.v_merge * c.v_merge);
  if ((rc = linear(e, y, mg, e->m_fc1w, e->m_fc1b, mlp, mg, (int)Nm, (int)mg, (int)mg, B200_EPI_GELU_EXACT, s)))
    return rc;
  if ((rc = linear(e, mlp, mg, e->m_fc2w, e->m_fc2b, (bf16*)feats_out, c.v_out, (int)Nm, c.v_out, (int)mg,
                   B200_EPI_NONE, s)))
    return rc;
  return B200_OK;
}

// one sequence of a batched prefill: tokens [off, off + T) of the concatenated batch go to KV pool row `row`
struct PreSeg { int off, T, row; };

static int prefill_layers_body(b200_engine* e, const int* pos3, int T, int ctx0, void* all_logits_out,
                               cudaStream_t s, const PreSeg* segs = nullptr, int n_seg = 0,
                               const void* tok_loc = nullptr);

static int prefill_layers(b200_engine* e, const void* embeds, const int* pos3, int T, int ctx0,
                          void* all_logits_out, cudaStream_t s) {
  const auto& c = e->cfg;
  const LmWs w = lm_ws(c, T);
  int* pos_stage = (int*)(e->ws + w.pos);
  // graph inputs at fixed workspace addresses: the embeddings (residual stream) and the position ids
  B200_CUDA(cudaMemcpyAsync(e->ws + w.h, embeds, (size_t)T * c.hidden * 2, cudaMemcpyDeviceToDevice, s));
  B200_CUDA(cudaMemcpyAsync(pos_stage, pos3, (size_t)3 * T * 4, cudaMemcpyDeviceToDevice, s));
  // where the cache lives travels through device memory (the captured graph survives a new pool)
  if (!e->kvref) {
    B200_CUDA(cudaMalloc(&e->kvref, sizeof(KvRef)));
    B200_CUDA(cudaMallocHost(&e->kvref_host, sizeof(KvRef)));
    B200_CUDA(cudaEventCreateWithFlags(&e->kvref_ev, cudaEventDisableTiming));
  } else {
    B200_CUDA(cudaEventSynchronize(e->kvref_ev));
  }
  e->kvref_host->k0 = e->kptr(0, e->kv_row);
  e->kvref_host->v_off = e->kv_off(0, 1, 0);
  e->kvref_host->layer_stride = e->kv_off(1, 0, 0);
  e->kvref_host->cap = e->kvb.cap;
  B200_CUDA(cudaMemcpyAsync(e->kvref, e->kvref_host, sizeof(KvRef), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaEventRecord(e->kvref_ev, s));
  if (all_logits_out || ctx0 != 0 || e->wt)  // all-row logits / a later chunk / 8-bit write-through: plain launches
    return prefill_layers_body(e, pos_stage, T, ctx0, all_logits_out, s);
  const std::vector<long> key = {(long)(uintptr_t)e->ws, (long)e->ws_bytes, (long)T};
  return seq_run(e, e->pre_graphs, key, s, [&]() { return prefill_layers_body(e, pos_stage, T, 0, nullptr, s); });
}

// segs == nullptr: ONE sequence bound to e->kv_row (graph-capturable: the cache is addressed through e->kvref).
// segs != nullptr (PromptProcessingBatch, ar.py:1581-2175): several fresh sequences concatenated along the token
// axis — every GEMM / norm / SwiGLU runs once over all T tokens (the weights are streamed once for the whole
// batch), M-RoPE + KV append scatter each token to (its row, its position) through `tok_loc`, and attention runs
// per sequence on its own block of the shared q / K / V^T buffers (block-diagonal causal).
static int prefill_layers_body(b200_engine* e, const int* pos3, int T, int ctx0, void* all_logits_out,
                               cudaStream_t s, const PreSeg* segs, int n_seg, const void* tok_loc) {
  const auto& c = e->cfg;
  const long H = c.hidden, I = c.inter, QH = (long)c.n_heads * c.head_dim;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  const int hd = c.head_dim, t_ld = (int)round8(T);
  const LmWs w = lm_ws(c, T);
  bf16* h = (bf16*)(e->ws + w.h);
  bf16* xn = (bf16*)(e->ws + w.xn);
  bf16* qkv = (bf16*)(e->ws + w.qkv);
  bf16* att = (bf16*)(e->ws + w.att);
  bf16* act = (bf16*)(e->ws + w.act);
  bf16* vt = (bf16*)(e->ws + w.vt);
  bf16* kws = (bf16*)(e->ws + w.kws);
  int rc;
  if ((rc = rms_norm(h, e->layers[0].ln1, xn, T, (int)H, c.rms_eps, s))) return rc;
  e->launches += 1;
  const float scale = 1.0f / sqrtf((float)hd);
  const float scale_bf = __bfloat162float(__float2bfloat16_rn(scale));
  const int S = ctx0 + T, cap = e->kvb.cap;
  for (int l = 0; l < c.n_layers; ++l) {
    const LayerW& lw = e->layers[l];
    bf16* kc = e->kptr(l, e->kv_row);
    bf16* vc = e->vptr(l, e->kv_row);
    if ((rc = linear(e, xn, H, lw.wqkv, lw.bqkv, qkv, QKV, T, (int)QKV, (int)H, B200_EPI_NONE, s))) return rc;
    if (e->qk_norm) {
      if ((rc = qk_norm(qkv, T, c.n_heads, c.n_kv_heads, hd, e->qn[l], e->kn[l], c.rms_eps, s))) return rc;
      e->launches += 1;
    }
    // the pipelined kernel needs V^T of EVERY key: available for a fresh prompt (ctx0 == 0).  It then
    // reads the chunk's own rotated K copy and V^T from the workspace, and the cache is addressed through
    // e->kvref: nothing about the KV pool is baked into the captured graph.
    const bool fa = ctx0 == 0 && !e->wt && attention_fa_supported(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld,
                                                        t_ld, att, QH, hd);
    if (segs) {
      B200_REQUIRE(fa, "prefill_batch: the pipelined attention kernel does not support this geometry");
      if ((rc = mrope_kv_write(qkv, pos3, e->lm_inv_freq, e->axis_sel, e->kptr(l, 0), e->vptr(l, 0), T, 0, cap,
                               c.n_heads, c.n_kv_heads, hd, s, scale_bf, vt, t_ld, nullptr, l, kws, tok_loc,
                               e->kv_off(0, 0, 1))))
        return rc;
      // all sequences in ONE launch: the (q0, Lq, k0, S) table follows the (row, position) table in `tok_loc`
      int longest = 0;
      for (int g = 0; g < n_seg; ++g) longest = segs[g].T > longest ? segs[g].T : longest;
      if ((rc = attention_fa(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld, t_ld, att, QH, c.n_heads,
                             c.n_kv_heads, hd, longest, longest, 1, s, 0, T, 0, T, (const int*)tok_loc + 2L * T, n_seg)))
        return rc;
      e->launches += 2;
    } else {
    if ((rc = mrope_kv_write(qkv, pos3, e->lm_inv_freq, e->axis_sel, kc, vc, T, ctx0, cap, c.n_heads,
                             c.n_kv_heads, hd, s, fa ? scale_bf : 0.f, fa ? vt : nullptr, t_ld,
                             fa ? e->kvref : nullptr, l, fa ? kws : nullptr)))
      return rc;
    if (e->wt && l < e->wt->n_layers) {  // an 8-bit layer: the chunk's rows are quantized before they are attended
      const KvWriteThrough& w8 = *e->wt;
      if ((rc = kvq_quantize_rows(kc, cap, e->q8_plane(w8.q8, l, 0, w8.row, w8.rows, w8.cap), w8.cap, c.n_kv_heads,
                                  ctx0, T, hd, true, s)) ||
          (rc = kvq_quantize_rows(vc, cap, e->q8_plane(w8.q8, l, 1, w8.row, w8.rows, w8.cap), w8.cap, c.n_kv_heads,
                                  ctx0, T, hd, true, s)))
        return rc;
      e->launches += 2;
    }
    if (fa) {
      rc = attention_fa(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld, t_ld, att, QH, c.n_heads,
                        c.n_kv_heads, hd, T, S, 1, s, 0, T, 0, S);
    } else {
      rc = attention(qkv, QKV, hd, kc, hd, (long)cap * hd, vc, hd, (long)cap * hd, att, QH, c.n_heads,
                     c.n_kv_heads, hd, T, S, 1, scale, s);
    }
    if (rc) return rc;
    e->launches += 2;
    }
    if ((rc = linear_residual_norm(e, att, QH, lw.wo, nullptr, h, H, B200_NORM_RMS, lw.ln2, nullptr, c.rms_eps, xn,
                                   H, T, (int)H, (int)QH, s)))
      return rc;
    {  // gate/up with SwiGLU fused in the epilogue
      if ((rc = gemm_wt_tuned(xn, H, lw.wgu, nullptr, nullptr, 0, act, I, nullptr, 0, T, (int)(2 * I), (int)H,
                              B200_EPI_NONE, B200_WT_SWIGLU, (int)I, false, e->sm_count, nullptr, s)))
        return rc;
      e->launches += 1;
    }
    const bool last = (l + 1 == c.n_layers);
    const bool want_norm = !last || all_logits_out;
    const bf16* nw = last ? e->norm : e->layers[l + 1].ln1;
    if ((rc = linear_residual_norm(e, act, I, lw.wd, nullptr, h, H, want_norm ? B200_NORM_RMS : B200_NORM_NONE, nw,
                                   nullptr, c.rms_eps, xn, H, T, (int)H, (int)I, s)))
      return rc;
  }
  if (all_logits_out) {  // the reference computes the head on every row (ar.py:358); xn = final norm
    // rows of the caller's buffer are round8(vocab) apart (16-byte aligned rows for any vocabulary)
    if ((rc = linear(e, xn, H, e->head, nullptr, (bf16*)all_logits_out, round8(c.vocab), T, c.vocab, (int)H,
                     B200_EPI_NONE, s)))
      return rc;
  }
  return B200_OK;
}

static bool kvq_group_ok(const b200_engine* e, int gs) {
  return (gs == 32 || gs == 64 || gs == 128) && e->cfg.head_dim % gs == 0;
}

// The one place the KV binding changes (the entry points have checked their arguments).  The decode graph is dropped
// when the binding differs from the bound one, a write-through is cleared, the 8-bit decode staging planes exist for
// the q8 kind only, and a selected row the new pool does not have goes back to row 0.
static int bind(b200_engine* e, const KvBinding& b) {
  if (!(b == e->kvb)) invalidate_graph(e);  // a row reset below also changes the rows
  e->wt.reset();
  if (e->kv_row >= b.rows) e->kv_row = 0;
  const long stage = b.kind == KvKind::q8 ? 2L * e->cfg.n_kv_heads * b.cap * e->cfg.head_dim : 0;
  if (stage > e->q8_stage_elems || (stage == 0 && e->q8_stage)) {
    e->kvb = KvBinding{};  // nothing is bound until the staging planes are in place
    if (e->q8_stage) B200_CUDA(cudaFree(e->q8_stage));
    e->q8_stage = nullptr;
    e->q8_stage_elems = 0;
    if (stage) B200_CUDA(cudaMalloc(&e->q8_stage, (size_t)stage * sizeof(bf16)));
    e->q8_stage_elems = stage;
  }
  e->kvb = b;
  return B200_OK;
}

static int set_write_through(b200_engine* e, const char* fn, void* codes, void* scales, void* biases, int group_size,
                             int rows, int cap, int row, int n_layers) {
  B200_REQUIRE(e->kvb.kind == KvKind::bf16, "%s: bind the bf16 pool first", fn);
  B200_REQUIRE(codes && scales && biases && rows >= 1 && cap >= 1 && row >= 0 && row < rows, "%s: bad arguments", fn);
  B200_REQUIRE(n_layers >= 1 && n_layers <= e->cfg.n_layers, "%s: %d 8-bit layers of %d", fn, n_layers,
               e->cfg.n_layers);
  B200_REQUIRE(kvq_group_ok(e, group_size), "%s: group size %d must be 32, 64 or 128 and divide head_dim %d", fn,
               group_size, e->cfg.head_dim);
  e->wt = KvWriteThrough{KvqPlanes{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size}, rows, cap, row, n_layers};
  return B200_OK;
}

extern "C" {

const char* b200_last_error(void) { return g_err; }
int b200_abi_version(void) { return B200_ABI_VERSION; }

int b200_device_check(int device, int* sm_count) {
  cudaDeviceProp prop;
  B200_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
              prop.minor);
    return B200_ERR_UNSUPPORTED;
  }
  if (sm_count) *sm_count = prop.multiProcessorCount;
  return B200_OK;
}

int b200_engine_create(const b200_qwen2vl_config* cfg, int device, b200_engine** out) {
  B200_REQUIRE(cfg && out, "engine_create: null argument");
  // the vocabulary may be any size (Idefics2: 32003): logits / logprobs rows are allocated to the next
  // multiple of 8 with the tail preset to -inf, which the vectorised sampler passes read as "never wins"
  B200_REQUIRE(cfg->hidden % 8 == 0 && cfg->inter % 8 == 0 && cfg->vocab > 0 &&
                   cfg->head_dim % 8 == 0 && cfg->n_heads % cfg->n_kv_heads == 0,
               "engine_create: dims must be multiples of 8 (hidden=%d inter=%d)",
               cfg->hidden, cfg->inter);
  int sm = 0;
  int rc = b200_device_check(device, &sm);
  if (rc) return rc;
  B200_CUDA(cudaSetDevice(device));
  b200_engine* e = new b200_engine();
  e->cfg = *cfg;
  e->device = device;
  e->sm_count = sm;
  decode_set_sm_count(sm);
  const auto& c = e->cfg;
  B200_CUDA(cudaMalloc(&e->st, sizeof(DecState)));
  B200_CUDA(cudaMemset(e->st, 0, sizeof(DecState)));
  B200_CUDA(cudaMalloc(&e->h, (size_t)c.hidden * 2));
  B200_CUDA(cudaMalloc(&e->qbuf, (size_t)c.n_heads * c.head_dim * 2));
  B200_CUDA(cudaMalloc(&e->attn, (size_t)c.n_heads * c.head_dim * 2));
  B200_CUDA(cudaMalloc(&e->act, (size_t)c.inter * 2));
  B200_CUDA(cudaMalloc(&e->logits, (size_t)round8(c.vocab) * 2));
  B200_CUDA(cudaMalloc(&e->logprobs, (size_t)round8(c.vocab) * 2));
  if ((rc = fill_bf16_neg_inf(e->logits, round8(c.vocab))) || (rc = fill_bf16_neg_inf(e->logprobs, round8(c.vocab))))
    return rc;
  B200_CUDA(cudaMalloc(&e->partials, (size_t)sm * 8 * sizeof(float2)));
  B200_CUDA(cudaMalloc(&e->token_log, (size_t)e->log_cap * 4));
  B200_CUDA(cudaMalloc(&e->force, (size_t)e->log_cap * 4));
  B200_CUDA(cudaMemset(e->token_log, 0, (size_t)e->log_cap * 4));
  B200_CUDA(cudaMemset(e->force, 0, (size_t)e->log_cap * 4));
  B200_CUDA(cudaMalloc(&e->lm_inv_freq, (size_t)(c.head_dim / 2) * 4));
  B200_CUDA(cudaMalloc(&e->axis_sel, (size_t)(c.head_dim / 2) * 4));
  const int vhd = c.v_embed / c.v_heads;
  B200_CUDA(cudaMalloc(&e->v_inv_freq, (size_t)(vhd / 4 > 0 ? vhd / 4 : 1) * 4));
  // default rope tables (the Python host overrides them with its own fp32 values so
  // that they are bit-identical to what it hands to the oracle / reference formula)
  std::vector<float> f(c.head_dim / 2);
  for (int i = 0; i < c.head_dim / 2; ++i)
    f[i] = 1.0f / powf(c.rope_theta, (float)(2 * i) / (float)c.head_dim);
  B200_CUDA(cudaMemcpy(e->lm_inv_freq, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
  std::vector<int> sel(c.head_dim / 2, 0);
  {  // _chunked_position_selector, rope_utils.py:519-526
    int off = c.mrope_section[0];
    for (int dim = 1; dim < 3; ++dim) {
      for (int i = off; i < off + c.mrope_section[dim] && i < c.head_dim / 2; ++i) sel[i] = dim;
      off += c.mrope_section[dim];
    }
  }
  B200_CUDA(cudaMemcpy(e->axis_sel, sel.data(), sel.size() * 4, cudaMemcpyHostToDevice));
  std::vector<float> vf(vhd / 4 > 0 ? vhd / 4 : 1);
  for (int i = 0; i < (int)vf.size(); ++i)
    vf[i] = 1.0f / powf(10000.0f, (float)(2 * i) / (float)(vhd / 2));
  B200_CUDA(cudaMemcpy(e->v_inv_freq, vf.data(), vf.size() * 4, cudaMemcpyHostToDevice));
  B200_CUDA(cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking));
  B200_CUDA(cudaEventCreate(&e->ev0));
  B200_CUDA(cudaEventCreate(&e->ev1));
  *out = e;
  return B200_OK;
}

int b200_engine_destroy(b200_engine* e) {
  if (!e) return B200_OK;
  cudaSetDevice(e->device);
  invalidate_graph(e);
  drop_seq_graphs(e);
  cudaFree(e->st); cudaFree(e->h); cudaFree(e->qbuf); cudaFree(e->attn); cudaFree(e->act);
  cudaFree(e->logits); cudaFree(e->logprobs); cudaFree(e->partials); cudaFree(e->token_log);
  cudaFree(e->force); cudaFree(e->lm_inv_freq); cudaFree(e->axis_sel); cudaFree(e->v_inv_freq);
  if (e->pos_hw) cudaFree(e->pos_hw);
  if (e->pos_hw_host) cudaFreeHost(e->pos_hw_host);
  if (e->pos_ev) cudaEventDestroy(e->pos_ev);
  if (e->loc_dev) cudaFree(e->loc_dev);
  if (e->loc_host) cudaFreeHost(e->loc_host);
  if (e->loc_ev) cudaEventDestroy(e->loc_ev);
  if (e->kvref) cudaFree(e->kvref);
  if (e->kvref_host) cudaFreeHost(e->kvref_host);
  if (e->kvref_ev) cudaEventDestroy(e->kvref_ev);
  if (e->att_part) cudaFree(e->att_part);
  if (e->att_stats) cudaFree(e->att_stats);
  if (e->bar) cudaFree(e->bar);
  if (e->dbg) cudaFree(e->dbg);
  if (e->q8_stage) cudaFree(e->q8_stage);
  if (e->batch) batch_decoder_destroy(e->batch);
  if (e->cap_stream) cudaStreamDestroy(e->cap_stream);
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  delete e;
  return B200_OK;
}

int b200_engine_set_weight(b200_engine* e, const char* name, const void* ptr, long n_elems) {
  B200_REQUIRE(e && name && ptr, "set_weight: null argument");
  B200_REQUIRE(((uintptr_t)ptr & 15) == 0, "set_weight: '%s' must be 16-byte aligned", name);
  e->w[name] = (const bf16*)ptr;
  e->wn[name] = n_elems;
  drop_seq_graphs(e);
  e->resolved = false;
  invalidate_graph(e);
  return B200_OK;
}

int b200_engine_set_rope_tables(b200_engine* e, const float* lm_inv_freq_host,
                                const float* v_inv_freq_host) {
  B200_REQUIRE(e, "set_rope_tables: null engine");
  const auto& c = e->cfg;
  if (lm_inv_freq_host)
    B200_CUDA(cudaMemcpy(e->lm_inv_freq, lm_inv_freq_host, (size_t)(c.head_dim / 2) * 4,
                         cudaMemcpyHostToDevice));
  if (v_inv_freq_host) {
    const int vhd = c.v_embed / c.v_heads;
    B200_CUDA(cudaMemcpy(e->v_inv_freq, v_inv_freq_host, (size_t)(vhd / 4) * 4,
                         cudaMemcpyHostToDevice));
  }
  return B200_OK;
}

int b200_engine_set_axis_sel(b200_engine* e, const int* axis_sel_host) {
  B200_REQUIRE(e && axis_sel_host, "set_axis_sel: null argument");
  const int n = e->cfg.head_dim / 2;
  for (int i = 0; i < n; ++i)
    B200_REQUIRE(axis_sel_host[i] >= 0 && axis_sel_host[i] <= 2, "set_axis_sel: entry %d is %d (0, 1 or 2)", i,
                 axis_sel_host[i]);
  B200_CUDA(cudaMemcpy(e->axis_sel, axis_sel_host, (size_t)n * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

long b200_engine_workspace_bytes(const b200_engine* e, int max_tokens, int max_patches) {
  const long lm = lm_ws(e->cfg, max_tokens).end, v = tower_ws(e->cfg, max_patches).end;
  return (lm > v ? lm : v) + WT_PARTIAL_BYTES + 4096;
}

int b200_engine_set_workspace(b200_engine* e, void* ptr, long bytes) {
  B200_REQUIRE(e && ptr && bytes > 0 && ((uintptr_t)ptr & 255) == 0,
               "set_workspace: need a 256-byte aligned buffer");
  drop_seq_graphs(e);
  e->ws = (uint8_t*)ptr;
  e->ws_bytes = bytes;
  return B200_OK;
}

int b200_engine_bind_kv(b200_engine* e, void* pool, int batch, int cap) {
  B200_REQUIRE(e && pool && batch >= 1 && cap >= 1 && ((uintptr_t)pool & 15) == 0,
               "bind_kv: bad arguments");
  return bind(e, KvBinding{KvKind::bf16, (bf16*)pool, {}, 0, batch, cap});
}

int b200_engine_bind_kvq(b200_engine* e, void* codes, void* scales, void* biases, int batch, int cap,
                         int group_size) {
  B200_REQUIRE(e && codes && scales && biases && batch >= 1 && cap >= 1 && ((uintptr_t)codes & 15) == 0,
               "bind_kvq: bad arguments");
  B200_REQUIRE(kvq_group_ok(e, group_size), "bind_kvq: group size %d must be 32, 64 or 128 and divide head_dim %d",
               group_size, e->cfg.head_dim);
  const KvqPlanes q8{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  return bind(e, KvBinding{KvKind::q8, nullptr, q8, e->cfg.n_layers, batch, cap});
}

int b200_engine_bind_batch_kvq(b200_engine* e, void* codes, void* scales, void* biases, int group_size, int n_q8_layers,
                               void* bf16_pool, int batch, int cap) {
  B200_REQUIRE(e && codes && scales && biases && batch >= 1 && cap >= 1 && ((uintptr_t)codes & 15) == 0 &&
                   ((uintptr_t)bf16_pool & 15) == 0,
               "bind_batch_kvq: bad arguments");
  const auto& c = e->cfg;
  B200_REQUIRE(kvq_group_ok(e, group_size),
               "bind_batch_kvq: group size %d must be 32, 64 or 128 and divide head_dim %d", group_size, c.head_dim);
  B200_REQUIRE(n_q8_layers >= 1 && n_q8_layers <= c.n_layers && (bf16_pool != nullptr) == (n_q8_layers < c.n_layers),
               "bind_batch_kvq: %d of %d layers 8-bit needs a bf16 pool for the rest (and only then)", n_q8_layers,
               c.n_layers);
  const KvqPlanes q8{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  return bind(e, KvBinding{KvKind::q8_batch, (bf16*)bf16_pool, q8, n_q8_layers, batch, cap});
}

int b200_engine_set_prefill_kvq_row(b200_engine* e, void* codes, void* scales, void* biases, int group_size, int rows,
                                    int cap, int row, int n_q8_layers) {
  B200_REQUIRE(e, "set_prefill_kvq_row: null engine");
  return set_write_through(e, "set_prefill_kvq_row", codes, scales, biases, group_size, rows, cap, row, n_q8_layers);
}

int b200_engine_set_prefill_kvq(b200_engine* e, void* codes, void* scales, void* biases, int group_size) {
  B200_REQUIRE(e, "set_prefill_kvq: null engine");
  if (!codes) {
    e->wt.reset();
    return B200_OK;
  }
  return set_write_through(e, "set_prefill_kvq", codes, scales, biases, group_size, e->kvb.rows, e->kvb.cap, e->kv_row,
                           e->cfg.n_layers);
}

int b200_engine_vision(b200_engine* e, const float* pixel_values, const int* grid_thw_host,
                       int n_images, void* feats_out, void* stream) {
  B200_REQUIRE(e && pixel_values && grid_thw_host && n_images > 0 && feats_out,
               "engine_vision: null argument");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(!e->cfg.external_vision, "engine_vision: this engine was created without a vision tower");
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  const auto& c = e->cfg;
  long N = 0;
  for (int i = 0; i < n_images; ++i) {
    const int t = grid_thw_host[i * 3], h = grid_thw_host[i * 3 + 1], w = grid_thw_host[i * 3 + 2];
    B200_REQUIRE(t > 0 && h > 0 && w > 0 && h % c.v_merge == 0 && w % c.v_merge == 0,
                 "engine_vision: bad grid (%d,%d,%d)", t, h, w);
    N += (long)t * h * w;
  }
  B200_REQUIRE(e->ws && b200_engine_workspace_bytes(e, 1, (int)N) <= e->ws_bytes,
               "engine_vision: workspace too small for %ld patches", N);
  return vision(e, pixel_values, grid_thw_host, n_images, N, feats_out, s);
}

int b200_engine_prefill(b200_engine* e, const void* embeds, const int* pos3, int T, int ctx0,
                        int rope_delta, void* all_logits_out, void* stream) {
  B200_REQUIRE(e && embeds && pos3 && T > 0 && ctx0 >= 0, "engine_prefill: bad arguments");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(e->kvb.kind == KvKind::bf16, "engine_prefill: no bf16 KV pool bound (an 8-bit pool is decode-only)");
  B200_REQUIRE(ctx0 + T <= e->kvb.cap, "engine_prefill: ctx0+T=%d exceeds cache capacity %d",
               ctx0 + T, e->kvb.cap);
  B200_REQUIRE(!e->wt || ctx0 + T <= e->wt->cap,
               "engine_prefill: ctx0+T=%d exceeds the capacity %d of the 8-bit write-through pool", ctx0 + T,
               e->wt->cap);
  B200_REQUIRE(e->ws && b200_engine_workspace_bytes(e, T, 1) <= e->ws_bytes,
               "engine_prefill: workspace too small for %d tokens", T);
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  const auto& c = e->cfg;
  if ((rc = prefill_layers(e, embeds, pos3, T, ctx0, all_logits_out, s))) return rc;
  const bf16* h = (const bf16*)(e->ws + lm_ws(c, T).h);
  // last row through the fused head + sampler; arms the decode state
  const DecodeDims d = e->dims();
  if ((rc = decode_prepare())) return rc;
  e->ctx_host = ctx0 + T;
  e->pos_host = ctx0 + T + rope_delta;
  if ((rc = launch_set_state(e->st, 0, e->ctx_host, e->pos_host, 0, 0, e->embed, e->h, c.hidden, s)))
    return rc;
  if ((rc = launch_head(d, e->norm, e->head, h + (long)(T - 1) * c.hidden, e->logits, e->partials, s)))
    return rc;
  if ((rc = launch_sample(d, e->logits, e->partials, e->logprobs, e->embed, e->h, e->st,
                          e->token_log, e->log_cap, e->force, 0, s)))
    return rc;
  e->launches += 3;
  e->tokens_launched += 1;
  return B200_OK;
}

// PromptProcessingBatch (ar.py:1581-2175): n_seq FRESH prompts prefilled in one pass.  embeds = the sequences'
// embeddings concatenated along the token axis, EACH SEQUENCE PADDED TO A MULTIPLE OF 8 TOKENS (any finite values in
// the padding rows): [sum round8(T_g), hidden]; pos3 = (3, sum round8(T_g)) int32 device, laid out the same way;
// sequence g has seq_len[g] real tokens and fills KV pool row rows[g] from position 0.  The first token of every sequence goes through
// the fused head + sampler in order: token_log receives n_seq entries (tokens_launched += n_seq).
int b200_engine_prefill_batch(b200_engine* e, const void* embeds, const int* pos3, int n_seq, const int* seq_len,
                              const int* rows, void* stream) {
  B200_REQUIRE(e && embeds && pos3 && n_seq > 0 && seq_len && rows, "engine_prefill_batch: bad arguments");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(e->kvb.kind == KvKind::bf16, "engine_prefill_batch: no bf16 KV pool bound (an 8-bit pool is decode-only)");
  B200_REQUIRE(!e->wt, "engine_prefill_batch: no 8-bit write-through in the batched prefill");
  long T = 0;
  std::vector<PreSeg> segs(n_seq);
  for (int g = 0; g < n_seq; ++g) {
    B200_REQUIRE(seq_len[g] > 0 && seq_len[g] <= e->kvb.cap && rows[g] >= 0 && rows[g] < e->kvb.rows,
                 "engine_prefill_batch: sequence %d: %d tokens into row %d (capacity %d, %d rows)", g, seq_len[g], rows[g],
                 e->kvb.cap, e->kvb.rows);
    segs[g] = PreSeg{(int)T, seq_len[g], rows[g]};
    T += round8(seq_len[g]);   // every sequence starts at a multiple of 8 tokens: the V^T tiles are loaded by TMA
                               // with tokens innermost, and a box must start on a 16-byte boundary
  }
  B200_REQUIRE(e->ws && b200_engine_workspace_bytes(e, (int)T, 1) <= e->ws_bytes,
               "engine_prefill_batch: workspace too small for %ld tokens", T);
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  const auto& c = e->cfg;
  const long H = c.hidden;
  const LmWs w = lm_ws(c, T);
  bf16* h = (bf16*)(e->ws + w.h);
  int* pos_stage = (int*)(e->ws + w.pos);   // 3 * T ints; the tokens' (row, position) table lives in e->loc_dev
  B200_CUDA(cudaMemcpyAsync(h, embeds, (size_t)T * H * 2, cudaMemcpyDeviceToDevice, s));
  B200_CUDA(cudaMemcpyAsync(pos_stage, pos3, (size_t)3 * T * 4, cudaMemcpyDeviceToDevice, s));
  std::vector<int> loc(2 * (size_t)T, -1);   // padding tokens: row -1 = no cache write
  for (int g = 0; g < n_seq; ++g)
    for (int t = 0; t < segs[g].T; ++t) {
      loc[2 * ((size_t)segs[g].off + t)] = segs[g].row;
      loc[2 * ((size_t)segs[g].off + t) + 1] = t;
    }
  for (int g = 0; g < n_seq; ++g)   // attention segments (q0, Lq, k0, S), 16-byte aligned behind the table (T % 8 == 0)
    for (int v : {segs[g].off, segs[g].T, segs[g].off, segs[g].T}) loc.push_back(v);
  if ((rc = upload_loc(e, loc, s))) return rc;
  rc = prefill_layers_body(e, pos_stage, (int)T, 0, nullptr, s, segs.data(), n_seq, e->loc_dev);
  B200_CUDA(cudaEventRecord(e->loc_ev, s));   // the table (and its staging copy) may be rewritten after this point
  if (rc) return rc;
  const DecodeDims d = e->dims();
  if ((rc = decode_prepare())) return rc;
  for (int g = 0; g < n_seq; ++g) {   // first token of every sequence: fused head + sampler on its last row
    if ((rc = launch_set_state(e->st, 0, segs[g].T, segs[g].T, 0, 0, e->embed, e->h, c.hidden, s))) return rc;
    if ((rc = launch_head(d, e->norm, e->head, h + (long)(segs[g].off + segs[g].T - 1) * H, e->logits, e->partials, s)))
      return rc;
    if ((rc = launch_sample(d, e->logits, e->partials, e->logprobs, e->embed, e->h, e->st, e->token_log, e->log_cap,
                            e->force, 0, s)))
      return rc;
    e->launches += 3;
    e->tokens_launched += 1;
  }
  e->ctx_host = segs[n_seq - 1].T;
  e->pos_host = segs[n_seq - 1].T;
  return B200_OK;
}

int b200_engine_set_next(b200_engine* e, int token, int ctx, int position, void* stream) {
  B200_REQUIRE(e && token >= 0 && token < e->cfg.vocab && ctx >= 0, "set_next: bad arguments");
  int rc = resolve(e);
  if (rc) return rc;
  e->ctx_host = ctx;
  e->pos_host = position;
  e->launches += 1;
  return launch_set_state(e->st, token, ctx, position, 0, 1, e->embed, e->h, e->cfg.hidden,
                          (cudaStream_t)stream);
}

int b200_engine_decode(b200_engine* e, int n_steps, const int* force_tokens_host, void* stream) {
  B200_REQUIRE(e && n_steps > 0, "engine_decode: bad arguments");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(e->kvb.kind == KvKind::bf16 || e->kvb.kind == KvKind::q8, "engine_decode: KV pool not bound (a "
               "lock-step 8-bit batch pool serves b200_batch_decode only)");
  B200_REQUIRE(e->ctx_host + n_steps <= e->kvb.cap,
               "engine_decode: %d cached + %d steps exceeds cache capacity %d", e->ctx_host,
               n_steps, e->kvb.cap);
  B200_REQUIRE(n_steps < e->log_cap, "engine_decode: too many steps per call");
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  if (force_tokens_host) {
    // forced feed for the token sampled at log index n is force[n % cap]
    for (int i = 0; i < n_steps; ++i) {
      const long idx = (e->tokens_launched + i) % e->log_cap;
      B200_CUDA(cudaMemcpyAsync(e->force + idx, force_tokens_host + i, 4, cudaMemcpyHostToDevice, s));
    }
  }
  if ((rc = launch_set_state(e->st, 0, e->ctx_host, e->pos_host, force_tokens_host ? 1 : 0, 0,
                             e->embed, e->h, e->cfg.hidden, s)))
    return rc;
  if ((rc = decode_prepare())) return rc;
  if (e->use_mega && e->mega_fits && !e->mega_ready) {
    if ((rc = mega_prepare(e, s))) {
      // a geometry the persistent kernel cannot hold (very long cache: the attention scratch
      // leaves no room for the weight ring; > 132 attention CTAs; ...): same step, one kernel per
      // phase — still this library's CUDA path.  b200_last_error() keeps the reason.
      if (rc != B200_ERR_INVALID) return rc;
      e->mega_fits = false;
    }
  }
  if (!(e->use_graph && e->gexec)) {
    // the per-phase attention kernel: its capacity limit and shared memory apply to the steps it serves only, so a
    // cache that k_mega holds is not refused for being too long for k_attn
    if (!e->active_mega() && (rc = attn_prepare(e->dims(), e->attn_cluster, e->kvb.kind == KvKind::q8))) return rc;
  }
  if (e->use_graph && !e->gexec) {
    // capture one step on the engine's own stream (capture does not execute)
    cudaGraph_t graph = nullptr;
    B200_CUDA(cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeThreadLocal));
    rc = enqueue_step(e, e->cap_stream);
    cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (ce != cudaSuccess) return cuda_fail(ce, "cudaStreamEndCapture", __FILE__, __LINE__);
    ce = cudaGraphInstantiate(&e->gexec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) return cuda_fail(ce, "cudaGraphInstantiate", __FILE__, __LINE__);
  }
  B200_CUDA(cudaEventRecord(e->ev0, s));
  for (int i = 0; i < n_steps; ++i) {
    if (e->use_graph) {
      B200_CUDA(cudaGraphLaunch(e->gexec, s));
    } else {
      if ((rc = enqueue_step(e, s))) return rc;
    }
  }
  B200_CUDA(cudaEventRecord(e->ev1, s));
  e->last_steps = n_steps;
  e->timing_valid = true;
  e->ctx_host += n_steps;
  e->pos_host += n_steps;
  e->tokens_launched += n_steps;
  e->launches += (long)n_steps * kernels_per_step(e) + 1;
  return B200_OK;
}

const void* b200_engine_logits(const b200_engine* e) { return e ? e->logits : nullptr; }
const void* b200_engine_logprobs(const b200_engine* e) { return e ? e->logprobs : nullptr; }
const int* b200_engine_token_log(const b200_engine* e) { return e ? e->token_log : nullptr; }
int b200_engine_token_log_capacity(const b200_engine* e) { return e ? e->log_cap : 0; }
long b200_engine_tokens_launched(const b200_engine* e) { return e ? e->tokens_launched : 0; }
long b200_engine_launch_count(const b200_engine* e) { return e ? e->launches : 0; }
int b200_engine_set_graph(b200_engine* e, int enabled) {
  B200_REQUIRE(e, "set_graph: null engine");
  e->use_graph = enabled != 0;
  return B200_OK;
}
int b200_engine_set_mega(b200_engine* e, int enabled) {
  B200_REQUIRE(e, "set_mega: null engine");
  B200_REQUIRE(enabled == 0 || enabled == 1, "set_mega: mode %d (0: one kernel per phase, 1: k_mega)", enabled);
  e->use_mega = enabled;
  invalidate_graph(e);
  return B200_OK;
}
int b200_engine_debug_buffer(b200_engine* e, const char* name, void** ptr, long* bytes) {
  B200_REQUIRE(e && name && ptr && bytes, "debug_buffer: null argument");
  const std::string n(name);
  if (n == "h") { *ptr = e->h; *bytes = (long)e->cfg.hidden * 2; }
  else if (n == "act") { *ptr = e->act; *bytes = (long)e->cfg.inter * 2; }
  else if (n == "q") { *ptr = e->qbuf; *bytes = (long)e->cfg.n_heads * e->cfg.head_dim * 2; }
  else {
    set_error("debug_buffer: unknown or unallocated buffer '%s'", name);
    return B200_ERR_INVALID;
  }
  return B200_OK;
}
int b200_engine_device_error(b200_engine* e, int* out) {
  B200_REQUIRE(e && out, "device_error: null argument");
  DecState st;
  B200_CUDA(cudaMemcpy(&st, e->st, sizeof(st), cudaMemcpyDeviceToHost));
  *out = st.error;
  return B200_OK;
}
/* debugging aid: per-barrier globaltimer stamps of CTA 0 and the last CTA for the most
 * recent step; out_host must hold 2*1024*2 int64.  Enables stamping on first call. */
int b200_engine_mega_timeline(b200_engine* e, long long* out_host) {
  B200_REQUIRE(e, "mega_timeline: null engine");
  const size_t n = (size_t)(2 * 1024 * 2 + 256) * sizeof(long long);
  if (!e->dbg) {
    B200_CUDA(cudaMalloc(&e->dbg, n));
    B200_CUDA(cudaMemset(e->dbg, 0, n));
    invalidate_graph(e);
    return B200_OK;
  }
  if (out_host) B200_CUDA(cudaMemcpy(out_host, e->dbg, n, cudaMemcpyDeviceToHost));
  return B200_OK;
}
int b200_engine_set_pdl(b200_engine* e, int enabled) {
  B200_REQUIRE(e, "set_pdl: null engine");
  decode_set_pdl(enabled != 0);
  invalidate_graph(e);
  return B200_OK;
}
int b200_engine_set_attn_cluster(b200_engine* e, int cluster) {
  B200_REQUIRE(e && (cluster == 1 || cluster == 2 || cluster == 4 || cluster == 8),
               "set_attn_cluster: cluster must be 1, 2, 4 or 8");
  e->attn_cluster = cluster;
  invalidate_graph(e);
  return B200_OK;
}
int b200_engine_fetch_tokens(b200_engine* e, long start, int n, int* host_out, void* stream) {
  B200_REQUIRE(e && host_out && n > 0 && start >= 0 && n <= e->log_cap, "fetch_tokens: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long a = start % e->log_cap;
  const long first = (a + n <= e->log_cap) ? n : e->log_cap - a;
  B200_CUDA(cudaMemcpyAsync(host_out, e->token_log + a, (size_t)first * 4, cudaMemcpyDeviceToHost, s));
  if (first < n)
    B200_CUDA(cudaMemcpyAsync(host_out + first, e->token_log, (size_t)(n - first) * 4,
                              cudaMemcpyDeviceToHost, s));
  return B200_OK;
}
int b200_engine_set_kv_row(b200_engine* e, int row) {
  B200_REQUIRE(e && row >= 0 && (e->kvb.kind == KvKind::none || row < e->kvb.rows), "set_kv_row: row %d of %d", row,
               e ? e->kvb.rows : 0);
  if (row != e->kv_row) {  // the decode graph and a write-through were set up for the old row
    invalidate_graph(e);
    e->wt.reset();
  }
  e->kv_row = row;
  return B200_OK;
}

static void bd_model(b200_engine* e, BdModel* m) {
  const auto& c = e->cfg;
  m->d = e->dims();
  m->n_layers = c.n_layers;
  m->layers = e->layers.data();
  m->embed = e->embed; m->head = e->head; m->final_norm = e->norm;
  m->inv_freq = e->lm_inv_freq;
  const KvBinding& b = e->kvb;
  m->kv = b.kv;
  m->row_stride = e->kv_off(0, 0, 1);
  m->v_off = e->kv_off(0, 1, 0);
  m->layer_stride = e->kv_off(1, 0, 0);
  m->kv_batch = b.rows;
  m->sm_count = e->sm_count;
  m->qn = e->qk_norm ? e->qn.data() : nullptr;
  m->kn = e->qk_norm ? e->kn.data() : nullptr;
  m->q8_codes = b.q8.codes; m->q8_scales = b.q8.scales; m->q8_biases = b.q8.biases;
  m->q8_gs = b.q8.gs; m->q8_layers = b.n_q8;
}

static bool batch_kind(const b200_engine* e) {
  return e->kvb.kind == KvKind::bf16 || e->kvb.kind == KvKind::q8_batch;
}

int b200_batch_begin(b200_engine* e, int B, const int* tok, const int* ctx, const int* pos, const int* active,
                     void* stream) {
  B200_REQUIRE(e && tok && ctx && pos && active, "batch_begin: null argument");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(batch_kind(e), "batch_begin: KV pool not bound (bf16 or a lock-step 8-bit batch pool)");
  B200_CUDA(cudaSetDevice(e->device));
  BdModel m;
  bd_model(e, &m);
  if ((rc = batch_decoder_begin(&e->batch, m, B, tok, ctx, pos, active, (cudaStream_t)stream))) return rc;
  e->b_ctx.assign(ctx, ctx + B);
  e->b_active.assign(active, active + B);
  e->launches += 1;
  return B200_OK;
}

int b200_batch_decode(b200_engine* e, int n_steps, int want_logprobs, void* stream) {
  B200_REQUIRE(e && e->batch && n_steps > 0, "batch_decode: batch_begin first");
  B200_REQUIRE(batch_kind(e), "batch_decode: KV pool not bound (bf16 or a lock-step 8-bit batch pool)");
  for (size_t b = 0; b < e->b_ctx.size(); ++b)
    B200_REQUIRE(!e->b_active[b] || e->b_ctx[b] + n_steps <= e->kvb.cap,
                 "batch_decode: row %zu: %d cached + %d steps exceeds cache capacity %d", b, e->b_ctx[b], n_steps,
                 e->kvb.cap);
  B200_CUDA(cudaSetDevice(e->device));
  BdModel m;
  bd_model(e, &m);
  cudaStream_t s = (cudaStream_t)stream;
  B200_CUDA(cudaEventRecord(e->ev0, s));
  int rc = batch_decoder_step(e->batch, m, n_steps, want_logprobs != 0, s, e->cap_stream, &e->launches);
  if (rc) return rc;
  B200_CUDA(cudaEventRecord(e->ev1, s));
  e->last_steps = n_steps;
  e->timing_valid = true;
  for (size_t b = 0; b < e->b_ctx.size(); ++b)
    if (e->b_active[b]) e->b_ctx[b] += n_steps;
  return B200_OK;
}

int b200_batch_fetch(b200_engine* e, long first_step, int n_steps, int* tok_host, float* lp_host, void* stream) {
  B200_REQUIRE(e && e->batch && tok_host, "batch_fetch: batch_begin first");
  return batch_decoder_fetch(e->batch, first_step, n_steps, tok_host, lp_host, (cudaStream_t)stream);
}

int b200_batch_set_procs(b200_engine* e, const int* params, const float* penalties, const int* bias_ids,
                         const float* bias_vals, int bias_cap, int* hist, int* hist_len, int hist_cap, int top_k) {
  B200_REQUIRE(e && e->batch, "batch_set_procs: batch_begin first");
  BdProcs pr;
  pr.params = params; pr.penalties = penalties; pr.bias_ids = bias_ids; pr.bias_vals = bias_vals;
  pr.bias_cap = bias_cap; pr.hist = hist; pr.hist_len = hist_len; pr.hist_cap = hist_cap; pr.top_k = top_k;
  return batch_decoder_set_procs(e->batch, pr, e->cfg.vocab);
}

int b200_batch_fetch_topk(b200_engine* e, long first_step, int n_steps, int* ids_host, float* lp_host, void* stream) {
  B200_REQUIRE(e && e->batch && ids_host && lp_host, "batch_fetch_topk: batch_begin first");
  return batch_decoder_fetch_topk(e->batch, first_step, n_steps, ids_host, lp_host, (cudaStream_t)stream);
}

int b200_batch_procs_apply(void* logits, const void* logprobs, int B, int vocab, int ldv, const int* tok,
                           const int* active, const int* params, const float* penalties, const int* bias_ids,
                           const float* bias_vals, int bias_cap, int* hist, int* hist_len, int hist_cap, int top_k,
                           int* top_ids, float* top_lp, void* stream) {
  BdProcs pr;
  pr.params = params; pr.penalties = penalties; pr.bias_ids = bias_ids; pr.bias_vals = bias_vals;
  pr.bias_cap = bias_cap; pr.hist = hist; pr.hist_len = hist_len; pr.hist_cap = hist_cap; pr.top_k = top_k;
  return batch_procs_apply((bf16*)logits, (const bf16*)logprobs, B, vocab, ldv, tok, active, pr, top_ids, top_lp,
                           (cudaStream_t)stream);
}

const void* b200_batch_logits(b200_engine* e) { return e ? batch_decoder_buffer(e->batch, 0) : nullptr; }
const void* b200_batch_logprobs(b200_engine* e) { return e ? batch_decoder_buffer(e->batch, 1) : nullptr; }
/* device int32 [4096 steps][16 rows]: token of (step since the last begin, row) */
const int* b200_batch_token_log(b200_engine* e) { return e ? (const int*)batch_decoder_buffer(e->batch, 2) : nullptr; }

int b200_memcpy_d2d(void* dst, const void* src, long bytes, void* stream) {
  B200_REQUIRE(dst && src && bytes >= 0, "memcpy_d2d: bad arguments");
  B200_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return B200_OK;
}
float b200_engine_last_decode_ms(const b200_engine* e) {
  if (!e || !e->timing_valid || e->last_steps <= 0) return -1.0f;
  if (cudaEventSynchronize(e->ev1) != cudaSuccess) return -1.0f;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) != cudaSuccess) return -1.0f;
  return ms / (float)e->last_steps;
}

}  // extern "C"
