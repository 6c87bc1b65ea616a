// Engine: whole-tower / whole-step entry points of the C ABI (include/b200vlm.h).
// Owns the weight table, the decode state, the step buffers and the captured
// CUDA graph of one decode step.  The caller (Python, via ctypes) owns weights,
// workspace and the KV pool (torch-allocated device memory).
#include <stdarg.h>

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

struct VBlk {
  const bf16 *ln1w, *ln1b, *ln2w, *ln2b, *qkvw, *qkvb, *projw, *projb, *fc1w, *fc1b, *fc2w, *fc2b;
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
  // kv pool (caller-owned)
  bf16* kv = nullptr;
  int kv_batch = 0, kv_cap = 0;
  int kv_row = 0;        // row of the pool that prefill / single-row decode read and write
  // 8-bit pool (b200_engine_bind_kvq; replaces `kv` while bound) and the engine-owned bf16 staging planes
  // [2][n_kv][cap][hd] where the decode QKV kernel leaves the new K/V row before it is quantized
  KvqPlanes q8 = {};
  KvqPlanes pre_q8 = {};  // b200_engine_set_prefill_kvq: prefill writes its rows through to this 8-bit pool
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
  bool seq_graphs = true;       // B200_SEQ_GRAPH=0: plain launches
  KvRef* kvref = nullptr;       // device: where the bound pool row lives (read by the captured prefill)
  KvRef* kvref_host = nullptr;  // pinned staging
  cudaEvent_t kvref_ev = nullptr;
  bool v2 = true;               // weight-major GEMMs + pipelined attention (B200_PREFILL_V1=1: round-1 path)
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
  int prepared_cap = -1, prepared_cluster = -1;
  // megakernel
  int use_mega = 1;  // 0: one kernel per phase, 1: k_mega (CUDA cores), 2: k_mega_tc (wgmma)
  bool mega_fits = true;  // false: this shape / cache capacity does not fit the persistent kernel
  int active_mega() const { return mega_fits ? use_mega : 0; }
  MegaTcP tp;
  uint8_t* packed = nullptr;  // tile images of the LM weights (k_mega_tc)
  size_t packed_bytes = 0;
  bool packed_ready = false;
  long long* tc_acc = nullptr;  // fixed-point split-K accumulators (k_mega_tc)
  long tc_acc_rows = 0;
  int tc_alias = 1;
  int tc_inflight = 2;
  int fma_inflight = 0, l2_prefetch = 0, l2_skip = 2;
  int flow = 0;  // k_mega dataflow mode (set_mega(4) / B200_MEGA_FLOW=1): measured slower, see DESIGN.md
  unsigned long long* flow_words = nullptr;
  float* att_part = nullptr;
  float* att_stats = nullptr;
  unsigned long long* bar = nullptr;
  bool mega_ready = false;
  MegaP mp;
  long long* dbg = nullptr;

  DecodeDims dims() const {
    DecodeDims d;
    d.hidden = cfg.hidden; d.inter = cfg.inter; d.n_heads = cfg.n_heads; d.n_kv = cfg.n_kv_heads;
    d.hd = cfg.head_dim; d.vocab = cfg.vocab; d.cap = kv_cap; d.eps = cfg.rms_eps;
    d.scale_bf = __bfloat162float(__float2bfloat16_rn(1.0f / sqrtf((float)cfg.head_dim)));
    return d;
  }
  bf16* kptr(int layer, int row) const {
    return kv + (((long)layer * 2 + 0) * kv_batch + row) * cfg.n_kv_heads * (long)kv_cap * cfg.head_dim;
  }
  bf16* vptr(int layer, int row) const {
    return kv + (((long)layer * 2 + 1) * kv_batch + row) * cfg.n_kv_heads * (long)kv_cap * cfg.head_dim;
  }
  KvqPlanes q8_plane(int layer, int side, int row, const KvqPlanes& pool) const {
    const long plane = (((long)layer * 2 + side) * kv_batch + row) * cfg.n_kv_heads;
    KvqPlanes p = pool;
    p.codes += plane * kv_cap * cfg.head_dim;
    p.scales += plane * kv_cap * (cfg.head_dim / pool.gs);
    p.biases += plane * kv_cap * (cfg.head_dim / pool.gs);
    return p;
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
  B200_REQUIRE(!e->q8.codes, "mega: the persistent kernels read a bf16 KV pool; an 8-bit pool runs the per-phase kernels");
  B200_REQUIRE(!e->qk_norm || e->use_mega == 1,
               "mega: k_mega_tc has no q/k norm (Qwen3-VL); such a model runs k_mega or the per-phase kernels");
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
  p.kv_layer_stride = 2L * e->kv_batch * c.n_kv_heads * (long)e->kv_cap * c.head_dim;
  p.kv_v_offset = (long)e->kv_batch * c.n_kv_heads * (long)e->kv_cap * c.head_dim;
  p.partials = e->partials; p.st = e->st; p.token_log = e->token_log; p.log_cap = e->log_cap;
  p.force = e->force; p.inv_freq = e->lm_inv_freq; p.bar = e->bar; p.advance = 1;
  p.dbg = e->dbg;
  p.qk_norm = e->qk_norm;
  for (int l = 0; e->qk_norm && l < c.n_layers; ++l) {
    p.qn[l] = e->qn[l];
    p.kn[l] = e->kn[l];
  }
  // tuning aids
  p.max_inflight = e->fma_inflight;
  p.flow = e->flow;
  {
    const size_t nh = (size_t)c.hidden, nq = (size_t)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim / 2;
    if (!e->flow_words) {
      B200_CUDA(cudaMalloc(&e->flow_words, (2 * nh + nq) * sizeof(unsigned long long)));
      B200_CUDA(cudaMemset(e->flow_words, 0, (2 * nh + nq) * sizeof(unsigned long long)));
    }
    p.hmid_w = e->flow_words;
    p.hout_w = e->flow_words + nh;
    p.qkv_w = e->flow_words + 2 * nh;
  }
  p.l2_prefetch = e->l2_prefetch;
  p.l2_skip = e->l2_skip;
  int rc;
  if (e->use_mega == 2) {
    // ---- tensor-core variant: tile images of the weights + split-K partial buffers ----
    const int QKV = (c.n_heads + 2 * c.n_kv_heads) * c.head_dim, H = c.hidden, I = c.inter;
    const int OK_ = c.n_heads * c.head_dim;
    const size_t b_qkv = mega_tc_packed_bytes(QKV, H, false), b_o = mega_tc_packed_bytes(H, OK_, false);
    const size_t b_gu = mega_tc_packed_bytes(I, H, true), b_d = mega_tc_packed_bytes(H, I, false);
    const size_t b_head = mega_tc_packed_bytes(c.vocab, H, false);
    const size_t total = (size_t)c.n_layers * (b_qkv + b_o + b_gu + b_d) + b_head;
    if (!e->packed || e->packed_bytes < total) {
      if (e->packed) cudaFree(e->packed);
      e->packed = nullptr;
      B200_CUDA(cudaMalloc(&e->packed, total));
      e->packed_bytes = total;
      e->packed_ready = false;
    }
    MegaTcP& P = e->tp;
    memset(&P, 0, sizeof(P));
    uint8_t* w = e->packed;
    for (int l = 0; l < c.n_layers; ++l) {
      const LayerW& lw = e->layers[l];
      LayerWT& lt = P.lt[l];
      lt.wqkv = w; w += b_qkv;
      lt.wo = w; w += b_o;
      lt.wgu = w; w += b_gu;
      lt.wd = w; w += b_d;
      if (!e->packed_ready) {
        if ((rc = mega_tc_pack(lw.wqkv, nullptr, QKV, H, false, (void*)lt.wqkv, s))) return rc;
        if ((rc = mega_tc_pack(lw.wo, nullptr, H, OK_, false, (void*)lt.wo, s))) return rc;
        if ((rc = mega_tc_pack(lw.wgu, lw.wgu + (long)I * H, I, H, true, (void*)lt.wgu, s))) return rc;
        if ((rc = mega_tc_pack(lw.wd, nullptr, H, I, false, (void*)lt.wd, s))) return rc;
      }
    }
    P.head_t = w;
    if (!e->packed_ready)
      if ((rc = mega_tc_pack(e->head, nullptr, c.vocab, H, false, (void*)w, s))) return rc;
    e->packed_ready = true;
    const long acc_rows = ((long)(QKV > H ? QKV : H) + 127) & ~127L;
    if (!e->tc_acc || e->tc_acc_rows < acc_rows) {
      if (e->tc_acc) cudaFree(e->tc_acc);
      e->tc_acc = nullptr;
      B200_CUDA(cudaMalloc(&e->tc_acc, (size_t)3 * acc_rows * sizeof(long long)));
      e->tc_acc_rows = acc_rows;
    }
    // the kernel keeps the accumulators zero between uses; (re)establish that here
    B200_CUDA(cudaMemsetAsync(e->tc_acc, 0, (size_t)3 * acc_rows * sizeof(long long), s));
    P.qkv_acc = e->tc_acc;
    P.o_acc = e->tc_acc + acc_rows;
    P.d_acc = e->tc_acc + 2 * acc_rows;
    P.max_inflight = e->tc_inflight;  // clamped below to n_stages - 1 (a lagging slot must not be reused)
    P.x_kstride = e->tc_alias ? 1024 : 2048;
    P.x_sbo = e->tc_alias ? 0 : 1024;
    P.base = p;
    if ((rc = mega_tc_fill(P, e->sm_count))) return rc;
    if (P.max_inflight > P.base.n_stages - 1) P.max_inflight = P.base.n_stages - 1;
    if (P.max_inflight < 1) P.max_inflight = 1;
    e->mega_ready = true;
    return B200_OK;
  }
  rc = mega_fill(p, e->sm_count);
  if (rc) return rc;
  if (p.max_inflight >= p.n_stages) p.max_inflight = p.n_stages - 1;  // a lagging slot must not be reused
  e->mega_ready = true;
  return B200_OK;
}

// one decode step as plain launches on stream s (also what gets captured)
static int enqueue_step(b200_engine* e, cudaStream_t s) {
  const DecodeDims d = e->dims();
  const auto& c = e->cfg;
  int rc;
  if (e->active_mega() == 2) return mega_tc_launch(e->tp, e->sm_count, s);
  if (e->active_mega()) return mega_launch(e->mp, e->sm_count, s);
  if (e->q8.codes) {
    bf16* sk = e->q8_stage;
    bf16* sv = sk + (long)c.n_kv_heads * e->kv_cap * c.head_dim;
    for (int l = 0; l < c.n_layers; ++l) {
      const LayerW& lw = e->layers[l];
      if ((rc = launch_qkv(d, lw, e->h, e->qbuf, sk, sv, e->st, e->lm_inv_freq, s, e->qk_norm ? e->qn[l] : nullptr,
                           e->qk_norm ? e->kn[l] : nullptr)))
        return rc;
      if ((rc = launch_attn_q8(d, e->qbuf, e->q8_plane(l, 0, e->kv_row, e->q8), e->q8_plane(l, 1, e->kv_row, e->q8), sk, sv,
                               e->attn, e->st, e->attn_cluster, s)))
        return rc;
      if ((rc = launch_res(lw.wo, e->attn, e->h, c.hidden, c.n_heads * c.head_dim, s))) return rc;
      if ((rc = launch_gateup(d, lw, e->h, e->act, s))) return rc;
      if ((rc = launch_res(lw.wd, e->act, e->h, c.hidden, c.inter, s))) return rc;
    }
  } else {
  for (int l = 0; l < c.n_layers; ++l) {
    const LayerW& lw = e->layers[l];
    bf16* kc = e->kptr(l, e->kv_row);
    bf16* vc = e->vptr(l, e->kv_row);
    if ((rc = launch_qkv(d, lw, e->h, e->qbuf, kc, vc, e->st, e->lm_inv_freq, s, e->qk_norm ? e->qn[l] : nullptr,
                         e->qk_norm ? e->kn[l] : nullptr)))
      return rc;
    if ((rc = launch_attn(d, e->qbuf, kc, vc, e->attn, e->st, e->attn_cluster, s))) return rc;
    if ((rc = launch_res(lw.wo, e->attn, e->h, c.hidden, c.n_heads * c.head_dim, s))) return rc;
    if ((rc = launch_gateup(d, lw, e->h, e->act, s))) return rc;
    if ((rc = launch_res(lw.wd, e->act, e->h, c.hidden, c.inter, s))) return rc;
  }
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
// round-2 prefill / vision path: weight-major GEMMs (gemm_wt.cu), split-K partials finished by
// finish_rows (bias + residual + the NEXT norm fused), pipelined attention (attention_fa.cu)
// ---------------------------------------------------------------------------------------------
static long align256(long x) { return (x + 255) & ~255L; }
static const long WT_PARTIAL_BYTES = 48L << 20;  // fp32 split-K partial tiles (bounded: see gemm_wt_auto)
static long round8(long x) { return (x + 7) & ~7L; }
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
static int v2_linear(b200_engine* e, const bf16* x, long ldx, const bf16* W, const bf16* b, bf16* y, long ldy,
                     int T, int N, int K, int epi, cudaStream_t s) {
  e->launches += 1;
  return gemm_wt_tuned(x, ldx, W, b, nullptr, 0, y, ldy, nullptr, 0, T, N, K, epi, B200_WT_BF16, 0, false,
                       e->sm_count, nullptr, s);
}

// h = bf16(h + bf16(x . W^T + b)); xn = norm(h)   (split-K GEMM + one finishing row op)
static int v2_linear_residual_norm(b200_engine* e, const bf16* x, long ldx, const bf16* W, const bf16* b,
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

static int v2_upload_pos(b200_engine* e, const std::vector<int>& pos, cudaStream_t s) {
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
  if (!e->seq_graphs) return body();
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

static int vision_v2_body(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                          void* feats_out, cudaStream_t s);

static int vision_v2(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                     void* feats_out, cudaStream_t s) {
  const auto& c = e->cfg;
  // graph input / output live at fixed workspace addresses: stage them around the captured body
  uint8_t* p = e->ws;
  p += align256(N * (long)c.v_patch_dim * 2) + 2 * align256(N * (long)c.v_embed * 2) +
       align256(N * 3L * c.v_embed * 2) + align256(N * (long)c.v_mlp * 2) + align256(N * (long)c.v_embed * 2) +
       align256((long)c.v_embed * round8(N) * 2);
  float* xin = (float*)p; p += align256(N * (long)c.v_patch_dim * 4);
  bf16* fout = (bf16*)p;
  const long Nm = N / ((long)c.v_merge * c.v_merge);
  int rc;
  std::vector<int> pos;
  build_pos_hw(grid, n_images, c.v_merge, &pos);
  if ((rc = v2_upload_pos(e, pos, s))) return rc;
  B200_CUDA(cudaMemcpyAsync(xin, pixel_values, (size_t)N * c.v_patch_dim * 4, cudaMemcpyDeviceToDevice, s));
  std::vector<long> key = {(long)(uintptr_t)e->ws, (long)e->ws_bytes, N, (long)n_images, (long)(uintptr_t)e->pos_hw};
  for (int i = 0; i < n_images * 3; ++i) key.push_back(grid[i]);
  rc = seq_run(e, e->vis_graphs, key, s, [&]() { return vision_v2_body(e, xin, grid, n_images, N, fout, s); });
  if (rc) return rc;
  B200_CUDA(cudaMemcpyAsync(feats_out, fout, (size_t)Nm * c.v_out * 2, cudaMemcpyDeviceToDevice, s));
  return B200_OK;
}

static int vision_v2_body(b200_engine* e, const float* pixel_values, const int* grid, int n_images, long N,
                          void* feats_out, cudaStream_t s) {
  const auto& c = e->cfg;
  const long E = c.v_embed, Em = c.v_mlp;
  const int nh = c.v_heads, hd = c.v_embed / c.v_heads;
  const int t_ld = (int)round8(N);
  uint8_t* p = e->ws;
  bf16* x = (bf16*)p; p += align256(N * (long)c.v_patch_dim * 2);
  bf16* h = (bf16*)p; p += align256(N * E * 2);
  bf16* y = (bf16*)p; p += align256(N * E * 2);
  bf16* qkv = (bf16*)p; p += align256(N * 3 * E * 2);
  bf16* mlp = (bf16*)p; p += align256(N * Em * 2);
  bf16* att = (bf16*)p; p += align256(N * E * 2);
  bf16* vt = (bf16*)p; p += align256(E * (long)t_ld * 2);
  int rc;
  if ((rc = cast_f32_bf16(pixel_values, x, N * c.v_patch_dim, s))) return rc;
  if ((rc = v2_linear(e, x, c.v_patch_dim, e->v_patch, nullptr, h, E, (int)N, (int)E, c.v_patch_dim, B200_EPI_NONE, s)))
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
     // (8 tokens); frames with other offsets (e.g. a 6 x 6-patch image followed by another) take the round-1 kernel
    long o = 0;
    for (int im = 0; im < n_images && fa; ++im)
      for (int tt = 0; tt < grid[im * 3]; ++tt) {
        if (o % 8) fa = false;
        o += (long)grid[im * 3 + 1] * grid[im * 3 + 2];
      }
  }
  for (int i = 0; i < c.v_depth; ++i) {
    const VBlk& b = e->vblk[i];
    if ((rc = v2_linear(e, y, E, b.qkvw, b.qkvb, qkv, 3 * E, (int)N, (int)(3 * E), (int)E, B200_EPI_NONE, s))) return rc;
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
    if ((rc = v2_linear_residual_norm(e, att, E, b.projw, b.projb, h, E, B200_NORM_LN, b.ln2w, b.ln2b, c.v_ln_eps,
                                      y, E, (int)N, (int)E, (int)E, s)))
      return rc;
    if ((rc = v2_linear(e, y, E, b.fc1w, b.fc1b, mlp, Em, (int)N, (int)Em, (int)E, B200_EPI_GELU_FAST, s))) return rc;
    const bool last = (i + 1 == c.v_depth);
    const bf16* nw = last ? e->m_lnw : e->vblk[i + 1].ln1w;
    const bf16* nb = last ? e->m_lnb : e->vblk[i + 1].ln1b;
    if ((rc = v2_linear_residual_norm(e, mlp, Em, b.fc2w, b.fc2b, h, E, B200_NORM_LN, nw, nb,
                                      last ? 1e-6f : c.v_ln_eps, y, E, (int)N, (int)E, (int)Em, s)))
      return rc;
  }
  // PatchMerger (vision.py:105-120): y already holds LayerNorm(h) of the last block
  const long mg = (long)c.v_merge * c.v_merge * E;
  const long Nm = N / ((long)c.v_merge * c.v_merge);
  if ((rc = v2_linear(e, y, mg, e->m_fc1w, e->m_fc1b, mlp, mg, (int)Nm, (int)mg, (int)mg, B200_EPI_GELU_EXACT, s)))
    return rc;
  if ((rc = v2_linear(e, mlp, mg, e->m_fc2w, e->m_fc2b, (bf16*)feats_out, c.v_out, (int)Nm, c.v_out, (int)mg,
                      B200_EPI_NONE, s)))
    return rc;
  return B200_OK;
}

// one sequence of a batched prefill: tokens [off, off + T) of the concatenated batch go to KV pool row `row`
struct PreSeg { int off, T, row; };

static int prefill_layers_v2_body(b200_engine* e, const int* pos3, int T, int ctx0, void* all_logits_out,
                                  cudaStream_t s, const PreSeg* segs = nullptr, int n_seg = 0,
                                  const void* tok_loc = nullptr);

static int prefill_layers_v2(b200_engine* e, const void* embeds, const int* pos3, int T, int ctx0,
                             void* all_logits_out, bf16** h_out, cudaStream_t s) {
  const auto& c = e->cfg;
  const long H = c.hidden, I = c.inter, QH = (long)c.n_heads * c.head_dim;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  uint8_t* p = e->ws;
  bf16* h = (bf16*)p;
  p += 2 * align256((long)T * H * 2) + align256((long)T * QKV * 2) + align256((long)T * QH * 2) +
       align256((long)T * 2 * I * 2) + align256((long)T * I * 2);
  int* pos_stage = (int*)p;
  // graph inputs at fixed workspace addresses: the embeddings (residual stream) and the position ids
  B200_CUDA(cudaMemcpyAsync(h, embeds, (size_t)T * H * 2, cudaMemcpyDeviceToDevice, s));
  B200_CUDA(cudaMemcpyAsync(pos_stage, pos3, (size_t)3 * T * 4, cudaMemcpyDeviceToDevice, s));
  *h_out = h;
  // where the cache lives travels through device memory (the captured graph survives a new pool)
  if (!e->kvref) {
    B200_CUDA(cudaMalloc(&e->kvref, sizeof(KvRef)));
    B200_CUDA(cudaMallocHost(&e->kvref_host, sizeof(KvRef)));
    B200_CUDA(cudaEventCreateWithFlags(&e->kvref_ev, cudaEventDisableTiming));
  } else {
    B200_CUDA(cudaEventSynchronize(e->kvref_ev));
  }
  e->kvref_host->k0 = e->kptr(0, e->kv_row);
  e->kvref_host->v_off = (long)e->kv_batch * c.n_kv_heads * (long)e->kv_cap * c.head_dim;
  e->kvref_host->layer_stride = 2L * e->kvref_host->v_off;
  e->kvref_host->cap = e->kv_cap;
  B200_CUDA(cudaMemcpyAsync(e->kvref, e->kvref_host, sizeof(KvRef), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaEventRecord(e->kvref_ev, s));
  if (all_logits_out || ctx0 != 0 || e->pre_q8.codes)  // all-row logits / a later chunk / 8-bit write-through: plain launches
    return prefill_layers_v2_body(e, pos_stage, T, ctx0, all_logits_out, s);
  const std::vector<long> key = {(long)(uintptr_t)e->ws, (long)e->ws_bytes, (long)T};
  return seq_run(e, e->pre_graphs, key, s, [&]() { return prefill_layers_v2_body(e, pos_stage, T, 0, nullptr, s); });
}

// segs == nullptr: ONE sequence bound to e->kv_row (graph-capturable: the cache is addressed through e->kvref).
// segs != nullptr (PromptProcessingBatch, ar.py:1581-2175): several fresh sequences concatenated along the token
// axis — every GEMM / norm / SwiGLU runs once over all T tokens (the weights are streamed once for the whole
// batch), M-RoPE + KV append scatter each token to (its row, its position) through `tok_loc`, and attention runs
// per sequence on its own block of the shared q / K / V^T buffers (block-diagonal causal).
static int prefill_layers_v2_body(b200_engine* e, const int* pos3, int T, int ctx0, void* all_logits_out,
                                  cudaStream_t s, const PreSeg* segs, int n_seg, const void* tok_loc) {
  const auto& c = e->cfg;
  const long H = c.hidden, I = c.inter, QH = (long)c.n_heads * c.head_dim;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  const int hd = c.head_dim, t_ld = (int)round8(T);
  uint8_t* p = e->ws;
  bf16* h = (bf16*)p; p += align256((long)T * H * 2);
  bf16* xn = (bf16*)p; p += align256((long)T * H * 2);
  bf16* qkv = (bf16*)p; p += align256((long)T * QKV * 2);
  bf16* att = (bf16*)p; p += align256((long)T * QH * 2);
  p += align256((long)T * 2 * I * 2);  // (gate/up buffer of the round-1 path)
  bf16* act = (bf16*)p; p += align256((long)T * I * 2);
  p += align256(3L * T * 4);
  bf16* vt = (bf16*)p; p += align256((long)c.n_kv_heads * hd * t_ld * 2);
  bf16* kws = (bf16*)p; p += align256((long)c.n_kv_heads * hd * T * 2);
  int rc;
  if ((rc = rms_norm(h, e->layers[0].ln1, xn, T, (int)H, c.rms_eps, s))) return rc;
  e->launches += 1;
  const float scale = 1.0f / sqrtf((float)hd);
  const float scale_bf = __bfloat162float(__float2bfloat16_rn(scale));
  const int S = ctx0 + T;
  for (int l = 0; l < c.n_layers; ++l) {
    const LayerW& lw = e->layers[l];
    bf16* kc = e->kptr(l, e->kv_row);
    bf16* vc = e->vptr(l, e->kv_row);
    if ((rc = v2_linear(e, xn, H, lw.wqkv, lw.bqkv, qkv, QKV, T, (int)QKV, (int)H, B200_EPI_NONE, s))) return rc;
    if (e->qk_norm) {
      if ((rc = qk_norm(qkv, T, c.n_heads, c.n_kv_heads, hd, e->qn[l], e->kn[l], c.rms_eps, s))) return rc;
      e->launches += 1;
    }
    // the pipelined kernel needs V^T of EVERY key: available for a fresh prompt (ctx0 == 0).  It then
    // reads the chunk's own rotated K copy and V^T from the workspace, and the cache is addressed through
    // e->kvref: nothing about the KV pool is baked into the captured graph.
    const bool fa = ctx0 == 0 && !e->pre_q8.codes && attention_fa_supported(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld,
                                                        t_ld, att, QH, hd);
    if (segs) {
      B200_REQUIRE(fa, "prefill_batch: the pipelined attention kernel does not support this geometry");
      const long row_stride = (long)c.n_kv_heads * e->kv_cap * hd;
      if ((rc = mrope_kv_write(qkv, pos3, e->lm_inv_freq, e->axis_sel, e->kptr(l, 0), e->vptr(l, 0), T, 0, e->kv_cap,
                               c.n_heads, c.n_kv_heads, hd, s, scale_bf, vt, t_ld, nullptr, l, kws, tok_loc, row_stride)))
        return rc;
      // all sequences in ONE launch: the (q0, Lq, k0, S) table follows the (row, position) table in `tok_loc`
      int longest = 0;
      for (int g = 0; g < n_seg; ++g) longest = segs[g].T > longest ? segs[g].T : longest;
      if ((rc = attention_fa(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld, t_ld, att, QH, c.n_heads,
                             c.n_kv_heads, hd, longest, longest, 1, s, 0, T, 0, T, (const int*)tok_loc + 2L * T, n_seg)))
        return rc;
      e->launches += 2;
    } else {
    if ((rc = mrope_kv_write(qkv, pos3, e->lm_inv_freq, e->axis_sel, kc, vc, T, ctx0, e->kv_cap, c.n_heads,
                             c.n_kv_heads, hd, s, fa ? scale_bf : 0.f, fa ? vt : nullptr, t_ld,
                             fa ? e->kvref : nullptr, l, fa ? kws : nullptr)))
      return rc;
    if (e->pre_q8.codes) {  // an 8-bit cache: the chunk's rows are quantized before they are attended
      if ((rc = kvq_quantize_rows(kc, e->kv_cap, e->q8_plane(l, 0, e->kv_row, e->pre_q8), c.n_kv_heads, ctx0, T, hd,
                                  true, s)) ||
          (rc = kvq_quantize_rows(vc, e->kv_cap, e->q8_plane(l, 1, e->kv_row, e->pre_q8), c.n_kv_heads, ctx0, T, hd,
                                  true, s)))
        return rc;
      e->launches += 2;
    }
    if (fa) {
      rc = attention_fa(qkv, QKV, hd, kws, hd, (long)T * hd, vt, (long)hd * t_ld, t_ld, att, QH, c.n_heads,
                        c.n_kv_heads, hd, T, S, 1, s, 0, T, 0, S);
    } else {
      rc = attention(qkv, QKV, hd, kc, hd, (long)e->kv_cap * hd, vc, hd, (long)e->kv_cap * hd, att, QH, c.n_heads,
                     c.n_kv_heads, hd, T, S, 1, scale, s);
    }
    if (rc) return rc;
    e->launches += 2;
    }
    if ((rc = v2_linear_residual_norm(e, att, QH, lw.wo, nullptr, h, H, B200_NORM_RMS, lw.ln2, nullptr, c.rms_eps, xn,
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
    if ((rc = v2_linear_residual_norm(e, act, I, lw.wd, nullptr, h, H, want_norm ? B200_NORM_RMS : B200_NORM_NONE, nw,
                                      nullptr, c.rms_eps, xn, H, T, (int)H, (int)I, s)))
      return rc;
  }
  if (all_logits_out) {  // the reference computes the head on every row (ar.py:358); xn = final norm
    // rows of the caller's buffer are round8(vocab) apart (16-byte aligned rows for any vocabulary)
    if ((rc = v2_linear(e, xn, H, e->head, nullptr, (bf16*)all_logits_out, round8(c.vocab), T, c.vocab, (int)H,
                        B200_EPI_NONE, s)))
      return rc;
  }
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
  if (const char* v = getenv("B200_MEGA_FLOW")) e->flow = atoi(v) != 0;  // tuning aid (A/B)
  if (const char* v = getenv("B200_PREFILL_V1")) e->v2 = atoi(v) == 0;    // A/B: round-1 prefill kernels
  if (const char* v = getenv("B200_SEQ_GRAPH")) e->seq_graphs = atoi(v) != 0;
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
  if (e->packed) cudaFree(e->packed);
  if (e->tc_acc) cudaFree(e->tc_acc);
  if (e->flow_words) cudaFree(e->flow_words);
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
  e->packed_ready = false;
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
  const auto& c = e->cfg;
  const long T = max_tokens, N = max_patches;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  long lm = align256(T * c.hidden * 2) * 2 + align256(T * QKV * 2) +
            align256(T * (long)c.n_heads * c.head_dim * 2) + align256(T * 2L * c.inter * 2) +
            align256(T * (long)c.inter * 2) + align256(3L * T * 4);
  long v = align256(N * (long)c.v_patch_dim * 2) + align256(N * (long)c.v_embed * 2) * 2 +
           align256(N * 3L * c.v_embed * 2) + align256(N * (long)c.v_mlp * 2) +
           align256(N * (long)c.v_embed * 2);
  lm += align256((long)c.n_kv_heads * c.head_dim * round8(T) * 2);  // V^T of the prompt chunk
  lm += align256((long)c.n_kv_heads * c.head_dim * T * 2);          // rotated K of the prompt chunk
  v += align256((long)c.v_embed * round8(N) * 2);                   // V^T of the vision tower
  v += align256(N * (long)c.v_patch_dim * 4);                       // staged fp32 pixel_values (graph input)
  v += align256((N / ((long)c.v_merge * c.v_merge) + 1) * c.v_out * 2);  // staged features (graph output)
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
  if (pool != e->kv || batch != e->kv_batch || cap != e->kv_cap || e->q8.codes) invalidate_graph(e);
  if (e->q8_stage) {  // the 8-bit decode staging planes are not needed while a bf16 pool is bound
    B200_CUDA(cudaFree(e->q8_stage));
    e->q8_stage = nullptr;
    e->q8_stage_elems = 0;
  }
  e->kv = (bf16*)pool;
  e->kv_batch = batch;
  e->kv_cap = cap;
  e->q8 = KvqPlanes{};
  e->pre_q8 = KvqPlanes{};
  return B200_OK;
}

int b200_engine_set_prefill_kvq(b200_engine* e, void* codes, void* scales, void* biases, int group_size) {
  B200_REQUIRE(e, "set_prefill_kvq: null engine");
  if (!codes) {
    e->pre_q8 = KvqPlanes{};
    return B200_OK;
  }
  B200_REQUIRE(e->kv && scales && biases && e->v2, "set_prefill_kvq: bind the bf16 pool first / round-1 prefill selected");
  B200_REQUIRE((group_size == 32 || group_size == 64 || group_size == 128) && e->cfg.head_dim % group_size == 0,
               "set_prefill_kvq: group size %d must be 32, 64 or 128 and divide head_dim %d", group_size,
               e->cfg.head_dim);
  e->pre_q8 = KvqPlanes{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  return B200_OK;
}

int b200_engine_bind_kvq(b200_engine* e, void* codes, void* scales, void* biases, int batch, int cap,
                         int group_size) {
  B200_REQUIRE(e && codes && scales && biases && batch >= 1 && cap >= 1 && ((uintptr_t)codes & 15) == 0,
               "bind_kvq: bad arguments");
  const auto& c = e->cfg;
  B200_REQUIRE((group_size == 32 || group_size == 64 || group_size == 128) && c.head_dim % group_size == 0,
               "bind_kvq: group size %d must be 32, 64 or 128 and divide head_dim %d", group_size, c.head_dim);
  B200_REQUIRE(e->kv_row < batch, "bind_kvq: bound row %d of %d", e->kv_row, batch);
  const long stage = 2L * c.n_kv_heads * cap * c.head_dim;
  if (stage > e->q8_stage_elems) {
    if (e->q8_stage) B200_CUDA(cudaFree(e->q8_stage));
    e->q8_stage = nullptr;
    e->q8_stage_elems = 0;
    B200_CUDA(cudaMalloc(&e->q8_stage, (size_t)stage * sizeof(bf16)));
    e->q8_stage_elems = stage;
  }
  if (codes != e->q8.codes || batch != e->kv_batch || cap != e->kv_cap || group_size != e->q8.gs)
    invalidate_graph(e);
  e->kv = nullptr;
  e->kv_batch = batch;
  e->kv_cap = cap;
  e->q8 = KvqPlanes{(uint8_t*)codes, (bf16*)scales, (bf16*)biases, group_size};
  return B200_OK;
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
  if (e->v2) return vision_v2(e, pixel_values, grid_thw_host, n_images, N, feats_out, s);
  const long E = c.v_embed, Em = c.v_mlp;
  const int nh = c.v_heads, hd = c.v_embed / c.v_heads;
  uint8_t* p = e->ws;
  bf16* x = (bf16*)p; p += align256(N * (long)c.v_patch_dim * 2);
  bf16* h = (bf16*)p; p += align256(N * E * 2);
  bf16* y = (bf16*)p; p += align256(N * E * 2);
  bf16* qkv = (bf16*)p; p += align256(N * 3 * E * 2);
  bf16* mlp = (bf16*)p; p += align256(N * Em * 2);
  bf16* att = (bf16*)p; p += align256(N * E * 2);
  // position ids -> device
  std::vector<int> pos;
  build_pos_hw(grid_thw_host, n_images, c.v_merge, &pos);
  if ((long)pos.size() > e->pos_hw_cap) {
    if (e->pos_hw) B200_CUDA(cudaFree(e->pos_hw));
    B200_CUDA(cudaMalloc(&e->pos_hw, pos.size() * 4));
    e->pos_hw_cap = (long)pos.size();
  }
  B200_CUDA(cudaMemcpyAsync(e->pos_hw, pos.data(), pos.size() * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaStreamSynchronize(s));  // `pos` is a stack-lifetime pageable buffer

  if ((rc = cast_f32_bf16(pixel_values, x, N * c.v_patch_dim, s))) return rc;
  if ((rc = gemm_bf16_tn(x, c.v_patch_dim, e->v_patch, nullptr, nullptr, 0, h, E, (int)N, (int)E,
                         c.v_patch_dim, B200_EPI_NONE, s)))
    return rc;
  e->launches += 2;
  const float scale = 1.0f / sqrtf((float)hd);
  for (int i = 0; i < c.v_depth; ++i) {
    const VBlk& b = e->vblk[i];
    if ((rc = layer_norm(h, b.ln1w, b.ln1b, y, (int)N, (int)E, c.v_ln_eps, s))) return rc;
    if ((rc = gemm_bf16_tn(y, E, b.qkvw, b.qkvb, nullptr, 0, qkv, 3 * E, (int)N, (int)(3 * E),
                           (int)E, B200_EPI_NONE, s)))
      return rc;
    if ((rc = vision_rope(qkv, e->pos_hw, e->v_inv_freq, (int)N, nh, hd, s))) return rc;
    long off = 0;
    for (int im = 0; im < n_images; ++im) {
      const int t = grid_thw_host[im * 3];
      const int seg = grid_thw_host[im * 3 + 1] * grid_thw_host[im * 3 + 2];
      for (int tt = 0; tt < t; ++tt) {  // one attention segment per frame (vision.py:270-281)
        const bf16* qb = qkv + off * 3 * E;
        if ((rc = attention(qb, 3 * E, hd, qb + E, 3 * E, hd, qb + 2 * E, 3 * E, hd,
                            att + off * E, E, nh, nh, hd, seg, seg, 0, scale, s)))
          return rc;
        off += seg;
        e->launches += 1;
      }
    }
    if ((rc = gemm_bf16_tn(att, E, b.projw, b.projb, h, E, h, E, (int)N, (int)E, (int)E,
                           B200_EPI_NONE, s)))
      return rc;
    if ((rc = layer_norm(h, b.ln2w, b.ln2b, y, (int)N, (int)E, c.v_ln_eps, s))) return rc;
    if ((rc = gemm_bf16_tn(y, E, b.fc1w, b.fc1b, nullptr, 0, mlp, Em, (int)N, (int)Em, (int)E,
                           B200_EPI_GELU_FAST, s)))
      return rc;
    if ((rc = gemm_bf16_tn(mlp, Em, b.fc2w, b.fc2b, h, E, h, E, (int)N, (int)E, (int)Em,
                           B200_EPI_NONE, s)))
      return rc;
    e->launches += 7;
  }
  // PatchMerger (vision.py:105-120)
  const long mg = (long)c.v_merge * c.v_merge * E;
  const long Nm = N / ((long)c.v_merge * c.v_merge);
  if ((rc = layer_norm(h, e->m_lnw, e->m_lnb, y, (int)N, (int)E, 1e-6f, s))) return rc;
  if ((rc = gemm_bf16_tn(y, mg, e->m_fc1w, e->m_fc1b, nullptr, 0, mlp, mg, (int)Nm, (int)mg,
                         (int)mg, B200_EPI_GELU_EXACT, s)))
    return rc;
  if ((rc = gemm_bf16_tn(mlp, mg, e->m_fc2w, e->m_fc2b, nullptr, 0, feats_out, c.v_out, (int)Nm,
                         c.v_out, (int)mg, B200_EPI_NONE, s)))
    return rc;
  e->launches += 3;
  return B200_OK;
}

int b200_engine_prefill(b200_engine* e, const void* embeds, const int* pos3, int T, int ctx0,
                        int rope_delta, void* all_logits_out, void* stream) {
  B200_REQUIRE(e && embeds && pos3 && T > 0 && ctx0 >= 0, "engine_prefill: bad arguments");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(e->kv, "engine_prefill: KV pool not bound");
  B200_REQUIRE(ctx0 + T <= e->kv_cap, "engine_prefill: ctx0+T=%d exceeds cache capacity %d",
               ctx0 + T, e->kv_cap);
  B200_REQUIRE(e->ws && b200_engine_workspace_bytes(e, T, 1) <= e->ws_bytes,
               "engine_prefill: workspace too small for %d tokens", T);
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  const auto& c = e->cfg;
  const long H = c.hidden, I = c.inter, QH = (long)c.n_heads * c.head_dim;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  uint8_t* p = e->ws;
  bf16* h = (bf16*)p; p += align256((long)T * H * 2);
  bf16* xn = (bf16*)p; p += align256((long)T * H * 2);
  bf16* qkv = (bf16*)p; p += align256((long)T * QKV * 2);
  bf16* att = (bf16*)p; p += align256((long)T * QH * 2);
  bf16* gu = (bf16*)p; p += align256((long)T * 2 * I * 2);
  bf16* act = (bf16*)p; p += align256((long)T * I * 2);
  if (e->v2) {
    if ((rc = prefill_layers_v2(e, embeds, pos3, T, ctx0, all_logits_out, &h, s))) return rc;
  } else {
  B200_CUDA(cudaMemcpyAsync(h, embeds, (size_t)T * H * 2, cudaMemcpyDeviceToDevice, s));
  const float scale = 1.0f / sqrtf((float)c.head_dim);
  const int S = ctx0 + T;
  for (int l = 0; l < c.n_layers; ++l) {
    const LayerW& lw = e->layers[l];
    bf16* kc = e->kptr(l, e->kv_row);
    bf16* vc = e->vptr(l, e->kv_row);
    if ((rc = rms_norm(h, lw.ln1, xn, T, (int)H, c.rms_eps, s))) return rc;
    if ((rc = gemm_bf16_tn(xn, H, lw.wqkv, lw.bqkv, nullptr, 0, qkv, QKV, T, (int)QKV, (int)H,
                           B200_EPI_NONE, s)))
      return rc;
    if (e->qk_norm && (rc = qk_norm(qkv, T, c.n_heads, c.n_kv_heads, c.head_dim, e->qn[l], e->kn[l], c.rms_eps, s)))
      return rc;
    if ((rc = mrope_kv_write(qkv, pos3, e->lm_inv_freq, e->axis_sel, kc, vc, T, ctx0, e->kv_cap,
                             c.n_heads, c.n_kv_heads, c.head_dim, s)))
      return rc;
    if ((rc = attention(qkv, QKV, c.head_dim, kc, c.head_dim, (long)e->kv_cap * c.head_dim, vc,
                        c.head_dim, (long)e->kv_cap * c.head_dim, att, QH, c.n_heads,
                        c.n_kv_heads, c.head_dim, T, S, 1, scale, s)))
      return rc;
    if ((rc = gemm_bf16_tn(att, QH, lw.wo, nullptr, h, H, h, H, T, (int)H, (int)QH, B200_EPI_NONE,
                           s)))
      return rc;
    if ((rc = rms_norm(h, lw.ln2, xn, T, (int)H, c.rms_eps, s))) return rc;
    if ((rc = gemm_bf16_tn(xn, H, lw.wgu, nullptr, nullptr, 0, gu, 2 * I, T, (int)(2 * I), (int)H,
                           B200_EPI_NONE, s)))
      return rc;
    if ((rc = swiglu(gu, act, T, (int)I, s))) return rc;
    if ((rc = gemm_bf16_tn(act, I, lw.wd, nullptr, h, H, h, H, T, (int)H, (int)I, B200_EPI_NONE,
                           s)))
      return rc;
    e->launches += 9;
  }
  if (all_logits_out) {  // the reference computes the head on every row (ar.py:358)
    if ((rc = rms_norm(h, e->norm, xn, T, (int)H, c.rms_eps, s))) return rc;
    B200_REQUIRE(c.vocab % 8 == 0, "prefill (round-1 kernels): all-row logits need vocab %% 8 == 0");
    if ((rc = gemm_bf16_tn(xn, H, e->head, nullptr, nullptr, 0, all_logits_out, c.vocab, T,
                           c.vocab, (int)H, B200_EPI_NONE, s)))
      return rc;
    e->launches += 2;
  }
  }
  // last row through the fused head + sampler; arms the decode state
  const DecodeDims d = e->dims();
  if (e->prepared_cap != e->kv_cap || e->prepared_cluster != e->attn_cluster) {
    if ((rc = decode_prepare(d, e->attn_cluster))) return rc;
    e->prepared_cap = e->kv_cap;
    e->prepared_cluster = e->attn_cluster;
  }
  e->ctx_host = ctx0 + T;
  e->pos_host = ctx0 + T + rope_delta;
  if ((rc = launch_set_state(e->st, 0, e->ctx_host, e->pos_host, 0, 0, e->embed, e->h, c.hidden, s)))
    return rc;
  if ((rc = launch_head(d, e->norm, e->head, h + (long)(T - 1) * H, e->logits, e->partials, s)))
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
  B200_REQUIRE(e->kv && e->v2, "engine_prefill_batch: KV pool not bound / round-1 prefill kernels selected");
  B200_REQUIRE(!e->pre_q8.codes, "engine_prefill_batch: no 8-bit write-through in the batched prefill");
  long T = 0;
  std::vector<PreSeg> segs(n_seq);
  for (int g = 0; g < n_seq; ++g) {
    B200_REQUIRE(seq_len[g] > 0 && seq_len[g] <= e->kv_cap && rows[g] >= 0 && rows[g] < e->kv_batch,
                 "engine_prefill_batch: sequence %d: %d tokens into row %d (capacity %d, %d rows)", g, seq_len[g], rows[g],
                 e->kv_cap, e->kv_batch);
    segs[g] = PreSeg{(int)T, seq_len[g], rows[g]};
    T += round8(seq_len[g]);   // every sequence starts at a multiple of 8 tokens: the V^T tiles are loaded by TMA
                               // with tokens innermost, and a box must start on a 16-byte boundary
  }
  B200_REQUIRE(e->ws && b200_engine_workspace_bytes(e, (int)T, 1) <= e->ws_bytes,
               "engine_prefill_batch: workspace too small for %ld tokens", T);
  B200_CUDA(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  const auto& c = e->cfg;
  const long H = c.hidden, I = c.inter, QH = (long)c.n_heads * c.head_dim;
  const long QKV = (long)(c.n_heads + 2 * c.n_kv_heads) * c.head_dim;
  uint8_t* p = e->ws;
  bf16* h = (bf16*)p;
  p += 2 * align256(T * H * 2) + align256(T * QKV * 2) + align256(T * QH * 2) + align256(T * 2 * I * 2) +
       align256(T * I * 2);
  int* pos_stage = (int*)p;   // 3 * T ints; the tokens' (row, position) table lives in e->loc_dev
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
  rc = prefill_layers_v2_body(e, pos_stage, (int)T, 0, nullptr, s, segs.data(), n_seq, e->loc_dev);
  B200_CUDA(cudaEventRecord(e->loc_ev, s));   // the table (and its staging copy) may be rewritten after this point
  if (rc) return rc;
  const DecodeDims d = e->dims();
  if (e->prepared_cap != e->kv_cap || e->prepared_cluster != e->attn_cluster) {
    if ((rc = decode_prepare(d, e->attn_cluster))) return rc;
    e->prepared_cap = e->kv_cap;
    e->prepared_cluster = e->attn_cluster;
  }
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
  B200_REQUIRE(e->kv || e->q8.codes, "engine_decode: KV pool not bound");
  B200_REQUIRE(e->ctx_host + n_steps <= e->kv_cap,
               "engine_decode: %d cached + %d steps exceeds cache capacity %d", e->ctx_host,
               n_steps, e->kv_cap);
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
  if (e->prepared_cap != e->kv_cap || e->prepared_cluster != e->attn_cluster) {
    if ((rc = decode_prepare(e->dims(), e->attn_cluster))) return rc;
    e->prepared_cap = e->kv_cap;
    e->prepared_cluster = e->attn_cluster;
  }
  if (e->use_mega && e->mega_fits && !e->mega_ready) {
    if ((rc = mega_prepare(e, s))) {
      // a geometry the persistent kernel cannot hold (very long cache: the attention scratch
      // leaves no room for the weight ring; > 132 attention CTAs; ...): same step, one kernel per
      // phase — still this library's CUDA path.  b200_last_error() keeps the reason.
      if (rc != B200_ERR_INVALID) return rc;
      e->mega_fits = false;
    }
  }
  if (e->q8.codes && !(e->use_graph && e->gexec))
    if ((rc = kvq_decode_prepare(e->dims(), e->attn_cluster))) return rc;
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
  B200_REQUIRE(enabled >= 0 && enabled <= 4,
               "set_mega: mode %d (0 off, 1 k_mega, 2 k_mega_tc, 3 k_mega_tc with a 16-row operand, 4 k_mega dataflow)",
               enabled);
  e->use_mega = enabled == 3 ? 2 : (enabled == 4 ? 1 : enabled);
  e->tc_alias = enabled == 3 ? 0 : 1;
  e->flow = enabled == 4 ? 1 : 0;
  if (const char* v = getenv("B200_TC_INFLIGHT")) e->tc_inflight = atoi(v) > 0 ? atoi(v) : 2;  // tuning aids
  if (const char* v = getenv("B200_FMA_INFLIGHT")) e->fma_inflight = atoi(v);

  if (const char* v = getenv("B200_L2_PREFETCH")) e->l2_prefetch = atoi(v);
  if (const char* v = getenv("B200_L2_SKIP")) e->l2_skip = atoi(v);
  invalidate_graph(e);
  return B200_OK;
}
int b200_engine_debug_buffer(b200_engine* e, const char* name, void** ptr, long* bytes) {
  B200_REQUIRE(e && name && ptr && bytes, "debug_buffer: null argument");
  const std::string n(name);
  if (n == "h") { *ptr = e->h; *bytes = (long)e->cfg.hidden * 2; }
  else if (n == "act") { *ptr = e->act; *bytes = (long)e->cfg.inter * 2; }
  else if (n == "tc_acc" && e->tc_acc) { *ptr = e->tc_acc; *bytes = 3 * e->tc_acc_rows * 8; }
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
  B200_REQUIRE(e && row >= 0 && (e->kv_batch == 0 || row < e->kv_batch), "set_kv_row: row %d of %d", row,
               e ? e->kv_batch : 0);
  if (row != e->kv_row) invalidate_graph(e);
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
  m->kv = e->kptr(0, 0);
  m->row_stride = (long)c.n_kv_heads * e->kv_cap * c.head_dim;
  m->v_off = (long)e->kv_batch * m->row_stride;
  m->layer_stride = 2L * m->v_off;
  m->kv_batch = e->kv_batch;
  m->sm_count = e->sm_count;
  m->qn = e->qk_norm ? e->qn.data() : nullptr;
  m->kn = e->qk_norm ? e->kn.data() : nullptr;
}

int b200_batch_begin(b200_engine* e, int B, const int* tok, const int* ctx, const int* pos, const int* active,
                     void* stream) {
  B200_REQUIRE(e && tok && ctx && pos && active, "batch_begin: null argument");
  int rc = resolve(e);
  if (rc) return rc;
  B200_REQUIRE(e->kv, "batch_begin: KV pool not bound");
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
  for (size_t b = 0; b < e->b_ctx.size(); ++b)
    B200_REQUIRE(!e->b_active[b] || e->b_ctx[b] + n_steps <= e->kv_cap,
                 "batch_decode: row %zu: %d cached + %d steps exceeds cache capacity %d", b, e->b_ctx[b], n_steps,
                 e->kv_cap);
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

const void* b200_batch_logits(b200_engine* e) { return e ? batch_decoder_buffer(e->batch, 0) : nullptr; }
const void* b200_batch_logprobs(b200_engine* e) { return e ? batch_decoder_buffer(e->batch, 1) : nullptr; }
/* device int32 [4096 steps][16 rows]: token of (step since the last begin, row) */
const int* b200_batch_token_log(b200_engine* e) { return e ? (const int*)batch_decoder_buffer(e->batch, 2) : nullptr; }

/* cache management of the batched pool (the reference's BatchKVCache.filter / extend / extract,
 * models/cache.py:1077-1201, move rows between arrays): copy the first n_tokens positions of one row
 * of a pool (n_layers, 2, batch, n_kv, cap, hd) into a row of another (or the same) pool */
int b200_kv_copy_row(void* dst_pool, int dst_batch, int dst_cap, int dst_row, const void* src_pool, int src_batch,
                     int src_cap, int src_row, int n_layers, int n_kv, int hd, int n_tokens, void* stream) {
  B200_REQUIRE(dst_pool && src_pool && dst_row >= 0 && dst_row < dst_batch && src_row >= 0 && src_row < src_batch &&
                   n_tokens >= 0 && n_tokens <= dst_cap && n_tokens <= src_cap,
               "kv_copy_row: bad arguments");
  if (n_tokens == 0) return B200_OK;
  const size_t w = (size_t)n_tokens * hd * 2;
  for (int l = 0; l < n_layers; ++l)
    for (int kv = 0; kv < 2; ++kv) {
      const char* sp = (const char*)src_pool + ((((size_t)l * 2 + kv) * src_batch + src_row) * n_kv) * (size_t)src_cap * hd * 2;
      char* dp = (char*)dst_pool + ((((size_t)l * 2 + kv) * dst_batch + dst_row) * n_kv) * (size_t)dst_cap * hd * 2;
      B200_CUDA(cudaMemcpy2DAsync(dp, (size_t)dst_cap * hd * 2, sp, (size_t)src_cap * hd * 2, w, n_kv,
                                  cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    }
  return B200_OK;
}

int b200_memcpy_d2d(void* dst, const void* src, long bytes, void* stream) {
  B200_REQUIRE(dst && src && bytes >= 0, "memcpy_d2d: bad arguments");
  B200_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return B200_OK;
}
int b200_memcpy_h2d(void* dst, const void* src_host, long bytes, void* stream) {
  B200_REQUIRE(dst && src_host && bytes >= 0, "memcpy_h2d: bad arguments");
  B200_CUDA(cudaMemcpyAsync(dst, src_host, (size_t)bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
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
