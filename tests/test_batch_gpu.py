"""Lock-step batched decode on the GPU (csrc/decode_batch.cu; SURVEY §8 a15, config C5): rows that
share one weight stream must produce what each request produces alone.

The batch-1 path (persistent k_mega) and the batched path (weight-major wgmma GEMMs + bd_attn)
are different kernels: both are within the per-op bar of the oracle, so a row's tokens are required
to be equal until the first near-tie (the batched token's logprob on the batch-1 path within two
bf16 ulps of the maximum), exactly like the oracle comparisons of test_engine_gpu.py."""
import types

import numpy as np
import pytest
import torch

from _util import cmp_noise, rl2
from test_engine_gpu import _build, _to_model_config, _token_ok
from test_gate_gpu import _cfg_7b_geometry

pytestmark = pytest.mark.gpu


def _alone(model, ids, kw, n):
    from mlx_vlm_b200.generate import generate_step
    toks, lps = [], []
    for t, lp in generate_step(ids, model, kw.get("pixel_values"), None, max_tokens=n,
                               image_grid_thw=kw.get("image_grid_thw")):
        toks.append(t)
        lps.append(lp.float().cpu())
    return toks, lps


def _same_until_tie(got, want, want_lps, name):
    assert len(got) == len(want), (name, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            assert _token_ok(g, want_lps[i]), f"{name}: token {i}: batched {g} vs alone {w} is not a near-tie"
            print(f"{name}: near-tie at token {i} ({g} vs {w}); histories diverge legitimately")
            return i
    return len(got)


def _requests(c, req, n_rows, seed=3):
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    pvd = torch.from_numpy(pv).cuda()
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n_rows):
        if i % 2 == 0:
            rows.append((ids, {"pixel_values": pvd, "image_grid_thw": grid}, 6 + 3 * i))
        else:
            rows.append((rng.integers(0, 900, size=(1, 9 + 7 * i)), {}, 5 + 2 * i))
    return rows


@pytest.mark.parametrize("kind", ["tiny", "wide2", "7b", "oddvocab"])
def test_lock_step_rows_equal_single_requests(kind):
    from mlx_vlm_b200.generate_batch import BatchGenerator
    from oracle import qwen2vl as O
    if kind == "7b":
        from mlx_vlm_b200.models.qwen2_vl import Model
        c = _cfg_7b_geometry()
        W = O.init_weights(c, 0, norm_jitter=0.05)
        model = Model(_to_model_config(c), device="cuda:0")
        model.load_weights(W)
        req = O.synthetic_request(c, 10, image_hw=(56, 56), seed=0)
    else:
        c, W, model, req = _build(kind, 10, (56, 56))
    rows = _requests(c, req, 5)
    want = [_alone(model, r[0], r[1], r[2]) for r in rows]
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    for slice_, cbs in ((1, 3), (4, 5)):
        g = BatchGenerator(model, proc, completion_batch_size=cbs, prefill_batch_size=2, decode_slice=slice_)
        assert g._lockstep
        l0 = model.engine.launch_count
        uids = g.insert([r[0] for r in rows], [r[2] for r in rows], [r[1] for r in rows])
        got = {u: [] for u in uids}
        while g.has_work:
            _, rs = g.next()
            for r in rs:
                got[r.uid].append(r.token)
        assert model.engine.device_error() == 0
        agree = 0
        for u, (wt, wl) in zip(uids, want):
            agree += _same_until_tie(got[u], wt, wl, f"{kind} slice={slice_} row {u}")
        total = sum(len(w[0]) for w in want)
        print(f"{kind}: slice={slice_} cbs={cbs}: {agree}/{total} tokens identical to the batch-1 path, "
              f"{model.engine.launch_count - l0} launches")
        assert agree >= 0.7 * total


def test_batched_step_logits_against_oracle():
    """B = 4 rows of different lengths, one lock-step step: each row's logits vs the oracle's decode
    step on that row alone (teacher-forced), and the appended K/V rows of layer 0 to the 1e-3 bar."""
    from oracle import qwen2vl as O
    from _util import cmp_bf16
    c, W, model, req = _build("wide2", 10, (56, 56))
    lm, eng = model.language_model, model.engine
    rows_req = _requests(c, req, 4)
    rows, caches = lm.make_batch_cache(4, 256)
    refs = []
    rng = np.random.default_rng(5)
    B = len(rows_req)
    rows.lengths = [0] * B
    feed = []
    for b, (ids, kw, _) in enumerate(rows_req):
        pv = kw.get("pixel_values")
        grid = kw.get("image_grid_thw")
        pv_np = None if pv is None else pv.cpu().numpy()
        forced = int(rng.integers(0, 900))
        ref = O.greedy_generate(c, W, ids, pv_np, grid, 2, force_tokens=[forced, forced])
        ex = O.greedy_generate(c, W, ids, pv_np, grid, 2, dtype="f32", force_tokens=[forced, forced])
        refs.append((ref, ex))
        feed.append(forced)
        emb = model.get_input_embeddings(ids, pv, image_grid_thw=grid)
        rc = lm.make_cache_row(rows.pool, b)
        lm._rope_deltas, lm._position_ids = None, None
        lm(ids, inputs_embeds=emb.inputs_embeds, cache=rc, position_ids=emb.position_ids,
           rope_deltas=emb.rope_deltas, logits_to_keep=1, reserve_tokens=256)
        rows.lengths[b] = ids.shape[1]
    rows._touch()
    deltas = np.asarray([[int(r[0]["prefill"].rope_deltas[0, 0])] for r in refs])
    out = lm(np.asarray(feed)[:, None], cache=caches, rope_deltas=deltas)
    eng.stream.synchronize()
    assert out.logits.shape == (B, 1, c.text.vocab_size)
    for b, (ref, ex) in enumerate(refs):
        cmp_noise(out.logits[b, 0], ref["logits"][1][0], ex["logits"][1][0], f"batched step row {b} logits")
        T = rows_req[b][0].shape[1]
        cmp_bf16(caches[0].keys[b, :, T:T + 1], ref["cache"][0].keys[0, :, T:T + 1], f"row {b} appended K, layer 0",
                 rel_l2=1e-3, max_mismatch=0.05)
        cmp_bf16(caches[0].values[b, :, T:T + 1], ref["cache"][0].values[0, :, T:T + 1], f"row {b} appended V, layer 0",
                 rel_l2=1e-3, max_mismatch=0.05)
    assert rows.lengths == [r[0].shape[1] + 1 for r in rows_req]


def test_fused_greedy_decode_hook_batched_and_cache_surgery():
    """the reference's `_fused_greedy_step` convention with B = 3 rows (ar.py:1015-1042), then
    BatchKVCache.filter / extend / extract semantics on the device pool (cache.py:1077-1201):
    dropping a row and appending another must not disturb the surviving rows' tokens."""
    c, W, model, req = _build("tiny", 10, (56, 56))
    lm, eng = model.language_model, model.engine
    rows_req = _requests(c, req, 4)
    want = [_alone(model, r[0], r[1], 8) for r in rows_req]
    rows, caches = lm.make_batch_cache(4, 256)
    ids_list = [r[0] for r in rows_req[:3]]
    L = max(i.shape[1] for i in ids_list)
    ids = np.zeros((3, L), dtype=np.int64)
    mask = np.zeros((3, L), dtype=np.int64)
    for b, i in enumerate(ids_list):
        ids[b, L - i.shape[1]:] = i[0]
        mask[b, L - i.shape[1]:] = 1
    # rows with an image need their embeddings: prefill them one by one through the row caches instead
    firsts, deltas = [], []
    rows.lengths = [0, 0, 0]
    for b, (rid, kw, _) in enumerate(rows_req[:3]):
        emb = model.get_input_embeddings(rid, kw.get("pixel_values"), image_grid_thw=kw.get("image_grid_thw"))
        rc = lm.make_cache_row(rows.pool, b)
        lm._rope_deltas, lm._position_ids = None, None
        lm(rid, inputs_embeds=emb.inputs_embeds, cache=rc, position_ids=emb.position_ids,
           rope_deltas=emb.rope_deltas, logits_to_keep=1, reserve_tokens=256)
        eng.stream.synchronize()
        firsts.append(int(eng.token_log_view()[(eng.tokens_launched - 1) % eng.token_log_capacity]))
        deltas.append(int(np.asarray(emb.rope_deltas).reshape(-1)[0]))
        rows.lengths[b] = rid.shape[1]
    rows._touch()
    got = [[f] for f in firsts]
    fwd = {"rope_deltas": np.asarray(deltas)[:, None]}
    inputs = np.asarray(firsts)
    for _ in range(3):
        sampled = lm.fused_greedy_decode(inputs[:, None], cache=caches, **fwd)
        assert sampled is not None and tuple(sampled.shape) == (3,)
        eng.stream.synchronize()
        for b in range(3):
            got[b].append(int(sampled[b]))
        inputs = sampled
    # drop row 1, admit request 3 as a single-request cache, extend
    for cch in caches:
        cch.filter([0, 2])
    assert rows.B == 2 and rows.lengths == [rows_req[0][0].shape[1] + 3, rows_req[2][0].shape[1] + 3]
    rid, kw, _ = rows_req[3]
    single = lm.make_cache()
    emb = model.get_input_embeddings(rid, kw.get("pixel_values"), image_grid_thw=kw.get("image_grid_thw"))
    lm._rope_deltas, lm._position_ids = None, None
    lm(rid, inputs_embeds=emb.inputs_embeds, cache=single, position_ids=emb.position_ids,
       rope_deltas=emb.rope_deltas, logits_to_keep=1)
    eng.stream.synchronize()
    first3 = int(eng.token_log_view()[(eng.tokens_launched - 1) % eng.token_log_capacity])
    from mlx_vlm_b200.models.cache import RowBatchKVCache
    other = [RowBatchKVCache.merge([single[l]], engine=eng) if l == 0 else None for l in range(len(single))]
    other_rows = other[0]._rows
    for l, cch in enumerate(caches):
        cch.extend(RowBatchKVCache(other_rows, l))
    assert rows.B == 3
    ex = caches[0].extract(1)
    assert ex.offset == rows.lengths[1]
    assert torch.equal(ex.keys[0, :, :ex.offset], caches[0].keys[1, :, :ex.offset])
    got3 = [first3]
    keep_rows = [0, 2]
    inputs = np.asarray([got[0][-1], got[2][-1], first3])
    fwd = {"rope_deltas": np.asarray([deltas[0], deltas[2], int(np.asarray(emb.rope_deltas).reshape(-1)[0])])[:, None]}
    for _ in range(4):
        sampled = lm.fused_greedy_decode(inputs[:, None], cache=caches, **fwd)
        eng.stream.synchronize()
        got[0].append(int(sampled[0]))
        got[2].append(int(sampled[1]))
        got3.append(int(sampled[2]))
        inputs = sampled
    _same_until_tie(got[0], want[0][0][:len(got[0])], want[0][1], "row 0 across filter/extend")
    _same_until_tie(got[1], want[1][0][:len(got[1])], want[1][1], "row 1 before the filter")
    _same_until_tie(got[2], want[2][0][:len(got[2])], want[2][1], "row 2 across filter/extend")
    _same_until_tie(got3, want[3][0][:len(got3)], want[3][1], "row admitted by extend")


def test_server_loop_streams_concurrent_requests():
    """mlx_vlm_b200/server.py (reference server/generation.py:1730-1918) on the real engine: the GPU thread
    owns the lock-step BatchGenerator; three caller threads stream their own request and must see the tokens
    the request produces alone; the vision cache is filled on a miss and used on the repeat."""
    import threading
    from mlx_vlm_b200.server import GenerationArguments, ResponseGenerator
    from mlx_vlm_b200.vision_cache import VisionFeatureCache
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _requests(c, req, 3)
    want = [_alone(model, r[0], r[1], r[2]) for r in rows]
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    srv = ResponseGenerator(model, proc, max_num_seqs=4, decode_slice=2, vision_cache=VisionFeatureCache())
    got = {}

    def client(i):
        ids, kw, n = rows[i]
        raw = {"input_ids": ids, **kw}
        got[i] = [e.token for e in srv.generate(raw, GenerationArguments(max_tokens=n), timeout=60)]

    th = [threading.Thread(target=client, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(120)
    srv.stop_and_join()
    assert srv._error is None, srv._error
    for i in range(3):
        _same_until_tie(got[i], want[i][0], want[i][1], f"server request {i}")
    assert model.engine.device_error() == 0


def test_batched_prefill_equals_single_prefills():
    """`b200_engine_prefill_batch` (reference PromptProcessingBatch, ar.py:1581-2175): four prompts of different
    lengths (two with an image) prefilled in ONE pass land in their pool rows exactly like four single prefills:
    K/V rows to the per-op bar, first tokens equal up to a near-tie; the following lock-step steps run on them."""
    c, W, model, req = _build("wide2", 10, (56, 56))
    lm, eng = model.language_model, model.engine
    rows_req = _requests(c, req, 4)
    # reference: every prompt alone in a single-row cache
    singles, firsts = [], []
    for ids, kw, _ in rows_req:
        emb = model.get_input_embeddings(ids, kw.get("pixel_values"), image_grid_thw=kw.get("image_grid_thw"))
        cache = lm.make_cache()
        lm._rope_deltas, lm._position_ids = None, None
        lm(ids, inputs_embeds=emb.inputs_embeds, cache=cache, position_ids=emb.position_ids,
           rope_deltas=emb.rope_deltas, logits_to_keep=1)
        eng.stream.synchronize()
        firsts.append(int(eng.token_log_view()[(eng.tokens_launched - 1) % eng.token_log_capacity]))
        lp = eng.logprobs_view().float().cpu().clone()
        singles.append((cache, emb, lp))
    rows, caches = lm.make_batch_cache(4, 256)
    row_caches = [lm.make_cache_row(rows.pool, b) for b in range(4)]
    toks = lm.prefill_rows([r[0] for r in rows_req], [s[1].inputs_embeds for s in singles], row_caches,
                           [s[1].position_ids for s in singles], [s[1].rope_deltas for s in singles], reserve_tokens=256)
    eng.stream.synchronize()
    for b, (ids, _, _) in enumerate(rows_req):
        L = ids.shape[1]
        assert row_caches[b][0].offset == L
        for layer in (0, 1):
            k1 = singles[b][0][layer].keys[0, :, :L].float().cpu()
            v1 = singles[b][0][layer].values[0, :, :L].float().cpu()
            k2 = row_caches[b][layer].keys[0, :, :L].float().cpu()
            v2 = row_caches[b][layer].values[0, :, :L].float().cpu()
            assert rl2(k2, k1) <= 1e-3 and rl2(v2, v1) <= 1e-3, (b, layer, rl2(k2, k1), rl2(v2, v1))
        assert _token_ok(toks[b], singles[b][2]), (b, toks[b], firsts[b])
    print("batched prefill first tokens", toks, "single", firsts)
