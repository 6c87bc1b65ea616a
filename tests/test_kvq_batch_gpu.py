"""8-bit KV cache in the lock-step batch (kv_bits=8 on BatchGenerator; csrc/decode_batch.cu Q8 variant of
bd_attn_kernel): the reference's batch rule (ar.py:751-859 `_make_cache`, models/cache.py:8-21) with every 8-bit
layer quantized from the first prefill on.

  * op level: the 8-bit lock-step attention appends codes / scales / biases bit-exact with b200_kvq_quantize of the
    same bf16 row, stays within relative L2 1e-3 of sdpa over the dequantized cache, and agrees with the single-row
    8-bit attention (b200_kvq_decode_attention) row by row;
  * end to end: greedy rows against an oracle loop that applies the batch rule to each row alone (tests/kvq_ref.py
    arithmetic), tokens equal until the first near-tie, step-0 logprobs on the noise bar;
  * lifecycle: joins, finishes with compaction, pool growth past 256 positions with live rows, filter / extend /
    extract byte-exact, extract continuing under generate_step(kv_bits=8), chunked admission == one-shot;
  * memory: nbytes of the batch cache."""
import types

import numpy as np
import pytest
import torch

from _util import cmp_noise, rl2
from test_engine_gpu import _build, _to_model_config, _token_ok

pytestmark = pytest.mark.gpu


def _bf(x):
    return x.to(torch.bfloat16).float()


def _quantize(x, gs):
    """x (P, n, hd) bf16 cuda -> (codes, scales, biases) through b200_kvq_quantize"""
    from mlx_vlm_b200 import _native as N
    P, n, hd = x.shape
    codes = torch.zeros(P, n, hd, dtype=torch.uint8, device="cuda")
    scales = torch.zeros(P, n, hd // gs, dtype=torch.bfloat16, device="cuda")
    biases = torch.zeros_like(scales)
    N.check(N.lib().b200_kvq_quantize(x.contiguous().data_ptr(), n, codes.data_ptr(), scales.data_ptr(),
                                      biases.data_ptr(), n, P, n, hd, gs, torch.cuda.current_stream().cuda_stream))
    return codes, scales, biases


def _dequant(codes, scales, biases, gs):
    s = scales.float().repeat_interleave(gs, -1)
    b = biases.float().repeat_interleave(gs, -1)
    return _bf(s * codes.float() + b)


@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("hd,gs", [(64, 32), (64, 64), (128, 32), (128, 64), (128, 128)])
def test_batch_kvq_attention_op(B, hd, gs):
    from mlx_vlm_b200 import _native as N
    from oracle import mlx_semantics as S
    from _util import cmp_bf16
    lib = N.lib()
    torch.manual_seed(B * 1000 + hd + gs)
    nkv, nh, cap = 2, (4 if hd == 64 else 8), 512
    QKV = (nh + 2 * nkv) * hd
    rng = np.random.default_rng(B + hd + gs)
    ctx = rng.integers(0, 400, size=B).astype(np.int32)
    ctx[0] = 0 if B > 1 else ctx[0]
    # cache content of every row, quantized by the conversion kernel
    cache = (torch.randn(2, B, nkv, cap, hd, device="cuda") * 0.8).to(torch.bfloat16)
    codes, scales, biases = (t.view(2, B, nkv, cap, -1).contiguous()
                             for t in _quantize(cache.view(-1, cap, hd), gs))
    before = [t.clone() for t in (codes, scales, biases)]
    qkv = _bf(torch.randn(B, QKV, device="cuda"))
    bias = torch.zeros(QKV, dtype=torch.bfloat16, device="cuda")
    inv_freq = torch.rand(hd // 2, device="cuda")
    ctx_d = torch.from_numpy(ctx).cuda()
    pos_d = torch.zeros(B, dtype=torch.int32, device="cuda")   # position 0: the rotary is the identity
    out = torch.zeros(B, nh * hd, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200_batch_kvq_attention(qkv.data_ptr(), bias.data_ptr(), inv_freq.data_ptr(), ctx_d.data_ptr(),
                                         pos_d.data_ptr(), codes.data_ptr(), scales.data_ptr(), biases.data_ptr(), gs,
                                         B, cap, out.data_ptr(), B, nh, nkv, hd, None, None, 1e-6, s),
            "batch_kvq_attention")
    torch.cuda.synchronize()
    for b in range(B):
        c = int(ctx[b])
        q = qkv[b, :nh * hd].view(nh, hd)
        k_new = qkv[b, nh * hd:(nh + nkv) * hd].view(nkv, hd).to(torch.bfloat16)
        v_new = qkv[b, (nh + nkv) * hd:].view(nkv, hd).to(torch.bfloat16)
        # the appended row: bit-exact with the conversion kernel on the same bf16 row
        for side, row in ((0, k_new), (1, v_new)):
            want = _quantize(row.view(nkv, 1, hd), gs)
            for got_t, want_t in zip((codes, scales, biases), want):
                assert torch.equal(got_t[side, b, :, c], want_t[:, 0]), (b, side)
            # nothing else of the row changed
            for got_t, old_t in zip((codes, scales, biases), before):
                assert torch.equal(got_t[side, b, :, :c], old_t[side, b, :, :c])
        # sdpa (the oracle's, bf16 rounding points) over the dequantized cache, the new row included
        K = _dequant(codes[0, b, :, :c + 1], scales[0, b, :, :c + 1], biases[0, b, :, :c + 1], gs).cpu()
        V = _dequant(codes[1, b, :, :c + 1], scales[1, b, :, :c + 1], biases[1, b, :, :c + 1], gs).cpu()
        want = S.sdpa(S.Rounder("bf16"), q.float().cpu()[None, :, None, :], K[None], V[None], hd ** -0.5, causal=False)
        cmp_bf16(out[b].view(nh, hd).cpu(), want[0, :, 0], f"B={B} hd={hd} gs={gs} row {b} ctx={c}", rel_l2=1e-3,
                 max_mismatch=0.05)
        # the single-row 8-bit attention on the row alone
        stage = torch.zeros(2, nkv, cap, hd, dtype=torch.bfloat16, device="cuda")
        stage[0, :, c] = k_new
        stage[1, :, c] = v_new
        pl = [t[:, b].clone() for t in before]   # (2, nkv, cap, ...) planes before the append
        one = torch.zeros(nh * hd, dtype=torch.bfloat16, device="cuda")
        N.check(lib.b200_kvq_decode_attention(q.to(torch.bfloat16).contiguous().data_ptr(), pl[0][0].data_ptr(),
                                              pl[1][0].data_ptr(), pl[2][0].data_ptr(), pl[0][1].data_ptr(),
                                              pl[1][1].data_ptr(), pl[2][1].data_ptr(), stage[0].data_ptr(),
                                              stage[1].data_ptr(), one.data_ptr(), nh, nkv, hd, cap, c, gs, 4, s),
                "kvq_decode_attention")
        cmp_bf16(out[b].cpu(), one.cpu(), f"B={B} hd={hd} gs={gs} row {b}: batched vs single-row", rel_l2=1e-3,
                 max_mismatch=0.05)


def _rope_ref(x, pos, inv_freq):
    """warp_head_rope (csrc/common.cuh): rotate_half at one position, rounding points of the kernel; x (..., hd)"""
    h = x.shape[-1] // 2
    ang = pos * inv_freq
    c, sn = _bf(torch.cos(ang)), _bf(torch.sin(ang))
    y1, y2 = x[..., :h], x[..., h:]
    return torch.cat([_bf(_bf(y1 * c) + _bf(-y2 * sn)), _bf(_bf(y2 * c) + _bf(y1 * sn))], -1)


def _rms_ref(x, w, eps):
    """warp_head_rms (csrc/common.cuh): RMSNorm of each head, two roundings"""
    rs = 1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + eps)
    return _bf(_bf(x * rs) * w.float())


@pytest.mark.parametrize("hd", [64, 128])
def test_batch_kvq_attention_op_qk_norm_rope_bias(hd):
    """the 8-bit lock-step attention with what a Qwen3-VL layer adds (q/k RMSNorm per head) and what every layer has
    (bias, M-RoPE at each row's own position): the appended V row is bit-exact (bias only); the appended K row is the
    quantization of the normalised, rotated key within the noise of two fp32 evaluations of the norm and rotary; the
    output is within relative L2 1e-3 of sdpa over the dequantized cache with q normalised and rotated the same way.
    A kernel that skipped the norm, the rotary or the bias fails all three by orders of magnitude."""
    from mlx_vlm_b200 import _native as N
    from oracle import mlx_semantics as S
    from _util import cmp_bf16, rl2
    lib = N.lib()
    torch.manual_seed(hd)
    B, gs, nkv, nh, cap, eps = 3, 64, 2, (4 if hd == 64 else 8), 512, 1e-6
    QKV = (nh + 2 * nkv) * hd
    ctx = np.asarray([0, 137, 380], dtype=np.int32)
    pos = np.asarray([5, 150, 1021], dtype=np.int32)
    cache = (torch.randn(2, B, nkv, cap, hd, device="cuda") * 0.8).to(torch.bfloat16)
    codes, scales, biases = (t.view(2, B, nkv, cap, -1).contiguous()
                             for t in _quantize(cache.view(-1, cap, hd), gs))
    qkv = _bf(torch.randn(B, QKV, device="cuda") * 2.0)
    bias = (torch.randn(QKV, device="cuda") * 0.5).to(torch.bfloat16)
    inv_freq = (1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda", dtype=torch.float32) / hd))).contiguous()
    qn = (1.0 + 0.3 * torch.randn(hd, device="cuda")).to(torch.bfloat16)
    kn = (1.0 + 0.3 * torch.randn(hd, device="cuda")).to(torch.bfloat16)
    ctx_d, pos_d = torch.from_numpy(ctx).cuda(), torch.from_numpy(pos).cuda()
    out = torch.zeros(B, nh * hd, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200_batch_kvq_attention(qkv.data_ptr(), bias.data_ptr(), inv_freq.data_ptr(), ctx_d.data_ptr(),
                                         pos_d.data_ptr(), codes.data_ptr(), scales.data_ptr(), biases.data_ptr(), gs,
                                         B, cap, out.data_ptr(), B, nh, nkv, hd, qn.data_ptr(), kn.data_ptr(), eps, s),
            "batch_kvq_attention")
    torch.cuda.synchronize()
    scale_bf = float(torch.tensor(hd ** -0.5).to(torch.bfloat16))
    a = _bf(qkv + bias.float())
    for b in range(B):
        c, p = int(ctx[b]), float(pos[b])
        q = _bf(_rope_ref(_rms_ref(a[b, :nh * hd].view(nh, hd), qn, eps), p, inv_freq) * scale_bf)
        k = _rope_ref(_rms_ref(a[b, nh * hd:(nh + nkv) * hd].view(nkv, hd), kn, eps), p, inv_freq)
        v = a[b, (nh + nkv) * hd:].view(nkv, hd)
        for got_t, want_t in zip((codes, scales, biases), _quantize(v.to(torch.bfloat16).view(nkv, 1, hd), gs)):
            assert torch.equal(got_t[1, b, :, c], want_t[:, 0]), (b, "V")
        kq = _quantize(k.to(torch.bfloat16).view(nkv, 1, hd), gs)
        got_k = _dequant(codes[0, b, :, c], scales[0, b, :, c], biases[0, b, :, c], gs)
        want_k = _dequant(kq[0][:, 0], kq[1][:, 0], kq[2][:, 0], gs)
        same = (codes[0, b, :, c] == kq[0][:, 0]).float().mean().item()
        print(f"hd={hd} row {b}: appended K codes equal to the restatement's: {same:.4f}, rel_l2 {rl2(got_k, want_k):.2e}")
        assert rl2(got_k, want_k) <= 1e-2 and same >= 0.95, (b, same, rl2(got_k, want_k))
        K = _dequant(codes[0, b, :, :c + 1], scales[0, b, :, :c + 1], biases[0, b, :, :c + 1], gs).cpu()
        V = _dequant(codes[1, b, :, :c + 1], scales[1, b, :, :c + 1], biases[1, b, :, :c + 1], gs).cpu()
        # q arrives already scaled and rounded: sdpa with scale 1 keeps that one rounding
        want = S.sdpa(S.Rounder("bf16"), q.cpu()[None, :, None, :], K[None], V[None], 1.0, causal=False)
        cmp_bf16(out[b].view(nh, hd).cpu(), want[0, :, 0], f"qk-norm hd={hd} row {b} ctx={c} pos={int(p)}",
                 rel_l2=1e-3, max_mismatch=0.05)


# ------------------------------------------------------------------------------------------ end to end
def _oracle_batch_rule(c, W, ids, pv, grid, n, gs, dtype="bf16"):
    """oracle greedy loop of ONE row under the batch rule: every layer where should_quantize_kv_layer holds keeps its
    rows in quantized form from the first prefill on (QuantOracleCache converted while empty)"""
    from kvq_ref import QuantOracleCache
    from oracle import mlx_semantics as S
    from oracle import qwen2vl as O
    from mlx_vlm_b200.models.cache import should_quantize_kv_layer
    R = S.Rounder(dtype)
    ids = np.asarray(ids, dtype=np.int64)
    L = c.text.num_hidden_layers
    embeds, _, pos, deltas = O.get_input_embeddings(c, W, ids, pv, grid, R)
    cache = [QuantOracleCache(gs) for _ in range(L)]
    for l, cc in enumerate(cache):
        cc.quantized = should_quantize_kv_layer(l, L)
    hidden = O.lm_layers_forward(c, W, embeds, pos, cache, R)
    logits = O.lm_head(c, W, hidden[:, -1, :], R)
    toks, lps = [], []
    for i in range(n):
        lp = O.logprobs_from_logits(R, logits)
        y = S.argmax_lowest(lp)
        toks.append(int(y[0]))
        lps.append(lp[0].float())
        if i == n - 1:
            break
        e = W["language_model.model.embed_tokens.weight"][y][:, None, :]
        hidden = O.lm_layers_forward(c, W, e, O.decode_position_ids(cache[0].offset, deltas, 1), cache, R)
        logits = O.lm_head(c, W, hidden[:, -1, :], R)
    return toks, lps, cache


def _wide3():
    from oracle import qwen2vl as O
    from mlx_vlm_b200.models.qwen2_vl import Model
    c = O.qwen2_vl_2b()
    c.text.num_hidden_layers = 3   # 2B widths, 3 layers: the last one stays bf16 under the batch rule
    c.vision.depth = 1
    W = O.init_weights(c, 0, norm_jitter=0.05)
    model = Model(_to_model_config(c), device="cuda:0")
    model.load_weights(W)
    return c, W, model, O.synthetic_request(c, 10, image_hw=(56, 56), seed=0)


def _rows(c, req, lens, seed=3):
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    rng = np.random.default_rng(seed)
    rows = [(ids, {"pixel_values": torch.from_numpy(pv).cuda(), "image_grid_thw": grid}, 8)]
    for i, n in enumerate(lens):
        rows.append((rng.integers(0, 900, size=(1, n)), {}, 6 + 3 * i))
    return rows


def _run_gen(model, rows, **kw):
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    g = BatchGenerator(model, proc, compute_logprobs=True, **kw)
    assert g._lockstep
    uids = g.insert([r[0] for r in rows], [r[2] for r in rows], [r[1] for r in rows])
    got = {u: [] for u in uids}
    while g.has_work:
        _, rs = g.next()
        for r in rs:
            got[r.uid].append((r.token, r.token_logprob))
    assert model.engine.device_error() == 0
    return [got[u] for u in uids], g


def _check_rows(c, W, rows, got, gs, name):
    for i, ((ids, kw, n), g) in enumerate(zip(rows, got)):
        pv = kw.get("pixel_values")
        toks, lps, _ = _oracle_batch_rule(c, W, ids, None if pv is None else pv.cpu().numpy(),
                                          kw.get("image_grid_thw"), n, gs)
        assert len(g) == n
        for t, ((gt, _), wt) in enumerate(zip(g, toks)):
            if gt != wt:
                assert _token_ok(gt, lps[t]), f"{name} row {i} token {t}: {gt} vs oracle {wt} is not a near-tie"
                break


@pytest.mark.parametrize("kind,gs", [("tiny", 64), ("wide3", 64), ("tiny", 32)])
def test_batch_generator_kv8_against_batch_rule_oracle(kind, gs):
    from oracle import qwen2vl as O
    if kind == "wide3":
        c, W, model, req = _wide3()
    else:
        c, W, model, req = _build(kind, 10, (56, 56))
    rows = _rows(c, req, [9, 23, 14])
    # step-0 logprobs of every row on the noise bar (a row prefilled into an 8-bit batch pool)
    lm, eng = model.language_model, model.engine
    from mlx_vlm_b200.models.cache import BatchKVQPool
    pool = BatchKVQPool(c.text.num_hidden_layers, lm.n_kv_heads, lm.head_dim, eng.device, group_size=gs, batch=4,
                        capacity=256, stream=eng.stream)
    for b, (ids, kw, _) in enumerate(rows):
        emb = model.get_input_embeddings(ids, kw.get("pixel_values"), image_grid_thw=kw.get("image_grid_thw"))
        rc = lm.make_cache_row(pool, b)
        lm._rope_deltas, lm._position_ids = None, None
        lm(ids, inputs_embeds=emb.inputs_embeds, cache=rc, position_ids=emb.position_ids,
           rope_deltas=emb.rope_deltas, logits_to_keep=1, reserve_tokens=64)
        eng.stream.synchronize()
        lp0 = eng.logprobs_view().float().cpu().clone()
        pv = kw.get("pixel_values")
        pv = None if pv is None else pv.cpu().numpy()
        _, ref, ocache = _oracle_batch_rule(c, W, ids, pv, kw.get("image_grid_thw"), 1, gs)
        _, ex, _ = _oracle_batch_rule(c, W, ids, pv, kw.get("image_grid_thw"), 1, gs, dtype="f32")
        # The noise bar of a bf16 pipeline is slack 1.5 (two independent rounding realisations).  An 8-bit cache adds
        # one more noise source: a K/V element one bf16 ulp apart between the two pipelines can move its code by a
        # whole quantization step (~range / 255, far above an ulp).  Where such flips are measured in the prompt's
        # layer-0 keys, the bar widens to slack 2.0; without flips the bf16 bar applies unchanged.
        T = int(rc[0].offset)
        q = pool.q
        mine = _dequant(q.codes[0, 0, b, :, :T], q.scales[0, 0, b, :, :T], q.biases[0, 0, b, :, :T], gs).cpu()
        flips = (mine != ocache[0].keys[0, :, :T].float()).float().mean().item()
        d_pair, d_ref = rl2(lp0, ref[0]), rl2(ref[0], ex[0])
        print(f"{kind} gs={gs} row {b}: layer-0 K elements off by a quantization step: {flips:.4f}, "
              f"|cuda-oracle_bf16| / |oracle_bf16-exact| = {d_pair / d_ref:.2f}")
        cmp_noise(lp0, ref[0], ex[0], f"{kind} row {b} step-0 logprobs", slack=1.5 if flips == 0 else 2.0)
    got, _ = _run_gen(model, rows, kv_bits=8, kv_group_size=gs, completion_batch_size=4, decode_slice=4)
    _check_rows(c, W, rows, got, gs, kind)


def test_batch_generator_kv8_lifecycle_growth_and_chunked_admission():
    """5 rows through 3 slots: rows join while others decode and finish with compaction; the longest prompt joins
    last and grows the pool past 256 positions while other rows are live.  Chunked admission (prefill_step_size
    smaller than the prompts) gives the same tokens and logprobs bit for bit."""
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _rows(c, req, [12, 30, 19, 230])
    rows[-1] = (rows[-1][0], {}, 40)   # 230 + 40 + 1 > 256: the pool grows when this row is admitted
    got, g = _run_gen(model, rows, kv_bits=8, completion_batch_size=3, prefill_batch_size=2, decode_slice=3)
    assert g._pool.capacity >= 512 and g._pool.bf is None   # 2 layers: every layer 8-bit
    _check_rows(c, W, rows, got, 64, "lifecycle")
    chunked, _ = _run_gen(model, rows, kv_bits=8, completion_batch_size=3, prefill_batch_size=2, decode_slice=3,
                          prefill_step_size=16)
    assert chunked == got


def _row_bytes(pool, b, n):
    out = [t[:, :, b, :, :n].clone() for t in (pool.q.codes, pool.q.scales, pool.q.biases)]
    if pool.bf is not None:
        out.append(pool.bf.buf[:, :, b, :, :n].clone())
    return out


def test_cache_surgery_is_byte_exact_and_nbytes():
    c, W, model, req = _wide3()
    lm, eng = model.language_model, model.engine
    rows_req = _rows(c, req, [9, 21, 13])
    rows, caches = lm.make_batch_cache(3, 256, kv_bits=8, kv_group_size=64)
    from mlx_vlm_b200.models.cache import BatchQuantizedKVCache, RowBatchKVCache
    assert [type(x) for x in caches] == [BatchQuantizedKVCache, BatchQuantizedKVCache, RowBatchKVCache]
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
    inputs = np.asarray(firsts)
    for _ in range(3):
        inputs = lm.fused_greedy_decode(inputs[:, None], cache=caches, rope_deltas=np.asarray(deltas)[:, None])
    eng.stream.synchronize()
    assert eng.device_error() == 0
    # memory: 8-bit planes for layers 0, 1, bf16 for layer 2 (0.53x bf16 on the 8-bit layers at group size 64)
    nb = [x.nbytes for x in caches]
    assert nb[0] == nb[1] and abs(nb[0] / nb[2] - 0.53125) < 1e-9
    lens = list(rows.lengths)
    snap = {b: _row_bytes(rows.pool, b, lens[b]) for b in (0, 2)}
    for x in caches:
        x.filter([0, 2])
    for new_b, old_b in enumerate((0, 2)):
        for a, w in zip(_row_bytes(rows.pool, new_b, lens[old_b]), snap[old_b]):
            assert torch.equal(a, w)
    # extend by a one-row batch of its own
    other, oc = lm.make_batch_cache(1, 256, kv_bits=8, kv_group_size=64)
    rid, kw, _ = rows_req[1]
    other.lengths = [0]
    lm._rope_deltas, lm._position_ids = None, None
    lm(rid, cache=lm.make_cache_row(other.pool, 0), logits_to_keep=1, reserve_tokens=256)
    other.lengths = [rid.shape[1]]
    eng.stream.synchronize()
    osnap = _row_bytes(other.pool, 0, rid.shape[1])
    for x, y in zip(caches, oc):
        x.extend(y)
    eng.stream.synchronize()
    assert rows.B == 3
    for a, w in zip(_row_bytes(rows.pool, 2, rid.shape[1]), osnap):
        assert torch.equal(a, w)
    for new_b, old_b in enumerate((0, 2)):
        for a, w in zip(_row_bytes(rows.pool, new_b, lens[old_b]), snap[old_b]):
            assert torch.equal(a, w)
    ex = caches[0].extract(1)
    eng.stream.synchronize()
    n = ex.offset
    assert n == rows.lengths[1]
    for a, w in zip(ex.keys, caches[0].keys):
        assert torch.equal(a[0, :, :n], w[1, :, :n])


def test_extract_follows_decode_and_continues_under_generate_step():
    """every layer of a 2-layer stack is 8-bit, so an extracted row is a complete single-request 8-bit cache.  An
    extract, three lock-step steps, then a second extract: the second holds the row as it is now, byte for byte, in a
    pool of its own, and the first is untouched.  The first extract, continued under generate_step(kv_bits=8), gives
    the tokens the lock-step batch gave that row (up to a near-tie)."""
    from mlx_vlm_b200.generate import generate_step
    c, W, model, req = _build("tiny", 10, (56, 56))
    lm, eng = model.language_model, model.engine
    rows, caches = lm.make_batch_cache(2, 256, kv_bits=8, kv_group_size=64)
    rng = np.random.default_rng(1)
    prompts = [rng.integers(0, 900, size=(1, 17)), rng.integers(0, 900, size=(1, 11))]
    rows.lengths = [0, 0]
    firsts = []
    for b, p in enumerate(prompts):
        lm._rope_deltas, lm._position_ids = None, None
        lm(p, cache=lm.make_cache_row(rows.pool, b), logits_to_keep=1, reserve_tokens=256)
        eng.stream.synchronize()
        firsts.append(int(eng.token_log_view()[(eng.tokens_launched - 1) % eng.token_log_capacity]))
        rows.lengths[b] = p.shape[1]
    rows._touch()
    a = [x.extract(1) for x in caches]
    eng.stream.synchronize()
    assert all(e._pool is a[0]._pool for e in a) and a[0].offset == 11
    a_bytes = [t.clone() for t in (a[0]._pool.codes, a[0]._pool.scales, a[0]._pool.biases)]
    inputs, steps = np.asarray(firsts), []
    for _ in range(3):
        inputs = lm.fused_greedy_decode(inputs[:, None], cache=caches, rope_deltas=np.zeros((2, 1), np.int64))
        eng.stream.synchronize()
        steps.append(int(inputs[1]))
    assert rows.lengths == [20, 14]
    bq = [x.extract(1) for x in caches]
    eng.stream.synchronize()
    assert bq[0]._pool is not a[0]._pool and bq[0].offset == 14
    q = rows.pool.q
    for got, pool_t in zip((bq[0]._pool.codes, bq[0]._pool.scales, bq[0]._pool.biases), (q.codes, q.scales, q.biases)):
        assert torch.equal(got[:, :, 0, :, :14], pool_t[:, :, 1, :, :14])
    for got, was, pool_t in zip((a[0]._pool.codes, a[0]._pool.scales, a[0]._pool.biases), a_bytes,
                                (q.codes, q.scales, q.biases)):
        assert torch.equal(got, was) and torch.equal(got[:, :, 0, :, :11], pool_t[:, :, 1, :, :11])
    toks, lps = [], []
    for t, lp in generate_step(np.asarray([[firsts[1]]]), model, None, None, max_tokens=3, prompt_cache=a,
                               kv_bits=8, kv_group_size=64, quantized_kv_start=0):
        toks.append(int(t))
        lps.append(lp.float().cpu())
    assert eng.device_error() == 0
    for i, (g, w) in enumerate(zip(toks, steps)):
        if g != w:
            assert _token_ok(w, lps[i]), f"continued row: token {i} {g} vs lock-step {w} is not a near-tie"
            break


def test_qwen3_vl_lockstep_kv8_runs_clean():
    """a Qwen3-VL geometry that runs lock-step (head_dim == hidden / heads) end to end with kv_bits=8: every row gets
    all its tokens, from a batch pool with both layers 8-bit, with no device error.  The arithmetic of the 8-bit
    kernel's q/k-norm branch is checked at op level (test_batch_kvq_attention_op_qk_norm_rope_bias)."""
    from test_qwen3_vl_gpu import _model
    from mlx_vlm_b200.models.cache import BatchKVQPool
    cfg, W, model = _model("tiny")
    rng = np.random.default_rng(0)
    rows = [(rng.integers(0, 900, size=(1, n)), {}, 8) for n in (7, 19, 12)]
    got8, g8 = _run_gen(model, rows, kv_bits=8, completion_batch_size=3)
    assert isinstance(g8._pool, BatchKVQPool) and g8._pool.n_q == 2 and g8._pool.bf is None
    assert [len(r) for r in got8] == [8, 8, 8]
