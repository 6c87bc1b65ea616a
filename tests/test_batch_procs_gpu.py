"""Per-row logits processors and top-k logprobs in the lock-step batch (csrc/decode_batch.cu `bd_procs_kernel`,
`bd_topk_*`): the device path must compute what the same processors compute as torch ops.

The torch restatement is the processors themselves, run by the batch's host path: a processor list that does not
lower (here the same closures wrapped in plain functions) runs as torch ops on the row's logits, one step at a time.
Both paths share the lock-step head, so a row's tokens, token logprobs and top-k ids must be identical; logprobs are
held to one bf16 ulp because the host path takes its logsumexp with torch and the device path with bd_sample.
Against the single-request path (`generate_step`, a different decode kernel) rows agree until the first near-tie,
as in test_batch_gpu.py."""
import threading
import types

import numpy as np
import pytest

from test_batch_gpu import _requests, _same_until_tie
from test_engine_gpu import _build

pytestmark = pytest.mark.gpu

K_TOP = 5


def _settings(n, hist_ids):
    """per-row processor settings: none, each penalty alone, all four, an unknown callable"""
    from mlx_vlm_b200.sample_utils import make_logits_processors
    bias = {int(hist_ids[0]): 2.5, int(hist_ids[-1]): -1.75, 7: 0.5}   # ids that are also in the history
    table = [
        {},
        {"repetition_penalty": 1.3, "repetition_context_size": 8},
        {"presence_penalty": 0.7, "presence_context_size": 64},
        {"frequency_penalty": 0.45, "frequency_context_size": 1000},
        {"logit_bias": bias},
        {"logit_bias": bias, "repetition_penalty": 0.8, "presence_penalty": -0.3, "frequency_penalty": 0.6},
        "unknown",
        {},
    ]
    out = []
    for i in range(n):
        s = table[i % len(table)]
        if s == "unknown":
            rep = make_logits_processors(repetition_penalty=1.5)[0]
            out.append([lambda toks, lg, p=rep: p(toks, lg)])
        else:
            out.append(make_logits_processors(**s) or None)
    return out


def _as_host(procs):
    """the same processors as callables the batch does not recognise: the torch path"""
    return [None if p is None else [lambda toks, lg, q=q: q(toks, lg) for q in p] for p in procs]


def _run(model, rows, procs, *, decode_slice, top_k=K_TOP, kv_bits=None, insert_late=0, **kw):
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    g = BatchGenerator(model, proc, completion_batch_size=8, prefill_batch_size=3, decode_slice=decode_slice,
                       top_logprobs_k=top_k, kv_bits=kv_bits, **kw)
    n0 = len(rows) - insert_late
    uids = g.insert([r[0] for r in rows[:n0]], [r[2] for r in rows[:n0]], [r[1] for r in rows[:n0]],
                    logits_processors=procs[:n0])
    got = {}
    steps = 0
    while g.has_work:
        _, rs = g.next()
        steps += 1
        if steps == 3 and insert_late:   # insertion while other rows decode
            uids += g.insert([r[0] for r in rows[n0:]], [r[2] for r in rows[n0:]], [r[1] for r in rows[n0:]],
                             logits_processors=procs[n0:])
        for r in rs:
            got.setdefault(r.uid, []).append((r.token, r.token_logprob, r.top_logprobs))
    assert model.engine.device_error() == 0
    return [got[u] for u in uids]


def _ulp_close(a, b):
    return abs(a - b) <= abs(b) * 2.0 ** -7 + 1e-6


def _same(dev, host, name, exact_lp=False):
    assert len(dev) == len(host)
    for b, (d, h) in enumerate(zip(dev, host)):
        assert [t for t, _, _ in d] == [t for t, _, _ in h], f"{name} row {b}: tokens differ"
        for i, ((_, ld, td), (_, lh, th)) in enumerate(zip(d, h)):
            assert (ld == lh) if exact_lp else _ulp_close(ld, lh), f"{name} row {b} step {i}: logprob {ld} vs {lh}"
            if td is not None or th is not None:
                assert [x for x, _ in td] == [x for x, _ in th], f"{name} row {b} step {i}: top-k ids {td} vs {th}"
                assert all(_ulp_close(x, y) for (_, x), (_, y) in zip(td, th))


@pytest.mark.parametrize("kind", ["tiny", "oddvocab"])
def test_device_processors_equal_torch_processors(kind):
    """8 lock-step rows, images in some, mixed settings: the device path (8-step device loop and one step at a
    time) against the torch path; rows leave at different lengths (filter) and join during generation"""
    c, W, model, req = _build(kind, 10, (56, 56))
    rows = _requests(c, req, 8)
    procs = _settings(8, np.asarray(req["input_ids"]).reshape(-1))
    dev8 = _run(model, rows, procs, decode_slice=8, insert_late=3)
    dev1 = _run(model, rows, procs, decode_slice=1, insert_late=3)
    host = _run(model, rows, _as_host(procs), decode_slice=1, insert_late=3)
    _same(dev8, dev1, f"{kind} device loop", exact_lp=True)
    _same(dev8, host, f"{kind} device vs torch")
    for b, r in enumerate(dev8):
        assert all(top is not None and len(top) == K_TOP for _, _, top in r)
        for tok, lp, top in r:   # the order the kernel defines: logprob descending, lower id first on ties
            assert all((x[1] > y[1]) or (x[1] == y[1] and x[0] < y[0]) for x, y in zip(top, top[1:]))


def test_rows_without_processors_unchanged():
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _requests(c, req, 8)
    procs = _settings(8, np.asarray(req["input_ids"]).reshape(-1))
    # one admission path for both runs (rows with processors are prefilled one at a time)
    mixed = _run(model, rows, procs, decode_slice=8, top_k=0, batched_prefill=False)
    plain = _run(model, rows, [None] * 8, decode_slice=8, top_k=0, batched_prefill=False)
    for b, p in enumerate(procs):
        if p is None:
            assert mixed[b] == plain[b], f"row {b} without processors changed"


def test_batch_rows_equal_single_requests():
    """each row against generate_step with the same processors (until the first near-tie)"""
    from mlx_vlm_b200.generate import generate_step
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _requests(c, req, 8)
    procs = _settings(8, np.asarray(req["input_ids"]).reshape(-1))
    got = _run(model, rows, procs, decode_slice=8)
    agree = total = 0
    for b, ((ids, kw, n), p) in enumerate(zip(rows, procs)):
        toks, lps = [], []
        for t, lp in generate_step(ids, model, kw.get("pixel_values"), None, max_tokens=n,
                                   image_grid_thw=kw.get("image_grid_thw"), logits_processors=p):
            toks.append(t)
            lps.append(lp.float().cpu())
        agree += _same_until_tie([t for t, _, _ in got[b]], toks, lps, f"row {b}")
        total += n
    print(f"{agree}/{total} tokens identical to the single-request path")
    assert agree >= 0.7 * total


def test_kv8_lockstep_penalised_batch():
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _requests(c, req, 4)
    procs = _settings(6, np.asarray(req["input_ids"]).reshape(-1))[1:5]
    out = _run(model, rows, procs, decode_slice=4, kv_bits=8)
    assert [len(r) for r in out] == [r[2] for r in rows]


def test_time_multiplexed_penalised_batch():
    """rows over the single-request path (the engines without the batched decoder) run their processors as torch ops"""
    c, W, model, req = _build("tiny", 10, (56, 56))
    rows = _requests(c, req, 4)
    procs = _settings(6, np.asarray(req["input_ids"]).reshape(-1))[1:5]
    out = _run(model, rows, procs, decode_slice=4, time_multiplex=True)
    assert [len(r) for r in out] == [r[2] for r in rows]
    assert all(top is not None and len(top) == K_TOP for r in out for _, _, top in r)


def test_response_generator_penalties_and_top_logprobs():
    from mlx_vlm_b200.server import GenerationArguments, ResponseGenerator
    c, W, model, req = _build("tiny", 10, (56, 56))
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    rg = ResponseGenerator(model, proc, completion_batch_size=8, decode_slice=4)
    results, errors = {}, []

    def caller(i):
        try:
            ids = np.random.default_rng(i).integers(0, 900, size=(1, 8 + i))
            args = GenerationArguments(max_tokens=6 + i)
            if i % 2:
                args.repetition_penalty, args.logit_bias, args.top_logprobs = 1.2, {5: 1.0}, 3 + i
            results[i] = (args, list(rg.generate({"input_ids": ids}, args)))
        except Exception as e:   # reported below
            errors.append(e)

    ts = [threading.Thread(target=caller, args=(i,)) for i in range(6)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(300)
    rg.stop_and_join()
    assert not errors, errors
    for i, (args, events) in results.items():
        assert len(events) == args.max_tokens
        k = args.top_k()
        for e in events:
            assert (e.top_logprobs is None) if k == 0 else len(e.top_logprobs) == k
    assert model.engine.device_error() == 0


@pytest.mark.parametrize("V", [151936, 32003])
def test_kernels_against_torch_restatement(V):
    """bd_procs_kernel and the top-k kernels on synthetic bf16 logits (b200_batch_procs_apply), bit for bit against
    `make_logits_processors` and `top_logprobs`: negative logits, repeated history tokens, a history longer than the
    device ring, windows longer than the history, bias ids that are also in the history, an inactive row (no append),
    and ties at the maximum placed in different 8192-token slices of the top-k part kernel"""
    import torch
    from mlx_vlm_b200 import _native as N
    from mlx_vlm_b200.models.cache import BatchProcState
    from mlx_vlm_b200.sample_utils import lower_logits_processors, make_logits_processors, top_logprobs
    lib, dev = N.lib(), "cuda:0"
    ldv, B, cap = (V + 7) // 8 * 8, 6, BatchProcState.HIST_CAP
    g = torch.Generator().manual_seed(V)
    logits = (torch.randn(B, V, generator=g) * 3 - 1).to(torch.bfloat16)
    ties = (3, 8191, 8192, 16384, V - 1)
    for b in range(B):
        logits[b, list(ties)] = float(logits[b].float().max()) + 1
    long = torch.randint(0, V, (cap + 476,), generator=g).tolist()
    long[-40:] = [8192] * 10 + long[-30:]
    hists = [[5, 5, 5, 8191, 3, 9], long, [11, 12, 11, 8192], [3, 16384, 7, 7, 100], [1, 2, 3], long[:300] * 4]
    settings = [dict(repetition_penalty=1.3, repetition_context_size=6),
                dict(presence_penalty=0.7, presence_context_size=1000, frequency_penalty=0.45,
                     frequency_context_size=cap),
                dict(repetition_penalty=0.8, repetition_context_size=50, frequency_penalty=-0.3,
                     frequency_context_size=64),
                dict(logit_bias={3: 2.5, 16384: -1.75, V - 1: 0.3, 7: 0.1}, presence_penalty=0.2,
                     presence_context_size=3),
                {},
                dict(logit_bias={8191: -3.0, long[5]: 1.0}, repetition_penalty=1.1, repetition_context_size=900,
                     presence_penalty=-0.5, presence_context_size=20, frequency_penalty=0.6,
                     frequency_context_size=700)]
    procs = [make_logits_processors(**s) for s in settings]
    tok = [8192, 8192, 11, 3, 4, 77]
    active = [1, 1, 1, 1, 1, 0]
    st = BatchProcState(dev)
    for b in range(B):
        st.set_row(b, lower_logits_processors(procs[b]), hists[b], V)
    dl = torch.full((B, ldv), float("-inf"), dtype=torch.bfloat16, device=dev)
    dl[:, :V] = logits.to(dev)
    t_tok = torch.tensor(tok, dtype=torch.int32, device=dev)
    t_act = torch.tensor(active, dtype=torch.int32, device=dev)
    ids = torch.zeros(B, 20, dtype=torch.int32, device=dev)
    lps = torch.zeros(B, 20, dtype=torch.float32, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200_batch_procs_apply(dl.data_ptr(), None, B, V, ldv, t_tok.data_ptr(), t_act.data_ptr(),
                                       st.params.data_ptr(), st.penalties.data_ptr(), st.bias_ids.data_ptr(),
                                       st.bias_vals.data_ptr(), st.BIAS_CAP, st.hist.data_ptr(),
                                       st.hist_len.data_ptr(), cap, 0, None, None, s), "procs_apply")
    torch.cuda.synchronize()
    want_lp = []
    for b in range(B):
        ctx = hists[b] + ([tok[b]] if active[b] else [])
        want = logits[b:b + 1].to(dev)
        for p in procs[b]:
            want = p(ctx, want)
        got = dl[b:b + 1, :V]
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
            f"row {b}: {(got != want).sum().item()} logits differ"
        assert torch.equal(dl[b, V:].float(), torch.full((ldv - V,), float("-inf"), device=dev))
        if procs[b]:
            assert st.history(b) == ctx[-cap:], f"row {b}: device history"
        want_lp.append(want - torch.logsumexp(want.float(), dim=-1, keepdim=True).to(want.dtype))
    lp = torch.full((B, ldv), float("-inf"), dtype=torch.bfloat16, device=dev)
    lp[:, :V] = torch.cat(want_lp)
    N.check(lib.b200_batch_procs_apply(None, lp.data_ptr(), B, V, ldv, None, None, None, None, None, None, 0, None,
                                       None, 0, 20, ids.data_ptr(), lps.data_ptr(), s), "procs_apply top-k")
    torch.cuda.synchronize()
    for b in range(B):
        ref = top_logprobs(lp[b, :V], 20)
        assert list(zip(ids[b].tolist(), lps[b].tolist())) == ref, f"row {b}: top-k"
    assert [i for i, _ in top_logprobs(lp[4, :V], 5)] == sorted(ties)   # the untouched row keeps its ties
