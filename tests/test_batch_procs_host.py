"""CPU: per-row logits processors and top-k logprobs of the batch — lowering of `make_logits_processors` to the
lock-step kernel's parameters, the per-row device state (`BatchProcState`) and how it moves with rows, the
reference's token-context and processor-list bookkeeping (ar.py:995-1013, 1070-1074, 1174-1278), and a server
request that sets penalties and top_logprobs, on the engine stand-in of test_batch_host.py."""
import itertools
import threading

import numpy as np
import pytest
import torch

from test_batch_host import _fake_model

KINDS = ("bias", "repetition", "presence", "frequency")


def _procs(kinds):
    from mlx_vlm_b200.sample_utils import make_logits_processors
    kw = {}
    if "bias" in kinds:
        kw["logit_bias"] = {3: 1.5, 9: -2.0}
    if "repetition" in kinds:
        kw.update(repetition_penalty=1.25, repetition_context_size=7)
    if "presence" in kinds:
        kw.update(presence_penalty=0.5, presence_context_size=11)
    if "frequency" in kinds:
        kw.update(frequency_penalty=0.3, frequency_context_size=13)
    return make_logits_processors(**kw)


@pytest.mark.parametrize("kinds", [c for n in range(5) for c in itertools.combinations(KINDS, n)])
def test_lowering_every_combination(kinds):
    from mlx_vlm_b200.sample_utils import lower_logits_processors
    low = lower_logits_processors(_procs(kinds))
    assert set(low) == set(kinds)
    if "bias" in kinds:
        assert low["bias"] == ({3: 1.5, 9: -2.0},)
    if "repetition" in kinds:
        assert low["repetition"] == (1.25, 7)
    if "presence" in kinds:
        assert low["presence"] == (0.5, 11)
    if "frequency" in kinds:
        assert low["frequency"] == (0.3, 13)


def test_unknown_or_reordered_processors_do_not_lower():
    from mlx_vlm_b200.sample_utils import lower_logits_processors
    rep = _procs(("repetition",))
    assert lower_logits_processors(rep + [lambda toks, lg: lg]) is None
    assert lower_logits_processors(_procs(("presence",)) + rep) is None      # the kernel's order is fixed
    assert lower_logits_processors(rep + rep) is None
    assert lower_logits_processors([]) == {}


def test_row_values_round_as_the_torch_ops():
    from mlx_vlm_b200.models.cache import BatchProcState
    low = {"bias": ({3: 0.1, 9: -2.0},), "repetition": (1.1, 20), "frequency": (0.3, 5)}
    par, pen, ids, vals = BatchProcState.row_values(low, 100)
    assert par[0] == 1 | 2 | 8 and par[1] == 20 and par[3] == 5 and par[4] == 2
    assert ids == [3, 9]
    assert vals == [float(torch.tensor(0.1, dtype=torch.bfloat16)), -2.0]
    assert pen[0] == np.float32(1.1) and pen[1] == np.float32(1) / np.float32(1.1) and pen[3] == np.float32(0.3)
    with pytest.raises(ValueError):
        BatchProcState.row_values({"bias": ({100: 1.0},)}, 100)
    assert not BatchProcState.fits({"repetition": (1.1, 0)})        # the whole history: torch path
    assert not BatchProcState.fits({"presence": (0.5, BatchProcState.HIST_CAP + 1)})


def test_history_ring_seed_and_moves():
    from mlx_vlm_b200.models.cache import BatchProcState
    st = BatchProcState("cpu")
    long = list(range(5000, 5000 + BatchProcState.HIST_CAP + 37))
    st.set_row(0, {"repetition": (1.1, 20)}, [1, 2, 3], 10 ** 5)
    st.set_row(1, {"presence": (0.5, 20)}, long, 10 ** 5)
    st.set_row(2, {}, [7], 10 ** 5)
    assert st.history(0) == [1, 2, 3]
    assert st.history(1) == long[-BatchProcState.HIST_CAP:]
    assert int(st.params[2, 0]) == 0
    st.move_rows(st, [0, 1], [1, 0])   # rows swap with their state
    assert st.history(0) == long[-BatchProcState.HIST_CAP:] and st.history(1) == [1, 2, 3]
    assert int(st.params[0, 0]) == 4 and int(st.params[1, 0]) == 2
    other = BatchProcState("cpu")
    other.move_rows(st, [5], [1])
    assert other.history(5) == [1, 2, 3]


def test_insert_alignment():
    """insert gives each prompt the generator's list or checks the per-prompt lists as the reference does
    (ar.py:2584-2604); the batch bookkeeping after insertion is checked against the reference's golden below"""
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model, proc = _fake_model()
    rep = _procs(("repetition",))
    g = BatchGenerator(model, proc, max_tokens=4, decode_slice=1, logits_processors=rep)
    with pytest.raises(ValueError):
        g.insert([[1, 2], [3]], logits_processors=[rep])
    g.insert([[1, 2, 3]])                                      # the generator's list
    g.insert([[4, 5], [6]], logits_processors=[None, rep])
    assert [r.procs for r in g.unprocessed_prompts] == [rep, None, rep]   # shortest first
    assert all(r.lowered == {"repetition": (1.25, 7)} for r in g.unprocessed_prompts if r.procs)


@pytest.mark.parametrize("lockstep", [False, True])
def test_token_context_grows_by_each_input_token(lockstep):
    """a processor sees the prompt, then each step's input token before it runs (ar.py:1070-1074)"""
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model, proc = _fake_model(lockstep=lockstep)
    seen = []

    def spy(tokens, logits):
        seen.append(list(tokens))
        return logits
    g = BatchGenerator(model, proc, max_tokens=4, decode_slice=2)
    g.insert([[5, 6, 7]], logits_processors=[[spy]])
    toks = []
    while g.has_work:
        _, rs = g.next()
        toks += [r.token for r in rs]
    assert seen == [[5, 6, 7] + toks[:i] for i in range(4)]


def test_server_accepts_penalties_and_top_logprobs():
    from mlx_vlm_b200.server import GenerationArguments
    from test_server_host import _server
    srv, _ = _server(lockstep=False)
    out = {}

    def client(i):
        args = GenerationArguments(max_tokens=5)
        if i:
            args.repetition_penalty, args.presence_penalty, args.frequency_penalty = 1.2, 0.1, 0.2
            args.logit_bias, args.top_logprobs = {"4": 0.5}, 3 if i == 1 else 50
        out[i] = (args, list(srv.generate({"input_ids": np.asarray([[1, 2, 3 + i]])}, args, timeout=20)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join(30)
    srv.stop_and_join()
    assert sorted(out) == [0, 1, 2]
    for i, (args, evs) in out.items():
        assert len(evs) == 5
        k = {0: 0, 1: 3, 2: 20}[i]
        assert args.top_k() == k
        for e in evs:
            assert (e.top_logprobs is None) if k == 0 else [len(e.top_logprobs)] == [k]
            if k:
                assert e.top_logprobs[0][0] == e.token


def test_server_rejects_a_bad_logit_bias_alone():
    """a logit bias outside the vocabulary fails its own request at insertion; a request running next to it
    completes"""
    from mlx_vlm_b200.server import GenerationArguments
    from test_batch_host import V
    from test_server_host import _server
    import types
    srv, model = _server(lockstep=False)
    model.language_model.args = types.SimpleNamespace(vocab_size=V)
    out = {}

    def client(i, bias):
        args = GenerationArguments(max_tokens=6, logit_bias=bias, repetition_penalty=1.1)
        try:
            out[i] = [e.token for e in srv.generate({"input_ids": np.asarray([[1, 2, 3 + i]])}, args, timeout=20)]
        except Exception as e:   # the bad request hears about its own error
            out[i] = e

    th = [threading.Thread(target=client, args=(i, b)) for i, b in enumerate([{V: 1.0}, {"-2": 1.0}, {4: 0.5}])]
    for t in th:
        t.start()
    for t in th:
        t.join(30)
    srv.stop_and_join()
    assert isinstance(out[0], ValueError) and isinstance(out[1], ValueError)
    assert isinstance(out[2], list) and len(out[2]) == 6


def test_bookkeeping_against_reference_golden():
    """tests/golden/batch_procs_golden.json (the reference's GenerationBatch executed by
    make_batch_procs_golden.py): processor-list alignment and token context through steps, extend and filter, the
    context each processor call sees, and the top-k ids"""
    import json
    import os
    from mlx_vlm_b200.generate_batch import GenerationBatch, _Row
    from mlx_vlm_b200.sample_utils import top_logprobs
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "batch_procs_golden.json")))
    tr = iter(g["trace"])
    prompts = {int(k): v for k, v in g["prompts"].items()}
    seen = []

    def proc(tokens, logits):
        return logits
    rows = {u: _Row(u, prompts[u], 8, {}, procs=[proc] if u == 0 else None) for u in prompts}

    def check(batch, ctx_of_row0_call=False):
        t = next(tr)
        assert [r.uid for r in batch.rows] == t["uids"], t["op"]
        assert [p is not None for p in batch.logits_processors] == t["has_processors"], t["op"]
        assert batch.token_context == t["token_context"], t["op"]
        return t

    def step(batch):
        t = g["trace"][len(done)]
        batch.record_inputs([(r, [x]) for r, x in zip(batch.rows, t["inputs"])])
        if any(r.uid == 0 for r in batch.rows):
            seen.append(list(rows[0].context))   # what row 0's processor is given at this step
        for lp, want in zip(t["logprobs"], t["next_top_idx"]):
            assert [i for i, _ in top_logprobs(torch.tensor(lp), g["top_k"])] == want
        done.append(check(batch))

    done = []
    a = GenerationBatch.admitted([rows[0], rows[1]])
    done.append(check(a))
    step(a)
    step(a)
    b = GenerationBatch.admitted([rows[2]])
    done.append(check(b))
    step(b)
    a.extend(b)
    done.append(check(a))
    step(a)
    a.filter([2, 0])
    done.append(check(a))
    step(a)
    a.filter([0])
    done.append(check(a))
    assert seen == [c["tokens"] for c in g["processor_calls"]]
