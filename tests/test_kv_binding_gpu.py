"""The engine's KV binding through Engine and the C ABI, on tiny Qwen2-VL and Qwen3-VL configs: which calls each
binding kind accepts, that every bind and a row change switch a prefill write-through off, that a bind selects row 0
when the new pool has no selected row, and that rebinding a pool decodes bit for bit like an engine that never saw
another pool."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 8      # prompt tokens of every prefill here (a multiple of 8: the batched prefill takes it unpadded)
CAP = 256
GS = 64


def _model(kind, seed=0):
    if kind == "qwen2":
        from test_engine_gpu import _build
        return _build("tiny", 12, (56, 56), seed=seed)[2]
    from test_qwen3_vl_gpu import _model as q3
    return q3("tiny", seed=seed)[2]


def _dims(eng):
    c = eng.cfg
    return c.n_layers, c.n_kv_heads, c.head_dim


def _bf16(eng, rows=1, cap=CAP):
    from mlx_vlm_b200.models.cache import KVPool
    with torch.cuda.stream(eng.stream):
        return KVPool(*_dims(eng), eng.device, batch=rows, capacity=cap, stream=eng.stream)


def _q8(eng, rows=1, cap=CAP):
    from mlx_vlm_b200.models.cache import QuantizedKVPool
    return QuantizedKVPool(*_dims(eng), eng.device, group_size=GS, batch=rows, capacity=cap, stream=eng.stream)


def _batch_q8(eng, rows=1, cap=CAP, tail=False):
    """the lock-step 8-bit batch pool; tail: layer 0 only 8-bit, the others in a bf16 pool (the tiny configs have two
    layers, where the batch rule quantizes every layer)"""
    from mlx_vlm_b200.models.cache import BatchKVQPool, KVPool, QuantizedKVPool
    L, nkv, hd = _dims(eng)
    p = BatchKVQPool(L, nkv, hd, eng.device, group_size=GS, batch=rows, capacity=cap, stream=eng.stream)
    if tail:
        p.n_q = 1
        p.q = QuantizedKVPool(1, nkv, hd, eng.device, group_size=GS, batch=rows, capacity=cap, stream=eng.stream)
        with torch.cuda.stream(eng.stream):
            p.bf = KVPool(L - 1, nkv, hd, eng.device, batch=rows, capacity=cap, stream=eng.stream)
    return p


def _prompt(eng, seed=0):
    g = torch.Generator().manual_seed(seed)
    emb = (torch.randn(T, eng.cfg.hidden, generator=g) * 0.5).to(torch.bfloat16).to(eng.device)
    pos3 = torch.arange(T, dtype=torch.int32).repeat(3, 1).contiguous().to(eng.device)
    return emb, pos3


def _accepts(fn):
    from mlx_vlm_b200._native import B200Error
    try:
        fn()
    except B200Error:
        return False
    return True


# binding kind -> (prefill, prefill_batch, decode, batch_begin) accepted; the rules of the parent commit
MATRIX = {
    "bf16 batch 1": (True, True, True, True),
    "bf16 batch 4": (True, True, True, True),
    "8-bit single request": (False, False, True, False),
    "8-bit batch": (False, False, False, True),
    "8-bit batch + bf16 tail": (False, False, False, True),
}


def _pool_of(eng, kind):
    return {"bf16 batch 1": lambda: _bf16(eng, 1), "bf16 batch 4": lambda: _bf16(eng, 4),
            "8-bit single request": lambda: _q8(eng, 1), "8-bit batch": lambda: _batch_q8(eng, 4),
            "8-bit batch + bf16 tail": lambda: _batch_q8(eng, 4, tail=True)}[kind]()


@pytest.mark.parametrize("model_kind", ["qwen2", "qwen3"])
def test_kind_call_matrix(model_kind):
    model = _model(model_kind)
    eng = model.engine
    emb, pos3 = _prompt(eng)
    for kind, want in MATRIX.items():
        pool = _pool_of(eng, kind)
        eng.bind_pool(pool)
        eng.set_kv_row(0)
        eng.set_next(1, 0, 0)
        rows = pool.batch
        got = (_accepts(lambda: eng.prefill(emb, pos3, 0, 0)),
               _accepts(lambda: eng.prefill_batch(emb, pos3, [T], [0])),
               _accepts(lambda: eng.decode(1)),
               _accepts(lambda: eng.batch_begin(np.ones(rows), np.zeros(rows), np.zeros(rows), np.ones(rows))))
        eng.stream.synchronize()
        assert got == want, f"{model_kind} {kind}: (prefill, prefill_batch, decode, batch_begin) {got}, want {want}"
    assert eng.device_error() == 0


def _planes(q):
    return [t.clone() for t in (q.codes, q.scales, q.biases)]


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("model_kind", ["qwen2", "qwen3"])
def test_every_bind_and_a_row_change_switch_the_write_through_off(model_kind):
    model = _model(model_kind)
    eng = model.engine
    emb, pos3 = _prompt(eng)
    pool = _bf16(eng, 2)

    def run(between):
        """write-through into an 8-bit pool, `between`, then a prefill on `pool`: did the 8-bit pool change?"""
        q = _q8(eng, 2)
        eng.bind_pool(pool)
        eng.set_kv_row(0)
        eng.set_prefill_kvq(q, 0)
        between()
        before = _planes(q)
        eng.prefill(emb, pos3, 0, 0)
        eng.stream.synchronize()
        changed = not _same(before, _planes(q))
        eng.set_prefill_kvq(None)
        return changed

    assert run(lambda: None), "the write-through writes the 8-bit pool"
    rebinds = {
        "bind_kv (the same pool)": lambda: eng.bind_pool(pool),
        "bind_kv (another pool)": lambda: (eng.bind_pool(_bf16(eng, 2)), eng.bind_pool(pool)),
        "bind_kvq": lambda: (eng.bind_pool(_q8(eng, 2)), eng.bind_pool(pool)),
        "bind_batch_kvq": lambda: (eng.bind_pool(_batch_q8(eng, 2)), eng.bind_pool(pool)),
        "set_kv_row to another row": lambda: eng.set_kv_row(1),
    }
    for name, between in rebinds.items():
        assert not run(between), f"{model_kind}: the write-through survives {name}"
    # the bound-pool form of the C ABI (b200_engine_set_prefill_kvq): its target row is the row selected when it is
    # set, and selecting another row switches it off as well
    from mlx_vlm_b200 import _native as N
    q = _q8(eng, 2)
    eng.bind_pool(pool)
    eng.set_kv_row(0)
    N.check(eng.lib.b200_engine_set_prefill_kvq(eng.h, q.codes.data_ptr(), q.scales.data_ptr(), q.biases.data_ptr(),
                                                GS), "set_prefill_kvq")
    eng.set_kv_row(1)
    before = _planes(q)
    eng.prefill(emb, pos3, 0, 0)
    eng.stream.synchronize()
    assert _same(before, _planes(q)), f"{model_kind}: b200_engine_set_prefill_kvq survives a row change"
    assert eng.device_error() == 0


def _written_rows(pool):
    """rows of a bf16 pool holding any non-zero value"""
    buf = pool.buf.float()
    return [r for r in range(pool.batch) if bool(buf[:, :, r].abs().sum() > 0)]


@pytest.mark.parametrize("model_kind", ["qwen2", "qwen3"])
def test_a_bind_without_the_selected_row_selects_row_0(model_kind):
    model = _model(model_kind)
    eng = model.engine
    emb, pos3 = _prompt(eng)
    for kind in ("bf16", "8-bit single request", "8-bit batch"):
        four = _bf16(eng, 4)
        eng.bind_pool(four)
        eng.set_kv_row(3)
        one = {"bf16": lambda: _bf16(eng, 1), "8-bit single request": lambda: _q8(eng, 1),
               "8-bit batch": lambda: _batch_q8(eng, 1)}[kind]()
        eng.bind_pool(one)   # accepted: the selected row 3 does not exist in a 1-row pool
        if kind == "bf16":   # a prefill writes row 0 of the new pool
            eng.prefill(emb, pos3, 0, 0)
            eng.stream.synchronize()
            assert _written_rows(one) == [0], f"{model_kind} {kind}"
        probe = _bf16(eng, 4)   # row 0 stays selected across a bind of a pool that has it
        eng.bind_pool(probe)
        eng.prefill(emb, pos3, 0, 0)
        eng.stream.synchronize()
        assert _written_rows(probe) == [0], f"{model_kind} {kind}: rows written {_written_rows(probe)}"
    assert eng.device_error() == 0


def _greedy(eng, pool_a, pool_b=None, n=6):
    """prefill + n greedy steps on pool_a; with pool_b, bind it and pool_a again half way"""
    emb, pos3 = _prompt(eng, seed=1)
    eng.bind_pool(pool_a)
    eng.set_kv_row(0)
    start = eng.tokens_launched
    eng.prefill(emb, pos3, 0, 0)
    eng.decode(n // 2)
    if pool_b is not None:
        eng.bind_pool(pool_b)
        eng.bind_pool(pool_a)
    eng.decode(n - n // 2)
    lp = eng.snapshot("logprobs")
    host = torch.empty(n + 1, dtype=torch.int32).pin_memory()
    eng.fetch_tokens(start, n + 1, host)
    eng.stream.synchronize()
    assert eng.device_error() == 0
    return host.tolist(), lp.cpu()


@pytest.mark.parametrize("model_kind", ["qwen2", "qwen3"])
@pytest.mark.parametrize("kv8", [False, True])
def test_rebinding_a_pool_decodes_like_a_fresh_engine(model_kind, kv8):
    """greedy decode on pool A, bind pool B (another capacity) and A again, decode on: the decode graph of A is
    dropped and re-captured, and tokens and logprobs equal those of a fresh engine that only saw A, bit for bit.
    kv8: A and B are 8-bit pools (decode on A8; the prefill runs on a bf16 pool that writes A8 through)"""
    models = [_model(model_kind) for _ in range(3)]   # warm-up, fresh, rebound: the same seeded weights
    warm, fresh, used = (m.engine for m in models)

    def run(eng, rebind):
        if not kv8:
            return _greedy(eng, _bf16(eng), _bf16(eng, cap=2 * CAP) if rebind else None)
        a8, pre = _q8(eng), _bf16(eng)
        emb, pos3 = _prompt(eng, seed=1)
        eng.bind_pool(pre)
        eng.set_kv_row(0)
        eng.set_prefill_kvq(a8, 0)
        start = eng.tokens_launched
        eng.prefill(emb, pos3, 0, 0)
        eng.set_prefill_kvq(None)
        eng.bind_pool(a8)
        eng.decode(3)
        if rebind:
            eng.bind_pool(_q8(eng, cap=2 * CAP))
            eng.bind_pool(a8)
        eng.decode(3)
        lp = eng.snapshot("logprobs")
        host = torch.empty(7, dtype=torch.int32).pin_memory()
        eng.fetch_tokens(start, 7, host)
        eng.stream.synchronize()
        assert eng.device_error() == 0
        return host.tolist(), lp.cpu()

    run(warm, False)   # the GEMM configurations are tuned once per process: both engines below run the tuned ones
    want_tok, want_lp = run(fresh, False)
    got_tok, got_lp = run(used, True)
    assert got_tok == want_tok
    assert torch.equal(got_lp, want_lp)
