"""kv_bits=8 in the lock-step batch, host side: the reference's layer rule (models/cache.py:8-21
`should_quantize_kv_layer`), the arguments BatchGenerator accepts and refuses, and the layout and byte count of the
mixed-format batch pool (8-bit layers, bf16 last layer); the layer rule and the batch cache's update / extract /
filter / extend bookkeeping against tests/golden/kvq_batch_golden.json (the reference's own source, executed)."""
import json
import os

import numpy as np
import pytest
import torch

from test_batch_host import _fake_model


@pytest.mark.parametrize("n,want", [(1, [True]), (2, [True, True]), (3, [True, True, False]),
                                    (28, [True] * 27 + [False])])
def test_layer_rule(n, want):
    from mlx_vlm_b200.models.cache import BatchKVQPool, should_quantize_kv_layer
    assert [should_quantize_kv_layer(i, n) for i in range(n)] == want
    pool = BatchKVQPool(n, 2, 64, torch.device("cpu"), group_size=64, batch=2, capacity=256)
    assert pool.n_q == sum(want) and (pool.bf is None) == all(want)
    assert pool.q.n_layers == pool.n_q and (pool.bf is None or pool.bf.n_layers == n - pool.n_q)


def _lockstep_model(head_dim=128):
    model, proc = _fake_model(lockstep=True)
    model.language_model.head_dim = head_dim
    return model, proc


def test_batch_generator_kv_arguments():
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model, proc = _lockstep_model()
    for bits in (8, 8.0):
        for gs in (32, 64, 128):
            for scheme in (None, "uniform"):
                g = BatchGenerator(model, proc, kv_bits=bits, kv_group_size=gs, kv_quant_scheme=scheme,
                                   quantized_kv_start=1000)
                assert g.kv_bits == 8 and g.kv_group_size == gs
    assert BatchGenerator(model, proc).kv_bits is None
    for kw in ({"kv_bits": 4}, {"kv_bits": 8.5}, {"kv_bits": 6}, {"kv_bits": 8, "kv_quant_scheme": "turboquant"},
               {"kv_bits": 8, "kv_key_bits": 8}, {"kv_bits": 8, "kv_value_bits": 8}, {"kv_key_bits": 4}):
        with pytest.raises(NotImplementedError):
            BatchGenerator(model, proc, **kw)
    for gs in (16, 48, 256):
        with pytest.raises(ValueError):
            BatchGenerator(model, proc, kv_bits=8, kv_group_size=gs)
    with pytest.raises(ValueError):   # the group size must divide head_dim
        BatchGenerator(*_lockstep_model(head_dim=64), kv_bits=8, kv_group_size=128)


def test_time_multiplexed_rows_refuse_kv_bits():
    """no batched decoder (or a Qwen3-VL geometry that runs time-multiplexed): the single-request path would apply a
    different 8-bit policy, so the option is refused with the reason"""
    from mlx_vlm_b200.generate_batch import BatchGenerator
    model, proc = _fake_model()
    model.language_model.head_dim = 128
    with pytest.raises(NotImplementedError, match="lock-step"):
        BatchGenerator(model, proc, kv_bits=8)
    model, proc = _lockstep_model()
    with pytest.raises(NotImplementedError, match="lock-step"):
        BatchGenerator(model, proc, kv_bits=8, time_multiplex=True)


@pytest.mark.parametrize("gs", [32, 64, 128])
def test_batch_cache_surface_and_nbytes(gs):
    from mlx_vlm_b200.models.cache import (BatchKVQPool, BatchQuantizedKVCache, BatchRows, KVPool,
                                           RowBatchKVCache)
    L, nkv, hd, rows, cap = 3, 2, 128, 4, 256
    pool = BatchKVQPool(L, nkv, hd, torch.device("cpu"), group_size=gs, batch=rows, capacity=cap)
    r = BatchRows(pool, None, lengths=[5, 9, 3])
    caches = r.layer_caches()
    assert [type(c) for c in caches] == [BatchQuantizedKVCache, BatchQuantizedKVCache, RowBatchKVCache]
    k = caches[0].keys
    assert k[0].dtype == torch.uint32 and tuple(k[0].shape) == (3, nkv, cap, hd // 4)
    assert tuple(k[1].shape) == (3, nkv, cap, hd // gs) and k[1].dtype == torch.bfloat16
    assert list(caches[0].offset) == [5, 9, 3] and not np.any(caches[0].left_padding)
    assert caches[0].size() == 9 and caches[0].bits == 8 and caches[0].group_size == gs
    # 8-bit layers: codes + bf16 scales / biases; the last layer: bf16
    q_bytes = 2 * 3 * nkv * cap * (hd + 4 * (hd // gs))
    assert caches[0].nbytes == caches[1].nbytes == q_bytes
    assert caches[2].nbytes == 2 * 3 * nkv * cap * hd * 2
    if gs == 64:
        assert caches[0].nbytes / caches[2].nbytes == 0.53125
    bf16 = KVPool(L, nkv, hd, torch.device("cpu"), batch=rows, capacity=cap)
    assert pool.bytes_per_position() == 2 * nkv * (2 * (hd + 4 * (hd // gs)) + 2 * hd)
    assert bf16.buf.numel() * 2 / (rows * cap) == L * 2 * nkv * hd * 2
    # growth keeps the two parts at one capacity
    pool.reserve(300, live_tokens=9)
    assert pool.capacity == pool.bf.capacity == 512


# ----------------------------------------------------------------- against the reference's own source
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kvq_batch_golden.json")


class _HostRowCopies:
    """the engine's row copies (b200_pool_copy_row / b200_kv_copy_row) restated with torch on host pools: this test
    checks which rows the cache operations move where; the device copies are checked byte for byte on the GPU"""
    stream = None

    def kvq_copy_row(self, dst, dst_row, src, src_row, n):
        for name in ("codes", "scales", "biases"):
            getattr(dst, name)[:, :, dst_row, :, :n].copy_(getattr(src, name)[:, :, src_row, :, :n].clone())

    def kv_copy_row(self, dst, dst_row, src, src_row, n):
        self.kvq_copy_row(dst.q, dst_row, src.q, src_row, n)
        if dst.bf is not None:
            dst.bf.buf[:, :, dst_row, :, :n].copy_(src.bf.buf[:, :, src_row, :, :n].clone())


def _write_rows(pool, keys, values, gs, start=0):
    """quantize (B, n_kv, n, hd) rows with the reference arithmetic into layer 0 of the 8-bit pool at `start`,
    as the kernels append them"""
    from kvq_ref import quantize
    for side, x in ((0, keys), (1, values)):
        x = np.asarray(x, dtype=np.float32)
        c, s, b = quantize(x, gs)
        n = x.shape[2]
        B = x.shape[0]
        pool.q.codes[0, side, :B, :, start:start + n] = torch.from_numpy(c)
        pool.q.scales[0, side, :B, :, start:start + n] = torch.from_numpy(s).to(torch.bfloat16)
        pool.q.biases[0, side, :B, :, start:start + n] = torch.from_numpy(b).to(torch.bfloat16)


def _same(cache, snap, name):
    n = snap["idx"]
    assert list(cache.offset) == snap["offset"], name
    assert list(cache.left_padding) == snap["left_padding"], name
    for got, want in ((cache.keys, snap["keys"]), (cache.values, snap["values"])):
        w = [np.asarray(x) for x in want]
        assert np.array_equal(got[0][..., :n, :].numpy().astype(np.int64), w[0].astype(np.int64)), name
        assert np.array_equal(got[1][..., :n, :].float().numpy(), w[1].astype(np.float32)), name
        assert np.array_equal(got[2][..., :n, :].float().numpy(), w[2].astype(np.float32)), name
        assert [list(got[0].shape[:2]), got[0].shape[-1], got[1].shape[-1]] == [
            snap["shapes"][0][:2], snap["shapes"][0][-1], snap["shapes"][1][-1]], name


def test_layer_rule_against_reference_golden():
    from mlx_vlm_b200.models.cache import BatchKVQPool, should_quantize_kv_layer
    with open(GOLDEN) as f:
        g = json.load(f)
    for n, want in g["layer_rule"].items():
        n = int(n)
        assert [should_quantize_kv_layer(i, n) for i in range(n)] == want
        assert BatchKVQPool(n, 1, 64, torch.device("cpu"), capacity=256).n_q == sum(want)


def test_batch_cache_bookkeeping_against_reference_golden():
    """update / extract / filter / extend of the reference's BatchQuantizedKVCache (executed from its source) against
    the product's BatchQuantizedKVCache over a host pool: codes as uint32 words, scales, biases, offsets, padding"""
    from mlx_vlm_b200.models.cache import BatchKVQPool, BatchRows, QuantizedKVCache
    with open(GOLDEN) as f:
        g = json.load(f)
    gs, hd, nkv = g["group_size"], g["head_dim"], g["n_kv"]
    inp, tr = g["inputs"], g["trace"]
    eng = _HostRowCopies()
    pool = BatchKVQPool(2, nkv, hd, torch.device("cpu"), group_size=gs, batch=3, capacity=256)
    rows = BatchRows(pool, eng, lengths=[0, 0, 0])
    caches = rows.layer_caches()
    _write_rows(pool, inp["prefill"]["keys"], inp["prefill"]["values"], gs)
    rows.lengths = [5, 5, 5]
    _same(caches[0], tr[0], tr[0]["op"])
    _write_rows(pool, inp["decode"]["keys"], inp["decode"]["values"], gs, start=5)
    rows.lengths = [6, 6, 6]
    _same(caches[0], tr[1], tr[1]["op"])
    ex = caches[0].extract(1)
    want = tr[2]
    assert isinstance(ex, QuantizedKVCache) and ex.offset == want["offset"]
    assert (ex.group_size, ex.bits) == (want["group_size"], want["bits"])
    for got, w in ((ex.keys, want["keys"]), (ex.values, want["values"])):
        n = ex.offset
        assert np.array_equal(got[0][..., :n, :].numpy().astype(np.int64), np.asarray(w[0]).astype(np.int64))
        assert np.array_equal(got[1][..., :n, :].float().numpy(), np.asarray(w[1], dtype=np.float32))
        assert np.array_equal(got[2][..., :n, :].float().numpy(), np.asarray(w[2], dtype=np.float32))
    for c in caches:
        c.filter(np.array([0, 2]))
    _same(caches[0], tr[3], tr[3]["op"])
    opool = BatchKVQPool(2, nkv, hd, torch.device("cpu"), group_size=gs, batch=1, capacity=256)
    orows = BatchRows(opool, eng, lengths=[0])
    _write_rows(opool, inp["other"]["keys"], inp["other"]["values"], gs)
    orows.lengths = [6]
    for c, o in zip(caches, orows.layer_caches()):
        c.extend(o)
    _same(caches[0], tr[4], tr[4]["op"])


def test_extract_sweeps_are_fresh_and_follow_the_length():
    """every extract sweep copies the row as it is now (decode steps grow a row without a structural change) into
    its own pool; the layers of one sweep share that pool"""
    from mlx_vlm_b200.models.cache import BatchKVQPool, BatchRows
    pool = BatchKVQPool(2, 2, 64, torch.device("cpu"), group_size=64, batch=2, capacity=256)
    rows = BatchRows(pool, _HostRowCopies(), lengths=[4, 3])
    caches = rows.layer_caches()
    pool.q.codes[:, :, 1, :, :3] = 11
    a = [c.extract(1) for c in caches]
    assert a[0]._pool is a[1]._pool and a[0].offset == 3
    pool.q.codes[:, :, 1, :, 3:5] = 22        # two lock-step steps append to row 1
    rows.lengths = [6, 5]
    b = [c.extract(1) for c in caches]
    assert b[0]._pool is b[1]._pool and b[0]._pool is not a[0]._pool and b[0].offset == 5
    assert torch.equal(b[0]._pool.codes[:, :, 0, :, :5], pool.q.codes[:, :, 1, :, :5])
    c2 = [c.extract(1) for c in caches]       # same state again: still a pool of its own
    assert c2[0]._pool is not b[0]._pool and torch.equal(c2[0]._pool.codes, b[0]._pool.codes)
