"""8-bit KV cache (kv_bits=8) without a GPU: the reference arithmetic, the argument checks, the single-request
conversion policy and the QuantizedKVCache surface on CPU tensors."""
import numpy as np
import pytest
import torch

import kvq_ref as K


@pytest.mark.parametrize("gs", [32, 64, 128])
def test_reference_quantize_properties(gs):
    w = K.special_groups(gs, 21)
    codes, scales, biases = K.quantize(w, gs)
    assert codes.dtype == np.uint8 and scales.shape == (21, 1) and biases.shape == (21, 1)
    deq = K.dequantize(codes, scales, biases, gs)
    span = (w.max(1) - w.min(1))[:, None]
    # every element is reconstructed to within one quantization step (plus the bf16 rounding of the result)
    assert np.all(np.abs(deq - w) <= span / 255 * 1.01 + np.abs(w) * 2.0 ** -7 + 1e-6)
    assert np.all(deq[2::7] == 0)                        # all-zero groups stay zero
    const = w[1::7]
    assert np.all(K.dequantize(*K.quantize(const, gs), gs) == const)
    tie = w[6::7]
    c, s, b = K.quantize(tie, gs)
    assert np.all(s == 1 / 64) and np.all(b == -255 / 64)
    # (w - bias) / scale = 254.5, 253.5, ...: round half to even
    x = (tie - b) / s
    half = np.abs(x - np.floor(x) - 0.5) < 1e-6
    assert half.any()
    assert np.all(c[half] == np.rint(x[half]))


def test_packed_word_layout():
    """codes viewed as uint32: element 4i+j sits in bits 8j of word i (mx.quantize with bits=8)"""
    codes = torch.arange(16, dtype=torch.uint8).reshape(1, 1, 1, 16)
    words = codes.view(torch.uint32)
    assert words.shape == (1, 1, 1, 4)
    w0 = int(words[0, 0, 0, 1].item())
    assert [(w0 >> (8 * j)) & 0xFF for j in range(4)] == [4, 5, 6, 7]


def test_kv_quant_args():
    from mlx_vlm_b200.generate import kv_quant_args
    assert kv_quant_args(None, 64, None, 128) is None
    assert kv_quant_args(8, 64, None, 128) == 8
    assert kv_quant_args(8.0, 32, "uniform", 64) == 8
    for bits in (4, 4.5, 2, 6):
        with pytest.raises(NotImplementedError):
            kv_quant_args(bits, 64, None, 128)
    with pytest.raises(NotImplementedError):
        kv_quant_args(8, 64, "turboquant", 128)
    for gs in (16, 48, 256):
        with pytest.raises(ValueError):
            kv_quant_args(8, gs, None, 128)
    with pytest.raises(ValueError):
        kv_quant_args(8, 128, None, 64)


class _FakeLayer:
    def __init__(self):
        self.offset = 0
        self._pool = None

    def to_quantized(self, group_size, bits):
        q = _FakeQ()
        q.offset, q.group_size, q.bits = self.offset, group_size, bits
        return q


class _FakeQ:
    pass


@pytest.mark.parametrize("delta", [None, -1, 0, 5])
def test_single_request_switch_point(delta):
    """generate/common.py:174-183 after every forward: all layers convert at the first forward whose resulting
    offset reaches quantized_kv_start; the prefill (T tokens) always runs in bf16."""
    from mlx_vlm_b200.generate import maybe_quantize_kv_cache
    T = 9
    start = 0 if delta is None else T + delta
    cache = [_FakeLayer() for _ in range(3)]
    switched_at = None
    for fwd in range(12):           # prefill, then one decode step per forward
        L = T if fwd == 0 else 1
        for c in cache:
            c.offset += L
        before = isinstance(cache[0], _FakeQ)
        maybe_quantize_kv_cache(cache, start, 64, 8)
        if not before and isinstance(cache[0], _FakeQ):
            switched_at = cache[0].offset
        assert all(isinstance(c, _FakeQ) for c in cache) == isinstance(cache[0], _FakeQ)
    assert switched_at == max(T, start)
    assert all(c.bits == 8 and c.group_size == 64 for c in cache)
    maybe_quantize_kv_cache(cache, start, 64, None)   # kv_bits=None: nothing happens


def test_quantized_cache_surface_cpu():
    from mlx_vlm_b200.models.cache import QuantizedKVCache, QuantizedKVPool
    pool = QuantizedKVPool(3, 2, 128, "cpu", group_size=64, capacity=10)
    assert pool.capacity == 256
    c = QuantizedKVCache(group_size=64, bits=8, pool=pool, layer=1)
    c.offset = 7
    k, v = c.keys, c.values
    assert k[0].dtype == torch.uint32 and k[0].shape == (1, 2, 256, 32)
    assert k[1].shape == (1, 2, 256, 2) and k[1].dtype == torch.bfloat16 and v[2].shape == (1, 2, 256, 2)
    sk, sv = c.state
    assert sk[0].shape == (1, 2, 7, 32)
    assert c.meta_state == ("7", "64", "8")
    assert c.trim(3) == 3 and c.offset == 4 and c.size() == 4 and c.is_trimmable()
    assert c.make_mask(1) is None and c.make_mask(5) == "causal"
    bf16_layer_bytes = 2 * 2 * 256 * 128 * 2
    assert c.nbytes == 2 * 2 * 256 * (128 + 2 * 2 * 2)
    assert c.nbytes / bf16_layer_bytes == 0.53125
    assert pool.bytes_per_position() * 256 == 3 * c.nbytes
    with pytest.raises(NotImplementedError):
        QuantizedKVCache(group_size=64, bits=4)


def test_to_quantized_rejects_other_widths():
    from mlx_vlm_b200.models.cache import KVCache
    c = KVCache()
    c.update_and_fetch(torch.zeros(1, 2, 3, 64), torch.zeros(1, 2, 3, 64))
    with pytest.raises(NotImplementedError):
        c.to_quantized()                    # the reference's default bits=4
    with pytest.raises(ValueError):
        c.to_quantized(group_size=48, bits=8)
