"""Reference arithmetic of the 8-bit KV cache for the tests (the product never imports this).

`quantize` / `dequantize` restate mx.quantize / mx.dequantize with bits=8 (affine mode, MLX's CPU quantize
routine as remembered, not checked against a running mlx: unpinned at the mlx boundary), in numpy fp32:

  per group of gs consecutive elements: w_max, w_min; mask = |w_min| > |w_max|
  scale = max((w_max - w_min) / 255, 1e-7), negated unless mask
  edge = mask ? w_min : w_max; q0 = rint(edge / scale)
  q0 != 0: scale = edge / q0, bias = edge; otherwise bias = 0
  code = clamp(rint((w - bias) / scale), 0, 255); scale, bias rounded to bf16 only when stored

Dequantized element: bf16(fp32(scale * code + bias)) with the stored scale and bias; scale * code is exact in
fp32, so that is the fp32 rounding of the sum followed by the bf16 rounding.  This rounding is the project's
choice, also unpinned: MLX dequantizes in the storage dtype and may round scale * code to bf16 first.  Quantized
attention (quantized_scaled_dot_product_attention) is taken as `sdpa` over the dequantized K / V with sdpa's
rounding points; MLX's quantized_matmul folds scale and bias into the dot product instead.  How far either MLX
form lies from this one is not measured.

`greedy_generate_kvq` is oracle.qwen2vl.greedy_generate with the single-request policy of
generate/common.py:174-183 (every layer converts once its offset reaches quantized_kv_start, after a forward)
and QuantizedKVCache.update_and_fetch (a converted layer quantizes new rows before they are attended).
"""
import numpy as np
import torch


def _bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def quantize(w, gs):
    """w (..., hd) fp32 -> codes uint8 (..., hd), scales / biases fp32 of the bf16 values (..., hd / gs)"""
    w = np.asarray(w, dtype=np.float32)
    hd = w.shape[-1]
    g = w.reshape(-1, gs)
    w_max, w_min = g.max(axis=1), g.min(axis=1)
    mask = np.abs(w_min) > np.abs(w_max)
    scale = np.maximum((w_max - w_min) / np.float32(255), np.float32(1e-7)).astype(np.float32)
    scale = np.where(mask, scale, -scale).astype(np.float32)
    edge = np.where(mask, w_min, w_max).astype(np.float32)
    q0 = np.rint(edge / scale).astype(np.float32)
    nz = q0 != 0
    scale = np.where(nz, edge / np.where(nz, q0, np.float32(1)), scale).astype(np.float32)
    bias = np.where(nz, edge, np.float32(0)).astype(np.float32)
    codes = np.clip(np.rint((g - bias[:, None]) / scale[:, None]), 0, 255).astype(np.uint8)
    lead = w.shape[:-1]
    return (codes.reshape(w.shape), _bf16(scale).reshape(lead + (hd // gs,)),
            _bf16(bias).reshape(lead + (hd // gs,)))


def dequantize(codes, scales, biases, gs):
    c = np.asarray(codes).astype(np.float32)
    s = np.repeat(np.asarray(scales, dtype=np.float32), gs, axis=-1)
    b = np.repeat(np.asarray(biases, dtype=np.float32), gs, axis=-1)
    return _bf16((s * c + b).astype(np.float32))


def qdq(x: torch.Tensor, gs: int) -> torch.Tensor:
    """the dequantized form of an fp32 tensor (..., hd)"""
    return torch.from_numpy(dequantize(*quantize(x.numpy(), gs), gs))


def special_groups(gs: int, n: int, seed: int = 0) -> np.ndarray:
    """(n, gs) fp32 groups of bf16 values: random, constant, all-zero, negative- and positive-dominant,
    one-outlier and groups whose (w - bias) / scale lands on .5 ties"""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        kind = i % 7
        if kind == 0:
            g = rng.standard_normal(gs) * 0.7
        elif kind == 1:
            g = np.full(gs, rng.choice([0.75, -3.5, 1e-3]))
        elif kind == 2:
            g = np.zeros(gs)
        elif kind == 3:
            g = rng.standard_normal(gs) * 0.1
            g[rng.integers(gs)] = -6.0
        elif kind == 4:
            g = rng.standard_normal(gs) * 0.1
            g[rng.integers(gs)] = 6.0
        elif kind == 5:
            g = np.zeros(gs)
            g[rng.integers(gs)] = rng.choice([40.0, -40.0])
        else:
            # w_min = -255/64 -> scale 1/64, bias w_min: w = -(2k+1)/128 gives codes 254.5, 253.5, ...
            g = -(2 * rng.integers(0, 8, size=gs) + 1) / 128.0
            g[0] = -255.0 / 64.0
            g[1] = 0.0
        rows.append(g)
    return _bf16(np.stack(rows))


class QuantOracleCache:
    """OracleKVCache whose layer converts to 8 bits at the policy point: from then on its stored rows and every
    appended row are kept in dequantized form (what quantized attention reads)."""

    def __init__(self, gs: int):
        from oracle.qwen2vl import OracleKVCache
        self.c = OracleKVCache()
        self.gs = gs
        self.quantized = False

    @property
    def offset(self):
        return self.c.offset

    @property
    def keys(self):
        return self.c.keys

    @property
    def values(self):
        return self.c.values

    def convert(self):
        n = self.c.offset
        self.c.keys[..., :n, :] = qdq(self.c.keys[..., :n, :].contiguous(), self.gs)
        self.c.values[..., :n, :] = qdq(self.c.values[..., :n, :].contiguous(), self.gs)
        self.quantized = True

    def update_and_fetch(self, k, v):
        if self.quantized:
            k, v = qdq(k.contiguous(), self.gs), qdq(v.contiguous(), self.gs)
        return self.c.update_and_fetch(k, v)


def greedy_generate_kvq(cfg, W, input_ids, pixel_values, grid_thw, max_tokens, gs, quantized_kv_start,
                        dtype="bf16", force_tokens=None, prefill_step_size=None):
    """oracle.qwen2vl.greedy_generate with kv_bits=8 (single-request policy); returns the same dict plus
    `switch_offset` (the cache offset at which the layers converted, None if they never did).  With
    prefill_step_size < T the prompt is prefilled in chunks as generate_step does (ar.py:426-472): chunks of
    min(step, left - 1) tokens while more than one token is left, then the last token, the policy after each."""
    from oracle import mlx_semantics as S
    from oracle import qwen2vl as O
    R = S.Rounder(dtype)
    ids = np.asarray(input_ids, dtype=np.int64)
    B, T = ids.shape
    embeds, feats, pos, deltas = O.get_input_embeddings(cfg, W, ids, pixel_values, grid_thw, R)
    cache = [QuantOracleCache(gs) for _ in range(cfg.text.num_hidden_layers)]
    switch = []

    def policy():
        for c in cache:
            if not c.quantized and c.offset >= quantized_kv_start:
                c.convert()
                if not switch:
                    switch.append(c.offset)

    a = 0
    if prefill_step_size is not None and T > prefill_step_size:
        while T - a > 1:
            n = min(prefill_step_size, T - a - 1)
            O.lm_layers_forward(cfg, W, embeds[:, a:a + n], pos[:, :, a:a + n], cache, R)
            policy()
            a += n
    hidden = O.lm_layers_forward(cfg, W, embeds[:, a:], pos[:, :, a:], cache, R)
    policy()
    logits = O.lm_head(cfg, W, hidden[:, -1, :], R)
    toks, all_logits, all_lp = [], [], []
    for n in range(max_tokens):
        lp = O.logprobs_from_logits(R, logits)
        y = S.argmax_lowest(lp)
        toks.append(y.clone())
        all_logits.append(logits.clone())
        all_lp.append(lp)
        if n == max_tokens - 1:
            break
        feed = y if force_tokens is None else torch.full_like(y, int(force_tokens[n]))
        e = W["language_model.model.embed_tokens.weight"][feed][:, None, :]
        p = O.decode_position_ids(cache[0].offset, deltas, B)
        hidden = O.lm_layers_forward(cfg, W, e, p, cache, R)
        policy()
        logits = O.lm_head(cfg, W, hidden[:, -1, :], R)
    return dict(tokens=torch.stack(toks, 1), logits=all_logits, logprobs=all_lp, cache=cache,
                switch_offset=switch[0] if switch else None)
