"""Qwen2-VL language model — Python face of the reference's
mlx_vlm/models/qwen2_vl/language.py (`LanguageModel` :203-530).

Host-side integer logic (M-RoPE position ids, decode position bookkeeping) is
restated here in numpy and is bit-exact with the reference (tests pin it on the
reference's known-answer vectors).  The transformer arithmetic runs in
libb200vlm.so: `b200_engine_prefill` for L > 1, the captured decode-step graph
(`b200_engine_decode`) for L == 1.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from ..base import LanguageModelOutput
from ..cache import (BatchKVQPool, BatchQuantizedKVCache, BatchRows, KVCache, KVPool, QuantizedKVCache,
                     QuantizedKVPool, RowBatchKVCache)
from .config import ModelConfig, TextConfig


def _np(x, dtype=np.int64):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy().astype(dtype)
    return np.asarray(x, dtype=dtype)


class LanguageModel:
    # generate_step passes logits_to_keep=1 when this is set (ar.py:341-342), so the
    # head runs on the last prompt row only; all rows are still available on request.
    supports_logits_to_keep = True

    def __init__(self, args: TextConfig, config: ModelConfig, engine_getter):
        self.args = args
        self.config = config
        self.model_type = args.model_type
        self._rope_deltas = None
        self._position_ids = None
        self._engine = engine_getter
        self._pool: Optional[KVPool] = None

    # ------------------------------------------------------------------ rope
    def get_rope_index(self, input_ids, image_grid_thw=None, video_grid_thw=None,
                       attention_mask=None):
        """language.py:216-402.  Returns numpy int64 (position_ids, rope_deltas):
        (3,B,T),(B,1) with vision grids, else the 2-D text branch."""
        cfg = self.config
        ids = _np(input_ids)
        B, T = ids.shape
        ms = cfg.vision_config.spatial_merge_size
        img_id, vid_id = cfg.image_token_id, cfg.video_token_id
        vs_id = cfg.vision_start_token_id
        igrid, vgrid = _np(image_grid_thw), _np(video_grid_thw)
        amask = _np(attention_mask)
        if igrid is not None or vgrid is not None:
            if amask is None:
                amask = np.ones_like(ids)
            pos = np.ones((3, B, T), dtype=np.int64)
            deltas: List[int] = []
            ii = vi = 0
            for i in range(B):
                row_mask = amask[i].tolist()
                toks = [t for t, keep in zip(ids[i].tolist(), row_mask) if keep == 1]
                follow = [toks[j + 1] for j, t in enumerate(toks[:-1]) if t == vs_id]
                n_img = sum(t == img_id for t in follow)
                n_vid = sum(t == vid_id for t in follow)
                parts: List[np.ndarray] = []
                st = 0
                left_i, left_v = n_img, n_vid
                for _ in range(n_img + n_vid):
                    e_img = toks.index(img_id, st) if (img_id in toks and left_i > 0) else len(toks) + 1
                    e_vid = toks.index(vid_id, st) if (vid_id in toks and left_v > 0) else len(toks) + 1
                    if e_img < e_vid:
                        t, h, w = (int(v) for v in igrid[ii])
                        ii += 1
                        left_i -= 1
                        ed = e_img
                    else:
                        t, h, w = (int(v) for v in vgrid[vi])
                        vi += 1
                        left_v -= 1
                        ed = e_vid
                    gt, gh, gw = t, h // ms, w // ms
                    n_text = ed - st
                    base = int(parts[-1].max()) + 1 if parts else 0
                    parts.append(np.tile(np.arange(n_text), (3, 1)) + base)
                    grid = np.indices((gt, gh, gw)).reshape(3, -1)  # rows: t, h, w
                    parts.append(grid + n_text + base)
                    st = ed + gt * gh * gw
                if st < len(toks):
                    base = int(parts[-1].max()) + 1 if parts else 0
                    parts.append(np.tile(np.arange(len(toks) - st), (3, 1)) + base)
                if not parts:
                    deltas.append(0)
                    continue
                compact = np.concatenate(parts, axis=1).reshape(3, -1)
                keep_cols = [c for c, k in enumerate(row_mask) if k == 1]
                pos[:, i, keep_cols] = compact[:, :len(keep_cols)]
                deltas.append(int(compact.max()) + 1 - len(toks))
            return pos, np.asarray(deltas, dtype=np.int64).reshape(-1, 1)
        if amask is not None:
            pos = np.cumsum(amask, axis=-1) - 1
            pos = np.where(amask == 0, 1, pos)
            return pos, pos.max(axis=-1, keepdims=True) + 1 - amask.shape[-1]
        pos = np.tile(np.arange(T), (B, 1))
        return pos, np.zeros((B, 1), dtype=np.int64)

    # ----------------------------------------------------------------- cache
    def make_cache(self):
        """One device pool per request; per-layer KVCache views (models/cache.py)."""
        eng = self._engine()
        pool = KVPool(self.args.num_hidden_layers, self.args.num_key_value_heads, self.head_dim,
                      eng.device, batch=1, stream=eng.stream)
        self._pool = pool
        return [KVCache(pool, l) for l in range(self.args.num_hidden_layers)]

    def make_cache_row(self, pool: KVPool, row: int):
        """per-layer KVCache views of ROW `row` of a batched pool (a request admitted to a batch); on a kv_bits=8
        batch pool (BatchKVQPool) QuantizedKVCache views on its 8-bit layers"""
        if isinstance(pool, BatchKVQPool):
            return pool.row_caches(row)
        return [KVCache(pool, l, row=row) for l in range(self.args.num_hidden_layers)]

    def make_batch_cache(self, rows: int, capacity: int = 0, kv_bits=None, kv_group_size: int = 64):
        """device-resident batch cache for `rows` requests: (BatchRows, per-layer caches) — RowBatchKVCache, or with
        kv_bits=8 the reference's batch rule (BatchQuantizedKVCache where `should_quantize_kv_layer` holds)"""
        eng = self._engine()
        if kv_bits is not None:
            from ..cache import _kvq_check
            _kvq_check(kv_group_size, kv_bits, self.head_dim)
            pool = BatchKVQPool(self.args.num_hidden_layers, self.args.num_key_value_heads, self.head_dim, eng.device,
                                group_size=kv_group_size, batch=rows, capacity=max(capacity, KVPool.step),
                                stream=eng.stream)
        else:
            pool = KVPool(self.args.num_hidden_layers, self.args.num_key_value_heads, self.head_dim, eng.device,
                          batch=rows, capacity=max(capacity, KVPool.step))
        r = BatchRows(pool, eng)
        return r, r.layer_caches()

    def _bind(self, cache, need_tokens: int, decode: bool = False, chunk_end: Optional[int] = None) -> KVPool:
        c0 = cache[0]
        pool = getattr(c0, "_pool", None)
        if pool is None:
            raise ValueError("b200 LanguageModel needs caches from make_prompt_cache(language_model)")
        eng = self._engine()
        if getattr(c0, "_batch_pool", None) is not None:
            return self._bind_batch_row(cache, need_tokens, decode, chunk_end)
        if any(isinstance(c, QuantizedKVCache) for c in cache):
            return self._bind_q8(cache, need_tokens, decode)
        if pool.capacity < need_tokens:
            eng.stream.synchronize()
            with torch.cuda.stream(eng.stream):
                # a batched pool moves as a whole: keep every row's live prefix
                live = c0.offset if pool.batch == 1 else pool.capacity
                pool.reserve(need_tokens, live_tokens=live)
        eng.bind_pool(pool)
        eng.set_kv_row(c0._row or 0)
        return pool

    def _bind_q8(self, cache, need_tokens: int, decode: bool):
        """an 8-bit cache: every layer a view of ONE QuantizedKVPool.  Decode steps bind it directly.  A prefill
        call gets a bf16 pool holding the dequantized prefix and writes its own rows through to the 8-bit pool
        (quantized before they are attended); that bf16 pool lives until the next bind."""
        c0 = cache[0]
        pool = c0._pool
        if not all(isinstance(c, QuantizedKVCache) and c._pool is pool for c in cache):
            raise NotImplementedError("a cache that mixes 8-bit and bf16 layers is not built for single requests")
        eng = self._engine()
        if pool.capacity < need_tokens:
            eng.stream.synchronize()
            pool.reserve(need_tokens, live_tokens=c0.offset)
        if decode:
            eng.bind_kvq(pool)
            eng.set_kv_row(c0._row or 0)
            return pool
        prefix = pool.to_bf16_pool(int(c0.offset))
        eng.bind_pool(prefix)
        eng.set_kv_row(c0._row or 0)
        eng.set_prefill_kvq(pool)
        return prefix

    def _bind_batch_row(self, cache, need_tokens: int, decode: bool, chunk_end: Optional[int]):
        """the prefill of a row admitted to a kv_bits=8 batch pool (BatchKVQPool): the chunks run on a batch-1 bf16
        pool of this admission and write the 8-bit layers' rows through to the batch pool's row, quantized before
        they are attended (their dequantized values stay in the bf16 pool as the prefix of the next chunk); the
        bf16 layers are copied to the batch pool after each chunk (`_finish_batch_row`).  The transient pool holds
        the prompt only (`chunk_end`: the end of this chunk), grown chunk by chunk; `need_tokens` (which includes
        the tokens still to be generated) sizes the batch pool"""
        c0 = cache[0]
        bp, row, off = c0._batch_pool, c0._row, int(c0.offset)
        if decode or chunk_end is None:
            raise NotImplementedError("a row of a kv_bits=8 batch pool decodes in the lock-step batch only")
        eng = self._engine()
        adm = getattr(bp, "_admit", None)
        if off == 0 or adm is None or adm[0] != row:
            if off != 0:
                raise NotImplementedError("a prefill chunk of a kv_bits=8 batch row must continue that row's admission")
            with torch.cuda.stream(eng.stream):
                tmp = KVPool(self.args.num_hidden_layers, self.args.num_key_value_heads, self.head_dim, eng.device,
                             batch=1, capacity=chunk_end, stream=eng.stream)
            bp._admit = (row, tmp)
        else:
            tmp = adm[1]
            if tmp.capacity < chunk_end:
                eng.stream.synchronize()
                with torch.cuda.stream(eng.stream):
                    tmp.reserve(chunk_end, live_tokens=off)
        if bp.capacity < need_tokens:
            raise ValueError(f"kv_bits=8 batch pool holds {bp.capacity} positions per row, the row needs {need_tokens}")
        eng.bind_pool(tmp)
        eng.set_kv_row(0)
        eng.set_prefill_kvq_row(bp, row)
        return tmp

    def _finish_batch_row(self, cache, n_tokens: int):
        """after a prefill chunk of a kv_bits=8 batch row: its bf16 layers move to the batch pool's row"""
        eng = self._engine()
        bp = cache[0]._batch_pool
        eng.set_prefill_kvq(None)
        if bp.bf is None:
            return
        from ... import _native as Nn
        tmp = bp._admit[1]
        src = tmp.buf[bp.n_q:]
        Nn.check(eng.lib.b200_pool_copy_row(bp.bf.buf.data_ptr(), bp.batch, bp.capacity, int(cache[0]._row),
                                            src.data_ptr(), 1, tmp.capacity, 0, bp.n_layers - bp.n_q, bp.n_kv,
                                            2 * bp.hd, int(n_tokens), eng.s), "pool_copy_row")

    # ------------------------------------------------------------------ call
    def __call__(self, inputs, inputs_embeds=None, mask=None, cache=None, **kwargs):
        position_ids = kwargs.pop("position_ids", None)
        pixel_values = kwargs.pop("pixel_values", None)
        image_grid_thw = kwargs.pop("image_grid_thw", None)
        video_grid_thw = kwargs.pop("video_grid_thw", None)
        rope_deltas_kw = kwargs.pop("rope_deltas", None)
        logits_to_keep = kwargs.pop("logits_to_keep", None)
        reserve_tokens = kwargs.pop("reserve_tokens", 0)
        eng = self._engine()
        if pixel_values is not None:  # new image/video: reset (language.py:418-420)
            self._rope_deltas = None
            self._position_ids = None
        if rope_deltas_kw is not None:
            self._rope_deltas = _np(rope_deltas_kw)
        if cache is None or cache[0] is None:
            cache = self.make_cache()  # stateless call: throw-away cache
        ids_host = _np(inputs)
        if ids_host.ndim == 1:
            ids_host = ids_host[None]
        B, L = ids_host.shape
        if isinstance(cache[0], (RowBatchKVCache, BatchQuantizedKVCache)):
            return self._call_batch(ids_host, inputs_embeds, mask, cache, rope_deltas_kw, position_ids,
                                    reserve_tokens)
        cache_offset = int(cache[0].offset)
        if B != 1:
            raise ValueError("a batch of rows needs a batch cache: LanguageModel.make_batch_cache(rows) "
                             "(device-resident RowBatchKVCache)")
        position_ids, delta0 = self.resolve_position_ids(ids_host, cache_offset, position_ids, mask,
                                                         image_grid_thw, video_grid_thw, rope_deltas_kw)

        need = max(cache_offset + L, reserve_tokens)
        self._bind(cache, need, decode=(L == 1 and inputs_embeds is None), chunk_end=cache_offset + L)
        V = self.args.vocab_size
        if L == 1 and inputs_embeds is None:
            # ---- decode step through the captured graph ----
            pos = int(position_ids[0, 0, 0])
            eng.set_next(int(ids_host[0, 0]), cache_offset, pos)
            eng.decode(1)
            logits = eng.snapshot("logits").view(1, 1, V)
        else:
            if inputs_embeds is None:
                from .qwen2_vl import embed_tokens
                inputs_embeds = embed_tokens(eng, ids_host)
            emb = inputs_embeds.reshape(-1, inputs_embeds.shape[-1])
            assert emb.shape[0] == L and emb.dtype == torch.bfloat16 and emb.is_cuda
            pos3 = torch.from_numpy(np.ascontiguousarray(position_ids[:, 0, :], dtype=np.int32))
            with torch.cuda.stream(eng.stream):
                pos3 = pos3.to(eng.device, non_blocking=False)
            keep_all = logits_to_keep is None or logits_to_keep != 1
            Vp = (V + 7) // 8 * 8     # device rows are 16-byte aligned for any vocabulary
            all_logits = eng.empty((L, Vp)) if keep_all else None
            eng.prefill(emb.contiguous(), pos3, cache_offset, delta0, all_logits)
            if getattr(cache[0], "_batch_pool", None) is not None:
                self._finish_batch_row(cache, cache_offset + L)
            elif isinstance(cache[0], QuantizedKVCache):
                eng.set_prefill_kvq(None)
            logits = (all_logits[:, :V].unsqueeze(0) if keep_all
                      else eng.snapshot("logits").view(1, 1, V))
        for c in cache:
            c.offset += L
        return LanguageModelOutput(logits=logits)

    def prefill_rows(self, ids_list, embeds_list, caches, position_ids_list=None, rope_deltas_list=None,
                     reserve_tokens: int = 0) -> List[int]:
        """The reference's `PromptProcessingBatch` (ar.py:1581-2175) for FRESH prompts that live in rows of ONE
        batched pool: all prompts are prefilled in one pass over the weights (tokens concatenated, block-diagonal
        causal attention, every token scattered to its own row / position of the pool).  `caches[g]` are the
        per-layer row caches of prompt g (`make_cache_row`); returns the first greedy token of every prompt
        (host ints; one device->host fetch for the whole group)."""
        eng = self._engine()
        n = len(ids_list)
        assert n == len(embeds_list) == len(caches) and n > 0
        pools = {id(c[0]._pool) for c in caches}
        if len(pools) != 1 or any(int(c[0].offset) != 0 for c in caches):
            raise ValueError("prefill_rows: fresh prompts in rows of one pool only")
        lens, pos, embs, deltas = [], [], [], []
        for g in range(n):
            ids = _np(ids_list[g])
            if ids.ndim == 1:
                ids = ids[None]
            L = ids.shape[1]
            self._rope_deltas, self._position_ids = None, None
            p3, d0 = self.resolve_position_ids(
                ids, 0, None if position_ids_list is None else position_ids_list[g], None, None, None,
                None if rope_deltas_list is None else rope_deltas_list[g])
            if rope_deltas_list is not None and rope_deltas_list[g] is not None:
                d0 = int(np.asarray(rope_deltas_list[g]).reshape(-1)[0])
            e = embeds_list[g].reshape(-1, embeds_list[g].shape[-1])
            assert e.shape[0] == L and e.dtype == torch.bfloat16 and e.is_cuda
            pad = (-L) % 8            # sequences start at multiples of 8 tokens in the concatenated batch
            p3 = np.asarray(p3)[:, 0, :].astype(np.int32)
            lens.append(L)
            pos.append(np.ascontiguousarray(np.pad(p3, ((0, 0), (0, pad)))))
            embs.append((e, pad))
            deltas.append(d0)
        need = max(max(lens), reserve_tokens)
        self._bind(caches[0], need)
        pos3 = torch.from_numpy(np.ascontiguousarray(np.concatenate(pos, axis=1)))
        with torch.cuda.stream(eng.stream):
            pos3 = pos3.to(eng.device)
            parts = []
            for e, pad in embs:
                parts.append(e)
                if pad:
                    parts.append(torch.zeros(pad, e.shape[1], dtype=e.dtype, device=e.device))
            emb = torch.cat(parts, 0) if len(parts) > 1 else parts[0].contiguous()
        start = eng.tokens_launched
        eng.prefill_batch(emb, pos3, lens, [int(c[0]._row or 0) for c in caches])
        for g in range(n):
            for c in caches[g]:
                c.offset += lens[g]
        host = torch.empty(n, dtype=torch.int32).pin_memory()
        eng.fetch_tokens(start, n, host)
        eng.stream.synchronize()
        self._rope_deltas, self._position_ids = None, None
        self.last_prefill_deltas = deltas
        return [int(t) for t in host]

    def resolve_position_ids(self, ids_host: np.ndarray, cache_offset: int, position_ids=None, mask=None,
                             image_grid_thw=None, video_grid_thw=None, rope_deltas_kw=None):
        """Position bookkeeping of `LanguageModel.__call__` (reference language.py:404-518), pure host
        logic: returns ((3, B, L) int positions, M-RoPE delta of row 0) and records `_rope_deltas` /
        `_position_ids` like the reference.
          * explicit `position_ids` longer than the chunk are sliced at the cache offset;
          * first call of a request (cache empty or no delta yet): the stored ids of the request
            (chunked prefill) or `get_rope_index`;
          * afterwards (decode / later chunks): arange(L) + cache_offset + rope_delta on all three axes;
          * 2-D (text-only) positions are broadcast to the three M-RoPE axes."""
        B, L = ids_host.shape
        position_ids = _np(position_ids)
        if position_ids is not None and position_ids.shape[-1] > L:
            position_ids = position_ids[..., cache_offset:cache_offset + L]
        rope_mask = mask
        if mask is not None and _np(mask).shape[-1] != L:
            rope_mask = None
        if position_ids is None and (rope_mask is None or _np(rope_mask).ndim == 2):
            if cache_offset == 0 or self._rope_deltas is None:
                if self._position_ids is not None:
                    position_ids = self._position_ids[..., cache_offset:cache_offset + L]
                else:
                    position_ids, deltas = self.get_rope_index(ids_host, image_grid_thw,
                                                               video_grid_thw, rope_mask)
                    self._rope_deltas = deltas
                    self._position_ids = position_ids
            else:
                src = _np(rope_deltas_kw) if rope_deltas_kw is not None else self._rope_deltas
                delta = cache_offset + np.asarray(src).reshape(-1)[:B]
                position_ids = np.arange(L)[None, :] + delta[:, None]  # (B, L)
                position_ids = np.broadcast_to(position_ids[None], (3, B, L))
        if position_ids.ndim == 2:  # text-only: the same scalar position on every axis
            position_ids = np.broadcast_to(position_ids[None], (3,) + position_ids.shape)
        delta0 = int(np.asarray(self._rope_deltas).reshape(-1)[0]) if self._rope_deltas is not None else 0
        return position_ids, delta0

    # -------------------------------------------------- fused greedy decoding
    def fused_greedy_decode(self, inputs, cache=None, **kwargs):
        """The reference's operator hook, with its contract (generate/ar.py:1015-1042,
        `GenerationBatch._fused_greedy_step`):

            sampled = language_model.fused_greedy_decode(inputs[:, None], cache=prompt_cache,
                                                         **fwd_kwargs)   # fwd_kwargs: rope_deltas

        `inputs` (B, 1) token ids -> greedy token ids (B,) of the NEXT position as an int32 device
        tensor (or None when this call cannot be served, which makes the reference fall back to
        `__call__`).  One persistent-kernel launch: forward, logprobs and argmax never leave the
        device.  When `inputs` is (a view of) the tensor this method returned last time (the
        reference feeds `_next_tokens[:, None]` straight back), the token is already in the device
        state and no host round trip happens at all."""
        if cache is None or kwargs.get("logits_processors"):
            return None
        eng = self._engine()
        last = getattr(self, "_fused_last", None)
        chained = (last is not None and isinstance(inputs, torch.Tensor) and inputs.is_cuda
                   and inputs.numel() == 1 and inputs.data_ptr() == last.data_ptr())
        if not chained:
            ids = _np(inputs)
            if ids.ndim == 1:
                ids = ids[:, None]
            if ids.shape[1] != 1:
                return None
            if ids.shape[0] != 1:
                return self._fused_greedy_batch(ids, cache, _inputs_tensor=inputs, **kwargs)
        rd = kwargs.get("rope_deltas", None)
        if rd is not None:
            self._rope_deltas = _np(rd)
        off = int(cache[0].offset)
        self._bind(cache, max(off + 1, int(kwargs.get("reserve_tokens", 0))), decode=True)
        if not chained:
            delta = int(np.asarray(self._rope_deltas).reshape(-1)[0]) if self._rope_deltas is not None else 0
            eng.set_next(int(ids[0, 0]), off, off + delta)
        idx = eng.tokens_launched
        eng.decode(1)
        for c in cache:
            c.offset += 1
        out = eng.token_log_view()[idx % eng.token_log_capacity: idx % eng.token_log_capacity + 1]
        self._fused_last = out
        return out

    # ----------------------------------------------------------- batched rows
    def _arm_batch(self, rows: BatchRows, toks, deltas, need: int):
        eng = self._engine()
        B = rows.B
        d = np.zeros(B, dtype=np.int64) if deltas is None else np.asarray(deltas, dtype=np.int64).reshape(-1)[:B]
        if d.shape[0] < B:
            d = np.resize(d, B)
        rows.ensure(B, need)
        eng.bind_pool(rows.pool)
        ctx = np.asarray(rows.lengths, dtype=np.int64)
        eng.batch_begin(np.asarray(toks).reshape(-1)[:B], ctx, ctx + d, np.ones(B, dtype=np.int32))
        self._batch_key = (id(rows), rows.version, rows.key())
        self._batch_step = 0

    def _fused_greedy_batch(self, ids, cache, **kwargs):
        """B > 1 rows in lock step (csrc/decode_batch.cu): ONE weight stream per step for all rows.
        cache: per-layer RowBatchKVCache of `make_batch_cache` / `RowBatchKVCache.merge`."""
        rows = getattr(cache[0], "_rows", None)
        if rows is None or rows.B != ids.shape[0]:
            return None
        eng = self._engine()
        inputs = kwargs.get("_inputs_tensor", None)
        last = getattr(self, "_fused_last", None)
        key = (id(rows), rows.version, rows.key())
        chained = (last is not None and isinstance(inputs, torch.Tensor) and inputs.is_cuda and
                   inputs.data_ptr() == last.data_ptr() and getattr(self, "_batch_key", None) == key and
                   self._batch_step + 1 < eng.BATCH_LOG_STEPS and
                   max(rows.lengths) + 1 <= rows.pool.capacity)
        if not chained:
            self._arm_batch(rows, ids[:, 0], kwargs.get("rope_deltas", None),
                            max(max(rows.lengths) + 1, int(kwargs.get("reserve_tokens", 0))))
        eng.batch_decode(1)
        out = eng.batch_token_log_view()[self._batch_step, :rows.B]
        self._batch_step += 1
        rows.lengths = [n + 1 for n in rows.lengths]
        self._fused_last = out
        return out

    def _call_batch(self, ids_host, inputs_embeds, mask, cache, rope_deltas_kw, position_ids, reserve_tokens):
        """LanguageModel.__call__ for B rows with a device batch cache (language.py:404-518, batched
        decode branch).  L == 1: one lock-step step, logits (B, 1, V).  L > 1: rows are prefilled
        one by one into their pool rows (`mask` (B, L) marks each row's real, right-aligned tokens)."""
        rows: BatchRows = cache[0]._rows
        eng = self._engine()
        B, L = ids_host.shape
        V = self.args.vocab_size
        if L == 1 and inputs_embeds is None:
            assert B == rows.B, (B, rows.B)
            self._arm_batch(rows, ids_host[:, 0], rope_deltas_kw,
                            max(max(rows.lengths) + 1, int(reserve_tokens)))
            eng.batch_decode(1)
            self._batch_step = 1
            self._fused_last = None
            rows.lengths = [n + 1 for n in rows.lengths]
            rows_logits = eng.empty((B, V))
            from ... import _native as Nn
            Nn.check(eng.lib.b200_memcpy_d2d(rows_logits.data_ptr(), eng.lib.b200_batch_logits(eng.h), B * V * 2,
                                             eng.s), "memcpy_d2d")
            return LanguageModelOutput(logits=rows_logits.view(B, 1, V))
        # ---- prompt rows: batch-1 prefills into the pool rows (admission) ----
        m = np.ones((B, L), dtype=np.int64) if mask is None else _np(mask)
        if rows.B == 0:
            rows.lengths = [0] * B
        assert rows.B == B
        rows.ensure(B, max(int(reserve_tokens), max(rows.lengths) + L))
        out = eng.empty((B, 1, V))
        from ... import _native as Nn
        deltas = []
        for b in range(B):
            n = int(m[b].sum())
            sub = ids_host[b:b + 1, L - n:]
            emb = None if inputs_embeds is None else inputs_embeds[b:b + 1, L - n:]
            saved = (self._rope_deltas, self._position_ids)
            self._rope_deltas, self._position_ids = None, None
            rc = self.make_cache_row(rows.pool, b)
            for c in rc:
                c.offset = rows.lengths[b]
            pid = None if position_ids is None else _np(position_ids)[:, b:b + 1, L - n:]
            o = self(sub, inputs_embeds=emb, cache=rc, position_ids=pid, logits_to_keep=1,
                     reserve_tokens=rows.pool.capacity)
            Nn.check(eng.lib.b200_memcpy_d2d(out[b].data_ptr(), o.logits.data_ptr(), V * 2, eng.s), "memcpy_d2d")
            deltas.append(0 if self._rope_deltas is None else int(np.asarray(self._rope_deltas).reshape(-1)[0]))
            self._rope_deltas, self._position_ids = saved
            rows.lengths[b] += n
        rows._touch()
        self._batch_rope_deltas = np.asarray(deltas, dtype=np.int64).reshape(-1, 1)
        return LanguageModelOutput(logits=out)

    def fused_greedy_decode_n(self, n_steps: int, cache, reserve_tokens: int = 0):
        """`n_steps` greedy decode steps entirely on the device (token feedback through device
        memory, no host round trip between steps).  Tokens land in the engine's token log."""
        eng = self._engine()
        off = int(cache[0].offset)
        self._bind(cache, max(off + n_steps, reserve_tokens), decode=True)
        eng.decode(n_steps)
        self._fused_last = None
        for c in cache:
            c.offset += n_steps

    @property
    def layers(self):
        return list(range(self.args.num_hidden_layers))

    @property
    def head_dim(self):
        return self.args.hidden_size // self.args.num_attention_heads

    @property
    def n_kv_heads(self):
        return self.args.num_key_value_heads
