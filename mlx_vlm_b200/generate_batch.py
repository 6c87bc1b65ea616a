"""Continuous batching surface of the reference (generate/ar.py: `BatchGenerator` :2178-2887,
`GenerationBatch.Response` :937-944, `BatchStats` / `BatchResponse` / `PromptProgress` :863-914,
`BatchGenerationResult` :519-545, `_left_pad_prompts` / `_right_pad_prompts` :548-560,
`batch_generate` :2890-3097).

With `kv_bits=8` the pool follows the reference's batch rule (`_make_cache`, ar.py:751-859): the layers where
`should_quantize_kv_layer` holds are 8-bit from the first prefill on (models/cache.py `BatchKVQPool`), the last
layer of a deeper stack stays bf16.

How the rows run on the CUDA engine: LOCK STEP on the device (csrc/decode_batch.cu).  All active
rows live in ONE batched KV pool (layers, 2, rows, kv heads, capacity, head_dim), each with its own
length (no left padding); a decode step is one captured CUDA graph that streams the weights ONCE
for all rows (weight-major wgmma GEMMs with the rows as a 16-wide token tile), so B rows cost
about one batch-1 step.  Admission of a request = a batch-1 prefill straight into a free row of
the pool; a finished row is replaced by the last row (one row copy); the device state is re-armed
only when the set of rows changes.  Tokens are produced in slices of `decode_slice` steps and
surfaced one per row per `next()` call.  Scheduling policy is the reference's: decode-first, then
admit up to `prefill_batch_size` waiting prompts (shortest first) while fewer than
`completion_batch_size` rows are active.  Engines without the batched decoder (the CPU stand-in
of the host-logic tests) run the rows time-multiplexed over the batch-1 path instead.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .models import cache as cache_mod

DEFAULT_MAX_TOKENS = 256
DEFAULT_COMPLETION_BATCH_SIZE = 32
DEFAULT_PREFILL_BATCH_SIZE = 8


def _host_buf(n: int) -> torch.Tensor:
    t = torch.empty(n, dtype=torch.int32)
    return t.pin_memory() if torch.cuda.is_available() else t


def _left_pad_prompts(prompts, max_length=None):
    """ar.py:548-553: rows right-aligned, zeros in front."""
    if max_length is None:
        max_length = max(len(p) for p in prompts)
    return np.asarray([[0] * (max_length - len(p)) + list(p) for p in prompts])


def _right_pad_prompts(prompts, max_length=None):
    """ar.py:555-560."""
    if max_length is None:
        max_length = max(len(p) for p in prompts)
    return np.asarray([list(p) + [0] * (max_length - len(p)) for p in prompts])


@dataclass
class BatchGenerationResult:
    texts: List[str]
    tokens: List[Optional[int]]
    logprobs: List[Optional[List[float]]]
    prompt_tokens: List[int]
    generation_tokens: List[int]
    total_tokens: List[int]
    prompt_tps: List[float]
    generation_tps: List[float]
    peak_memory: float = 0.0
    image_sizes: Optional[List[Tuple[int, int]]] = None


@dataclass
class BatchStats:
    prompt_tokens: int = 0
    prompt_tps: float = 0
    prompt_time: float = 0
    generation_tokens: int = 0
    generation_tps: float = 0
    generation_time: float = 0
    peak_memory: float = 0


@dataclass
class BatchResponse:
    texts: List[str]
    stats: BatchStats
    image_sizes: Optional[List[Tuple[int, int]]] = None


@dataclass
class PromptProgress:
    uid: int
    prompt_tokens: int
    prompt_tps: float = 0.0
    prompt_time: float = 0.0
    cached_tokens: int = 0


@dataclass
class _Row:
    uid: int
    ids: List[int]
    max_tokens: int
    kwargs: Dict[str, Any]
    cache: Optional[list] = None
    delta: Optional[int] = 0   # M-RoPE delta of the row (None: the model has no M-RoPE state)
    n_tokens: int = 0          # tokens surfaced so far
    n_decoded: int = 0         # tokens computed so far (>= n_tokens: the slice buffer)
    last_token: int = -1       # last computed token (input of the next decode step)
    buffer: List[Tuple[int, float]] = field(default_factory=list)
    reserve: int = 0
    ctx: int = 0               # tokens in the row's KV cache (lock-step mode)


class GenerationBatch:
    """The set of rows that are decoding (reference ar.py:929-1390).  Observable bookkeeping of the
    reference object — `uids`, `max_tokens`, `_num_tokens`, per-row `_rope_deltas` (B, 1), `filter`,
    `extend`, `empty` — over rows that each own their KV pool (so `filter` / `extend` move no cache
    memory here; the reference's versions also re-pack a `BatchKVCache`)."""

    @dataclass
    class Response:
        uid: int
        token: int
        token_logprob: float
        finish_reason: Optional[str]
        top_logprobs: Optional[List[Tuple[int, float]]] = None

    def __init__(self, rows: Optional[List[_Row]] = None):
        self.rows: List[_Row] = list(rows or [])

    @classmethod
    def empty(cls, *_, **__) -> "GenerationBatch":
        return cls([])

    def __len__(self) -> int:
        return len(self.rows)

    @property
    def uids(self) -> List[int]:
        return [r.uid for r in self.rows]

    @property
    def max_tokens(self) -> List[int]:
        return [r.max_tokens for r in self.rows]

    @property
    def _num_tokens(self) -> List[int]:
        return [r.n_tokens for r in self.rows]

    @property
    def _rope_deltas(self) -> Optional[np.ndarray]:
        if not self.rows or self.rows[0].delta is None:
            return None
        return np.asarray([[r.delta] for r in self.rows], dtype=np.int32)

    def filter(self, keep: List[int]) -> None:
        self.rows = [self.rows[i] for i in keep]

    def extend(self, other: "GenerationBatch") -> None:
        if self.rows and other.rows and (self.rows[0].delta is None) != (other.rows[0].delta is None):
            raise RuntimeError("extend() mixes MRoPE and non-MRoPE batches; both sides must carry "
                               "rope_deltas or neither side may.")
        self.rows.extend(other.rows)


class BatchGenerator:
    """`insert()` prompts (token-id lists), then call `next()` until `has_work` is False.

    next() -> (prompt_responses: List[PromptProgress], generation_responses:
    List[GenerationBatch.Response]) — one response per active row per call; a row's last
    response carries finish_reason "stop" (EOS) or "length"."""

    def __init__(self, model, processor, *, max_tokens: int = DEFAULT_MAX_TOKENS,
                 stop_tokens: Optional[set] = None, sampler: Optional[Callable] = None,
                 completion_batch_size: int = DEFAULT_COMPLETION_BATCH_SIZE,
                 prefill_batch_size: int = DEFAULT_PREFILL_BATCH_SIZE,
                 prefill_step_size: Optional[int] = None, compute_logprobs: bool = False,
                 top_logprobs_k: int = 0, logits_processors=None, greedy_sampling: bool = False,
                 decode_slice: int = 16, batched_prefill: bool = True, kv_bits=None, kv_group_size: int = 64,
                 kv_quant_scheme: Optional[str] = None, quantized_kv_start: int = 0, **unsupported):
        for k in ("kv_key_bits", "kv_value_bits", "draft_model", "apc_manager", "prompt_cache"):
            if unsupported.pop(k, None) is not None:
                raise NotImplementedError(f"BatchGenerator: `{k}` is outside this engine's hot-path scope")
        # kv_bits=8: the reference's batch rule (ar.py:751-859 `_make_cache`): every layer where
        # `should_quantize_kv_layer` holds keeps an 8-bit cache from the first prefill on; `quantized_kv_start`
        # plays no part in it (accepted for the reference's signature)
        from .generate import kv_quant_args
        self.kv_bits = kv_quant_args(kv_bits, kv_group_size, kv_quant_scheme,
                                     getattr(getattr(model, "language_model", None), "head_dim", None) or 128)
        self.kv_group_size = int(kv_group_size)
        if logits_processors:
            raise NotImplementedError("BatchGenerator: logits processors run on the single-request path only")
        if top_logprobs_k:
            raise NotImplementedError("BatchGenerator: top_logprobs_k > 0 is not supported")
        self.model, self.processor = model, processor
        self.max_tokens = max_tokens
        self.sampler = sampler
        self.greedy_sampling = greedy_sampling or sampler is None or getattr(sampler, "is_greedy", False)
        self.compute_logprobs = compute_logprobs
        self.completion_batch_size = completion_batch_size
        self.prefill_batch_size = prefill_batch_size
        self.prefill_step_size = prefill_step_size
        self.decode_slice = max(1, int(decode_slice))
        self.batched_prefill = bool(batched_prefill)
        self.tokenizer = processor.tokenizer if hasattr(processor, "tokenizer") else processor
        from .utils import StoppingCriteria
        if getattr(self.tokenizer, "stopping_criteria", None) is None:
            eos = getattr(getattr(model, "config", None), "eos_token_id", None)
            self.tokenizer.stopping_criteria = StoppingCriteria(eos if eos is not None else [], self.tokenizer)
        if stop_tokens:
            self.tokenizer.stopping_criteria.add_eos_token_ids(list(stop_tokens))
        eng = getattr(model, "engine", None)
        lm = getattr(model, "language_model", None)
        # lock-step batched decode needs the native batched decoder (<= 16 rows per weight stream)
        self._lockstep = (hasattr(eng, "batch_begin") and hasattr(lm, "make_cache_row")
                          and getattr(lm, "lockstep_supported", True)
                          and not unsupported.pop("time_multiplex", False))
        if self.kv_bits is not None and not self._lockstep:
            raise NotImplementedError(
                "BatchGenerator(kv_bits=8) runs in the lock-step batch only; this model / engine runs its rows "
                "time-multiplexed over the single-request path (no batched decoder, or a Qwen3-VL head_dim other "
                "than hidden / heads), whose 8-bit policy is the single-request one")
        if self._lockstep:
            self.completion_batch_size = min(self.completion_batch_size, 16)
        self._pool = None          # the shared batched KV pool (lock-step mode)
        self._armed_key = None     # (uids, live flags) the device state was armed for
        self._steps_since_begin = 0
        self.uid_count = 0
        self._unprocessed_sequences: List[_Row] = []
        self._generation_batch = GenerationBatch.empty()
        self._prompt_tokens_counter = 0
        self._prompt_time_counter = 0.0
        self._gen_tokens_counter = 0
        self._gen_time_counter = 0.0

    # ------------------------------------------------------------------ queueing
    def insert(self, prompts, max_tokens: Union[List[int], int, None] = None,
               prompt_kwargs: Optional[List[dict]] = None) -> List[int]:
        if max_tokens is None or isinstance(max_tokens, int):
            max_tokens = [max_tokens or self.max_tokens] * len(prompts)
        if prompt_kwargs is None:
            prompt_kwargs = [{} for _ in prompts]
        if len(max_tokens) != len(prompts) or len(prompt_kwargs) != len(prompts):
            raise ValueError("insert: max_tokens / prompt_kwargs must match the number of prompts")
        uids = []
        for p, m, kw in zip(prompts, max_tokens, prompt_kwargs):
            ids = np.asarray(p.cpu() if isinstance(p, torch.Tensor) else p).reshape(-1).tolist()
            self._unprocessed_sequences.append(_Row(self.uid_count, ids, int(m), dict(kw or {})))
            uids.append(self.uid_count)
            self.uid_count += 1
        self._unprocessed_sequences.sort(key=lambda r: len(r.ids))  # shortest first (ar.py:2620-2623)
        return uids

    @property
    def _active(self) -> List[_Row]:
        return self._generation_batch.rows

    def remove(self, uid) -> bool:
        for i, r in enumerate(self._unprocessed_sequences):   # waiting in the queue
            if r.uid == uid:
                self._unprocessed_sequences.pop(i)
                return True
        if uid in self._generation_batch.uids:                 # already decoding
            idx = self._generation_batch.uids.index(uid)
            self._generation_batch.filter([i for i in range(len(self._generation_batch)) if i != idx])
            if self._lockstep:
                self._compact()
            return True
        return False

    @property
    def unprocessed_prompts(self):
        return self._unprocessed_sequences

    @property
    def has_pending_prompts(self) -> bool:
        return len(self._unprocessed_sequences) > 0

    @property
    def has_work(self) -> bool:
        return bool(self._active) or bool(self._unprocessed_sequences)

    @property
    def active_uids(self) -> List[int]:
        return [r.uid for r in self._active]

    def stats(self) -> BatchStats:
        s = BatchStats()
        s.prompt_tokens = self._prompt_tokens_counter
        s.prompt_time = self._prompt_time_counter
        s.prompt_tps = s.prompt_tokens / s.prompt_time if s.prompt_time > 0 else 0
        s.generation_tokens = self._gen_tokens_counter
        s.generation_time = self._gen_time_counter
        s.generation_tps = s.generation_tokens / s.generation_time if s.generation_time > 0 else 0
        eng = getattr(self.model, "engine", None)
        if eng is not None and torch.cuda.is_available():
            s.peak_memory = torch.cuda.max_memory_allocated(eng.device) / 1e9
        return s

    def close(self):
        self._generation_batch.filter([])
        self._unprocessed_sequences.clear()

    # ------------------------------------------------------------------ device work
    def _logprob_of(self, tok: int) -> float:
        eng = self.model.engine
        lp = eng.snapshot("logprobs")
        with torch.cuda.stream(eng.stream):   # ordered after the snapshot copy; .item() syncs it
            return float(lp.view(-1)[tok].float().item())

    def _prefill(self, row: _Row) -> PromptProgress:
        """Embeddings + prefill for one row; the fused head + sampler leave the first token in
        the engine's token log."""
        model, lm, eng = self.model, self.model.language_model, self.model.engine
        tic = time.perf_counter()
        kw = dict(row.kwargs)
        ids = np.asarray([row.ids])
        emb = kw.pop("inputs_embeds", None)
        pos, deltas = kw.pop("position_ids", None), kw.pop("rope_deltas", None)
        if emb is None:
            out = model.get_input_embeddings(ids, kw.pop("pixel_values", None), mask=kw.pop("mask", None), **kw)
            emb, pos, deltas = out.inputs_embeds, out.position_ids, out.rope_deltas
        T = emb.shape[1]
        row.reserve = T + row.max_tokens + 1
        if self._lockstep:
            row.cache = lm.make_cache_row(self._pool_for(row.reserve), len(self._active) + self._admitting)
            self._admitting += 1
        else:
            row.cache = cache_mod.make_prompt_cache(lm)
        row.delta = int(np.asarray(deltas).reshape(-1)[0]) if deltas is not None else 0
        step = self.prefill_step_size
        ids_left = ids
        while step is not None and emb.shape[1] > step + 1:   # chunked prefill (ar.py:426-472)
            lm(ids_left[:, :step], inputs_embeds=emb[:, :step], cache=row.cache, position_ids=pos,
               rope_deltas=deltas, logits_to_keep=1, reserve_tokens=row.reserve)
            emb, ids_left = emb[:, step:], ids_left[:, step:]
        out = lm(ids_left, inputs_embeds=emb, cache=row.cache, position_ids=pos, rope_deltas=deltas,
                 logits_to_keep=1, reserve_tokens=row.reserve)
        if self.greedy_sampling:
            host = _host_buf(1)
            eng.fetch_tokens(eng.tokens_launched - 1, 1, host)
            eng.stream.synchronize()
            tok = int(host[0])
            lp = self._logprob_of(tok) if self.compute_logprobs else 0.0
        else:
            tok, lp = self._sample(out.logits[:, -1, :])
        row.last_token, row.n_decoded = tok, 1
        row.ctx = int(row.cache[0].offset)
        row.buffer.append((tok, lp))
        if self.kv_bits is not None and self._lockstep:
            self._pool._admit = None   # the bf16 pool of the admission (csrc: prefill write-through) is done
        dt = time.perf_counter() - tic
        self._prompt_tokens_counter += len(row.ids)
        self._prompt_time_counter += dt
        return PromptProgress(uid=row.uid, prompt_tokens=len(row.ids), prompt_time=dt,
                              prompt_tps=len(row.ids) / dt if dt > 0 else 0.0)

    def _prefill_group(self, rows: List[_Row]) -> List[PromptProgress]:
        """`PromptProcessingBatch` (ar.py:1581-2175): the rows admitted together are prefilled in ONE pass over the
        weights (tokens concatenated, block-diagonal causal attention, every token scattered to its own pool row);
        embeddings (vision tower + merge) are still produced per request."""
        model, lm, eng = self.model, self.model.language_model, self.model.engine
        tic = time.perf_counter()
        ids_l, emb_l, pos_l, del_l = [], [], [], []
        for row in rows:
            kw = dict(row.kwargs)
            ids = np.asarray([row.ids])
            emb = kw.pop("inputs_embeds", None)
            pos, deltas = kw.pop("position_ids", None), kw.pop("rope_deltas", None)
            if emb is None:
                out = model.get_input_embeddings(ids, kw.pop("pixel_values", None), mask=kw.pop("mask", None), **kw)
                emb, pos, deltas = out.inputs_embeds, out.position_ids, out.rope_deltas
            row.reserve = emb.shape[1] + row.max_tokens + 1
            row.delta = int(np.asarray(deltas).reshape(-1)[0]) if deltas is not None else 0
            ids_l.append(ids); emb_l.append(emb); pos_l.append(pos); del_l.append(deltas)
        pool = self._pool_for(max(r.reserve for r in rows))
        base = len(self._active)
        for i, row in enumerate(rows):
            row.cache = lm.make_cache_row(pool, base + i)
        toks = lm.prefill_rows(ids_l, emb_l, [r.cache for r in rows], pos_l, del_l,
                               reserve_tokens=max(r.reserve for r in rows))
        dt = time.perf_counter() - tic
        out = []
        for row, tok in zip(rows, toks):
            row.last_token, row.n_decoded = tok, 1
            row.ctx = int(row.cache[0].offset)
            row.buffer.append((tok, 0.0))
            self._prompt_tokens_counter += len(row.ids)
            out.append(PromptProgress(uid=row.uid, prompt_tokens=len(row.ids), prompt_time=dt / len(rows),
                                      prompt_tps=len(row.ids) * len(rows) / dt if dt > 0 else 0.0))
        self._prompt_time_counter += dt
        return out

    def _sample(self, logits: torch.Tensor) -> Tuple[int, float]:
        # torch ops on the engine's stream: ordered after the step that wrote `logits`
        with torch.cuda.stream(self.model.engine.stream):
            lf = logits.float()
            logprobs = logits - torch.logsumexp(lf, dim=-1, keepdim=True).to(logits.dtype)
            y = self.sampler(logprobs)
            tok = int(y.reshape(-1)[0].item())
            return tok, float(logprobs.reshape(-1)[tok].float().item())

    # ------------------------------------------------------------------ lock-step rows
    _admitting = 0

    def _pool_for(self, need_tokens: int):
        """the shared batched pool, with room for `need_tokens` positions per row"""
        lm, eng = self.model.language_model, self.model.engine
        step = cache_mod.KVPool.step
        cap = ((need_tokens + step - 1) // step) * step
        if self._pool is None and self.kv_bits is not None:
            self._pool = cache_mod.BatchKVQPool(lm.args.num_hidden_layers, lm.n_kv_heads, lm.head_dim, eng.device,
                                                group_size=self.kv_group_size, batch=self.completion_batch_size,
                                                capacity=cap, stream=eng.stream)
        elif self._pool is None:
            self._pool = cache_mod.KVPool(lm.args.num_hidden_layers, lm.n_kv_heads, lm.head_dim, eng.device,
                                          batch=self.completion_batch_size, capacity=cap)
        elif cap > self._pool.capacity:
            import contextlib
            eng.stream.synchronize()
            on = torch.cuda.stream(eng.stream) if torch.cuda.is_available() else contextlib.nullcontext()
            with on:
                self._pool.reserve(cap, live_tokens=self._pool.capacity)
            self._armed_key = None
        return self._pool

    def _compact(self):
        """rows are pool rows 0..B-1 in `_active` order: after a filter, move rows down"""
        eng = self.model.engine
        for slot, row in enumerate(self._active):
            cur = row.cache[0]._row
            if cur != slot:
                eng.kv_copy_row(self._pool, slot, self._pool, cur, row.ctx)
                for c in row.cache:
                    c._row = slot
                self._armed_key = None

    def _lockstep_slice(self):
        """one slice of lock-step decode steps for every row that still has tokens to compute"""
        eng = self.model.engine
        rows = self._active
        live = [r.n_decoded < r.max_tokens for r in rows]
        if not any(live):
            return
        k = min([self.decode_slice] + [r.max_tokens - r.n_decoded for r, a in zip(rows, live) if a])
        greedy = self.greedy_sampling
        if not greedy:
            k = 1
        key = (tuple(r.uid for r in rows), tuple(live))
        if key != self._armed_key or self._steps_since_begin + k > 4000 or not greedy:
            eng.bind_pool(self._pool)
            eng.batch_begin([r.last_token for r in rows], [r.ctx for r in rows],
                            [r.ctx + (r.delta or 0) for r in rows], [int(a) for a in live])
            self._armed_key = key
            self._steps_since_begin = 0
        eng.batch_decode(k, want_logprobs=not greedy)
        B = len(rows)
        if greedy:
            toks = _host_buf(k * B).view(k, B)
            lps = torch.empty(k, B, dtype=torch.float32)
            lps = lps.pin_memory() if torch.cuda.is_available() else lps
            eng.batch_fetch(self._steps_since_begin, k, toks, lps)
            eng.stream.synchronize()
            self._steps_since_begin += k
            for b, (r, a) in enumerate(zip(rows, live)):
                if not a:
                    continue
                col = toks[:, b].tolist()
                r.buffer.extend((int(t), float(l)) for t, l in zip(col, lps[:, b].tolist()))
                r.last_token, r.n_decoded, r.ctx = int(col[-1]), r.n_decoded + k, r.ctx + k
                for c in r.cache:
                    c.offset = r.ctx
        else:   # sampler on the host-visible logits of every row (one step at a time)
            logits = eng.batch_logits_view("logits")
            self._steps_since_begin += 1
            for b, (r, a) in enumerate(zip(rows, live)):
                if not a:
                    continue
                tok, lp = self._sample(logits[b:b + 1])
                r.buffer.append((tok, lp))
                r.last_token, r.n_decoded, r.ctx = tok, r.n_decoded + 1, r.ctx + 1
                for c in r.cache:
                    c.offset = r.ctx
            self._armed_key = None

    def _decode_slice(self, row: _Row):
        """Refill the row's token buffer: hand the engine to this row for up to `decode_slice`
        steps (device-resident token feedback when greedy)."""
        lm, eng = self.model.language_model, self.model.engine
        left = row.max_tokens - row.n_decoded
        if left <= 0:
            return
        ctx = int(row.cache[0].offset)
        if self.greedy_sampling and not self.compute_logprobs:
            k = min(self.decode_slice, left)
            eng.set_next(row.last_token, ctx, ctx + row.delta)
            base = eng.tokens_launched
            lm.fused_greedy_decode_n(k, row.cache, reserve_tokens=row.reserve)
            host = _host_buf(k)
            eng.fetch_tokens(base, k, host)
            eng.stream.synchronize()
            toks = [int(t) for t in host.tolist()]
            row.buffer.extend((t, 0.0) for t in toks)
            row.last_token, row.n_decoded = toks[-1], row.n_decoded + k
        else:
            out = lm(np.asarray([[row.last_token]]), cache=row.cache,
                     rope_deltas=np.asarray([[row.delta]]), reserve_tokens=row.reserve)
            if self.greedy_sampling:
                lp = eng.snapshot("logprobs").view(-1)
                with torch.cuda.stream(eng.stream):
                    tok = int(torch.argmax(lp.float()).item())
                    lpv = float(lp[tok].float().item())
            else:
                tok, lpv = self._sample(out.logits[:, -1, :])
            row.buffer.append((tok, lpv))
            row.last_token, row.n_decoded = tok, row.n_decoded + 1

    # ------------------------------------------------------------------ scheduling
    def next(self, **kwargs):
        prompt_responses: List[PromptProgress] = []
        generation_responses: List[GenerationBatch.Response] = []
        stop = self.tokenizer.stopping_criteria
        # 1. decode-first: one token per active row
        if self._active:
            tic = time.perf_counter()
            keep = []
            if self._lockstep and any(not r.buffer for r in self._active):
                self._lockstep_slice()
            for i, row in enumerate(self._active):
                if not row.buffer:
                    self._decode_slice(row)
                tok, lp = row.buffer.pop(0)
                row.n_tokens += 1
                finish = None
                if stop(tok):
                    finish = "stop"
                elif row.n_tokens >= row.max_tokens:
                    finish = "length"
                generation_responses.append(GenerationBatch.Response(
                    uid=row.uid, token=tok, token_logprob=lp, finish_reason=finish))
                if finish is None:
                    keep.append(i)
            self._gen_tokens_counter += len(self._active)
            self._gen_time_counter += time.perf_counter() - tic
            if len(keep) < len(self._generation_batch):
                self._generation_batch.filter(keep)
                if self._lockstep:
                    self._compact()
        # 2. admit waiting prompts while there is room (shortest first)
        room = self.completion_batch_size - len(self._active)
        n_admit = min(room, self.prefill_batch_size, len(self._unprocessed_sequences))
        admitted = []
        self._admitting = 0
        # kv_bits=8 rows are admitted one at a time (the grouped prefill has no 8-bit write-through)
        group = (self._lockstep and n_admit >= 2 and self.greedy_sampling and not self.compute_logprobs
                 and self.kv_bits is None
                 and hasattr(self.model.language_model, "prefill_rows") and self.batched_prefill
                 and (self.prefill_step_size is None
                      or all(len(r.ids) <= self.prefill_step_size + 1 for r in self._unprocessed_sequences[:n_admit])))
        if group:
            admitted = [self._unprocessed_sequences.pop(0) for _ in range(n_admit)]
            prompt_responses.extend(self._prefill_group(admitted))
        for _ in range(0 if group else max(0, n_admit)):
            row = self._unprocessed_sequences.pop(0)
            prompt_responses.append(self._prefill(row))
            admitted.append(row)
        self._admitting = 0
        if admitted:
            self._generation_batch.extend(GenerationBatch(admitted))
        return prompt_responses, generation_responses


def batch_generate(model, processor, images=None, prompts: Optional[List[str]] = None,
                   max_tokens: Union[int, List[int]] = 128, verbose: bool = False,
                   resize_shape=None, **kwargs) -> BatchResponse:
    """ar.py:2890-3097: one prompt (and optionally one image) per row -> texts in input order."""
    from .generate import _make_detokenizer
    from .utils import prepare_inputs
    if prompts is None:
        raise ValueError("batch_generate: prompts is required")
    if isinstance(prompts, str):
        prompts = [prompts]
    if images is not None and not isinstance(images, (list, tuple)):
        images = [images]
    if images is not None and len(images) not in (0, len(prompts)):
        raise ValueError("batch_generate: give one image per prompt (or none)")
    eng = model.engine
    gen = BatchGenerator(model, processor, max_tokens=max_tokens if isinstance(max_tokens, int) else DEFAULT_MAX_TOKENS,
                         **kwargs)
    ids_list, kw_list, sizes = [], [], []
    for i, prompt in enumerate(prompts):
        img = images[i] if images else None
        inp = prepare_inputs(processor, images=[img] if img is not None else None, prompts=prompt,
                             resize_shape=resize_shape, device=eng.device, stream=eng.stream)
        ids_list.append(np.asarray(inp["input_ids"].cpu() if isinstance(inp["input_ids"], torch.Tensor)
                                   else inp["input_ids"]).reshape(-1).tolist())
        kw_list.append({k: v for k, v in inp.items() if k not in ("input_ids", "attention_mask") and v is not None})
        if img is not None and hasattr(img, "shape"):
            sizes.append((int(img.shape[0]), int(img.shape[1])))
    uids = gen.insert(ids_list, max_tokens if not isinstance(max_tokens, int) else None, kw_list)
    if isinstance(max_tokens, int):
        for r in gen.unprocessed_prompts:
            r.max_tokens = max_tokens
    detok = {u: _make_detokenizer(processor) for u in uids}
    stop = gen.tokenizer.stopping_criteria
    while gen.has_work:
        _, responses = gen.next()
        for r in responses:
            if not (r.finish_reason == "stop" and stop(r.token)):
                detok[r.uid].add_token(r.token)
    texts = []
    for u in uids:
        detok[u].finalize()
        texts.append(detok[u].text)
    stats = gen.stats()
    if verbose:
        print(f"Prompt: {stats.prompt_tokens} tokens, {stats.prompt_tps:.1f} tokens-per-sec")
        print(f"Generation: {stats.generation_tokens} tokens, {stats.generation_tps:.1f} tokens-per-sec")
    return BatchResponse(texts=texts, stats=stats, image_sizes=sizes or None)
