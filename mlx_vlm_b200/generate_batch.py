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
about one batch-1 step.  `models/cache.py::BatchRows` owns the pool's rows: admission of a request =
a prefill straight into the next free row; after rows finish the remaining rows move down (row
copies); every row's length; and when the device state is re-armed (`BatchRows.arm`).  Tokens are
produced in slices of `decode_slice` steps and surfaced one per row per `next()` call.  Scheduling policy is the reference's: decode-first, then
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
from .sample_utils import greedy_sampler, lower_logits_processors, top_logprobs

DEFAULT_MAX_TOKENS = 256
DEFAULT_COMPLETION_BATCH_SIZE = 32
DEFAULT_PREFILL_BATCH_SIZE = 8
TOP_LOGPROBS_MAX = 20   # the reference server's cap (server/generation.py get_top_logprobs_k) and the kernel's


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
    buffer: List[Tuple[int, float, Optional[list]]] = field(default_factory=list)   # (token, logprob, top-k)
    reserve: int = 0
    procs: Optional[list] = None     # the row's logits processors (None: none)
    lowered: Optional[dict] = None   # their device form (lock-step rows; None: torch ops on the host)
    context: Optional[List[int]] = None   # the reference's token context of a row with processors


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

    # The reference keeps `logits_processors` / `token_context` as lists aligned with the rows (ar.py:995-1013):
    # a batch that had processors when it was formed or extended tracks a context for EVERY row (the prompt when the
    # row was admitted with processors in its group, else []), appended while any row has processors; a batch that
    # never had any tracks none.  Here a row's `context` is None when it is not tracked.
    @property
    def logits_processors(self) -> list:
        """one processor list (or None) per row; [] when the batch tracks no processors"""
        return [r.procs for r in self.rows] if any(r.context is not None for r in self.rows) else []

    @property
    def token_context(self) -> List[List[int]]:
        return [list(r.context) for r in self.rows] if any(r.context is not None for r in self.rows) else []

    @staticmethod
    def admitted(rows: List[_Row]) -> "GenerationBatch":
        """rows admitted together (a prefill batch): each is seeded with its prompt when any of them has processors
        (ar.py:1663-1667)"""
        track = any(r.procs for r in rows)
        for r in rows:
            r.context = list(r.ids) if track else None
        return GenerationBatch(rows)

    def record_inputs(self, inputs: List[Tuple[_Row, List[int]]]):
        """the input tokens of the step(s) about to run join every tracked row's context while any row has
        processors (ar.py:1070-1074)"""
        if any(r.procs for r in self.rows):
            for r, toks in inputs:
                if r.context is not None:
                    r.context.extend(toks)

    def filter(self, keep: List[int]) -> None:
        self.rows = [self.rows[i] for i in keep]

    def extend(self, other: "GenerationBatch") -> None:
        if self.rows and other.rows and (self.rows[0].delta is None) != (other.rows[0].delta is None):
            raise RuntimeError("extend() mixes MRoPE and non-MRoPE batches; both sides must carry "
                               "rope_deltas or neither side may.")
        track = any(r.procs for r in self.rows + other.rows)   # ar.py:1181-1202
        for r in self.rows + other.rows:
            r.context = (r.context if r.context is not None else []) if track else None
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
        if not 0 <= int(top_logprobs_k) <= TOP_LOGPROBS_MAX:
            raise ValueError(f"BatchGenerator: top_logprobs_k must lie in [0, {TOP_LOGPROBS_MAX}]")
        self.top_logprobs_k = int(top_logprobs_k)
        self.logits_processors = list(logits_processors) if logits_processors else None   # default of every row
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
        self._rows: Optional[cache_mod.BatchRows] = None   # the rows of the shared batched KV pool (lock-step mode)
        self.uid_count = 0
        self._unprocessed_sequences: List[_Row] = []
        self._generation_batch = GenerationBatch.empty()
        self._prompt_tokens_counter = 0
        self._prompt_time_counter = 0.0
        self._gen_tokens_counter = 0
        self._gen_time_counter = 0.0

    # ------------------------------------------------------------------ queueing
    def insert(self, prompts, max_tokens: Union[List[int], int, None] = None,
               prompt_kwargs: Optional[List[dict]] = None, logits_processors=None) -> List[int]:
        """`logits_processors`: one processor list (or None) per prompt; None gives every prompt the generator's
        own list (ar.py:2584-2604)"""
        if max_tokens is None or isinstance(max_tokens, int):
            max_tokens = [max_tokens or self.max_tokens] * len(prompts)
        if prompt_kwargs is None:
            prompt_kwargs = [{} for _ in prompts]
        if logits_processors is None:
            logits_processors = [self.logits_processors] * len(prompts)
        elif len(logits_processors) != len(prompts):
            raise ValueError("Insufficient number of logits_processors provided")
        if len(max_tokens) != len(prompts) or len(prompt_kwargs) != len(prompts):
            raise ValueError("insert: max_tokens / prompt_kwargs must match the number of prompts")
        uids = []
        for p, m, kw, procs in zip(prompts, max_tokens, prompt_kwargs, logits_processors):
            ids = np.asarray(p.cpu() if isinstance(p, torch.Tensor) else p).reshape(-1).tolist()
            row = _Row(self.uid_count, ids, int(m), dict(kw or {}), procs=list(procs) if procs else None)
            self._check_bias(row.procs)
            if row.procs:
                lowered = lower_logits_processors(row.procs)
                row.lowered = lowered if lowered is not None and cache_mod.BatchProcState.fits(lowered) else None
            self._unprocessed_sequences.append(row)
            uids.append(self.uid_count)
            self.uid_count += 1
        self._unprocessed_sequences.sort(key=lambda r: len(r.ids))  # shortest first (ar.py:2620-2623)
        return uids

    def _check_bias(self, procs):
        """a logit bias must name tokens of the vocabulary: refused here, so only the request that brings it fails"""
        lm = getattr(self.model, "language_model", None)
        vocab = getattr(getattr(lm, "args", None), "vocab_size", None)
        for p in procs or []:
            spec = getattr(p, "lowered", None)
            if isinstance(spec, tuple) and spec[0] == "bias":
                bad = [i for i in spec[1] if not (isinstance(i, (int, np.integer)) and i >= 0
                                                  and (vocab is None or i < vocab))]
                if bad:
                    raise ValueError(f"logit_bias: token ids {bad} outside the vocabulary [0, {vocab})")

    @property
    def _active(self) -> List[_Row]:
        return self._generation_batch.rows

    @property
    def _pool(self):
        """the shared batched KV pool of lock-step mode (owned by `_rows`; None before the first admission)"""
        return None if self._rows is None else self._rows.pool

    def remove(self, uid) -> bool:
        for i, r in enumerate(self._unprocessed_sequences):   # waiting in the queue
            if r.uid == uid:
                self._unprocessed_sequences.pop(i)
                return True
        if uid in self._generation_batch.uids:                 # already decoding
            idx = self._generation_batch.uids.index(uid)
            self._keep([i for i in range(len(self._generation_batch)) if i != idx])
            return True
        return False

    def _keep(self, keep: List[int]):
        """the active rows `keep` (ascending) stay; in lock-step mode their pool rows move down to stay compact"""
        self._generation_batch.filter(keep)
        if self._rows is not None:
            self._rows.filter(keep)

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
        self._keep([])
        self._unprocessed_sequences.clear()

    # ------------------------------------------------------------------ device work
    def _logprob_of(self, tok: int) -> float:
        eng = self.model.engine
        lp = eng.snapshot("logprobs")
        with torch.cuda.stream(eng.stream):   # ordered after the snapshot copy; .item() syncs it
            return float(lp.view(-1)[tok].float().item())

    def _embed(self, row: _Row):
        """the row's prompt embeddings (vision tower + merge unless the request brings `inputs_embeds`); sets the
        row's `reserve` and M-RoPE `delta`.  Returns (ids, embeddings, position_ids, rope_deltas)."""
        kw = dict(row.kwargs)
        ids = np.asarray([row.ids])
        emb = kw.pop("inputs_embeds", None)
        pos, deltas = kw.pop("position_ids", None), kw.pop("rope_deltas", None)
        if emb is None:
            out = self.model.get_input_embeddings(ids, kw.pop("pixel_values", None), mask=kw.pop("mask", None), **kw)
            emb, pos, deltas = out.inputs_embeds, out.position_ids, out.rope_deltas
        row.reserve = emb.shape[1] + row.max_tokens + 1
        row.delta = int(np.asarray(deltas).reshape(-1)[0]) if deltas is not None else 0
        return ids, emb, pos, deltas

    def _pool_rows(self, need_tokens: int) -> cache_mod.BatchRows:
        """the rows of the shared batched pool, with room for `need_tokens` positions per row: allocated with
        `completion_batch_size` rows at the first admission, grown (capacity doubling) when a row needs more"""
        if self._rows is None:
            lm = self.model.language_model
            self._rows = cache_mod.BatchRows.allocate(self.model.engine, lm.args.num_hidden_layers, lm.n_kv_heads,
                                                      lm.head_dim, self.completion_batch_size, need_tokens,
                                                      self.kv_bits, self.kv_group_size)
        else:
            self._rows.ensure(self._rows.B, need_tokens)
        return self._rows

    def _prefill(self, row: _Row) -> PromptProgress:
        """Embeddings + prefill for one row; the fused head + sampler leave the first token in
        the engine's token log.  In lock-step mode the row is prefilled into the next free row of the pool."""
        lm, eng = self.model.language_model, self.model.engine
        tic = time.perf_counter()
        ids, emb, pos, deltas = self._embed(row)
        if self._lockstep:
            rows = self._pool_rows(row.reserve)
            cache = lm.make_cache_row(rows.pool, rows.B)
        else:
            cache = row.cache = cache_mod.make_prompt_cache(lm)
        step = self.prefill_step_size
        ids_left = ids
        while step is not None and emb.shape[1] > step + 1:   # chunked prefill (ar.py:426-472)
            lm(ids_left[:, :step], inputs_embeds=emb[:, :step], cache=cache, position_ids=pos,
               rope_deltas=deltas, logits_to_keep=1, reserve_tokens=row.reserve)
            emb, ids_left = emb[:, step:], ids_left[:, step:]
        out = lm(ids_left, inputs_embeds=emb, cache=cache, position_ids=pos, rope_deltas=deltas,
                 logits_to_keep=1, reserve_tokens=row.reserve)
        row.context = list(row.ids) if row.procs else None   # seeded with the prompt (ar.py:1663-1667)
        top = None
        if self.greedy_sampling and not row.procs and not self.top_logprobs_k:
            host = _host_buf(1)
            eng.fetch_tokens(eng.tokens_launched - 1, 1, host)
            eng.stream.synchronize()
            tok = int(host[0])
            lp = self._logprob_of(tok) if self.compute_logprobs else 0.0
        else:   # the row's processors as torch ops over its prompt, as the single-request path runs them
            tok, lp, top = self._sample(out.logits[:, -1, :], row, row.procs)
        row.last_token, row.n_decoded = tok, 1
        row.buffer.append((tok, lp, top))
        if self._lockstep:
            rows.admit(int(cache[0].offset), row.lowered, row.context)
            if self.kv_bits is not None:
                rows.pool.end_admission()
        dt = time.perf_counter() - tic
        self._prompt_tokens_counter += len(row.ids)
        self._prompt_time_counter += dt
        return PromptProgress(uid=row.uid, prompt_tokens=len(row.ids), prompt_time=dt,
                              prompt_tps=len(row.ids) / dt if dt > 0 else 0.0)

    def _prefill_group(self, rows: List[_Row]) -> List[PromptProgress]:
        """`PromptProcessingBatch` (ar.py:1581-2175): the rows admitted together are prefilled in ONE pass over the
        weights (tokens concatenated, block-diagonal causal attention, every token scattered to its own pool row);
        embeddings (vision tower + merge) are still produced per request."""
        lm = self.model.language_model
        tic = time.perf_counter()
        ids_l, emb_l, pos_l, del_l = zip(*[self._embed(row) for row in rows])
        reserve = max(r.reserve for r in rows)
        pool_rows = self._pool_rows(reserve)
        caches = [lm.make_cache_row(pool_rows.pool, pool_rows.B + i) for i in range(len(rows))]
        toks = lm.prefill_rows(list(ids_l), list(emb_l), caches, list(pos_l), list(del_l), reserve_tokens=reserve)
        dt = time.perf_counter() - tic
        out = []
        for row, tok, cache in zip(rows, toks, caches):
            row.last_token, row.n_decoded = tok, 1
            pool_rows.admit(int(cache[0].offset))
            row.buffer.append((tok, 0.0, None))
            self._prompt_tokens_counter += len(row.ids)
            out.append(PromptProgress(uid=row.uid, prompt_tokens=len(row.ids), prompt_time=dt / len(rows),
                                      prompt_tps=len(row.ids) * len(rows) / dt if dt > 0 else 0.0))
        self._prompt_time_counter += dt
        return out

    def _sample(self, logits: torch.Tensor, row: Optional[_Row] = None, procs=None,
                want_top: bool = True) -> Tuple[int, float, Optional[list]]:
        """`procs` (torch ops over the row's token context), logprobs, the sampler and the top-k of one row"""
        # torch ops on the engine's stream: ordered after the step that wrote `logits`
        with torch.cuda.stream(self.model.engine.stream):
            for p in procs or []:
                logits = p(row.context, logits)
            lf = logits.float()
            logprobs = logits - torch.logsumexp(lf, dim=-1, keepdim=True).to(logits.dtype)
            y = (greedy_sampler if self.greedy_sampling or self.sampler is None else self.sampler)(logprobs)
            tok = int(y.reshape(-1)[0].item())
            top = top_logprobs(logprobs, self.top_logprobs_k) if self.top_logprobs_k and want_top else None
            return tok, float(logprobs.reshape(-1)[tok].float().item()), top

    # ------------------------------------------------------------------ lock-step rows
    def _lockstep_slice(self):
        """one slice of lock-step decode steps for every row that still has tokens to compute"""
        eng, rows = self.model.engine, self._rows
        active = self._active
        live = [r.n_decoded < r.max_tokens for r in active]
        if not any(live):
            return
        # rows whose processors do not lower run them as torch ops on their logits row, one step at a time
        host = [a and r.procs is not None and r.lowered is None for r, a in zip(active, live)]
        greedy = self.greedy_sampling and not any(host)
        k = min([self.decode_slice] + [r.max_tokens - r.n_decoded for r, a in zip(active, live) if a]) if greedy else 1
        # greedy: the device feeds each step's tokens to the next; otherwise the host's sampled tokens are uploaded
        rows.top_k = self.top_logprobs_k
        rows.arm(k, [r.last_token for r in active], [r.delta or 0 for r in active], live, fed_back=greedy)
        first = rows.steps
        eng.batch_decode(k, want_logprobs=not self.greedy_sampling)
        rows.advance(k, live)
        B = len(active)
        top_ids = top_lp = None
        if self.top_logprobs_k:
            top_ids = _host_buf(k * B * TOP_LOGPROBS_MAX).view(k, B, TOP_LOGPROBS_MAX)
            top_lp = torch.empty(k, B, TOP_LOGPROBS_MAX, dtype=torch.float32)
            top_lp = top_lp.pin_memory() if torch.cuda.is_available() else top_lp
            eng.batch_fetch_topk(first, k, top_ids, top_lp)

        def device_top(step, b):
            if top_ids is None:
                return None
            n = self.top_logprobs_k
            return list(zip(top_ids[step, b, :n].tolist(), top_lp[step, b, :n].tolist()))

        if self.greedy_sampling:
            toks = _host_buf(k * B).view(k, B)
            lps = torch.empty(k, B, dtype=torch.float32)
            lps = lps.pin_memory() if torch.cuda.is_available() else lps
            eng.batch_fetch(first, k, toks, lps)
        eng.stream.synchronize()
        logits = None if greedy else eng.batch_logits_view("logits")
        for b, (r, a) in enumerate(zip(active, live)):
            if not a:
                continue
            if self.greedy_sampling and not host[b]:   # the device's tokens (its processors applied)
                col = [int(t) for t in toks[:, b].tolist()]
                entries = [(t, float(l), device_top(i, b)) for i, (t, l) in enumerate(zip(col, lps[:, b].tolist()))]
            else:   # the sampler (and a host row's processors) on the row's logits
                entries = []
            # the step's input tokens join the token context before the processors run
            self._generation_batch.record_inputs([(r, [r.last_token] + [t for t, _, _ in entries[:-1]])])
            if not entries:
                tok, lp, top = self._sample(logits[b:b + 1], r, r.procs if host[b] else None, want_top=host[b])
                entries = [(tok, lp, top if host[b] else device_top(0, b))]
            r.buffer.extend(entries)
            r.last_token, r.n_decoded = entries[-1][0], r.n_decoded + len(entries)

    def _decode_slice(self, row: _Row):
        """Refill the row's token buffer: hand the engine to this row for up to `decode_slice`
        steps (device-resident token feedback when greedy)."""
        lm, eng = self.model.language_model, self.model.engine
        left = row.max_tokens - row.n_decoded
        if left <= 0:
            return
        ctx = int(row.cache[0].offset)
        if self.greedy_sampling and not self.compute_logprobs and not row.procs and not self.top_logprobs_k:
            k = min(self.decode_slice, left)
            eng.set_next(row.last_token, ctx, ctx + row.delta)
            base = eng.tokens_launched
            lm.fused_greedy_decode_n(k, row.cache, reserve_tokens=row.reserve)
            host = _host_buf(k)
            eng.fetch_tokens(base, k, host)
            eng.stream.synchronize()
            toks = [int(t) for t in host.tolist()]
            row.buffer.extend((t, 0.0, None) for t in toks)
            row.last_token, row.n_decoded = toks[-1], row.n_decoded + k
        else:
            out = lm(np.asarray([[row.last_token]]), cache=row.cache,
                     rope_deltas=np.asarray([[row.delta]]), reserve_tokens=row.reserve)
            self._generation_batch.record_inputs([(row, [row.last_token])])
            top = None
            if self.greedy_sampling and not row.procs and not self.top_logprobs_k:
                lp = eng.snapshot("logprobs").view(-1)
                with torch.cuda.stream(eng.stream):
                    tok = int(torch.argmax(lp.float()).item())
                    lpv = float(lp[tok].float().item())
            else:
                tok, lpv, top = self._sample(out.logits[:, -1, :], row, row.procs)
            row.buffer.append((tok, lpv, top))
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
                tok, lp, top = row.buffer.pop(0)
                row.n_tokens += 1
                finish = None
                if stop(tok):
                    finish = "stop"
                elif row.n_tokens >= row.max_tokens:
                    finish = "length"
                generation_responses.append(GenerationBatch.Response(
                    uid=row.uid, token=tok, token_logprob=lp, finish_reason=finish, top_logprobs=top))
                if finish is None:
                    keep.append(i)
            self._gen_tokens_counter += len(self._active)
            self._gen_time_counter += time.perf_counter() - tic
            if len(keep) < len(self._generation_batch):
                self._keep(keep)
        # 2. admit waiting prompts while there is room (shortest first)
        room = self.completion_batch_size - len(self._active)
        n_new = min(room, self.prefill_batch_size, len(self._unprocessed_sequences))
        admitted = []
        # kv_bits=8 rows are admitted one at a time (the grouped prefill has no 8-bit write-through)
        group = (self._lockstep and n_new >= 2 and self.greedy_sampling and not self.compute_logprobs
                 and self.kv_bits is None and not self.top_logprobs_k
                 and not any(r.procs for r in self._unprocessed_sequences[:n_new])
                 and hasattr(self.model.language_model, "prefill_rows") and self.batched_prefill
                 and (self.prefill_step_size is None
                      or all(len(r.ids) <= self.prefill_step_size + 1 for r in self._unprocessed_sequences[:n_new])))
        if group:
            admitted = [self._unprocessed_sequences.pop(0) for _ in range(n_new)]
            prompt_responses.extend(self._prefill_group(admitted))
        for _ in range(0 if group else max(0, n_new)):
            row = self._unprocessed_sequences.pop(0)
            prompt_responses.append(self._prefill(row))
            admitted.append(row)
        if admitted:
            self._generation_batch.extend(GenerationBatch.admitted(admitted))
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
    # the request's penalties and logit bias become every row's processors (ar.py:2890-3097, make_logits_processors)
    from .sample_utils import make_logits_processors
    procs = make_logits_processors(kwargs.pop("logit_bias", None), kwargs.pop("repetition_penalty", None),
                                   kwargs.pop("repetition_context_size", 20), kwargs.pop("presence_penalty", None),
                                   kwargs.pop("presence_context_size", 20), kwargs.pop("frequency_penalty", None),
                                   kwargs.pop("frequency_context_size", 20))
    procs += list(kwargs.pop("logits_processors", None) or [])
    gen = BatchGenerator(model, processor, max_tokens=max_tokens if isinstance(max_tokens, int) else DEFAULT_MAX_TOKENS,
                         logits_processors=procs or None, **kwargs)
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
