"""The server's GPU-thread loop (reference mlx_vlm/server/generation.py:1730-1918, `ResponseGenerator`):
ONE thread owns the engine and its `BatchGenerator`; caller threads tokenise / preprocess on their own
and hand over a request; the loop admits waiting requests between decode steps (continuous batching),
runs the vision tower for a new request on the GPU thread (`_gpu_embed`, generation.py:1636-1675),
streams every generated token back through the request's own queue, honours cancellation and a
`max_num_seqs` admission cap (back-pressure: the rest stay queued), and reports an engine error to every
request it affects.  The HTTP / OpenAI front end is outside the hot-path scope (SURVEY section 8(f2): the
loop is the part that touches the path); `ResponseGenerator.generate()` is what such a front end calls.

Differences from the reference, by design: no speculative / diffusion / APC branches (out of scope), the
sampler is the engine's fused greedy sampler unless a request asks for temperature > 0 (then the batch
falls back to the time-multiplexed sampler path of `BatchGenerator`)."""
from __future__ import annotations

import queue
import threading
from dataclasses import dataclass, field
from typing import Any, Dict, Iterator, List, Optional, Tuple

import numpy as np

from .generate_batch import TOP_LOGPROBS_MAX, BatchGenerator


@dataclass
class GenerationArguments:
    max_tokens: int = 256
    temperature: float = 0.0
    logprobs: bool = False
    top_logprobs: int = 0          # capped to [0, 20] as the reference server caps it (get_top_logprobs_k)
    repetition_penalty: Optional[float] = None
    repetition_context_size: int = 20
    presence_penalty: Optional[float] = None
    presence_context_size: int = 20
    frequency_penalty: Optional[float] = None
    frequency_context_size: int = 20
    logit_bias: Optional[Dict[int, float]] = None

    def logits_processors(self) -> list:
        """the request's penalties and logit bias as processors (server/generation.py:689-761)"""
        from .sample_utils import make_logits_processors
        bias = {int(k): float(v) for k, v in self.logit_bias.items()} if self.logit_bias else None
        return make_logits_processors(bias, self.repetition_penalty, self.repetition_context_size,
                                      self.presence_penalty, self.presence_context_size, self.frequency_penalty,
                                      self.frequency_context_size)

    def top_k(self) -> int:
        return max(0, min(int(self.top_logprobs or 0), TOP_LOGPROBS_MAX))


@dataclass
class GenerationContext:
    """first item a request receives (generation.py `GenerationContext`): its uid and prompt length"""
    uid: int
    prompt_tokens: int


@dataclass
class TokenEvent:
    token: int
    logprob: float
    finish_reason: Optional[str]
    text: str = ""
    top_logprobs: Optional[List[Tuple[int, float]]] = None


@dataclass
class _Request:
    raw_inputs: Dict[str, Any]
    args: GenerationArguments
    images: Any = None
    rqueue: "queue.Queue" = field(default_factory=queue.Queue)
    cancelled: threading.Event = field(default_factory=threading.Event)


class ResponseGenerator:
    def __init__(self, model, processor, *, max_num_seqs: Optional[int] = 16, vision_cache=None,
                 completion_batch_size: int = 16, prefill_batch_size: int = 8, decode_slice: int = 8,
                 idle_timeout: float = 0.05, batch_generator_factory=None, start: bool = True):
        self.model, self.processor = model, processor
        self.max_num_seqs = max_num_seqs
        self.vision_cache = vision_cache
        self.completion_batch_size = completion_batch_size
        self.prefill_batch_size = prefill_batch_size
        self.decode_slice = decode_slice
        self.idle_timeout = idle_timeout
        self._factory = batch_generator_factory
        self.requests: "queue.Queue[Optional[_Request]]" = queue.Queue()
        self._stop = False
        self._ready = threading.Event()
        self._error: Optional[BaseException] = None
        self.steps = 0
        self.peak_active = 0
        self._thread = threading.Thread(target=self._run, name="b200-generation", daemon=True)
        if start:
            self._thread.start()

    # ------------------------------------------------------------------ caller side
    def submit(self, raw_inputs: Dict[str, Any], args: Optional[GenerationArguments] = None, images=None) -> _Request:
        """queue a request prepared on the caller's thread (`prepare_inputs` output: input_ids +
        pixel_values / image_grid_thw / ...); returns the handle whose `rqueue` receives a
        GenerationContext, then TokenEvents, then None"""
        if self._stop:
            raise RuntimeError("ResponseGenerator is stopped")
        req = _Request(raw_inputs=dict(raw_inputs), args=args or GenerationArguments(), images=images)
        self.requests.put(req)
        return req

    def generate(self, raw_inputs, args: Optional[GenerationArguments] = None, images=None,
                 timeout: Optional[float] = 120.0) -> Iterator[TokenEvent]:
        """blocking iterator over one request's tokens (what an HTTP handler streams)"""
        req = self.submit(raw_inputs, args, images)
        try:
            while True:
                item = req.rqueue.get(timeout=timeout)
                if item is None:
                    return
                if isinstance(item, BaseException):
                    raise item
                if isinstance(item, GenerationContext):
                    continue
                yield item
                if item.finish_reason is not None:
                    return
        finally:
            req.cancelled.set()     # a consumer that walks away frees its row at the next step

    def cancel(self, req: _Request):
        req.cancelled.set()

    def stop_and_join(self, timeout: float = 30.0):
        self._stop = True
        self.requests.put(None)
        self._thread.join(timeout)

    # ------------------------------------------------------------------ GPU thread
    def _gpu_embed(self, req: _Request):
        """vision tower + merge on the GPU thread; the embeddings travel to BatchGenerator as prompt kwargs"""
        raw = req.raw_inputs
        ids = raw.get("input_ids")
        pv = raw.get("pixel_values")
        data = {k: v for k, v in raw.items() if k not in ("input_ids", "pixel_values", "attention_mask")}
        extra = {}
        if pv is not None and self.vision_cache is not None and req.images is not None:
            hit = self.vision_cache.get(req.images)
            if hit is not None:
                extra["cached_image_features"] = hit
            elif hasattr(self.model, "encode_image"):
                feats = self.model.encode_image(pv)
                self.vision_cache.put(req.images, feats)
                extra["cached_image_features"] = feats
        emb = self.model.get_input_embeddings(ids, pv, mask=raw.get("attention_mask"), **data, **extra)
        kw = dict(data)
        kw.update({k: v for k, v in emb.to_dict().items() if v is not None})
        return np.asarray(ids).reshape(-1).tolist(), kw

    def _collect(self, active: bool, capacity: Optional[int]) -> (List[_Request], bool):
        got, stop = [], False

        def take(item):
            nonlocal stop
            if item is None:
                stop = self._stop
            else:
                got.append(item)

        room = lambda: capacity is None or len(got) < capacity   # noqa: E731
        try:
            if active:
                if room():
                    take(self.requests.get_nowait())
            else:
                take(self.requests.get(timeout=self.idle_timeout))
        except queue.Empty:
            pass
        while not stop and room():
            try:
                take(self.requests.get_nowait())
            except queue.Empty:
                break
        return got, stop

    def _make_batch_generator(self, args: GenerationArguments):
        if self._factory is not None:
            return self._factory(args)
        sampler = None
        if args.temperature > 0:
            from .sample_utils import make_sampler
            sampler = make_sampler(temp=args.temperature)
        return BatchGenerator(self.model, self.processor, sampler=sampler, compute_logprobs=bool(args.logprobs),
                              completion_batch_size=self.completion_batch_size,
                              prefill_batch_size=self.prefill_batch_size, decode_slice=self.decode_slice,
                              greedy_sampling=args.temperature == 0)

    def _run(self):
        gen = None
        active: Dict[int, _Request] = {}
        self._ready.set()
        while not (self._stop and not active and self.requests.empty()):
            new: List[_Request] = []
            try:
                cap = None if self.max_num_seqs is None else max(0, self.max_num_seqs - len(active))
                new, should_stop = self._collect(bool(active), cap)
                if should_stop and not active and not new:
                    break
                # abandoned requests free their rows before more work is done
                for uid in [u for u, r in active.items() if r.cancelled.is_set()]:
                    gen.remove(uid)
                    active.pop(uid).rqueue.put(None)
                for req in new:
                    if req.cancelled.is_set():
                        req.rqueue.put(None)
                        continue
                    if gen is None:
                        gen = self._make_batch_generator(req.args)
                    try:
                        ids, kw = self._gpu_embed(req)
                        procs = req.args.logits_processors()
                        (uid,) = gen.insert([ids], max_tokens=req.args.max_tokens, prompt_kwargs=[kw],
                                            logits_processors=[procs or None])
                    except Exception as e:     # a bad request must not take the loop down
                        req.rqueue.put(e)
                        continue
                    req.rqueue.put(GenerationContext(uid=uid, prompt_tokens=len(ids)))
                    active[uid] = req
                self.peak_active = max(self.peak_active, len(active))
                if not active or gen is None:
                    continue
                if hasattr(gen, "top_logprobs_k"):   # the widest top_logprobs any active request asks for
                    gen.top_logprobs_k = max(r.args.top_k() for r in active.values())
                _, responses = gen.next()
                self.steps += 1
                for r in responses:
                    req = active.get(r.uid)
                    if req is None:
                        continue
                    k = req.args.top_k()
                    top = getattr(r, "top_logprobs", None)
                    req.rqueue.put(TokenEvent(token=int(r.token), logprob=float(r.token_logprob),
                                              finish_reason=r.finish_reason,
                                              top_logprobs=list(top[:k]) if k and top else None))
                    if r.finish_reason is not None:
                        active.pop(r.uid)
                        req.rqueue.put(None)
                if gen is not None and not gen.has_work and not active:
                    gen.close()
                    gen = None
            except Exception as e:             # engine error: every request it touches hears about it
                self._error = e
                for req in list(active.values()) + [r for r in new if r not in active.values()]:
                    req.rqueue.put(e)
                    req.rqueue.put(None)
                active.clear()
                gen = None
        if gen is not None:
            gen.close()
