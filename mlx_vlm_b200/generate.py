"""Generation API with the reference's surface
(mlx_vlm/generate/ar.py:151-515 `generate_step`; generate/dispatch.py:694-1105
`stream_generate`, :1108-1228 `generate`; generate/common.py:216-263
`GenerationResult`, `PromptCacheState`).

Scheduling mirrors the reference: the step for token n+1 is enqueued BEFORE token
n is read on the host (`mx.async_eval`, ar.py:476,500 -> here: the decode-step
CUDA graph is launched, then an event on the previous step's 4-byte token copy is
waited on).  With the greedy sampler and no logits processors the token feedback
never leaves the device.
"""
from __future__ import annotations

import time
from dataclasses import dataclass
from typing import Any, Callable, Dict, Generator, List, Optional, Tuple, Union

import numpy as np
import torch

from .models import cache as cache_mod
from .sample_utils import make_logits_processors, make_sampler

DEFAULT_MAX_TOKENS = 2048
DEFAULT_TEMPERATURE = 0.0
DEFAULT_TOP_P = 1.0
DEFAULT_TOP_K = 0
DEFAULT_MIN_P = 0.0
DEFAULT_TOP_N_SIGMA = 0.0
DEFAULT_REPETITION_CONTEXT_SIZE = 20
DEFAULT_PREFILL_STEP_SIZE = 2048
DEFAULT_SEED = 0
DEFAULT_KV_GROUP_SIZE = 64
DEFAULT_QUANTIZED_KV_START = 5000


@dataclass
class GenerationResult:
    text: str = ""
    token: Optional[int] = None
    logprobs: Optional[Any] = None
    prompt_tokens: int = 0
    generation_tokens: int = 0
    total_tokens: int = 0
    prompt_tps: float = 0.0
    generation_tps: float = 0.0
    peak_memory: float = 0.0
    cached_tokens: int = 0
    finish_reason: Optional[str] = None


class PromptCacheState:
    """generate/common.py:243-263."""

    def __init__(self):
        self.cache: Optional[List[Any]] = None
        self.token_ids: Optional[List[int]] = None

    def find_prefix_length(self, new_ids: list) -> int:
        if self.token_ids is None:
            return 0
        max_len = min(len(self.token_ids), len(new_ids))
        for i in range(max_len):
            if self.token_ids[i] != new_ids[i]:
                return i
        return max_len

    def update(self, token_ids: list, kv_cache: list):
        self.token_ids = list(token_ids)
        self.cache = kv_cache


_UNSUPPORTED = ("max_kv_size", "kv_key_bits", "kv_value_bits", "draft_model")


def kv_quant_args(kv_bits, kv_group_size, kv_quant_scheme, head_dim: int):
    """Validate the KV-quantization kwargs: returns the bit width (None: bf16 cache).  Only the uniform 8-bit
    scheme is built; other widths and schemes raise NotImplementedError, a bad group size ValueError."""
    if kv_bits is None:
        return None
    if kv_bits != 8:
        raise NotImplementedError(f"kv_bits={kv_bits}: only the uniform 8-bit KV cache is built")
    if kv_quant_scheme not in (None, "uniform"):
        raise NotImplementedError(f"kv_quant_scheme={kv_quant_scheme!r}: only the uniform scheme is built")
    if kv_group_size not in (32, 64, 128) or head_dim % kv_group_size:
        raise ValueError(f"kv_group_size={kv_group_size}: must be 32, 64 or 128 and divide head_dim={head_dim}")
    return 8


def maybe_quantize_kv_cache(prompt_cache, quantized_kv_start, kv_group_size, kv_bits,
                            kv_quant_scheme: str = "uniform", kv_key_bits=None, kv_value_bits=None,
                            kv_key_scheme=None, kv_value_scheme=None):
    """generate/common.py:77-183, uniform branch: every layer whose offset reached `quantized_kv_start` is
    replaced by its 8-bit form.  The layers of a request share one pool: once all of them are converted the
    bf16 pool is released (the replaced bf16 views are empty afterwards)."""
    if kv_bits is None:
        return
    if kv_key_bits is not None or kv_value_bits is not None or kv_key_scheme is not None or \
            kv_value_scheme is not None:
        raise NotImplementedError("per-side KV quantization (kv_key_bits / kv_value_bits / schemes) is not built")
    pools = set()
    for index, layer_cache in enumerate(prompt_cache):
        if hasattr(layer_cache, "to_quantized") and layer_cache.offset >= quantized_kv_start:
            prompt_cache[index] = layer_cache.to_quantized(group_size=kv_group_size, bits=int(kv_bits))
            pools.add(layer_cache._pool)
    for pool in pools:
        if pool is not None and not any(getattr(c, "_pool", None) is pool for c in prompt_cache):
            pool.buf = None
            pool.__dict__.pop("_q8", None)


def generate_step(
    input_ids,
    model,
    pixel_values,
    mask,
    *,
    max_tokens: int = DEFAULT_MAX_TOKENS,
    temperature: float = DEFAULT_TEMPERATURE,
    repetition_penalty: Optional[float] = None,
    repetition_context_size: Optional[int] = DEFAULT_REPETITION_CONTEXT_SIZE,
    presence_penalty: Optional[float] = None,
    presence_context_size: Optional[int] = DEFAULT_REPETITION_CONTEXT_SIZE,
    frequency_penalty: Optional[float] = None,
    frequency_context_size: Optional[int] = DEFAULT_REPETITION_CONTEXT_SIZE,
    top_p: float = DEFAULT_TOP_P,
    min_p: float = DEFAULT_MIN_P,
    top_k: int = DEFAULT_TOP_K,
    top_n_sigma: float = DEFAULT_TOP_N_SIGMA,
    p_less: bool = False,
    typical_p: float = 1.0,
    logit_bias: Optional[Dict[int, float]] = None,
    prompt_cache: Optional[List[Any]] = None,
    sampler: Optional[Callable] = None,
    logits_processors: Optional[List[Callable]] = None,
    prefill_step_size: Optional[int] = DEFAULT_PREFILL_STEP_SIZE,
    seed: Optional[int] = None,
    verbose: bool = False,
    return_logprobs: bool = True,
    **kwargs,
) -> Generator[Tuple[int, Any], None, None]:
    """Yields (token id, logprobs (vocab,) bf16 device tensor) like ar.py:151-515."""
    for k in _UNSUPPORTED:
        if kwargs.pop(k, None) is not None:
            raise NotImplementedError(f"generate_step: `{k}` is outside this engine's hot-path scope")
    kv_bits = kwargs.pop("kv_bits", None)
    kv_group_size = kwargs.pop("kv_group_size", DEFAULT_KV_GROUP_SIZE)
    kv_quant_scheme = kwargs.pop("kv_quant_scheme", None)
    quantized_kv_start = kwargs.pop("quantized_kv_start", DEFAULT_QUANTIZED_KV_START)
    if kv_bits is not None:
        kv_bits = kv_quant_args(kv_bits, kv_group_size, kv_quant_scheme, model.language_model.head_dim)
    for k in ("kv_key_scheme", "kv_value_scheme", "draft_kind", "draft_block_size", "prompt_cache_checkpoint",
              "prompt_cache_checkpoint_len", "thinking_budget_criteria"):
        kwargs.pop(k, None)
    if seed is not None:
        torch.manual_seed(seed)

    sampler_is_greedy = (sampler is None and temperature == 0) or getattr(sampler, "is_greedy", False)
    if sampler is None:
        sampler = make_sampler(temp=temperature, top_p=top_p, min_p=min_p, top_k=top_k,
                               top_n_sigma=top_n_sigma, p_less=p_less, typical_p=typical_p)
    processors = make_logits_processors(logit_bias, repetition_penalty, repetition_context_size,
                                        presence_penalty, presence_context_size,
                                        frequency_penalty, frequency_context_size)
    if logits_processors is not None:
        processors.extend(logits_processors)

    lm = model.language_model
    eng = model.engine
    if prompt_cache is None:
        prompt_cache = cache_mod.make_prompt_cache(lm)

    embedding_output = model.get_input_embeddings(input_ids, pixel_values, mask=mask, **kwargs)
    inputs_embeds = embedding_output.inputs_embeds
    kwargs.update({k: v for k, v in embedding_output.to_dict().items()
                   if k != "inputs_embeds" and v is not None})
    ids_host = input_ids.cpu().numpy() if isinstance(input_ids, torch.Tensor) else np.asarray(input_ids)
    if ids_host.ndim == 1:
        ids_host = ids_host[None]
    T = inputs_embeds.shape[1]
    reserve = int(prompt_cache[0].offset) + T + max_tokens + 1
    step_kwargs = dict(kwargs)
    if getattr(lm, "supports_logits_to_keep", False):
        step_kwargs["logits_to_keep"] = 1

    def quantize_policy():
        # ar.py:366,457: after every forward
        maybe_quantize_kv_cache(prompt_cache, quantized_kv_start, kv_group_size, kv_bits)

    # ---- prefill (chunked above prefill_step_size, ar.py:426-472) ----
    if prefill_step_size is not None and T > prefill_step_size:
        while inputs_embeds.shape[1] > 1:
            n = min(prefill_step_size, inputs_embeds.shape[1] - 1)
            lm(ids_host[:, :n], inputs_embeds=inputs_embeds[:, :n], cache=prompt_cache,
               n_to_process=n, reserve_tokens=reserve, **step_kwargs)
            quantize_policy()
            inputs_embeds = inputs_embeds[:, n:]
            ids_host = ids_host[:, n:]
        ids_host = ids_host[:, -1:]
    outputs = lm(ids_host, inputs_embeds=inputs_embeds, cache=prompt_cache,
                 reserve_tokens=reserve, **step_kwargs)
    quantize_policy()

    fast = sampler_is_greedy and not processors
    if fast:
        yield from _greedy_device_loop(eng, lm, prompt_cache, max_tokens, reserve, return_logprobs,
                                       quantize_policy if kv_bits is not None else None)
        return

    # ---- general path: torch samplers / logits processors on the ENGINE's stream ----
    # The engine enqueues its kernels and the logits copy on `eng.stream` (non-blocking); every
    # torch op that touches those logits runs inside `torch.cuda.stream(eng.stream)` so it is
    # stream-ordered after the step that produced them, and `.item()` synchronises that stream.
    # The stream context never spans a `yield`.
    # Token history of the processors (ar.py:357-361): the reference concatenates the ids fed to
    # EVERY `_step`, so it starts with the prompt (its last chunk) and then holds each fed token.
    tokens: List[int] = [int(t) for t in np.asarray(ids_host).reshape(-1)] if processors else []

    def _sample(logits):
        with torch.cuda.stream(eng.stream):
            for p in processors:
                logits = p(tokens, logits)
            lf = logits.float()
            logprobs = (logits - torch.logsumexp(lf, dim=-1, keepdim=True).to(logits.dtype))
            y = sampler(logprobs)
            tok = int(y.reshape(-1)[0].item())   # synchronises eng.stream
        return tok, logprobs

    logits = outputs.logits[:, -1, :]
    n = 0
    while n < max_tokens:
        tok, logprobs = _sample(logits)
        yield tok, logprobs.squeeze(0)
        n += 1
        if n == max_tokens:
            break
        if processors:
            tokens.append(tok)
        outputs = lm(np.asarray([[tok]]), cache=prompt_cache, reserve_tokens=reserve)
        quantize_policy()
        logits = outputs.logits[:, -1, :]


def _greedy_device_loop(eng, lm, prompt_cache, max_tokens, reserve, return_logprobs, after_step=None):
    """Decode loop with device-resident token feedback, one step ahead of the host.  `after_step` runs after
    every enqueued step (the KV quantization policy: stream-ordered, no host synchronisation)."""
    if max_tokens <= 0:
        return
    host = torch.empty(max_tokens + 2, dtype=torch.int32).pin_memory()
    base = eng.tokens_launched - 1  # log index of the token sampled by the prefill call
    events = [torch.cuda.Event() for _ in range(max_tokens + 1)]
    lp = eng.snapshot("logprobs") if return_logprobs else None
    eng.fetch_tokens(base, 1, host[0:1])
    events[0].record(eng.stream)
    n = 0
    while True:
        next_lp = None
        if n != max_tokens:
            lm.fused_greedy_decode_n(1, prompt_cache, reserve_tokens=reserve)
            if after_step is not None:
                after_step()
            next_lp = eng.snapshot("logprobs") if return_logprobs else None
            eng.fetch_tokens(base + n + 1, 1, host[n + 1:n + 2])
            events[n + 1].record(eng.stream)
        if n == max_tokens:
            break
        events[n].synchronize()
        yield int(host[n]), lp
        lp = next_lp
        n += 1


def stream_generate(model, processor, prompt: str, image: Union[str, List[str], Any] = None,
                    audio=None, video=None, **kwargs) -> Generator[GenerationResult, None, None]:
    """generate/dispatch.py:694-1105 (vision/text requests; audio/video out of scope)."""
    from .utils import StoppingCriteria, prepare_inputs
    if audio is not None or video is not None:
        raise NotImplementedError("audio / video inputs are outside this engine's hot-path scope")
    tokenizer = processor.tokenizer if hasattr(processor, "tokenizer") else processor
    skip_special_token_ids = (set(getattr(tokenizer, "all_special_ids", []))
                              if kwargs.pop("skip_special_tokens", False) else set())
    prompt_cache_state: Optional[PromptCacheState] = kwargs.pop("prompt_cache_state", None)
    vision_cache = kwargs.pop("vision_cache", None)
    eos_tokens = kwargs.pop("eos_tokens", None)
    if not hasattr(tokenizer, "stopping_criteria") or tokenizer.stopping_criteria is None:
        eos = getattr(model.config, "eos_token_id", None)
        if eos is None:
            eos = getattr(tokenizer, "eos_token_id", None)
        tokenizer.stopping_criteria = StoppingCriteria(eos if eos is not None else [], tokenizer)
    if eos_tokens is not None:
        tokenizer.stopping_criteria.add_eos_token_ids(eos_tokens)

    input_ids = kwargs.pop("input_ids", None)
    pixel_values = kwargs.pop("pixel_values", None)
    mask = kwargs.pop("mask", None)
    resize_shape = kwargs.pop("resize_shape", None)
    if input_ids is None:
        inputs = prepare_inputs(processor, images=image, prompts=prompt, resize_shape=resize_shape,
                                device=model.engine.device, stream=model.engine.stream)
        input_ids = inputs.pop("input_ids")
        pixel_values = inputs.pop("pixel_values", None)
        mask = inputs.pop("attention_mask", None)
        kwargs.update({k: v for k, v in inputs.items() if v is not None})
    ids_list = np.asarray(input_ids.cpu() if isinstance(input_ids, torch.Tensor) else input_ids
                          ).reshape(-1).tolist()

    # vision feature reuse across turns (dispatch.py:800-809): a hit is handed to the model as
    # `cached_image_features`; a miss is filled only by models that expose `encode_image`
    # (Qwen2-VL does not, in the reference either)
    if vision_cache is not None and image is not None and pixel_values is not None:
        cached = vision_cache.get(image)
        if cached is not None:
            kwargs["cached_image_features"] = cached
        elif hasattr(model, "encode_image"):
            features = model.encode_image(pixel_values)
            vision_cache.put(image, features)
            kwargs["cached_image_features"] = features

    # prefix reuse across turns (dispatch.py:861-882): trim the cached KV to the
    # common prefix and only prefill the new suffix (text-only suffixes).
    reused = 0
    if prompt_cache_state is not None and prompt_cache_state.cache is not None and pixel_values is None:
        reused = prompt_cache_state.find_prefix_length(ids_list)
        reused = min(reused, len(ids_list) - 1)
        pc = prompt_cache_state.cache
        if reused > 0 and all(c.is_trimmable() for c in pc):
            extra = pc[0].offset - reused
            if extra >= 0:
                for c in pc:
                    c.trim(extra)
                kwargs["prompt_cache"] = pc
                input_ids = np.asarray([ids_list[reused:]])
            else:
                reused = 0
        else:
            reused = 0
    if "prompt_cache" not in kwargs:
        kwargs["prompt_cache"] = cache_mod.make_prompt_cache(model.language_model)
    tracked_cache = kwargs["prompt_cache"]
    total_prompt_tokens = len(ids_list)

    detokenizer = _make_detokenizer(processor)
    gen = generate_step(input_ids, model, pixel_values, mask, **kwargs)
    tic = time.perf_counter()
    generated: List[int] = []
    finish_reason = None
    prompt_tps = 0.0
    token, logprobs, n = None, None, -1
    for n, (token, logprobs) in enumerate(gen):
        if n == 0:
            prompt_time = time.perf_counter() - tic
            prompt_tps = total_prompt_tokens / prompt_time
            tic = time.perf_counter()
        generated.append(token)
        if tokenizer.stopping_criteria(token):
            finish_reason = "stop"
            break
        detokenizer.add_token(token, skip_special_token_ids=skip_special_token_ids)
        yield GenerationResult(
            text=detokenizer.last_segment, token=token, logprobs=logprobs,
            prompt_tokens=total_prompt_tokens, generation_tokens=n + 1,
            total_tokens=total_prompt_tokens + n + 1, prompt_tps=prompt_tps,
            generation_tps=(n + 1) / (time.perf_counter() - tic),
            peak_memory=torch.cuda.max_memory_allocated(model.engine.device) / 1e9,
            cached_tokens=reused)
    else:
        finish_reason = "length"
    if not generated:
        prompt_time = time.perf_counter() - tic
        yield GenerationResult(prompt_tokens=total_prompt_tokens, total_tokens=total_prompt_tokens,
                               prompt_tps=total_prompt_tokens / prompt_time if prompt_time > 0 else 0.0,
                               finish_reason="length", cached_tokens=reused)
        return
    detokenizer.finalize()
    yield GenerationResult(
        text=detokenizer.last_segment, token=token, logprobs=logprobs,
        prompt_tokens=total_prompt_tokens, generation_tokens=n + 1,
        total_tokens=total_prompt_tokens + n + 1, prompt_tps=prompt_tps,
        generation_tps=(n + 1) / (time.perf_counter() - tic),
        peak_memory=torch.cuda.max_memory_allocated(model.engine.device) / 1e9,
        cached_tokens=reused, finish_reason=finish_reason)
    if prompt_cache_state is not None:
        prompt_cache_state.update(ids_list + generated, tracked_cache)


def generate(model, processor, prompt: str, image=None, audio=None, video=None,
             verbose: bool = False, **kwargs) -> GenerationResult:
    """generate/dispatch.py:1108-1228: run stream_generate to completion."""
    tokenizer = processor.tokenizer if hasattr(processor, "tokenizer") else processor
    sc = getattr(tokenizer, "stopping_criteria", None)
    if sc is not None and hasattr(sc, "reset"):
        eos = getattr(model.config, "eos_token_id", None)
        if eos is not None:
            sc.reset(eos)
    text = ""
    last = None
    for resp in stream_generate(model, processor, prompt, image, audio, video, **kwargs):
        text += resp.text
        if verbose:
            print(resp.text, end="", flush=True)
        last = resp
    if last is None:
        return GenerationResult()
    if verbose:
        print("\n" + "=" * 10)
        print(f"Prompt: {last.prompt_tokens} tokens, {last.prompt_tps:.3f} tokens-per-sec")
        print(f"Generation: {last.generation_tokens} tokens, {last.generation_tps:.3f} tokens-per-sec")
        print(f"Peak memory: {last.peak_memory:.3f} GB")
    return GenerationResult(
        text=text, token=last.token, logprobs=last.logprobs, prompt_tokens=last.prompt_tokens,
        generation_tokens=last.generation_tokens, total_tokens=last.total_tokens,
        prompt_tps=last.prompt_tps, generation_tps=last.generation_tps,
        peak_memory=last.peak_memory, cached_tokens=last.cached_tokens,
        finish_reason=last.finish_reason)


# --------------------------------------------------------------------------
class _NaiveDetokenizer:
    """Streaming detokenizer with the reference's observable behaviour (tokenizer_utils.py:48-118,
    `StreamingDetokenizer.last_segment` + `NaiveStreamingDetokenizer`; pinned by the golden trace
    `detokenizer_trace`): the pending tokens are re-decoded on every read and folded into the
    settled text at a newline; a segment is only released when the text does not end in an
    incomplete UTF-8 sequence (U+FFFD)."""

    _REPLACEMENT = "\ufffd"

    def __init__(self, tokenizer):
        self._tok = tokenizer
        self.reset()

    def reset(self):
        self.offset = 0
        self._settled_tokens: List[int] = []
        self._settled_text = ""
        self._pending: List[int] = []
        self._pending_text = ""

    def add_token(self, token, skip_special_token_ids=()):
        if token not in skip_special_token_ids:
            self._pending.append(token)

    def _settle(self, text: str):
        self._settled_tokens.extend(self._pending)
        self._settled_text += text
        self._pending = []
        self._pending_text = ""

    def finalize(self):
        self._settle(self._tok.decode(self._pending))

    @property
    def text(self) -> str:
        if self._pending:
            self._pending_text = self._tok.decode(self._pending)
        if self._pending_text.endswith("\n"):
            self._settle(self._pending_text)
        return self._settled_text + self._pending_text

    @property
    def tokens(self) -> List[int]:
        return self._settled_tokens

    @property
    def last_segment(self) -> str:
        text = self.text
        if not text or text.endswith(self._REPLACEMENT):
            return ""
        seg = text[self.offset:]
        self.offset = len(text)
        return seg


def _make_detokenizer(processor):
    d = getattr(processor, "detokenizer", None)
    if d is not None:
        d.reset()
        return d
    tokenizer = processor.tokenizer if hasattr(processor, "tokenizer") else processor
    return _NaiveDetokenizer(tokenizer)
