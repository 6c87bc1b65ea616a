"""Samplers and logits processors with the reference's API
(mlx_vlm/sample_utils.py: make_sampler :10-89, make_logits_processors :92-146,
apply_top_k :149-175, apply_top_n_sigma :178-211, apply_p_less :214-231,
apply_min_p :234-286, apply_top_p :289-318, apply_typical_p :321-347, apply_xtc
:350-386, categorical_sampling :385-387, penalties :390-475, top_p_sampling :478).

The benchmarked sampler is greedy (`temp == 0`), which the CUDA step kernel fuses
(k_sample: logprobs + lowest-index argmax).  The functions here serve the other
sampling modes; they operate on device tensors with torch tensor ops (API-parity
code, off the measured path).
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional

import torch


def make_sampler(temp: float = 0.0, top_p: float = 0.0, min_p: float = 0.0,
                 min_tokens_to_keep: int = 1, top_k: int = 0, top_n_sigma: float = 0.0,
                 p_less: bool = False, typical_p: float = 1.0, xtc_probability: float = 0.0,
                 xtc_threshold: float = 0.0, xtc_special_tokens: Optional[List[int]] = None,
                 ) -> Callable[[torch.Tensor], torch.Tensor]:
    if xtc_special_tokens is None:
        xtc_special_tokens = []
    if temp == 0:
        return greedy_sampler
    methods = []
    if top_n_sigma > 0.0:
        methods.append(lambda x: apply_top_n_sigma(x, top_n_sigma))
    if p_less:
        methods.append(lambda x: apply_p_less(x, temp))
    if 0.0 < typical_p < 1.0:
        methods.append(lambda x: apply_typical_p(x, typical_p))
    if 0 < top_p < 1.0:
        methods.append(lambda x: apply_top_p(x, top_p))
    if min_p != 0.0:
        methods.append(lambda x: apply_min_p(x, min_p, min_tokens_to_keep))
    if xtc_probability > 0.0:
        methods.append(lambda x: apply_xtc(x, xtc_probability, xtc_threshold, xtc_special_tokens))
    if top_k > 0:
        methods.append(lambda x: apply_top_k(x, top_k))

    def sampler(logprobs):
        for m in methods:
            logprobs = m(logprobs)
        return categorical_sampling(logprobs, temp)

    return sampler


def greedy_sampler(x: torch.Tensor) -> torch.Tensor:
    """mx.argmax(x, axis=-1): first maximum (lowest index on ties)."""
    m = x.max(dim=-1, keepdim=True).values
    idx = torch.arange(x.shape[-1], device=x.device).expand_as(x)
    return torch.where(x == m, idx, torch.full_like(idx, x.shape[-1])).min(dim=-1).values


greedy_sampler.is_greedy = True  # lets generate_step route to the fused CUDA sampler


def make_logits_processors(logit_bias: Optional[Dict[int, float]] = None,
                           repetition_penalty: Optional[float] = None,
                           repetition_context_size: Optional[int] = 20,
                           presence_penalty: Optional[float] = None,
                           presence_context_size: Optional[int] = 20,
                           frequency_penalty: Optional[float] = None,
                           frequency_context_size: Optional[int] = 20):
    procs = []
    if logit_bias:
        keys = list(logit_bias.keys())
        vals = list(logit_bias.values())

        def logit_bias_processor(_, logits):
            idx = torch.tensor(keys, device=logits.device)
            v = torch.tensor(vals, device=logits.device, dtype=logits.dtype)
            out = logits.clone()
            out[:, idx] += v
            return out

        logit_bias_processor.lowered = ("bias", dict(zip(keys, vals)))
        procs.append(logit_bias_processor)
    for make, pen, ctx in ((make_repetition_penalty, repetition_penalty, repetition_context_size),
                           (make_presence_penalty, presence_penalty, presence_context_size),
                           (make_frequency_penalty, frequency_penalty, frequency_context_size)):
        if pen is not None and pen != 0:
            procs.append(make(pen, ctx))
    return procs


def top_logprobs(logprobs: torch.Tensor, k: int):
    """[(token id, logprob)] of the k largest entries of a (vocab,) logprob row, largest first, the lower token id
    first among equal logprobs (the order of the lock-step batch's top-k kernel)."""
    v, i = torch.sort(logprobs.reshape(-1).float(), descending=True, stable=True)
    return [(int(a), float(b)) for a, b in zip(i[:k].tolist(), v[:k].tolist())]


LOWERED_ORDER = ("bias", "repetition", "presence", "frequency")


def lower_logits_processors(procs) -> Optional[Dict[str, tuple]]:
    """The parameters of a processor list that the lock-step batch applies on the device (csrc/decode_batch.cu
    `bd_procs_kernel`): {"bias": ({id: value},), "repetition" | "presence" | "frequency": (penalty, context size)}.
    Only closures of `make_logits_processors` / `make_*_penalty` lower, each kind at most once and in the order
    make_logits_processors returns them (the order the kernel applies them).  None when the list holds anything
    else: that row runs its processors as torch ops."""
    out: Dict[str, tuple] = {}
    last = -1
    for p in procs or []:
        spec = getattr(p, "lowered", None)
        if not isinstance(spec, tuple) or spec[0] not in LOWERED_ORDER:
            return None
        at = LOWERED_ORDER.index(spec[0])
        if at <= last:
            return None
        last = at
        out[spec[0]] = tuple(spec[1:])
    return out


def apply_top_k(logprobs: torch.Tensor, top_k: int) -> torch.Tensor:
    vocab = logprobs.shape[-1]
    if not isinstance(top_k, int) or not (0 < top_k < vocab):
        raise ValueError(f"`top_k` has to be an integer in the (0, {vocab}] interval,"
                         f" but is {top_k}.")
    keep = torch.topk(logprobs, top_k, dim=-1).indices
    out = torch.full_like(logprobs, -float("inf"))
    return out.scatter(-1, keep, logprobs.gather(-1, keep))


def apply_top_n_sigma(logits: torch.Tensor, n_sigma: float) -> torch.Tensor:
    if n_sigma < 0:
        raise ValueError(f"`top_n_sigma` has to be a non-negative float, but is {n_sigma}")
    f = logits.float()
    top = f.max(dim=-1, keepdim=True).values
    std = f.std(dim=-1, keepdim=True, unbiased=False)
    return torch.where(f < top - n_sigma * std, torch.full_like(logits, -float("inf")), logits)


def apply_p_less(logits: torch.Tensor, temp: float) -> torch.Tensor:
    probs = torch.softmax(logits.float() * (1.0 / temp), dim=-1)
    thr = (probs * probs).sum(dim=-1, keepdim=True)
    return torch.where(probs < thr, torch.full_like(logits, -float("inf")), logits)


def apply_min_p(logprobs: torch.Tensor, min_p: float, min_tokens_to_keep: int = 1) -> torch.Tensor:
    if not (0 <= min_p <= 1.0):
        raise ValueError(f"`min_p` has to be a float in the [0, 1] interval, but is {min_p}")
    if not isinstance(min_tokens_to_keep, int) or (min_tokens_to_keep < 1):
        raise ValueError("`min_tokens_to_keep` has to be a positive integer, "
                         f"but is {min_tokens_to_keep}")
    top = logprobs.max(dim=-1, keepdim=True).values
    remove = logprobs < (top + math.log(min_p))
    if min_tokens_to_keep > 1:
        keep = torch.topk(logprobs, min_tokens_to_keep, dim=-1).indices
        remove = remove.scatter(-1, keep, False)
    return torch.where(remove, torch.full_like(logprobs, -float("inf")), logprobs)


def _cum_in_original_order(p_sorted, sorted_idx):
    cum = torch.cumsum(p_sorted, dim=-1)
    inv = torch.zeros_like(sorted_idx).scatter(
        -1, sorted_idx, torch.arange(sorted_idx.shape[-1], device=sorted_idx.device
                                     ).expand_as(sorted_idx))
    return cum.gather(-1, inv)


def apply_top_p(logprobs: torch.Tensor, top_p: float) -> torch.Tensor:
    lp = logprobs.float()
    probs = torch.exp(lp)
    sorted_idx = torch.argsort(lp, dim=-1, stable=True)
    cum = _cum_in_original_order(probs.gather(-1, sorted_idx), sorted_idx)
    return torch.where(cum > 1 - top_p, logprobs, torch.full_like(logprobs, -float("inf")))


def apply_typical_p(logprobs: torch.Tensor, typical_p: float) -> torch.Tensor:
    if not (0.0 < typical_p <= 1.0):
        raise ValueError(f"`typical_p` has to be a float in the (0, 1] interval, but is {typical_p}")
    lp = logprobs.float()
    p = torch.exp(lp)
    ent = -(p * torch.where(p > 0, lp, torch.zeros_like(lp))).sum(dim=-1, keepdim=True)
    shifted = (-lp - ent).abs()
    sorted_idx = torch.argsort(shifted, dim=-1, stable=True)
    cum = _cum_in_original_order(p.gather(-1, sorted_idx), sorted_idx)
    return torch.where(cum - p < typical_p, logprobs, torch.full_like(logprobs, -float("inf")))


def apply_xtc(logits, xtc_probability: float, xtc_threshold: float, xtc_special_tokens: List[int]):
    if not (0 <= xtc_threshold <= 0.5):
        raise ValueError(f"`threshold` has to be a float in the [0, 0.5] interval, but is {xtc_threshold}")
    if not (0 <= xtc_probability <= 1.0):
        raise ValueError(f"`probability` has to be a float in the [0, 1] interval, but is {xtc_probability}")
    probs = torch.softmax(logits.float(), -1)
    inf = torch.full_like(probs, float("inf"))
    mask = probs > torch.where(probs > xtc_threshold, probs, inf).min()
    if xtc_special_tokens:
        mask[..., xtc_special_tokens] = False
    if float(torch.rand(())) > xtc_probability:
        return logits
    return torch.where(mask, torch.full_like(logits, -float("inf")), logits)


def categorical_sampling(logits: torch.Tensor, temp: float) -> torch.Tensor:
    """mx.random.categorical(logits / temp) via the Gumbel-max trick."""
    z = logits.float() * (1.0 / temp)
    u = torch.rand(z.shape, device=z.device).clamp_min(1e-20)
    return torch.argmax(z - torch.log(-torch.log(u)), dim=-1)


def make_repetition_penalty(penalty: float, context_size: int = 20):
    if penalty < 0 or not isinstance(penalty, (int, float)):
        raise ValueError(f"penalty must be a non-negative float, got {penalty}")

    def repetition_penalty_processor(tokens, logits):
        if len(tokens) > 0:
            t = torch.as_tensor(tokens[-context_size:], device=logits.device, dtype=torch.long)
            sel = logits[:, t]
            sel = torch.where(sel < 0, sel * penalty, sel / penalty)
            logits = logits.clone()
            logits[:, t] = sel
        return logits

    repetition_penalty_processor.lowered = ("repetition", penalty, context_size)
    return repetition_penalty_processor


def make_presence_penalty(penalty: float, context_size: int = 20):
    def presence_penalty_processor(tokens, logits):
        if len(tokens) > 0:
            t = torch.unique(torch.as_tensor(tokens[-context_size:], device=logits.device,
                                             dtype=torch.long))
            logits = logits.clone()
            logits[:, t] -= penalty
        return logits

    presence_penalty_processor.lowered = ("presence", penalty, context_size)
    return presence_penalty_processor


def make_frequency_penalty(penalty: float, context_size: int = 20):
    def frequency_penalty_processor(tokens, logits):
        if len(tokens) > 0:
            t = torch.as_tensor(tokens[-context_size:], device=logits.device, dtype=torch.long)
            sub = torch.zeros_like(logits[0], dtype=torch.float32)
            sub.index_add_(0, t, torch.full((t.numel(),), float(penalty), device=logits.device))
            logits = (logits.float() - sub[None]).to(logits.dtype)
        return logits

    frequency_penalty_processor.lowered = ("frequency", penalty, context_size)
    return frequency_penalty_processor


def top_p_sampling(logits: torch.Tensor, top_p: float, temperature: float) -> torch.Tensor:
    unbatched = logits.ndim == 1
    if unbatched:
        logits = logits[None]
    probs = torch.softmax(logits.float() / temperature, dim=-1)
    sorted_idx = torch.argsort(probs, dim=-1, stable=True)
    sp = probs.gather(-1, sorted_idx)
    cum = torch.cumsum(sp, dim=-1)
    top = torch.where(cum > 1 - top_p, sp, torch.zeros_like(sp))
    pos = categorical_sampling(torch.log(top), 1.0)
    tok = sorted_idx.gather(-1, pos[..., None]).squeeze(-1)
    return tok.squeeze(0) if unbatched else tok
