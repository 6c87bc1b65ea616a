"""Reference arithmetic of the Qwen3-VL decoder for the tests (the product never imports this).

Restates reference mlx_vlm/models/qwen3_vl/language.py for text prompts with the rounding points of
oracle/mlx_semantics.py: bf16 Linear projections without bias, q_norm / k_norm as mx.fast.rms_norm over each head
(:84-89), the interleaved M-RoPE (rope_utils.py:511-516 selector; cos / sin cast to bf16, three roundings in the
rotation like oracle.qwen2vl.apply_mrope), the CPU-fallback SDPA, SwiGLU MLP and the tied or untied head.
Rounder("f32") gives the un-rounded evaluation that tests compare with HuggingFace transformers.
"""
import numpy as np
import torch

from oracle import mlx_semantics as S
from oracle.mlx_semantics import Rounder
from oracle.qwen2vl import OracleKVCache, _rotate_half, logprobs_from_logits


def interleaved_selector(section, freq_dim):
    sel = [0] * freq_dim
    for dim, offset in enumerate((1, 2), start=1):
        for idx in range(offset, min(section[dim] * 3, freq_dim), 3):
            sel[idx] = dim
    return np.asarray(sel, dtype=np.int64)


def cos_sin(t, position_ids, R):
    """position_ids (3, B, L) or (B, L) -> cos, sin (B, L, head_dim), cast to the activation dtype"""
    hd = t.head_dim
    inv = 1.0 / (t.rope_theta ** (torch.arange(0, hd, 2).to(torch.float32) / hd))
    pos = torch.as_tensor(np.array(position_ids))
    if pos.ndim == 2:
        freqs = pos.to(torch.float32)[..., None] * inv
    else:
        sel = torch.from_numpy(interleaved_selector(t.mrope_section, inv.shape[0]))
        freqs = pos[sel].permute(1, 2, 0).to(torch.float32) * inv
    emb = torch.cat([freqs, freqs], dim=-1)
    return R.r(torch.cos(emb)), R.r(torch.sin(emb))


def rope(R, x, cos, sin):
    c, s = cos[:, None], sin[:, None]
    return R.r(R.r(x * c) + R.r(_rotate_half(x) * s))


def lm_forward(t, W, h, position_ids, cache, R, collect_k=None):
    """Qwen3VLModel.__call__ without the embedding: h (B, L, H) -> final-normed (B, L, H)"""
    B, L, H = h.shape
    nh, nkv, hd = t.num_attention_heads, t.num_key_value_heads, t.head_dim
    cos, sin = cos_sin(t, position_ids, R)
    for i in range(t.num_hidden_layers):
        p = f"language_model.model.layers.{i}."
        x = S.rms_norm(R, h, W[p + "input_layernorm.weight"], t.rms_norm_eps)
        q = S.linear(R, x, W[p + "self_attn.q_proj.weight"]).reshape(B, L, nh, hd)
        k = S.linear(R, x, W[p + "self_attn.k_proj.weight"]).reshape(B, L, nkv, hd)
        v = S.linear(R, x, W[p + "self_attn.v_proj.weight"]).reshape(B, L, nkv, hd).transpose(1, 2)
        q = S.rms_norm(R, q, W[p + "self_attn.q_norm.weight"], t.rms_norm_eps).transpose(1, 2)
        k = S.rms_norm(R, k, W[p + "self_attn.k_norm.weight"], t.rms_norm_eps).transpose(1, 2)
        q, k = rope(R, q, cos, sin), rope(R, k, cos, sin)
        keys, values = cache[i].update_and_fetch(k, v)
        if collect_k is not None:
            collect_k.append(k)
        o = S.sdpa(R, q, keys, values, hd ** -0.5, causal=(L > 1))
        o = o.transpose(1, 2).reshape(B, L, nh * hd)
        h = R.r(h + S.linear(R, o, W[p + "self_attn.o_proj.weight"]))
        x = S.rms_norm(R, h, W[p + "post_attention_layernorm.weight"], t.rms_norm_eps)
        g = S.linear(R, x, W[p + "mlp.gate_proj.weight"])
        u = S.linear(R, x, W[p + "mlp.up_proj.weight"])
        h = R.r(h + S.linear(R, S.swiglu(R, g, u), W[p + "mlp.down_proj.weight"]))
    return S.rms_norm(R, h, W["language_model.model.norm.weight"], t.rms_norm_eps)


def head(t, W, hidden, R):
    w = W["language_model.model.embed_tokens.weight"] if t.tie_word_embeddings else W["language_model.lm_head.weight"]
    return S.linear(R, hidden, w)


def host_weights(config, seed=0, std=0.02):
    """the product's random_weights on the CPU, as fp32 tensors holding bf16 values"""
    from mlx_vlm_b200.models.qwen3_vl.weights import random_weights
    return {k: v.float() for k, v in random_weights(config, seed, std, "cpu").items()}


def greedy_generate(config, W, input_ids, max_tokens, dtype="bf16"):
    """generate_step's greedy loop over a text prompt: tokens (B, n) and the logprobs of every step"""
    R = Rounder(dtype)
    t = config.text_config
    ids = torch.as_tensor(np.asarray(input_ids, dtype=np.int64))
    B, T = ids.shape
    cache = [OracleKVCache() for _ in range(t.num_hidden_layers)]
    pos = np.broadcast_to(np.arange(T)[None], (B, T))
    logits = head(t, W, lm_forward(t, W, W["language_model.model.embed_tokens.weight"][ids], pos, cache, R)[:, -1], R)
    toks, lps = [], []
    for n in range(max_tokens):
        lp = logprobs_from_logits(R, logits)
        y = S.argmax_lowest(lp)
        toks.append(y.clone())
        lps.append(lp)
        if n == max_tokens - 1:
            break
        p = np.full((3, B, 1), cache[0].offset, dtype=np.int64)
        e = W["language_model.model.embed_tokens.weight"][y][:, None, :]
        logits = head(t, W, lm_forward(t, W, e, p, cache, R)[:, -1], R)
    return torch.stack(toks, 1), lps
