"""Seeded random weights at the Qwen3-VL decoder shapes under the reference's names (benchmarks / tests)."""
from __future__ import annotations

import torch


def weight_shapes(config):
    t = config.text_config
    H, hd = t.hidden_size, t.head_dim
    s = {"language_model.model.embed_tokens.weight": (t.vocab_size, H)}
    for i in range(t.num_hidden_layers):
        p = f"language_model.model.layers.{i}."
        s[p + "input_layernorm.weight"], s[p + "post_attention_layernorm.weight"] = (H,), (H,)
        for n, rows in (("q", t.num_attention_heads * hd), ("k", t.num_key_value_heads * hd),
                        ("v", t.num_key_value_heads * hd)):
            s[p + f"self_attn.{n}_proj.weight"] = (rows, H)
        s[p + "self_attn.q_norm.weight"], s[p + "self_attn.k_norm.weight"] = (hd,), (hd,)
        s[p + "self_attn.o_proj.weight"] = (H, t.num_attention_heads * hd)
        s[p + "mlp.gate_proj.weight"], s[p + "mlp.up_proj.weight"] = (t.intermediate_size, H), (t.intermediate_size, H)
        s[p + "mlp.down_proj.weight"] = (H, t.intermediate_size)
    s["language_model.model.norm.weight"] = (H,)
    if not t.tie_word_embeddings:
        s["language_model.lm_head.weight"] = (t.vocab_size, H)
    return s


def random_weights(config, seed=0, std=0.02, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    W = {}
    for name, shape in weight_shapes(config).items():
        r = torch.randn(shape, generator=g, device=device, dtype=torch.float32) * std
        W[name] = (r + 1.0 if name.endswith("norm.weight") else r).to(torch.bfloat16)
    return W
