"""Qwen3-VL `Model` (reference mlx_vlm/models/qwen3_vl/qwen3_vl.py) for text prompts.

The decoder differs from Qwen2-VL's in three ways the engine covers here: no q/k/v bias, an RMSNorm over every q and
k head before the rotary (language.py:59-60,84-89; engine weights lm.<i>.qn / lm.<i>.kn) and the interleaved M-RoPE
frequency-to-axis table (rope_utils.py:511-516; b200_engine_set_axis_sel).  `head_dim` comes from the config.

Not built yet, and refused with NotImplementedError: image and video input (the Qwen3-VL vision tower with its
DeepStack feature sets), and `qwen3_vl_moe`.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from ... import _native as N
from ..base import InputEmbeddingsFeatures
from ..qwen2_vl.language import _np
from ..qwen2_vl.qwen2_vl import Model as _Qwen2VLModel, embed_tokens
from .config import ModelConfig
from .language import LanguageModel

_NO_VISION = ("qwen3_vl: image and video input are not supported by the CUDA engine yet (the Qwen3-VL vision tower "
              "and its DeepStack features are not built); text prompts are")


def interleaved_position_selector(mrope_section, freq_dim: int) -> np.ndarray:
    """_interleaved_position_selector (rope_utils.py:511-516): frequency i rotates with the t, h or w position id"""
    selector = [0] * freq_dim
    for dim, offset in enumerate((1, 2), start=1):
        for idx in range(offset, min(mrope_section[dim] * 3, freq_dim), 3):
            selector[idx] = dim
    return np.asarray(selector, dtype=np.int32)


def weight_manifest(c: N.Qwen2VLConfig):
    """(engine name, shape) of every engine tensor: Qwen2-VL's decoder-only layout plus the q/k norm weights"""
    H, I = c.hidden, c.inter
    QKV = (c.n_heads + 2 * c.n_kv_heads) * c.head_dim
    out = [("lm.embed", (c.vocab, H)), ("lm.norm", (H,))]
    if not c.tie_embeddings:
        out.append(("lm.head", (c.vocab, H)))
    for i in range(c.n_layers):
        q = f"lm.{i}."
        out += [(q + "ln1", (H,)), (q + "ln2", (H,)), (q + "wqkv", (QKV, H)), (q + "bqkv", (QKV,)),
                (q + "wo", (H, c.n_heads * c.head_dim)), (q + "wgu", (2 * I, H)), (q + "wd", (H, I)),
                (q + "qn", (c.head_dim,)), (q + "kn", (c.head_dim,))]
    return out


class Model(_Qwen2VLModel):
    def __init__(self, config: ModelConfig, device=None):
        if config.model_type != "qwen3_vl":
            raise NotImplementedError(f"{config.model_type}: only dense qwen3_vl is supported by the CUDA engine "
                                      "(qwen3_vl_moe is not built)")
        self.config = config
        self._device = torch.device(device) if device is not None else torch.device("cuda", 0)
        self._eng = None
        self.vision_tower = None
        self.language_model = LanguageModel(config.text_config, config, self._engine)

    def native_config(self) -> N.Qwen2VLConfig:
        t = self.config.text_config
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = t.hidden_size, t.num_hidden_layers, t.intermediate_size
        c.n_heads, c.n_kv_heads = t.num_attention_heads, t.num_key_value_heads
        c.head_dim = t.head_dim
        c.vocab = t.vocab_size
        c.rms_eps, c.rope_theta = t.rms_norm_eps, t.rope_theta
        sec = t.mrope_section
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = sec[0], sec[1], sec[2]
        c.tie_embeddings = int(t.tie_word_embeddings)
        c.external_vision = 1
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = t.hidden_size, 1e-6
        return c

    def _engine(self):
        if self._eng is None:
            eng = super()._engine()
            sel = interleaved_position_selector(self.config.text_config.mrope_section, eng.cfg.head_dim // 2)
            N.check(eng.lib.b200_engine_set_axis_sel(eng.h, sel.ctypes.data), "set_axis_sel")
        return self._eng

    def _arena(self):
        if getattr(self, "_weights", None) is None:
            from ..qwen2_vl.qwen2_vl import WeightArena
            self._weights = WeightArena(weight_manifest(self.native_config()), self._engine().device)
        return self._weights

    def sanitize(self, weights):
        """HF names -> the reference's (qwen3_vl.py:238-252): in keys containing `model`, `model.language_model` ->
        `language_model.model` or else `model.visual` -> `vision_tower`; other keys: `lm_head` ->
        `language_model.lm_head`."""
        out = {}
        for key, value in weights.items():
            if "model" in key:
                if "model.language_model" in key:
                    key = key.replace("model.language_model", "language_model.model")
                elif "model.visual" in key:
                    key = key.replace("model.visual", "vision_tower")
            elif "lm_head" in key:
                key = key.replace("lm_head", "language_model.lm_head")
            out[key] = value
        return out

    def load_weights(self, weights: Dict[str, torch.Tensor], strict: bool = True):
        """Pack reference-named decoder tensors into the engine layout (q/k/v rows fused, zero qkv bias, q/k norm
        weights); the vision tower's tensors are not used (no tower yet)."""
        eng = self._engine()
        t = self.config.text_config
        dev = eng.device

        def get(name):
            if name not in weights:
                raise KeyError(f"missing weight {name}")
            return weights[name]

        put = self._put
        put("lm.embed", get("language_model.model.embed_tokens.weight"))
        put("lm.norm", get("language_model.model.norm.weight"))
        if not t.tie_word_embeddings:
            put("lm.head", get("language_model.lm_head.weight"))
        qkv_rows = (t.num_attention_heads + 2 * t.num_key_value_heads) * t.head_dim
        for i in range(t.num_hidden_layers):
            p, q = f"language_model.model.layers.{i}.", f"lm.{i}."
            put(q + "ln1", get(p + "input_layernorm.weight"))
            put(q + "ln2", get(p + "post_attention_layernorm.weight"))
            put(q + "wqkv", torch.cat([get(p + f"self_attn.{n}_proj.weight").to(dev) for n in "qkv"], 0))
            put(q + "bqkv", torch.zeros(qkv_rows, dtype=torch.bfloat16, device=dev))
            put(q + "qn", get(p + "self_attn.q_norm.weight"))
            put(q + "kn", get(p + "self_attn.k_norm.weight"))
            put(q + "wo", get(p + "self_attn.o_proj.weight"))
            put(q + "wgu", torch.cat([get(p + "mlp.gate_proj.weight").to(dev), get(p + "mlp.up_proj.weight").to(dev)], 0))
            put(q + "wd", get(p + "mlp.down_proj.weight"))
        torch.cuda.synchronize(dev)

    def init_random(self, seed: int = 0, std: float = 0.02):
        """Seeded random weights at the configured shapes (benchmarks; no checkpoints offline): N(0, std), norm
        weights 1 + N(0, std) so that the q/k norms are not the identity, qkv bias 0."""
        from .weights import random_weights
        self.load_weights(random_weights(self.config, seed, std, self._engine().device))
        return self

    # ------------------------------------------------------------- contract
    def get_input_embeddings(self, input_ids=None, pixel_values=None, **kwargs):
        """qwen3_vl.py:44-162, text branch: embedding lookup and the text position ids"""
        if pixel_values is not None or kwargs.get("pixel_values_videos", None) is not None:
            raise NotImplementedError(_NO_VISION)
        if kwargs.get("cached_image_features", None) is not None:
            raise NotImplementedError("qwen3_vl: VisionFeatureCache is not supported (no vision tower yet)")
        eng = self._engine()
        ids_host = _np(input_ids)
        if ids_host.ndim == 1:
            ids_host = ids_host[None]
        position_ids, rope_deltas = self.language_model.get_rope_index(ids_host, attention_mask=kwargs.get("mask"))
        return InputEmbeddingsFeatures(inputs_embeds=embed_tokens(eng, ids_host), position_ids=position_ids,
                                       rope_deltas=rope_deltas)

    def encode_image(self, *args, **kwargs):
        raise NotImplementedError(_NO_VISION)
