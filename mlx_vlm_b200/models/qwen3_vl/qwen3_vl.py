"""Qwen3-VL `Model` (reference mlx_vlm/models/qwen3_vl/qwen3_vl.py) for text prompts.

The decoder differs from Qwen2-VL's in three ways the engine covers here: no q/k/v bias, an RMSNorm over every q and
k head before the rotary (language.py:59-60,84-89; engine weights lm.<i>.qn / lm.<i>.kn) and the interleaved M-RoPE
frequency-to-axis table (rope_utils.py:511-516; b200_engine_set_axis_sel).  `head_dim` comes from the config.

Not built yet, and refused with NotImplementedError: image and video input (the Qwen3-VL vision tower with its
DeepStack feature sets), and `qwen3_vl_moe`.
"""
from __future__ import annotations

import numpy as np

from ... import _native as N
from ..base import InputEmbeddingsFeatures
from ..engine_model import _np, embed_tokens
from ..qwen2_vl.qwen2_vl import Model as _Qwen2VLModel
from .config import ModelConfig
from .language import LanguageModel
from .weights import random_weights

_NO_VISION = ("qwen3_vl: image and video input are not supported by the CUDA engine yet (the Qwen3-VL vision tower "
              "and its DeepStack features are not built); text prompts are")


def interleaved_position_selector(mrope_section, freq_dim: int) -> np.ndarray:
    """_interleaved_position_selector (rope_utils.py:511-516): frequency i rotates with the t, h or w position id"""
    selector = [0] * freq_dim
    for dim, offset in enumerate((1, 2), start=1):
        for idx in range(offset, min(mrope_section[dim] * 3, freq_dim), 3):
            selector[idx] = dim
    return np.asarray(selector, dtype=np.int32)


class Model(_Qwen2VLModel):
    LanguageModel = LanguageModel
    VisionModel = None
    random_weights = staticmethod(random_weights)   # norm weights 1 + N(0, std): q/k norms are not the identity
    qkv_bias = False
    qk_norm = True
    builtin_tower = False

    def __init__(self, config: ModelConfig, device=None):
        if config.model_type != "qwen3_vl":
            raise NotImplementedError(f"{config.model_type}: only dense qwen3_vl is supported by the CUDA engine "
                                      "(qwen3_vl_moe is not built)")
        super().__init__(config, device)

    def _engine(self):
        if self._eng is None:
            eng = super()._engine()
            sel = interleaved_position_selector(self.config.text_config.mrope_section, eng.cfg.head_dim // 2)
            N.check(eng.lib.b200_engine_set_axis_sel(eng.h, sel.ctypes.data), "set_axis_sel")
        return self._eng

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

    def _load_vision(self, weights):
        """no vision tower yet: its tensors are not used"""

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
