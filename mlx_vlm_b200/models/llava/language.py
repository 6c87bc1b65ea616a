"""Llama language model of LLaVA-1.5 (reference mlx_vlm/models/llava/language.py:16-150) on the shared
decoder engine: a Llama layer is the Qwen2 layer with zero q/k/v bias, and nn.RoPE(traditional=False)
is the multimodal rotary with the same position on all three axes."""
from __future__ import annotations

import numpy as np

from ..engine_model import _np
from ..qwen2_vl.language import LanguageModel as _DecoderLM


class LanguageModel(_DecoderLM):
    def get_rope_index(self, input_ids, image_grid_thw=None, video_grid_thw=None, attention_mask=None):
        """1-D positions (language.py:66-79: the cache offset + arange); no M-RoPE delta"""
        ids = _np(input_ids)
        B, T = ids.shape
        amask = _np(attention_mask)
        if amask is not None:
            pos = np.cumsum(amask, axis=-1) - 1
            pos = np.where(amask == 0, 1, pos)
            return pos, np.zeros((B, 1), dtype=np.int64)
        return np.tile(np.arange(T), (B, 1)), np.zeros((B, 1), dtype=np.int64)
