"""Language model of LLaVA-Next (reference mlx_vlm/models/llava_next/language.py): the same Llama / Mistral decoder as
LLaVA-1.5 on the shared decoder engine.  One difference in the calling convention: the merge of LLaVA-Next makes the
embedded sequence LONGER than `input_ids` (every <image> token becomes a block of rows), and the reference's language
model takes its length from `inputs_embeds` (language.py:131-140), so the ids are only a placeholder here."""
from __future__ import annotations

import numpy as np

from ..engine_model import _np
from ..llava.language import LanguageModel as _LlavaLM


class LanguageModel(_LlavaLM):
    def __call__(self, inputs, inputs_embeds=None, mask=None, cache=None, **kwargs):
        if inputs_embeds is not None:
            ids = _np(inputs)
            if ids.ndim == 1:
                ids = ids[None]
            T = int(inputs_embeds.shape[-2])
            if ids.shape[1] != T:        # positions are arange(T) + cache offset: the token ids are not looked at
                inputs = np.zeros((ids.shape[0], T), dtype=np.int64)
        return super().__call__(inputs, inputs_embeds=inputs_embeds, mask=mask, cache=cache, **kwargs)
