"""LLaVA-Next (LLaVA-1.6) `Model` — a sibling of LLaVA-1.5 that shares its kernels (SURVEY §8 f4; reference
mlx_vlm/models/llava_next/llava_next.py:32-144).  What differs from LLaVA-1.5, all of it host logic around the same
device ops:
  * `pixel_values` is (1, N, C, H, W): the N crops of ONE image (base view + any-resolution tiles); the tower and the
    projector run on the N crops as a batch;
  * the learned `image_newline` vector is broadcast to the features' shape and concatenated along the CROP axis
    (N crops -> 2N blocks of P rows; llava_next.py:84-90);
  * the merge REPLACES every <image> token by one block of P rows, so the sequence grows; `zip(text segments, blocks)`
    pairs the first min(#tokens, #blocks) and keeps only the tail after the LAST <image> token (llava_next.py:98-121).
Both are pinned by executing the reference's source (tests/golden/make_llava_next_golden.py)."""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
import torch

from ..base import InputEmbeddingsFeatures
from ..engine_model import _np, embed_merge, embed_tokens
from ..llava.llava import Model as _LlavaModel
from .config import ModelConfig
from .language import LanguageModel


def merge_plan(input_ids, image_token_index: int, n_blocks: int, rows_per_block: int) -> Tuple[List[int], int]:
    """The merged sequence of llava_next.py:98-121 as a list of source ids: text positions keep their token id, every
    image row is the image token id; returns (ids of the merged sequence, number of blocks used).  Pure indexing."""
    ids = _np(input_ids)
    if ids.ndim == 2:
        ids = ids[0]
    ids = ids.tolist()
    positions = [i for i, t in enumerate(ids) if t == image_token_index]
    out: List[int] = []
    start = 0
    used = min(len(positions), n_blocks)
    for k in range(used):                       # zip(text_segments, image_embeddings)
        out += ids[start:positions[k]]
        out += [image_token_index] * rows_per_block
        start = positions[k] + 1
    if positions:
        start = positions[-1] + 1               # `final_embeddings += [inputs_embeds[:, start_idx:]]`: after the LAST token
    out += ids[start:]
    return out, used


class Model(_LlavaModel):
    LanguageModel = LanguageModel

    def __init__(self, config: ModelConfig, device=None):
        super().__init__(config, device)
        self.image_newline: torch.Tensor = None   # (hidden,) bf16 on the device, set by load_weights

    def load_weights(self, weights: Dict[str, torch.Tensor], strict: bool = True):
        super().load_weights(weights, strict)
        self.image_newline = weights["image_newline"].to(device=self._engine().device, dtype=torch.bfloat16).contiguous()
        torch.cuda.synchronize(self._engine().device)

    def init_random(self, seed: int = 0, std: float = 0.02):
        W = self.random_weights(self.config, seed, std, self._engine().device)
        g = torch.Generator(device=self._engine().device).manual_seed(seed + 1)
        H = self.config.text_config.hidden_size
        W["image_newline"] = (torch.randn(H, generator=g, device=self._engine().device) / H ** 0.5).to(torch.bfloat16)
        self.load_weights(W)
        return self

    def encode_image(self, pixel_values) -> torch.Tensor:
        """(1, N, C, H, W) or (N, C, H, W) fp32 -> (2N, P, hidden) bf16: the projected crops, then the newline blocks"""
        pv = pixel_values
        if pv.dim() == 5:
            pv = pv[0]                                      # `pixel_values[0]`: the crops of one image
        feats = super().encode_image(pv)                    # (N, P, hidden) bf16, one rounding (astype at the merge)
        eng = self._engine()
        with torch.cuda.stream(eng.stream):                 # layout only: the newline vector repeated N * P times
            nl = self.image_newline.to(feats.dtype).expand(feats.shape[0], feats.shape[1], -1)
            return torch.cat([feats, nl], dim=0).contiguous()

    def get_input_embeddings(self, input_ids=None, pixel_values=None, **kwargs):
        eng = self._engine()
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        if pixel_values is None:
            return InputEmbeddingsFeatures(inputs_embeds=embed_tokens(eng, ids))
        if self.vision_feature_select_strategy not in ("default", "full"):
            raise ValueError(f"Unexpected feature selection strategy: {self.vision_feature_select_strategy}")
        cached = kwargs.get("cached_image_features", None)
        blocks = cached if cached is not None else self.encode_image(pixel_values)
        return InputEmbeddingsFeatures(inputs_embeds=self._merge_input_ids_with_image_features(blocks, None, ids))

    def _merge_input_ids_with_image_features(self, image_features, inputs_embeds, input_ids):
        """llava_next.py:98-121 on the device: host plan (merge_plan) + the shared gather kernel"""
        if inputs_embeds is not None:
            raise NotImplementedError("llava_next merge: pass inputs_embeds=None (the embedding lookup is fused)")
        n_blocks, P, H = int(image_features.shape[0]), int(image_features.shape[1]), int(image_features.shape[2])
        tok = int(self.config.image_token_index)
        plan, used = merge_plan(input_ids, tok, n_blocks, P)
        return embed_merge(self._engine(), np.asarray([plan], dtype=np.int64),
                           image_features[:max(used, 1)].reshape(-1, H), used * P, tok)
