"""LLaVA-1.5 `Model` — the per-model contract of the reference (mlx_vlm/models/llava/llava.py:32-150):
`get_input_embeddings` (CLIP tower -> feature layer -2 without the class token -> projector -> merge),
`_merge_input_ids_with_image_features`, `vision_tower`, `language_model`, `layers`, `sanitize`."""
from __future__ import annotations

from typing import Dict

import torch

from ... import _native as N
from ..base import InputEmbeddingsFeatures
from ..engine_model import EngineModel, _np, embed_merge, embed_tokens
from ..tower_ops import EPI_GELU_EXACT, SplitBuf, TowerOps
from .config import ModelConfig
from .language import LanguageModel
from .vision import VisionModel
from .weights import random_weights


class Model(EngineModel):
    LanguageModel = LanguageModel
    VisionModel = VisionModel
    random_weights = staticmethod(random_weights)

    def __init__(self, config: ModelConfig, device=None):
        super().__init__(config, device)
        self.vision_tower = self.VisionModel(config.vision_config, self._engine)
        self.proj: Dict[str, torch.Tensor] = {}
        self.vision_feature_layer = config.vision_feature_layer
        self.vision_feature_select_strategy = config.vision_feature_select_strategy

    def _load_vision(self, weights: Dict[str, torch.Tensor]):
        """reference-named tensors vision_tower.* / multi_modal_projector.*"""
        dev = self._engine().device
        self.vision_tower.load(self.vision_tower.sanitize({k: v for k, v in weights.items() if k.startswith("vision_tower")}))
        for n in ("linear_1", "linear_2"):
            self.proj[n + ".w"] = weights[f"multi_modal_projector.{n}.weight"].to(device=dev, dtype=torch.bfloat16).contiguous()
            self.proj[n + ".b"] = weights[f"multi_modal_projector.{n}.bias"].to(device=dev, dtype=torch.bfloat16).contiguous()

    # ------------------------------------------------------------- contract
    def encode_image(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """pixel_values (B, C, H, W) fp32 -> projected image features (B, P, hidden) bf16 (llava.py:59-83)"""
        eng = self._engine()
        ops = TowerOps(eng)
        v = self.config.vision_config
        with torch.cuda.stream(eng.stream):
            x = pixel_values.to(torch.float32).permute(0, 2, 3, 1).contiguous()   # NHWC, like llava.py:62
        B = x.shape[0]
        _, _, states = self.vision_tower(x, output_hidden_states=True, feature_layer=self.vision_feature_layer)
        if not isinstance(self.vision_feature_layer, int):
            raise NotImplementedError("a list of vision feature layers is outside this engine's hot-path scope")
        sel = states[self.vision_feature_layer]
        P = (x.shape[1] // v.patch_size) * (x.shape[2] // v.patch_size)
        L = P + 1
        skip = 1 if self.vision_feature_select_strategy == "default" else 0
        rows = L - skip
        E, H = v.hidden_size, self.config.text_config.hidden_size
        xs = SplitBuf(eng, B * rows, E)
        for b in range(B):   # drop the class token of every image (llava.py:66-68)
            N.check(eng.lib.b200_f32_split(sel[b * L + skip:].data_ptr(), E, xs.t[b * rows:].data_ptr(), xs.ld, xs.n_pad,
                                           rows, E, eng.s), "f32_split")
        mid = SplitBuf(eng, B * rows, H)
        ops.linear(xs, self.proj["linear_1.w"], self.proj["linear_1.b"], out_split=mid, epi=EPI_GELU_EXACT)
        feats32 = ops.f32(B * rows, H)
        ops.linear(mid, self.proj["linear_2.w"], self.proj["linear_2.b"], out32=feats32)
        feats = eng.empty((B, rows, H))
        N.check(eng.lib.b200_cast_f32_bf16(feats32.data_ptr(), feats.data_ptr(), B * rows * H, eng.s), "cast")
        return feats   # astype(inputs_embeds.dtype): the ONE rounding of the vision path (llava.py:101-104)

    def get_input_embeddings(self, input_ids=None, pixel_values=None, **kwargs):
        eng = self._engine()
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        if pixel_values is None:
            return InputEmbeddingsFeatures(inputs_embeds=embed_tokens(eng, ids))
        cached = kwargs.get("cached_image_features", None)
        feats = cached if cached is not None else self.encode_image(pixel_values)
        final = self._merge_input_ids_with_image_features(feats, None, ids)
        return InputEmbeddingsFeatures(inputs_embeds=final)

    def _merge_input_ids_with_image_features(self, image_features, inputs_embeds, input_ids):
        """llava.py:90-116: the k-th <image> position takes the k-th feature row (batch 1)."""
        eng = self._engine()
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        tok = self.config.image_token_index
        n_pos = int((ids == tok).sum())
        flat = image_features.reshape(-1, image_features.shape[-1])
        if flat.shape[0] > n_pos:
            raise ValueError("Llava model supports only one image per input. Please check your input_ids and "
                             "pixel_values.")
        if flat.shape[0] < n_pos:
            raise ValueError(f"shape mismatch: {flat.shape[0]} image feature rows cannot fill {n_pos} <image> "
                             "positions")
        if inputs_embeds is None:
            return embed_merge(eng, ids, flat, flat.shape[0], tok)
        return embed_merge(eng, ids, flat, flat.shape[0], inputs_embeds=inputs_embeds, rows=ids == tok)
