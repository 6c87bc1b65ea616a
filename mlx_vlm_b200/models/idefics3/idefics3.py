"""Idefics3 `Model` — the per-model contract of the reference (mlx_vlm/models/idefics3/idefics3.py:47-230):
`get_input_embeddings` (padding-image removal, pixel mask -> patch mask, SigLIP tower -> pixel shuffle + Linear ->
masked-scatter merge), `vision_model`, `language_model`, `connector`, `layers`, `sanitize`.  Everything around the
tower and the connector is Idefics2's (models/idefics2/idefics2.py); SmolVLM is this model under another name
(models/smolvlm)."""
from __future__ import annotations

from typing import Dict

import torch

from ..idefics2.idefics2 import Model as _Idefics2Model
from ..idefics2.idefics2 import patch_attention_mask, real_image_indices  # noqa: F401  (same rules, :104-140)
from ..tower_ops import SplitBuf, TowerOps
from .config import ModelConfig
from .language import LanguageModel
from .vision import VisionModel
from .weights import random_weights


class Connector:
    """pixel shuffle + modality projection (idefics3.py:21-70): tokens of an s x s neighbourhood are concatenated
    along the feature axis, then one Linear without bias, in fp32 on the bf16-valued tower output"""

    def __init__(self, config: ModelConfig, engine_getter):
        self.config = config
        self._engine = engine_getter
        self.w: Dict[str, torch.Tensor] = {}

    def load(self, weights, prefix="connector."):
        eng = self._engine()
        self.w["proj"] = weights[prefix + "modality_projection.proj.weight"].to(device=eng.device,
                                                                                dtype=torch.bfloat16).contiguous()

    def __call__(self, feats: torch.Tensor, n_img: int) -> torch.Tensor:
        """feats fp32 (n_img * P, E) -> fp32 (n_img * P / s^2, H)"""
        eng = self._engine()
        ops = TowerOps(eng)
        s = self.config.scale_factor
        E = feats.shape[1]
        P = feats.shape[0] // n_img
        side = int(P ** 0.5)
        if side * side != P or side % s:
            raise ValueError(f"pixel shuffle needs a square grid divisible by {s}, got {P} patches")
        rows = n_img * (side // s) ** 2
        xs = SplitBuf(eng, rows, E * s * s)
        ops.pixel_shuffle(feats, n_img, side, s, xs, round_in=True)
        out = ops.f32(rows, self.w["proj"].shape[0])
        ops.linear(xs, self.w["proj"], None, out32=out)
        return out


class Model(_Idefics2Model):
    LanguageModel = LanguageModel
    VisionModel = VisionModel
    Connector = Connector
    random_weights = staticmethod(random_weights)
