"""Qwen2.5-VL `Model` — the per-model contract of the reference (mlx_vlm/models/qwen2_5_vl/qwen2_5_vl.py:14-195).  Everything
but the vision tower is Qwen2-VL's (same `get_input_embeddings`, merge, M-RoPE index, `sanitize`, language model —
models/qwen2_vl/qwen2_vl.py); the tower (RMSNorm / SwiGLU blocks, windowed attention) is models/qwen2_5_vl/vision.py and
the decoder engine is created without its built-in Qwen2-VL tower."""
from __future__ import annotations

from typing import Dict

import torch

from ..qwen2_vl.qwen2_vl import Model as _Qwen2VLModel
from .vision import VisionModel
from .weights import random_weights


class Model(_Qwen2VLModel):
    VisionModel = VisionModel
    random_weights = staticmethod(random_weights)
    builtin_tower = False

    def _load_vision(self, weights: Dict[str, torch.Tensor]):
        self.vision_tower.load(self.vision_tower.sanitize({k: x for k, x in weights.items() if "vision_tower" in k}))
