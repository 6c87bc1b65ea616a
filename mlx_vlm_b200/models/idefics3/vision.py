"""SigLIP vision tower of Idefics3 / SmolVLM (reference mlx_vlm/models/idefics3/vision.py:67-185).

Host integer logic (bit-exact, pinned by tests/golden/idefics3_golden.json): the bucketed position ids.  Unlike
Idefics2 the buckets are `sum(frac >= boundaries)` (coordinate 0 -> bucket 0), the ids of the valid block are written
to the FIRST n_valid sequence positions (vision.py:128-131), and the position embedding of a padding patch is zeroed
(`position_embeddings * patch_mask`, :139-141).

Device: the layer structure is Idefics2's tower with GELU(approx="precise") (the tanh form) in the MLP, so it runs on
the same kernels (split-operand tensor-core GEMMs + fp32 row kernels).  The reference casts the embeddings to the
weight dtype and runs THIS encoder in bf16 (vision.py:176); here it is computed at fp32 accuracy — a superset: the
result differs from the reference's by the reference's own bf16 rounding noise, which is the tolerance of the parity
test — and the pooled output is rounded to bf16 where the reference hands it over (`pooler_output.astype(...)`)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ..idefics2.vision import VisionModel as _SiglipTower
from ..tower_ops import EPI_GELU_TANH


def _arange_f32(start: float, stop: float, step: float) -> np.ndarray:
    """`mx.arange` on python floats: float32, element i = start + i * step with the product rounded to float32 (the Metal
    kernel of the device the reference runs on).  The buckets below are decided by `>=` between float32 values and an image
    that fills the grid makes every comparison a tie, so this rounding is part of the reference's behaviour (DESIGN §7)."""
    n = max(int(np.ceil((stop - start) / step)), 0)
    first = np.float32(start)
    inc = np.float32(np.float32(start + step) - first)
    return np.array([np.float32(first + np.float32(np.float32(i) * inc)) for i in range(n)], dtype=np.float32)


def position_ids(patch_mask: np.ndarray, side: int, seq: int) -> np.ndarray:
    """vision.py:95-137.  patch_mask (B, ph, pw) bool -> (B, seq) int64"""
    m = np.asarray(patch_mask).astype(bool)
    edges = _arange_f32(1 / side, 1.0, 1 / side)
    top = np.float32(1.0 - 1e-6)
    ids = np.zeros((m.shape[0], seq), dtype=np.int64)
    for b in range(m.shape[0]):
        rows, cols = max(int(m[b, :, 0].sum()), 1), max(int(m[b, 0, :].sum()), 1)
        fr = np.minimum(np.arange(rows, dtype=np.float32) / np.float32(rows), top)
        fc = np.minimum(np.arange(cols, dtype=np.float32) / np.float32(cols), top)
        br = (fr[:, None] >= edges[None, :]).sum(axis=1)
        bc = (fc[:, None] >= edges[None, :]).sum(axis=1)
        flat = (br[:, None] * side + bc[None, :]).reshape(-1)
        n = min(flat.shape[0], seq)
        ids[b, :n] = flat[:n]
    return ids


class VisionModel(_SiglipTower):
    epi = EPI_GELU_TANH       # GELU(approx="precise"): the tanh form

    def load(self, weights, prefix: str = "vision_model."):
        super().load(weights, prefix)
        pos = self.w["pos"]
        self.n_pos = pos.shape[0]
        with torch.cuda.stream(self._engine().stream):      # one extra all-zero row: the "masked" position
            self.w["pos"] = torch.cat([pos, torch.zeros_like(pos[:1])], 0).contiguous()

    def patch_position_ids(self, patch_attention_mask: Optional[np.ndarray], B: int, gh: int, gw: int) -> np.ndarray:
        """vision.py:95-141: padding patches take the zero row"""
        P = gh * gw
        if patch_attention_mask is None:
            return np.tile(np.arange(P, dtype=np.int64), (B, 1))          # vision.py:99-103
        m = np.asarray(patch_attention_mask).astype(bool)
        ids = position_ids(m, self.config.image_size // self.config.patch_size, P)
        ids[~m.reshape(B, -1)[:, :P]] = self.n_pos                       # zero row
        return ids
