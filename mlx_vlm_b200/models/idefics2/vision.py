"""SigLIP vision tower of Idefics2 (reference mlx_vlm/models/idefics2/vision.py:20-215), in fp32 with
bf16-valued weights like the reference runs it (float32 `pixel_values` are never cast, idefics2.py:212-251).

Host integer logic (bit-exact, pinned by tests/golden): the bucketed fractional position ids
(vision.py:150-173).  Device: patch embedding with bias, position gather, N x {LN, MHA, LN, fast-GELU MLP},
post-LayerNorm — split-operand tensor-core GEMMs and fp32 kernels (models/tower_ops.py)."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from ..tower_ops import EPI_GELU_FAST, SplitBuf, TowerOps, encoder, pack_encoder_layers, sanitize
from .config import VisionConfig


def bucketed_position_ids(patch_mask: np.ndarray, side: int) -> np.ndarray:
    """vision.py:150-170.  patch_mask (B, ph, pw) bool -> (B, ph * pw) int64.  The valid nh x nw block of
    an image maps onto the side x side position grid through its fractional coordinates; the reference
    uses `np.digitize(frac, boundaries, right=True) - 1`, so coordinate 0 falls into bucket -1 and those
    ids are negative (they index the position table from its end, like the reference's mx gather)."""
    m = np.asarray(patch_mask).astype(bool)
    B, ph, pw = m.shape
    edges = np.linspace(1 / side, 1.0, side, endpoint=False)
    ids = np.zeros((B, ph * pw), dtype=np.int64)
    for b in range(B):
        rows, cols = int(m[b, :, 0].sum()), int(m[b, 0, :].sum())
        r = np.digitize(np.linspace(0, 1, rows, endpoint=False), edges, right=True) - 1
        c = np.digitize(np.linspace(0, 1, cols, endpoint=False), edges, right=True) - 1
        ids[b, m[b].reshape(-1)] = (r[:, None] * side + c[None, :]).reshape(-1)
    return ids


class VisionModel:
    epi = EPI_GELU_FAST       # the MLP's activation: GELU(approx="fast")

    def __init__(self, config: VisionConfig, engine_getter):
        self.config = config
        self.model_type = config.model_type
        self._engine = engine_getter
        self.w: Dict[str, torch.Tensor] = {}

    def sanitize(self, weights):
        return sanitize(weights, self.config.num_channels)

    def load(self, weights: Dict[str, torch.Tensor], prefix: str = "vision_model."):
        c, eng = self.config, self._engine()
        E, dev = c.hidden_size, eng.device

        def put(name, t):
            self.w[name] = t.to(device=dev, dtype=torch.bfloat16).contiguous()

        K = c.patch_size * c.patch_size * c.num_channels
        conv = weights[prefix + "embeddings.patch_embedding.weight"].reshape(E, K)
        convp = torch.zeros(E, (K + 7) // 8 * 8, dtype=conv.dtype)
        convp[:, :K] = conv
        put("patch", convp)
        put("patch.b", weights[prefix + "embeddings.patch_embedding.bias"])
        put("pos", weights[prefix + "embeddings.position_embedding.weight"])
        put("post.w", weights[prefix + "post_layernorm.weight"]); put("post.b", weights[prefix + "post_layernorm.bias"])
        pack_encoder_layers(weights, prefix, c.num_hidden_layers, put)

    def patch_position_ids(self, patch_attention_mask: Optional[np.ndarray], B: int, gh: int, gw: int) -> np.ndarray:
        """(B, gh * gw) rows of the position table"""
        if patch_attention_mask is None:
            patch_attention_mask = np.ones((B, gh, gw), dtype=bool)
        return bucketed_position_ids(patch_attention_mask, self.config.image_size // self.config.patch_size)

    def __call__(self, x: torch.Tensor, patch_attention_mask: Optional[np.ndarray] = None,
                 output_hidden_states: Optional[bool] = None):
        """x: NHWC fp32 (n_img, H, W, C) on the device -> (pooler_output fp32 (n_img * P, E), None, None).
        The reference calls the encoder WITHOUT an attention mask (vision.py:207): padded patches take
        part in attention, only their position id stays 0."""
        c, eng = self.config, self._engine()
        ops = TowerOps(eng)
        B, H, W, C = x.shape
        ps, E = c.patch_size, c.hidden_size
        gh, gw = H // ps, W // ps
        P = gh * gw
        T = B * P
        K = ps * ps * C
        w = self.w
        pos_ids = self.patch_position_ids(patch_attention_mask, B, gh, gw).astype(np.int32)
        pos_dev = torch.from_numpy(np.ascontiguousarray(pos_ids))
        with torch.cuda.stream(eng.stream):
            pos_dev = pos_dev.to(eng.device)
        x = x.contiguous()
        pat = SplitBuf(eng, T, K)
        ops.patchify(x, ps, pat)
        patch = ops.f32(T, E)
        ops.linear(pat, w["patch"], w["patch.b"], out32=patch, k_w=K)
        h = ops.f32(T, E)
        ops.embed(patch, None, w["pos"], pos_dev, h, B, P)
        encoder(ops, w, h, c.num_hidden_layers, n_heads=c.num_attention_heads, inter=c.intermediate_size, seg=P,
                eps=c.layer_norm_eps, epi=self.epi)
        pooled = ops.f32(T, E)
        ops.layer_norm(h, w["post.w"], w["post.b"], 1e-5, out32=pooled)   # nn.LayerNorm default eps (vision.py:184)
        return pooled, None, None
