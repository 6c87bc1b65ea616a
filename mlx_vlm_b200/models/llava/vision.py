"""CLIP ViT-L/14 vision tower of LLaVA-1.5 (reference mlx_vlm/models/llava/vision.py:108-221), as the
reference computes it for this model: in fp32 with bf16-valued weights (`pixel_values` is never cast,
llava.py:61-63).  GEMMs run on the tensor cores over split operands (models/tower_ops.py), the rest in
fp32 kernels (csrc/tower_f32.cu)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from ..tower_ops import EPI_GELU_FAST, SplitBuf, TowerOps, encoder, pack_encoder_layers, sanitize
from .config import VisionConfig


class _States(list):
    """hidden states of the encoder; only the layers that were asked for are materialised"""


class VisionModel:
    def __init__(self, config: VisionConfig, engine_getter):
        self.config = config
        self.model_type = config.model_type
        self._engine = engine_getter
        self.w: Dict[str, torch.Tensor] = {}

    def sanitize(self, weights):
        """reference vision.py:196-221"""
        return sanitize(weights, self.config.num_channels)

    def load(self, weights: Dict[str, torch.Tensor]):
        """weights: reference names below `vision_tower.vision_model.` (post-sanitize layouts)"""
        c, eng = self.config, self._engine()
        E = c.hidden_size
        dev = eng.device
        p = "vision_tower.vision_model."

        def put(name, t):
            self.w[name] = t.to(device=dev, dtype=torch.bfloat16).contiguous()

        K = c.patch_size * c.patch_size * c.num_channels
        conv = weights[p + "embeddings.patch_embedding.weight"].reshape(E, K)
        convp = torch.zeros(E, (K + 7) // 8 * 8, dtype=conv.dtype)
        convp[:, :K] = conv
        put("patch", convp)
        put("cls", weights[p + "embeddings.class_embedding"])
        put("pos", weights[p + "embeddings.position_embedding.weight"])
        for n in ("pre_layrnorm", "post_layernorm"):
            if p + n + ".weight" in weights:
                put(n + ".w", weights[p + n + ".weight"])
                put(n + ".b", weights[p + n + ".bias"])
        pack_encoder_layers(weights, p, c.num_hidden_layers, put)

    def __call__(self, x: torch.Tensor, output_hidden_states: Optional[bool] = None, feature_layer: int = -2):
        """x: pixel_values NHWC fp32 (B, H, W, C) on the device -> (None, selected state, states) where
        `states[feature_layer]` is the fp32 hidden state (B * (P + 1), E) after that encoder layer
        (index 0 = after the pre-LayerNorm).  The reference runs all layers and returns every state
        (vision.py:160-185); the layers after the selected one cannot influence it and are skipped."""
        c, eng = self.config, self._engine()
        ops = TowerOps(eng)
        B, H, W, C = x.shape
        ps, E = c.patch_size, c.hidden_size
        P = (H // ps) * (W // ps)
        L = P + 1
        T = B * L
        K = ps * ps * C
        w = self.w
        x = x.contiguous()
        pat = SplitBuf(eng, B * P, K)
        ops.patchify(x, ps, pat)
        patch = ops.f32(B * P, E)
        ops.linear(pat, w["patch"], None, out32=patch, k_w=K)
        emb = ops.f32(T, E)
        ops.embed(patch, w["cls"], w["pos"], None, emb, B, P)
        h = ops.f32(T, E)
        ops.layer_norm(emb, w["pre_layrnorm.w"], w["pre_layrnorm.b"], 1e-5, out32=h)   # nn.LayerNorm default eps
        n_states = c.num_hidden_layers + 1
        want = feature_layer % n_states
        encoder(ops, w, h, want, n_heads=c.num_attention_heads, inter=c.intermediate_size, seg=L, eps=c.layer_norm_eps,
                epi=EPI_GELU_FAST)
        states = _States([None] * n_states)
        states[want] = h
        return None, h, states
