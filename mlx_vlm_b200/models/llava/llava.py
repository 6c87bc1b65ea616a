"""LLaVA-1.5 `Model` — the per-model contract of the reference (mlx_vlm/models/llava/llava.py:32-150):
`get_input_embeddings` (CLIP tower -> feature layer -2 without the class token -> projector -> merge),
`_merge_input_ids_with_image_features`, `vision_tower`, `language_model`, `layers`, `sanitize`."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from ... import _native as N
from ...engine import Engine
from ..base import InputEmbeddingsFeatures
from ..qwen2_vl.language import _np
from ..qwen2_vl.qwen2_vl import WeightArena, _ids_to_device, weight_manifest
from ..tower_ops import EPI_GELU_EXACT, SplitBuf, TowerOps
from .config import ModelConfig
from .language import LanguageModel
from .vision import VisionModel


def embed_tokens(eng: Engine, ids_host: np.ndarray) -> torch.Tensor:
    ids_host = np.asarray(ids_host)
    if ids_host.ndim == 1:
        ids_host = ids_host[None]
    B, T = ids_host.shape
    out = eng.empty((B, T, eng.cfg.hidden))
    ids = _ids_to_device(eng, ids_host)
    N.check(eng.lib.b200_embed_merge(ids.data_ptr(), B, T, eng.weights["lm.embed"].data_ptr(), eng.cfg.hidden,
                                     0, 0, -1, -1, out.data_ptr(), 0, eng.s), "embed")
    return out


class Model:
    def __init__(self, config: ModelConfig, device=None):
        self.config = config
        self._device = torch.device(device) if device is not None else torch.device("cuda", 0)
        self._eng: Optional[Engine] = None
        self._weights: Optional[WeightArena] = None
        self.vision_tower = VisionModel(config.vision_config, self._engine)
        self.language_model = LanguageModel(config.text_config, config, self._engine)
        self.proj: Dict[str, torch.Tensor] = {}
        self.vision_feature_layer = config.vision_feature_layer
        self.vision_feature_select_strategy = config.vision_feature_select_strategy

    # ------------------------------------------------------------- engine (decoder only)
    def native_config(self) -> N.Qwen2VLConfig:
        t = self.config.text_config
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = t.hidden_size, t.num_hidden_layers, t.intermediate_size
        c.n_heads, c.n_kv_heads = t.num_attention_heads, t.num_key_value_heads
        c.head_dim = t.hidden_size // t.num_attention_heads
        c.vocab = t.vocab_size
        c.rms_eps, c.rope_theta = t.rms_norm_eps, t.rope_theta
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = c.head_dim // 2, 0, 0   # plain RoPE
        c.tie_embeddings = int(t.tie_word_embeddings)
        c.external_vision = 1
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = t.hidden_size, 1e-5
        return c

    def _engine(self) -> Engine:
        if self._eng is None:
            self._eng = Engine(self.native_config(), self._device)
        return self._eng

    @property
    def engine(self) -> Engine:
        return self._engine()

    def _arena(self) -> WeightArena:
        if self._weights is None:
            self._weights = WeightArena(weight_manifest(self.native_config()), self._engine().device)
        return self._weights

    @property
    def packed_weights(self) -> torch.Tensor:
        return self._arena().flat

    def _put(self, name, value):
        v = self._arena().view(name)
        v.copy_(value.reshape(v.shape).to(device=v.device, dtype=torch.bfloat16))
        self._engine().set_weight(name, v)

    # ------------------------------------------------------------- weights
    def sanitize(self, weights):
        return weights

    def load_weights(self, weights: Dict[str, torch.Tensor], strict: bool = True):
        """reference-named tensors (vision_tower.* / multi_modal_projector.* / language_model.*)"""
        eng = self._engine()
        t = self.config.text_config
        dev = eng.device
        hd = t.hidden_size // t.num_attention_heads
        QKV = (t.num_attention_heads + 2 * t.num_key_value_heads) * hd
        self.vision_tower.load(self.vision_tower.sanitize({k: v for k, v in weights.items() if k.startswith("vision_tower")}))
        for n in ("linear_1", "linear_2"):
            self.proj[n + ".w"] = weights[f"multi_modal_projector.{n}.weight"].to(device=dev, dtype=torch.bfloat16).contiguous()
            self.proj[n + ".b"] = weights[f"multi_modal_projector.{n}.bias"].to(device=dev, dtype=torch.bfloat16).contiguous()
        put = self._put
        put("lm.embed", weights["language_model.model.embed_tokens.weight"])
        put("lm.norm", weights["language_model.model.norm.weight"])
        if not t.tie_word_embeddings:
            put("lm.head", weights["language_model.lm_head.weight"])
        for i in range(t.num_hidden_layers):
            p, q = f"language_model.model.layers.{i}.", f"lm.{i}."
            put(q + "ln1", weights[p + "input_layernorm.weight"])
            put(q + "ln2", weights[p + "post_attention_layernorm.weight"])
            put(q + "wqkv", torch.cat([weights[p + f"self_attn.{n}_proj.weight"].to(dev) for n in "qkv"], 0))
            put(q + "bqkv", torch.zeros(QKV))      # Llama: no q/k/v bias
            put(q + "wo", weights[p + "self_attn.o_proj.weight"])
            put(q + "wgu", torch.cat([weights[p + "mlp.gate_proj.weight"].to(dev), weights[p + "mlp.up_proj.weight"].to(dev)], 0))
            put(q + "wd", weights[p + "mlp.down_proj.weight"])
        torch.cuda.synchronize(dev)

    def init_random(self, seed: int = 0, std: float = 0.02):
        """seeded random-init at the configured shapes (benchmarks; no checkpoints offline)"""
        from .weights import random_weights
        self.load_weights(random_weights(self.config, seed, std, self._engine().device))
        return self

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
        B, T = ids.shape
        tok = self.config.image_token_index
        n_pos = int((ids == tok).sum())
        flat = image_features.reshape(-1, image_features.shape[-1])
        if flat.shape[0] > n_pos:
            raise ValueError("Llava model supports only one image per input. Please check your input_ids and "
                             "pixel_values.")
        if flat.shape[0] < n_pos:
            raise ValueError(f"shape mismatch: {flat.shape[0]} image feature rows cannot fill {n_pos} <image> "
                             "positions")
        H = int(flat.shape[-1])
        out = eng.empty((B, T, H))
        feats = flat.contiguous()
        if inputs_embeds is None:
            ids_dev = _ids_to_device(eng, ids)
            N.check(eng.lib.b200_embed_merge(ids_dev.data_ptr(), B, T, eng.weights["lm.embed"].data_ptr(), H,
                                             feats.data_ptr(), flat.shape[0], int(tok), -1, out.data_ptr(), 0, eng.s),
                    "embed_merge")
            return out
        sent = B * T
        ids2 = np.where(ids == tok, sent, np.arange(B * T).reshape(B, T))
        ids_dev = _ids_to_device(eng, ids2)
        table = inputs_embeds.reshape(B * T, H).contiguous()
        N.check(eng.lib.b200_embed_merge(ids_dev.data_ptr(), B, T, table.data_ptr(), H, feats.data_ptr(), flat.shape[0],
                                         sent, sent, out.data_ptr(), 0, eng.s), "embed_merge")
        return out

    @property
    def layers(self):
        return self.language_model.layers

    def __call__(self, input_ids, pixel_values=None, mask=None, cache=None, **kwargs):
        feats = self.get_input_embeddings(input_ids, pixel_values, **kwargs)
        return self.language_model(input_ids, feats.inputs_embeds, mask=mask, cache=cache)
