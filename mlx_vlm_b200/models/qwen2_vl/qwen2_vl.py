"""Qwen2-VL `Model` — the per-model contract of the reference
(mlx_vlm/models/qwen2_vl/qwen2_vl.py:13-190): `get_input_embeddings`,
`merge_input_ids_with_image_features`, `vision_tower`, `language_model`, `layers`,
`sanitize`.  The decoder engine runs its built-in vision tower for this family only: the tower's
engine fields, arena rows and weight packing are here, the rest is models/engine_model.py.
"""
from __future__ import annotations

from typing import Dict

import torch

from ... import _native as N
from ...engine import Engine
from ..base import InputEmbeddingsFeatures
from ..engine_model import WeightArena  # noqa: F401  (the arena, importable from here as before)
from ..engine_model import EngineModel, _np, embed_merge, embed_tokens
from ..engine_model import weight_manifest as decoder_manifest
from .config import ModelConfig
from .language import LanguageModel
from .vision import VisionModel


def weight_manifest(c: N.Qwen2VLConfig, qk_norm: bool = False):
    """(engine name, shape) of every tensor of the engine layout, in a fixed order (DESIGN.md §3): the built-in
    vision tower and merger lead when the engine runs them (external_vision = 0), then the decoder"""
    if c.external_vision:
        return decoder_manifest(c, qk_norm)
    E, Em, mg = c.v_embed, c.v_mlp, c.v_merge ** 2 * c.v_embed
    out = [("v.patch_embed.w", (E, c.v_patch_dim))]
    for i in range(c.v_depth):
        q = f"v.blk.{i}."
        out += [(q + "ln1.w", (E,)), (q + "ln1.b", (E,)), (q + "ln2.w", (E,)), (q + "ln2.b", (E,)),
                (q + "qkv.w", (3 * E, E)), (q + "qkv.b", (3 * E,)), (q + "proj.w", (E, E)), (q + "proj.b", (E,)),
                (q + "fc1.w", (Em, E)), (q + "fc1.b", (Em,)), (q + "fc2.w", (E, Em)), (q + "fc2.b", (E,))]
    out += [("v.merger.ln.w", (E,)), ("v.merger.ln.b", (E,)), ("v.merger.fc1.w", (mg, mg)), ("v.merger.fc1.b", (mg,)),
            ("v.merger.fc2.w", (c.v_out, mg)), ("v.merger.fc2.b", (c.v_out,))]
    return out + decoder_manifest(c, qk_norm)


class Model(EngineModel):
    LanguageModel = LanguageModel
    VisionModel = VisionModel
    qkv_bias = True
    mrope = True
    forward_kwargs = True
    builtin_tower = True      # Qwen2.5-VL and Qwen3-VL run a decoder-only engine: their towers are their own

    def __init__(self, config: ModelConfig, device=None):
        super().__init__(config, device)
        self.vision_tower = self.VisionModel(config.vision_config, self._engine) if self.VisionModel else None

    # ------------------------------------------------------------- engine
    def native_config(self) -> N.Qwen2VLConfig:
        c = super().native_config()
        if self.builtin_tower:
            v = self.config.vision_config
            c.external_vision = 0
            c.v_depth, c.v_embed, c.v_heads = v.depth, v.embed_dim, v.num_heads
            c.v_mlp = int(v.embed_dim * v.mlp_ratio)
            c.v_patch_dim = v.in_channels * v.temporal_patch_size * v.patch_size * v.patch_size
            c.v_merge, c.v_out, c.v_ln_eps = v.spatial_merge_size, v.hidden_size, v.layer_norm_eps
        return c

    def _manifest(self):
        return weight_manifest(self.native_config(), self.qk_norm)

    # ------------------------------------------------------------ weights
    def sanitize(self, weights):
        """HF checkpoint names -> the reference's names (behaviour of qwen2_vl.py:179-190, pinned by
        tests/golden `sanitize_keys`): `visual.*` becomes `vision_tower.*`; tensors not yet under
        `language_model` get the `language_model.` prefix on their `model` / `lm_head` component."""
        renamed = {}
        for key, value in weights.items():
            name = key if "vision_tower" in key else key.replace("visual", "vision_tower")
            if "language_model" not in name:
                for part in ("model", "lm_head"):       # first match wins, like the reference's if/elif
                    if part in name:
                        name = name.replace(part, "language_model." + part)
                        break
            renamed[name] = value
        return renamed

    def _load_vision(self, weights: Dict[str, torch.Tensor]):
        """the built-in tower's and the merger's tensors, packed into the engine layout"""
        v = self.config.vision_config

        def get(name):
            if name not in w:
                raise KeyError(f"missing weight {name}")
            return w[name]

        w = self.vision_tower.sanitize({k: x for k, x in weights.items() if "vision_tower" in k})
        put = self._put
        put("v.patch_embed.w", get("vision_tower.patch_embed.proj.weight").reshape(v.embed_dim, -1))
        for i in range(v.depth):
            p, q = f"vision_tower.blocks.{i}.", f"v.blk.{i}."
            for a, b in (("norm1.weight", "ln1.w"), ("norm1.bias", "ln1.b"), ("norm2.weight", "ln2.w"),
                         ("norm2.bias", "ln2.b"), ("attn.qkv.weight", "qkv.w"), ("attn.qkv.bias", "qkv.b"),
                         ("attn.proj.weight", "proj.w"), ("attn.proj.bias", "proj.b"),
                         ("mlp.fc1.weight", "fc1.w"), ("mlp.fc1.bias", "fc1.b"),
                         ("mlp.fc2.weight", "fc2.w"), ("mlp.fc2.bias", "fc2.b")):
                put(q + b, get(p + a))
        for a, b in (("ln_q.weight", "ln.w"), ("ln_q.bias", "ln.b"), ("mlp.0.weight", "fc1.w"),
                     ("mlp.0.bias", "fc1.b"), ("mlp.2.weight", "fc2.w"), ("mlp.2.bias", "fc2.b")):
            put("v.merger." + b, get("vision_tower.merger." + a))

    def init_random(self, seed: int = 0, std: float = 0.02):
        """Seeded random-init at the configured shapes, generated on the device in arena order
        (benchmark weights; SURVEY §8d: N(0, 0.02), norm weights 1, norm biases 0).  A family without the
        built-in tower loads its reference-named `random_weights` instead."""
        if not self.builtin_tower:
            return super().init_random(seed, std)
        eng = self._engine()
        g = torch.Generator(device=eng.device).manual_seed(seed)
        arena = self._arena()
        for name, shape in self._manifest():
            v = arena.view(name)
            if name.endswith(("ln1.w", "ln2.w", "ln.w", ".ln1", ".ln2", "lm.norm")):
                v.fill_(1.0)              # norm weights 1
            elif name.endswith(("ln1.b", "ln2.b", "ln.b")):
                v.zero_()                 # norm biases 0
            else:
                v.copy_((torch.randn(shape, generator=g, device=eng.device, dtype=torch.float32) * std
                         ).to(torch.bfloat16))
            eng.set_weight(name, v)
        torch.cuda.synchronize(eng.device)
        return self

    # ------------------------------------------------------------- contract
    def get_input_embeddings(self, input_ids=None, pixel_values=None, **kwargs):
        """qwen2_vl.py:20-76."""
        if pixel_values is None:
            pixel_values = kwargs.get("pixel_values_videos", None)
        image_grid_thw = kwargs.get("image_grid_thw", None)
        video_grid_thw = kwargs.get("video_grid_thw", None)
        mask = kwargs.get("mask", None)
        grid_thw = image_grid_thw if image_grid_thw is not None else video_grid_thw
        eng = self._engine()
        ids_host = _np(input_ids)
        if ids_host.ndim == 1:
            ids_host = ids_host[None]
        lm = self.language_model
        if pixel_values is None:
            position_ids, rope_deltas = lm.get_rope_index(ids_host, attention_mask=mask)
            return InputEmbeddingsFeatures(inputs_embeds=embed_tokens(eng, ids_host),
                                           position_ids=position_ids, rope_deltas=rope_deltas)
        cached = kwargs.get("cached_image_features", None)
        if cached is not None:
            hidden_states = cached
        else:
            hidden_states = self.vision_tower(pixel_values, grid_thw, output_hidden_states=False)
        final = self.merge_input_ids_with_image_features(
            self.config.image_token_id, self.config.video_token_id, hidden_states, None, ids_host,
            _engine=eng)
        position_ids, rope_deltas = lm.get_rope_index(ids_host, image_grid_thw, video_grid_thw, mask)
        return InputEmbeddingsFeatures(inputs_embeds=final, position_ids=position_ids,
                                       rope_deltas=rope_deltas)

    @staticmethod
    def merge_input_ids_with_image_features(image_token_id, video_token_id, image_features,
                                            inputs_embeds, input_ids, _engine: Engine = None):
        """qwen2_vl.py:78-148.  Host: count validation (the reference's ValueError);
        device: one gather kernel (prefix sum of the image mask -> feature row).
        `inputs_embeds=None` fuses the embedding lookup into the same kernel."""
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        B, T = ids.shape
        mask = ids == image_token_id
        if mask.sum() == 0:
            mask = ids == video_token_id
        n_feats = int(image_features.shape[0])
        start = 0
        for b in range(B):
            n = int(mask[b].sum())
            if n > 0 and n_feats - start < n:
                raise ValueError(
                    f"Number of image token positions ({n}) does not match "
                    f"number of image features ({max(n_feats - start, 0)}) for batch {b}")
            start += n
        eng = _engine
        if eng is None:
            raise N.B200Error("merge_input_ids_with_image_features needs the model's engine "
                              "(call it through Model.get_input_embeddings or pass _engine=)")
        if inputs_embeds is None:       # the fused lookup: either token id takes a feature row
            return embed_merge(eng, ids, image_features, n_feats, image_token_id, video_token_id)
        return embed_merge(eng, ids, image_features, n_feats, inputs_embeds=inputs_embeds, rows=mask)
