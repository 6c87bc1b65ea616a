"""Idefics2 `Model` — the per-model contract of the reference (mlx_vlm/models/idefics2/idefics2.py:36-300):
`get_input_embeddings` (padding-image removal, pixel mask -> patch mask, SigLIP tower -> connector
(modality MLP + Perceiver resampler) -> masked-scatter merge), `vision_model`, `language_model`,
`connector`, `layers`, `sanitize`.  Tower and connector run in fp32 like the reference
(`pooler_output.astype(pixel_values.dtype)`, idefics2.py:251); the merge rounds to bf16 once."""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from ... import _native as N
from ..base import InputEmbeddingsFeatures
from ..engine_model import EngineModel, _np, embed_merge, embed_tokens
from ..tower_ops import SplitBuf, TowerOps
from .config import ModelConfig
from .language import LanguageModel
from .vision import VisionModel
from .weights import random_weights


def real_image_indices(pixel_values: np.ndarray) -> List[int]:
    """idefics2.py:204-210: an all-zero image is padding and is dropped.  pixel_values (B, N, C, H, W)."""
    pv = np.asarray(pixel_values)
    flat = pv.reshape(pv.shape[0] * pv.shape[1], -1)
    return np.flatnonzero((flat == 0.0).sum(axis=1) != flat.shape[1]).tolist()


def patch_attention_mask(pixel_attention_mask: np.ndarray, patch_size: int) -> np.ndarray:
    """idefics2.py:226-243: a patch is valid iff any of its pixels is.  (n, H, W) -> (n, H/ps, W/ps) bool"""
    m = np.asarray(pixel_attention_mask)
    n, H, W = m.shape
    ph, pw = H // patch_size, W // patch_size
    m = m[:, :ph * patch_size, :pw * patch_size].reshape(n, ph, patch_size, pw, patch_size)
    return m.sum(axis=(2, 4)) > 0


class Connector:
    """modality projection (SwiGLU MLP) + Perceiver resampler (idefics2.py:36-171), fp32"""

    def __init__(self, config: ModelConfig, engine_getter):
        self.config = config
        self._engine = engine_getter
        self.w: Dict[str, torch.Tensor] = {}

    def load(self, weights, prefix="connector."):
        eng = self._engine()
        pc = self.config.perceiver_config

        def put(name, t):
            self.w[name] = t.to(device=eng.device, dtype=torch.bfloat16).contiguous()

        m = prefix + "modality_projection."
        put("mp.gu", torch.cat([weights[m + "gate_proj.weight"], weights[m + "up_proj.weight"]], 0))
        put("mp.down", weights[m + "down_proj.weight"])
        r = prefix + "perceiver_resampler."
        put("latents", weights[r + "latents"])
        put("norm", weights[r + "norm.weight"])
        for i in range(pc.resampler_depth):
            q = r + f"layers.{i}."
            put(f"{i}.ln_lat", weights[q + "input_latents_norm.weight"])
            put(f"{i}.ln_ctx", weights[q + "input_context_norm.weight"])
            put(f"{i}.ln_post", weights[q + "post_attention_layernorm.weight"])
            put(f"{i}.q", weights[q + "self_attn.q_proj.weight"])
            put(f"{i}.kv", torch.cat([weights[q + "self_attn.k_proj.weight"], weights[q + "self_attn.v_proj.weight"]], 0))
            put(f"{i}.o", weights[q + "self_attn.o_proj.weight"])
            put(f"{i}.gu", torch.cat([weights[q + "mlp.gate_proj.weight"], weights[q + "mlp.up_proj.weight"]], 0))
            put(f"{i}.down", weights[q + "mlp.down_proj.weight"])

    def __call__(self, feats: torch.Tensor, n_img: int) -> torch.Tensor:
        """feats fp32 (n_img * P, E) -> fp32 (n_img * n_latents, H)"""
        cfg, eng = self.config, self._engine()
        ops = TowerOps(eng)
        t, pc = cfg.text_config, cfg.perceiver_config
        H, I = t.hidden_size, t.intermediate_size
        E = feats.shape[1]
        P = feats.shape[0] // n_img
        nl, nh, nkv, hd = pc.resampler_n_latents, pc.resampler_n_heads, pc.num_key_value_heads, pc.resampler_head_dim
        w = self.w
        eps = t.rms_norm_eps
        # ---- modality projection: x = down(silu(gate f) * up f)
        fs = SplitBuf(eng, n_img * P, E)
        ops.split(feats, fs)
        gu = ops.f32(n_img * P, 2 * I)
        ops.linear(fs, w["mp.gu"], None, out32=gu)
        act = SplitBuf(eng, n_img * P, I)
        ops.swiglu(gu, act)
        x = ops.f32(n_img * P, H)
        ops.linear(act, w["mp.down"], None, out32=x)
        # ---- perceiver resampler: latents attend to [context; latents]
        h = ops.f32(n_img * nl, H)
        for b in range(n_img):   # h[b] = the learned latents (an fp32 copy made once at load time)
            N.check(eng.lib.b200_memcpy_d2d(h[b * nl:].data_ptr(), self._latents32(eng).data_ptr(), nl * H * 4, eng.s),
                    "memcpy_d2d")
        S = P + nl
        kvin = SplitBuf(eng, n_img * S, H)
        lat = SplitBuf(eng, n_img * nl, H)
        q32 = ops.f32(n_img * nl, nh * hd)
        kv32 = ops.f32(n_img * S, 2 * nkv * hd)
        o = SplitBuf(eng, n_img * nl, nh * hd)
        y = SplitBuf(eng, n_img * nl, H)
        gu2 = ops.f32(n_img * nl, 8 * H)
        act2 = SplitBuf(eng, n_img * nl, 4 * H)
        for i in range(pc.resampler_depth):
            ops.rms_norm(h, w[f"{i}.ln_lat"], eps, out_split=lat)
            ops.rms_norm(x, w[f"{i}.ln_ctx"], eps, out_split=kvin, seg_in=P, seg_out=S, seg_off=0)
            ops.rms_norm(h, w[f"{i}.ln_lat"], eps, out_split=kvin, seg_in=nl, seg_out=S, seg_off=P)
            ops.linear(lat, w[f"{i}.q"], None, out32=q32)
            ops.linear(kvin, w[f"{i}.kv"], None, out32=kv32)
            ops.attention((q32, nh * hd, hd), (kv32, 2 * nkv * hd, hd), (kv32[:, nkv * hd:], 2 * nkv * hd, hd),
                          n_heads=nh, n_kv=nkv, hd=hd, Lq=nl, S=S, n_seg=n_img, q_seg=nl, k_seg=S, scale=hd ** -0.5,
                          out_split=o)
            ops.linear(o, w[f"{i}.o"], None, out32=h, res32=h)
            ops.rms_norm(h, w[f"{i}.ln_post"], eps, out_split=y)
            ops.linear(y, w[f"{i}.gu"], None, out32=gu2)
            ops.swiglu(gu2, act2)
            ops.linear(act2, w[f"{i}.down"], None, out32=h, res32=h)
        out = ops.f32(n_img * nl, H)
        ops.rms_norm(h, w["norm"], eps, out32=out)
        return out

    def _latents32(self, eng):
        if "latents32" not in self.w:
            with torch.cuda.stream(eng.stream):
                self.w["latents32"] = self.w["latents"].to(torch.float32).contiguous()   # once, at load time
            eng.stream.synchronize()
        return self.w["latents32"]


class Model(EngineModel):
    LanguageModel = LanguageModel
    VisionModel = VisionModel
    Connector = Connector
    random_weights = staticmethod(random_weights)
    decoder_prefix = "language_model."

    def __init__(self, config: ModelConfig, device=None):
        super().__init__(config, device)
        self.vision_model = self.VisionModel(config.vision_config, self._engine)
        self.connector = self.Connector(config, self._engine)

    def sanitize(self, weights):
        """reference idefics2.py sanitize: HF `model.*` prefixes are dropped, lm_head goes under language_model"""
        out = {}
        for k, v in weights.items():
            if k.startswith("model."):
                k = k[len("model."):]
            if k.startswith("text_model."):
                k = "language_model." + k[len("text_model."):]
            if k.startswith("lm_head."):
                k = "language_model." + k
            out[k] = v
        return out

    def _load_vision(self, weights: Dict[str, torch.Tensor]):
        self.vision_model.load(self.vision_model.sanitize({k: v for k, v in weights.items() if k.startswith("vision_model.")}))
        self.connector.load(weights)

    # ------------------------------------------------------------- contract
    def encode_image(self, pixel_values, pixel_attention_mask=None) -> torch.Tensor:
        """pixel_values (B, n, C, H, W) fp32 (device tensor or numpy) -> image features (n_real * n_latents, H) bf16"""
        eng = self._engine()
        cfg = self.config
        pv_host = pixel_values.detach().cpu().numpy() if isinstance(pixel_values, torch.Tensor) else np.asarray(pixel_values)
        B, n, C, Hh, Ww = pv_host.shape
        keep = real_image_indices(pv_host)
        if pixel_attention_mask is None:
            pam = np.ones((len(keep), Hh, Ww), dtype=bool)
        else:
            pam = _np(pixel_attention_mask, dtype=bool).reshape(B * n, Hh, Ww)[keep]
        pmask = patch_attention_mask(pam, cfg.vision_config.patch_size)
        if isinstance(pixel_values, torch.Tensor) and pixel_values.is_cuda:
            with torch.cuda.stream(eng.stream):
                x = pixel_values.reshape(B * n, C, Hh, Ww)[keep].to(torch.float32).permute(0, 2, 3, 1).contiguous()
        else:
            t = torch.from_numpy(np.ascontiguousarray(pv_host.reshape(B * n, C, Hh, Ww)[keep].transpose(0, 2, 3, 1),
                                                      dtype=np.float32)).pin_memory()
            with torch.cuda.stream(eng.stream):
                x = t.to(eng.device, non_blocking=True)
        pooled, _, _ = self.vision_model(x, patch_attention_mask=pmask, output_hidden_states=True)
        feats32 = self.connector(pooled, len(keep))
        feats = eng.empty(tuple(feats32.shape))
        N.check(eng.lib.b200_cast_f32_bf16(feats32.data_ptr(), feats.data_ptr(), feats32.numel(), eng.s), "cast")
        return feats

    def get_input_embeddings(self, input_ids=None, pixel_values=None, **kwargs):
        eng = self._engine()
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        if pixel_values is None:
            return InputEmbeddingsFeatures(inputs_embeds=embed_tokens(eng, ids))
        cached = kwargs.get("cached_image_features", None)
        feats = cached if cached is not None else self.encode_image(pixel_values, kwargs.get("pixel_attention_mask", None))
        return InputEmbeddingsFeatures(inputs_embeds=self._prepare_inputs_for_multimodal(feats, None, ids))

    def _prepare_inputs_for_multimodal(self, image_features, inputs_embeds, input_ids):
        """idefics2.py:263-280 + masked_scatter :15-33: the flattened features fill, in order, the <image> rows"""
        eng = self._engine()
        ids = _np(input_ids)
        if ids.ndim == 1:
            ids = ids[None]
        tok = self.config.image_token_index
        n_tok = int((ids == tok).sum())
        flat = image_features.reshape(-1, image_features.shape[-1])
        H = int(flat.shape[-1])
        if n_tok * H != flat.numel():
            raise ValueError(f"Image features and image tokens do not match: tokens: {n_tok}, features {flat.shape[0]}")
        if inputs_embeds is None:
            return embed_merge(eng, ids, flat, flat.shape[0], tok)
        return embed_merge(eng, ids, flat, flat.shape[0], inputs_embeds=inputs_embeds, rows=ids == tok)
