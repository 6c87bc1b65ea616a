"""What every model family shares on the one decoder engine (engine.py): the packed weight arena, the embedding
lookup and feature merge, and `EngineModel`, the base of every family's `Model`.

`EngineModel` owns the engine and its arena, the engine config and the decoder's weight loader.  A family swaps its
component classes (`LanguageModel`, `VisionModel`, `Connector`) and declares how its decoder differs:
  * `decoder_prefix`: where the decoder's tensors sit in the checkpoint (`language_model.model.` or `language_model.`);
  * `qkv_bias`: q/k/v biases read from the checkpoint, or zeros;
  * `qk_norm`: per-head q/k RMSNorm weights (engine weights lm.<i>.qn / lm.<i>.kn);
  * `mrope`: rope sections from the config's `mrope_section`, or plain RoPE on one axis (head_dim // 2, 0, 0).
`head_dim` is the language model's.  Only Qwen2-VL runs the engine's built-in vision tower; every other engine is
decoder-only (`external_vision = 1`) and its tower fields hold one placeholder set.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from .. import _native as N
from ..engine import Engine


def _np(x, dtype=np.int64):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy().astype(dtype)
    return np.asarray(x, dtype=dtype)


def _ids_to_device(eng: Engine, ids_host: np.ndarray) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(ids_host, dtype=np.int32))
    with torch.cuda.stream(eng.stream):
        return t.to(eng.device)


def embed_merge(eng: Engine, ids: np.ndarray, feats: Optional[torch.Tensor] = None, n_feats: int = 0,
                image_id: int = -1, video_id: int = -1, inputs_embeds: Optional[torch.Tensor] = None,
                rows: Optional[np.ndarray] = None) -> torch.Tensor:
    """ids (B, T) host -> (B, T, H) bf16 in one gather kernel (prefix sum of the feature mask -> feature row).
    `inputs_embeds=None`: every token is looked up in `lm.embed`, and the k-th token whose id is `image_id` or
    `video_id` takes feature row k instead.  Otherwise the given (B, T, H) embeddings are the table (row b * T + t)
    and the positions where `rows` is set take the feature rows in order: they point at the sentinel row B * T, which
    is the only id that selects a feature."""
    B, T = ids.shape
    H = eng.cfg.hidden if feats is None else int(feats.shape[-1])
    out = eng.empty((B, T, H))
    if feats is not None:
        feats = feats.contiguous()
    if inputs_embeds is None:
        ids_dev = _ids_to_device(eng, ids)
        table = eng.weights["lm.embed"]
    else:
        sent = B * T
        ids_dev = _ids_to_device(eng, np.where(rows, sent, np.arange(B * T).reshape(B, T)))
        table = inputs_embeds.reshape(B * T, H).contiguous()
        image_id = video_id = sent
    N.check(eng.lib.b200_embed_merge(ids_dev.data_ptr(), B, T, table.data_ptr(), H, N.ptr(feats), n_feats,
                                     int(image_id), int(video_id), out.data_ptr(), 0, eng.s), "embed_merge")
    return out


def embed_tokens(eng: Engine, ids_host: np.ndarray) -> torch.Tensor:
    """nn.Embedding lookup (qwen2_vl/language.py:183) through the merge kernel with no features."""
    ids_host = np.asarray(ids_host)
    if ids_host.ndim == 1:
        ids_host = ids_host[None]
    return embed_merge(eng, ids_host)


def weight_manifest(c: N.Qwen2VLConfig, qk_norm: bool = False):
    """(engine name, shape) of every decoder tensor of the engine layout, in a fixed order (DESIGN.md §3)"""
    H, I = c.hidden, c.inter
    QKV = (c.n_heads + 2 * c.n_kv_heads) * c.head_dim
    out = [("lm.embed", (c.vocab, H)), ("lm.norm", (H,))]
    if not c.tie_embeddings:
        out.append(("lm.head", (c.vocab, H)))
    for i in range(c.n_layers):
        q = f"lm.{i}."
        out += [(q + "ln1", (H,)), (q + "ln2", (H,)), (q + "wqkv", (QKV, H)), (q + "bqkv", (QKV,)),
                (q + "wo", (H, c.n_heads * c.head_dim)), (q + "wgu", (2 * I, H)), (q + "wd", (H, I))]
        if qk_norm:
            out += [(q + "qn", (c.head_dim,)), (q + "kn", (c.head_dim,))]
    return out


class WeightArena:
    """ONE device buffer for all weights of a replica (views at 256-byte aligned offsets): the
    multi-GPU start-up is then a single NCCL broadcast of `flat` (parallel.broadcast_packed)."""

    def __init__(self, manifest, device):
        self.offsets = {}
        off = 0
        for name, shape in manifest:
            n = int(np.prod(shape))
            self.offsets[name] = (off, shape)
            off += (n + 127) // 128 * 128
        self.flat = torch.empty(off, dtype=torch.bfloat16, device=device)

    def view(self, name: str) -> torch.Tensor:
        off, shape = self.offsets[name]
        return self.flat[off:off + int(np.prod(shape))].view(*shape)


class EngineModel:
    LanguageModel = None          # the family's component class, like its VisionModel / Connector
    random_weights = None         # the family's weights.random_weights, as a staticmethod
    decoder_prefix = "language_model.model."
    qkv_bias = False
    qk_norm = False
    mrope = False
    forward_kwargs = False        # __call__ hands its keyword arguments (position ids, rope deltas) to the decoder

    def __init__(self, config, device=None):
        self.config = config
        self._device = torch.device(device) if device is not None else torch.device("cuda", 0)
        self._eng: Optional[Engine] = None
        self._weights: Optional[WeightArena] = None
        self.language_model = self.LanguageModel(config.text_config, config, self._engine)

    # ------------------------------------------------------------- engine
    def native_config(self) -> N.Qwen2VLConfig:
        t = self.config.text_config
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = t.hidden_size, t.num_hidden_layers, t.intermediate_size
        c.n_heads, c.n_kv_heads = t.num_attention_heads, t.num_key_value_heads
        c.head_dim = self.language_model.head_dim
        c.vocab = t.vocab_size
        c.rms_eps, c.rope_theta = t.rms_norm_eps, t.rope_theta
        sec = t.mrope_section if self.mrope else (c.head_dim // 2, 0, 0)
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = sec[0], sec[1], sec[2]
        c.tie_embeddings = int(t.tie_word_embeddings)
        c.external_vision = 1      # placeholder tower: only the built-in tower's kernels read these fields
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = t.hidden_size, 1e-6
        return c

    def _engine(self) -> Engine:
        if self._eng is None:
            self._eng = Engine(self.native_config(), self._device)
        return self._eng

    @property
    def engine(self) -> Engine:
        return self._engine()

    def _manifest(self):
        return weight_manifest(self.native_config(), self.qk_norm)

    def _arena(self) -> WeightArena:
        if self._weights is None:
            self._weights = WeightArena(self._manifest(), self._engine().device)
        return self._weights

    @property
    def packed_weights(self) -> torch.Tensor:
        """the flat device buffer every engine weight is a view of"""
        return self._arena().flat

    def _put(self, name: str, value: torch.Tensor):
        """copy `value` into the arena view of `name` (bf16) and register it with the engine"""
        v = self._arena().view(name)
        v.copy_(value.reshape(v.shape).to(device=v.device, dtype=torch.bfloat16))
        self._engine().set_weight(name, v)

    # ------------------------------------------------------------ weights
    def sanitize(self, weights):
        return weights

    def _load_vision(self, weights: Dict[str, torch.Tensor]):
        """the tower's and the connector's tensors; a text-only family has none"""

    def load_weights(self, weights: Dict[str, torch.Tensor], strict: bool = True):
        """Pack reference-named tensors: the family's tower and connector, then the decoder into the engine layout
        (bf16, device): q/k/v rows fused into wqkv, gate/up rows into wgu (DESIGN.md §3)."""
        self._load_vision(weights)
        t = self.config.text_config
        dev = self._engine().device
        pre = self.decoder_prefix

        def get(name):
            if name not in weights:
                raise KeyError(f"missing weight {name}")
            return weights[name]

        put = self._put
        put("lm.embed", get(pre + "embed_tokens.weight"))
        put("lm.norm", get(pre + "norm.weight"))
        if not t.tie_word_embeddings:
            put("lm.head", get("language_model.lm_head.weight"))
        qkv_rows = (t.num_attention_heads + 2 * t.num_key_value_heads) * self.language_model.head_dim
        for i in range(t.num_hidden_layers):
            p, q = f"{pre}layers.{i}.", f"lm.{i}."
            put(q + "ln1", get(p + "input_layernorm.weight"))
            put(q + "ln2", get(p + "post_attention_layernorm.weight"))
            put(q + "wqkv", torch.cat([get(p + f"self_attn.{n}_proj.weight").to(dev) for n in "qkv"], 0))
            if self.qkv_bias:
                put(q + "bqkv", torch.cat([get(p + f"self_attn.{n}_proj.bias").to(dev) for n in "qkv"], 0))
            else:
                put(q + "bqkv", torch.zeros(qkv_rows, dtype=torch.bfloat16, device=dev))
            if self.qk_norm:
                put(q + "qn", get(p + "self_attn.q_norm.weight"))
                put(q + "kn", get(p + "self_attn.k_norm.weight"))
            put(q + "wo", get(p + "self_attn.o_proj.weight"))
            put(q + "wgu", torch.cat([get(p + "mlp.gate_proj.weight").to(dev), get(p + "mlp.up_proj.weight").to(dev)], 0))
            put(q + "wd", get(p + "mlp.down_proj.weight"))
        torch.cuda.synchronize(dev)

    def init_random(self, seed: int = 0, std: float = 0.02):
        """seeded random-init at the configured shapes (benchmarks; no checkpoints offline)"""
        self.load_weights(self.random_weights(self.config, seed, std, self._engine().device))
        return self

    # ------------------------------------------------------------- contract
    @property
    def layers(self):
        return self.language_model.layers

    def __call__(self, input_ids, pixel_values=None, mask=None, cache=None, **kwargs):
        feats = self.get_input_embeddings(input_ids, pixel_values, **kwargs)
        lm_kwargs = {"pixel_values": pixel_values, **kwargs} if self.forward_kwargs else {}
        return self.language_model(input_ids, feats.inputs_embeds, mask=mask, cache=cache, **lm_kwargs)
