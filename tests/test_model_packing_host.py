"""CPU: what every model family packs for the decoder engine, pinned by digest.

Each family's `Model` runs on a stand-in engine that records `set_weight` on the CPU, so `init_random` (and, for
LLaVA and Idefics2, `sanitize` + `load_weights` of a checkpoint with a PyTorch-layout patch conv) can be hashed
without a GPU: every engine weight (name, dtype, shape, bytes), every tensor the tower and the connector keep, the
LLaVA-Next newline vector, and every field of the engine config.  `v_ln_eps` is left out of an engine without its
built-in tower: only that tower reads it.  A change to how any family names, fuses, orders or rounds its weights
changes a digest."""
import hashlib
import importlib
import sys
import types

import pytest
import torch

FAMILIES = {
    "qwen2_vl": "c5fb10bf13b83aa9363adcf946f8453bda506aef2f3729f7f2a7420715be17e4",
    "qwen2_5_vl": "acb21bcebc68212f2175d7384818ada33f5f88ed7ba997f921780d175fac5eb6",
    "qwen3_vl": "b2a918d30a4e3dac3bc688bfcab5f6d6a6767d8e555f9346766f488aba9d7958",
    "llava": "1b2d0ad97d7ef24b90489e90ce0a4f62ebcb8c4d350831f9c27608dd947d0d9d",
    "llava_next": "bb5a057678e4c4600d65b02bf685d1549dfaa7a60a54ce371e624c0d0a0c1865",
    "idefics2": "e4038887ba599abe35744985e2c32d6332da3ab3b03ea33ebc12cc4703f6d7f8",
    "idefics3": "64875ff724d49044916010e8bacaabbfe0b8c56a3e8464fe08a66dc742273d9b",
    "smolvlm": "64875ff724d49044916010e8bacaabbfe0b8c56a3e8464fe08a66dc742273d9b",
}


class _StandInEngine:
    def __init__(self, cfg, device):
        self.cfg, self.device, self.stream, self.h = cfg, torch.device("cpu"), None, 0
        self.weights = {}
        self.lib = types.SimpleNamespace(b200_engine_set_axis_sel=lambda *a: 0)

    def set_weight(self, name, t):
        self.weights[name] = t


@pytest.fixture
def stand_in(monkeypatch):
    """Model classes of every family create a _StandInEngine; device syncs are no-ops."""
    for fam in FAMILIES:
        importlib.import_module(f"mlx_vlm_b200.models.{fam}")
    for name, mod in list(sys.modules.items()):
        if name.startswith("mlx_vlm_b200.models") and hasattr(mod, "Engine"):
            monkeypatch.setattr(mod, "Engine", _StandInEngine)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)


def _config(fam):
    C = importlib.import_module(f"mlx_vlm_b200.models.{fam}.config")
    t = dict(hidden_size=64, num_hidden_layers=2, intermediate_size=96, num_attention_heads=4, num_key_value_heads=2,
             vocab_size=100)
    qwen = fam.startswith("qwen")
    if fam in ("qwen2_vl", "qwen2_5_vl"):
        t["rope_scaling"] = {"type": "mrope", "mrope_section": [2, 3, 3]}
    if fam == "qwen3_vl":
        t.update(head_dim=32, rope_scaling={"rope_type": "default", "mrope_section": [4, 6, 6], "mrope_interleaved": True})
    if qwen:
        t.update(model_type=fam, rms_norm_eps=1e-6, rope_theta=10000.0, max_position_embeddings=4096)
    if fam == "qwen2_vl":
        v = dict(depth=2, embed_dim=32, hidden_size=64, num_heads=2)
    elif fam == "qwen2_5_vl":
        v = dict(depth=2, hidden_size=32, intermediate_size=48, num_heads=2, out_hidden_size=64, fullatt_block_indexes=[1])
    elif fam == "qwen3_vl":
        v = {}
    else:
        v = dict(hidden_size=32, num_hidden_layers=2, intermediate_size=48, num_attention_heads=2, image_size=28,
                 patch_size=14)
    kw = dict(text_config=C.TextConfig.from_dict(t) if qwen else C.TextConfig(**t),
              vision_config=C.VisionConfig.from_dict(v) if qwen else C.VisionConfig(**v))
    if qwen:
        kw["model_type"] = fam
    if fam == "idefics2":
        kw["perceiver_config"] = C.PerceiverConfig(resampler_n_latents=4, resampler_depth=1, resampler_n_heads=2,
                                                   resampler_head_dim=16, num_key_value_heads=1)
    return C.ModelConfig(**kw)


def _model(fam):
    M = importlib.import_module(f"mlx_vlm_b200.models.{fam}").Model
    return M(_config(fam), device="cpu")


def _digest(model):
    h = hashlib.sha256()

    def tensor(name, v):
        v = v.detach().contiguous()
        h.update(f"{name}|{v.dtype}|{tuple(v.shape)}|".encode())
        h.update(v.view(torch.uint8).numpy().tobytes())

    for name, v in sorted(model.engine.weights.items()):
        tensor(name, v)
    for owner in ("vision_tower", "vision_model", "connector"):
        for name, v in sorted(getattr(getattr(model, owner, None), "w", {}).items()):
            tensor(f"{owner}.{name}", v)
    if getattr(model, "image_newline", None) is not None:
        tensor("image_newline", model.image_newline)
    c = model.native_config()
    for field, _ in c._fields_:
        if field == "v_ln_eps" and c.external_vision == 1:
            continue
        value = getattr(c, field)
        h.update(f"{field}={list(value) if field == 'mrope_section' else value}|".encode())
    return h.hexdigest()


@pytest.mark.parametrize("fam", list(FAMILIES))
def test_init_random_packs_the_same_weights(stand_in, fam):
    assert _digest(_model(fam).init_random(1)) == FAMILIES[fam]


@pytest.mark.parametrize("fam", ["llava", "idefics2"])
def test_a_pytorch_layout_checkpoint_packs_like_init_random(stand_in, fam):
    """random_weights with the patch conv in the PyTorch [O, C, kH, kW] layout, through sanitize + load_weights"""
    model = _model(fam)
    W = importlib.import_module(f"mlx_vlm_b200.models.{fam}.weights").random_weights(model.config, 1, 0.02, "cpu")
    key = next(k for k in W if k.endswith("embeddings.patch_embedding.weight"))
    W[key] = W[key].permute(0, 3, 1, 2).contiguous()
    model.load_weights(model.sanitize(W))
    assert _digest(model) == FAMILIES[fam]
