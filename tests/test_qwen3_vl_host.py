"""Qwen3-VL host rules against the reference's own source (tests/golden/qwen3_vl_golden.json, made by
tests/golden/make_qwen3_vl_golden.py), and the decoder restatement of tests/qwen3vl_ref.py in fp32 against
HuggingFace transformers' Qwen3VLForConditionalGeneration on the same random weights."""
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "qwen3_vl_golden.json")))


def _tiny_config(tied=True, hd=64):
    from mlx_vlm_b200.models.qwen3_vl import ModelConfig, TextConfig, VisionConfig
    text = TextConfig(model_type="qwen3_vl", num_hidden_layers=2, hidden_size=256, intermediate_size=512,
                      num_attention_heads=4, rms_norm_eps=1e-6, vocab_size=512, num_key_value_heads=2, head_dim=hd,
                      rope_theta=5000000.0, max_position_embeddings=4096,
                      rope_scaling={"rope_type": "default", "mrope_section": [8, 12, 12], "mrope_interleaved": True},
                      tie_word_embeddings=tied)
    return ModelConfig(text_config=text, vision_config=VisionConfig(depth=1), model_type="qwen3_vl", vocab_size=512)


def test_interleaved_selector_matches_reference():
    from mlx_vlm_b200.models.qwen3_vl.qwen3_vl import interleaved_position_selector
    from qwen3vl_ref import interleaved_selector
    for case in G["selector"]:
        assert interleaved_position_selector(case["section"], case["freq_dim"]).tolist() == case["sel"]
        assert interleaved_selector(case["section"], case["freq_dim"]).tolist() == case["sel"]


def test_sanitize_matches_reference():
    from mlx_vlm_b200.models.qwen3_vl import Model
    out = Model.sanitize(None, {k: 0 for k in G["sanitize"]["in"]})
    assert list(out.keys()) == G["sanitize"]["out"]


def test_config_rules_match_reference():
    from mlx_vlm_b200.models.qwen3_vl import TextConfig
    for case in G["config"]:
        kw = dict(model_type="qwen3_vl", num_hidden_layers=1, hidden_size=8, intermediate_size=8, num_attention_heads=4,
                  rms_norm_eps=1e-6, vocab_size=8, num_key_value_heads=None, head_dim=2, rope_theta=1.0,
                  max_position_embeddings=8, rope_scaling=None if case["in"] is None else dict(case["in"]))
        if case["error"] is not None:
            with pytest.raises(ValueError):
                TextConfig(**kw)
            continue
        t = TextConfig(**kw)
        assert t.rope_scaling == case["out"] and t.num_key_value_heads == case["kv"]


def test_from_dict_nested_and_head_dim():
    from mlx_vlm_b200.models.qwen3_vl import ModelConfig, TextConfig, VisionConfig
    from mlx_vlm_b200.models.qwen3_vl.config import qwen3_vl_2b_config
    c = qwen3_vl_2b_config()
    d = {"model_type": "qwen3_vl", "text_config": dict(c.text_config.__dict__), "vision_config": dict(c.vision_config.__dict__),
         "image_token_id": 151655, "unknown_key": 1}
    m = ModelConfig.from_dict(d)
    assert isinstance(m.text_config, TextConfig) and isinstance(m.vision_config, VisionConfig)
    assert m.text_config.head_dim == 128 and m.vision_config.deepstack_visual_indexes == [5, 11, 17]
    assert m.image_token_index == 151655
    partial = {"model_type": "qwen3_vl", "text_config": {"hidden_size": 8}, "vision_config": {}}
    assert isinstance(ModelConfig.from_dict(partial).text_config, dict)   # the reference keeps an incomplete dict


def test_text_rope_index_matches_reference():
    from mlx_vlm_b200.models.qwen3_vl import LanguageModel
    cfg = _tiny_config()
    lm = LanguageModel(cfg.text_config, cfg, None)
    for case in G["rope_text"]:
        mask = None if case["mask"] is None else np.asarray(case["mask"])
        pos, deltas = lm.get_rope_index(np.asarray(case["ids"]), attention_mask=mask)
        assert np.asarray(pos).tolist() == case["pos"] and np.asarray(deltas).tolist() == case["deltas"]


def test_unsupported_inputs_raise():
    from mlx_vlm_b200.models.qwen3_vl import Model
    cfg = _tiny_config()
    cfg.model_type = "qwen3_vl_moe"
    with pytest.raises(NotImplementedError, match="qwen3_vl_moe"):
        Model(cfg, device="cpu")
    m = Model(_tiny_config(), device="cpu")
    with pytest.raises(NotImplementedError, match="qwen3_vl"):
        m.get_input_embeddings(np.zeros((1, 4), np.int64), pixel_values=np.zeros((4, 8), np.float32))
    from mlx_vlm_b200.utils import get_model_and_args
    with pytest.raises(ValueError, match="qwen3_vl_moe"):
        get_model_and_args({"model_type": "qwen3_vl_moe"})


@pytest.mark.parametrize("tied,hd", [(True, 64), (False, 128)])
def test_reference_fp32_matches_transformers(tied, hd):
    transformers = pytest.importorskip("transformers")
    from qwen3vl_ref import head, host_weights, lm_forward
    from oracle.mlx_semantics import Rounder
    from oracle.qwen2vl import OracleKVCache
    cfg = _tiny_config(tied, hd)
    t = cfg.text_config
    W = host_weights(cfg, seed=1, std=0.05)
    hf_cfg = transformers.Qwen3VLConfig(
        text_config=dict(hidden_size=t.hidden_size, num_hidden_layers=t.num_hidden_layers,
                         intermediate_size=t.intermediate_size, num_attention_heads=t.num_attention_heads,
                         num_key_value_heads=t.num_key_value_heads, head_dim=t.head_dim, vocab_size=t.vocab_size,
                         rms_norm_eps=t.rms_norm_eps, rope_theta=t.rope_theta,
                         rope_scaling={"rope_type": "default", "mrope_section": t.mrope_section, "mrope_interleaved": True},
                         max_position_embeddings=4096, tie_word_embeddings=tied),
        vision_config=dict(depth=1, hidden_size=64, intermediate_size=128, num_heads=2, out_hidden_size=t.hidden_size,
                           deepstack_visual_indexes=[]),
        tie_word_embeddings=tied)
    hf = transformers.Qwen3VLForConditionalGeneration(hf_cfg).float().eval()
    sd = {}
    for k, v in W.items():
        k2 = k.replace("language_model.model.", "model.language_model.").replace("language_model.lm_head", "lm_head")
        sd[k2] = v
    if tied:
        sd["lm_head.weight"] = W["language_model.model.embed_tokens.weight"]
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all(m.startswith("model.visual") for m in missing), (missing, unexpected)
    ids = torch.as_tensor(np.random.default_rng(0).integers(0, t.vocab_size, size=(1, 11)))
    with torch.no_grad():
        want = hf(input_ids=ids).logits[0].float()
    R = Rounder("f32")
    pos = np.broadcast_to(np.arange(11)[None], (1, 11))
    h = lm_forward(t, W, W["language_model.model.embed_tokens.weight"][ids], pos,
                   [OracleKVCache() for _ in range(t.num_hidden_layers)], R)
    got = head(t, W, h, R)[0]
    rel = float((got - want).norm() / want.norm())
    assert rel < 1e-5, rel
    # the interleaved table with three different position rows (an image's t / h / w ids) against HF's rotary
    p3 = np.stack([np.arange(11), np.arange(11) * 2 % 5, np.arange(11) * 3 % 7])[:, None, :]
    with torch.no_grad():
        want3 = hf.model.language_model(input_ids=ids, position_ids=torch.as_tensor(p3)).last_hidden_state[0]
    h3 = lm_forward(t, W, W["language_model.model.embed_tokens.weight"][ids], p3,
                    [OracleKVCache() for _ in range(t.num_hidden_layers)], R)[0]
    assert float((h3 - want3).norm() / want3.norm()) < 1e-5
