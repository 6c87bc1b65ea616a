"""The config classes of every model family on the CUDA path are generated from tables (models/config_schema.py); this pins
them field by field — names, order, defaults — against the reference's dataclasses as recorded with `ast` by
tests/golden/make_config_golden.py, and checks the behaviour attached to them."""
import dataclasses
import importlib
import json
import os

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "config_schema_golden.json")) as f:
    GOLD = json.load(f)

FAMILIES = ("llava", "llava_next", "idefics2", "idefics3", "smolvlm", "qwen2_5_vl", "qwen2_vl")


@pytest.mark.parametrize("family", FAMILIES)
def test_schema_matches_the_reference(family):
    mod = importlib.import_module(f"mlx_vlm_b200.models.{family}.config")
    for cname, rows in GOLD[family].items():
        cls = getattr(mod, cname)
        want, seen = [], set()
        for name, default in rows:            # a field the reference declares twice keeps its first position, last default
            if name in seen:
                want = [[n, default if n == name else d] for n, d in want]
                continue
            seen.add(name)
            want.append([name, default])
        got = dataclasses.fields(cls)
        assert [f.name for f in got] == [n for n, _ in want], (family, cname)
        for f, (name, default) in zip(got, want):
            if default == "<required>":
                continue                      # the product may add a convenience default where the reference has none
            if isinstance(default, dict) and "factory" in default:
                assert f.default_factory is not dataclasses.MISSING, (family, cname, name)
                made = f.default_factory()
                if isinstance(default["factory"], list):
                    assert made == default["factory"], (family, cname, name)
                else:                         # `TextConfig()` / `VisionConfig()`
                    assert type(made).__name__ == default["factory"].split("(")[0], (family, cname, name)
                continue
            assert f.default == default and type(f.default) is type(default), (family, cname, name, f.default, default)


def test_from_dict_keeps_every_known_key_and_builds_nested_configs():
    from mlx_vlm_b200.models import idefics2, idefics3, llava, llava_next, smolvlm
    for mod, extra in ((llava, {}), (llava_next, {}), (idefics3, {"scale_factor": 3}), (smolvlm, {"scale_factor": 3}),
                       (idefics2, {"perceiver_config": {"resampler_depth": 1, "junk": 0}})):
        raw = {"model_type": "x", "ignore_index": -7, "vocab_size": 11, "eos_token_id": [1, 2], "junk": 1,
               "text_config": {"hidden_size": 64, "num_attention_heads": 4, "num_key_value_heads": None, "junk": 2},
               "vision_config": {"hidden_size": 32, "junk": 3}, **extra}
        before = json.dumps(raw, sort_keys=True)
        c = mod.ModelConfig.from_dict(raw)
        assert json.dumps(raw, sort_keys=True) == before, "from_dict must not modify its argument"
        assert (c.model_type, c.ignore_index, c.vocab_size, c.eos_token_id) == ("x", -7, 11, [1, 2])
        assert c.text_config.hidden_size == 64 and c.text_config.num_key_value_heads == 4
        assert c.vision_config.hidden_size == 32
        if "scale_factor" in extra:
            assert c.scale_factor == 3
        if "perceiver_config" in extra:
            assert c.perceiver_config.resampler_depth == 1
    d = smolvlm.ModelConfig()                      # default factories
    assert d.text_config.num_attention_heads == 32 and d.vision_config.hidden_size == 1152 and d.image_token_index == 49153
    a, b = smolvlm.ModelConfig(), smolvlm.ModelConfig()
    assert a.text_config is not b.text_config


def test_list_defaults_are_not_shared():
    from mlx_vlm_b200.models.qwen2_5_vl import VisionConfig
    a, b = VisionConfig(), VisionConfig()
    a.fullatt_block_indexes.append(99)
    assert b.fullatt_block_indexes == [7, 15, 23, 31]


def test_llama_rope_scaling_rules():
    from mlx_vlm_b200.models.llava import TextConfig
    assert TextConfig().num_key_value_heads == 32
    assert TextConfig(rope_scaling={"type": "linear", "factor": 2.0}).rope_scaling["factor"] == 2.0
    with pytest.raises(ValueError, match="keys"):
        TextConfig(rope_scaling={"type": "linear"})
    with pytest.raises(ValueError, match="linear"):
        TextConfig(rope_scaling={"type": "yarn", "factor": 2.0})
