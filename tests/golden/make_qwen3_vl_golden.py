#!/usr/bin/env python
"""Golden vectors for the Qwen3-VL decoder's host rules: the reference's own `_interleaved_position_selector`
(mlx_vlm/models/rope_utils.py), `Model.sanitize` (models/qwen3_vl/qwen3_vl.py), `TextConfig.__post_init__`
(models/qwen3_vl/config.py) and the text branch of `LanguageModel.get_rope_index` (models/qwen3_vl/language.py) are
extracted with `ast` and EXECUTED over the numpy stand-in for mlx.core of make_golden.py.
Writes tests/golden/qwen3_vl_golden.json.   usage: python tests/golden/make_qwen3_vl_golden.py"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import load, make_mx, tolist  # noqa: E402

OUT = os.path.join(HERE, "qwen3_vl_golden.json")


def main():
    from typing import Optional, Sequence
    mx = make_mx()
    mx.arange = lambda *a, dtype=None: np.arange(*a, dtype=dtype)
    mx.array = lambda x, dtype=None: np.array(x, dtype=dtype)
    ns = {"mx": mx, "np": np, "Optional": Optional, "Sequence": Sequence}
    sel, w1 = load(ns, "models/rope_utils.py", "_interleaved_position_selector")
    san, w2 = load(ns, "models/qwen3_vl/qwen3_vl.py", "sanitize", "Model")
    post, w3 = load(ns, "models/qwen3_vl/config.py", "__post_init__", "TextConfig")
    rope, w4 = load(ns, "models/qwen3_vl/language.py", "get_rope_index", "LanguageModel")
    golden = {"_about": "reference qwen3_vl host rules executed over a numpy stand-in",
              "provenance": {"selector": w1, "sanitize": w2, "text_post_init": w3, "get_rope_index": w4}}
    golden["selector"] = [{"section": s, "freq_dim": f, "sel": tolist(sel(s, f))}
                          for s, f in (([24, 20, 20], 64), ([16, 24, 24], 64), ([8, 12, 12], 32), ([4, 6, 6], 16),
                                       ([24, 20, 20], 32))]
    keys = ["model.language_model.layers.0.self_attn.q_norm.weight", "model.language_model.embed_tokens.weight",
            "model.visual.blocks.0.attn.qkv.weight", "model.visual.deepstack_merger_list.0.norm.weight",
            "lm_head.weight", "language_model.model.norm.weight", "vision_tower.patch_embed.proj.weight",
            "model.language_model.norm.weight", "visual.merger.linear_fc1.weight"]
    golden["sanitize"] = {"in": keys, "out": list(san(None, {k: 0 for k in keys}).keys())}
    cases = []
    for rs in ({"rope_type": "default", "mrope_section": [24, 20, 20], "mrope_interleaved": True},
               {"type": "mrope", "mrope_section": [16, 24, 24]}, {"rope_type": "yarn", "mrope_section": [1, 2, 3]},
               {"mrope_section": [24, 20, 20]}, None):
        self = types.SimpleNamespace(num_key_value_heads=None, num_attention_heads=4, rope_scaling=None if rs is None else dict(rs))
        try:
            post(self)
            cases.append({"in": rs, "out": self.rope_scaling, "kv": self.num_key_value_heads, "error": None})
        except ValueError as e:
            cases.append({"in": rs, "out": None, "kv": None, "error": str(e)})
    golden["config"] = cases
    rcases = []
    for ids, mask in (([[5, 6, 7, 8]], None), ([[0, 0, 5, 6, 7], [5, 6, 7, 8, 9]], [[0, 0, 1, 1, 1], [1, 1, 1, 1, 1]])):
        self = types.SimpleNamespace(config=types.SimpleNamespace(
            vision_config=types.SimpleNamespace(spatial_merge_size=2), image_token_id=151655, video_token_id=151656,
            vision_start_token_id=151652))
        m = None if mask is None else np.asarray(mask, dtype=np.int64)
        pos, deltas = rope(self, np.asarray(ids, dtype=np.int64), None, None, m)
        rcases.append({"ids": ids, "mask": mask, "pos": tolist(pos), "deltas": tolist(deltas)})
    golden["rope_text"] = rcases
    with open(OUT, "w") as f:
        json.dump(golden, f)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
