"""Qwen3-VL configuration: the schema of reference mlx_vlm/models/qwen3_vl/config.py:30-127 as tables; `rope_scaling`
key normalisation ('rope_type' -> 'type') and validation; `head_dim` given explicitly (it need not be hidden / heads);
`text_config` deserialised only when it carries every required field, as in the reference."""
from __future__ import annotations

import inspect

from ..config_schema import config_class

_VISION = """
    model_type                str         'qwen3_vl'
    depth                     int         32
    hidden_size               int         1280
    intermediate_size         int         3420
    out_hidden_size           int         1536
    num_heads                 int         16
    image_size                int         384
    patch_size                int         14
    vocab_size                int         32000
    mlp_ratio                 float       4.0
    in_channels               int         3
    layer_norm_eps            float       1e-6
    spatial_patch_size        int         14
    spatial_merge_size        int         2
    tokens_per_second         int         2
    temporal_patch_size       int         2
    num_position_embeddings   int         2304
    window_size               int         112
    fullatt_block_indexes     List[int]   [7, 15, 23, 31]
    deepstack_visual_indexes  List[int]   []
"""
_TEXT = """
    model_type               str                                           -
    num_hidden_layers        int                                           -
    hidden_size              int                                           -
    intermediate_size        int                                           -
    num_attention_heads      int                                           -
    rms_norm_eps             float                                         -
    vocab_size               int                                           -
    num_key_value_heads      Optional[int]                                 -
    head_dim                 int                                           -
    rope_theta               float                                         -
    max_position_embeddings  int                                           -
    norm_topk_prob           bool                                          True
    rope_scaling             Optional[Dict[str,Union[float,str,bool,list]]]  {'type': 'default', 'mrope_section': [24, 20, 20]}
    tie_word_embeddings      bool                                          False
    attention_bias           bool                                          False
    hidden_act               str                                           'silu'
    use_final_norm           bool                                          True
"""
_MODEL = """
    text_config                      object                -
    vision_config                    object                -
    model_type                       str                   -
    ignore_index                     int                   -100
    image_token_id                   int                   151655
    video_token_id                   int                   151656
    image_token_index                Optional[int]         None
    video_token_index                Optional[int]         None
    vision_start_token_id            int                   151652
    vision_end_token_id              int                   151653
    vision_token_id                  int                   151654
    vision_feature_select_strategy   str                   'default'
    vision_feature_layer             int                   -2
    vocab_size                       int                   32000
    eos_token_id                     Optional[List[int]]   None
    skip_vision                      bool                  False
"""


def _text_rules(self):
    """config.py:76-90"""
    if self.num_key_value_heads is None:
        self.num_key_value_heads = self.num_attention_heads
    scaling = self.rope_scaling
    if scaling:
        if "type" not in scaling and "rope_type" in scaling:
            scaling["type"] = scaling.pop("rope_type")
        if not {"mrope_section", "type"} <= set(scaling):
            raise ValueError("rope_scaling must contain keys {'mrope_section', 'type'}")
        if scaling["type"] not in ("mrope", "default"):
            raise ValueError("rope_scaling type must be 'mrope' or 'default'")


def _mrope_section(self):
    """sections of the rotary half-dimension per position axis (default: rope_utils.py:1030-1040)"""
    return list((self.rope_scaling or {}).get("mrope_section") or (24, 20, 20))


def _model_rules(self):
    """config.py:112-116"""
    if self.image_token_index is None:
        self.image_token_index = self.image_token_id
    if self.video_token_index is None:
        self.video_token_index = self.video_token_id


def _kwargs(cls, params):
    return {k: v for k, v in params.items() if k in inspect.signature(cls).parameters}


def _from_dict(cls, params):
    """config.py:118-127: the vision dict is always deserialised, the text dict only when it has every required field"""
    params = dict(params)
    if isinstance(params.get("vision_config"), dict):
        params["vision_config"] = VisionConfig(**_kwargs(VisionConfig, params["vision_config"]))
    text = params.get("text_config")
    if isinstance(text, dict):
        required = [n for n, p in inspect.signature(TextConfig).parameters.items() if p.default is inspect.Parameter.empty]
        if all(n in text for n in required):
            params["text_config"] = TextConfig(**_kwargs(TextConfig, text))
    return cls(**_kwargs(cls, params))


VisionConfig = config_class("VisionConfig", __name__, _VISION)
TextConfig = config_class("TextConfig", __name__, _TEXT, _text_rules, {"mrope_section": property(_mrope_section)})
ModelConfig = config_class("ModelConfig", __name__, _MODEL, _model_rules, members={"from_dict": classmethod(_from_dict)})


def qwen3_vl_2b_config() -> "ModelConfig":
    """Qwen3-VL-2B-Instruct shapes, recalled from the checkpoint's published config.json (not checked against the
    file itself): text hidden 2048, 28 layers, 16 q / 8 kv heads of 128, intermediate 6144, tied head, rope theta
    5e6, interleaved M-RoPE sections [24, 20, 20]; vision depth 24 x 1024, 16 heads, intermediate 4096, patch 16,
    merge 2, DeepStack after blocks 5 / 11 / 17, 2304 position embeddings, output width 2048."""
    text = TextConfig(model_type="qwen3_vl", num_hidden_layers=28, hidden_size=2048, intermediate_size=6144,
                      num_attention_heads=16, rms_norm_eps=1e-6, vocab_size=151936, num_key_value_heads=8,
                      head_dim=128, rope_theta=5000000.0, max_position_embeddings=262144,
                      rope_scaling={"type": "default", "mrope_section": [24, 20, 20], "mrope_interleaved": True},
                      tie_word_embeddings=True)
    vision = VisionConfig(depth=24, hidden_size=1024, intermediate_size=4096, out_hidden_size=2048, num_heads=16,
                          patch_size=16, spatial_patch_size=16, spatial_merge_size=2, num_position_embeddings=2304,
                          deepstack_visual_indexes=[5, 11, 17])
    return ModelConfig(text_config=text, vision_config=vision, model_type="qwen3_vl", vocab_size=151936,
                       eos_token_id=[151645, 151643])
