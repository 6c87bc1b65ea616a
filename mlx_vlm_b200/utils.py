"""Load / input preparation with the reference's surface (mlx_vlm/utils.py:
`load` :1065-1119, `load_model` :736-987, `load_config` :1175-1210,
`prepare_inputs` :1918-2136, `load_image`/`process_image` :1503-1567,
`StoppingCriteria` :2191-2249).

Device-first differences: safetensors shards are memory-mapped on the host and every tensor is
packed (q/k/v and gate/up fused, conv layout fixed) straight into ONE device arena
(`Model.packed_weights`, bf16) — which is also what a multi-GPU start-up broadcasts with a single
NCCL call; inputs are moved to the device with one pinned-memory H2D copy per tensor on the
generation stream.  `lazy` has no meaning here (weights must be resident for the kernels);
`revision` is rejected (local directories only, no hub).
"""
from __future__ import annotations

import glob
import importlib
import json
import os
from typing import Any, Dict, List, Optional, Union

import numpy as np
import torch

MODEL_REMAPPING: Dict[str, str] = {}


def get_model_and_args(config: dict):
    """utils.py:588-635: import mlx_vlm_b200.models.<model_type>."""
    model_type = MODEL_REMAPPING.get(config["model_type"].lower(), config["model_type"].lower())
    try:
        arch = importlib.import_module(f"mlx_vlm_b200.models.{model_type}")
    except ImportError as e:
        raise ValueError(f"Model type {model_type} not supported by the CUDA engine yet.") from e
    return arch, model_type


def load_config(model_path: str) -> dict:
    with open(os.path.join(model_path, "config.json"), "r") as f:
        config = json.load(f)
    gen = os.path.join(model_path, "generation_config.json")
    if os.path.exists(gen):
        try:
            with open(gen, "r") as f:
                g = json.load(f)
            if "eos_token_id" in g:
                config["eos_token_id"] = g["eos_token_id"]
        except Exception:
            pass
    return config


def _read_safetensors(path: str) -> Dict[str, torch.Tensor]:
    from safetensors import safe_open
    out = {}
    with safe_open(path, framework="pt", device="cpu") as f:
        for k in f.keys():
            out[k] = f.get_tensor(k)
    return out


def load_model(model_path: str, lazy: bool = False, strict: bool = True, device=None, **kwargs):
    """config.json -> module -> safetensors -> sanitize -> engine weights."""
    config = load_config(model_path)
    files = sorted(glob.glob(os.path.join(model_path, "*.safetensors")))
    if not files:
        raise FileNotFoundError(f"No safetensors found in {model_path}")
    arch, _ = get_model_and_args(config)
    model_config = arch.ModelConfig.from_dict(config)
    model = arch.Model(model_config, device=device)
    weights: Dict[str, torch.Tensor] = {}
    for fpath in files:
        weights.update(_read_safetensors(fpath))
    weights = model.sanitize(weights)
    model.load_weights(weights, strict=strict)
    return model


def load_processor(model_path: str, **kwargs):
    from transformers import AutoProcessor
    processor = AutoProcessor.from_pretrained(model_path, **kwargs)
    tok = processor.tokenizer if hasattr(processor, "tokenizer") else processor
    eos = getattr(tok, "eos_token_id", None)
    tok.stopping_criteria = StoppingCriteria([] if eos is None else eos, tok)
    return processor


def load(path_or_hf_repo: str, adapter_path: Optional[str] = None, lazy: bool = False,
         revision: Optional[str] = None, strict: bool = True, **kwargs):
    """utils.py:1065-1072 signature.  Local directories only (no network); the
    pseudo-path `synthetic:qwen2-vl-2b` / `synthetic:qwen2-vl-7b` builds a seeded
    random-init model with a SyntheticProcessor (benchmarks, no checkpoint)."""
    if adapter_path is not None:
        raise NotImplementedError("adapters (LoRA) are outside this engine's hot-path scope")
    if revision is not None:
        raise NotImplementedError("`revision` needs the hub; only local model directories are supported")
    if path_or_hf_repo.startswith("synthetic:"):
        return load_synthetic(path_or_hf_repo.split(":", 1)[1], **kwargs)
    if not os.path.isdir(path_or_hf_repo):
        raise FileNotFoundError(
            f"{path_or_hf_repo}: only local model directories are supported (no hub download)")
    processor = kwargs.pop("processor", None)   # a ready ProcessorLike (tests / custom pipelines)
    model = load_model(path_or_hf_repo, lazy=lazy, strict=strict, device=kwargs.pop("device", None))
    if processor is None:
        processor = load_processor(path_or_hf_repo)
    return model, processor


def load_synthetic(name: str, seed: int = 0, device=None, n_text_tokens: int = 128, config=None):
    from .models.qwen2_vl import Model
    from .models.qwen2_vl.config import qwen2_vl_2b_config, qwen2_vl_7b_config
    from .models.qwen2_vl.processing_qwen2_vl import SyntheticProcessor
    if config is None:
        table = {"qwen2-vl-2b": qwen2_vl_2b_config, "qwen2-vl-7b": qwen2_vl_7b_config}
        if name.lower() not in table:
            raise ValueError(f"unknown synthetic model {name}; have {sorted(table)}")
        config = table[name.lower()]()
    model = Model(config, device=device).init_random(seed)
    processor = SyntheticProcessor(config, n_text_tokens=n_text_tokens, seed=seed)
    processor.tokenizer.stopping_criteria = StoppingCriteria([], processor.tokenizer)
    return model, processor


# --------------------------------------------------------------------------
def load_image(image_source, timeout: int = 10):
    from PIL import Image
    if isinstance(image_source, Image.Image):
        return image_source
    if isinstance(image_source, np.ndarray):
        return image_source
    if isinstance(image_source, str) and os.path.exists(image_source):
        return Image.open(image_source).convert("RGB")
    raise ValueError(f"cannot load image {image_source!r} (URLs need network access)")


def process_image(img, resize_shape, image_processor=None):
    img = load_image(img)
    if resize_shape is not None and hasattr(img, "resize"):
        img = img.resize(resize_shape)
    return img


def _to_device(arr, device, stream, dtype):
    t = torch.from_numpy(np.ascontiguousarray(arr)).to(dtype)
    t = t.pin_memory() if device.type == "cuda" else t
    if stream is not None:
        with torch.cuda.stream(stream):
            return t.to(device, non_blocking=True)
    return t.to(device)


def prepare_inputs(processor, images=None, audio=None, prompts=None, image_token_index=None,
                   resize_shape=None, add_special_tokens=False, padding=True,
                   padding_side="left", pad_to_uniform_size=False, device=None, stream=None,
                   **kwargs) -> Dict[str, Any]:
    """utils.py:1918-2136 for text / image requests.  Returns input_ids and
    attention_mask as host numpy (the rope-index / merge bookkeeping is host logic,
    like the reference's `.tolist()`), pixel_values as a device fp32 tensor."""
    if audio is not None:
        raise NotImplementedError("audio inputs are outside this engine's hot-path scope")
    if images is not None and not isinstance(images, (list, tuple)):
        images = [images]
    if images is not None:
        images = [process_image(im, resize_shape) for im in images]
        if len(images) == 0:
            images = None
    if isinstance(prompts, str):
        prompts = [prompts]
    try:
        inputs = processor(text=prompts, images=images, padding=padding, return_tensors="np")
    except TypeError:
        inputs = processor(text=prompts, images=images)
    out: Dict[str, Any] = {}
    out["input_ids"] = np.asarray(inputs["input_ids"], dtype=np.int64)
    if "attention_mask" in inputs:
        out["attention_mask"] = np.asarray(inputs["attention_mask"], dtype=np.int64)
    dev = torch.device(device) if device is not None else torch.device("cuda", 0)
    if inputs.get("pixel_values", None) is not None:
        out["pixel_values"] = _to_device(np.asarray(inputs["pixel_values"], dtype=np.float32), dev,
                                         stream, torch.float32)
    if "pixel_values" not in inputs and inputs.get("images", None) is not None:   # utils.py:2113-2115
        out["pixel_values"] = _to_device(np.asarray(inputs["images"], dtype=np.float32), dev, stream, torch.float32)
    for k in ("image_grid_thw", "video_grid_thw"):
        if inputs.get(k, None) is not None:
            out[k] = np.asarray(inputs[k], dtype=np.int64)
    # every other key the processor produced travels on to the model as a kwarg (utils.py:2124-2134), as host
    # arrays: Idefics2's `pixel_attention_mask`, LLaVA-Next's `image_sizes`, ...
    for k in inputs.keys():
        if k in out or k in ("input_ids", "attention_mask", "pixel_values", "images"):
            continue
        v = inputs[k]
        out[k] = v if v is None or isinstance(v, (str, list)) else np.asarray(v)
    return out


class StoppingCriteria:
    """utils.py:2191-2249."""

    def __init__(self, eos_token_ids: Union[int, List[int]], tokenizer=None,
                 additional_eos_token_ids: Optional[List[int]] = None):
        self.tokenizer = tokenizer
        self.additional_eos_token_ids = list(dict.fromkeys(additional_eos_token_ids or ()))
        self.reset(eos_token_ids)

    def add_eos_token_ids(self, new_eos_token_ids=None):
        if new_eos_token_ids is None:
            return
        if self.tokenizer is None:
            raise ValueError("Processor is not provided")
        if isinstance(new_eos_token_ids, (str, int)):
            new_eos_token_ids = [new_eos_token_ids]
        for token in new_eos_token_ids:
            if isinstance(token, int):
                self.eos_token_ids.append(token)
            elif isinstance(token, str):
                self.eos_token_ids.append(
                    self.tokenizer.encode(" " + token, add_special_tokens=False)[-1])

    def reset(self, eos_token_ids=None):
        eos_token_ids = eos_token_ids if eos_token_ids is not None else self.tokenizer.eos_token_ids
        if isinstance(eos_token_ids, int):
            eos_token_ids = [eos_token_ids]
        resolved = list(eos_token_ids)
        resolved.extend(t for t in self.additional_eos_token_ids if t not in resolved)
        if getattr(self, "eos_token_ids", None) != resolved:
            self.eos_token_ids = resolved

    def __call__(self, input_ids) -> bool:
        return input_ids in self.eos_token_ids
