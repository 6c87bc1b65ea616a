"""Idefics3 (and, through models/smolvlm, SmolVLM) on the CUDA engine: tower + pixel-shuffle connector + Llama LM."""
from .idefics3 import Connector, Model
from .vision import VisionModel, position_ids
from .language import LanguageModel
from .config import ModelConfig, TextConfig, VisionConfig, idefics3_8b_config

__all__ = ["Model", "Connector", "VisionModel", "LanguageModel", "ModelConfig", "TextConfig", "VisionConfig",
           "idefics3_8b_config", "position_ids"]
