from .config import ModelConfig, TextConfig, VisionConfig
from .language import LanguageModel
from .qwen3_vl import Model
