"""mlx_vlm_b200 — H100-native drop-in for the generate path of Blaizzy/mlx-vlm.

`import mlx_vlm_b200 as mlx_vlm` gives the reference's generate-path surface
(reference mlx_vlm/__init__.py:7-20): load, generate, stream_generate,
generate_step, batch_generate / BatchGenerator, prepare_inputs, GenerationResult,
PromptCacheState.  The
arithmetic lives in libb200vlm.so (hand-written sm_90a CUDA behind the C ABI of
include/b200vlm.h); importing the package does not need a GPU, calling a model
does (there is no CPU fallback).
"""
from .generate import (GenerationResult, PromptCacheState, generate, generate_step,
                       stream_generate)
from .generate_batch import (BatchGenerator, BatchResponse, BatchStats, GenerationBatch,
                             PromptProgress, batch_generate)
from .prompt_utils import apply_chat_template, get_message_json
from .utils import load, load_synthetic, prepare_inputs, process_image
from .version import __version__
from .vision_cache import VisionFeatureCache

__all__ = ["BatchGenerator", "BatchResponse", "BatchStats", "GenerationBatch", "PromptProgress",
           "batch_generate", "GenerationResult", "PromptCacheState", "generate", "generate_step",
           "stream_generate", "VisionFeatureCache", "apply_chat_template", "get_message_json", "load", "load_synthetic", "prepare_inputs", "process_image",
           "__version__"]
