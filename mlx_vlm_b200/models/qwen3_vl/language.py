"""Qwen3-VL language model on the shared decoder engine.  Host bookkeeping (position ids, KV pool, prefill / decode
calls) is Qwen2-VL's: for text prompts the reference's `get_rope_index` (qwen3_vl/language.py:299-485) takes the same
text branch.  What differs is `head_dim`, which Qwen3-VL configs give explicitly (Qwen3-VL-4B: hidden 2560, 32 heads of
128), and, inside the engine, the q/k RMSNorm per head (lm.<i>.qn / lm.<i>.kn) and the interleaved M-RoPE axis table
(b200_engine_set_axis_sel), both set up by models/qwen3_vl/qwen3_vl.py."""
from ..qwen2_vl.language import LanguageModel as _Qwen2VLLanguageModel


class LanguageModel(_Qwen2VLLanguageModel):
    @property
    def head_dim(self):
        """the configured head width (Attention.head_dim, language.py:49-51), which sizes the KV pools"""
        return self.args.head_dim

    @property
    def lockstep_supported(self):
        """The lock-step batch (batched prefill + decode_batch.cu) is verified only for head_dim == hidden / heads;
        at other widths it produced wrong first tokens, so BatchGenerator runs such models time-multiplexed."""
        return self.args.head_dim * self.args.num_attention_heads == self.args.hidden_size
