"""Decode step time of Qwen2-VL-2B (synthetic weights) with a bf16 KV cache (k_mega, and the per-phase kernels)
and with the 8-bit cache (per-phase kernels + k_attn_q8), alternating the arms at the same context.  Prints one
JSON line.

    python tools/kvq_decode_probe.py [ctx ...]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mlx_vlm_b200.generate import maybe_quantize_kv_cache  # noqa: E402
from mlx_vlm_b200.models.cache import make_prompt_cache  # noqa: E402
from mlx_vlm_b200.utils import load_synthetic  # noqa: E402

STEPS, WINDOWS = 64, 5


def main():
    ctxs = [int(a) for a in sys.argv[1:]] or [4096, 16384]
    dev = torch.device("cuda", 0)
    model, _ = load_synthetic("qwen2-vl-2b", seed=0, device=dev, n_text_tokens=16)
    lm, eng = model.language_model, model.engine
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "model": "Qwen2-VL-2B (synthetic weights), batch 1", "steps_per_window": STEPS,
           "windows": WINDOWS, "ctx": {}}
    for ctx in ctxs:
        ids = np.random.default_rng(ctx).integers(0, 1000, size=(1, ctx))
        caches = {}
        for arm in ("bf16", "q8"):
            c = make_prompt_cache(lm)
            lm(ids, cache=c, reserve_tokens=ctx + STEPS + 1, logits_to_keep=1)
            if arm == "q8":
                maybe_quantize_kv_cache(c, 0, 64, 8)
            caches[arm] = c
        times = {"bf16": [], "bf16_per_phase": [], "q8": []}
        for w in range(WINDOWS + 1):
            for arm in times:
                eng.set_mega(arm != "bf16_per_phase")
                lm._bind(caches["q8" if arm == "q8" else "bf16"], ctx + STEPS, decode=True)
                eng.set_next(1, ctx, ctx)
                eng.decode(STEPS)
                ms = eng.last_decode_ms()
                if w > 0:   # window 0 warms up (graph capture, first launches)
                    times[arm].append(ms)
        eng.set_mega(True)
        assert eng.device_error() == 0
        q = caches["q8"][0]._pool
        out["ctx"][ctx] = {
            **{f"{a}_ms_per_step": float(np.median(t)) for a, t in times.items()},
            "bf16_kv_bytes_per_pos": 28 * 2 * 2 * 128 * 2, "q8_kv_bytes_per_pos": q.bytes_per_position(),
            "spread_ms": {a: [min(t), max(t)] for a, t in times.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
