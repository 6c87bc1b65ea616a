"""GPU time of the C2 vision tower and LM prefill in isolation (CUDA events around N back-to-back
calls with no Python work in between; the sequences replay as captured graphs from their second call).
usage: python tools/prefill_breakdown.py"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mlx_vlm_b200.models.cache import make_prompt_cache
from mlx_vlm_b200.utils import load_synthetic, prepare_inputs

model, proc = load_synthetic("qwen2-vl-2b", seed=0, device="cuda:0", n_text_tokens=128)
eng = model.engine
img = np.random.default_rng(0).integers(0, 256, size=(336, 336, 3), dtype=np.uint8)
inp = prepare_inputs(proc, images=[img], prompts="x", device=eng.device, stream=eng.stream)
ids, pvd, grid = inp["input_ids"], inp["pixel_values"], inp["image_grid_thw"]
T = ids.shape[1]
emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
cache = make_prompt_cache(model.language_model)
lm = model.language_model


def vis():
    return model.vision_tower(pvd, grid)


def pre():
    for c in cache:
        c.offset = 0
    lm._rope_deltas, lm._position_ids = None, None
    lm(ids, inputs_embeds=emb.inputs_embeds, cache=cache, position_ids=emb.position_ids, rope_deltas=emb.rope_deltas,
       logits_to_keep=1, reserve_tokens=T + 600)


for name, fn in (("vision tower (32 blocks + merger)", vis), ("LM prefill T=272 (28 layers + head)", pre)):
    for _ in range(4):
        fn()
    eng.stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    t0 = time.perf_counter()
    e0.record(eng.stream)
    for _ in range(n):
        fn()
    e1.record(eng.stream)
    t1 = time.perf_counter()
    eng.stream.synchronize()
    print(f"{name}: {e0.elapsed_time(e1) / n:.3f} ms GPU per call, host enqueue {1e3 * (t1 - t0) / n:.3f} ms per call",
          flush=True)
