"""Per-phase timeline of one decode step of the persistent megakernel (globaltimer
stamps at every grid barrier).  Prints mean compute / barrier-wait per phase kind."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mlx_vlm_b200 import _native as N
from mlx_vlm_b200.models.cache import make_prompt_cache
from mlx_vlm_b200.utils import load_synthetic, prepare_inputs
model, proc = load_synthetic("qwen2-vl-2b", seed=0, device="cuda:0", n_text_tokens=128)
eng = model.engine
eng.set_graph(False)
N.check(eng.lib.b200_engine_mega_timeline(eng.h, 0))
img = np.random.default_rng(0).integers(0, 256, size=(336, 336, 3), dtype=np.uint8)
inp = prepare_inputs(proc, images=[img], prompts="x", device=eng.device, stream=eng.stream)
ids, pvd, grid = inp["input_ids"], inp["pixel_values"], inp["image_grid_thw"]
T = ids.shape[1]
cache = make_prompt_cache(model.language_model)
emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=cache, position_ids=emb.position_ids,
                     rope_deltas=emb.rope_deltas, logits_to_keep=1, reserve_tokens=T + 600)
model.language_model.fused_greedy_decode_n(200, cache, reserve_tokens=T + 600)
eng.stream.synchronize()
raw = np.zeros(2 * 1024 * 2 + 256, dtype=np.int64)
buf = raw[:4096].reshape(2, 1024, 2)
N.check(eng.lib.b200_engine_mega_timeline(eng.h, raw.ctypes.data))
L = 28
names, per = ["qkv", "attn", "ores", "gateup", "dres"], 5
for cta in (0, 1):
    a = buf[cta]
    nb = per * L + 2
    arrive, release = a[:nb, 0], a[:nb, 1]
    comp = np.empty(nb); comp[0] = np.nan
    comp[1:] = arrive[1:] - release[:-1]
    wait = release - arrive
    print(f"--- CTA {'0' if cta == 0 else 'last'}: step span {(release[nb-1]-arrive[0])/1e3:.1f} us (first arrive -> last release)")
    for k, nm in enumerate(names):
        idx = np.arange(L) * per + k
        c = comp[idx[1:] if k == 0 else idx]
        print(f"  {nm:28s} compute {np.nanmean(c)/1e3:7.2f} us  barrier wait {wait[idx].mean()/1e3:7.2f} us")
    print(f"  head (+ last down)           compute {comp[per*L]/1e3:7.2f} us  wait {wait[per*L]/1e3:7.2f} us; sample compute {comp[per*L+1]/1e3:7.2f} wait {wait[per*L+1]/1e3:7.2f}")
    print("  layer 5 raw (compute, wait) us:", [(round(float(comp[per*5+k])/1e3,2), round(float(wait[per*5+k])/1e3,2)) for k in range(per)])

for name, off in (("gateup CTA0", 4096), ("gateup CTA77", 4096 + 32), ("dres CTA0", 4096 + 64)):
    t = raw[off:off + 28]
    t = t[t > 0]
    if len(t) > 2:
        d = np.diff(t) / 1e3
        print(f"{name}: prologue {d[0]:.2f} us; then (wait, compute) per tile:", [(round(d[i],2), round(d[i+1],2)) for i in range(1, len(d)-1, 2)])

t = raw[4096 + 96:4096 + 126]; t = t[t > 0]
c = raw[4096:4096 + 30]; c = c[c > 0]
b = buf[0]
print("layer-5 CTA0 absolute us (relative to the first barrier release of layer 5):")
t0 = b[per * 5, 1]
print("  barrier releases:", [round(float(b[per * 5 + k, 1] - t0) / 1e3, 2) for k in range(per)])
print("  producer issue times of gate/up tiles:", [round((x - t0) / 1e3, 2) for x in t])
print("  consumer gate/up stamps (start, prologue end, then wait-done/compute-done):", [round((x - t0) / 1e3, 2) for x in c])

names = ["start", "q loaded", "scores", "local stats", "group barrier", "stats read", "PV", "partial written", "counter", "end"]
for cta in (0, 1):
    t = raw[4096 + 128 + 32 * cta:4096 + 128 + 32 * cta + 12]; t = t[t > 0]
    if len(t) > 2:
        print(f"attention CTA{cta} (layer 5) step durations us:", list(zip(names[1:], [round(x / 1e3, 2) for x in np.diff(t)])))
