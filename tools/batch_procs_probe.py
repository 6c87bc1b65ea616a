"""Cost of per-row logits processors and top-k logprobs in the lock-step batch (Qwen2-VL-7B shapes, synthetic
weights, 8 rows of ~1k context, greedy).  Arms, alternated over 5 windows (median reported):
  a  greedy, no processors
  b  repetition_penalty=1.1 on every row, lowered to the device kernel (k-step device loop kept)
  c  the same penalty as torch ops on each row's logits (the path of processors the batch cannot lower)
  d  greedy with top_logprobs_k=5
Per-step time = CUDA events around the decode loop of one window (every row admitted first) over its steps;
the loop ends in a device synchronise, so host work between steps is part of the number.
usage: python tools/batch_procs_probe.py [out.json]"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

ROWS, CTX, STEPS, WINDOWS = 8, 1000, 64, 5


def main():
    from mlx_vlm_b200.generate_batch import BatchGenerator
    from mlx_vlm_b200.sample_utils import make_logits_processors
    from mlx_vlm_b200.utils import load_synthetic
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    model, proc = load_synthetic("qwen2-vl-7b", seed=1, device="cuda:0")
    model.config.eos_token_id = []
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, 30000, size=CTX + 8 * i).tolist() for i in range(ROWS)]
    rep = make_logits_processors(repetition_penalty=1.1)
    wrapped = [lambda toks, lg, p=rep[0]: p(toks, lg)]
    arms = {"a_greedy": ({}, None), "b_rep_device": ({}, rep), "c_rep_torch": ({}, wrapped),
            "d_top5": ({"top_logprobs_k": 5}, None)}

    def window(kw, procs):
        g = BatchGenerator(model, proc, max_tokens=STEPS + 1, completion_batch_size=ROWS, prefill_batch_size=ROWS,
                           decode_slice=32, **kw)
        g.insert(prompts, logits_processors=[procs] * ROWS)
        g.next()   # admission: every row prefilled
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(model.engine.stream)
        n = 0
        while g.has_work:
            g.next()
            n += 1
        e1.record(model.engine.stream)
        torch.cuda.synchronize()
        assert model.engine.device_error() == 0
        return e0.elapsed_time(e1) / STEPS

    for kw, procs in arms.values():   # warm-up: GEMM configurations, graphs
        window(kw, procs)
    ms = {k: [] for k in arms}
    for _ in range(WINDOWS):
        for k, (kw, procs) in arms.items():
            ms[k].append(window(kw, procs))
    out = {"gpu": gpu, "rows": ROWS, "context": CTX, "steps": STEPS,
           "ms_per_step_median": {k: statistics.median(v) for k, v in ms.items()}, "ms_per_step": ms}
    print(json.dumps(out))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
