"""Decode-step and prefill time of the Qwen3-VL decoder at the Qwen3-VL-2B shapes (random weights), with the device
name and power limit read in the same run.  Qwen3-VL's step runs on k_mega (q/k norm in its own phase) and on the
per-phase kernels; the Qwen2-VL-2B step on both is timed alongside for comparison.
Text prompt of 128 tokens (the vision tower is not built), greedy, 1 + 256 generated tokens.

usage: python tools/qwen3_vl_probe.py [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(model, ids, n):
    from mlx_vlm_b200.generate import generate_step
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in generate_step(ids, model, None, None, max_tokens=n):
        pass
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _measure(model, ids, n_dec=256, reps=5):
    _time(model, ids, 8)                      # warm-up: GEMM configurations measured, graphs captured
    _time(model, ids, n_dec + 1)
    pre, full = [], []
    for _ in range(reps):                     # alternate the two lengths; medians
        pre.append(_time(model, ids, 1))
        full.append(_time(model, ids, n_dec + 1))
    pre_ms, full_ms = 1e3 * float(np.median(pre)), 1e3 * float(np.median(full))
    return {"prefill_plus_first_token_ms": round(pre_ms, 3), "decode_ms_per_token": round((full_ms - pre_ms) / n_dec, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    ids = np.random.default_rng(0).integers(0, 150000, size=(1, 128))
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}
    from mlx_vlm_b200.models.qwen3_vl import Model
    from mlx_vlm_b200.models.qwen3_vl.config import qwen3_vl_2b_config
    m3 = Model(qwen3_vl_2b_config(), device="cuda:0").init_random(0)
    res["qwen3_vl_2b_k_mega"] = _measure(m3, ids)
    m3.engine.set_mega(0)
    res["qwen3_vl_2b_per_phase"] = _measure(m3, ids)
    del m3
    torch.cuda.empty_cache()
    from mlx_vlm_b200.models.qwen2_vl import Model as Q2
    from mlx_vlm_b200.models.qwen2_vl.config import qwen2_vl_2b_config
    m2 = Q2(qwen2_vl_2b_config(), device="cuda:0").init_random(0)
    res["qwen2_vl_2b_k_mega"] = _measure(m2, ids)
    m2.engine.set_mega(0)
    res["qwen2_vl_2b_per_phase"] = _measure(m2, ids)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "qwen3_vl_probe.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
