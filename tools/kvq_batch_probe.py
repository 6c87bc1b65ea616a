#!/usr/bin/env python
"""Lock-step decode step time with a bf16 batch pool vs a kv_bits=8 batch pool (Qwen2-VL-7B geometry, synthetic
weights): `rows` rows at `ctx` cached positions each, one greedy lock-step step timed with CUDA events over windows
of `steps` steps (each after an untimed window that captures the step graph).  The two arms alternate window by window in one process; the medians are reported, with the KV
bytes per row-position of each pool and the GPU name and power limit read in the same run.  The pool contents are
zeros: the step's work does not depend on the values.
usage: python tools/kvq_batch_probe.py [--rows 8 16] [--ctx 1024 4096] [--windows 5] [--steps 32]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def _gpu():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as exc:   # the numbers are still device-timed; say what could not be read
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({exc})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--ctx", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--group-size", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kvq_batch_probe: needs a CUDA device")
    from mlx_vlm_b200.models.cache import BatchKVQPool, KVPool
    from mlx_vlm_b200.utils import load_synthetic
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model, _ = load_synthetic("qwen2-vl-7b", seed=1, device=dev, n_text_tokens=16)
    lm, eng = model.language_model, model.engine
    L, nkv, hd = lm.args.num_hidden_layers, lm.n_kv_heads, lm.head_dim
    results = []
    for rows in args.rows:
        for ctx in args.ctx:
            cap = ((ctx + (args.windows + 1) * args.steps * 2 + 8 + 255) // 256) * 256
            pools = {}
            with torch.cuda.stream(eng.stream):
                pools["bf16"] = KVPool(L, nkv, hd, dev, batch=rows, capacity=cap)
                pools["kv8"] = BatchKVQPool(L, nkv, hd, dev, group_size=args.group_size, batch=rows, capacity=cap,
                                            stream=eng.stream)
            bpp = {"bf16": L * 2 * nkv * hd * 2, "kv8": pools["kv8"].bytes_per_position()}
            times = {k: [] for k in pools}
            n_ctx = {k: ctx for k in pools}
            tok = np.ones(rows, dtype=np.int32)
            for w in range(args.windows + 1):     # window 0 warms up (graph capture, GEMM configurations)
                for arm in ("bf16", "kv8"):
                    eng.bind_pool(pools[arm])
                    c = np.full(rows, n_ctx[arm], dtype=np.int32)
                    eng.batch_begin(tok, c, c, np.ones(rows, dtype=np.int32))
                    eng.batch_decode(args.steps)   # untimed: the bind re-captures the step graph
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(eng.stream)
                    eng.batch_decode(args.steps)
                    e1.record(eng.stream)
                    e1.synchronize()
                    n_ctx[arm] += 2 * args.steps
                    if w:
                        times[arm].append(e0.elapsed_time(e1) / args.steps)
            assert eng.device_error() == 0
            r = {"rows": rows, "ctx": ctx, "ms_per_step": {k: float(np.median(v)) for k, v in times.items()},
                 "spread_ms": {k: [float(min(v)), float(max(v))] for k, v in times.items()},
                 "kv_bytes_per_row_position": bpp}
            results.append(r)
            print(json.dumps(r), flush=True)
            del pools
            torch.cuda.empty_cache()
    out = {"gpu": _gpu(), "model": "Qwen2-VL-7B geometry, synthetic weights", "group_size": args.group_size,
           "windows": args.windows, "steps_per_window": args.steps, "results": results}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
