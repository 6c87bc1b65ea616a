#!/usr/bin/env python
"""Golden vectors for the 8-bit lock-step batch cache: the reference's own `should_quantize_kv_layer` and
`BatchQuantizedKVCache` / `QuantizedKVCache` (mlx_vlm/models/cache.py) are extracted with `ast` and EXECUTED over the
numpy stand-in for mlx.core of make_golden.py, with `mx.quantize` bound to tests/kvq_ref.py's restatement (codes
packed into uint32 words the way mx.quantize packs bits=8: element 4i+j in bits 8j of word i).
The trace: rows of equal length (the product keeps no left padding) through update (prefill of 5 positions, then one
decode position), extract, filter and extend.
Writes tests/golden/kvq_batch_golden.json.   usage: python tests/golden/make_kvq_batch_golden.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import extract, make_mx, tolist  # noqa: E402

OUT = os.path.join(HERE, "kvq_batch_golden.json")
GS, HD, NKV = 32, 64, 2


class _U32:
    """mx.uint32 of the stand-in: `.size` (bytes) as mlx's dtype has it; arrays are numpy uint32"""
    size = 4


def main():
    from typing import List
    import kvq_ref
    mx = make_mx()
    mx.uint32 = _U32
    mx.zeros = lambda shape, dtype=None: np.zeros(shape, dtype=np.uint32 if dtype is _U32 else dtype)

    def quantize(w, group_size=64, bits=8):
        assert bits == 8
        codes, scales, biases = kvq_ref.quantize(np.asarray(w, dtype=np.float32), group_size)
        return np.ascontiguousarray(codes).view(np.uint32), scales, biases
    mx.quantize = quantize
    ns = {"mx": mx, "np": np, "List": List, "Optional": None, "_BaseCache": object,
          "tree_map": lambda f, t: tuple(tuple(f(x) for x in p) for p in t)}
    prov = {}
    for name in ("should_quantize_kv_layer", "QuantizedKVCache", "BatchQuantizedKVCache"):
        code, where = extract("models/cache.py", name)
        exec(compile(code, f"<reference {where}>", "exec"), ns)
        prov[name] = where
    rule, BQ = ns["should_quantize_kv_layer"], ns["BatchQuantizedKVCache"]
    golden = {"_about": "reference 8-bit batch cache executed over a numpy stand-in, mx.quantize = tests/kvq_ref.py",
              "provenance": prov, "group_size": GS, "head_dim": HD, "n_kv": NKV,
              "layer_rule": {str(n): [bool(rule(i, n)) for i in range(n)] for n in (1, 2, 3, 28)}}
    rng = np.random.default_rng(0)

    def rows(B, n):
        # bf16-representable values, so the product's bf16 pool holds exactly what was quantized
        k = kvq_ref._bf16(rng.standard_normal((B, NKV, n, HD)) * 0.7)
        v = kvq_ref._bf16(rng.standard_normal((B, NKV, n, HD)) * 0.7)
        return k, v

    def snap(c, tag):
        n = int(c._idx)
        return {"op": tag, "idx": n, "offset": tolist(c.offset), "left_padding": tolist(c.left_padding),
                "keys": [tolist(x[..., :n, :]) for x in c.keys], "values": [tolist(x[..., :n, :]) for x in c.values],
                "shapes": [list(x.shape) for x in c.keys]}

    trace, inputs = [], {}
    c = BQ([0, 0, 0], group_size=GS, bits=8)
    k, v = rows(3, 5)
    inputs["prefill"] = {"keys": tolist(k), "values": tolist(v)}
    c.update_and_fetch(k, v)
    trace.append(snap(c, "update: prefill 5 positions of 3 rows"))
    k, v = rows(3, 1)
    inputs["decode"] = {"keys": tolist(k), "values": tolist(v)}
    c.update_and_fetch(k, v)
    trace.append(snap(c, "update: one decode position"))
    ex = c.extract(1)
    trace.append({"op": "extract row 1", "offset": int(ex.offset), "group_size": ex.group_size, "bits": ex.bits,
                  "keys": [tolist(x) for x in ex.keys], "values": [tolist(x) for x in ex.values]})
    c.filter(np.array([0, 2]))
    trace.append(snap(c, "filter keep rows 0, 2"))
    o = BQ([0], group_size=GS, bits=8)
    k, v = rows(1, 6)
    inputs["other"] = {"keys": tolist(k), "values": tolist(v)}
    o.update_and_fetch(k, v)
    c.extend(o)
    trace.append(snap(c, "extend with a 1-row cache of 6 positions"))
    golden["inputs"], golden["trace"] = inputs, trace
    with open(OUT, "w") as f:
        json.dump(golden, f)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
