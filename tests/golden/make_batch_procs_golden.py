#!/usr/bin/env python
"""Golden vectors for the per-row logits processors of the batch: the reference's own `GenerationBatch`
(mlx_vlm/generate/ar.py) and `_sample_with_positions` are extracted with `ast` and EXECUTED over the numpy stand-in
for mlx.core of make_golden.py, with a stand-in language model (deterministic distinct logits per input token) and a
processor that records the token context it is given.
The trace: a batch of two rows (one with processors, its token context seeded with the prompts as
PromptProcessingBatch seeds it, ar.py:1663-1667) steps twice; a batch without processors steps once and joins it
(extend); the three rows step; filter keeps rows 2, 0, then row 0 only.  Recorded: every processor call's token
context, the batch's `logits_processors` alignment and `token_context` after each operation, and the top-k ids.
Writes tests/golden/batch_procs_golden.json.   usage: python tests/golden/make_batch_procs_golden.py"""
import json
import os
import sys
import types
from dataclasses import dataclass
from typing import Any, Callable, List, Optional, Tuple

import numpy as np
from scipy.special import logsumexp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import extract, make_mx  # noqa: E402

OUT = os.path.join(HERE, "batch_procs_golden.json")
V, K = 50, 3


def logits_of(tokens, step):
    """distinct logits per row, a function of the row's input token and the step"""
    out = np.zeros((len(tokens), V), np.float32)
    for b, t in enumerate(tokens):
        perm = np.random.default_rng(int(t) * 7 + step).permutation(V)
        out[b] = perm.astype(np.float32) * 0.25 - 6.0
    return out


def main():
    mx = make_mx()
    mx.logsumexp = lambda a, axis=None, keepdims=False: logsumexp(a, axis=axis, keepdims=keepdims).astype(a.dtype)
    mx.async_eval = lambda *a, **k: None
    array = type("array", (np.ndarray,), {})   # mx.array as a type (isinstance) and a constructor
    array.__new__ = lambda cls, x, dtype=None: np.asarray(np.array(x, dtype=dtype))
    mx.array = array
    ns = {"mx": mx, "np": np, "List": List, "Optional": Optional, "Callable": Callable, "Any": Any, "Tuple": Tuple,
          "dataclass": dataclass, "nn": types.SimpleNamespace(Module=object), "_extend_cache": lambda a, b: []}
    prov = {}
    for name in ("_sample_with_positions", "GenerationBatch"):
        code, where = extract("generate/ar.py", name)
        exec(compile(code, f"<reference {where}>", "exec"), ns)
        prov[name] = where
    GB = ns["GenerationBatch"]
    calls = []
    step = [0]

    class LM:
        def __call__(self, inputs, cache=None, **kw):
            step[0] += 1
            return types.SimpleNamespace(logits=logits_of(np.asarray(inputs).reshape(-1).tolist(), step[0])[:, None])

    def recorder(uid):
        def proc(tokens, logits):
            calls.append({"uid": uid, "tokens": np.asarray(tokens).tolist()})
            return logits
        return proc

    model = types.SimpleNamespace(language_model=LM())
    argmax = lambda lp: np.argmax(lp, axis=-1)   # noqa: E731
    trace = []
    prompts = {0: [5, 6, 7], 1: [8, 9], 2: [10, 11, 12, 13]}
    firsts = {0: 21, 1: 22, 2: 23}

    def snap(g, op, extra=None):
        d = {"op": op, "uids": list(g.uids),
             "has_processors": [p is not None for p in g.logits_processors],
             "token_context": [list(map(int, c)) for c in g.token_context]}
        d.update(extra or {})
        trace.append(d)

    def step_(g, op):
        toks, _, top_idx, _ = g._step()
        lg = logits_of(toks, step[0])
        snap(g, op, {"inputs": [int(t) for t in toks],
                     "logprobs": (lg - logsumexp(lg, axis=-1, keepdims=True)).astype(np.float32).tolist(),
                     "next_top_idx": np.asarray(g._next_top_idx).tolist()})

    a = GB(model, [0, 1], np.array([firsts[0], firsts[1]]), [], argmax, None, [8, 8], top_logprobs_k=K,
           token_context=[prompts[0], prompts[1]], logits_processors=[[recorder(0)], None])
    snap(a, "new batch: row 0 with processors, row 1 without")
    step_(a, "step")
    step_(a, "step")
    b = GB(model, [2], np.array([firsts[2]]), [], argmax, None, [8], top_logprobs_k=K, token_context=[],
           logits_processors=[])
    snap(b, "new batch without processors")
    step_(b, "step")
    a.extend(b)
    snap(a, "extend")
    step_(a, "step")
    a.filter([2, 0])
    snap(a, "filter [2, 0]")
    step_(a, "step")
    a.filter([0])
    snap(a, "filter [0]")
    golden = {"_about": "reference GenerationBatch executed over a numpy stand-in; logits: make_batch_procs_golden.py "
                        "logits_of(input token, step counter)",
              "provenance": prov, "vocab": V, "top_k": K, "prompts": {str(k): v for k, v in prompts.items()},
              "trace": trace, "processor_calls": calls}
    with open(OUT, "w") as f:
        json.dump(golden, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
