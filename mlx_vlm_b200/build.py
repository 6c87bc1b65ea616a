"""Build libb200vlm.so (sm_90a only) in-tree with nvcc.

`python -m mlx_vlm_b200.build` or `build()`; the .so lands next to this file so
it travels with the repo snapshot to the GPU box (it is git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200vlm.so")
SOURCES = ["engine.cu", "rowops.cu", "attention.cu", "decode.cu", "decode_mega.cu",
           "attention_tc.cu", "gemm_wt.cu", "attention_fa.cu", "decode_batch.cu", "tower_f32.cu", "kvq.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _fingerprint() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp = LIB + ".stamp"
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as f:
            if f.read().strip() == fp:
                return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src} ---\n{out.decode()}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libb200vlm.so")
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
           "-Xcompiler", "-fPIC"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(fp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
