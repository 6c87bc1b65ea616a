"""Back-to-back timing (CUDA events, warm) of the prefill-side attention and row ops at the C2 shapes, through
the C ABI.  The GEMMs (gemm_wt) have their own sweep, tools/wt_sweep.py.
usage: python tools/op_sweep.py [iters]   -> one line per op: us per call, TFLOP/s"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from mlx_vlm_b200 import _native as N

lib = N.lib()
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 40
dev = "cuda:0"


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev, dtype=torch.float32) * scale).to(torch.bfloat16)


def timeit(fn, n=iters):
    for i in range(4):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def attn_case(name, heads, kv, hd, L, S, causal):
    q = bf(L, heads * hd)
    k = bf(kv, S, hd)
    v = bf(kv, S, hd)
    o = torch.empty(L, heads * hd, device=dev, dtype=torch.bfloat16)

    def fn(i):
        N.check(lib.b200_attention(q.data_ptr(), heads * hd, hd, k.data_ptr(), hd, S * hd, v.data_ptr(), hd,
                                   S * hd, o.data_ptr(), heads * hd, heads, kv, hd, L, S, causal,
                                   1.0 / hd ** 0.5, 0), "attn")
    us = timeit(fn)
    fl = 4.0 * L * S * hd * heads * (0.5 if causal else 1.0)
    print(f"attn {name:14s} h={heads} kv={kv} hd={hd} L={L} S={S}: {us:8.2f} us  {fl / us / 1e6:7.1f} TFLOP/s", flush=True)
    return us


def rowop_cases():
    x = bf(576, 1280)
    w, b = bf(1280), bf(1280)
    y = torch.empty_like(x)
    us = timeit(lambda i: N.check(lib.b200_layer_norm(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(),
                                                      576, 1280, 1e-6, 0), "ln"))
    print(f"layer_norm 576x1280: {us:.2f} us")
    x2 = bf(272, 1536)
    y2 = torch.empty_like(x2)
    w2 = bf(1536)
    us = timeit(lambda i: N.check(lib.b200_rms_norm(x2.data_ptr(), w2.data_ptr(), y2.data_ptr(), 272, 1536,
                                                    1e-6, 0), "rms"))
    print(f"rms_norm 272x1536: {us:.2f} us")
    gu = bf(272, 17920)
    act = torch.empty(272, 8960, device=dev, dtype=torch.bfloat16)
    us = timeit(lambda i: N.check(lib.b200_swiglu(gu.data_ptr(), act.data_ptr(), 272, 8960, 0), "swiglu"))
    print(f"swiglu 272x8960: {us:.2f} us")


if __name__ == "__main__":
    a_v = 32 * attn_case("vit", 16, 16, 80, 576, 576, 0)
    a_l = 28 * attn_case("lm", 12, 2, 128, 272, 272, 1)
    rowop_cases()
    print(f"sum: vit attn {a_v / 1e3:.2f} ms, lm attn {a_l / 1e3:.2f} ms")
