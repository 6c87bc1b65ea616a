"""GPU parity of the round-2 ops (weight-major GEMM, finish_rows, pipelined attention, qkv post
kernel) against the oracle's restatement, through the C ABI.  Same bar as test_kernels_gpu.py:
relative L2 <= 1e-3 with the oracle's rounding points mirrored."""
import ctypes as C

import numpy as np
import pytest
import torch

from _util import cmp_bf16, to_dev
from test_kernels_gpu import R, lib, rnd  # noqa: F401  (fixture + helpers)

pytestmark = pytest.mark.gpu
BF16, PARTIAL, SWIGLU = 0, 1, 2


def _cfg(c):
    return (C.c_int * 4)(*c) if c else None


@pytest.mark.parametrize("T,N,K,epi,bias,res,cfg", [
    (576, 3840, 1280, 0, True, False, None),            # ViT qkv, automatic configuration
    (576, 5120, 1280, 1, True, False, (192, 2, 2, 1)),  # fc1 + gelu_fast
    (576, 1280, 5120, 0, True, True, (144, 1, 3, 1)),   # fc2 + residual, direct epilogue
    (144, 5120, 5120, 2, True, False, None),            # merger fc1 + exact gelu
    (272, 2048, 1536, 0, True, False, (96, 2, 3, 1)),   # LM qkv
    (1, 256, 64, 0, True, False, (16, 1, 3, 1)),        # single row
    (130, 200, 72, 1, True, True, (144, 1, 2, 1)),      # ragged T / N / K
    (8, 1536, 1536, 0, True, False, (16, 2, 6, 1)),     # decode batch
    (576, 1280, 1176, 0, False, False, None),           # patch embed (K tail 1176 = 18*64+24)
    (700, 1000, 520, 1, True, True, (256, 1, 2, 1)),    # large token tile, ragged N, gelu + residual
    (272, 1536, 8960, 0, False, True, None),            # LM down + residual, no bias
    (3600, 3584, 1024, 0, False, "inplace", None),      # 7B o_proj / down of a long chunk: h = h + x.W^T in place
])
def test_gemm_wt_bf16(lib, T, N, K, epi, bias, res, cfg):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    X, W = rnd(T, K, seed=1), rnd(N, K, scale=0.05, seed=2)
    b = rnd(N, scale=0.5, seed=3) if bias else None
    resid = rnd(T, N, seed=4) if res else None
    want = S.linear(r, X, W, b)
    if epi == 1:
        want = S.gelu_fast(r, want)
    elif epi == 2:
        want = S.gelu_exact(r, want)
    if res:
        want = r.r(resid + want)
    dX, dW = to_dev(X), to_dev(W)
    db = to_dev(b) if bias else None
    ldn = ((N + 7) // 8) * 8
    Cc = torch.zeros(T, ldn, dtype=torch.bfloat16, device="cuda")
    dr = None
    if res:
        dr = torch.zeros(T, ldn, dtype=torch.bfloat16, device="cuda")
        dr[:, :N] = to_dev(resid)
        if res == "inplace":   # the output is its own residual, as in the engine's long-chunk residual add
            Cc = dr
    Nn.check(lib.b200_gemm_wt(dX.data_ptr(), K, dW.data_ptr(), Nn.ptr(db), Nn.ptr(dr), ldn, Cc.data_ptr(), ldn, 0,
                              T, N, K, epi, BF16, 0, _cfg(cfg), 0, 0), "gemm_wt")
    torch.cuda.synchronize()
    cmp_bf16(Cc[:, :N], want, f"gemm_wt {T}x{N}x{K} epi={epi} cfg={cfg}")


@pytest.mark.parametrize("T,N,K,cfg,kind", [
    (272, 1536, 8960, (144, 2, 3, 6), "rms"),    # LM down: split-K 6 + residual + RMSNorm of the next layer
    (576, 1280, 5120, (192, 2, 2, 4), "ln"),     # ViT fc2: split-K 4 + residual + LayerNorm
    (8, 1536, 8960, (16, 2, 6, 10), "rms"),      # decode batch
    (272, 1536, 1536, (96, 2, 3, 4), "none"),    # o_proj, no norm
    (272, 1536, 1536, (96, 2, 3, 4), "rms_inplace"),  # o_proj, residual added in place (h_out == resid), as in the engine
])
def test_gemm_wt_partial_and_finish_rows(lib, T, N, K, cfg, kind):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    X, W = rnd(T, K, seed=5), rnd(N, K, scale=0.05, seed=6)
    b, h = rnd(N, scale=0.5, seed=7), rnd(T, N, seed=8)
    nw = r.r(1.0 + 0.1 * torch.randn(N, generator=torch.Generator().manual_seed(9)))
    nb = rnd(N, scale=0.1, seed=10)
    hw = r.r(h + S.linear(r, X, W, b))
    dX, dW, db, dh, dnw, dnb = (to_dev(t) for t in (X, W, b, h, nw, nb))
    P = torch.full((cfg[3], T, N), 7.0, dtype=torch.float32, device="cuda")
    Nn.check(lib.b200_gemm_wt(dX.data_ptr(), K, dW.data_ptr(), 0, 0, 0, 0, 0, P.data_ptr(), T, N, K, 0, PARTIAL,
                              0, _cfg(cfg), 0, 0), "gemm_wt partial")
    norm, inplace = kind.removesuffix("_inplace"), kind.endswith("_inplace")
    hout, xn = dh if inplace else torch.zeros_like(dh), torch.zeros_like(dh)
    k = {"none": 0, "rms": 1, "ln": 2}[norm]
    Nn.check(lib.b200_finish_rows(P.data_ptr(), cfg[3], db.data_ptr(), dh.data_ptr(), N, hout.data_ptr(), N, k,
                                  dnw.data_ptr(), dnb.data_ptr() if norm == "ln" else 0, 1e-6, xn.data_ptr(),
                                  N, T, N, 0), "finish_rows")
    torch.cuda.synchronize()
    cmp_bf16(hout, hw, f"finish_rows h {T}x{N} split={cfg[3]} {kind}")
    got_h = hout.float().cpu()
    if norm == "rms":    # the norm is checked on the kernel's own h (identical inputs)
        cmp_bf16(xn, S.rms_norm(r, got_h, nw, 1e-6), "finish_rows rms_norm")
    elif norm == "ln":
        cmp_bf16(xn, S.layer_norm(r, got_h, nw, nb, 1e-6), "finish_rows layer_norm")


@pytest.mark.parametrize("T,I,K,cfg", [(272, 8960, 1536, None), (8, 8960, 1536, (16, 2, 6, 1)),
                                       (100, 200, 64, (112, 1, 2, 1))])
def test_gemm_wt_swiglu(lib, T, I, K, cfg):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    X, W = rnd(T, K, seed=11), rnd(2 * I, K, scale=0.05, seed=12)
    want = S.swiglu(r, S.linear(r, X, W[:I]), S.linear(r, X, W[I:]))
    dX, dW = to_dev(X), to_dev(W)
    act = torch.zeros(T, I, dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_gemm_wt(dX.data_ptr(), K, dW.data_ptr(), 0, 0, 0, act.data_ptr(), I, 0, T, 2 * I, K, 0,
                              SWIGLU, I, _cfg(cfg), 0, 0), "gemm_wt swiglu")
    torch.cuda.synchronize()
    cmp_bf16(act, want, f"gemm_wt swiglu {T}x{I}x{K}")


@pytest.mark.parametrize("Lq,S_,nh,nkv,hd,causal", [
    (576, 576, 16, 16, 80, 0),   # ViT block
    (272, 272, 12, 2, 128, 1),   # LM prefill
    (17, 17, 4, 2, 64, 1),       # ragged tile
    (300, 300, 28, 4, 128, 1),   # Qwen2-VL-7B head geometry
    (33, 33, 4, 4, 72, 0),       # head dim 72 (SigLIP-SO400M): padded to 80 for the P.V MMA
    (577, 577, 16, 16, 64, 0),   # CLIP-L/14-336: 577 tokens
])
def test_attention_fa(lib, Lq, S_, nh, nkv, hd, causal):
    """pipelined attention: q pre-scaled (qs = bf16(q * bf16(scale))), V passed transposed"""
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    q = rnd(1, nh, Lq, hd, seed=12)
    k = rnd(1, nkv, S_, hd, seed=13)
    v = rnd(1, nkv, S_, hd, seed=14)
    scale = hd ** -0.5
    want = S.sdpa(r, q, k, v, scale, bool(causal))  # (1,nh,Lq,hd)
    qs = r.r(q * r.scalar(scale))
    dq = to_dev(qs[0].transpose(0, 1))      # (Lq, nh, hd)
    dk = to_dev(k[0].transpose(0, 1))       # (S, nkv, hd)  token-major, like a packed qkv buffer
    s_ld = (S_ + 7) // 8 * 8
    vt = torch.zeros(nkv, hd, s_ld, dtype=torch.bfloat16, device="cuda")
    vt[:, :, :S_] = to_dev(v[0].transpose(1, 2))
    out = torch.zeros(Lq, nh * hd, dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_attention_fa(dq.data_ptr(), nh * hd, hd, dk.data_ptr(), nkv * hd, hd, vt.data_ptr(),
                                   hd * s_ld, s_ld, out.data_ptr(), nh * hd, nh, nkv, hd, Lq, S_, causal, 0),
             "attention_fa")
    torch.cuda.synchronize()
    cmp_bf16(out.view(Lq, nh, hd), want[0].transpose(0, 1), f"attention_fa Lq={Lq} S={S_} hd={hd}")


def test_vision_qkv_post(lib):
    """rotary (vision.py:35-50) on q,k in place, q pre-scaled, V^T emitted"""
    from mlx_vlm_b200 import _native as Nn
    from oracle import qwen2vl as O
    cfg = O.qwen2_vl_2b()
    v = cfg.vision
    grid = [[1, 24, 22]]
    N, nh, hd = 24 * 22, v.num_heads, v.embed_dim // v.num_heads
    r = R()
    qkv = rnd(N, 3, nh, hd, seed=15)
    freqs = O.vision_rotary_freqs(grid, v)
    cos = torch.cos(freqs).repeat(1, 2)[:, None, :]
    sin = torch.sin(freqs).repeat(1, 2)[:, None, :]
    want = qkv.clone()
    for w in (0, 1):
        x = qkv[:, w]
        want[:, w] = r.r(x * cos + O._rotate_half(x) * sin)
    scale = hd ** -0.5
    want[:, 0] = r.r(want[:, 0] * r.scalar(scale))
    d = to_dev(qkv)
    pos = torch.from_numpy(O.rot_pos_ids(grid, v.spatial_merge_size).astype(np.int32)).cuda()
    dim = hd // 2
    inv = (1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))).cuda()
    t_ld = (N + 7) // 8 * 8
    vt = torch.full((nh, hd, t_ld), 3.0, dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_vision_qkv_post(d.data_ptr(), pos.data_ptr(), inv.data_ptr(), N, nh, hd, float(scale),
                                      vt.data_ptr(), t_ld, 0), "qkv_post")
    torch.cuda.synchronize()
    cmp_bf16(d[:, :2], want[:, :2], "qkv_post q (scaled), k", max_mismatch=0.01)
    assert torch.equal(d[:, 2].cpu().float(), qkv[:, 2]), "V must stay untouched"
    assert torch.equal(vt[:, :, :N].cpu().float(), qkv[:, 2].permute(1, 2, 0)), "V^T must be an exact transpose"
