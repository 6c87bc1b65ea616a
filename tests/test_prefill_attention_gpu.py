"""The bf16 prefill attention of every path against sdpa at long and boundary lengths, through the C ABI and through
the real engine.

Kernels (C ABI):
  attention_fa   b200_attention_fa: a fresh prompt (Lq = S), TMA-fed, a 2-slot K / V^T ring that each CTA walks twice
                 (pass 1: row max and sum, pass 2: P.V); b200_attention_fa_seg: the same kernel on a part of larger
                 tensors (the vision tower's frames at q0 = k0 = offset) and with a segment table (the batched
                 prefill's block-diagonal causal attention)
  attention_tc   b200_attention with hd % 16 == 0: a chunk over the KV pool (K / V planes of one row, k_hs = cap*hd,
                 q a packed qkv row), bottom-right causal; and the vision tower's fallback for frames whose offset is
                 not a multiple of 8 (non-causal, q / k / v at qkv + off*3E)
  two-pass       b200_attention with hd % 16 != 0: scores of ATT_QT rows kept in shared memory, so S is bounded

Inputs sit on the quarter grid of `_grid` (values in [-2, 2]): with hd <= 128 every score, of pre-scaled q too (a
2^-15 grid, sums below 2^21 of it), is exact in fp32 in any summation order.  Every byte a call must not read holds
NaN (pool positions >= S and the other pool row, V^T columns [S, s_ld), everything past q_tot / k_tot inside an
allocation), and the output is pre-filled with a sentinel that rows and head columns the call does not own must keep.
The one exception is the caller contract of segmented attention: a key tile may run past a segment's S into the next
segment (or its padding tokens) within k_tot; those scores are masked, but their V^T columns must be finite, because
a NaN times a zero probability is NaN.  Long cases compute the reference on selected rows only: every row at a
query or key tile edge +-1, the first and last rows, and 32 random rows.

Engine (a one-layer rig): pos3 = 0 (the rotary is the identity), embeddings of +-1 rows (ln1 leaves them unchanged),
wqkv a selection matrix with quarter-grid weights (each output column reads one input column, so q / k / v are exact
on the grid), wo = I, a zero MLP, and a head [I; 0] behind a unit final norm: logits[t, :H] = rms_norm(bf16(x_t +
att_t)).  The workspace is poisoned with NaN before every call, the KV pool is NaN outside the rows written, and the
K / V rows written must be exact.

The bar is the decode file's (`_compare`), measured for the prefill paths on an H100 (see `_compare`)."""
import numpy as np
import pytest
import torch

from _util import cmp_bf16
from test_decode_attention_gpu import GEOMS, _grid, _rms_ref

pytestmark = pytest.mark.gpu

# ---- tiling constants -----------------------------------------------------------------------------------------------
FA_TQ, FA_TK = 128, 128          # attention_fa.cu: query rows per CTA, keys per tile (a ring of 2 K / V^T slots)
TC_TQ, TC_TK = 128, 128          # attention_tc.cu: TQ, TK
ATT_QT = 16                      # attention.cu: query rows per CTA of the two-pass attention_kernel
ATT_SMEM_MAX = 220 * 1024        # attention.cu: the two-pass kernel's shared-memory limit
B200_ERR_INVALID = 1             # include/b200vlm.h
assert (FA_TQ, FA_TK) == (TC_TQ, TC_TK)   # sel_rows serves both tensor-core kernels
SENTINEL = -7.0


def cdiv(a, b):
    return -(-a // b)


def round8(x):
    return cdiv(x, 8) * 8


def two_pass_smem(hd, S):        # attention.cu attention(): q tile in fp32 + ATT_QT rows of S bf16 scores
    return ATT_QT * hd * 4 + ATT_QT * S * 2


def two_pass_max_s(hd):
    S = 1
    while two_pass_smem(hd, S + 1) <= ATT_SMEM_MAX:
        S += 1
    return S


def test_two_pass_limit_matches_the_kernel_formula():
    """the two-pass kernel's largest S at the head dims that reach it (hd % 16 != 0); a change of its shared-memory
    layout shows here first"""
    assert [two_pass_max_s(hd) for hd in (72, 88)] == [6896, 6864]


# ---- reference --------------------------------------------------------------------------------------------------------
def _lib():
    from mlx_vlm_b200 import _native as N
    return N.lib()


def _check(rc, what):
    from mlx_vlm_b200 import _native as N
    N.check(rc, what)


# The bar.  The kernels sum the softmax denominator and P.V in fp32 in another order than the oracle (and the
# pipelined kernel takes exp2 from the SFU): now and then a probability rounds to the neighbouring bf16 value, and
# when it is one of the larger ones most outputs of that q head row move by an ulp.  Measured on an H100 80GB HBM3
# (700 W) over the 124 comparisons of this file (two runs, identical results): at most rel L2 2.3e-4 and 0.37 %
# differing elements (the two-pass kernel, hd 72, S = 1000); the engine rig's outputs stay below rel L2 4e-5.  The
# bar is the decode file's: rel L2 <= 2e-3 and at most 2 % plus one q head of differing elements.  A key tile dropped
# or counted twice moves the selected rows of a causal prompt of 385 or 2049 tokens by rel L2 0.12 to 0.28 (computed
# with the oracle).
def _compare(got, want, name, n_heads):
    return cmp_bf16(got, want, name, rel_l2=2e-3, max_mismatch=0.02 + 1 / n_heads)


def sel_rows(Lq, S, causal, seed):
    """query rows where the tiling changes: query tile edges +-1, rows whose visible key count crosses a key tile
    edge +-1, the first and last rows, 32 random rows"""
    s = {0, Lq - 1}
    for e in range(FA_TQ, Lq + 1, FA_TQ):
        s |= {e - 2, e - 1, e, e + 1}
    if causal:   # row i sees S - Lq + i + 1 keys
        for e in range(FA_TK, S + 2, FA_TK):
            for n in (e - 1, e, e + 1):
                s.add(n - 1 - (S - Lq))
    s |= set(np.random.default_rng(seed).integers(0, Lq, 32).tolist())
    return sorted(x for x in s if 0 <= x < Lq)


def sdpa_rows(q, k, v, causal, rows=None):
    """oracle sdpa: q (Lq, nh, hd) unscaled, k / v (S, nkv, hd), fp32 CPU; the output rows `rows` (all: None),
    (n_rows, nh, hd).  Row i sees S - Lq + i + 1 keys when causal (bottom-right)."""
    from oracle import mlx_semantics as Sm
    R = Sm.Rounder("bf16")
    Lq, nh, hd = q.shape
    S = k.shape[0]
    scale = hd ** -0.5
    qh, kh, vh = q.transpose(0, 1)[None], k.transpose(0, 1)[None], v.transpose(0, 1)[None]
    if rows is None:
        return Sm.sdpa(R, qh, kh, vh, scale, causal)[0].transpose(0, 1)
    out = []
    for i in rows:
        n = S - Lq + i + 1 if causal else S
        out.append(Sm.sdpa(R, qh[:, :, i:i + 1], kh[:, :, :n], vh[:, :, :n], scale, False)[0, :, 0])
    return torch.stack(out)


def _want_rows(Lq, S, nh, causal, seed, full_limit=3e6):
    """None (every row) when the full reference is cheap, else the selected rows"""
    return None if Lq * S * nh <= full_limit else sel_rows(Lq, S, causal, seed)


def _prescale(q):
    """bf16(q * bf16(scale)): what the rotary kernels hand the pipelined kernel"""
    from oracle import mlx_semantics as Sm
    R = Sm.Rounder("bf16")
    return R.r(q * R.scalar(q.shape[-1] ** -0.5))


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")


def _rand(gen, *shape):
    return _grid(torch.randn(*shape, generator=gen)).float()


def _out(rows, o_ts):
    return torch.full((rows, o_ts), SENTINEL, dtype=torch.bfloat16, device="cuda")


def _check_out(out, owned_rows, width, want, name, nh, rows=None):
    """rows `owned_rows` (a list) columns [0, width) against want (rows: the compared subset of owned_rows); every
    other element keeps the sentinel"""
    o = out.float().cpu()
    keep = torch.ones_like(o, dtype=torch.bool)
    keep[torch.as_tensor(owned_rows, dtype=torch.long), :width] = False
    assert bool((o[keep] == SENTINEL).all()), f"{name}: wrote rows or columns it does not own"
    got = o[torch.as_tensor(owned_rows if rows is None else rows, dtype=torch.long), :width]
    return _compare(got, want.reshape(got.shape), name, nh)


# ---- attention_fa: fresh prompt -----------------------------------------------------------------------------------------
FA_LENGTHS = (1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 384, 385, 2047, 2048, 2049)
FA_HEADS = [(hd, G) for hd in (64, 72, 80, 128) for G in (1, 2, 6, 7, 8)]   # hd 72 is padded to 80 for the MMAs


def _heads(G):
    nkv = 1 if G == 8 else 2
    return G * nkv, nkv


def _fa_cases():
    out = []
    for i, L in enumerate(FA_LENGTHS):
        for causal in (1, 0):   # every (hd, G) once causal and once not
            hd, G = FA_HEADS[(i + 10 * causal) % len(FA_HEADS)]
            out.append((L, causal, hd) + _heads(G))
    for causal in (1, 0):
        out.append((8192, causal, 128, 2, 1))
    return out


def _fa_inputs(L, nh, nkv, hd, seed):
    gen = torch.Generator().manual_seed(seed)
    return _rand(gen, L, nh, hd), _rand(gen, L, nkv, hd), _rand(gen, L, nkv, hd)


def _fa_operands(q, k, v, extra=16):
    """the engine's layout: q pre-scaled in a packed qkv row (q_ts = QKV), K as the workspace copy (kv head, token,
    dim), V^T (kv head, dim, token) with s_ld = round8(tokens); NaN past the tokens, in the V^T padding columns and in
    one more kv head of each allocation"""
    T, nh, hd = q.shape
    nkv = k.shape[1]
    QKV = (nh + 2 * nkv) * hd
    s_ld = round8(T)
    qkv = _nan(T + extra, QKV)
    qkv[:T, :nh * hd] = _prescale(q).reshape(T, -1).to(torch.bfloat16).cuda()
    kws = _nan(nkv + 1, T + extra, hd)
    kws[:nkv, :T] = k.transpose(0, 1).to(torch.bfloat16).cuda()
    vt = _nan(nkv + 1, hd, s_ld)
    vt[:nkv, :, :T] = v.permute(1, 2, 0).to(torch.bfloat16).cuda()
    return qkv, QKV, kws, (T + extra) * hd, vt, s_ld


@pytest.mark.parametrize("L,causal,hd,nh,nkv", _fa_cases(),
                         ids=[f"L{c[0]}-{'causal' if c[1] else 'full'}-hd{c[2]}-{c[3]}x{c[4]}" for c in _fa_cases()])
def test_attention_fa_fresh_prompt(L, causal, hd, nh, nkv):
    q, k, v = _fa_inputs(L, nh, nkv, hd, seed=L * 7 + causal)
    qkv, QKV, kws, k_hs, vt, s_ld = _fa_operands(q, k, v)
    o_ts = nh * hd + 8
    out = _out(L + 8, o_ts)
    torch.cuda.synchronize()
    _check(_lib().b200_attention_fa(qkv.data_ptr(), QKV, hd, kws.data_ptr(), hd, k_hs, vt.data_ptr(), hd * s_ld, s_ld,
                                    out.data_ptr(), o_ts, nh, nkv, hd, L, L, causal, 0), "attention_fa")
    torch.cuda.synchronize()
    rows = _want_rows(L, L, nh, causal, seed=L)
    want = sdpa_rows(q, k, v, bool(causal), rows)
    _check_out(out, list(range(L)), nh * hd, want, f"attention_fa L={L} causal={causal} hd={hd} {nh}x{nkv}", nh,
               rows)


# ---- attention_fa on parts of larger tensors: vision frames, the batched prefill's segment table -------------------------
def test_attention_fa_vision_frames():
    """three frames of one image batch at token offsets 0, 64, 264 (multiples of 8) in a 397-token qkv buffer: the
    middle frame's last key tile reads into the last frame, the last frame's tiles read past k_tot; once per frame
    (q0 = k0 = offset, as the vision tower calls it) and once through a segment table"""
    lib = _lib()
    nh, hd = 16, 80
    E = nh * hd
    lens = [64, 200, 133]
    offs = [0, 64, 264]
    N = sum(lens)
    t_ld = round8(N)
    gen = torch.Generator().manual_seed(3)
    q, k, v = _rand(gen, N, nh, hd), _rand(gen, N, nh, hd), _rand(gen, N, nh, hd)
    qkv = _nan(N + 16, 3 * E)
    qkv[:N, :E] = _prescale(q).reshape(N, E).to(torch.bfloat16).cuda()
    qkv[:N, E:2 * E] = k.reshape(N, E).to(torch.bfloat16).cuda()
    qkv[:N, 2 * E:] = v.reshape(N, E).to(torch.bfloat16).cuda()
    vt = _nan(nh + 1, hd, t_ld)
    vt[:nh, :, :N] = v.permute(1, 2, 0).to(torch.bfloat16).cuda()
    want = torch.cat([sdpa_rows(q[o:o + n], k[o:o + n], v[o:o + n], False) for o, n in zip(offs, lens)])
    segs = torch.tensor([[o, n, o, n] for o, n in zip(offs, lens)], dtype=torch.int32, device="cuda")
    k_ptr = qkv.data_ptr() + E * 2
    for mode in ("per frame", "table"):
        out = _out(N + 8, E + 8)
        torch.cuda.synchronize()
        if mode == "per frame":
            for o, n in zip(offs, lens):
                _check(lib.b200_attention_fa_seg(qkv.data_ptr(), 3 * E, hd, k_ptr, 3 * E, hd, vt.data_ptr(), hd * t_ld,
                                                 t_ld, out.data_ptr(), E + 8, nh, nh, hd, n, n, 0, o, N, o, N, None, 0,
                                                 0), "attention_fa_seg")
        else:
            _check(lib.b200_attention_fa_seg(qkv.data_ptr(), 3 * E, hd, k_ptr, 3 * E, hd, vt.data_ptr(), hd * t_ld,
                                             t_ld, out.data_ptr(), E + 8, nh, nh, hd, max(lens), max(lens), 0, 0, N, 0,
                                             N, segs.data_ptr(), len(lens), 0), "attention_fa_seg")
        torch.cuda.synchronize()
        _check_out(out, list(range(N)), E, want, f"attention_fa vision frames {lens} ({mode})", nh)


@pytest.mark.parametrize("nh,nkv,hd", [(12, 2, 128), (28, 4, 128), (8, 1, 64)])
def test_attention_fa_prefill_batch_table(nh, nkv, hd):
    """the batched prefill's launch: sequences of 1, 9, 127, 129 and 300 tokens, each padded to a multiple of 8 with
    finite padding tokens, block-diagonal causal through the (q0, Lq, k0, S) table; padding rows keep the sentinel"""
    lens = [1, 9, 127, 129, 300]
    offs = [int(o) for o in np.cumsum([0] + [round8(n) for n in lens[:-1]])]
    T = offs[-1] + round8(lens[-1])
    q, k, v = _fa_inputs(T, nh, nkv, hd, seed=nh + hd)
    qkv, QKV, kws, k_hs, vt, s_ld = _fa_operands(q, k, v)
    segs = torch.tensor([[o, n, o, n] for o, n in zip(offs, lens)], dtype=torch.int32, device="cuda")
    o_ts = nh * hd + 8
    out = _out(T + 8, o_ts)
    torch.cuda.synchronize()
    _check(_lib().b200_attention_fa_seg(qkv.data_ptr(), QKV, hd, kws.data_ptr(), hd, k_hs, vt.data_ptr(), hd * s_ld,
                                        s_ld, out.data_ptr(), o_ts, nh, nkv, hd, max(lens), max(lens), 1, 0, T, 0, T,
                                        segs.data_ptr(), len(lens), 0), "attention_fa_seg")
    torch.cuda.synchronize()
    owned = [o + i for o, n in zip(offs, lens) for i in range(n)]
    want = torch.cat([sdpa_rows(q[o:o + n], k[o:o + n], v[o:o + n], True) for o, n in zip(offs, lens)])
    _check_out(out, owned, nh * hd, want, f"attention_fa batch table {lens} {nh}x{nkv} hd={hd}", nh)


# ---- b200_attention -> attention_tc: a chunk over the KV pool ------------------------------------------------------------
TC_GEOMS = [(12, 2, 128), (28, 4, 128), (16, 8, 128), (8, 1, 64), (16, 16, 64)]


def _tc_cases():
    out = []
    for Lq in (1, 8, 127, 128, 129, 2048):
        for ctx0 in (1, 127, 128, 2048, 4095):
            out.append((Lq, ctx0) + TC_GEOMS[len(out) % len(TC_GEOMS)])
    return out


def _pool_case(Lq, ctx0, nh, nkv, hd, seed):
    """K / V planes (2, rows 2, n_kv, cap, hd) holding S = ctx0 + Lq keys in row 1 and NaN elsewhere, q a packed qkv
    row (unscaled), NaN past Lq"""
    S = ctx0 + Lq
    cap = cdiv(S + 1, 256) * 256
    gen = torch.Generator().manual_seed(seed)
    q, k, v = _rand(gen, Lq, nh, hd), _rand(gen, S, nkv, hd), _rand(gen, S, nkv, hd)
    kv = _nan(2, 2, nkv, cap, hd)
    kv[0, 1, :, :S] = k.transpose(0, 1).to(torch.bfloat16).cuda()
    kv[1, 1, :, :S] = v.transpose(0, 1).to(torch.bfloat16).cuda()
    QKV = (nh + 2 * nkv) * hd
    qkv = _nan(Lq + 8, QKV)
    qkv[:Lq, :nh * hd] = q.reshape(Lq, -1).to(torch.bfloat16).cuda()
    return q, k, v, kv, cap, qkv, QKV


def _run_attention(qkv, QKV, kv, cap, out, o_ts, nh, nkv, hd, Lq, S, causal):
    return _lib().b200_attention(qkv.data_ptr(), QKV, hd, kv[0, 1].data_ptr(), hd, cap * hd, kv[1, 1].data_ptr(), hd,
                                 cap * hd, out.data_ptr(), o_ts, nh, nkv, hd, Lq, S, causal, float(hd ** -0.5), 0)


@pytest.mark.parametrize("Lq,ctx0,nh,nkv,hd", _tc_cases(),
                         ids=[f"Lq{c[0]}-ctx{c[1]}-{c[2]}x{c[3]}-hd{c[4]}" for c in _tc_cases()])
def test_attention_tc_chunk_over_pool(Lq, ctx0, nh, nkv, hd):
    """the engine's later prefill chunk: q from packed qkv rows, K / V straight out of the pool (k_hs = cap*hd),
    bottom-right causal"""
    S = ctx0 + Lq
    q, k, v, kv, cap, qkv, QKV = _pool_case(Lq, ctx0, nh, nkv, hd, seed=Lq * 31 + ctx0)
    o_ts = nh * hd + 8
    out = _out(Lq + 8, o_ts)
    torch.cuda.synchronize()
    _check(_run_attention(qkv, QKV, kv, cap, out, o_ts, nh, nkv, hd, Lq, S, 1), "attention")
    torch.cuda.synchronize()
    rows = _want_rows(Lq, S, nh, True, seed=Lq + ctx0)
    want = sdpa_rows(q, k, v, True, rows)
    _check_out(out, list(range(Lq)), nh * hd, want, f"attention_tc Lq={Lq} ctx0={ctx0} {nh}x{nkv} hd={hd}", nh, rows)


@pytest.mark.parametrize("nh,hd,off,seg", [(16, 80, 36, 196), (16, 64, 36, 129), (16, 80, 100, 300)])
def test_attention_tc_vision_frame_fallback(nh, hd, off, seg):
    """a frame at a token offset that is not a multiple of 8 (after a 6 x 6-patch image): the vision tower calls
    b200_attention at qkv + off*3E, non-causal; every other row of the buffer is NaN"""
    E = nh * hd
    N = off + seg + 20
    gen = torch.Generator().manual_seed(off + seg)
    q, k, v = _rand(gen, seg, nh, hd), _rand(gen, seg, nh, hd), _rand(gen, seg, nh, hd)
    qkv = _nan(N, 3 * E)
    qkv[off:off + seg] = torch.cat([q.reshape(seg, E), k.reshape(seg, E), v.reshape(seg, E)], 1).to(
        torch.bfloat16).cuda()
    out = _out(N, E + 8)
    base = qkv.data_ptr() + off * 3 * E * 2
    torch.cuda.synchronize()
    _check(_lib().b200_attention(base, 3 * E, hd, base + E * 2, 3 * E, hd, base + 2 * E * 2, 3 * E, hd,
                                 out.data_ptr() + off * (E + 8) * 2, E + 8, nh, nh, hd, seg, seg, 0,
                                 float(hd ** -0.5), 0), "attention")
    torch.cuda.synchronize()
    want = sdpa_rows(q, k, v, False)
    _check_out(out, list(range(off, off + seg)), E, want, f"attention_tc vision frame off={off} seg={seg} hd={hd}", nh)


# ---- the two-pass attention_kernel (hd % 16 != 0) ------------------------------------------------------------------------
@pytest.mark.parametrize("hd", [72, 88])
@pytest.mark.parametrize("Lq,S", [(17, 1000), (40, "max")])
def test_attention_two_pass(hd, Lq, S):
    nh, nkv = 4, 2
    S = two_pass_max_s(hd) if S == "max" else S
    q, k, v, kv, cap, qkv, QKV = _pool_case(Lq, S - Lq, nh, nkv, hd, seed=hd + S)
    o_ts = nh * hd + 8
    out = _out(Lq + 8, o_ts)
    torch.cuda.synchronize()
    _check(_run_attention(qkv, QKV, kv, cap, out, o_ts, nh, nkv, hd, Lq, S, 1), "attention")
    torch.cuda.synchronize()
    want = sdpa_rows(q, k, v, True)
    _check_out(out, list(range(Lq)), nh * hd, want, f"attention two-pass Lq={Lq} S={S} hd={hd}", nh)


@pytest.mark.parametrize("hd", [72, 88])
def test_attention_two_pass_refuses_one_past_its_limit(hd):
    nh, nkv, Lq = 4, 2, 8
    S = two_pass_max_s(hd) + 1
    _, _, _, kv, cap, qkv, QKV = _pool_case(Lq, S - Lq, nh, nkv, hd, seed=1)
    out = _out(Lq, nh * hd)
    torch.cuda.synchronize()
    rc = _run_attention(qkv, QKV, kv, cap, out, nh * hd, nh, nkv, hd, Lq, S, 1)
    assert rc == B200_ERR_INVALID
    assert b"too long for the two-pass kernel" in _lib().b200_last_error()
    torch.cuda.synchronize()
    assert bool((out.float() == SENTINEL).all())


# ---- the engine's prefill paths ----------------------------------------------------------------------------------------
class Rig:
    """one-layer engine of geometry g whose all-row logits are rms_norm(bf16(x + attention)) (module docstring)"""
    EPS = 1e-6
    INTER = 256

    def __init__(self, g):
        from mlx_vlm_b200 import _native as N
        from mlx_vlm_b200.engine import Engine
        from mlx_vlm_b200.models.qwen2_vl.qwen2_vl import WeightArena, weight_manifest
        nh, nkv, hd, qk = GEOMS[g]
        self.g, self.nh, self.nkv, self.hd, self.qk = g, nh, nkv, hd, qk
        self.H = H = nh * hd
        self.QKV = QKV = (nh + 2 * nkv) * hd
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = H, 1, self.INTER
        c.n_heads, c.n_kv_heads, c.head_dim = nh, nkv, hd
        c.vocab = H + 8
        c.rms_eps, c.rope_theta = self.EPS, 1000000.0
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = hd // 2, 0, 0
        c.tie_embeddings = 0
        c.external_vision = 1
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = H, 1e-5
        self.eng = eng = Engine(c, torch.device("cuda", 0))
        arena = WeightArena(weight_manifest(c), eng.device)
        gen = torch.Generator().manual_seed(sum(map(ord, g)) + 1)
        # output column j of qkv reads input column sel[j] with weight w[j]
        self.sel = torch.randint(0, H, (QKV,), generator=gen)
        self.w = _rand(gen, QKV)
        if qk:   # q / k heads of +-1: their RMSNorm is exactly +-(norm weight)
            self.w[:(nh + nkv) * hd] = torch.randint(0, 2, ((nh + nkv) * hd,), generator=gen) * 2.0 - 1.0
        wqkv = torch.zeros(QKV, H)
        wqkv[torch.arange(QKV), self.sel] = self.w
        fill = {"lm.embed": torch.zeros(c.vocab, H), "lm.norm": torch.ones(H),
                "lm.head": torch.cat([torch.eye(H), torch.zeros(8, H)]),
                "lm.0.ln1": torch.ones(H), "lm.0.ln2": torch.ones(H),
                "lm.0.wqkv": wqkv, "lm.0.bqkv": torch.zeros(QKV), "lm.0.wo": torch.eye(H),
                "lm.0.wgu": torch.zeros(2 * self.INTER, H), "lm.0.wd": torch.zeros(H, self.INTER)}
        for name, t in fill.items():
            v = arena.view(name)
            v.copy_(t.to(torch.bfloat16))
            eng.set_weight(name, v)
        self.arena = arena
        if qk:
            self.qn = (1.0 + torch.randint(-3, 4, (hd,), generator=gen) / 8).to(torch.bfloat16)
            self.kn = (1.0 + torch.randint(-3, 4, (hd,), generator=gen) / 8).to(torch.bfloat16)
            self.qn_d, self.kn_d = self.qn.cuda(), self.kn.cuda()
            eng.set_weight("lm.0.qn", self.qn_d)
            eng.set_weight("lm.0.kn", self.kn_d)
        self.gen = gen
        torch.cuda.synchronize()

    def embeds(self, T):
        return torch.randint(0, 2, (T, self.H), generator=self.gen).float() * 2 - 1

    def qkv_ref(self, x):
        """q (T, nh, hd), k, v (T, nkv, hd) of embeddings x: exact (selection, rotary at position 0)"""
        T = x.shape[0]
        a = x[:, self.sel] * self.w
        nq, nk = self.nh * self.hd, self.nkv * self.hd
        q = a[:, :nq].reshape(T, self.nh, self.hd)
        k = a[:, nq:nq + nk].reshape(T, self.nkv, self.hd)
        v = a[:, nq + nk:].reshape(T, self.nkv, self.hd)
        if self.qk:
            q, k = _rms_ref(q, self.qn.float(), self.EPS), _rms_ref(k, self.kn.float(), self.EPS)
        return q, k, v

    def pool(self, cap, rows):
        from mlx_vlm_b200.models.cache import KVPool
        p = KVPool(1, self.nkv, self.hd, self.eng.device, batch=rows, capacity=cap)
        p.buf.fill_(float("nan"))
        return p

    def poison_workspace(self, T):
        self.eng.ensure_workspace(tokens=T)
        self.eng.workspace.fill_(0xFF)   # bf16 0xFFFF and fp32 0xFFFFFFFF are NaN
        torch.cuda.synchronize()

    def ws_bytes(self, offset, nbytes):
        ws = self.eng.workspace
        base = ((ws.data_ptr() + 255) & ~255) - ws.data_ptr()
        return ws[base + offset:base + offset + nbytes]

    def lm_ws(self, T):
        """csrc/engine.cu lm_ws: byte offsets of the residual stream h (the first carve) and of the T x 2 x inter pad
        that no kernel addresses (after h, xn, qkv, att)"""
        a = lambda n: cdiv(n, 256) * 256
        H, QKV, QH = self.H, self.QKV, self.nh * self.hd
        pad = 2 * a(T * H * 2) + a(T * QKV * 2) + a(T * QH * 2)
        return 0, pad, T * 2 * self.INTER * 2

    def h_rows(self, T):
        return self.ws_bytes(0, T * self.H * 2).view(torch.bfloat16).view(T, self.H).float().cpu()

    def check_pad(self, T, name):
        _, off, n = self.lm_ws(T)
        pad = self.ws_bytes(off, n)
        assert bool((pad == 0xFF).all()), f"{name}: a kernel wrote the unaddressed pad of lm_ws"


_RIGS = {}


def rig(g):
    if g not in _RIGS:
        _RIGS[g] = Rig(g)
    return _RIGS[g]


def _residual_ref(x, att):
    from oracle import mlx_semantics as Sm
    R = Sm.Rounder("bf16")
    return R.r(x + att.reshape(att.shape[0], -1))


def _logits_ref(r, h):
    from oracle import mlx_semantics as Sm
    return Sm.rms_norm(Sm.Rounder("bf16"), h, torch.ones(r.H), r.EPS)


def _check_kv(r, pool, row, pos0, k, v, before, name):
    """pool row `row` positions [pos0, pos0 + len(k)) hold k / v exactly; nothing else changed (before: int16 bits)"""
    T = k.shape[0]
    buf = pool.buf
    assert torch.equal(buf[0, 0, row, :, pos0:pos0 + T].float().cpu(), k.transpose(0, 1)), f"{name}: K rows"
    assert torch.equal(buf[0, 1, row, :, pos0:pos0 + T].float().cpu(), v.transpose(0, 1)), f"{name}: V rows"
    changed = buf.view(torch.int16) != before
    changed[0, :, row, :, pos0:pos0 + T] = False
    assert not bool(changed.any()), f"{name}: the prefill wrote other pool positions"


def _prefill(r, pool, row, x, ctx0, name, rows=None):
    """prefill of embeddings x at ctx0 into pool row `row` (positions < ctx0 already filled) with all-row logits on a
    poisoned workspace; checks K / V, the logits and the residual stream h of the workspace on `rows`"""
    eng = r.eng
    T = x.shape[0]
    eng.bind_pool(pool)
    eng.set_kv_row(row)
    r.poison_workspace(T)
    before = pool.buf.view(torch.int16).clone()
    logits = torch.full((T, round8(r.H + 8)), SENTINEL, dtype=torch.bfloat16, device="cuda")
    emb = x.to(torch.bfloat16).cuda()
    pos3 = torch.zeros(3, T, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.prefill(emb, pos3, ctx0, 0, logits)
    eng.stream.synchronize()
    assert eng.device_error() == 0
    q, k, v = r.qkv_ref(x)
    _check_kv(r, pool, row, ctx0, k, v, before, name)
    K = pool.buf[0, 0, row, :, :ctx0 + T].float().cpu().transpose(0, 1)
    V = pool.buf[0, 1, row, :, :ctx0 + T].float().cpu().transpose(0, 1)
    sel = list(range(T)) if rows is None else rows
    att = sdpa_rows(q, K, V, True, rows)
    h = _residual_ref(x[sel], att)
    _compare(r.h_rows(T)[sel], h, f"{name} residual h", r.nh)
    _compare(logits[sel, :r.H], _logits_ref(r, h), f"{name} logits", r.nh)
    r.check_pad(T, name)


@pytest.mark.parametrize("g", ["2b", "7b", "q3"])
def test_engine_fresh_prompt(g):
    """ctx0 = 0: the pipelined kernel on the chunk's own K copy and V^T, row 1 of a two-row pool"""
    r = rig(g)
    T = 300
    pool = r.pool(512, 2)
    _prefill(r, pool, 1, r.embeds(T), 0, f"engine fa {g} T={T}")


@pytest.mark.parametrize("g", ["2b", "7b", "q3"])
@pytest.mark.parametrize("ctx0,T", [(300, 200), (2048, 129)])
def test_engine_second_chunk(g, ctx0, T):
    """ctx0 > 0: attention() over the pool row, which holds ctx0 earlier keys and the chunk's appended rows"""
    r = rig(g)
    pool = r.pool(cdiv(ctx0 + T + 1, 256) * 256, 2)
    gen = torch.Generator(device="cuda").manual_seed(ctx0 + T)
    pool.buf[0, :, 1, :, :ctx0] = _grid(torch.randn(2, r.nkv, ctx0, r.hd, device="cuda", generator=gen))
    _prefill(r, pool, 1, r.embeds(T), ctx0, f"engine attention() {g} ctx0={ctx0} T={T}")


@pytest.mark.parametrize("g", ["2b", "7b", "q3"])
def test_engine_prefill_batch(g):
    """four fresh prompts into permuted rows of a five-row pool in one pass; the residual stream h is read from the
    workspace (its offset is checked against a single prefill by test_engine_fresh_prompt)"""
    r = rig(g)
    eng = r.eng
    lens, rows = [9, 130, 1, 300], [3, 0, 4, 1]
    offs = [int(o) for o in np.cumsum([0] + [round8(n) for n in lens[:-1]])]
    T = offs[-1] + round8(lens[-1])
    pool = r.pool(512, 5)
    eng.bind_pool(pool)
    x = r.embeds(T)   # the padding rows are finite too
    r.poison_workspace(T)
    before = pool.buf.view(torch.int16).clone()
    emb = x.to(torch.bfloat16).cuda()
    pos3 = torch.zeros(3, T, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.prefill_batch(emb, pos3, lens, rows)
    eng.stream.synchronize()
    assert eng.device_error() == 0
    h = r.h_rows(T)
    changed = pool.buf.view(torch.int16) != before
    for o, n, row in zip(offs, lens, rows):
        name = f"engine prefill_batch {g} seq {n} tokens -> row {row}"
        q, k, v = r.qkv_ref(x[o:o + n])
        assert torch.equal(pool.buf[0, 0, row, :, :n].float().cpu(), k.transpose(0, 1)), f"{name}: K rows"
        assert torch.equal(pool.buf[0, 1, row, :, :n].float().cpu(), v.transpose(0, 1)), f"{name}: V rows"
        changed[0, :, row, :, :n] = False
        _compare(h[o:o + n], _residual_ref(x[o:o + n], sdpa_rows(q, k, v, True)), name, r.nh)
    assert not bool(changed.any()), f"prefill_batch {g}: wrote pool positions outside the sequences"
    r.check_pad(T, f"prefill_batch {g}")


def test_engine_large_prompt_in_place_residual():
    """7B geometry (hidden 3584), T = 3600: T * hidden * 4 B > 48 MiB, so o_proj and down_proj add the residual in the
    bf16 GEMM epilogue in place (h = h + x.W^T).  The first call of the problem class measures the GEMM's candidate
    configurations on the caller's operands; those launches must not overwrite h.  The second call uses the cached
    configuration.  Both must give the same, correct rows."""
    r = rig("7b")
    T = 3600
    assert T * r.H * 4 > 48 << 20
    rows = sel_rows(T, T, True, seed=5)
    for call in ("first (measures)", "second (cached)"):
        pool = r.pool(cdiv(T + 1, 256) * 256, 2)
        _prefill(r, pool, 1, r.embeds(T), 0, f"engine 7b T={T} {call} call", rows=rows)
        del pool
