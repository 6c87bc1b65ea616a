"""The weight-major wgmma GEMM `gemm_wt` (csrc/gemm_wt.cu) and its split-K row op `finish_rows`, in every
configuration the measured choice can run, at every family's shapes, against an exact float64 reference.

`gemm_wt_tuned` times a candidate list on the device and caches the winner per (64-token bucket, N, K, mode); a later
call in the bucket reuses it with TN clamped to round16(T) and the split re-fitted to the partial buffer.  So every
candidate of every T in a bucket must be right.  The list comes from the library itself (b200_gemm_wt_candidates,
the same function the tuner times); the bucket reuse is restated in `reuse` below from gemm_wt_tuned's two lines.

THE BAR.  Every operand sits on a grid: X and W are small integers times a per-tensor power of two, bias and
residual are bf16 values on grids of their own.  Every product is then a multiple of one unit u, and while
sum_k |x w| < 2^24 u (asserted per case, `unit_bound`) every partial sum in any order is exact in fp32: in any wgmma
accumulation order, any split, any finish_rows order.  So the accumulator equals the float64 product exactly and the
only roundings left are the kernels' own rounding points:

  BF16 EPI_NONE, bias, residual (separate and in place), PARTIAL tiles and the finish_rows h, F32 EPI_NONE with
  bias and res32, SPLIT EPI_NONE:   bit-exact against float64 rounded at the kernel's points (single fp32 adds
  mirrored in float32; the integer sums land on many bf16 ties, so round-half-to-even is checked too).
  SwiGLU, bf16 GELU fast / exact, the finish_rows RMSNorm:   the intervals of tests/test_decode_gemv_gpu.py.
  finish_rows LayerNorm (`ln_iv`):  mu = fl(sum h) / N is within e_mu = gamma(N) sum|h| / N + |mu| u of the mean;
      the two-pass variance about the computed mean is (1/N) sum (h - mu_c)^2 (1 + theta), |theta| <= gamma(N + 3)
      (the difference, its square or an FMA, the sum, the division), and sum (h - mu_c)^2 = sum (h - mu)^2 +
      N (mu - mu_c)^2; rstd = 1 / sqrtf(var + eps) adds three correctly rounded operations and the square root halves
      the relative error of its argument: delta_r = (gamma(N + 3) + e_mu^2 / (var + eps)) / 2 + 3u.  Then
      y = fl(fl(h - mu_c) rstd) lies within rstd e_mu + |h - mu| rstd (delta_r + 2u) of (h - mu) rstd, is rounded to
      bf16, and x w and + b follow with their roundings (`corners`).
  erff / tanhf:  within 2 ulp (CUDA C++ Programming Guide, mathematical functions): |f| 2^-22.
  The fp32 tower epilogues (`f32_epi_band`, absolute bands on an fp32 result that is never rounded to bf16):
      GELU fast   v sigmoid(fl(1.702f v)):  the argument carries |g| u, which moves sigmoid by at most
                  sigma (1 - sigma) |g| u <= sigma |g| u; __expf / + 1 / __fdividef give sigmoid_band(g); the
                  product one u:  |out| (sigmoid_band(g) + |g| u + u).
      GELU exact  v (1 + erff(fl(v / sqrt2f))) 0.5:  the quotient carries |a| u, erf' <= 2 / sqrt(pi), erff 2 ulp,
                  1 + e one u of its result, the product one u:
                  0.5 |v| (1.13 |a| u e^(-a^2) + |erf a| 2^-22 + |1 + erf a| u) + |out| u.
      GELU tanh   0.5 v (1 + tanhf(0.79788f (v + 0.044715f v v v))):  the cubic is three products (3u relative) and
                  nvcc may contract it with + v into one FMA (--fmad=true, no fast-math in build.py), so the sum is
                  within |s| u + 3.01 |c| u either way; the scaling one u, tanh' <= 1 - t^2, tanhf 2 ulp, 1 + t one
                  u, the product one u.
  Each band is widened by 1 % (_BAND_SLACK) for the second-order terms.  test_the_wt_bands_on_the_host shows they
  admit fp32 restatements of the kernel formulas in two summation orders, with and without FMA, and refuse an
  element two ulps off.
  SPLIT operands in F32 / SPLIT:  x_hi in {-1, 0, 1} s and x_lo in {-1, 0, 1} s 2^-9, which keeps n_parts = 2 exact.
  SPLIT with a GELU must give hi = bf16(v') and lo = bf16(v' - hi) for one fp32 v' within the band.

Exactness rests on one assumption: the bf16 wgmma keeps every bit of fp32 sums below 2^24 u, in any order it adds.
test_exactness_probe runs K = 64 and K = 18944 first; with it failing, every exact check below would fail too.

Output the call does not own starts as a sentinel and must keep it; partial buffers start as NaN, and X columns
beyond K (ldx > K) hold NaN, so a read there poisons the result.  Each check prints its count of elements that differ
from the float64-then-round reference and the worst band ratio, as test_decode_gemv_gpu.py does."""
import ctypes as C
import math
import os
import zlib
from typing import NamedTuple

import pytest
import torch

from test_decode_gemv_gpu import U, Iv, check, corners, rbf, rms_iv, rounded, sigmoid_band, swiglu_iv, bf16_round, \
    bf16_step, gamma, _BAND_SLACK

BF16, PARTIAL, SWIGLU, F32, SPLIT = 0, 1, 2, 3, 4
EPI_NONE, GELU_FAST, GELU_EXACT, GELU_TANH = 0, 1, 2, 3
NORM_NONE, NORM_RMS, NORM_LN = 0, 1, 2
MODE_NAME = {BF16: "BF16", PARTIAL: "PARTIAL", SWIGLU: "SWIGLU", F32: "F32", SPLIT: "SPLIT"}
EPI_NAME = {EPI_NONE: "none", GELU_FAST: "gelu_fast", GELU_EXACT: "gelu_exact", GELU_TANH: "gelu_tanh"}

# ---- constants and formulas of the host code ------------------------------------------------------------------------
WT_BK, WT_ROWS, WT_TN_AUTO, WT_EPI_TOK = 64, 128, 128, 64
FIN_N_MAX = 8192                    # gemm_wt.cu finish_rows: N <= FIN_N_MAX
PREFILL_PARTIAL = 48 << 20          # engine.cu WT_PARTIAL_BYTES
BATCH_PARTIAL = 64 << 20            # decode_batch.cu partial_bytes
TOWER_SMS = 132                     # tower_f32.cu b200_gemm_wt_f32: the measured choice is made for 132 SMs
EPS = 1e-6


def cdiv(a, b):
    return -(-a // b)


def round16(x):
    return (x + 15) & ~15


def round8(x):
    return (x + 7) & ~7


def pad64(n):
    return cdiv(n, 64) * 64


_LIB = None


def lib():
    """the library, built if needed (the candidate list is host code: it runs without a GPU)"""
    global _LIB
    if _LIB is None:
        from mlx_vlm_b200.build import build
        from mlx_vlm_b200 import _native as N
        build()
        _LIB = N.lib()
    return _LIB


def ncheck(rc, what):
    from mlx_vlm_b200 import _native as N
    N.check(rc, what)


def candidates(T, N, K, mode, inter, allow_split, sms, partial_bytes):
    """the configurations gemm_wt_tuned times for this problem, the cost model's choice first"""
    buf, n = (C.c_int * 256)(), C.c_int()
    ncheck(lib().b200_gemm_wt_candidates(T, N, K, mode, inter, int(allow_split), sms, partial_bytes, buf, 64,
                                         C.byref(n)), "gemm_wt_candidates")
    assert n.value <= 64
    return [tuple(buf[4 * i:4 * i + 4]) for i in range(n.value)]


def fits(split, T, N, mode, partial_bytes):
    return not (mode == PARTIAL and split * T * N * 4 > partial_bytes)


def reuse(cfg, T, N, K, mode, partial_bytes):
    """gemm_wt_tuned's two lines for a configuration cached at another T of the bucket: TN clamped to round16(T),
    the split re-fitted to the partial buffer (None: the call refuses)"""
    TN, KS, st, sp = cfg
    kbt = cdiv(K, WT_BK)
    TN = min(TN, round16(T))
    while sp > 1 and not fits(sp, T, N, mode, partial_bytes):
        sp = cdiv(kbt, cdiv(kbt, sp - 1))
    return (TN, KS, st, sp) if fits(sp, T, N, mode, partial_bytes) else None


# ---- the case table ----------------------------------------------------------------------------------------------------
class Gemm(NamedTuple):
    """one GEMM as a caller runs it"""
    name: str
    mode: int
    N: int
    K: int                  # columns of W (towers: K_w)
    epi: int = EPI_NONE
    bias: bool = False
    res: str = ""           # BF16: "sep" / "inplace"; F32: "res32" (in place, as every tower caller)
    inter: int = 0          # SWIGLU
    norm: int = NORM_NONE   # PARTIAL: the finish_rows norm of the caller
    ln_w: bool = True
    ln_b: bool = True
    ldc: int = 0            # 0: N (SWIGLU: inter)
    ldx: int = 0            # 0: K
    pbytes: int = 0         # PARTIAL: the caller's partial buffer
    split_ok: bool = False
    n_parts: int = 2        # F32 / SPLIT
    tower_sms: bool = False # the measured choice at 132 SMs whatever the device (b200_gemm_wt_f32)


class Family(NamedTuple):
    name: str
    hidden: int
    inter: int
    nh: int
    nkv: int
    hd: int
    vocab: int
    qkv_bias: bool


FAMILIES = [
    Family("qwen2vl-2b", 1536, 8960, 12, 2, 128, 151936, True),
    Family("qwen2vl-7b", 3584, 18944, 28, 4, 128, 152064, True),
    Family("qwen3vl-2b", 2048, 6144, 16, 8, 128, 151936, False),
    Family("qwen3vl-4b", 2560, 9728, 32, 8, 128, 151936, False),
    Family("mistral-7b", 4096, 14336, 32, 8, 128, 32003, False),
    Family("llama-7b", 4096, 11008, 32, 32, 128, 32064, False),
    Family("smolvlm-256m", 576, 1536, 9, 3, 64, 49280, False),
    Family("smolvlm-2.2b", 2048, 8192, 32, 32, 64, 49280, False),
]
PREFILL_T = (1, 16, 17, 48, 49, 96, 97, 128, 129, 577, 1000)
BATCH_B = (1, 3, 8, 16)
HEAD_T_MAX = 129


def lm_prefill(f):
    """engine.cu prefill: linear (qkv, head), linear_residual_norm (o_proj, down: PARTIAL + finish_rows, or the in-place
    bf16 epilogue once T N 4 > 48 MiB), gate/up with SwiGLU"""
    H, I, QKV, QH = f.hidden, f.inter, (f.nh + 2 * f.nkv) * f.hd, f.nh * f.hd
    pre = dict(pbytes=PREFILL_PARTIAL, split_ok=True)
    return [Gemm("qkv", BF16, QKV, H, bias=f.qkv_bias),
            Gemm("o_proj", PARTIAL, H, QH, norm=NORM_RMS, **pre),
            Gemm("o_proj in place", BF16, H, QH, res="inplace"),
            Gemm("gate/up", SWIGLU, 2 * I, H, inter=I),
            Gemm("down", PARTIAL, H, I, norm=NORM_RMS, **pre),
            Gemm("down, last layer", PARTIAL, H, I, norm=NORM_NONE, **pre),
            Gemm("head", BF16, f.vocab, H, ldc=round8(f.vocab))]


def lm_batch(f):
    """decode_batch.cu bd_enqueue_step: qkv, o_proj and down as split-K partials (o_proj and down finished with the
    residual and RMSNorm; the qkv partials are summed by the attention kernel), gate/up with SwiGLU, the head"""
    H, I, QKV, QH = f.hidden, f.inter, (f.nh + 2 * f.nkv) * f.hd, f.nh * f.hd
    bd = dict(pbytes=BATCH_PARTIAL, split_ok=True)
    return [Gemm("qkv partials", PARTIAL, QKV, H, **bd),
            Gemm("o_proj", PARTIAL, H, QH, norm=NORM_RMS, **bd),
            Gemm("gate/up", SWIGLU, 2 * I, H, inter=I),
            Gemm("down", PARTIAL, H, I, norm=NORM_RMS, **bd),
            Gemm("head", BF16, f.vocab, H, ldc=round8(f.vocab))]


def prefill_ts(f, g):
    if g.name == "head":
        return [t for t in PREFILL_T if t <= HEAD_T_MAX]
    if g.name == "o_proj in place":
        return [3511] if f.name == "qwen2vl-7b" else []    # T N 4 = 48 MiB + 2 KiB: the in-place bf16 path
    ts = list(PREFILL_T)
    if f.name == "qwen2vl-7b" and g.name == "o_proj":
        ts.append(3510)                                     # the partial buffer exactly full
    return ts


def tower_rows():
    """(tower, Gemm, T list).  Qwen2-VL's bf16 ViT and merger (engine.cu vision); the fp32-accurate towers through
    b200_gemm_wt_f32 (models/tower_ops.py encoder, llava, idefics2 / 3, qwen2_5_vl)"""
    vit = dict(pbytes=PREFILL_PARTIAL, split_ok=True)
    T2 = (64, 577, 1000)
    out = [("qwen2vl-vit", Gemm("patch", BF16, 1280, 1176), T2),
           ("qwen2vl-vit", Gemm("qkv", BF16, 3840, 1280, bias=True), T2),
           ("qwen2vl-vit", Gemm("proj + LN", PARTIAL, 1280, 1280, bias=True, norm=NORM_LN, **vit), T2),
           ("qwen2vl-vit", Gemm("fc1 gelu_fast", BF16, 5120, 1280, GELU_FAST, bias=True), T2),
           ("qwen2vl-vit", Gemm("fc2 + LN", PARTIAL, 1280, 5120, bias=True, norm=NORM_LN, **vit), T2),
           ("qwen2vl-vit", Gemm("merger fc1 gelu_exact", BF16, 5120, 5120, GELU_EXACT, bias=True), (16, 144, 250)),
           ("qwen2vl-vit", Gemm("merger fc2", BF16, 1536, 5120, bias=True), (16, 144, 250))]
    tw = dict(tower_sms=True)
    for tower, E, M, epi, Kp in (("clip-l", 1024, 4096, GELU_FAST, 588), ("siglip", 1152, 4304, GELU_TANH, 588)):
        Ts = (97, 577)
        out += [(tower, Gemm("patch", F32, E, Kp, **tw), Ts),
                (tower, Gemm("qkv", F32, 3 * E, E, bias=True, **tw), Ts),
                (tower, Gemm("out + res32", F32, E, E, bias=True, res="res32", **tw), Ts),
                (tower, Gemm(f"fc1 {EPI_NAME[epi]}", SPLIT, M, E, epi, bias=True, **tw), Ts),
                (tower, Gemm("fc2 + res32", F32, E, M, bias=True, res="res32", **tw), Ts)]
    out += [("llava-projector", Gemm("linear_1 gelu_exact", SPLIT, 4096, 1024, GELU_EXACT, bias=True, **tw), (577,)),
            ("idefics3-connector", Gemm("proj", F32, 2048, 4608, **tw), (64, 169)),
            ("smolvlm-connector", Gemm("proj", F32, 576, 12288, **tw), (64, 169)),
            ("qwen2.5vl", Gemm("patch, n_parts 1", F32, 1280, 1176, n_parts=1, **tw), (64, 577)),
            ("qwen2.5vl", Gemm("gate/up", F32, 2 * 3424, 1280, bias=True, **tw), (64, 577)),
            ("qwen2.5vl", Gemm("down + res32", F32, 1280, 3424, bias=True, res="res32", **tw), (64, 577)),
            ("qwen2.5vl", Gemm("merger fc1 gelu_exact", SPLIT, 5120, 5120, GELU_EXACT, bias=True, **tw), (16, 145))]
    return out


def edge_rows():
    """shapes no family has, for the cases the code distinguishes: K < 64, N < 128 with N % 8 != 0, ldc % 8 != 0 and
    ldx > K in bf16, SwiGLU with inter % 64 != 0, finish_rows at N = FIN_N_MAX and LayerNorm without weight / bias"""
    e = dict(pbytes=PREFILL_PARTIAL, split_ok=True)
    return [("edge", Gemm("K 40, N 100, residual", BF16, 100, 40, bias=True, res="sep"), (1, 17, 130)),
            ("edge", Gemm("N 200 ldc 204 ldx 584, gelu_fast", BF16, 200, 520, GELU_FAST, bias=True, res="sep",
                          ldc=204, ldx=584), (17, 130)),
            ("edge", Gemm("swiglu inter 200", SWIGLU, 400, 1000, inter=200), (7, 130)),
            ("edge", Gemm("finish N 8192 + RMS", PARTIAL, FIN_N_MAX, 2048, bias=True, norm=NORM_RMS, **e), (17, 129)),
            ("edge", Gemm("LN without weight", PARTIAL, 1024, 3000, bias=True, norm=NORM_LN, ln_w=False, **e),
             (9, 97)),
            ("edge", Gemm("LN without bias", PARTIAL, 1032, 3000, norm=NORM_LN, ln_b=False, **e), (9, 97)),
            ("edge", Gemm("F32 N 1000 + res32, gelu_tanh", F32, 1000, 520, GELU_TANH, bias=True, res="res32",
                          tower_sms=True), (17, 130)),
            ("edge", Gemm("SPLIT N 302", SPLIT, 302, 200, tower_sms=True), (17, 130))]


def table():
    """[(row id, Gemm, [T])] of every shape the families run"""
    out = []
    for f in FAMILIES:
        for g in lm_prefill(f):
            ts = prefill_ts(f, g)
            if ts:
                out.append((f"{f.name} prefill {g.name}", g, ts))
        for g in lm_batch(f):
            out.append((f"{f.name} lock-step {g.name}", g, list(BATCH_B)))
    for tower, g, ts in tower_rows() + edge_rows():
        out.append((f"{tower} {g.name}", g, list(ts)))
    return out


def kdim(g):
    """the K the GEMM sees: the split operand repeats the weight k-blocks n_parts times"""
    return g.n_parts * pad64(g.K) if g.mode in (F32, SPLIT) else g.K


def sms_for(g, sms):
    return TOWER_SMS if g.tower_sms else sms


def runnable(g, T, sms):
    """every configuration that can run at T: the candidates of each T' of T's 64-bucket, reused at T"""
    K, out = kdim(g), []
    tb = (T + 63) // 64
    for t2 in range(64 * (tb - 1) + 1, 64 * tb + 1):
        for c in candidates(t2, g.N, K, g.mode, g.inter, g.split_ok, sms_for(g, sms), g.pbytes):
            r = reuse(c, T, g.N, K, g.mode, g.pbytes)
            if r is not None and r not in out:
                out.append(r)
    return out


WIDE = ((144, 1, 4, 1), (192, 1, 3, 1), (256, 1, 2, 1), (256, 2, 2, 1))   # the 16-chunk instantiation


def plan(g, ts, sms):
    """{T: [configurations]}: at every T the cost model's choice; every other configuration that can run at some T of
    the row once, at the first T whose own candidates hold it, else at the first T it can run at"""
    K = kdim(g)
    out, seen = {}, set()
    cands = {T: candidates(T, g.N, K, g.mode, g.inter, g.split_ok, sms_for(g, sms), g.pbytes) for T in ts}
    for T in ts:
        out[T] = cands[T][:1]
        seen |= set(out[T])
    for T in ts:
        for c in cands[T]:
            if c not in seen:
                out[T].append(c)
                seen.add(c)
    for T in ts:
        for c in runnable(g, T, sms):
            if c not in seen:
                out[T].append(c)
                seen.add(c)
    return out


def plan_wide(g, ts):
    """explicit 16-chunk configurations on the bf16 shapes of the Qwen2-VL ViT, the edge rows and the towers' fc2"""
    return {T: [c for c in WIDE if fits(c[3], T, g.N, g.mode, g.pbytes)] for T in ts if T > 128}


def full_table(sms):
    rows = []
    for rid, g, ts in table():
        p = plan(g, ts, sms)
        if rid.startswith(("qwen2vl-vit", "edge", "clip-l fc2")) and g.mode != SWIGLU:
            for T, cs in plan_wide(g, ts).items():
                p[T] += [c for c in cs if c not in p[T]]
        rows.append((rid, g, p))
    return rows


# ---- what the table reaches ----------------------------------------------------------------------------------------------
def features(g, T, cfg):
    """the cases of gemm_wt / finish_rows one launch takes"""
    TN, KS, st, sp = cfg
    K = kdim(g)
    kbt = cdiv(K, WT_BK)
    kbps = cdiv(kbt, sp)
    lens = [min(kbt, (s + 1) * kbps) - s * kbps for s in range(sp)]
    n_it = [cdiv(n, KS) for n in lens]
    tower = g.mode in (F32, SPLIT)
    f = {f"gemm_wt_kernel<{'true' if tower else 'false'}, {16 if TN > 128 else 8}>",
         f"{MODE_NAME[g.mode]} epilogue {EPI_NAME[g.epi]}", f"{MODE_NAME[g.mode]} bias {g.bias}"}
    if g.res:
        f.add(f"{MODE_NAME[g.mode]} residual {g.res}")
    ldc = g.ldc or (g.inter if g.mode == SWIGLU else g.N)
    if g.mode == BF16:
        if g.N % 8:
            f.add("element-wise store of the last chunk (N % 8 != 0)")
        if ldc % 8:
            f.add("element-wise stores (ldc % 8 != 0)")
    if g.mode in (F32, SPLIT, PARTIAL) and g.N % 4:
        f.add("element-wise fp32 tail (N % 4 != 0)")
    if g.N < 128:
        f.add("N < 128")
    if g.N % 128:
        f.add("N % 128 != 0")
    if g.mode == SWIGLU and g.inter % 64:
        f.add("SwiGLU inter % 64 != 0")
    if K < 64:
        f.add("K < 64")
    if K % 64:
        f.add("K % 64 != 0")
    if (g.ldx or (2 * pad64(g.K) if tower else K)) > K:
        f.add("ldx > K")
    if min(n_it) < st:
        f.add("n_it < stages")
    if max(n_it) > 2 * st:
        f.add("ring wraps twice")
    if KS == 2 and any(n % 2 for n in lens):
        f.add("short last KS = 2 stage")
    if len(set(lens)) > 1:
        f.add("splits of unequal length")
    if TN % 64:
        f.add("TN % 64 != 0 (a partial epilogue pass)")
    if T < TN:
        f.add("T < TN")
    if T % TN:
        f.add("T % TN != 0")
    if g.mode == PARTIAL and g.N <= FIN_N_MAX:
        f.add(f"finish_rows<{'1024, 2' if T <= 32 else '256, 8'}>")
        if sp == 1:
            f.add("finish_rows S = 1")
        if sp in (8, 9):
            f.add(f"finish_rows S = {sp}")
        if sp > 16:
            f.add("finish_rows S > 16")
        if g.N == FIN_N_MAX:
            f.add("finish_rows N = FIN_N_MAX")
        if g.norm == NORM_LN:
            f.add(f"finish_rows LN weight {g.ln_w} bias {g.ln_b}")
        else:
            f.add(f"finish_rows norm {g.norm}")
    return f


def reached(sms):
    """{case: bool} over the planned launches, and every distinct configuration of every shape's runnable set"""
    want = {f"gemm_wt_kernel<{a}, {b}>" for a in ("false", "true") for b in (8, 16)}
    want |= {f"{MODE_NAME[m]} epilogue {EPI_NAME[e]}" for m, e in ((BF16, EPI_NONE), (BF16, GELU_FAST),
             (BF16, GELU_EXACT), (PARTIAL, EPI_NONE), (SWIGLU, EPI_NONE), (F32, EPI_NONE), (F32, GELU_TANH),
             (SPLIT, EPI_NONE), (SPLIT, GELU_FAST), (SPLIT, GELU_EXACT), (SPLIT, GELU_TANH))}
    want |= {f"{MODE_NAME[m]} bias {b}" for m in (BF16, F32, SPLIT, PARTIAL) for b in (True, False)}
    want |= {"BF16 residual sep", "BF16 residual inplace", "F32 residual res32"}
    want |= {"element-wise store of the last chunk (N % 8 != 0)", "element-wise stores (ldc % 8 != 0)",
             "element-wise fp32 tail (N % 4 != 0)", "N < 128", "N % 128 != 0", "SwiGLU inter % 64 != 0", "K < 64",
             "K % 64 != 0", "ldx > K", "n_it < stages", "ring wraps twice", "short last KS = 2 stage",
             "splits of unequal length", "TN % 64 != 0 (a partial epilogue pass)", "T < TN", "T % TN != 0",
             "finish_rows<1024, 2>", "finish_rows<256, 8>", "finish_rows S = 1", "finish_rows S = 8",
             "finish_rows S = 9", "finish_rows S > 16", "finish_rows N = FIN_N_MAX", "finish_rows norm 0",
             "finish_rows norm 1", "finish_rows LN weight True bias True", "finish_rows LN weight False bias True",
             "finish_rows LN weight True bias False"}
    got = set()
    runs = {}
    all_runnable_covered = True
    for rid, g, p in full_table(sms):
        for T, cs in p.items():
            for c in cs:
                got |= features(g, T, c)
                runs.setdefault(rid, set()).add(c)
        need = set()
        for T in p:
            need |= set(runnable(g, T, sms))
        if not need <= runs[rid]:
            all_runnable_covered = False
    out = {w: w in got for w in sorted(want)}
    out["every runnable configuration of every shape runs"] = all_runnable_covered
    return out


@pytest.mark.parametrize("sms", [132, 114])
def test_case_table_reaches_every_case(sms):
    """the table reaches every instantiation, mode x epilogue, store path, tiling edge and finish_rows case, and runs
    every configuration the measured choice can pick for each shape, at the SM counts of the H100 SXM (132) and
    PCIe (114)"""
    got = reached(sms)
    for case, ok in got.items():
        print(f"{sms} SMs  {'reached' if ok else 'MISSED '}  {case}")
    assert all(got.values()), [c for c, ok in got.items() if not ok]
    n_shapes = n_launch = 0
    cfgs = set()
    for rid, g, p in full_table(sms):
        n_shapes += 1
        for T, cs in p.items():
            n_launch += len(cs)
            cfgs |= set(cs)
    print(f"{sms} SMs: {n_shapes} shapes, {len(cfgs)} distinct configurations, {n_launch} launches")


def test_candidate_spot_values():
    """worked by hand from gemm_wt.cu: qwen2vl-2b lock-step down (B = 8, N = 1536, K = 8960, 64 MiB).  140 k-blocks,
    12 row blocks, one 16-token tile; the splits for one and two waves are 132 / 12 = 11 and 264 / 12 = 22, re-fitted
    to cdiv(140, cdiv(140, 22)) = 20 (7 k-blocks each, so KS = 2 ends on a half stage); KS = 2 gets 208 KB / 36 KB = 5
    stages, KS = 1 110 KB / 18 KB = 6.  At 114 SMs: 9 and 19 -> cdiv(140, 8) = 18."""
    for sms, (a, b) in ((132, (11, 20)), (114, (9, 18))):
        got = candidates(8, 1536, 8960, PARTIAL, 0, True, sms, BATCH_PARTIAL)
        rest = [c for s in (1, a, b) for c in ((16, 2, 5, s), (16, 1, 6, s))]
        model = got[0]
        assert model in rest, (sms, got)
        assert got == [model] + [c for c in rest if c != model], (sms, got)
    # the bucket reuse: a configuration cached at T = 100 reused at T = 70 is clamped to TN 80; a split that no longer
    # fits the buffer is re-fitted
    assert reuse((128, 2, 4, 1), 70, 1536, 8960, BF16, 0) == (80, 2, 4, 1)
    assert reuse((96, 1, 6, 20), 600, 18944, 3584, PARTIAL, PREFILL_PARTIAL) == (96, 1, 6, 1)
    # the engine's boundary between the partial path and the in-place bf16 path (7B o_proj, N = 3584)
    assert 3510 * 3584 * 4 <= PREFILL_PARTIAL < 3511 * 3584 * 4
    # the list is the tuner's: a partial buffer too small for one split gives none
    assert candidates(3511, 3584, 3584, PARTIAL, 0, True, 132, PREFILL_PARTIAL) == []


# ---- the grid data ----------------------------------------------------------------------------------------------------------
def wmax_for(g):
    """the widest integer range of W that keeps sum |x w| < 2^24 u (the split operand: |x| <= 1 + 2^-9 in units
    2^9 u, so each product is at most |w| (2^9 + 1) u)"""
    K = g.K
    for w in (8, 4, 2, 1):
        per = w * ((2 ** 9 + 1) if (g.mode in (F32, SPLIT) and g.n_parts == 2) else (1 if g.mode in (F32, SPLIT)
                                                                                      else 8))
        if K * per < 2 ** 24:
            return w
    raise AssertionError(g)


def unit_bound(X, W, x_unit, w_unit):
    """max over outputs of sum_k |x w| in units u = x_unit w_unit (must stay below 2^24 for exact fp32 sums)"""
    m = 0.0
    for i in range(0, W.shape[0], 8192):
        m = max(m, float((X.abs().double() @ W[i:i + 8192].abs().double().T).max()))
    return m / (x_unit * w_unit)


class Data(NamedTuple):
    X: torch.Tensor         # the operand as launched ([T, ldx] bf16; NaN beyond the valid columns)
    W: torch.Tensor         # [N, ldw] bf16, K_w valid columns
    Xv: torch.Tensor        # float64 [T, K_w] values that multiply W (the split operand: hi + lo; n_parts 1: hi)
    bias: torch.Tensor
    res: torch.Tensor       # bf16 [T, ldc] or fp32 [T, N]
    nw: torch.Tensor
    nb: torch.Tensor


def make(g, T, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, device="cuda", generator=gen).double()
    Kw, N = g.K, g.N
    wm = wmax_for(g)
    tower = g.mode in (F32, SPLIT)
    # magnitudes: the accumulator's standard deviation a few units, so GELU and SwiGLU see their curved range
    if tower:
        s = 2.0 ** -int(math.log2(max(1.0, math.sqrt(Kw) * wm / 2)))
        hi, lo = ri(-1, 1, T, Kw) * s, ri(-1, 1, T, Kw) * s * 2.0 ** -9
        if g.n_parts == 1:
            lo = torch.zeros_like(lo)
        ldx = 2 * pad64(Kw)
        X = torch.full((T, ldx), float("nan"), dtype=torch.bfloat16, device="cuda")
        X[:, :pad64(Kw)] = 0
        X[:, :Kw] = hi.to(torch.bfloat16)
        if g.n_parts == 2:
            X[:, pad64(Kw):pad64(Kw) + Kw] = lo.to(torch.bfloat16)
            X[:, pad64(Kw) + Kw:] = 0
        Xv, x_unit = hi + lo, s * 2.0 ** -9
        # rows round8(K_w) apart, as the callers pad them (a 16-byte row pitch); NaN past K_w
        W = torch.full((N, round8(Kw)), float("nan"), dtype=torch.bfloat16, device="cuda")
        W[:, :Kw] = (ri(-wm, wm, N, Kw) * 2.0 ** -2).to(torch.bfloat16)
        w_unit = 2.0 ** -2
    else:
        ex = -int(math.log2(max(1.0, math.sqrt(Kw) * 24 / 2)))
        ldx = g.ldx or Kw
        X = torch.full((T, ldx), float("nan"), dtype=torch.bfloat16, device="cuda")
        Xv = ri(-8, 8, T, Kw) * 2.0 ** ex
        X[:, :Kw] = Xv.to(torch.bfloat16)
        x_unit = 2.0 ** ex
        W = ri(-wm, wm, N, Kw).to(torch.bfloat16)
        w_unit = 1.0
    bound = unit_bound(Xv, W[:, :Kw], x_unit, w_unit)
    assert bound < 2 ** 24, f"sum |x w| = {bound} u: fp32 sums would not be exact"
    bias = (ri(-64, 64, N) * 2.0 ** -5).to(torch.bfloat16) if g.bias else None
    res = None
    ldc = g.ldc or (g.inter if g.mode == SWIGLU else N)
    if g.res in ("sep", "inplace") or g.mode == PARTIAL:
        res = (ri(-255, 255, T, ldc) * 2.0 ** -5).to(torch.bfloat16)
    elif g.res == "res32":
        res = (ri(-2 ** 20, 2 ** 20, T, N) * 2.0 ** -17).float()
    nw = (1 + ri(-32, 32, N) / 64).to(torch.bfloat16) if g.norm != NORM_NONE and g.ln_w else None
    nb = (ri(-32, 32, N) / 16).to(torch.bfloat16) if g.norm == NORM_LN and g.ln_b else None
    return Data(X, W, Xv, bias, res, nw, nb)


# ---- float64 references and bands ---------------------------------------------------------------------------------------
def acc64(d, k0=0, k1=None):
    """the exact accumulator [T, N] over columns [k0, k1) of W (float64: every partial sum is exact)"""
    k1 = d.Xv.shape[1] if k1 is None else k1
    return d.Xv[:, k0:k1] @ d.W[:, k0:k1].double().T


def f32(x):
    return x.float()


def ln_iv(h, w, b, eps):
    """finish_rows LayerNorm of exact bf16 rows h (float64 [T, N]): see the module docstring"""
    N = h.shape[-1]
    eps = float(torch.tensor(eps, dtype=torch.float32))
    mu = h.mean(-1, keepdim=True)
    e_mu = gamma(N) * h.abs().sum(-1, keepdim=True) / N + mu.abs() * U
    var = ((h - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    d_r = (gamma(N + 3) + e_mu ** 2 / (var + eps)) / 2 + 3 * U
    y = (h - mu) * rstd
    band = rstd * e_mu + (h - mu).abs() * rstd * (d_r + 2 * U)
    o = rounded(y, band)
    o = Iv(o.lo, o.hi, o.ref)
    if w is not None:
        o = corners(lambda a, ww: rbf(a.float() * ww.float()), o, Iv.exact(w.double().expand_as(h)))
    if b is not None:
        o = corners(lambda a, bb: rbf(a.float() + bb.float()), o, Iv.exact(b.double().expand_as(h)))
    return o


def gelu_fast_iv(v):
    """gelu_fast_bf (common.cuh) of exact bf16 values: rbf(x rbf(sigmoid_f(rbf(1.703125 x))))"""
    g = rbf(f32(v) * 1.703125)
    sg = torch.sigmoid(g)
    band = sigmoid_band(g) * _BAND_SLACK
    s = Iv(bf16_round(sg * (1 - band)), bf16_round(sg * (1 + band)), bf16_round(sg))
    return corners(lambda a, b: rbf(a.float() * b.float()), Iv.exact(v), s)


def gelu_exact_iv(v):
    """gelu_exact_bf (common.cuh): a = rbf(x / 1.4140625f), rbf(erff(a)) within 2 ulp, then three roundings"""
    a = rbf(f32(v) / 1.4140625)
    e = torch.erf(a)
    ei = rounded(e, e.abs() * 2.0 ** -22)
    ei = Iv(ei.lo, ei.hi, ei.ref)
    c = corners(lambda t: rbf(1.0 + t.float()), ei)
    dd = corners(lambda x, cc: rbf(x.float() * cc.float()), Iv.exact(v), c)
    return corners(lambda t: rbf(t.float() * 0.5), dd)


SQRT2F = float(torch.tensor(1.41421356237309515, dtype=torch.float32))
C1702, C0797, C0044 = (float(torch.tensor(x, dtype=torch.float32)) for x in (1.702, 0.7978845608028654, 0.044715))


def f32_epi_band(v, epi):
    """(reference, band) of the fp32 tower epilogue (wt_stage_f32) at exact fp32 values v (float64)"""
    if epi == GELU_FAST:
        g = v * C1702
        ref = v * torch.sigmoid(g)
        band = ref.abs() * (sigmoid_band(g) + g.abs() * U + U)
    elif epi == GELU_EXACT:
        a = v / SQRT2F
        e = torch.erf(a)
        ref = v * (1 + e) * 0.5
        band = 0.5 * v.abs() * (1.13 * a.abs() * U * torch.exp(-a * a) + e.abs() * 2.0 ** -22 + (1 + e).abs() * U) \
            + ref.abs() * U
    elif epi == GELU_TANH:
        c = C0044 * v * v * v
        s = v + c
        uu = C0797 * s
        t = torch.tanh(uu)
        ref = 0.5 * v * (1 + t)
        d_uu = uu.abs() * U + C0797 * (s.abs() * U + 3.01 * c.abs() * U)
        band = 0.5 * v.abs() * (t.abs() * 2.0 ** -22 + (1 - t * t) * d_uu + (1 + t).abs() * U) + ref.abs() * U
    else:
        return v, torch.zeros_like(v)
    return ref, band * _BAND_SLACK + 2.0 ** -140


def check_f32(got, ref, band, name):
    """|got - ref| <= band elementwise (fp32 results never rounded to bf16)"""
    got = got.double().reshape(ref.shape)
    err = (got - ref).abs()
    ok = err <= band
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:8].tolist()
        lines = [f"  {tuple(i)}: got {got[tuple(i)].item():.9g}, reference {ref[tuple(i)].item():.9g}, band "
                 f"{band[tuple(i)].item():.3g}" for i in bad]
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements outside the band\n" + "\n".join(lines))
    ratio = (err / band.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    diff = int((got.float().double() != ref.float().double()).sum())
    print(f"{name}: {diff} / {ok.numel()} differ from float64-then-round, worst band ratio {ratio:.3g}")
    return diff, ratio


def exact(got, want, name):
    return check(got, Iv.exact(want), name)


def two_ulps_off(t, i):
    """t with element i moved two bf16 ulps up"""
    t = t.clone()
    one = torch.ones(1, dtype=torch.float64, device=t.device)
    t.view(-1)[i] = bf16_step(bf16_step(t.double().view(-1)[i:i + 1], one), one).to(t.dtype)[0]
    return t


def test_the_wt_bands_on_the_host():
    """the LayerNorm band admits fp32 restatements of finish_rows in two summation orders with and without FMA; the
    fp32 GELU bands admit the restated epilogues with and without FMA; each refuses an element two ulps off"""
    g = torch.Generator().manual_seed(1)
    T, N = 8, 4096
    h = (torch.randn(T, N, generator=g) * 3 + 0.7).to(torch.bfloat16).double()
    w = (1 + torch.randn(N, generator=g) * 0.2).to(torch.bfloat16)
    b = (torch.randn(N, generator=g) * 0.5).to(torch.bfloat16)
    iv = ln_iv(h, w, b, EPS)
    hf = h.float()
    crossed = 0
    for order in ("forward", "reversed"):
        for fma in (False, True):
            idx = torch.arange(N) if order == "forward" else torch.arange(N - 1, -1, -1)
            s1 = torch.zeros(T)
            for k in idx:
                s1 = s1 + hf[:, k]
            mu = s1 / N
            v = torch.zeros(T)
            for k in idx:
                dk = hf[:, k] - mu
                v = (v.double() + dk.double() * dk.double()).float() if fma else v + dk * dk
            rstd = 1.0 / torch.sqrt(v / N + torch.tensor(EPS, dtype=torch.float32))
            o = ((hf - mu[:, None]) * rstd[:, None]).to(torch.bfloat16).float()
            o = (o * w.float()).to(torch.bfloat16).float()
            o = (o + b.float()).to(torch.bfloat16)
            n, _ = check(o, iv, f"host LN, {order}, fma={fma}")
            crossed += n
    assert crossed > 0, "no element differs from the float64 reference: the case does not test the band"
    i = int(iv.ref.abs().argmax())
    with pytest.raises(AssertionError, match="1 of"):
        check(two_ulps_off(iv.hi.to(torch.bfloat16), i), Iv(iv.lo, iv.hi, iv.ref), "host LN, two ulps off")
    # the fp32 epilogues on exact fp32 inputs
    v = (torch.randn(1 << 16, generator=g) * 3).double().float().double()
    vf = v.float()
    outs = {
        GELU_FAST: [vf * torch.sigmoid(vf * C1702)],
        GELU_EXACT: [vf * (1.0 + torch.erf(vf / SQRT2F)) * 0.5],
    }
    c2 = (C0044 * vf) * vf
    no_fma = vf + c2 * vf
    with_fma = (vf.double() + c2.double() * vf.double()).float()
    outs[GELU_TANH] = [0.5 * vf * (1.0 + torch.tanh(C0797 * s)) for s in (no_fma, with_fma)]
    for epi, cands in outs.items():
        ref, band = f32_epi_band(v, epi)
        for got in cands:
            check_f32(got, ref, band, f"host fp32 {EPI_NAME[epi]}")
        # the band is a few dozen fp32 ulps wide at most where the output is not a cancellation (v >= 0.5; __expf's
        # error grows with |g|), 2^-17 relative: far inside one bf16 ulp ...
        pos = v >= 0.5
        ulps = (band[pos] / (ref[pos].abs() * 2.0 ** -23)).max().item()
        print(f"host fp32 {EPI_NAME[epi]}: the band is at most {ulps:.2f} ulps of the output for v >= 0.5")
        assert ulps < 64
        # ... and an element two ulps past its edge is refused
        bad = cands[0].clone()
        j = int(pos.nonzero()[0])
        up = torch.tensor([math.inf])
        edge = torch.tensor([(ref[j] + band[j]).item()], dtype=torch.float64).float()
        bad[j] = float(torch.nextafter(torch.nextafter(edge, up), up))
        with pytest.raises(AssertionError, match="1 of"):
            check_f32(bad, ref, band, f"host fp32 {EPI_NAME[epi]}, two ulps past the band")
    # the split-operand exactness assertion refuses a case that breaks the bound (the SmolVLM connector at |w| = 4)
    assert wmax_for(Gemm("proj", F32, 576, 12288)) == 2 and wmax_for(Gemm("proj", F32, 2048, 4608)) == 4
    assert 12288 * 4 * (2 ** 9 + 1) >= 2 ** 24 > 12288 * 2 * (2 ** 9 + 1)


# ---- the GPU runs ---------------------------------------------------------------------------------------------------------
SENT_BF16 = 0x7B7B            # a finite bf16 (~1.3e36) no output takes
STATS = {}


def _note(key, res):
    n, w = res
    s = STATS.setdefault(key, [0, 0.0, 0])
    s[0] += n
    s[1] = max(s[1], w)
    s[2] += 1


def sentinel(shape):
    return torch.full(shape, SENT_BF16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def keep_sentinel(buf, owned, name):
    """every element of buf outside the owned index region still holds the sentinel"""
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[owned] = False
    bits = buf.view(torch.int16) if buf.dtype == torch.bfloat16 else buf.view(torch.int32)
    want = SENT_BF16 if buf.dtype == torch.bfloat16 else None
    if want is None:
        assert bool(torch.isnan(buf[mask]).all()), f"{name}: wrote outside its output"
    else:
        assert bool((bits[mask] == want).all()), f"{name}: wrote outside its output"


def _cfg(c):
    return (C.c_int * 4)(*c)


class Ref:
    """the references of one (shape, T), computed once and shared by every configuration"""

    def __init__(self, g, T, d):
        self.g, self.T, self.d = g, T, d
        A = acc64(d)
        N = g.N
        if g.mode == BF16:
            v = f32(A) + (f32(d.bias.double()) if d.bias is not None else 0)
            v = rbf(v)
            if g.epi == GELU_FAST:
                self.iv = gelu_fast_iv(v)
            elif g.epi == GELU_EXACT:
                self.iv = gelu_exact_iv(v)
            else:
                self.iv = Iv.exact(v)
            if g.res:
                r = d.res[:, :N].double()
                self.iv = corners(lambda a, rr: rbf(rr.float() + a.float()), self.iv, Iv.exact(r))
        elif g.mode == SWIGLU:
            I = g.inter
            self.iv = swiglu_iv(Iv.exact(rbf(f32(A[:, :I]))), Iv.exact(rbf(f32(A[:, I:]))))
        elif g.mode == PARTIAL:
            self.A = A
            h = rbf(f32(A) + (f32(d.bias.double()) if d.bias is not None else 0))
            self.h = rbf(f32(d.res[:, :N].double()) + f32(h))
            if g.norm == NORM_RMS:
                self.xn = rms_iv(Iv.exact(self.h), d.nw.double().expand_as(self.h), N)
            elif g.norm == NORM_LN:
                self.xn = ln_iv(self.h, d.nw, d.nb, EPS)
        else:
            v = f32(A) + (f32(d.bias.double()) if d.bias is not None else 0)
            self.v = v.double()
            if g.epi == EPI_NONE:
                out = self.v
                if g.res:
                    out = (f32(out) + d.res).double()
                self.out = out
            else:
                self.ref, self.band = f32_epi_band(self.v, g.epi)
                if g.res:     # + res32: one more fp32 rounding
                    self.ref = self.ref + d.res.double()
                    self.band = self.band + self.ref.abs() * U


def run_case(L, g, T, d, ref, cfg, tag):
    N, K = g.N, kdim(g)
    TN, KS, st, sp = cfg
    key = MODE_NAME[g.mode] + (f" {EPI_NAME[g.epi]}" if g.epi else "")
    if g.mode in (BF16, SWIGLU):
        cols = g.inter if g.mode == SWIGLU else N
        ldc = g.ldc or cols
        if g.res == "inplace":
            Cb = torch.cat([d.res.clone(), sentinel((2, ldc))])
            Cb[:T, cols:] = sentinel((T, ldc - cols))
        else:
            Cb = sentinel((T + 2, ldc))
        resid = Cb if g.res == "inplace" else (d.res if g.res == "sep" else None)
        if resid is not None and g.res == "sep":
            resid = d.res.clone()
            resid[:, cols:] = float("nan")
        ncheck(L.b200_gemm_wt(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), d.bias.data_ptr() if d.bias is not None
                              else None, resid.data_ptr() if resid is not None else None, ldc, Cb.data_ptr(), ldc, None,
                              T, N, K, g.epi, g.mode, g.inter, _cfg(cfg), 0, None), tag)
        torch.cuda.synchronize()
        _note(key + (" + residual" if g.res else ""), check(Cb[:T, :cols], ref.iv, tag))
        keep_sentinel(Cb, (slice(0, T), slice(0, cols)), tag)
    elif g.mode == PARTIAL:
        P = torch.full((sp * T * N + 64,), float("nan"), dtype=torch.float32, device="cuda")
        ncheck(L.b200_gemm_wt(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), None, None, 0, None, 0, P.data_ptr(), T,
                              N, K, EPI_NONE, PARTIAL, 0, _cfg(cfg), 0, None), tag)
        torch.cuda.synchronize()
        assert bool(torch.isnan(P[sp * T * N:]).all()), f"{tag}: wrote past its partial tiles"
        kbps = cdiv(cdiv(K, WT_BK), sp) * WT_BK
        Pv = P[:sp * T * N].view(sp, T, N)
        for s in range(sp):
            want = ref.A if sp == 1 else acc64(ref.d, s * kbps, min(K, (s + 1) * kbps))
            if not torch.equal(Pv[s].double(), want):
                bad = int((Pv[s].double() != want).sum())
                raise AssertionError(f"{tag}: split {s} of {sp}: {bad} of {T * N} partial sums differ from the exact "
                                     f"sum over k-blocks [{s * kbps // 64}, {min(K, (s + 1) * kbps) // 64})")
        _note("PARTIAL tiles", (0, 0.0))
        if N > FIN_N_MAX:
            return
        h = torch.cat([d.res.clone(), sentinel((1, N))])
        xn = sentinel((T + 1, N))
        ncheck(L.b200_finish_rows(P.data_ptr(), sp, d.bias.data_ptr() if d.bias is not None else None, h.data_ptr(), N,
                                  h.data_ptr(), N, g.norm, d.nw.data_ptr() if d.nw is not None else None,
                                  d.nb.data_ptr() if d.nb is not None else None, EPS,
                                  xn.data_ptr() if g.norm != NORM_NONE else None, N, T, N, None), tag + " finish_rows")
        torch.cuda.synchronize()
        _note("finish_rows h", exact(h[:T], ref.h, tag + " finish_rows h"))
        keep_sentinel(h, (slice(0, T),), tag + " finish_rows h")
        if g.norm != NORM_NONE:
            _note(f"finish_rows {'RMS' if g.norm == NORM_RMS else 'LN'}", check(xn[:T], ref.xn, tag + " finish_rows xn"))
            keep_sentinel(xn, (slice(0, T),), tag + " finish_rows xn")
        else:
            keep_sentinel(xn, (slice(0, 0),), tag + " finish_rows xn")
    else:
        ext = None
        if g.mode == F32:
            out = torch.full((T + 1, N + 4), float("nan"), dtype=torch.float32, device="cuda")
            ldo = N + 4
            if g.res:
                out[:T, :N] = d.res
            ncheck(L.b200_gemm_wt_f32(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), d.W.stride(0),
                                      d.bias.data_ptr() if d.bias is not None else None,
                                      out.data_ptr() if g.res else None, ldo, out.data_ptr(), ldo, None, 0, 0, T, N,
                                      g.K, g.n_parts, g.epi, F32, _cfg(cfg), None), tag)
            torch.cuda.synchronize()
            got = out[:T, :N]
            if g.epi == EPI_NONE:
                _note(key + (" + res32" if g.res else ""), check_f32(got, ref.out, torch.zeros_like(ref.out), tag))
            else:
                _note(key, check_f32(got, ref.ref, ref.band, tag))
            keep_sentinel(out, (slice(0, T), slice(0, N)), tag)
        else:
            n_pad = pad64(N)
            sp_buf = sentinel((T + 1, 2 * n_pad + 8))
            ncheck(L.b200_gemm_wt_f32(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), d.W.stride(0),
                                      d.bias.data_ptr() if d.bias is not None else None, None, 0, None, 0,
                                      sp_buf.data_ptr(), sp_buf.stride(0), n_pad, T, N, g.K, g.n_parts, g.epi, SPLIT,
                                      _cfg(cfg), None), tag)
            torch.cuda.synchronize()
            hi, lo = sp_buf[:T, :N].double(), sp_buf[:T, n_pad:n_pad + N].double()
            if g.epi == EPI_NONE:
                v = f32(ref.v)
                whi = rbf(v)
                _note(key + " hi", exact(sp_buf[:T, :N], whi, tag + " hi"))
                _note(key + " lo", exact(sp_buf[:T, n_pad:n_pad + N], rbf(v - whi.float()), tag + " lo"))
            else:
                # hi = bf16(v'), lo = bf16(v' - hi) for an fp32 v' within the band: v' - hi is exact in fp32, so
                # v' lies within half an ulp of lo from hi + lo, and hi must be v's rounding
                # (the wider of the two spacings around lo: at a power of two they differ)
                ulp_lo = torch.maximum((bf16_step(lo, torch.ones_like(lo)) - lo).abs(),
                                       (bf16_step(lo, -torch.ones_like(lo)) - lo).abs())
                _note(key, check_f32(hi + lo, ref.ref, ref.band + ulp_lo / 2 * 1.0001, tag + " hi + lo"))
                vlo, vhi = hi + lo - ulp_lo / 2, hi + lo + ulp_lo / 2
                ok = (bf16_round(vlo) == hi) | (bf16_round(vhi) == hi) | ((vlo <= hi) & (hi <= vhi))
                assert bool(ok.all()), f"{tag}: hi is not the rounding of hi + lo"
            keep_sentinel(sp_buf, (slice(0, T), [*range(N), *range(n_pad, n_pad + N)]), tag)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


ROWS = [rid for rid, _, _ in table()]


@pytest.mark.gpu
def test_exactness_probe():
    """the bf16 wgmma keeps every bit of fp32 sums below 2^24 u: K = 64 and K = 18944 (the qwen2vl-7b down) with
    all-positive and mixed-sign integer operands, every configuration of the shape, against the float64 sums"""
    L = lib()
    for K, sign in ((64, False), (64, True), (18944, False), (18944, True)):
        g = Gemm("probe", BF16, 256, K)
        T = 48
        gen = torch.Generator(device="cuda").manual_seed(K + sign)
        lo = -8 if sign else 1
        Xi = torch.randint(lo, 9, (T, K), device="cuda", generator=gen).double()
        Wi = torch.randint(lo, 9, (256, K), device="cuda", generator=gen).double()
        bound = float((Xi.abs() @ Wi.abs().T).max())
        assert bound < 2 ** 24
        P = torch.full((T * 256,), float("nan"), dtype=torch.float32, device="cuda")
        want = Xi @ Wi.T
        X, W = Xi.to(torch.bfloat16), Wi.to(torch.bfloat16)
        for cfg in [(48, 1, 6, 1), (48, 2, 5, 1), (16, 1, 6, 1), (64, 4, 2, 1)]:
            ncheck(L.b200_gemm_wt(X.data_ptr(), K, W.data_ptr(), None, None, 0, None, 0, P.data_ptr(), T, 256, K, 0,
                                  PARTIAL, 0, _cfg(cfg), 0, None), "probe")
            torch.cuda.synchronize()
            got = P.view(T, 256).double()
            nd = int((got != want).sum())
            print(f"probe K={K} {'mixed' if sign else 'positive'} cfg={cfg}: sums up to {bound:.0f} u, {nd} of "
                  f"{T * 256} differ from float64, worst {float((got - want).abs().max()):.3g} u")
            assert nd == 0, f"K={K}: the wgmma fp32 sums are not exact below 2^24 u"


@pytest.mark.gpu
@pytest.mark.parametrize("rid", ROWS)
def test_gemm_wt_row(rid):
    """every planned configuration of one shape at its T edges, element by element against the float64 reference"""
    L = lib()
    sms = _sms()
    g, p = next((g, p) for r, g, p in full_table(sms) if r == rid)
    n = 0
    for T, cfgs in p.items():
        d = make(g, T, zlib.crc32(f"{rid} {T}".encode()))
        ref = Ref(g, T, d)
        for cfg in cfgs:
            run_case(L, g, T, d, ref, cfg, f"{rid} T={T} cfg={cfg}")
            n += 1
        del d, ref
    torch.cuda.empty_cache()
    print(f"{rid}: {n} launches at {sms} SMs; per mode: " +
          "; ".join(f"{k}: {v[0]} differ, worst ratio {v[1]:.3g}" for k, v in sorted(STATS.items())))


def _tune_off():
    return os.environ.get("B200_WT_TUNE", "") not in ("",) and int(os.environ["B200_WT_TUNE"]) == 0


@pytest.mark.gpu
def test_tuned_choice_and_bucket_reuse():
    """the measured choice: the first call of a class runs a member of its candidate list, a second call at another T
    of the bucket the cached choice clamped and re-fitted; both exact.  Each (N, K) is used by no other test, so the
    class really tunes"""
    if _tune_off():
        pytest.skip("B200_WT_TUNE=0: the cost model decides, nothing is measured")
    L = lib()
    sms = _sms()
    st = torch.cuda.Stream()
    for g, T1, T2, pbytes in ((Gemm("tuned bf16", BF16, 776, 1096, bias=True), 120, 70, 0),
                              (Gemm("tuned partial", PARTIAL, 1160, 5128, bias=True, norm=NORM_RMS,
                                    pbytes=24 << 20, split_ok=True), 128, 66, 24 << 20),
                              (Gemm("tuned swiglu", SWIGLU, 2 * 712, 904, inter=712), 100, 65, 0)):
        for T in (T1, T2):
            d = make(g, T, T)
            ref = Ref(g, T, d)
            out = (C.c_int * 4)()
            cols = g.inter if g.mode == SWIGLU else g.N
            Cb = sentinel((T + 1, cols))
            P = torch.full((max(pbytes // 4, 1) + 64,), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            ncheck(L.b200_gemm_wt_tuned(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(),
                                        d.bias.data_ptr() if d.bias is not None and g.mode == BF16 else None, None, 0,
                                        Cb.data_ptr() if g.mode != PARTIAL else None, cols,
                                        P.data_ptr() if g.mode == PARTIAL else None, pbytes, T, g.N, g.K, g.epi,
                                        g.mode, g.inter, int(g.split_ok), sms, out, st.cuda_stream), g.name)
            torch.cuda.synchronize()
            cfg = tuple(out)
            if T == T1:
                cand = candidates(T, g.N, g.K, g.mode, g.inter, g.split_ok, sms, pbytes)
                assert cfg in cand, f"{g.name}: ran {cfg}, not one of its candidates {cand}"
                first = cfg
            else:
                want = reuse(first, T, g.N, g.K, g.mode, pbytes)
                assert cfg == want, f"{g.name}: T={T} ran {cfg}, the cached {first} reused is {want}"
            print(f"{g.name} T={T}: ran {cfg}")
            tag = f"{g.name} T={T} tuned {cfg}"
            if g.mode == PARTIAL:
                run_case(L, g, T, d, ref, cfg, tag + " (replayed explicitly)")
                sp = cfg[3]
                kbps = cdiv(cdiv(g.K, WT_BK), sp) * WT_BK
                Pv = P[:sp * T * g.N].view(sp, T, g.N)
                for s in range(sp):
                    assert torch.equal(Pv[s].double(), acc64(d, s * kbps, min(g.K, (s + 1) * kbps))), tag
            else:
                check(Cb[:T], ref.iv, tag)
                keep_sentinel(Cb, (slice(0, T),), tag)


@pytest.mark.gpu
def test_tuned_in_place_residuals():
    """on the call that tunes, an in-place bf16 residual (C == residual) and an in-place fp32 res32 are added exactly
    once: the timing launches must not touch the caller's output"""
    if _tune_off():
        pytest.skip("B200_WT_TUNE=0: the cost model decides, nothing is measured")
    L = lib()
    sms = _sms()
    st = torch.cuda.Stream()
    g = Gemm("tuned in place", BF16, 1048, 1224, bias=True, res="inplace")
    T = 200
    d = make(g, T, 5)
    ref = Ref(g, T, d)
    Cb = d.res.clone()
    out = (C.c_int * 4)()
    torch.cuda.synchronize()
    ncheck(L.b200_gemm_wt_tuned(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), d.bias.data_ptr(), Cb.data_ptr(),
                                g.N, Cb.data_ptr(), g.N, None, 0, T, g.N, g.K, 0, BF16, 0, 0, sms, out, st.cuda_stream),
           g.name)
    torch.cuda.synchronize()
    check(Cb, ref.iv, f"{g.name} bf16 C == residual, tuned {tuple(out)}")
    g = Gemm("tuned res32", F32, 1096, 1176, bias=True, res="res32")
    d = make(g, T, 6)
    ref = Ref(g, T, d)
    o = d.res.clone()
    torch.cuda.synchronize()
    ncheck(L.b200_gemm_wt_f32(d.X.data_ptr(), d.X.stride(0), d.W.data_ptr(), d.W.stride(0), d.bias.data_ptr(),
                              o.data_ptr(), g.N, o.data_ptr(), g.N, None, 0, 0, T, g.N, g.K, 2, 0, F32, None,
                              st.cuda_stream),
           g.name)
    torch.cuda.synchronize()
    check_f32(o, ref.out, torch.zeros_like(ref.out), f"{g.name} fp32 C32 == res32, tuned")
