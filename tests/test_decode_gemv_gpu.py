"""Every weight-streaming GEMV stage of the batch-1 decode step, on k_mega and on the per-phase kernels, against a
float64 reference of the same operation, element by element.

The stages: qkv with RMSNorm and the rotary (and the q/k norm of Qwen3-VL), o_proj plus residual, gate/up with
SwiGLU, down plus residual, and the head with its logsumexp, logprobs and argmax.  Each case runs a ONE-LAYER engine
at a family's real hidden / inter / vocab, through its normal launch code, with weights that isolate one stage:

  qkv        the fed token's embedding row is +-1 (its RMS statistic is exact, so the normalised input is exactly
             +-ln1); random wqkv and bias.  Observed: the K and V rows the step appends at ctx (0, 37 and the
             last pool position) and the q heads (debug_buffer "q"), at rotary positions up to 10^5; the rest of the
             pool unchanged bit for bit.
  o_proj     ctx = 0, so the attention output is the V row exactly (read back from the pool); random wo, zero MLP,
             head [I; 0] behind a unit final norm: logits[:hidden] = rms_norm(bf16(h + bf16(Wo . v))).
  gate/up    zero qkv (the attention output is 0, h1 = h); random ln2 and wgu: act = swiglu of exact inputs.
  down       the same step, random wd: logits[:hidden] = rms_norm(bf16(h + bf16(Wd . act))), act read back.
  head       a zero layer (h stays the +-1 embedding row), random final norm and head, tied and untied: logits,
             the logsumexp, every logprob, the token (planted ties across head CTAs, inside a head tile, across
             sampler warps and across sampler CTAs), the token log and the next step's h; also through a prefill
             call, whose last row runs the same head and sampler.

THE BAR.  Every stage sees exactly known inputs, so the only legitimate difference from the float64 reference is
fp32 summation order.  Each rounding point of the kernel gets the interval of bf16 values that an fp32 result within
the error band of the exact value can round to: one value, or the two values on either side of a rounding boundary
inside the band (more only where cancellation leaves the exact value far smaller than the band).  Where a rounding
feeds SwiGLU, a residual add, an RMSNorm or the rotary, the interval is carried through the kernel's next operations,
rounded at the kernel's points (`Iv`, `corners`).  An element must lie in its interval.  The bands:

  dot products   the kernels sum the exact products (fmaf) in a tree: a chain of at most CHX <= 10 FMAs per lane and
                 accumulator, 3 pairwise levels, a 5-level warp butterfly, the S <= 8 K slices in sequence and the bias:
                 at most 27 additions on any path (decode.cu k_stream, decode_mega.cu consume_phase).  For a tree of
                 depth d, |err| <= gamma(d) (sum |w_i x_i| + |b|), gamma(d) = d u / (1 - d u), u = 2^-24 (Higham,
                 Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 4.2); DOT_DEPTH is twice 27.
  RMS statistic  rs = 1 / sqrtf(ss / K + eps) with ss = sum x_i^2 in fp32 (k_stream, consume_phase and
                 common.cuh warp_head_rms, in different orders and depths up to K).  The terms are positive, so ss
                 carries a relative error of at most gamma(K - 1); ss / K, + eps, sqrtf and 1 / x are correctly
                 rounded (no fast-math): one u each, and the square root halves the relative error of its argument.
                 So rs is within delta = gamma(K + 1) / 2 + 3u of exact (first order; _BAND_SLACK covers the rest),
                 and fl(x rs) within |x rs| (delta + u).  Where the input elements are themselves intervals, ss moves
                 by at most sum max |x'^2 - x^2| over them, which is added to the relative error of ss.
  sigmoid        __fdividef(1, 1 + __expf(-g)): __expf is within (2 + 1.173 |g|) ulp, the add 1/2 ulp, __fdividef
                 2 ulp (CUDA C++ Programming Guide, intrinsic functions), so sigma is within
                 (2 + 1.173 |g|) 2^-23 + 2^-24 + 2^-22 relative.
  cosf / sinf    within 2 ulp (same guide): |c| 2^-22.

A rel-L2 bar over 152k logits does not see one wrong row; this bar does.  Each check prints its count of
band-explained differences (elements that differ from the float64-then-round reference) and the worst band ratio
next to the rel L2, a summary only.  For a dot product the ratio is the distance of the exact value from the rounding
boundary the element crossed, over the band; after a chain of roundings it is how far the element went into the
admissible side of the reference (1: its edge).

The tile geometries (rows per tile, K slices, register chunks, kernel instantiation, tiles per CTA) are restated from
the C host code below, and test_geometry_table_reaches_every_case (no GPU) checks that the geometry table reaches
every case the kernels distinguish.  The vocabularies that target a tiles-per-CTA count are derived from the SM
count, so the GPU tests build them for the device they run on."""
import itertools
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch

from _util import rl2

# ---- tiling constants and formulas of the host code ------------------------------------------------------------------
STREAM_SMEM_BUDGET = 100 * 1024     # decode.cu: the ring of one k_stream CTA
STREAM_STAGE_MAX = 50 * 1024        # decode.cu stream_geometry: a tile <= 50 KB (and <= STREAM_SMEM_BUDGET / 2)
MEGA_STAGE = 48 * 1024              # mega_common.cuh: one k_mega ring stage
MEGA_SMEM = 227 * 1024 - 2048       # decode_mega.cu mega_fill / launch_k_mega: dynamic shared memory
MEGA_ATT_G, ATT_UN = 4, 8           # mega_common.cuh: q heads per attention CTA, key ranges per (kv head, group)
MAX_CHX = 10                        # the largest k_stream / k_mega register-chunk instantiation
STREAM_INST = (2, 6, 10)            # decode.cu launch_stream: k_stream<MODE, 2 | 6 | 10>
MEGA_INST = ((2, 2), (6, 10), (8, 10), (10, 10))   # decode_mega.cu mega_launch: k_mega<CHH, CHI>, first that fits
CAP = 256                           # KV pool capacity of every rig
EPS = 1e-6


def cdiv(a, b):
    return -(-a // b)


def chunks(K, S):
    """16-byte activation chunks per lane of one K slice: decode.cu launch_stream `chx`, decode_mega.cu mega_chx"""
    return cdiv(cdiv(K >> 3, S), 32)


def tile_rows(K, pair, units, stage_max):
    """R, rows (QKV / GATEUP: row pairs) per tile: decode.cu stream_geometry (stage_max 50 KB) and decode_mega.cu
    mega_geometry (48 KB).  None where the host refuses the width."""
    unit = K * 2 * (2 if pair else 1)
    R = 8
    while R > 1 and (R * unit > stage_max or R > units):
        R >>= 1
    while R > 1 and chunks(K, 8 // R) > MAX_CHX:
        R >>= 1
    return R if R * unit <= stage_max else None


def stream_inst(chx):
    """decode.cu launch_stream: the k_stream<MODE, CHX> instantiation"""
    return next((c for c in STREAM_INST if chx <= c), None)


class Phase(NamedTuple):
    name: str      # qkv, o_proj, gateup, down, head
    mode: str      # the kernel mode: QKV, ORES, DRES, GATEUP, HEAD
    K: int
    N: int         # output rows (QKV: row pairs of all head slots)
    R: int
    S: int
    chx: int
    tiles: int
    grid: int      # CTAs that take tiles

    def ragged(self):
        return self.mode != "QKV" and self.N % self.R != 0

    def counts(self):
        """the tiles per CTA that occur (CTA b takes tiles b, b + grid, ...)"""
        return {self.tiles // self.grid, cdiv(self.tiles, self.grid)} if self.tiles >= self.grid else {0, 1}


class Row(NamedTuple):
    name: str
    hidden: int
    inter: int
    vocab: int
    nh: int
    nkv: int
    hd: int
    qk: bool       # Qwen3-VL q / k RMSNorm
    tied: bool     # head = embedding


def phases(row, path, sms):
    """{name: Phase} of the step on `path` ("stream": the per-phase kernels, "mega": k_mega), or None where the host
    refuses a width.  decode.cu launch_qkv / launch_res / launch_gateup / launch_head / head_ctas and decode_mega.cu
    mega_fill."""
    H, I, V, nh, nkv, hd = row.hidden, row.inter, row.vocab, row.nh, row.nkv, row.hd
    stage = STREAM_STAGE_MAX if path == "stream" else MEGA_STAGE
    half = hd // 2
    out = {}
    for name, K, N, pair, units in (("qkv", H, (nh + 2 * nkv) * half, True, half), ("o_proj", nh * hd, H, False, H),
                                    ("gateup", H, I, True, I), ("down", I, H, False, H), ("head", H, V, False, V)):
        R = tile_rows(K, pair, units, stage)
        if R is None or (name == "qkv" and half % R):
            return None
        S = 8 // R
        tiles = cdiv(N, R)
        if path == "mega":
            grid = sms
        else:
            grid = min(tiles, 2 * sms if name == "head" else sms)
        if name == "qkv":
            mode = "QKV"
        elif name in ("o_proj", "down"):
            # per-phase: launch_res picks ORES / DRES by S == 1; k_mega: the o_proj phase by S == 1, the down phase
            # always consume_phase<PH_DRES, CHI>
            mode = "ORES" if S == 1 and not (path == "mega" and name == "down") else "DRES"
        else:
            mode = name.upper()
        out[name] = Phase(name, mode, K, N, R, S, chunks(K, S), tiles, grid)
    if path == "stream" and any(stream_inst(p.chx) is None for p in out.values()):
        return None
    return out


def mega_inst(ph):
    """decode_mega.cu mega_launch: CHH over qkv, o_proj, gateup and head, CHI of down"""
    chh = max(ph[n].chx for n in ("qkv", "o_proj", "gateup", "head"))
    chi = ph["down"].chx
    return next((m for m in MEGA_INST if chh <= m[0] and chi <= m[1]), None)


def mega_attn_ctas(row):
    """decode_mega.cu mega_fill: attention CTAs (must be <= the SM count)"""
    G = row.nh // row.nkv
    hs = cdiv(G, MEGA_ATT_G)
    if hs == 1 and G % 2 == 0 and G >= 4:
        hs = 2
    return row.nkv * hs * ATT_UN


def mega_ring_stages(row, cap=CAP):
    """decode_mega.cu mega_fill / mega_attn_scratch / mega_spare_bytes: weight ring stages (>= 2 to run)"""
    att = (MEGA_ATT_G * cdiv(cap, ATT_UN) + 8 * MEGA_ATT_G * row.hd + (MEGA_ATT_G + 2) * row.hd) * 4
    xs = max(row.inter, row.hidden, row.nh * row.hd) * 2
    scratch = cdiv(max(att, xs), 128) * 128
    spare = cdiv(row.hidden * 2, 128) * 128
    return (MEGA_SMEM - scratch - spare) // MEGA_STAGE


def mega_accepts(row, sms, cap=CAP):
    """whether the engine runs this row's step on k_mega (engine.cu: otherwise it falls back to the per-phase kernels)"""
    ph = phases(row, "mega", sms)
    return (ph is not None and mega_inst(ph) is not None and mega_attn_ctas(row) <= sms and row.hd in (64, 128)
            and mega_ring_stages(row, cap) >= 2)


def _tiles_for(m, sms, mult):
    """the smallest tile count, a multiple of mult, that gives CTA 0 of an sms-CTA grid m tiles and the last CTA m - 1"""
    t = (m - 1) * sms + 1
    return t + (-t) % mult


def rows(sms):
    """the geometry table (hidden, inter, vocab, heads, kv heads, head_dim, q/k norm, tied); the last rows size their
    vocabulary / inter from the SM count"""
    out = [
        Row("qwen2vl-2b", 1536, 8960, 151936, 12, 2, 128, False, True),
        Row("qwen2vl-7b", 3584, 18944, 152064, 28, 4, 128, False, False),
        Row("qwen3vl-2b", 2048, 6144, 151936, 16, 8, 128, True, True),
        Row("qwen3vl-4b", 2560, 9728, 151936, 32, 8, 128, True, True),
        Row("mistral-7b", 4096, 14336, 32003, 32, 8, 128, False, False),     # Idefics2: odd vocab
        Row("llama-7b", 4096, 11008, 32064, 32, 32, 128, False, False),      # LLaVA: 256 attention CTAs
        Row("smolvlm-256m", 576, 1536, 49280, 9, 3, 64, False, True),
        Row("smolvlm-2.2b", 2048, 8192, 49280, 32, 32, 64, False, True),
        # every phase within 2 chunks (k_mega<2,2>), a head of fewer tiles than CTAs, odd vocab
        Row("tiny", 256, 512, 8 * (sms // 2) + 3, 4, 2, 64, False, False),
        # o_proj of 5120: 4 rows x 2 slices of 10 chunks (k_mega<10,10> at any SM count)
        Row("w5120", 5120, 13824, 32000, 40, 4, 128, False, False),
        # per-phase: qkv and gate/up of 2 row pairs x 4 slices of 7 chunks, exactly one 50 KB tile (k_stream<., 10>);
        # k_mega: one row pair per tile
        Row("w6400", 6400, 6400, 6408, 32, 4, 128, False, False),
        # qkv and gate/up of one row pair per tile on both paths
        Row("w8192", 8192, 8192, 8200, 32, 4, 128, False, False),
    ]
    # k_mega's deferred epilogue flushes every 32 tiles: the head (4 rows per tile at 4096) and gate/up (2 row pairs)
    # at 32k - 1, 32k and 32k + 1 tiles per CTA; vocab = 4 T - 1 leaves a ragged last head tile
    for name, mh, mg in (("edge32a", 33, 32), ("edge32b", 32, 33), ("edge64a", 65, 64), ("edge64b", 64, 65)):
        out.append(Row(name, 4096, 2 * _tiles_for(mg, sms, 4), 4 * _tiles_for(mh, sms, 1) - 1, 32, 4, 128, False,
                       False))
    return out


def _selectable(mode):
    """the k_stream<MODE, CHX> instantiations launch_stream can select for `mode`, over every width"""
    out = set()
    for K in range(8, 65537, 8):
        pair = mode in ("QKV", "GATEUP")
        for units in ((32, 64) if mode == "QKV" else (1 << 20,)):
            R = tile_rows(K, pair, units, STREAM_STAGE_MAX)
            if R is None or (mode == "ORES") != (R == 8) or (mode == "QKV" and units % R):
                continue
            inst = stream_inst(chunks(K, 8 // R))
            if inst is not None:
                out.add(inst)
    return out


def reached(sms):
    """what the table reaches at this SM count, as {case: bool}"""
    table = rows(sms)
    got = {}
    mega_rows = [r for r in table if mega_accepts(r, sms)]
    for path in ("stream", "mega"):
        pr = table if path == "stream" else mega_rows
        ph = [phases(r, path, sms) for r in pr]
        assert all(p is not None for p in ph), f"{path}: a table row is refused by the host"
        for R in (8, 4, 2, 1):
            got[f"{path}: QKV R={R}"] = any(p["qkv"].R == R for p in ph)
            got[f"{path}: GATEUP R={R}"] = any(p["gateup"].R == R for p in ph)
            got[f"{path}: residual R={R}"] = any(p[n].R == R for p in ph for n in ("o_proj", "down"))
        for m in ("ORES", "DRES"):
            got[f"{path}: {m}"] = any(p[n].mode == m for p in ph for n in ("o_proj", "down"))
        got[f"{path}: ragged last head tile"] = any(p["head"].ragged() for p in ph)
        got[f"{path}: odd vocab"] = any(r.vocab % 2 for r in pr)
        got[f"{path}: tied and untied head"] = {r.tied for r in pr} == {True, False}
        got[f"{path}: q/k norm"] = any(r.qk for r in pr)
        got[f"{path}: head_dim 64 and 128"] = {r.hd for r in pr} == {64, 128}
    for mode in ("QKV", "ORES", "DRES", "GATEUP", "HEAD"):
        used = {stream_inst(p.chx) for r in table for p in phases(r, "stream", sms).values() if p.mode == mode}
        for c in sorted(_selectable(mode)):
            got[f"stream: k_stream<{mode}, {c}>"] = c in used
    insts = {mega_inst(phases(r, "mega", sms)) for r in mega_rows}
    for m in MEGA_INST:
        got[f"mega: k_mega<{m[0]}, {m[1]}>"] = m in insts
    mph = [phases(r, "mega", sms) for r in mega_rows]
    got["mega: head with fewer tiles than CTAs"] = any(p["head"].tiles < p["head"].grid for p in mph)
    for k in (1, 2):
        for n in (32 * k - 1, 32 * k, 32 * k + 1):
            got[f"mega: head at {n} tiles per CTA"] = any(n in p["head"].counts() for p in mph)
            got[f"mega: gateup at {n} tiles per CTA"] = any(n in p["gateup"].counts() for p in mph)
    return got


@pytest.mark.parametrize("sms", [132, 114])
def test_geometry_table_reaches_every_case(sms):
    """the table reaches every tile geometry, instantiation and tiles-per-CTA edge the kernels distinguish, at the
    SM counts of the H100 SXM (132) and PCIe (114)"""
    got = reached(sms)
    for case, ok in got.items():
        print(f"{sms} SMs  {'reached' if ok else 'MISSED '}  {case}")
    assert all(got.values()), [c for c, ok in got.items() if not ok]
    # a ragged last tile can only occur in the head: hidden and inter are multiples of 8 (b200_engine_create) and
    # R divides 8, so o_proj, gate/up and down always end on a full tile
    for r in rows(sms):
        assert r.hidden % 8 == 0 and r.inter % 8 == 0
        for path in ("stream", "mega"):
            assert not any(p.ragged() for p in phases(r, path, sms).values() if p.name != "head")


def test_geometry_of_the_issue_table():
    """spot values of the formulas, computed by hand from the C code"""
    t = {r.name: r for r in rows(132)}
    for path in ("stream", "mega"):
        p = phases(t["qwen2vl-7b"], path, 132)
        assert (p["qkv"].R, p["qkv"].S, p["qkv"].chx) == (2, 4, 4)
        assert (p["o_proj"].R, p["o_proj"].S, p["o_proj"].chx, p["o_proj"].mode) == (4, 2, 7, "DRES")
        assert (p["down"].R, p["down"].S, p["down"].chx) == (1, 8, 10)
        assert phases(t["mistral-7b"], path, 132)["down"][4:7] == (1, 8, 7)
        assert phases(t["qwen3vl-4b"], path, 132)["head"].chx == 10
        assert phases(t["smolvlm-256m"], path, 132)["o_proj"].chx == 3
    assert mega_inst(phases(t["qwen2vl-7b"], "mega", 132)) == (8, 10)
    assert mega_inst(phases(t["qwen3vl-4b"], "mega", 132)) == (10, 10)
    assert mega_inst(phases(t["tiny"], "mega", 132)) == (2, 2)
    assert stream_inst(phases(t["smolvlm-256m"], "stream", 132)["o_proj"].chx) == 6
    assert not mega_accepts(t["llama-7b"], 132) and not mega_accepts(t["smolvlm-2.2b"], 132)
    assert mega_accepts(t["qwen2vl-2b"], 132) and mega_accepts(t["w5120"], 114)


# ---- admissible intervals: the results a chain of fp32 operations and roundings may give ------------------------------
U = 2.0 ** -24
_BAND_SLACK = 1.01
DOT_DEPTH = 2 * (MAX_CHX + 3 + 5 + 8 + 1)


def gamma(n):
    return n * U / (1 - n * U)


def bf16_round(s):
    """float64 -> the float64 value of its round-to-nearest-even bf16 (no double rounding through fp32)"""
    _, e = torch.frexp(s)
    q = torch.ldexp(torch.ones_like(s), torch.clamp(e, min=-125) - 8)   # bf16 spacing in [2^(e-1), 2^e)
    return torch.round(s / q) * q


def bf16_step(v, d):
    """the bf16 neighbour of bf16 values v in direction d (+-1)"""
    t = v.float().view(torch.int32)
    away = (torch.sign(v) == d) | (v == 0)
    n = torch.where(away, t + 65536, t - 65536).view(torch.float32).double()
    return torch.where(v == 0, d * 2.0 ** -133, n)


def rbf(x):
    """fp32 -> bf16 -> float64 (the kernels' rbf / f2bf)"""
    return x.float().to(torch.bfloat16).double()


class Iv(NamedTuple):
    """every value the kernel may produce lies in [lo, hi] (bf16 values, as float64); ref: the float64 computation
    rounded at the kernel's rounding points"""
    lo: torch.Tensor
    hi: torch.Tensor
    ref: torch.Tensor
    s: torch.Tensor = None      # a rounding of a dot product: the exact value and its band
    band: torch.Tensor = None

    @staticmethod
    def exact(x):
        x = x.double()
        return Iv(x, x, x)

    def sel(self, f):
        """f (a view or an index) applied to every field"""
        return Iv(*(None if t is None else f(t) for t in self))


def rounded(s, band):
    """bf16 rounding of the fp32 computation of exact values s, known to within `band`"""
    band = band * _BAND_SLACK
    return Iv(bf16_round(s - band), bf16_round(s + band), bf16_round(s), s, band)


def corners(f, *ivs):
    """f of intervals, for f monotone in each argument when the others are fixed (sums, products, monotone
    roundings): its extremes lie on the corners of the box"""
    vals = torch.stack([f(*c) for c in itertools.product(*[(a.lo, a.hi) for a in ivs])])
    return Iv(vals.amin(0), vals.amax(0), f(*[a.ref for a in ivs]))


def check(got, iv, name):
    """every element of got lies in its admissible interval; prints the count of elements that differ from the
    float64-then-round reference and the worst band ratio (how far into the admissible side an element went)"""
    got = got.double().reshape(iv.ref.shape)
    ok = (got >= iv.lo) & (got <= iv.hi)
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        lines = [f"  {tuple(i)}: got {got[tuple(i)].item():.6g}, reference {iv.ref[tuple(i)].item():.6g}, admissible "
                 f"[{iv.lo[tuple(i)].item():.6g}, {iv.hi[tuple(i)].item():.6g}]" for i in bad[:8].tolist()]
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements outside the bar\n" + "\n".join(lines))
    diff = got != iv.ref
    if iv.s is not None:
        # the farthest rounding boundary the element crossed, its distance from the exact value over the band
        nb = bf16_step(got, torch.sign(iv.ref - got))
        ratio = (iv.s - (got + nb) / 2).abs() / iv.band.clamp_min(1e-300)
    else:
        # after a chain: how far into the admissible side of the reference the element went (1: its edge)
        side = torch.where(got > iv.ref, iv.hi - iv.ref, iv.ref - iv.lo)
        ratio = (got - iv.ref).abs() / side.clamp_min(1e-300)
    ratio = torch.where(diff, ratio, torch.zeros_like(ratio))
    worst = ratio.max().item() if ratio.numel() else 0.0
    e = rl2(got.float().cpu(), iv.ref.float().cpu())
    print(f"{name}: {int(diff.sum())} / {ok.numel()} band-explained differences, worst band ratio {worst:.3g}, "
          f"rel L2 {e:.2e}")
    return int(diff.sum()), worst


# ---- float64 references of the stages ---------------------------------------------------------------------------------
def dot64(W, x, chunk=8192):
    """W (N, K) bf16 on the device, x (K,) float64: exact sums and sum |w x| (float64; its own error K 2^-53 sum|w x|
    is far inside the fp32 band)"""
    s, a = [], []
    for i in range(0, W.shape[0], chunk):
        w = W[i:i + chunk].double()
        s.append(w @ x)
        a.append(w.abs() @ x.abs())
    return torch.cat(s), torch.cat(a)


def gemv_iv(W, x, bias=None, depth=DOT_DEPTH):
    """bf16(fp32(W . x + b)) for a summation tree of the given depth: within gamma(depth) (sum |w x| + |b|)"""
    s, a = dot64(W, x)
    if bias is not None:
        b = bias.double()
        s, a = s + b, a + b.abs()
    return rounded(s, gamma(depth) * a)


def rms_iv(iv, w, K, eps=EPS):
    """bf16(bf16(fl32(x rs)) w) over the admissible x, with rs = 1 / sqrtf(ss / K + eps) within its band (the
    RMSNorm of every NORM phase and of warp_head_rms; the last dim is the normalised vector)"""
    x = iv.ref
    ss = (x * x).sum(-1, keepdim=True)
    moved = torch.maximum((iv.lo ** 2 - x * x).abs(), (iv.hi ** 2 - x * x).abs()).sum(-1, keepdim=True)
    rs = 1.0 / torch.sqrt(ss / K + eps)
    delta = (gamma(K + 1) / 2 + 3 * U + moved / (2 * ss.clamp_min(1e-300))) * _BAND_SLACK
    rsi = Iv(rs * (1 - delta), rs * (1 + delta), rs)
    y = corners(lambda a, r: a * r, iv, rsi)
    y = Iv(rbf(y.lo - y.lo.abs() * U), rbf(y.hi + y.hi.abs() * U), rbf(y.ref))    # the fp32 product, then bf16
    return corners(lambda a, b: rbf(a.float() * b.float()), y, Iv.exact(w))


def residual_iv(h, iv):
    """bf16(h + r) over the admissible r (ORES / DRES epilogue: rbf(h + rbf(acc)))"""
    return corners(lambda a, b: rbf(a.float() + b.float()), Iv.exact(h), iv)


def rope_iv(iv, pos, inv_freq):
    """rotate_half at one position, three roundings (decode.cu k_stream QKV, common.cuh warp_head_rope), with
    ang = fp32(pos * inv_freq[j]) and cosf / sinf within 2 ulp"""
    ang = (torch.tensor(float(pos), dtype=torch.float32) * inv_freq.float().cpu()).double().to(iv.ref.device)
    c, s = torch.cos(ang), torch.sin(ang)
    ci, si = rounded(c, c.abs() * 2.0 ** -22), rounded(s, s.abs() * 2.0 ** -22)
    h = iv.ref.shape[-1] // 2
    y1, y2 = iv.sel(lambda t: t[..., :h]), iv.sel(lambda t: t[..., h:])
    f = lambda a, b: rbf(a.float() * b.float())
    o1 = corners(lambda a, b, co, sn: rbf(f(a, co).float() + f(-b, sn).float()), y1, y2, ci, si)
    o2 = corners(lambda a, b, co, sn: rbf(f(b, co).float() + f(a, sn).float()), y1, y2, ci, si)
    return Iv(*(torch.cat([a, b], -1) for a, b in zip(o1[:3], o2[:3])))


def sigmoid_band(g):
    return (2 + 1.173 * g.abs()) * 2.0 ** -23 + 2.0 ** -24 + 2.0 ** -22


def swiglu_iv(g, u):
    """swiglu_bf (common.cuh): s = rbf(g rbf(sigmoid(g))), act = rbf(s u), the sigmoid from __expf / __fdividef"""
    lo, hi = torch.sigmoid(g.lo), torch.sigmoid(g.hi)
    sg = Iv(bf16_round(lo * (1 - sigmoid_band(g.lo) * _BAND_SLACK)),
            bf16_round(hi * (1 + sigmoid_band(g.hi) * _BAND_SLACK)), bf16_round(torch.sigmoid(g.ref)))
    mul = lambda a, b: rbf(a.float() * b.float())
    return corners(mul, corners(mul, g, sg), u)


def lse_check(logits, logprobs, name):
    """the kernel's bf16 lse is within one bf16 ulp of the float64 logsumexp of its own logits, and every logprob is
    bf16(fp32(logit - lse)) exactly; returns that lse"""
    want = torch.logsumexp(logits.double(), 0).reshape(1).cpu()
    c0 = bf16_round(want)
    cands = (c0, bf16_step(c0, -torch.ones(1, dtype=torch.float64)), bf16_step(c0, torch.ones(1, dtype=torch.float64)))
    for lam in cands:
        lp = rbf(logits.float() - lam.float().to(logits.device))
        if torch.equal(lp, logprobs.double()):
            ulp = (cands[2] - cands[1]).item() / 2
            assert abs(lam.item() - want.item()) <= ulp * 1.0001, f"{name}: lse {lam.item()} vs float64 {want.item()}"
            print(f"{name}: lse {lam.item()} (float64 {want.item():.6f}), every logprob = bf16(logit - lse)")
            return lam.item()
    diff = (rbf(logits.float() - c0.float().to(logits.device)) != logprobs.double()).nonzero()
    raise AssertionError(f"{name}: no bf16 lse within one ulp of {want.item()} gives the logprobs (first differing "
                         f"indices {diff[:4].flatten().tolist()})")


def test_the_bar_on_the_host():
    """fp32 sums of a GEMV in two orders cross bf16 rounding boundaries: the bar admits every crossing (each within
    its band), the exact-rounding bar refuses them, and one element two ulps off is refused; the three-rounding
    rotary at a large position is admitted"""
    from mlx_vlm_b200.engine import _inv_freq
    g = torch.Generator().manual_seed(0)
    N, K = 8192, 4096
    W = torch.randn(N, K, generator=g).to(torch.bfloat16)
    x = torch.randn(K, generator=g).to(torch.bfloat16).double()
    iv = gemv_iv(W, x, depth=K)      # sequential sums below
    exact = gemv_iv(W, x, depth=0)
    Wf, xf = W.float(), x.float()
    for order in (range(K), reversed(range(K))):
        acc = torch.zeros(N)
        for k in order:
            acc = acc + Wf[:, k] * xf[k]
        got = acc.to(torch.bfloat16)
        crossed, worst = check(got, iv, "host GEMV, sequential fp32")
        assert crossed > 0 and 0 < worst <= 1, "no rounding boundary crossed: the case does not test the band"
        with pytest.raises(AssertionError, match=f"{crossed} of {N} elements outside the bar"):
            check(got, exact, "host GEMV against the exact rounding alone")
    bad = got.clone()
    i = int(iv.ref.abs().argmax())
    bad[i] = bf16_step(bf16_step(iv.hi[i:i + 1], torch.ones(1)), torch.ones(1)).float()[0]
    with pytest.raises(AssertionError, match=f"1 of {N} elements outside the bar"):
        check(bad, iv, "host GEMV, one element two ulps off")
    heads = rms_iv(iv.sel(lambda t: t[:256].view(2, 128)), torch.ones(2, 128, dtype=torch.float64), 128)
    inv = torch.from_numpy(_inv_freq(128, 1e6))
    y, ang = heads.ref.float(), torch.tensor(100003.0) * inv
    co, si = rbf(torch.cos(ang)).float(), rbf(torch.sin(ang)).float()
    o1 = rbf(rbf(y[:, :64] * co).float() + rbf(-y[:, 64:] * si).float())
    o2 = rbf(rbf(y[:, 64:] * co).float() + rbf(y[:, :64] * si).float())
    check(torch.cat([o1, o2], -1), rope_iv(heads, 100003, inv), "host rotary at 100003")


# ---- the one-layer engine -----------------------------------------------------------------------------------------------
class GemvRig:
    """one-layer engine of a table row; weights are reset per case"""

    def __init__(self, row):
        from mlx_vlm_b200 import _native as N
        from mlx_vlm_b200.engine import Engine, _inv_freq
        from mlx_vlm_b200.models.cache import KVPool
        from mlx_vlm_b200.models.qwen2_vl.qwen2_vl import WeightArena, weight_manifest
        self.row = r = row
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = r.hidden, 1, r.inter
        c.n_heads, c.n_kv_heads, c.head_dim = r.nh, r.nkv, r.hd
        c.vocab = r.vocab
        c.rms_eps, c.rope_theta = EPS, 1000000.0
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = r.hd // 2, 0, 0
        c.tie_embeddings = int(r.tied)
        c.external_vision = 1
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = r.hidden, 1e-5
        self.H, self.QKV = r.hidden, (r.nh + 2 * r.nkv) * r.hd
        self.eng = eng = Engine(c, torch.device("cuda", 0))
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.inv_freq = torch.from_numpy(_inv_freq(r.hd, c.rope_theta)).cuda()
        self.arena = WeightArena(weight_manifest(c), eng.device)
        self.gen = torch.Generator(device="cuda").manual_seed(sum(map(ord, r.name)))
        self.w = {name: self.arena.view(name) for name in self.arena.offsets}
        self.w["lm.head"] = self.w["lm.embed"] if r.tied else self.w["lm.head"]
        if r.qk:
            self.w["lm.0.qn"] = torch.empty(r.hd, dtype=torch.bfloat16, device="cuda")
            self.w["lm.0.kn"] = torch.empty(r.hd, dtype=torch.bfloat16, device="cuda")
        for t in self.w.values():
            t.zero_()
        for name, t in self.w.items():
            if not (r.tied and name == "lm.head"):
                eng.set_weight(name, t)
        self.pool = KVPool(1, r.nkv, r.hd, eng.device, batch=1, capacity=CAP)
        eng.bind_pool(self.pool)
        eng.set_kv_row(0)
        self.tok = r.hidden        # the fed token: its embedding row is +-1 in every case (below the [I; 0] head)
        torch.cuda.synchronize()

    # -- weights
    def randn(self, *shape, scale=1.0):
        return (torch.randn(*shape, device="cuda", generator=self.gen) * scale).to(torch.bfloat16)

    def signs(self, *shape):
        return (torch.randint(0, 2, shape, device="cuda", generator=self.gen) * 2 - 1).to(torch.bfloat16)

    def norm_w(self, n):
        """RMSNorm weights around 1"""
        return (1.0 + torch.randn(n, device="cuda", generator=self.gen) * 0.25).to(torch.bfloat16)

    def set(self, **kw):
        """set(lm__0__wo=t): copy into the bound weight lm.0.wo"""
        for name, t in kw.items():
            self.w[name.replace("__", ".")].copy_(t)
        torch.cuda.synchronize()

    def layer_zero(self):
        for n in ("lm.0.wqkv", "lm.0.bqkv", "lm.0.wo", "lm.0.wgu", "lm.0.wd"):
            self.w[n].zero_()
        for n in ("lm.0.ln1", "lm.0.ln2", "lm.norm") + (("lm.0.qn", "lm.0.kn") if self.row.qk else ()):
            self.w[n].fill_(1.0)

    def identity_head(self):
        """head [I; 0] behind a unit final norm: logits[:hidden] = rms_norm(h); the embedding rows from `hidden` on
        (the fed token's among them) are +-1"""
        H, V = self.H, self.row.vocab
        E, head = self.w["lm.embed"], self.w["lm.head"]
        if self.row.tied:     # one matrix: [I; +-1 rows]
            E[H:].copy_(self.signs(V - H, H))
        else:
            E.copy_(self.signs(V, H))
            head.zero_()
        head[:H].copy_(torch.eye(H, dtype=torch.bfloat16, device="cuda"))
        self.w["lm.norm"].fill_(1.0)

    # -- steps
    def fresh_pool(self, ctx=0):
        """NaN everywhere but positions < ctx of row 0, which hold zero keys and values"""
        self.pool.buf.fill_(float("nan"))
        self.pool.buf[0, :, 0, :, :ctx] = 0
        torch.cuda.synchronize()
        return self.pool.buf.view(torch.int16).clone()

    def decode(self, path, ctx=0, pos=0, force=None, tok=None):
        eng = self.eng
        eng.set_mega(path == "mega")
        eng.set_next(self.tok if tok is None else tok, ctx, pos)
        n0, t0 = eng.launch_count, eng.tokens_launched
        eng.decode(1, None if force is None else np.asarray([force]))
        eng.stream.synchronize()
        per_phase = 1 * (6 if self.row.qk else 5) + 2
        want = (1 if path == "mega" else per_phase) + 1       # + the state kernel of the call
        assert eng.launch_count - n0 == want, f"{path} expected, {eng.launch_count - n0} launches"
        assert eng.device_error() == 0
        return t0

    def h(self):
        return self.eng.debug_buffer("h", torch.bfloat16)

    def logits(self):
        return self.eng.logits_view().clone()

    def final_rms(self, hc):
        """logits[:hidden] of a unit final norm and the [I; 0] head"""
        return rms_iv(hc, torch.ones(self.H, device="cuda", dtype=torch.float64), self.H)


def _paths(r, sms):
    return ("mega", "stream") if mega_accepts(r, sms) else ("stream",)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _row(name):
    return next(r for r in rows(_sms()) if r.name == name)


ROW_NAMES = [r.name for r in rows(132)]
# (rotary position, ctx): the append lands at ctx, row offset (slot * cap + ctx) * hd
STEPS = ((0, 0), (1, 0), (4095, 37), (32767, 0), (100003, CAP - 1))


def _run_paths(r, fn):
    """fn(rig, path) on each path the row runs (k_mega where it fits); prints which"""
    sms = _sms()
    paths = _paths(r, sms)
    print(f"{r.name}: {' and '.join(paths)} at {sms} SMs")
    rig = GemvRig(r)
    try:
        for path in paths:
            fn(rig, path)
    finally:
        rig.eng.set_mega(1)
        del rig
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROW_NAMES)
def test_qkv_and_o_proj(name):
    """qkv (RMSNorm, bias, rotary or q/k norm + rotary, the K/V append at ctx) at rotary positions up to 10^5, then
    o_proj + residual on the appended V row"""
    r = _row(name)

    def run(rig, path):
        H, hd, nh, nkv = rig.H, r.hd, r.nh, r.nkv
        rig.layer_zero()
        rig.identity_head()
        h = rig.w["lm.embed"][rig.tok].double()
        ln1, W, b = rig.norm_w(H), rig.randn(rig.QKV, H, scale=0.05), rig.randn(rig.QKV)
        Wo = rig.randn(H, nh * hd, scale=1.0 / math.sqrt(nh * hd))
        rig.set(lm__0__ln1=ln1, lm__0__wqkv=W, lm__0__bqkv=b, lm__0__wo=Wo)
        if r.qk:
            rig.set(lm__0__qn=rig.norm_w(hd), lm__0__kn=rig.norm_w(hd))
        # the +-1 row's RMS statistic: rs rounds every element back to +-1, so the normalised input is h * ln1
        rs = 1.0 / math.sqrt(1.0 + np.float32(EPS))
        assert abs(rs - 1.0) < 2.0 ** -10
        x = h * ln1.double()
        Y = gemv_iv(W, x, b)
        Y = Y.sel(lambda t: t.view(nh + 2 * nkv, hd))
        qk = Y.sel(lambda t: t[:nh + nkv])
        if r.qk:
            qk = rms_iv(qk, torch.cat([rig.w["lm.0.qn"].double()[None].expand(nh, hd),
                                          rig.w["lm.0.kn"].double()[None].expand(nkv, hd)]), hd)
        for pos, ctx in STEPS:
            before = rig.fresh_pool(ctx)
            rig.decode(path, ctx, pos)
            tag = f"{r.name} {path} pos={pos} ctx={ctx}"
            buf = rig.pool.buf
            changed = buf.view(torch.int16) != before
            changed[0, :, 0, :, ctx] = False
            assert not bool(changed.any()), f"{tag}: the step wrote pool positions other than ctx={ctx}"
            rot = rope_iv(qk, pos, rig.inv_freq)
            q = rig.eng.debug_buffer("q", torch.bfloat16).view(nh, hd)
            check(q, rot.sel(lambda t: t[:nh]), f"{tag} qkv: q heads")
            check(buf[0, 0, 0, :, ctx], rot.sel(lambda t: t[nh:]), f"{tag} qkv: K row")
            vrow = buf[0, 1, 0, :, ctx]
            check(vrow, Y.sel(lambda t: t[nh + nkv:]), f"{tag} qkv: V row")
            if ctx == 0 and pos in (0, 32767):
                # attention over one key is its V row exactly (each q head: the row of its kv head); zero MLP;
                # logits[:H] = rms_norm(h + bf16(Wo . att))
                att = vrow.repeat_interleave(nh // nkv, 0).reshape(-1).double()
                h1 = residual_iv(h, gemv_iv(Wo, att))
                check(rig.logits()[:H], rig.final_rms(h1), f"{tag} o_proj + residual")

    _run_paths(r, run)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROW_NAMES)
def test_gateup_and_down(name):
    """gate/up with SwiGLU (debug_buffer "act"), then down + residual on the act read back"""
    r = _row(name)

    def run(rig, path):
        H, I = rig.H, r.inter
        rig.layer_zero()
        rig.identity_head()
        h = rig.w["lm.embed"][rig.tok].double()
        ln2 = rig.norm_w(H)
        Wgu = rig.randn(2 * I, H, scale=2.0 / math.sqrt(H))
        Wd = rig.randn(H, I, scale=1.0 / math.sqrt(I))
        rig.set(lm__0__ln2=ln2, lm__0__wgu=Wgu, lm__0__wd=Wd)
        x = h * ln2.double()
        G, Ug = gemv_iv(Wgu[:I], x), gemv_iv(Wgu[I:], x)
        for pos in (0, 7):
            rig.fresh_pool()
            rig.decode(path, 0, pos)
            tag = f"{r.name} {path} pos={pos}"
            act = rig.eng.debug_buffer("act", torch.bfloat16)
            check(act, swiglu_iv(G, Ug), f"{tag} gate/up")
            h2 = residual_iv(h, gemv_iv(Wd, act.double()))
            check(rig.logits()[:H], rig.final_rms(h2), f"{tag} down + residual")

    _run_paths(r, run)


def _cta_of(index, ph):
    return (index // ph.R) % ph.grid


SAMPLER_WARP, SAMPLER_CTA = 32 * 8, 256 * 8   # k_sample / mega_sample_finalize: logits per warp and per CTA pass


def _tie_cases(ph, tok):
    """pairs (i, j), i < j, of head rows planted equal and maximal.  Head GEMV tiles (they write the logits and the
    logsumexp partials): in different CTAs with the lower index in the higher-numbered CTA, in different CTAs the
    other way round, and inside one tile (one CTA when R == 1).  Sampler (the packed argmax, 8 logits per thread):
    in two warps of one CTA, so that the block's shared atomicMax decides, and in two CTAs, so that the global
    atomicMax decides (one CTA pass covers 2048 logits; every vocabulary here is below SMs x 2048, so the lower index
    always sits in the lower sampler CTA)"""
    R, grid, tiles, V = ph.R, ph.grid, ph.tiles, ph.N
    out = {}
    out["tie across sampler warps"] = (3, 3 + SAMPLER_WARP * min(7, (V - 4) // SAMPLER_WARP))
    if V > 2 * SAMPLER_CTA + 8:
        last = (V - 1) // SAMPLER_CTA * SAMPLER_CTA
        out["tie across sampler CTAs"] = (SAMPLER_CTA + 5, min(last + 6, V - 1))
    if tiles > grid:
        i, j = (grid - 1) * R + R // 2, grid * R
        if j < V:
            out["tie, lower index in a higher CTA"] = (i, j)
    if tiles >= 3:
        out["tie across CTAs"] = (R + R // 2, 2 * R + R - 1)
    t = min(tiles - 2, 5)
    out["tie inside a tile" if R > 1 else "tie inside a CTA"] = ((t * R, t * R + R - 1) if R > 1
                                                                 else (t, t + grid))
    return {k: (i, j) for k, (i, j) in out.items() if j < V and tok not in (i, j)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROW_NAMES)
def test_head_and_sampler(name):
    """head GEMV, logsumexp, logprobs, argmax (planted ties), token log and the next h; then a prefill call"""
    r = _row(name)
    sms = _sms()

    def run(rig, path):
        H, V = rig.H, r.vocab
        eng = rig.eng
        rig.layer_zero()
        E = rig.w["lm.embed"]
        E.copy_(rig.signs(V, H))
        head = rig.w["lm.head"]
        if not r.tied:
            head.copy_(rig.randn(V, H, scale=1.0 / math.sqrt(H)))
        rig.set(lm__norm=rig.norm_w(H))
        head0 = head.clone()
        ph = phases(r, path, sms)["head"]
        x = E[rig.tok].double() * rig.w["lm.norm"].double()
        pad = (V + 7) // 8 * 8
        for what, tie, force in [("sampled", None, None), ("forced", None, 3)] + \
                                [(k, ij, None) for k, ij in _tie_cases(ph, rig.tok).items()]:
            head.copy_(head0)
            if tie is not None:
                assert rig.tok not in tie
                dom = torch.sign(x).to(torch.bfloat16) * (2.0 if r.tied else 4.0 / math.sqrt(H))
                head[list(tie)] = dom
            torch.cuda.synchronize()
            tag = f"{r.name} {path} head {what}"
            rig.fresh_pool()
            t0 = rig.decode(path, 0, 0, force=force)
            lg = rig.logits()
            check(lg, gemv_iv(head, x), f"{tag}: logits")
            lp = eng.logprobs_view().clone()
            lse_check(lg, lp, tag)
            full = (eng._view(eng.lib.b200_engine_logits(eng.h), pad, torch.bfloat16),
                    eng._view(eng.lib.b200_engine_logprobs(eng.h), pad, torch.bfloat16))
            for t in full:
                assert bool((t[V:].float() == -math.inf).all()), f"{tag}: the padding past the vocabulary is not -inf"
            top = lp.float().max()
            want = int((lp.float() == top).nonzero()[0])
            tok = int(eng.token_log_view()[t0 % eng.token_log_capacity])
            assert tok == want, f"{tag}: token {tok}, lowest index of the maximum logprob {want}"
            if tie is not None:
                assert lg[tie[0]] == lg[tie[1]] and want == tie[0], f"{tag}: the planted tie {tie} is not the argmax"
                print(f"{tag}: rows {tie} in head CTAs {_cta_of(tie[0], ph)} / {_cta_of(tie[1], ph)}, sampler CTAs "
                      f"{tie[0] // SAMPLER_CTA} / {tie[1] // SAMPLER_CTA} -> token {tok}")
            feed = tok if force is None else force
            assert torch.equal(rig.h().view(torch.int16), E[feed].view(torch.int16)), \
                f"{tag}: h is not the embedding row of the fed token {feed}"
        head.copy_(head0)
        if path == "stream":
            # prefill: the last row through the same head and sampler, advance 0
            T = 3
            emb = rig.signs(T, H)
            pos3 = torch.arange(T, dtype=torch.int32, device="cuda").repeat(3, 1).contiguous()
            rig.fresh_pool()
            torch.cuda.synchronize()
            t0 = eng.tokens_launched
            eng.prefill(emb, pos3, 0, 0)
            eng.stream.synchronize()
            tag = f"{r.name} prefill head"
            lg = rig.logits()
            check(lg, gemv_iv(head, emb[-1].double() * rig.w["lm.norm"].double()), f"{tag}: logits")
            lp = eng.logprobs_view().clone()
            lse_check(lg, lp, tag)
            want = int((lp.float() == lp.float().max()).nonzero()[0])
            tok = int(eng.token_log_view()[t0 % eng.token_log_capacity])
            assert tok == want, f"{tag}: token {tok}, lowest index of the maximum logprob {want}"
            assert torch.equal(rig.h().view(torch.int16), E[tok].view(torch.int16)), f"{tag}: h"
            assert eng.device_error() == 0

    _run_paths(r, run)
