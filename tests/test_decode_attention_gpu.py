"""The bf16 decode attention of every path, read out of the real engine, against sdpa at long and boundary contexts.

k_mega never writes the attention vector to memory, so each case runs a ONE-LAYER decoder-only engine whose weights
make the logits a known function of it: a zero embedding (h = 0, so q, k and v are the qkv bias rotated at the
position), o_proj = identity (the residual is the bf16 attention vector exactly), a zero MLP, and a head [I; 0] behind
a unit final norm, so logits[:hidden] = rms_norm(attention).  Every path runs through its normal launch code (graph
capture, the decode state, the K/V append at ctx, the rotary at pos):

  k_mega    the persistent step kernel: ATT_UN key ranges per (kv head, q-head group) exchange softmax statistics
  k_attn1   per-phase kernel, capacity <= 4096: one CTA per (kv head, q-head group), 256-key passes
  k_attn    per-phase kernel, capacity > 4096: a cluster of 1/2/4/8 CTAs splits the keys
  bd_attn   lock-step batched decode, one CTA per (row, kv head, q-head group)

Pool positions past the context, and every other row of the pool, hold NaN: a key or value read past the context
poisons the output.  The reference is oracle sdpa over the keys read back from the pool after the step (the
appended row included), then the oracle rms_norm, compared with cmp_bf16 at the fixed bar of `_compare`.  The
boundary contexts, needle
positions and capacity limits are derived from the kernels' tiling constants and shared-memory formulas (cited
below), so they follow the code."""
import numpy as np
import pytest
import torch

from _util import cmp_bf16, rl2

pytestmark = pytest.mark.gpu

# ---- tiling constants -----------------------------------------------------------------------------------------------
ATT_UN, UNR, VPRE, MEGA_ATT_G = 8, 2, 8, 4   # mega_common.cuh: key ranges, 32-key trips in flight, V rows per warp
MEGA_STAGE = 48 * 1024                        # mega_common.cuh: one weight ring stage
ATT1_MAX_CAP, ATT1_G = 4096, 4                # decode.cu: k_attn1 up to this capacity, q heads per CTA
ATT_MAXG, ATT_MAXCL = 8, 8                    # decode.cu: k_attn q heads per CTA, cluster size
BLOCK = 256                                   # k_attn1 / bd_attn: keys per pass (8 warps x 32 lanes)
BD_AG_MAX = 4                                 # decode_batch.cu
POOL_STEP = 256                               # KVPool.step: capacities are multiples of it
CLUSTERS = (1, 2, 4, 8)
NEEDLE_SCORE = 40.0   # score of a needle key with every q head of its group: it leads the other keys' maximum by > 25

# name: (n_heads, n_kv, head_dim, q/k norm)
GEOMS = {
    "2b": (12, 2, 128, False),      # Qwen2-VL-2B: G = 6
    "7b": (28, 4, 128, False),      # Qwen2-VL-7B: G = 7, uneven 4 + 3 split in k_mega and bd_attn
    "q3": (16, 8, 128, True),       # Qwen3-VL: q/k RMSNorm (k_qk_norm_rope, qk_norm_phase)
    "mha64": (16, 16, 64, False),   # MHA: 128 attention CTAs in k_mega
    "g8": (8, 1, 64, False),        # G = 8
    "7b64": (28, 4, 64, False),     # G = 7 at head_dim 64: the lock-step head grouping AG = 2 at hd 64
}
SINGLE = ("2b", "7b", "q3", "mha64", "g8")


def cdiv(a, b):
    return -(-a // b)


# ---- capacity limits: the formulas of the C functions ------------------------------------------------------------------
def attn1_smem(hd, cap):                      # decode.cu attn1_smem
    return (ATT1_G * hd + ATT1_G * cap + 8 * ATT1_G * hd) * 4


def attn_smem(hd, cap, cl):                   # decode.cu attn_smem_bytes(d, cdiv(cap, cluster), false)
    return (ATT_MAXG * cdiv(cap, cl) + ATT_MAXCL * ATT_MAXG * 2 + ATT_MAXCL * ATT_MAXG * hd + 8 * ATT_MAXG * hd) * 4


def per_phase_fits(g, cap, cl):               # decode.cu attn_prepare: <= 220 KiB
    hd = GEOMS[g][2]
    return (attn1_smem(hd, cap) if cap <= ATT1_MAX_CAP else attn_smem(hd, cap, cl)) <= 220 * 1024


def mega_hsplit(g):                           # decode_mega.cu mega_fill
    nh, nkv = GEOMS[g][:2]
    G = nh // nkv
    hs = cdiv(G, MEGA_ATT_G)
    return 2 if hs == 1 and G % 2 == 0 and G >= 4 else hs


def mega_ctas(g):                             # decode_mega.cu mega_fill: attention CTAs, at most one per SM
    return GEOMS[g][1] * mega_hsplit(g) * ATT_UN


def mega_cap_fits(g, cap):                    # decode_mega.cu mega_fill / mega_attn_scratch / mega_spare_bytes
    nh, nkv, hd, _ = GEOMS[g]
    H, inter = nh * hd, 256
    att = (MEGA_ATT_G * cdiv(cap, ATT_UN) + 8 * MEGA_ATT_G * hd + (MEGA_ATT_G + 2) * hd) * 4
    scratch = cdiv(max(att, max(inter, H, nh * hd) * 2), 128) * 128
    spare = cdiv(H * 2, 128) * 128
    return (227 * 1024 - 2048 - scratch - spare) // MEGA_STAGE >= 2


def mega_fits(g, cap, sms):
    return mega_ctas(g) <= sms and mega_cap_fits(g, cap)


def bd_smem(hd, cap, ag):                     # decode_batch.cu bd_attn_smem
    return ((ag + 2) * hd + ag * cap + 8 * ag * hd) * 4


def bd_fits(g, cap):                          # decode_batch.cu batch_decoder_begin: bd_attn_smem(d, 4) <= 200 KiB
    return bd_smem(GEOMS[g][2], cap, BD_AG_MAX) <= 200 * 1024


def bd_heads_per_cta(g, B, sms):              # decode_batch.cu bd_attn_heads_per_cta
    nh, nkv = GEOMS[g][:2]
    for ag in (1, 2, 4):
        if nkv * cdiv(nh // nkv, ag) * B <= sms:
            return ag
    return BD_AG_MAX


def max_cap(fits):
    """the largest multiple of POOL_STEP that `fits`"""
    cap = POOL_STEP
    while fits(cap + POOL_STEP):
        cap += POOL_STEP
    assert fits(cap)
    return cap


def k_attn_max(g, cl):
    return max_cap(lambda c: per_phase_fits(g, c, cl))


def test_capacity_limits_match_the_kernel_formulas():
    """the limits the cases below are built on (hd 128 / 64 at clusters 1, 2, 4, 8; k_mega for the 2B geometry;
    bd_attn); a change of a kernel's shared-memory layout shows here first"""
    assert [k_attn_max("2b", cl) for cl in CLUSTERS] == [4864, 9728, 19712, 39680]
    assert [k_attn_max("g8", cl) for cl in CLUSTERS] == [5888, 11776, 23808, 47872]
    assert max_cap(lambda c: mega_cap_fits("2b", c)) == 54784
    assert max_cap(lambda c: bd_fits("2b", c)) == 11520 and max_cap(lambda c: bd_fits("g8", c)) == 12032


# ---- the one-layer engine ----------------------------------------------------------------------------------------------
def _bf(x):
    return x.to(torch.bfloat16).float()


def _grid(t):
    """random values on the grid of quarters in [-2, 2]: with such keys and q heads every score is a sum that fp32
    holds exactly in any order, so the kernel and the reference round the same scores (an order-dependent rounding
    flip of one score moves a whole head of the output by an ulp)"""
    return ((t * 4).round().clamp(-8, 8) / 4).to(torch.bfloat16)


def needle_keys(q, nkv):
    """(n_kv, hd) keys whose unscaled score with every q head of their group is NEEDLE_SCORE (least-norm solution)"""
    nh, hd = q.shape
    Q = q.view(nkv, nh // nkv, hd)
    want = torch.full((nkv, nh // nkv, 1), NEEDLE_SCORE * hd ** 0.5)
    return (torch.linalg.pinv(Q) @ want)[..., 0]


def _rope_ref(x, pos, inv_freq):
    """warp_head_rope / the QKV epilogue (csrc): rotate_half at one position with the kernels' rounding points"""
    h = x.shape[-1] // 2
    ang = pos * inv_freq
    c, sn = _bf(torch.cos(ang)), _bf(torch.sin(ang))
    y1, y2 = x[..., :h], x[..., h:]
    return torch.cat([_bf(_bf(y1 * c) + _bf(-y2 * sn)), _bf(_bf(y2 * c) + _bf(y1 * sn))], -1)


def _rms_ref(x, w, eps):
    """warp_head_rms (csrc/common.cuh): RMSNorm of each head, two roundings"""
    rs = 1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + eps)
    return _bf(_bf(x * rs) * w)


class Rig:
    """one-layer engine of geometry g whose logits are rms_norm(attention output)"""
    EPS = 1e-6

    def __init__(self, g):
        from mlx_vlm_b200 import _native as N
        from mlx_vlm_b200.engine import Engine, _inv_freq
        from mlx_vlm_b200.models.qwen2_vl.qwen2_vl import WeightArena, weight_manifest
        nh, nkv, hd, qk = GEOMS[g]
        self.g, self.nh, self.nkv, self.hd, self.qk = g, nh, nkv, hd, qk
        self.H = H = nh * hd
        c = N.Qwen2VLConfig()
        c.hidden, c.n_layers, c.inter = H, 1, 256
        c.n_heads, c.n_kv_heads, c.head_dim = nh, nkv, hd
        c.vocab = H + 8
        c.rms_eps, c.rope_theta = self.EPS, 1000000.0
        c.mrope_section[0], c.mrope_section[1], c.mrope_section[2] = hd // 2, 0, 0
        c.tie_embeddings = 0
        c.external_vision = 1
        c.v_depth, c.v_embed, c.v_heads, c.v_mlp, c.v_patch_dim, c.v_merge = 0, 8, 1, 8, 8, 1
        c.v_out, c.v_ln_eps = H, 1e-5
        self.eng = eng = Engine(c, torch.device("cuda", 0))
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.inv_freq = torch.from_numpy(_inv_freq(hd, c.rope_theta))
        arena = WeightArena(weight_manifest(c), eng.device)
        gen = torch.Generator().manual_seed(sum(map(ord, g)))
        QKV = (nh + 2 * nkv) * hd
        fill = {"lm.embed": torch.zeros(c.vocab, H), "lm.norm": torch.ones(H),
                "lm.head": torch.cat([torch.eye(H), torch.zeros(8, H)]),
                "lm.0.ln1": torch.ones(H), "lm.0.ln2": torch.ones(H),
                "lm.0.wqkv": torch.randn(QKV, H, generator=gen),   # multiplies x = 0: must not matter
                "lm.0.bqkv": torch.zeros(QKV), "lm.0.wo": torch.eye(H),
                "lm.0.wgu": torch.zeros(2 * 256, H), "lm.0.wd": torch.zeros(H, 256)}
        for name, t in fill.items():
            v = arena.view(name)
            v.copy_(t.to(torch.bfloat16))
            eng.set_weight(name, v)
        self.arena = arena
        self.bias = arena.view("lm.0.bqkv")
        if qk:
            # q / k norm weights on eighths: the normalised q heads (see new_bias) stay on a coarse grid
            self.qn = (1.0 + torch.randint(-3, 4, (hd,), generator=gen) / 8).to(torch.bfloat16)
            self.kn = (1.0 + torch.randint(-3, 4, (hd,), generator=gen) / 8).to(torch.bfloat16)
            self.qn_d, self.kn_d = self.qn.cuda(), self.kn.cuda()
            eng.set_weight("lm.0.qn", self.qn_d)
            eng.set_weight("lm.0.kn", self.kn_d)
        self.gen = gen
        self.new_bias()
        torch.cuda.synchronize()

    def new_bias(self, needle_new=False):
        """random q / k / v bias; needle_new: the new key (bias k) points along its q heads so that it dominates"""
        nh, nkv, hd = self.nh, self.nkv, self.hd
        b = _grid(torch.randn((nh + 2 * nkv) * hd, generator=self.gen)).float()
        if self.qk:   # q and k heads of +-1: their RMSNorm is exactly +-(norm weight)
            b[:(nh + nkv) * hd] = torch.randint(0, 2, ((nh + nkv) * hd,), generator=self.gen) * 2.0 - 1.0
        if needle_new:
            b[nh * hd:(nh + nkv) * hd] = needle_keys(self.q_ref(_bf(b), 0), nkv).reshape(-1)
        self.bias.copy_(b.to(torch.bfloat16))
        self.b = self.bias.float().cpu()
        torch.cuda.synchronize()

    # reference q / new key / new value of the step (pos: the rotary position)
    def q_ref(self, b, pos):
        q = b[:self.nh * self.hd].view(self.nh, self.hd)
        if self.qk:
            q = _rms_ref(q, self.qn.float(), self.EPS)
        return _rope_ref(q, pos, self.inv_freq) if pos else q

    def k_ref(self, pos):
        k = self.b[self.nh * self.hd:(self.nh + self.nkv) * self.hd].view(self.nkv, self.hd)
        if self.qk:
            k = _rms_ref(k, self.kn.float(), self.EPS)
        return _rope_ref(k, pos, self.inv_freq) if pos else k

    def v_ref(self):
        return self.b[(self.nh + self.nkv) * self.hd:].view(self.nkv, self.hd)

    @staticmethod
    def exact(pos):
        """no rotary at position 0: the step's q and new key are the (normalised) bias, on the grid"""
        return pos == 0

    def pool(self, cap, batch=1):
        from mlx_vlm_b200.models.cache import KVPool
        return KVPool(1, self.nkv, self.hd, self.eng.device, batch=batch, capacity=cap)


_RIGS = {}


def rig(g):
    if g not in _RIGS:
        _RIGS[g] = Rig(g)
    return _RIGS[g]


def _kv_base(r, cap, seed):
    """random bf16 keys and values of one row: (2, n_kv, cap, hd)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return _grid(torch.randn(2, r.nkv, cap, r.hd, device="cuda", generator=gen))


def _fill(pool, row, ctx, base, scale_range=None, needle=None, r=None, q=None):
    """row `row` positions < ctx from `base`, everything else NaN; scale_range (a, b): keys a..b-1 x 8;
    needle j: key j dominates every q head of its kv head (q: the step's q heads)"""
    buf = pool.buf
    buf.fill_(float("nan"))
    buf[0, :, row, :, :ctx] = base[:, :, :ctx]
    if scale_range is not None:
        a, b = scale_range
        buf[0, 0, row, :, a:b] = (buf[0, 0, row, :, a:b].float() * 8).to(torch.bfloat16)
    if needle is not None:
        buf[0, 0, row, :, needle] = needle_keys(q, r.nkv).to(torch.bfloat16).cuda()
    torch.cuda.synchronize()
    return buf.view(torch.int16).clone()


def _check_row(r, pool, row, ctx, pos, before, got, name, dominant=None):
    """appended row, untouched rest of the pool (before: its int16 bits before the step; None: checked by the
    caller), and the attention output (got: logits[:hidden]) against sdpa"""
    from oracle import mlx_semantics as S
    buf = pool.buf
    if before is not None:
        changed = buf.view(torch.int16) != before
        changed[0, :, row, :, ctx] = False
        assert not bool(changed.any()), f"{name}: the step wrote pool positions other than ctx={ctx} of row {row}"
    K = buf[0, 0, row, :, :ctx + 1].float().cpu()
    V = buf[0, 1, row, :, :ctx + 1].float().cpu()
    assert torch.equal(V[:, ctx], r.v_ref()), f"{name}: appended V row is not the bias"
    kw = r.k_ref(pos)
    if r.exact(pos):
        assert torch.equal(K[:, ctx], kw), f"{name}: appended K row is not the bias"
    else:
        same = (K[:, ctx] == kw).float().mean().item()
        assert rl2(K[:, ctx], kw) <= 1e-2 and same >= 0.95, f"{name}: appended K row: {same:.3f} equal"
    R = S.Rounder("bf16")
    q = r.q_ref(r.b, pos)
    att = S.sdpa(R, q[None, :, None, :], K[None], V[None], r.hd ** -0.5, causal=False)[0, :, 0].reshape(-1)
    if dominant is not None:   # the needle case is built right: the output is that value row
        vr = V[:, dominant].repeat_interleave(r.nh // r.nkv, 0).reshape(-1)
        assert rl2(att, vr) < 0.1, f"{name}: the needle does not dominate the reference"
    _compare(got, S.rms_norm(R, att, torch.ones(r.H), r.EPS), name, r.nh)


# The bar.  The kernels sum the softmax denominator and P.V in fp32 in another order than the oracle (and take expf
# from the device library): now and then a probability rounds to the neighbouring bf16 value, and when it is one of
# the larger probabilities most outputs of that q head move by an ulp.  Measured on an H100 over 11453 comparisons of
# this file (two runs): at most rel L2 1.27e-3 and 4.9 % differing elements with random keys (g8, 8 heads: 1/8 of
# the outputs is one head), and 1.42e-3 and 6.8 % (two heads of 28) when one range is scaled x 8 so that a handful
# of keys carry the softmax.  The bar sits above those: rel L2 <= 2e-3, and at most 2 % plus one q head (two heads
# with a scaled range) of differing elements.  One key dropped or counted twice among 54784 random keys moves the
# output by rel L2 ~6e-3; a key given to the wrong owner, a missed range or a statistics word of another step moves
# it by order 1.
def _compare(got, want, name, n_heads):
    heads = 2 if "scaled" in name else 1
    cmp_bf16(got, want, name, rel_l2=2e-3, max_mismatch=0.02 + heads / n_heads)


def _decode_one(r, pool, row, ctx, pos, path):
    eng = r.eng
    eng.set_next(0, ctx, pos)
    n0 = eng.launch_count
    eng.decode(1)
    eng.stream.synchronize()
    per_phase = 1 * (6 if r.qk else 5) + 2
    want = (1 if path == "k_mega" else per_phase) + 1   # + the state kernel of the call
    assert eng.launch_count - n0 == want, f"{path} expected, {eng.launch_count - n0} launches"
    return eng.logits_view()[:r.H].float().cpu()


# ---- contexts and needle positions derived from the tiling -------------------------------------------------------------
BASE_CTX = (0, 1, 6, 7, 8, 31, 32, 63, 64, 255, 256, 257, 511, 512, 513)


def contexts(path, cap, cl=1):
    """contexts (cached keys; the step attends to ctx + 1) where the path splits its work differently"""
    s = set(BASE_CTX) | {cap - 1, cap - 2, cap - BLOCK - 1}
    if path == "k_mega":
        # per = keys of one range: 1, one V prefetch (VPRE rows per warp x 8 warps), one and two score trips
        for per in (1, VPRE, 32, 32 * UNR, 2 * 32 * UNR, VPRE * 8 + 32):
            for n in (ATT_UN * (per - 1) + 1, ATT_UN * per, ATT_UN * per + 1):
                s.add(n - 1)
    elif path == "k_attn":
        # chunk = keys of one rank; n = cl + 1 leaves trailing ranks with no keys
        for chunk in (1, 2, 8, 32, BLOCK, 2 * BLOCK + 1):
            for n in (cl * (chunk - 1) + 1, cl * chunk, cl * chunk + 1):
                s.add(n - 1)
        s.add(cl)
    else:
        for k in range(1, cap // BLOCK + 1):
            s |= {k * BLOCK - 1, k * BLOCK}
    return sorted(c for c in s if 0 <= c < cap)


def owner_edges(path, nkeys, cl=1):
    """key positions at the edges of the work split for nkeys keys"""
    if path == "k_mega":
        per = cdiv(nkeys, ATT_UN)
        e = set()
        for u in range(ATT_UN):
            e |= {u * per - 1, u * per, u * per + 63, u * per + 64}
        return e
    if path == "k_attn":
        chunk = cdiv(nkeys, cl)
        return {x for rk in range(1, cl) for x in (rk * chunk - 1, rk * chunk)}
    return {x for k in range(1, cdiv(nkeys, BLOCK)) for x in (k * BLOCK - 1, k * BLOCK)}


def scaled_range(path, nkeys, cl=1):
    """the keys of one owner (range / rank / 256-key block), scaled x 8 so that the owners' maxima differ by tens"""
    if path == "k_mega":
        per = cdiv(nkeys, ATT_UN)
        u = ATT_UN // 2 if ATT_UN // 2 * per < nkeys - 1 else 0
        return u * per, min(nkeys - 1, (u + 1) * per)
    if path == "k_attn":
        chunk = cdiv(nkeys, cl)
        rk = cl // 2 if cl // 2 * chunk < nkeys - 1 else 0
        return rk * chunk, min(nkeys - 1, (rk + 1) * chunk)
    k = 1 if BLOCK < nkeys - 1 else 0
    return k * BLOCK, min(nkeys - 1, (k + 1) * BLOCK)


# ---- single request: k_mega, k_attn1, k_attn ---------------------------------------------------------------------------
def _single_cases():
    out = []
    for g in SINGLE:
        m = max_cap(lambda c: mega_cap_fits(g, c))
        for cap in (256, 4096, 8192, m):
            out.append((g, "k_mega", cap, 8))
        for cap in (256, ATT1_MAX_CAP):
            out.append((g, "k_attn1", cap, 8))
        for cl in CLUSTERS:
            out.append((g, "k_attn", ATT1_MAX_CAP + POOL_STEP, cl))
            out.append((g, "k_attn", k_attn_max(g, cl), cl))
        out.append((g, "k_attn", 8192, 8))
    return out


def _run_single(r, path, cap, cl, ctxs, seed, needles=True, scaled=True):
    """every context of `ctxs` (plain, one owner's keys scaled, and with a needle at each boundary) on row 1 of a
    two-row pool"""
    eng = r.eng
    pool = r.pool(cap, batch=2)
    r.eng.bind_pool(pool)
    eng.set_kv_row(1)
    base = _kv_base(r, cap, seed)
    tag = f"{path} {r.g} cap={cap} cluster={cl}"
    needle_ctx = max(c for c in ctxs if c < 8192)   # the needle cases: the largest context below 8192 keys
    for ctx in ctxs:
        n = ctx + 1
        variants = [("", None, None)]
        if scaled and n >= 16:
            variants.append(("scaled", scaled_range(path, n, cl), None))
        if needles and ctx == needle_ctx:
            for j in sorted({0, ctx - 1} | {x for x in owner_edges(path, n, cl) if 0 <= x < ctx}):
                variants.append((f"needle@{j}", None, j))
        for what, sr, j in variants:
            before = _fill(pool, 1, ctx, base, sr, j, r, r.q_ref(r.b, 0))
            got = _decode_one(r, pool, 1, ctx, 0, path)
            _check_row(r, pool, 1, ctx, 0, before, got, f"{tag} ctx={ctx} {what}", dominant=j)
    if needles and not r.qk:   # the new key itself dominates (through the bias; a k norm would fix its length)
        ctx = needle_ctx
        r.new_bias(needle_new=True)
        try:
            before = _fill(pool, 1, ctx, base)
            got = _decode_one(r, pool, 1, ctx, 0, path)
            _check_row(r, pool, 1, ctx, 0, before, got, f"{tag} ctx={ctx} needle@ctx (new key)", dominant=ctx)
        finally:
            r.new_bias()
    return pool


@pytest.mark.parametrize("g,path,cap,cl", _single_cases(),
                         ids=[f"{g}-{p}-cap{c}-cl{cl}" for g, p, c, cl in _single_cases()])
def test_single_request_attention(g, path, cap, cl):
    r = rig(g)
    if path == "k_mega":
        if mega_ctas(g) > r.sms:
            pytest.skip(f"k_mega runs {mega_ctas(g)} attention CTAs of {g}; this GPU has {r.sms} SMs")
        assert mega_fits(g, cap, r.sms)
    else:
        assert per_phase_fits(g, cap, cl)
        assert (path == "k_attn1") == (cap <= ATT1_MAX_CAP)
    r.eng.set_mega(path == "k_mega")
    r.eng.set_attn_cluster(cl)
    try:
        _run_single(r, path, cap, cl, contexts(path, cap, cl), seed=cap + cl)
        assert r.eng.device_error() == 0
    finally:
        r.eng.set_mega(1)
        r.eng.set_attn_cluster(8)


@pytest.mark.parametrize("g", ["2b", "q3", "g8"])
def test_mega_consecutive_steps(g):
    """decode(1) three times on k_mega: each step appends its row and attends to the previous steps' rows, the
    statistics words of consecutive steps carry alternating epochs; pos = ctx + delta with delta < 0 (Qwen2-VL rope
    deltas); one key range scaled x 8"""
    r = rig(g)
    cap, ctx0, delta = 2048, 1500, -37
    pool = r.pool(cap, batch=2)
    r.eng.bind_pool(pool)
    r.eng.set_kv_row(1)
    base = _kv_base(r, cap, 7)
    before = _fill(pool, 1, ctx0, base, scaled_range("k_mega", ctx0 + 1))
    r.eng.set_next(0, ctx0, ctx0 + delta)
    for i in range(3):
        ctx, pos = ctx0 + i, ctx0 + i + delta
        n0 = r.eng.launch_count
        r.eng.decode(1)
        r.eng.stream.synchronize()
        assert r.eng.launch_count - n0 == 2, "k_mega expected"
        got = r.eng.logits_view()[:r.H].float().cpu()
        _check_row(r, pool, 1, ctx, pos, before, got, f"k_mega {r.g} cap={cap} step {i} ctx={ctx} pos={pos} scaled")
        before = pool.buf.view(torch.int16).clone()
    assert r.eng.device_error() == 0


# ---- lock-step batch: bd_attn ------------------------------------------------------------------------------------------
LOCKSTEP = [("7b", 4), ("7b", 8), ("7b", 16), ("2b", 3), ("2b", 16), ("q3", 5), ("q3", 16), ("mha64", 8),
            ("mha64", 12), ("7b64", 4), ("7b64", 8), ("7b64", 16), ("g8", 16)]


def test_lockstep_cases_reach_every_head_grouping():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for hd in (64, 128):
        ags = {bd_heads_per_cta(g, B, sms) for g, B in LOCKSTEP if GEOMS[g][2] == hd}
        assert ags == {1, 2, 4}, (hd, ags)


def _run_lockstep(r, B, cap, ctx_rounds, pos_of=lambda c: 0, needle_rounds=None, new_key=False):
    """one batch_begin + batch_decode(1) per round: row b at context ctx_rounds[i][b] (its keys random, all else
    NaN, row B never attended), with a needle at needle_rounds[i][b] when given; new_key: the bias makes every
    row's new key dominate (Rig.new_bias(needle_new=True))"""
    eng = r.eng
    pool = r.pool(cap, batch=B + 1)   # row B is never attended: NaN throughout
    eng.bind_pool(pool)
    base = [_kv_base(r, cap, 100 + b) for b in range(B)]
    ag = bd_heads_per_cta(r.g, B, r.sms)
    q = r.q_ref(r.b, 0)
    for rnd, ctxs in enumerate(ctx_rounds):
        pool.buf.fill_(float("nan"))
        needles = {}
        for b, c in enumerate(ctxs):
            pool.buf[0, :, b, :, :c] = base[b][:, :, :c]
            if needle_rounds is not None:
                j = needle_rounds[rnd][b]
                if j is not None:
                    assert j < c and pos_of(c) == 0
                    pool.buf[0, 0, b, :, j] = needle_keys(q, r.nkv).to(torch.bfloat16).cuda()
                    needles[b] = j
        torch.cuda.synchronize()
        before = pool.buf.view(torch.int16).clone()
        pos = [pos_of(c) for c in ctxs]
        eng.batch_begin(np.zeros(B), np.asarray(ctxs), np.asarray(pos), np.ones(B))
        eng.batch_decode(1)
        eng.stream.synchronize()
        logits = eng.batch_logits_view()[:, :r.H].float().cpu()
        changed = pool.buf.view(torch.int16) != before
        for b, c in enumerate(ctxs):
            changed[0, :, b, :, c] = False
        assert not bool(changed.any()), f"bd_attn {r.g} B={B}: positions other than each row's ctx were written"
        if new_key:
            needles = dict(enumerate(ctxs))
        for b, c in enumerate(ctxs):
            _check_row(r, pool, b, c, pos[b], None, logits[b],
                       f"bd_attn {r.g} AG={ag} B={B} cap={cap} row {b} ctx={c} pos={pos[b]}"
                       + (f" needle@{needles[b]}" if b in needles else ""), dominant=needles.get(b))
    assert eng.device_error() == 0


def _lockstep_suite(r, B, cap):
    """the contexts of the rows walk the boundary list; needles at 0, ctx - 1, every 256-key block edge and (without
    a q/k norm, which fixes the new key's length) the new key itself; one round at rotary positions > 0"""
    ctxs = contexts("bd_attn", cap)
    rounds = [[ctxs[(i * B + b) % len(ctxs)] for b in range(B)] for i in range(cdiv(len(ctxs), B))]
    _run_lockstep(r, B, cap, rounds)
    # needles at 0, ctx - 1 and every 256-key block edge, B of them per round, each row at its own context
    ctxs = [cap - 1 - b for b in range(B)]
    spots = [0, None] + sorted(x for x in owner_edges("bd_attn", cap) if x < ctxs[-1])
    n_rounds = cdiv(len(spots), B)
    needles = [[ctxs[b] - 1 if spots[(i * B + b) % len(spots)] is None else spots[(i * B + b) % len(spots)]
                for b in range(B)] for i in range(n_rounds)]
    _run_lockstep(r, B, cap, [ctxs] * n_rounds, needle_rounds=needles)
    if not r.qk:
        r.new_bias(needle_new=True)
        try:
            _run_lockstep(r, B, cap, [[0] + [cap - 1 - b * (cap // B) for b in range(1, B)]], new_key=True)
        finally:
            r.new_bias()
    _run_lockstep(r, B, cap, [[min(cap - 1, 300 + 97 * b) for b in range(B)]], pos_of=lambda c: c - 11)


@pytest.mark.parametrize("g,B", LOCKSTEP, ids=[f"{g}-B{B}" for g, B in LOCKSTEP])
def test_lockstep_attention(g, B):
    """every row attends to its own keys at its own context"""
    _lockstep_suite(rig(g), B, 2048)


@pytest.mark.parametrize("g,B", [("7b", 16), ("g8", 16), ("mha64", 4)])
@pytest.mark.parametrize("cap", [4096, 8192])
def test_lockstep_capacities(g, B, cap):
    """bd_attn keeps AG x cap scores in shared memory: larger pools place each head's scores further apart"""
    _lockstep_suite(rig(g), B, cap)


@pytest.mark.parametrize("g", ["7b", "g8"])
def test_lockstep_at_capacity_limit(g):
    """bd_attn at its largest capacity (bd_attn_smem(d, 4) <= 200 KiB) and the clean refusal one step above it"""
    from mlx_vlm_b200 import _native as N
    r = rig(g)
    cap = max_cap(lambda c: bd_fits(g, c))
    _run_lockstep(r, 16, cap, [[cap - 1 - 257 * b for b in range(16)]])
    r.eng.bind_pool(r.pool(cap + POOL_STEP, batch=2))
    with pytest.raises(N.B200Error, match="capacity"):
        r.eng.batch_begin(np.zeros(2), np.asarray([5, 9]), np.zeros(2), np.ones(2))
    assert r.eng.device_error() == 0
    _run_lockstep(r, 2, 512, [[100, 511]])


# ---- capacity edges ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", ["2b", "mha64"])
def test_capacity_edges(g):
    """one pool step above each single-request path's largest capacity the decode call fails with B200Error naming
    the capacity, the device error stays 0, and the engine decodes correctly after a rebind to a smaller pool"""
    from mlx_vlm_b200 import _native as N
    r = rig(g)
    try:
        for mega, cl in [(1, 8)] + [(0, cl) for cl in CLUSTERS]:
            r.eng.set_mega(mega)
            r.eng.set_attn_cluster(cl)
            if mega:   # past k_mega's limit the step falls back to the per-phase kernels, whose limit is lower
                top = max_cap(lambda c: mega_fits(g, c, r.sms))
                assert not per_phase_fits(g, top + POOL_STEP, cl)
            else:
                top = k_attn_max(g, cl)
            pool = r.pool(top + POOL_STEP)
            r.eng.bind_pool(pool)
            r.eng.set_kv_row(0)
            pool.buf.zero_()
            r.eng.set_next(0, 100, 0)
            with pytest.raises(N.B200Error, match=f"cache capacity {top + POOL_STEP} too large"):
                r.eng.decode(1)
            r.eng.stream.synchronize()
            assert r.eng.device_error() == 0
            del pool
            _run_single(r, "k_mega" if mega else "k_attn1", 1024, cl, [0, 257, 1000], seed=cl, needles=False)
    finally:
        r.eng.set_mega(1)
        r.eng.set_attn_cluster(8)


def test_cache_longer_than_k_attn_holds():
    """2B geometry, capacity 40960: above k_attn's limit at cluster 8 (39680), within k_mega's (54784).  A short
    prefill is accepted, k_mega decodes it within the bar, and only a step forced onto the per-phase kernels is
    refused"""
    from mlx_vlm_b200 import _native as N
    r = rig("2b")
    cap = 40960
    assert mega_fits("2b", cap, r.sms) and not per_phase_fits("2b", cap, 8)
    pool = r.pool(cap)
    r.eng.bind_pool(pool)
    r.eng.set_kv_row(0)
    pool.buf.zero_()
    T = 8
    emb = torch.zeros(T, r.H, dtype=torch.bfloat16, device="cuda")
    pos3 = torch.arange(T, dtype=torch.int32, device="cuda").repeat(3, 1).contiguous()
    torch.cuda.synchronize()
    r.eng.prefill(emb, pos3, 0, 0)
    r.eng.stream.synchronize()
    assert torch.equal(pool.buf[0, 1, 0, :, :T].float().cpu(), r.v_ref()[:, None].expand(-1, T, -1)), \
        "the prefill did not append its rows"
    base = _kv_base(r, cap, 11)
    for ctx in (T, 20000, cap - 1):
        before = _fill(pool, 0, ctx, base, scaled_range("k_mega", ctx + 1))
        got = _decode_one(r, pool, 0, ctx, 0, "k_mega")
        _check_row(r, pool, 0, ctx, 0, before, got, f"k_mega 2b cap={cap} ctx={ctx} scaled")
    r.eng.set_mega(0)
    try:
        r.eng.set_next(0, 100, 0)
        with pytest.raises(N.B200Error, match=f"cache capacity {cap} too large"):
            r.eng.decode(1)
        assert r.eng.device_error() == 0
    finally:
        r.eng.set_mega(1)


def test_pool_growth_past_k_attn_limit():
    """a conversation that grows from 20480 to 20481 cached tokens: LanguageModel._bind doubles the pool to 40960
    (KVPool.reserve), and the next decode step runs on the default path within the bar"""
    import types
    from mlx_vlm_b200.models.cache import KVCache
    from mlx_vlm_b200.models.qwen2_vl.language import LanguageModel
    r = rig("2b")
    pool = r.pool(20480)
    lm = LanguageModel(types.SimpleNamespace(model_type="qwen2_vl"), None, lambda: r.eng)
    cache = [KVCache(pool, 0)]
    base = _kv_base(r, 20480, 13)
    pool.buf[0, :, 0] = base
    cache[0].offset = ctx = 20480
    torch.cuda.synchronize()
    assert lm._bind(cache, ctx + 1, decode=True) is pool and pool.capacity == 40960
    assert torch.equal(pool.buf[0, :, 0, :, :ctx], base), "the grown pool lost the cached rows"
    pool.buf[0, :, 0, :, ctx:] = float("nan")
    torch.cuda.synchronize()
    before = pool.buf.view(torch.int16).clone()
    got = _decode_one(r, pool, 0, ctx, 0, "k_mega")
    _check_row(r, pool, 0, ctx, 0, before, got, f"k_mega 2b grown pool cap={pool.capacity} ctx={ctx}")
    assert r.eng.device_error() == 0


def test_set_attn_cluster_rejects_other_sizes():
    from mlx_vlm_b200 import _native as N
    r = rig("g8")
    for bad in (0, 3, 16):
        with pytest.raises(N.B200Error, match="cluster must be 1, 2, 4 or 8"):
            r.eng.set_attn_cluster(bad)
