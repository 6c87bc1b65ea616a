"""8-bit KV cache (kv_bits=8) on the GPU: the bulk conversion kernels bit-exact against the reference arithmetic
(tests/kvq_ref.py), and generate_step(kv_bits=8) end to end against the oracle with the single-request policy."""
import numpy as np
import pytest
import torch

import kvq_ref as K
from _util import cmp_noise

pytestmark = pytest.mark.gpu


def _quantize_dev(x: torch.Tensor, gs: int, cap: int):
    """x (planes, n, hd) bf16 cuda -> 8-bit planes of capacity cap through b200_kvq_quantize"""
    from mlx_vlm_b200 import _native as N
    P, n, hd = x.shape
    src = torch.zeros(P, cap + 3, hd, dtype=torch.bfloat16, device="cuda")   # a different source capacity
    src[:, :n] = x
    codes = torch.full((P, cap, hd), 7, dtype=torch.uint8, device="cuda")
    scales = torch.zeros(P, cap, hd // gs, dtype=torch.bfloat16, device="cuda")
    biases = torch.zeros_like(scales)
    N.check(N.lib().b200_kvq_quantize(src.data_ptr(), cap + 3, codes.data_ptr(), scales.data_ptr(),
                                      biases.data_ptr(), cap, P, n, hd, gs, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return codes, scales, biases


@pytest.mark.parametrize("hd,gs", [(64, 32), (64, 64), (128, 32), (128, 64), (128, 128)])
def test_quantize_dequantize_kernels_bit_exact(hd, gs):
    from mlx_vlm_b200 import _native as N
    P, n, cap = 3, 40, 48
    groups = K.special_groups(gs, P * n * hd // gs, seed=hd + gs)
    x32 = groups.reshape(P, n, hd)
    x = torch.from_numpy(x32).to(device="cuda", dtype=torch.bfloat16)
    codes, scales, biases = _quantize_dev(x, gs, cap)
    rc, rs, rb = K.quantize(x32, gs)
    assert np.array_equal(codes[:, :n].cpu().numpy(), rc)
    assert np.array_equal(scales[:, :n].float().cpu().numpy(), rs)
    assert np.array_equal(biases[:, :n].float().cpu().numpy(), rb)
    assert bool((codes[:, n:] == 7).all()), "positions past n are not written"
    out = torch.zeros(P, n, hd, dtype=torch.bfloat16, device="cuda")
    N.check(N.lib().b200_kvq_dequantize(codes.data_ptr(), scales.data_ptr(), biases.data_ptr(), cap,
                                        out.data_ptr(), n, P, n, hd, gs, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert np.array_equal(out.float().cpu().numpy(), K.dequantize(rc, rs, rb, gs))


def _build(kind, n_text, hw, seed=0):
    from mlx_vlm_b200.models.qwen2_vl import Model
    from oracle import qwen2vl as O
    from test_engine_gpu import _mk_cfg, _to_model_config
    c = _mk_cfg(kind)
    W = O.init_weights(c, seed, norm_jitter=0.05)
    model = Model(_to_model_config(c), device="cuda:0")
    model.load_weights(W)
    req = O.synthetic_request(c, n_text, image_hw=hw, seed=seed)
    return c, W, model, req


def _token_ok(tok, oracle_lp):
    m = float(oracle_lp.max())
    return float(oracle_lp[tok]) >= m - (2 * abs(m) * 2.0 ** -7 + 1e-6)


@pytest.mark.parametrize("kind,gs,after", [("tiny", 64, None), ("tiny", 32, 3), ("wide2", 64, None),
                                           ("wide2", 128, 3)])
def test_generate_kv8_against_oracle(kind, gs, after):
    """generate_step(kv_bits=8, quantized_kv_start=s) for s = 0 (the cache converts after the prefill) and
    s = T + 3: tokens equal the oracle's until the first near-tie, every step's logprobs within the noise bar,
    and every step before the switch bit-exact with a kv_bits=None run."""
    from mlx_vlm_b200.generate import generate_step
    from mlx_vlm_b200.models.cache import QuantizedKVCache, make_prompt_cache
    c, W, model, req = _build(kind, 12 if kind == "tiny" else 32, (56, 84) if kind == "tiny" else (112, 112))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    T = ids.shape[1]
    start = 0 if after is None else T + after
    n_dec = 10
    ref = K.greedy_generate_kvq(c, W, ids, pv, grid, n_dec, gs, start)
    toks = ref["tokens"][0].tolist()
    ex = K.greedy_generate_kvq(c, W, ids, pv, grid, n_dec, gs, start, dtype="f32", force_tokens=toks)
    assert ref["switch_offset"] == max(T, start)
    pvd = torch.from_numpy(pv).cuda()
    base = [(t, lp.clone()) for t, lp in generate_step(ids, model, pvd, None, max_tokens=n_dec, image_grid_thw=grid)]
    cache = make_prompt_cache(model.language_model)
    got = []
    for tok, lp in generate_step(ids, model, pvd, None, max_tokens=n_dec, image_grid_thw=grid, prompt_cache=cache,
                                 kv_bits=8, kv_group_size=gs, quantized_kv_start=start):
        n = len(got)
        got.append(tok)
        cmp_noise(lp, ref["logprobs"][n][0], ex["logprobs"][n][0], f"{kind} gs={gs} step {n} logprobs")
        if T + n <= start:   # computed before the cache converted (the forward of token n ends at offset T + n)
            assert tok == base[n][0] and torch.equal(lp, base[n][1]), f"step {n} before the switch differs"
        assert _token_ok(tok, ref["logprobs"][n][0]), f"token {n}: got {tok}, oracle {toks[n]}"
        if tok != toks[n]:
            break
    print(f"{kind} gs={gs} start={start}: tokens {got} oracle {toks}")
    assert all(isinstance(x, QuantizedKVCache) for x in cache)
    q = cache[0]
    assert q.group_size == gs and q.bits == 8 and q.offset == T + len(got)   # the loop runs one step ahead
    assert model.engine.device_error() == 0
    # the pool holds the oracle's (dequantized) K/V of the positions written for the same tokens
    eq = next((i for i, (a, b) in enumerate(zip(got, toks)) if a != b), len(got))
    n_same = min(T + eq, T + n_dec - 1)
    _check_pool(model, c, q._pool, ref, n_same)


def _check_pool(model, c, pool, ref, n):
    """the pool holds the oracle's dequantized K/V (upstream bf16 noise flips an occasional code)"""
    deq = pool.to_bf16_pool(n).buf[..., :n, :]
    model.engine.stream.synchronize()
    for layer in range(c.text.num_hidden_layers):
        for side, want in ((0, ref["cache"][layer].keys), (1, ref["cache"][layer].values)):
            d = (deq[layer, side, 0].float().cpu() - want[0, :, :n]).norm() / want[0, :, :n].norm()
            assert d <= 2e-2, f"layer {layer} side {side}: pool vs oracle rel L2 {float(d):.3e}"


@pytest.mark.parametrize("hd,gs", [(64, 32), (64, 64), (128, 32), (128, 64), (128, 128)])
# past 4096 positions: trailing ranks of 8 with few keys, one rank holding 4600, two ranks of 4500
@pytest.mark.parametrize("ctx,cluster", [(5, 1), (300, 8), (1000, 4), (4500, 8), (4600, 1), (9000, 2)])
# q heads per kv head: 6 (two CTAs of 3), 7 (one CTA), 1, 8 (two CTAs of 4)
@pytest.mark.parametrize("n_heads,n_kv", [(12, 2), (28, 4), (16, 16), (8, 1)])
def test_decode_attention_kernel(hd, gs, ctx, cluster, n_heads, n_kv):
    """The 8-bit k_attn on its own: the new row (staging plane, position ctx) is appended bit-exact to what the
    reference quantize gives, the rows before it are untouched, and the output is sdpa over the dequantized K/V (the
    new row included) within relative L2 1e-3.  The pool's scales and biases at ctx and past it hold NaN before the
    call, so a read of the pool there poisons the output."""
    from mlx_vlm_b200 import _native as N
    from oracle import mlx_semantics as S
    from _util import cmp_bf16
    cap = ((ctx + 256) // 256) * 256
    ng = hd // gs
    rng = np.random.default_rng(ctx + hd + gs)
    bf = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32)).to(torch.bfloat16)
    kv = bf(rng.standard_normal((2, n_kv, cap, hd)) * 0.8)
    codes, scales, biases = (np.zeros((2, n_kv, cap, hd), np.uint8) + 7, np.full((2, n_kv, cap, ng), np.nan, np.float32),
                             np.full((2, n_kv, cap, ng), np.nan, np.float32))
    c_, s_, b_ = K.quantize(kv.float().numpy()[:, :, :ctx], gs)
    codes[:, :, :ctx], scales[:, :, :ctx], biases[:, :, :ctx] = c_, s_, b_
    stage = torch.zeros(2, n_kv, cap, hd, dtype=torch.bfloat16)
    stage[:, :, ctx] = bf(rng.standard_normal((2, n_kv, hd)) * 0.8)
    q = bf(rng.standard_normal((n_heads, hd)))
    dc = torch.from_numpy(codes).cuda()
    ds, db = bf(scales).cuda(), bf(biases).cuda()
    dstage, dq = stage.cuda(), q.cuda()
    out = torch.zeros(n_heads, hd, dtype=torch.bfloat16, device="cuda")
    N.check(N.lib().b200_kvq_decode_attention(dq.data_ptr(), dc[0].data_ptr(), ds[0].data_ptr(), db[0].data_ptr(),
                                              dc[1].data_ptr(), ds[1].data_ptr(), db[1].data_ptr(),
                                              dstage[0].data_ptr(), dstage[1].data_ptr(), out.data_ptr(), n_heads,
                                              n_kv, hd, cap, ctx, gs, cluster, torch.cuda.current_stream().cuda_stream),
            "kvq_decode_attention")
    torch.cuda.synchronize()
    nc, ns, nb = K.quantize(stage[:, :, ctx].float().numpy(), gs)
    gc, gsc, gb = dc.cpu().numpy(), ds.float().cpu().numpy(), db.float().cpu().numpy()
    assert np.array_equal(gc[:, :, ctx], nc) and np.array_equal(gsc[:, :, ctx], ns) and np.array_equal(gb[:, :, ctx], nb)
    assert np.array_equal(gc[:, :, :ctx], codes[:, :, :ctx]) and np.array_equal(gc[:, :, ctx + 1:], codes[:, :, ctx + 1:])
    assert np.isnan(gsc[:, :, ctx + 1:]).all() and np.isnan(gb[:, :, ctx + 1:]).all()
    deq = torch.from_numpy(K.dequantize(gc[:, :, :ctx + 1], gsc[:, :, :ctx + 1], gb[:, :, :ctx + 1], gs))
    R = S.Rounder("bf16")
    want = S.sdpa(R, q.float()[None, :, None, :], deq[0][None], deq[1][None], hd ** -0.5, causal=False)
    cmp_bf16(out, want[0, :, 0], f"8-bit k_attn heads={n_heads}/{n_kv} hd={hd} gs={gs} ctx={ctx} cluster={cluster}", rel_l2=1e-3)


@pytest.mark.parametrize("kind,gs,step,before", [("tiny", 64, 5, 7), ("wide2", 128, 16, 20)])
def test_chunked_prefill_over_8bit_prefix(kind, gs, step, before):
    """prefill_step_size < T with quantized_kv_start inside the prompt: the chunks after the switch (and the last
    prompt token) attend to the 8-bit prefix and to their own rows in quantized form, as in the oracle"""
    from mlx_vlm_b200.generate import generate_step
    from mlx_vlm_b200.models.cache import make_prompt_cache
    c, W, model, req = _build(kind, 12 if kind == "tiny" else 32, (56, 84) if kind == "tiny" else (112, 112))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    T = ids.shape[1]
    assert T > 2 * step and before < T - step
    n_dec = 6
    ref = K.greedy_generate_kvq(c, W, ids, pv, grid, n_dec, gs, before, prefill_step_size=step)
    toks = ref["tokens"][0].tolist()
    ex = K.greedy_generate_kvq(c, W, ids, pv, grid, n_dec, gs, before, dtype="f32", force_tokens=toks,
                               prefill_step_size=step)
    assert ref["switch_offset"] < T - 1
    pvd = torch.from_numpy(pv).cuda()
    cache = make_prompt_cache(model.language_model)
    got = []
    for tok, lp in generate_step(ids, model, pvd, None, max_tokens=n_dec, image_grid_thw=grid, prompt_cache=cache,
                                 kv_bits=8, kv_group_size=gs, quantized_kv_start=before, prefill_step_size=step):
        n = len(got)
        got.append(tok)
        cmp_noise(lp, ref["logprobs"][n][0], ex["logprobs"][n][0], f"{kind} chunked step {n} logprobs")
        assert _token_ok(tok, ref["logprobs"][n][0]), f"token {n}: got {tok}, oracle {toks[n]}"
        if tok != toks[n]:
            break
    print(f"{kind} chunked: tokens {got} oracle {toks}")
    assert model.engine.device_error() == 0
    _check_pool(model, c, cache[0]._pool, ref, T)


def test_kv8_nbytes_and_refusals():
    """the 8-bit pool is 0.53125x the bf16 one at gs=64; a suffix prefill over it runs; other widths are refused"""
    from mlx_vlm_b200.generate import generate_step
    from mlx_vlm_b200.models.cache import make_prompt_cache
    c, W, model, req = _build("tiny", 12, (56, 84))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    T = ids.shape[1]
    pvd = torch.from_numpy(pv).cuda()
    cache = make_prompt_cache(model.language_model)
    list(generate_step(ids, model, pvd, None, max_tokens=3, image_grid_thw=grid, prompt_cache=cache))
    bf16_bytes = sum(x.nbytes for x in cache)
    cache8 = make_prompt_cache(model.language_model)
    list(generate_step(ids, model, pvd, None, max_tokens=3, image_grid_thw=grid, prompt_cache=cache8,
                       kv_bits=8, quantized_kv_start=0))
    assert sum(x.nbytes for x in cache8) / bf16_bytes == 0.53125
    # a suffix prefilled over the 8-bit cache (PromptCacheState reuse) runs and keeps the cache 8-bit
    off = cache8[0].offset
    out = list(generate_step(ids[:, -3:], model, None, None, max_tokens=2, prompt_cache=cache8, kv_bits=8,
                             quantized_kv_start=0))
    assert len(out) == 2 and cache8[0].offset == off + 3 + 2 and model.engine.device_error() == 0
    with pytest.raises(NotImplementedError):
        list(generate_step(ids, model, pvd, None, max_tokens=2, image_grid_thw=grid, kv_bits=4))
