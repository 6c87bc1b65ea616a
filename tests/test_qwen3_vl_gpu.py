"""Qwen3-VL decoder on the GPU, every call through the C ABI, against tests/qwen3vl_ref.py: the q/k norm + interleaved
M-RoPE + KV append op on identical inputs (relative L2 1e-3), greedy generation at tiny, head_dim != hidden / heads
and 2B widths (first-step logprobs on the noise bar of tests/_util.cmp_noise, tokens equal above the two-ulp margin),
k_mega == the per-phase step (tokens, logprobs, K / V rows, bit for bit), chunked prefill == one-shot prefill, the
lock-step batch against requests run alone, and an 8-bit KV run."""
import types

import numpy as np
import pytest
import torch

from _util import cmp_noise, rl2
from test_engine_gpu import _token_ok

pytestmark = pytest.mark.gpu


def _config(kind):
    from mlx_vlm_b200.models.qwen3_vl import ModelConfig, TextConfig, VisionConfig
    if kind == "tiny":
        dims = dict(num_hidden_layers=2, hidden_size=256, intermediate_size=512, num_attention_heads=4,
                    num_key_value_heads=2, head_dim=64, vocab_size=1024, sec=[8, 12, 12])
    elif kind == "hd128":   # head_dim given explicitly and != hidden / heads (as in Qwen3-VL-4B: 2560 / 32 heads of 128)
        dims = dict(num_hidden_layers=2, hidden_size=256, intermediate_size=512, num_attention_heads=4,
                    num_key_value_heads=2, head_dim=128, vocab_size=1024, sec=[24, 20, 20])
    else:   # the Qwen3-VL-2B decoder widths, 3 of its 28 layers
        dims = dict(num_hidden_layers=3, hidden_size=2048, intermediate_size=6144, num_attention_heads=16,
                    num_key_value_heads=8, head_dim=128, vocab_size=4096, sec=[24, 20, 20])
    sec = dims.pop("sec")
    text = TextConfig(model_type="qwen3_vl", rms_norm_eps=1e-6, rope_theta=5000000.0, max_position_embeddings=8192,
                      rope_scaling={"rope_type": "default", "mrope_section": sec, "mrope_interleaved": True},
                      tie_word_embeddings=(kind == "tiny"), **dims)
    return ModelConfig(text_config=text, vision_config=VisionConfig(depth=1), model_type="qwen3_vl",
                       vocab_size=dims["vocab_size"], eos_token_id=[])


def _model(kind, seed=0):
    from qwen3vl_ref import host_weights
    from mlx_vlm_b200.models.qwen3_vl import Model
    cfg = _config(kind)
    W = host_weights(cfg, seed=seed, std=0.05)
    model = Model(cfg, device="cuda:0")
    model.load_weights({k: v.to(torch.bfloat16) for k, v in W.items()})
    return cfg, W, model


def _run(model, ids, n, **kw):
    from mlx_vlm_b200.generate import generate_step
    toks, lps = [], []
    for t, lp in generate_step(ids, model, None, None, max_tokens=n, **kw):
        toks.append(int(t))
        lps.append(lp.float().cpu())
    assert model.engine.device_error() == 0
    return toks, lps


@pytest.mark.parametrize("hd,nh,nkv", [(64, 4, 2), (128, 16, 8)])
def test_qk_norm_interleaved_rope_append_op(hd, nh, nkv):
    from qwen3vl_ref import interleaved_selector
    from oracle import mlx_semantics as S
    from oracle.mlx_semantics import Rounder
    from oracle.qwen2vl import _rotate_half
    from mlx_vlm_b200 import _native as N
    lib = N.lib()
    g = torch.Generator().manual_seed(hd)
    T, ctx0, cap, eps = 37, 5, 64, 1e-6
    qkv = (torch.randn(T, (nh + 2 * nkv) * hd, generator=g) * 2).to(torch.bfloat16)
    qn = (1 + 0.3 * torch.randn(hd, generator=g)).to(torch.bfloat16)
    kn = (1 + 0.3 * torch.randn(hd, generator=g)).to(torch.bfloat16)
    pos3 = torch.stack([torch.arange(T) + 3, torch.arange(T) * 2 % 11, torch.arange(T) * 5 % 13]).to(torch.int32)
    sec = [8, 12, 12] if hd == 64 else [24, 20, 20]
    sel = torch.from_numpy(interleaved_selector(sec, hd // 2).astype(np.int32))
    inv = 1.0 / (5000000.0 ** (torch.arange(0, hd, 2).to(torch.float32) / hd))
    d = {k: v.cuda() for k, v in dict(qkv=qkv.clone(), qn=qn, kn=kn, pos3=pos3, sel=sel, inv=inv).items()}
    kc = torch.zeros(nkv, cap, hd, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    N.check(lib.b200_qk_norm(d["qkv"].data_ptr(), T, nh, nkv, hd, d["qn"].data_ptr(), d["kn"].data_ptr(), eps, 0))
    N.check(lib.b200_mrope_kv_write(d["qkv"].data_ptr(), d["pos3"].data_ptr(), d["inv"].data_ptr(), d["sel"].data_ptr(),
                                    kc.data_ptr(), vc.data_ptr(), T, ctx0, cap, nh, nkv, hd, 0))
    torch.cuda.synchronize()
    R = Rounder("bf16")
    x = qkv.float()
    q = S.rms_norm(R, x[:, :nh * hd].reshape(T, nh, hd), qn.float(), eps)
    k = S.rms_norm(R, x[:, nh * hd:(nh + nkv) * hd].reshape(T, nkv, hd), kn.float(), eps)
    freqs = pos3.long()[torch.from_numpy(interleaved_selector(sec, hd // 2))].T.float() * inv
    emb = torch.cat([freqs, freqs], -1)
    c, s = R.r(torch.cos(emb))[:, None], R.r(torch.sin(emb))[:, None]
    q = R.r(R.r(q * c) + R.r(_rotate_half(q) * s))
    k = R.r(R.r(k * c) + R.r(_rotate_half(k) * s))
    got_q = d["qkv"].float().cpu()[:, :nh * hd].reshape(T, nh, hd)
    assert rl2(got_q, q) < 1e-3
    assert rl2(kc.float().cpu()[:, ctx0:ctx0 + T].transpose(0, 1), k) < 1e-3
    assert torch.equal(vc.cpu()[:, ctx0:ctx0 + T].transpose(0, 1), qkv[:, (nh + nkv) * hd:].reshape(T, nkv, hd))
    assert float(kc[:, :ctx0].abs().sum()) == 0 and float(kc[:, ctx0 + T:].abs().sum()) == 0


@pytest.mark.parametrize("kind", ["tiny", "hd128", "2b"])
def test_greedy_against_reference(kind):
    from qwen3vl_ref import greedy_generate
    cfg, W, model = _model(kind)
    ids = np.random.default_rng(1).integers(0, cfg.text_config.vocab_size, size=(1, 29))
    n = 10
    toks, lps = _run(model, ids, n)
    want, want_lps = greedy_generate(cfg, W, ids, n, "bf16")
    _, f32_lps = greedy_generate(cfg, W, ids, 1, "f32")
    cmp_noise(lps[0], want_lps[0][0].float(), f32_lps[0][0].float(), f"{kind} step-0 logprobs")
    for i, t in enumerate(toks):
        if t != int(want[0, i]):
            assert _token_ok(t, want_lps[i][0].float()), f"{kind}: token {i}: {t} vs reference {int(want[0, i])}"
            break


def _kv_rows(model, n):
    pool = model.language_model._pool
    return pool.buf[:, :, :, :, :n].clone()


@pytest.mark.parametrize("kind", ["tiny", "hd128", "2b"])
def test_k_mega_equals_per_phase_and_chunked_prefill_is_exact(kind):
    """k_mega (one launch per step, q/k norm in its own phase) against the per-phase step: tokens, logprobs and every
    appended K / V row bit for bit; chunked prefill against one-shot prefill, bit for bit"""
    cfg, W, model = _model(kind)
    ids = np.random.default_rng(2).integers(0, cfg.text_config.vocab_size, size=(1, 41))
    n = 8
    model.engine.set_mega(0)
    t0, l0 = _run(model, ids, n)
    kv0 = _kv_rows(model, 41 + n - 1)
    model.engine.set_mega(1)
    c0 = model.engine.launch_count
    t1, l1 = _run(model, ids, n)
    kv1 = _kv_rows(model, 41 + n - 1)
    assert t1 == t0 and all(torch.equal(a, b) for a, b in zip(l1, l0))
    assert torch.equal(kv1, kv0)
    per_step_mega = model.engine.launch_count - c0
    model.engine.set_mega(0)
    c0 = model.engine.launch_count
    _run(model, ids, n)
    per_step_phase = model.engine.launch_count - c0
    # the persistent kernel ran: one launch per decode step instead of 6 per layer + 2
    saved = per_step_phase - per_step_mega
    assert saved > 0 and saved % (6 * cfg.text_config.num_hidden_layers + 2 - 1) == 0, (per_step_phase, per_step_mega)
    model.engine.set_mega(1)
    tc, lc = _run(model, ids, n, prefill_step_size=16)   # windows of 16 + 16 + 9 tokens
    assert tc == t0 and all(torch.equal(a, b) for a, b in zip(lc, l0))
    assert torch.equal(_kv_rows(model, 41 + n - 1), kv0)


@pytest.mark.parametrize("kind", ["tiny", "hd128"])
def test_lock_step_rows_equal_single_requests(kind):
    from mlx_vlm_b200.generate_batch import BatchGenerator
    cfg, W, model = _model(kind)
    rng = np.random.default_rng(3)
    rows = [(rng.integers(0, cfg.text_config.vocab_size, size=(1, 7 + 5 * i)), 6 + 2 * i) for i in range(4)]
    want = [_run(model, ids, n) for ids, n in rows]
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    g = BatchGenerator(model, proc, completion_batch_size=4, prefill_batch_size=2, decode_slice=1)
    assert g._lockstep == (kind != "hd128")   # head_dim != hidden / heads: time-multiplexed rows
    uids = g.insert([r[0] for r in rows], [r[1] for r in rows], [{} for _ in rows])
    got = {u: [] for u in uids}
    while g.has_work:
        _, rs = g.next()
        for r in rs:
            got[r.uid].append(r.token)
    assert model.engine.device_error() == 0
    for u, (wt, wl) in zip(uids, want):
        assert len(got[u]) == len(wt)
        for i, (a, b) in enumerate(zip(got[u], wt)):
            if a != b:
                assert _token_ok(a, wl[i]), f"row {u} token {i}: batched {a} vs alone {b}"
                break


@pytest.mark.parametrize("kind", ["tiny", "hd128"])
def test_kv8_generation_runs_and_matches_before_the_switch(kind):
    cfg, W, model = _model(kind)
    ids = np.random.default_rng(4).integers(0, cfg.text_config.vocab_size, size=(1, 20))
    t0, l0 = _run(model, ids, 8)
    t8, l8 = _run(model, ids, 8, kv_bits=8, kv_group_size=64, quantized_kv_start=24)
    # positions 0..23 are cached in bf16: the steps before the conversion are the bf16 run's bits
    assert t8[:4] == t0[:4] and all(torch.equal(a, b) for a, b in zip(l8[:4], l0[:4]))
    for i in range(4, 8):
        if t8[i] != t0[i]:
            assert _token_ok(t8[i], l0[i])
            break
