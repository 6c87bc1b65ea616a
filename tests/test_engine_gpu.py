"""GPU parity of the whole generate path (vision tower -> merge -> rope index ->
prefill -> decode -> greedy sampling) against the oracle on the same seeded
weights and inputs, through the reference-shaped Python surface
(Model.get_input_embeddings / language_model / generate_step) which calls the C ABI.

Bars
  * integer outputs (merge indices, position ids, rope deltas, cache offsets):
    bit-exact;
  * stages whose INPUTS are identical to the oracle's (one decoder layer fed the
    oracle's hidden state, the fused head fed the oracle's final hidden state):
    relative L2 <= 1e-3 (the north star's bar);
  * deep end-to-end outputs (ViT features after 32 blocks, logits after 28
    layers): `_util.cmp_noise` — a bf16 pipeline is chaotic (see its docstring), so
    the CUDA path must be no further from the oracle's bf16 result than that
    result is from the exact fp32 evaluation;
  * greedy token ids: equal to the oracle's whenever the oracle's top-2 logprob
    margin exceeds two bf16 ulps.
"""
import numpy as np
import pytest
import torch

from _util import cmp_bf16, cmp_noise, rl2

pytestmark = pytest.mark.gpu


def _mk_cfg(kind):
    from oracle import qwen2vl as O
    if kind == "tiny":
        return O.tiny_cfg()
    if kind == "tiny1":  # one decoder layer / one ViT block: no deep cascade
        c = O.tiny_cfg()
        c.text.num_hidden_layers = 1
        c.vision.depth = 1
        return c
    if kind == "wide1":  # real Qwen2-VL-2B widths, 1 LM layer + 1 ViT block
        c = O.qwen2_vl_2b()
        c.text.num_hidden_layers = 1
        c.vision.depth = 1
        return c
    if kind == "wide2":
        c = O.qwen2_vl_2b()
        c.text.num_hidden_layers = 2
        c.vision.depth = 2
        return c
    if kind == "mha32":  # 32 kv heads (Llama-7B-like MHA): more attention CTAs than SMs -> the
        c = O.tiny_cfg()  # persistent kernel does not fit and the engine falls back per phase
        c.text.hidden_size, c.text.num_attention_heads, c.text.num_key_value_heads = 2048, 32, 32
        c.text.intermediate_size, c.text.num_hidden_layers = 512, 1
        c.text.mrope_section = (8, 12, 12)
        c.vision.hidden_size = 2048
        c.vision.depth = 1
        return c
    if kind == "oddvocab":  # vocabulary that is not a multiple of 8 (Idefics2's is 32003)
        c = O.tiny_cfg()
        c.text.vocab_size += 3
        return c
    if kind == "full":
        return O.qwen2_vl_2b()
    raise ValueError(kind)


def _to_model_config(c):
    from mlx_vlm_b200.models.qwen2_vl.config import ModelConfig, TextConfig, VisionConfig
    t, v = c.text, c.vision
    text = TextConfig(model_type="qwen2_vl", hidden_size=t.hidden_size,
                      num_hidden_layers=t.num_hidden_layers, intermediate_size=t.intermediate_size,
                      num_attention_heads=t.num_attention_heads, rms_norm_eps=t.rms_norm_eps,
                      vocab_size=t.vocab_size, num_key_value_heads=t.num_key_value_heads,
                      rope_theta=t.rope_theta,
                      rope_scaling={"type": "mrope", "mrope_section": list(t.mrope_section)},
                      tie_word_embeddings=t.tie_word_embeddings)
    vis = VisionConfig(depth=v.depth, embed_dim=v.embed_dim, hidden_size=v.hidden_size,
                       num_heads=v.num_heads, patch_size=v.patch_size, mlp_ratio=v.mlp_ratio,
                       spatial_merge_size=v.spatial_merge_size,
                       temporal_patch_size=v.temporal_patch_size)
    return ModelConfig(text_config=text, vision_config=vis, model_type="qwen2_vl",
                       image_token_id=c.image_token_id, video_token_id=c.video_token_id,
                       vision_start_token_id=c.vision_start_token_id, vocab_size=t.vocab_size)


def _build(kind, n_text, hw, seed=0, jitter=0.05):
    from mlx_vlm_b200.models.qwen2_vl import Model
    from oracle import qwen2vl as O
    c = _mk_cfg(kind)
    W = O.init_weights(c, seed, norm_jitter=jitter)
    model = Model(_to_model_config(c), device="cuda:0")
    model.load_weights(W)
    req = O.synthetic_request(c, n_text, image_hw=hw, seed=seed)
    return c, W, model, req


def _token_ok(tok, oracle_lp):
    """greedy token acceptable: its oracle logprob is within 2 bf16 ulps of the max."""
    m = float(oracle_lp.max())
    tol = 2 * abs(m) * 2.0 ** -7 + 1e-6
    return float(oracle_lp[tok]) >= m - tol


@pytest.mark.parametrize("kind,n_text,hw", [("tiny1", 12, (56, 84)), ("wide1", 32, (112, 112))])
def test_shallow_stages_identical_inputs(kind, n_text, hw):
    """One ViT block + merger, one decoder layer + head.  The K/V cache (RMSNorm ->
    QKV GEMM -> M-RoPE on the oracle's own embeddings) is held to the 1e-3 bar; the
    outputs further down the layer to the noise-relative bar."""
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    c, W, model, req = _build(kind, n_text, hw)
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    eng = model.engine
    ref = O.greedy_generate(c, W, ids, pv, grid, 3)
    toks = ref["tokens"][0].tolist()
    ex = O.greedy_generate(c, W, ids, pv, grid, 3, dtype="f32", force_tokens=toks)
    pre, pre32 = ref["prefill"], ex["prefill"]
    pvd = torch.from_numpy(pv).cuda()
    feats = model.vision_tower(pvd, grid)
    eng.stream.synchronize()
    cmp_noise(feats, pre.image_features, pre32.image_features, f"{kind} vision features (1 block)")
    # LM fed the ORACLE's merged embeddings -> identical inputs
    emb_or = pre.inputs_embeds.to(device="cuda", dtype=torch.bfloat16)
    cache = make_prompt_cache(model.language_model)
    out = model.language_model(ids, inputs_embeds=emb_or, cache=cache,
                               position_ids=pre.position_ids, rope_deltas=pre.rope_deltas)
    eng.stream.synchronize()
    T = ids.shape[1]
    cmp_bf16(cache[0].keys[0, :, :T], ref["cache"][0].keys[0, :, :T], f"{kind} K cache",
             rel_l2=1e-3, max_mismatch=0.02)
    cmp_bf16(cache[0].values[0, :, :T], ref["cache"][0].values[0, :, :T], f"{kind} V cache",
             rel_l2=1e-3, max_mismatch=0.02)
    cmp_noise(out.logits[0, -1], pre.logits_last[0], pre32.logits_last[0], f"{kind} prefill logits")
    cmp_noise(eng.logits_view(), pre.logits_last[0], pre32.logits_last[0], f"{kind} fused-head logits")
    # decode steps, teacher forced
    delta = int(pre.rope_deltas[0, 0])
    eng.set_next(toks[0], T, T + delta)
    for n in range(1, 3):
        eng.decode(1, force_tokens=np.asarray([toks[n]], dtype=np.int32))
        eng.stream.synchronize()
        cmp_noise(eng.logits_view(), ref["logits"][n][0], ex["logits"][n][0],
                  f"{kind} decode step {n} logits")


@pytest.mark.parametrize("kind,n_text,hw,n_dec", [("tiny", 12, (56, 84), 12),
                                                   ("wide2", 32, (112, 112), 8)])
def test_generate_path_parity(kind, n_text, hw, n_dec):
    from mlx_vlm_b200.generate import generate_step
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    c, W, model, req = _build(kind, n_text, hw)
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    eng = model.engine
    ref = O.greedy_generate(c, W, ids, pv, grid, n_dec)
    toks = ref["tokens"][0].tolist()
    ex = O.greedy_generate(c, W, ids, pv, grid, n_dec, dtype="f32", force_tokens=toks[:])
    pre, pre32 = ref["prefill"], ex["prefill"]
    # ---------------- vision tower
    pvd = torch.from_numpy(pv).cuda()
    feats = model.vision_tower(pvd, grid)
    eng.stream.synchronize()
    cmp_noise(feats, pre.image_features, pre32.image_features, f"{kind} vision features")
    # ---------------- input embeddings: merge indexing, rope index (bit-exact)
    emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
    eng.stream.synchronize()
    assert np.array_equal(np.asarray(emb.position_ids), pre.position_ids)
    assert np.array_equal(np.asarray(emb.rope_deltas), pre.rope_deltas)
    src = O.merge_indices(c, ids)[0]
    e = emb.inputs_embeds[0].float().cpu()
    table = W["language_model.model.embed_tokens.weight"]
    text_rows = np.where(src < 0)[0]
    assert torch.equal(e[text_rows], table[torch.from_numpy(ids[0][text_rows])])
    img_rows = np.where(src >= 0)[0]
    assert torch.equal(e[img_rows], feats.float().cpu()[torch.from_numpy(src[img_rows])]), \
        "image rows must be exact copies of the feature rows selected by cumsum(mask)-1"
    # ---------------- prefill: all-row logits through LanguageModel.__call__
    cache = make_prompt_cache(model.language_model)
    out = model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=cache,
                               position_ids=emb.position_ids, rope_deltas=emb.rope_deltas)
    eng.stream.synchronize()
    T = ids.shape[1]
    assert out.logits.shape == (1, T, c.text.vocab_size) and cache[0].offset == T
    cmp_noise(out.logits[0, -1], pre.logits_last[0], pre32.logits_last[0], f"{kind} prefill logits")
    cmp_noise(eng.logits_view(), pre.logits_last[0], pre32.logits_last[0], f"{kind} fused head")
    assert rl2(eng.logits_view(), out.logits[0, -1]) <= 1e-3, "GEMM head vs fused GEMV head"
    # ---------------- decode, teacher-forced with the oracle's tokens
    delta = int(pre.rope_deltas[0, 0])
    eng.set_next(toks[0], T, T + delta)
    for n in range(1, n_dec):
        eng.decode(1, force_tokens=np.asarray([toks[n]], dtype=np.int32))
        eng.stream.synchronize()
        cmp_noise(eng.logits_view(), ref["logits"][n][0], ex["logits"][n][0],
                  f"{kind} decode step {n} logits")
    # ---------------- free-running greedy through generate_step (public API)
    got = []
    for tok, lp in generate_step(ids, model, pvd, None, max_tokens=n_dec, image_grid_thw=grid):
        got.append(tok)
        n = len(got) - 1
        assert _token_ok(tok, ref["logprobs"][n][0]), f"token {n}: got {tok}, oracle {toks[n]}"
        if tok != toks[n]:
            break  # a (near-)tie: histories legitimately diverge from here
    print(f"{kind}: tokens {got} oracle {toks}")
    assert eng.device_error() == 0


def test_multi_kernel_decode_equals_megakernel():
    """The per-phase kernels (decode.cu) and the persistent megakernel
    (decode_mega.cu) share device code and tile geometry: same tokens, same logits."""
    from mlx_vlm_b200.generate import generate_step
    c, W, model, req = _build("wide2", 16, (56, 56))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    pvd = torch.from_numpy(pv).cuda()
    eng = model.engine
    runs = []
    for mega in (True, False):
        eng.set_mega(mega)
        toks, lps = [], []
        for tok, lp in generate_step(ids, model, pvd, None, max_tokens=6, image_grid_thw=grid):
            toks.append(tok)
            lps.append(lp.float().cpu())
        err = eng.device_error()
        assert err == 0, f"device error flag {err} (mega={mega})"
        runs.append((toks, lps))
    eng.set_mega(True)
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert rl2(a, b) <= 1e-3


@pytest.mark.parametrize("kind,mode", [("tiny", 2), ("wide2", 2), ("wide2", 3), ("tiny", 4), ("wide2", 4)])
def test_tensor_core_megakernel_parity(kind, mode):
    """Alternative decode-step kernels — k_mega_tc (modes 2/3; decode_mega_tc.cu: wgmma GEMV
    phases on pre-packed weight tile images, exact fixed-point split-K accumulation) and k_mega
    in dataflow mode (mode 4: polled self-validating activation words) — against the oracle, teacher-forced, and against
    k_mega on the same cache; the appended K/V rows of layer 0 must be bit-identical (same
    inputs, one Linear + rotary, fp32 accumulation differences stay below one bf16 ulp almost
    everywhere)."""
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    n_dec = 5
    c, W, model, req = _build(kind, 16, (56, 56))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    eng = model.engine
    ref = O.greedy_generate(c, W, ids, pv, grid, n_dec)
    toks = ref["tokens"][0].tolist()
    ex = O.greedy_generate(c, W, ids, pv, grid, n_dec, dtype="f32", force_tokens=toks[:])
    pvd = torch.from_numpy(pv).cuda()
    T = ids.shape[1]
    delta = int(ref["prefill"].rope_deltas[0, 0])
    got = {}
    try:
        for m in (1, mode):
            eng.set_mega(m)
            cache = make_prompt_cache(model.language_model)
            emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
            model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=cache,
                                 position_ids=emb.position_ids, rope_deltas=emb.rope_deltas)
            eng.set_next(toks[0], T, T + delta)
            logs = []
            for n in range(1, n_dec):
                eng.decode(1, force_tokens=np.asarray([toks[n]], dtype=np.int32))
                eng.stream.synchronize()
                logs.append(eng.logits_view().float().cpu().clone())
                if m == mode:
                    cmp_noise(logs[-1], ref["logits"][n][0], ex["logits"][n][0],
                              f"{kind} k_mega_tc (mode {mode}) decode step {n} logits")
            assert eng.device_error() == 0, f"device error flag (mode {m})"
            got[m] = (logs, cache[0].keys[0, :, T:T + n_dec - 1].float().cpu().clone(),
                      cache[0].values[0, :, T:T + n_dec - 1].float().cpu().clone())
    finally:
        eng.set_mega(1)
    for a, b in zip(got[1][0], got[mode][0]):
        assert rl2(a, b) <= 2e-2, "k_mega_tc vs k_mega logits"
    cmp_bf16(got[mode][1], got[1][1], f"{kind} appended K rows, layer 0", rel_l2=1e-3, max_mismatch=0.02)
    cmp_bf16(got[mode][2], got[1][2], f"{kind} appended V rows, layer 0", rel_l2=1e-3, max_mismatch=0.02)


def test_batch_generator_rows_equal_single_requests():
    """Continuous batching (SURVEY §8 a15) on the real engine: three requests (two with an
    image, different lengths / max_tokens) time-multiplexed through BatchGenerator produce
    exactly the tokens each produces alone through generate_step."""
    import types
    from mlx_vlm_b200.generate import generate_step
    from mlx_vlm_b200.generate_batch import BatchGenerator
    c, W, model, req = _build("tiny", 10, (56, 56))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    pvd = torch.from_numpy(pv).cuda()
    rng = np.random.default_rng(3)
    text_ids = rng.integers(0, 900, size=(1, 23))
    rows = [(ids, {"pixel_values": pvd, "image_grid_thw": grid}, 9),
            (text_ids, {}, 14),
            (ids[:, :ids.shape[1]], {"pixel_values": pvd, "image_grid_thw": grid}, 5)]
    want = []
    for r_ids, kw, m in rows:
        toks = [t for t, _ in generate_step(r_ids, model, kw.get("pixel_values"), None, max_tokens=m,
                                            image_grid_thw=kw.get("image_grid_thw"))]
        want.append(toks)
    model.config.eos_token_id = []
    proc = types.SimpleNamespace(tokenizer=types.SimpleNamespace(stopping_criteria=None))
    for slice_ in (1, 4):
        g = BatchGenerator(model, proc, completion_batch_size=2, prefill_batch_size=2, decode_slice=slice_)
        uids = g.insert([r[0] for r in rows], [r[2] for r in rows], [r[1] for r in rows])
        got = {u: [] for u in uids}
        while g.has_work:
            _, rs = g.next()
            for r in rs:
                got[r.uid].append(r.token)
        assert model.engine.device_error() == 0
        for u, w in zip(uids, want):
            assert got[u] == w, (slice_, u, got[u], w)


@pytest.mark.parametrize("sizes", [((56, 84), (84, 56)), ((84, 84), (56, 56))])
def test_two_images_of_different_size_in_one_prompt(sizes):
    """Multi-image request (the case of the reference's TestMultiImageMRoPE, test_models.py:11866):
    two images with different grids -> per-image (block-diagonal) vision attention, features
    concatenated, merge by cumsum(mask)-1, position ids / delta bit-exact, prefill logits in noise.
    The second case starts its second image at patch 36 (not a multiple of 8): the pipelined attention
    kernel cannot load V^T tiles there and the tower must take the fallback kernel."""
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    c, W, model, _ = _build("tiny", 8, (56, 56))
    eng = model.engine
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, size=(3,) + sizes[0], dtype=np.uint8),
            rng.integers(0, 256, size=(3,) + sizes[1], dtype=np.uint8)]
    pvs, grids = zip(*[O.preprocess_image(im, c.vision) for im in imgs])
    pv = np.concatenate(pvs, axis=0)
    grid = np.asarray(grids, dtype=np.int64)
    text = rng.integers(0, 900, size=12).tolist()
    ids = text[:3] + [c.vision_start_token_id, c.image_token_id, c.vision_end_token_id] + text[3:7] + \
        [c.vision_start_token_id, c.image_token_id, c.vision_end_token_id] + text[7:]
    ids = np.asarray([O.expand_image_tokens(ids, grids, c)], dtype=np.int64)
    ref = O.greedy_generate(c, W, ids, pv, grid, 2)
    ex = O.greedy_generate(c, W, ids, pv, grid, 2, dtype="f32", force_tokens=ref["tokens"][0].tolist())
    pre, pre32 = ref["prefill"], ex["prefill"]
    pvd = torch.from_numpy(pv).cuda()
    feats = model.vision_tower(pvd, grid)
    eng.stream.synchronize()
    assert feats.shape[0] == int(sum(np.prod(g) for g in grids)) // 4
    cmp_noise(feats, pre.image_features, pre32.image_features, "two-image vision features")
    emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
    eng.stream.synchronize()
    assert np.array_equal(np.asarray(emb.position_ids), pre.position_ids)
    assert np.array_equal(np.asarray(emb.rope_deltas), pre.rope_deltas)
    src = O.merge_indices(c, ids)[0]
    img_rows = np.where(src >= 0)[0]
    e = emb.inputs_embeds[0].float().cpu()
    assert torch.equal(e[img_rows], feats.float().cpu()[torch.from_numpy(src[img_rows])])
    cache = make_prompt_cache(model.language_model)
    out = model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=cache,
                               position_ids=emb.position_ids, rope_deltas=emb.rope_deltas)
    eng.stream.synchronize()
    cmp_noise(out.logits[0, -1], pre.logits_last[0], pre32.logits_last[0], "two-image prefill logits")


def test_geometry_that_does_not_fit_the_persistent_kernel_falls_back_per_phase():
    """32 kv heads x 8 key ranges > 132 SMs: k_mega cannot hold the step; the engine must run the
    same step as per-phase kernels (still the CUDA path) and stay in parity with the oracle."""
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    c, W, model, req = _build("mha32", 10, (56, 56))
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    eng = model.engine
    n_dec = 4
    ref = O.greedy_generate(c, W, ids, pv, grid, n_dec)
    toks = ref["tokens"][0].tolist()
    ex = O.greedy_generate(c, W, ids, pv, grid, n_dec, dtype="f32", force_tokens=toks[:])
    pvd = torch.from_numpy(pv).cuda()
    cache = make_prompt_cache(model.language_model)
    emb = model.get_input_embeddings(ids, pvd, image_grid_thw=grid)
    model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=cache,
                         position_ids=emb.position_ids, rope_deltas=emb.rope_deltas)
    T = ids.shape[1]
    eng.set_next(toks[0], T, T + int(ref["prefill"].rope_deltas[0, 0]))
    launches0 = eng.launch_count
    for n in range(1, n_dec):
        eng.decode(1, force_tokens=np.asarray([toks[n]], dtype=np.int32))
        eng.stream.synchronize()
        cmp_noise(eng.logits_view(), ref["logits"][n][0], ex["logits"][n][0], f"mha32 decode step {n}")
    assert eng.device_error() == 0
    per_step = (eng.launch_count - launches0) / (n_dec - 1)
    assert per_step > 2, f"expected the per-phase path (several launches per step), got {per_step}"


def test_text_only_and_cache_reuse():
    """text-only request (qwen2_vl.py:34-42) + chunked prefill == one-shot prefill
    (reference tests/cache_invariants.py:47-115)."""
    from mlx_vlm_b200.models.cache import make_prompt_cache
    from oracle import qwen2vl as O
    c, W, model, _ = _build("tiny", 8, (56, 56))
    eng = model.engine
    rng = np.random.default_rng(5)
    ids = rng.integers(0, 900, size=(1, 37))
    emb = model.get_input_embeddings(ids, None)
    assert np.asarray(emb.position_ids).shape == (1, 37)
    assert int(np.asarray(emb.rope_deltas)[0, 0]) == 0
    ref = O.greedy_generate(c, W, ids, None, None, 1)
    ex = O.greedy_generate(c, W, ids, None, None, 1, dtype="f32")
    c1 = make_prompt_cache(model.language_model)
    o1 = model.language_model(ids, inputs_embeds=emb.inputs_embeds, cache=c1,
                              position_ids=emb.position_ids)
    eng.stream.synchronize()
    cmp_noise(o1.logits[0, -1], ref["prefill"].logits_last[0], ex["prefill"].logits_last[0],
              "text-only logits")
    # chunked: 20 + 17 — same kernels on the same data => bit-identical to one-shot
    c2 = make_prompt_cache(model.language_model)
    model.language_model(ids[:, :20], inputs_embeds=emb.inputs_embeds[:, :20], cache=c2,
                         position_ids=emb.position_ids)
    o2 = model.language_model(ids[:, 20:], inputs_embeds=emb.inputs_embeds[:, 20:], cache=c2,
                              position_ids=emb.position_ids)
    eng.stream.synchronize()
    assert c2[0].offset == 37
    d = rl2(o2.logits[0, -1], o1.logits[0, -1])
    print(f"chunked vs one-shot prefill rel_l2={d:.3e}")
    assert d <= 1e-3
    cmp_bf16(c2[0].keys[0, :, :37], c1[0].keys[0, :, :37].float().cpu(), "chunked K cache layer 0",
             max_mismatch=0.0)


def test_merge_count_mismatch_raises():
    from mlx_vlm_b200.models.qwen2_vl import Model
    c, W, model, req = _build("tiny", 8, (56, 56))
    feats = torch.zeros(3, c.text.hidden_size, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="does not match"):
        Model.merge_input_ids_with_image_features(c.image_token_id, c.video_token_id, feats, None,
                                                  req["input_ids"], _engine=model.engine)


def test_full_size_c1():
    """BASELINE config C1: Qwen2-VL-2B shapes, 1 image 336x336, 32 text tokens (+144
    image tokens), 64 greedy tokens — oracle (CPU) vs CUDA path."""
    from mlx_vlm_b200.generate import generate_step
    from oracle import qwen2vl as O
    c, W, model, req = _build("full", 32, (336, 336), jitter=0.0)
    ids, pv, grid = req["input_ids"], req["pixel_values"], req["image_grid_thw"]
    assert ids.shape[1] == 32 + 144
    n_dec = 64
    ref = O.greedy_generate(c, W, ids, pv, grid, n_dec, keep_logits=True)
    toks = ref["tokens"][0].tolist()
    ex = O.greedy_generate(c, W, ids, pv, grid, 4, dtype="f32", force_tokens=toks[:])
    pvd = torch.from_numpy(pv).cuda()
    got, lps = [], []
    for tok, lp in generate_step(ids, model, pvd, None, max_tokens=n_dec, image_grid_thw=grid):
        got.append(tok)
        lps.append(lp)
    for n in range(n_dec):
        assert _token_ok(got[n], ref["logprobs"][n][0]), f"token {n}: {got[n]} vs {toks[n]}"
        if got[n] != toks[n]:
            break
        if n < 4:
            cmp_noise(lps[n], ref["logprobs"][n][0], ex["logprobs"][n][0], f"C1 logprobs step {n}")
        else:
            d = rl2(lps[n], ref["logprobs"][n][0])
            assert d <= 2e-2, f"C1 step {n}: logprobs rel-L2 {d:.3e}"
    print(f"C1: tokens equal to the oracle's: {got == toks}; first 8 {got[:8]} vs {toks[:8]}")
