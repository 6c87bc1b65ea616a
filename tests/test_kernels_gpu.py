"""GPU parity of each C-ABI op against the oracle's restatement (same seeded
inputs, sizes the oracle finishes in seconds).  Bar: see _util.cmp_bf16 —
relative L2 <= 1e-3 with the oracle's rounding points mirrored (most elements are
bit-identical; the rest differ by one bf16 ulp from fp32 summation order)."""
import math

import numpy as np
import pytest
import torch

from _util import cmp_bf16, to_dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from mlx_vlm_b200 import _native as N
    l = N.lib()
    sm = __import__("ctypes").c_int()
    N.check(l.b200_device_check(0, __import__("ctypes").byref(sm)), "device_check")
    return l


def R(dtype="bf16"):
    from oracle.mlx_semantics import Rounder
    return Rounder(dtype)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return R().r(torch.randn(*shape, generator=g) * scale)


@pytest.mark.parametrize("rows,dim", [(576, 1280), (3, 1536), (1, 256)])
def test_norms(lib, rows, dim):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    x = rnd(rows, dim, scale=2.0, seed=8)
    w = r.r(1.0 + 0.1 * torch.randn(dim, generator=torch.Generator().manual_seed(9)))
    b = rnd(dim, scale=0.1, seed=10)
    dx, dw, db = to_dev(x), to_dev(w), to_dev(b)
    y = torch.empty_like(dx)
    Nn.check(lib.b200_layer_norm(dx.data_ptr(), dw.data_ptr(), db.data_ptr(), y.data_ptr(), rows,
                                 dim, 1e-6, 0), "ln")
    torch.cuda.synchronize()
    cmp_bf16(y, S.layer_norm(r, x, w, b, 1e-6), "layer_norm")
    Nn.check(lib.b200_rms_norm(dx.data_ptr(), dw.data_ptr(), y.data_ptr(), rows, dim, 1e-6, 0), "rms")
    torch.cuda.synchronize()
    cmp_bf16(y, S.rms_norm(r, x, w, 1e-6), "rms_norm")


def test_cast(lib):
    from mlx_vlm_b200 import _native as Nn
    x = torch.randn(576 * 1176 + 3, generator=torch.Generator().manual_seed(11))
    dx = x.cuda()
    y = torch.empty(x.numel(), dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_cast_f32_bf16(dx.data_ptr(), y.data_ptr(), x.numel(), 0), "cast")
    torch.cuda.synchronize()
    assert torch.equal(y.cpu(), x.to(torch.bfloat16))


@pytest.mark.parametrize("Lq,S_,nh,nkv,hd,causal", [
    (576, 576, 16, 16, 80, 0),   # ViT block
    (272, 272, 12, 2, 128, 1),   # LM prefill
    (40, 300, 12, 2, 128, 1),    # chunk appended to an existing cache
    (17, 17, 4, 2, 64, 1),       # ragged tile
    (1, 33, 4, 4, 72, 0),
])
def test_attention(lib, Lq, S_, nh, nkv, hd, causal):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    q = rnd(1, nh, Lq, hd, seed=12)
    k = rnd(1, nkv, S_, hd, seed=13)
    v = rnd(1, nkv, S_, hd, seed=14)
    want = S.sdpa(r, q, k, v, hd ** -0.5, bool(causal))  # (1,nh,Lq,hd)
    dq = to_dev(q[0].transpose(0, 1))      # (Lq, nh, hd)
    dk, dv = to_dev(k[0]), to_dev(v[0])    # (nkv, S, hd)
    out = torch.zeros(Lq, nh * hd, dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_attention(dq.data_ptr(), nh * hd, hd, dk.data_ptr(), hd, S_ * hd,
                                dv.data_ptr(), hd, S_ * hd, out.data_ptr(), nh * hd, nh, nkv, hd,
                                Lq, S_, causal, float(hd ** -0.5), 0), "attention")
    torch.cuda.synchronize()
    cmp_bf16(out.view(Lq, nh, hd), want[0].transpose(0, 1), f"attention Lq={Lq} S={S_} hd={hd}")


def test_attention_two_pass_on_two_devices(lib):
    """b200_attention's two-pass kernel (head_dim 72: not a multiple of 16, so the tensor-core kernel declines) with
    S = 2048, i.e. 16 * 72 * 4 + 16 * 2048 * 2 = 70 KB of shared memory, on device 0 and then on device 1 of one
    process: the kernel's shared-memory limit is a per-device attribute, raised on each device it runs on"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    Lq, S_, nh, nkv, hd = 8, 2048, 4, 2, 72
    r = R()
    q = rnd(1, nh, Lq, hd, seed=40)
    k = rnd(1, nkv, S_, hd, seed=41)
    v = rnd(1, nkv, S_, hd, seed=42)
    want = S.sdpa(r, q, k, v, hd ** -0.5, False)[0].transpose(0, 1)
    for dev in (0, 1):
        with torch.cuda.device(dev):
            dq = to_dev(q[0].transpose(0, 1))
            dk, dv = to_dev(k[0]), to_dev(v[0])
            out = torch.zeros(Lq, nh * hd, dtype=torch.bfloat16, device="cuda")
            Nn.check(lib.b200_attention(dq.data_ptr(), nh * hd, hd, dk.data_ptr(), hd, S_ * hd, dv.data_ptr(), hd,
                                        S_ * hd, out.data_ptr(), nh * hd, nh, nkv, hd, Lq, S_, 0, float(hd ** -0.5),
                                        0), f"attention on device {dev}")
            torch.cuda.synchronize()
        cmp_bf16(out.view(Lq, nh, hd), want, f"two-pass attention on device {dev}")


def test_vision_rope(lib):
    from mlx_vlm_b200 import _native as Nn
    from oracle import qwen2vl as O
    cfg = O.qwen2_vl_2b()
    v = cfg.vision
    grid = [[1, 24, 24]]
    N, nh, hd = 576, v.num_heads, v.embed_dim // v.num_heads
    r = R()
    qkv = rnd(N, 3, nh, hd, seed=15)
    freqs = O.vision_rotary_freqs(grid, v)
    cos = torch.cos(freqs).repeat(1, 2)[:, None, :]
    sin = torch.sin(freqs).repeat(1, 2)[:, None, :]
    want = qkv.clone()
    for w in (0, 1):
        x = qkv[:, w]
        want[:, w] = r.r(x * cos + O._rotate_half(x) * sin)
    d = to_dev(qkv)
    pos = torch.from_numpy(O.rot_pos_ids(grid, v.spatial_merge_size).astype(np.int32)).cuda()
    dim = hd // 2
    inv = (1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))).cuda()
    Nn.check(lib.b200_vision_rope(d.data_ptr(), pos.data_ptr(), inv.data_ptr(), N, nh, hd, 0), "vrope")
    torch.cuda.synchronize()
    cmp_bf16(d, want, "vision_rope", max_mismatch=0.005)


def test_mrope_kv_write(lib):
    from mlx_vlm_b200 import _native as Nn
    from oracle import qwen2vl as O
    cfg = O.qwen2_vl_2b()
    t = cfg.text
    T, nh, nkv, hd, cap, ctx0 = 50, t.num_attention_heads, t.num_key_value_heads, 128, 256, 7
    r = R()
    rng = np.random.default_rng(0)
    pos = rng.integers(0, 900, size=(3, 1, T))
    qkv = rnd(T, (nh + 2 * nkv) * hd, seed=16)
    q = qkv[:, :nh * hd].reshape(1, T, nh, hd).transpose(1, 2)
    k = qkv[:, nh * hd:(nh + nkv) * hd].reshape(1, T, nkv, hd).transpose(1, 2)
    v = qkv[:, (nh + nkv) * hd:].reshape(1, T, nkv, hd).transpose(1, 2)
    cos, sin = O.mrope_cos_sin(t, pos, r)
    qe, ke = O.apply_mrope(r, q, k, cos, sin)
    d = to_dev(qkv)
    kc = torch.zeros(nkv, cap, hd, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    pos3 = torch.from_numpy(pos[:, 0].astype(np.int32)).cuda().contiguous()
    inv = (1.0 / (t.rope_theta ** (torch.arange(0, hd, 2).to(torch.float32) / hd))).cuda()
    sel = torch.from_numpy(O.mrope_selector(t.mrope_section, hd // 2).astype(np.int32)).cuda()
    Nn.check(lib.b200_mrope_kv_write(d.data_ptr(), pos3.data_ptr(), inv.data_ptr(), sel.data_ptr(),
                                     kc.data_ptr(), vc.data_ptr(), T, ctx0, cap, nh, nkv, hd, 0), "mrope")
    torch.cuda.synchronize()
    cmp_bf16(d[:, :nh * hd].view(T, nh, hd), qe[0].transpose(0, 1), "mrope q", max_mismatch=0.01)
    cmp_bf16(kc[:, ctx0:ctx0 + T], ke[0], "mrope k->cache", max_mismatch=0.01)
    assert torch.equal(vc[:, ctx0:ctx0 + T].cpu().float(), v[0]), "v copy must be exact"
    assert float(kc[:, :ctx0].abs().sum()) == 0 and float(kc[:, ctx0 + T:].abs().sum()) == 0


def test_swiglu(lib):
    from mlx_vlm_b200 import _native as Nn
    from oracle import mlx_semantics as S
    r = R()
    gu = rnd(37, 2 * 8960, scale=2.0, seed=17)
    want = S.swiglu(r, gu[:, :8960], gu[:, 8960:])
    d = to_dev(gu)
    out = torch.empty(37, 8960, dtype=torch.bfloat16, device="cuda")
    Nn.check(lib.b200_swiglu(d.data_ptr(), out.data_ptr(), 37, 8960, 0), "swiglu")
    torch.cuda.synchronize()
    cmp_bf16(out, want, "swiglu", max_mismatch=0.002)


@pytest.mark.parametrize("case", ["one_image", "two_images_batch2", "video_fallback", "text_only"])
def test_embed_merge_indices_bit_exact(lib, case):
    """integer indexing of merge_input_ids_with_image_features must be bit-exact."""
    from mlx_vlm_b200 import _native as Nn
    from oracle import qwen2vl as O
    cfg = O.tiny_cfg()
    H, V = 64, 1024
    img, vid = cfg.image_token_id, cfg.video_token_id
    rng = np.random.default_rng(3)
    if case == "one_image":
        ids = rng.integers(0, 900, size=(1, 40)); ids[0, 5:21] = img
    elif case == "two_images_batch2":
        ids = rng.integers(0, 900, size=(2, 33)); ids[0, 2:6] = img; ids[0, 20:28] = img; ids[1, 9:13] = img
    elif case == "video_fallback":
        ids = rng.integers(0, 900, size=(1, 25)); ids[0, 3:11] = vid
    else:
        ids = rng.integers(0, 900, size=(2, 19))
    want_src = O.merge_indices(cfg, ids)
    n_feats = int((want_src >= 0).sum())
    table = rnd(V, H, seed=18)
    feats = rnd(max(n_feats, 1), H, seed=19)
    B, T = ids.shape
    d_ids = torch.from_numpy(ids.astype(np.int32)).cuda()
    dt, df = to_dev(table), to_dev(feats)
    out = torch.zeros(B, T, H, dtype=torch.bfloat16, device="cuda")
    src = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    Nn.check(lib.b200_embed_merge(d_ids.data_ptr(), B, T, dt.data_ptr(), H, df.data_ptr(), n_feats,
                                  img, vid, out.data_ptr(), src.data_ptr(), 0), "embed_merge")
    torch.cuda.synchronize()
    assert np.array_equal(src.cpu().numpy().astype(np.int64), want_src)
    want = table[torch.from_numpy(ids)]
    if n_feats:
        want = O.merge_input_ids_with_image_features(cfg, feats[:n_feats], want, ids)
    assert torch.equal(out.cpu().float(), want), "merged embeddings are pure copies: bit-exact"
