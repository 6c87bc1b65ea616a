"""Thin Python face of the fp32-accurate tower ops (csrc/tower_f32.cu, gemm_wt.cu modes F32 / SPLIT).

Vocabulary: a *split operand* is an fp32 activation carried as two bf16 halves [hi | lo] in one
row (n_pad columns apart, n_pad = columns rounded up to 64): `SplitBuf`.  Weights are bf16 (exact),
so `linear()` = W.x_hi + W.x_lo on the tensor cores with fp32 accumulation; LayerNorm, residuals,
activations and attention are fp32.  torch is the memory container only.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _native as N

F32, SPLIT = 3, 4
EPI_NONE, EPI_GELU_FAST, EPI_GELU_EXACT, EPI_GELU_TANH = 0, 1, 2, 3


def pad64(n: int) -> int:
    return (n + 63) // 64 * 64


class SplitBuf:
    """[T, 2 * n_pad] bf16: hi half at columns [0, n), lo half at [n_pad, n_pad + n); padding is zero."""

    def __init__(self, eng, T: int, n: int):
        self.T, self.n, self.n_pad = T, n, pad64(n)
        with torch.cuda.stream(eng.stream):
            self.t = torch.zeros((T, 2 * self.n_pad), dtype=torch.bfloat16, device=eng.device)

    @property
    def ld(self) -> int:
        return 2 * self.n_pad


class TowerOps:
    def __init__(self, eng):
        self.eng = eng
        self.lib = eng.lib

    def f32(self, *shape) -> torch.Tensor:
        return self.eng.empty(shape, torch.float32)

    def layer_norm(self, x: torch.Tensor, w, b, eps: float, out32: Optional[torch.Tensor] = None,
                   out_split: Optional[SplitBuf] = None):
        T, n = x.shape
        N.check(self.lib.b200_f32_layer_norm(x.data_ptr(), x.stride(0), N.ptr(w), N.ptr(b), float(eps),
                                             N.ptr(out32), out32.stride(0) if out32 is not None else 0,
                                             N.ptr(out_split.t) if out_split else 0,
                                             out_split.ld if out_split else 0,
                                             out_split.n_pad if out_split else 0, T, n, self.eng.s), "f32_layer_norm")

    def rms_norm(self, x: torch.Tensor, w, eps: float, out32: Optional[torch.Tensor] = None,
                 out_split: Optional[SplitBuf] = None, seg_in: int = 0, seg_out: int = 0, seg_off: int = 0):
        T, n = x.shape
        N.check(self.lib.b200_f32_rms_norm(x.data_ptr(), x.stride(0), w.data_ptr(), float(eps), N.ptr(out32),
                                           out32.stride(0) if out32 is not None else 0,
                                           N.ptr(out_split.t) if out_split else 0, out_split.ld if out_split else 0,
                                           out_split.n_pad if out_split else 0, T, n, seg_in, seg_out, seg_off,
                                           self.eng.s), "f32_rms_norm")

    def swiglu(self, gu: torch.Tensor, out: SplitBuf):
        T = gu.shape[0]
        N.check(self.lib.b200_f32_swiglu_split(gu.data_ptr(), gu.stride(0), out.t.data_ptr(), out.ld, out.n_pad, T,
                                               out.n, self.eng.s), "f32_swiglu")

    def split(self, x: torch.Tensor, out: SplitBuf):
        T, n = x.shape
        N.check(self.lib.b200_f32_split(x.data_ptr(), x.stride(0), out.t.data_ptr(), out.ld, out.n_pad, T, n,
                                        self.eng.s), "f32_split")

    def linear(self, x: SplitBuf, w: torch.Tensor, bias, *, out32: Optional[torch.Tensor] = None,
               res32: Optional[torch.Tensor] = None, out_split: Optional[SplitBuf] = None, epi: int = EPI_NONE,
               k_w: Optional[int] = None, n_parts: int = 2):
        """y = act(W . x + bias) (+ res32): fp32 into `out32` or as a split operand into `out_split`.
        w: [N, ldw] bf16 with k_w valid columns (k_w defaults to x.n); n_parts = 1 reads only the hi half of x, i.e. the
        input rounded to bf16."""
        n_out = w.shape[0]
        k_w = x.n if k_w is None else k_w
        mode = F32 if out32 is not None else SPLIT
        N.check(self.lib.b200_gemm_wt_f32(
            x.t.data_ptr(), x.ld, w.data_ptr(), w.stride(0), N.ptr(bias), N.ptr(res32),
            res32.stride(0) if res32 is not None else 0, N.ptr(out32), out32.stride(0) if out32 is not None else 0,
            N.ptr(out_split.t) if out_split else 0, out_split.ld if out_split else 0,
            out_split.n_pad if out_split else 0, x.T, n_out, k_w, n_parts, epi, mode, None, self.eng.s), "gemm_wt_f32")

    def attention(self, q, k, v, *, n_heads: int, n_kv: int, hd: int, Lq: int, S: int, n_seg: int, q_seg: int,
                  k_seg: int, scale: float, out32: Optional[torch.Tensor] = None, out_split: Optional[SplitBuf] = None,
                  key_mask: Optional[torch.Tensor] = None):
        """q/k/v: (tensor, token stride, head stride) views into fp32 buffers"""
        (qt, q_ts, q_hs), (kt, k_ts, k_hs), (vt, v_ts, v_hs) = q, k, v
        N.check(self.lib.b200_attention_f32(
            qt.data_ptr(), q_ts, q_hs, kt.data_ptr(), k_ts, k_hs, vt.data_ptr(), v_ts, v_hs, N.ptr(out32),
            out32.stride(0) if out32 is not None else 0, N.ptr(out_split.t) if out_split else 0,
            out_split.ld if out_split else 0, out_split.n_pad if out_split else 0, n_heads, n_kv, hd, Lq, S, n_seg,
            q_seg, k_seg, N.ptr(key_mask), float(scale), self.eng.s), "attention_f32")

    def attention_varlen(self, q, k, v, *, n_heads: int, n_kv: int, hd: int, cu: torch.Tensor, n_seg: int, max_len: int,
                         scale: float, out32: Optional[torch.Tensor] = None, out_split: Optional[SplitBuf] = None):
        """self-attention inside each ragged segment [cu[z], cu[z+1]) (cu: device int32)"""
        (qt, q_ts, q_hs), (kt, k_ts, k_hs), (vt, v_ts, v_hs) = q, k, v
        N.check(self.lib.b200_attention_f32_varlen(
            qt.data_ptr(), q_ts, q_hs, kt.data_ptr(), k_ts, k_hs, vt.data_ptr(), v_ts, v_hs, N.ptr(out32),
            out32.stride(0) if out32 is not None else 0, N.ptr(out_split.t) if out_split else 0,
            out_split.ld if out_split else 0, out_split.n_pad if out_split else 0, n_heads, n_kv, hd, cu.data_ptr(),
            n_seg, max_len, float(scale), self.eng.s), "attention_f32_varlen")

    def vision_rope(self, qkv: torch.Tensor, pos_hw: torch.Tensor, inv_freq: torch.Tensor, n_heads: int, hd: int):
        N.check(self.lib.b200_f32_vision_rope(qkv.data_ptr(), qkv.stride(0), pos_hw.data_ptr(), inv_freq.data_ptr(),
                                              qkv.shape[0], n_heads, hd, self.eng.s), "f32_vision_rope")

    def gather_rows(self, x: torch.Tensor, idx: torch.Tensor, unit: int, out: torch.Tensor):
        N.check(self.lib.b200_f32_gather_rows(x.data_ptr(), x.stride(0), idx.data_ptr(), idx.numel(), unit, x.shape[1],
                                              out.data_ptr(), out.stride(0), self.eng.s), "f32_gather_rows")

    def pixel_shuffle(self, x: torch.Tensor, n_img: int, side: int, s: int, out: SplitBuf, round_in: bool = True):
        E = x.shape[-1]
        N.check(self.lib.b200_pixel_shuffle_split(x.data_ptr(), n_img, side, E, s, int(round_in), out.t.data_ptr(), out.ld,
                                                  out.n_pad, self.eng.s), "pixel_shuffle_split")

    def patchify(self, pix_nhwc: torch.Tensor, ps: int, out: SplitBuf):
        B, H, W, C = pix_nhwc.shape
        N.check(self.lib.b200_clip_patchify(pix_nhwc.data_ptr(), B, H, W, C, ps, out.t.data_ptr(), out.n_pad,
                                            self.eng.s), "clip_patchify")

    def embed(self, patch: torch.Tensor, cls, pos: torch.Tensor, pos_ids, emb: torch.Tensor, B: int, P: int):
        E = patch.shape[1]
        N.check(self.lib.b200_tower_embed(patch.data_ptr(), N.ptr(cls), pos.data_ptr(), N.ptr(pos_ids), emb.data_ptr(),
                                          B, P, E, pos.shape[0], self.eng.s), "tower_embed")


# ---------------------------------------------------------------- the CLIP / SigLIP encoder of LLaVA and Idefics
def sanitize(weights, num_channels: int):
    """reference clip / siglip `sanitize`: `position_ids` buffers are dropped and a PyTorch patch conv
    [O, C, kH, kW] becomes channels-last [O, kH, kW, C]"""
    out = {}
    for k, v in weights.items():
        if "position_ids" in k:
            continue
        if "patch_embedding.weight" in k and v.ndim == 4 and v.shape[1] == num_channels and v.shape[-1] != num_channels:
            v = v.permute(0, 2, 3, 1)
        out[k] = v
    return out


def pack_encoder_layers(weights, prefix: str, n_layers: int, put):
    """`{prefix}encoder.layers.{i}.*` -> the tower weights `{i}.*` (q/k/v rows and biases fused) through `put`"""
    for i in range(n_layers):
        q = prefix + f"encoder.layers.{i}."
        put(f"{i}.ln1.w", weights[q + "layer_norm1.weight"]); put(f"{i}.ln1.b", weights[q + "layer_norm1.bias"])
        put(f"{i}.ln2.w", weights[q + "layer_norm2.weight"]); put(f"{i}.ln2.b", weights[q + "layer_norm2.bias"])
        put(f"{i}.qkv.w", torch.cat([weights[q + f"self_attn.{n}_proj.weight"] for n in "qkv"], 0))
        put(f"{i}.qkv.b", torch.cat([weights[q + f"self_attn.{n}_proj.bias"] for n in "qkv"], 0))
        put(f"{i}.out.w", weights[q + "self_attn.out_proj.weight"]); put(f"{i}.out.b", weights[q + "self_attn.out_proj.bias"])
        put(f"{i}.fc1.w", weights[q + "mlp.fc1.weight"]); put(f"{i}.fc1.b", weights[q + "mlp.fc1.bias"])
        put(f"{i}.fc2.w", weights[q + "mlp.fc2.weight"]); put(f"{i}.fc2.b", weights[q + "mlp.fc2.bias"])


def encoder(ops: TowerOps, w, h: torch.Tensor, n_layers: int, *, n_heads: int, inter: int, seg: int, eps: float,
            epi: int):
    """encoder layers 0 .. n_layers - 1, in place on the fp32 residual stream h (T, E) of T / seg images of seg tokens
    each: LN -> qkv -> attention inside each image -> out + residual -> LN -> fc1 with the activation epilogue `epi`
    -> fc2 + residual"""
    eng = ops.eng
    T, E = h.shape
    hd = E // n_heads
    y, o, mlp = SplitBuf(eng, T, E), SplitBuf(eng, T, E), SplitBuf(eng, T, inter)
    qkv = ops.f32(T, 3 * E)
    for i in range(n_layers):
        ops.layer_norm(h, w[f"{i}.ln1.w"], w[f"{i}.ln1.b"], eps, out_split=y)
        ops.linear(y, w[f"{i}.qkv.w"], w[f"{i}.qkv.b"], out32=qkv)
        ops.attention((qkv, 3 * E, hd), (qkv[:, E:], 3 * E, hd), (qkv[:, 2 * E:], 3 * E, hd), n_heads=n_heads,
                      n_kv=n_heads, hd=hd, Lq=seg, S=seg, n_seg=T // seg, q_seg=seg, k_seg=seg, scale=hd ** -0.5,
                      out_split=o)
        ops.linear(o, w[f"{i}.out.w"], w[f"{i}.out.b"], out32=h, res32=h)
        ops.layer_norm(h, w[f"{i}.ln2.w"], w[f"{i}.ln2.b"], eps, out_split=y)
        ops.linear(y, w[f"{i}.fc1.w"], w[f"{i}.fc1.b"], out_split=mlp, epi=epi)
        ops.linear(mlp, w[f"{i}.fc2.w"], w[f"{i}.fc2.b"], out32=h, res32=h)
