"""Python handle of the native Qwen2-VL engine (C ABI in include/b200vlm.h).

Holds the torch tensors (weights, workspace, KV pool) whose device pointers the
native engine references — torch is the memory container only; every arithmetic
step is a kernel in libb200vlm.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _native as N
from .models.cache import BATCH_LOG_STEPS, BatchKVQPool, QuantizedKVPool


def _inv_freq(dim: int, base: float) -> np.ndarray:
    """compute_inv_freq (reference rope_utils.py:1042-1044), fp32."""
    t = 1.0 / (base ** (torch.arange(0, dim, 2).to(torch.float32) / dim))
    return t.numpy().astype(np.float32)


class Engine:
    def __init__(self, cfg: N.Qwen2VLConfig, device: torch.device):
        if device.type != "cuda":
            raise N.B200Error("the b200vlm engine needs a CUDA (sm_90a) device; no CPU fallback")
        self.lib = N.lib()
        self.cfg = cfg
        self.device = device
        self.index = device.index if device.index is not None else torch.cuda.current_device()
        h = C.c_void_p()
        N.check(self.lib.b200_engine_create(C.byref(cfg), self.index, C.byref(h)), "engine_create")
        self.h = h
        self.weights: Dict[str, torch.Tensor] = {}
        self.workspace: Optional[torch.Tensor] = None
        self._ws_tokens = 0
        self._ws_patches = 0
        self._bound = (None, -1)
        # rope tables computed with the reference's own formula on the host
        lm = _inv_freq(cfg.head_dim, cfg.rope_theta)
        vhd = cfg.v_embed // cfg.v_heads
        v = (1.0 / (10000.0 ** (torch.arange(0, vhd // 2, 2, dtype=torch.float32) / (vhd // 2))))
        v = v.numpy().astype(np.float32)
        N.check(self.lib.b200_engine_set_rope_tables(self.h, lm.ctypes.data, v.ctypes.data),
                "set_rope_tables")
        # a dedicated stream (the reference's `generation_stream`, generate/common.py:32)
        self.stream = torch.cuda.Stream(device=device)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.b200_engine_destroy(self.h)
                self.h = None
        except Exception:
            pass

    @property
    def s(self) -> int:
        return self.stream.cuda_stream

    def empty(self, shape, dtype=torch.bfloat16) -> torch.Tensor:
        """Allocate on the generation stream's pool (the kernels that fill the
        buffer run on that stream)."""
        with torch.cuda.stream(self.stream):
            return torch.empty(shape, dtype=dtype, device=self.device)

    # -- weights -------------------------------------------------------------
    def set_weight(self, name: str, t: torch.Tensor):
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.is_contiguous(), name
        self.weights[name] = t
        N.check(self.lib.b200_engine_set_weight(self.h, name.encode(), t.data_ptr(), t.numel()),
                f"set_weight({name})")

    # -- workspace -----------------------------------------------------------
    def ensure_workspace(self, tokens: int = 1, patches: int = 1):
        if self.workspace is not None and tokens <= self._ws_tokens and patches <= self._ws_patches:
            return
        tokens = max(tokens, self._ws_tokens)
        patches = max(patches, self._ws_patches)
        nbytes = self.lib.b200_engine_workspace_bytes(self.h, tokens, patches)
        torch.cuda.current_stream(self.device).synchronize()
        self.stream.synchronize()
        self.workspace = self.empty(nbytes + 256, torch.uint8)
        base = (self.workspace.data_ptr() + 255) & ~255
        N.check(self.lib.b200_engine_set_workspace(self.h, base, nbytes), "set_workspace")
        self._ws_tokens, self._ws_patches = tokens, patches

    # -- kv ------------------------------------------------------------------
    def _check_pool_shape(self, pool):
        # the C ABI takes no pool size: a pool laid out for other head counts / widths than the engine's would be
        # indexed past its end by the kernels
        c = self.cfg
        if (pool.n_layers, pool.n_kv, pool.hd) != (c.n_layers, c.n_kv_heads, c.head_dim):
            raise N.B200Error(f"KV pool (layers, kv heads, head_dim) = {(pool.n_layers, pool.n_kv, pool.hd)} does not "
                              f"match the engine's {(c.n_layers, c.n_kv_heads, c.head_dim)}")

    def bind_pool(self, pool):
        """bind a KVPool (bf16), a QuantizedKVPool (8-bit, single-request decode: the per-phase kernels with the
        8-bit attention) or a BatchKVQPool (the lock-step batch pool of kv_bits=8); see b200_engine_bind_kv"""
        # keyed on the device buffers themselves (not id(pool): CPython reuses ids of collected pools);
        # the engine keeps a strong reference to the bound buffers so their addresses cannot be recycled
        self._check_pool_shape(pool)
        if isinstance(pool, BatchKVQPool):
            q, bf = pool.q, (None if pool.bf is None else pool.bf.buf)
            bufs = (q.codes, q.scales, q.biases, bf)
            args = (q.codes.data_ptr(), q.scales.data_ptr(), q.biases.data_ptr(), pool.group_size, pool.n_q,
                    N.ptr(bf), pool.batch, pool.capacity)
            fn = "bind_batch_kvq"
        elif isinstance(pool, QuantizedKVPool):
            bufs = (pool.codes, pool.scales, pool.biases)
            args = (pool.codes.data_ptr(), pool.scales.data_ptr(), pool.biases.data_ptr(), pool.batch, pool.capacity,
                    pool.group_size)
            fn = "bind_kvq"
        else:
            bufs = (pool.buf,)
            args = (pool.buf.data_ptr(), pool.batch, pool.capacity)
            fn = "bind_kv"
        key = (type(pool),) + args
        if key != self._bound:
            N.check(getattr(self.lib, "b200_engine_" + fn)(self.h, *args), fn)
            self._bound = key
            self._bound_buf = bufs

    def set_prefill_kvq(self, pool, row: int = 0):
        """the next prefill calls quantize their K/V rows of the layers this 8-bit pool holds (a QuantizedKVPool:
        every layer; a BatchKVQPool: its 8-bit layers) into row `row` of it before they are attended; None: off.
        Any bind and a change of the selected row switch it off too (b200_engine_set_prefill_kvq_row)"""
        if pool is None:
            N.check(self.lib.b200_engine_set_prefill_kvq(self.h, None, None, None, 0), "set_prefill_kvq")
            return
        q = pool.q if isinstance(pool, BatchKVQPool) else pool
        N.check(self.lib.b200_engine_set_prefill_kvq_row(self.h, q.codes.data_ptr(), q.scales.data_ptr(),
                                                         q.biases.data_ptr(), q.group_size, q.batch, q.capacity,
                                                         int(row), q.n_layers), "set_prefill_kvq_row")
        self._bound = None   # the next bind_pool reaches the engine, which switches the write-through off

    # -- calls ---------------------------------------------------------------
    def vision(self, pixel_values: torch.Tensor, grid_thw: np.ndarray) -> torch.Tensor:
        grid = np.ascontiguousarray(np.asarray(grid_thw, dtype=np.int32).reshape(-1, 3))
        n_patches = int((grid[:, 0] * grid[:, 1] * grid[:, 2]).sum())
        assert pixel_values.dtype == torch.float32 and pixel_values.is_cuda
        assert pixel_values.shape[0] == n_patches and pixel_values.shape[1] == self.cfg.v_patch_dim
        pixel_values = pixel_values.contiguous()
        self.ensure_workspace(patches=n_patches)
        m2 = self.cfg.v_merge ** 2
        out = self.empty((n_patches // m2, self.cfg.v_out))
        N.check(self.lib.b200_engine_vision(self.h, pixel_values.data_ptr(), grid.ctypes.data,
                                            grid.shape[0], out.data_ptr(), self.s), "engine_vision")
        return out

    def prefill(self, embeds: torch.Tensor, pos3: torch.Tensor, ctx0: int, rope_delta: int,
                all_logits: Optional[torch.Tensor] = None):
        T = embeds.shape[0]
        self.ensure_workspace(tokens=T)
        N.check(self.lib.b200_engine_prefill(self.h, embeds.data_ptr(), pos3.data_ptr(), T, ctx0,
                                             rope_delta, N.ptr(all_logits), self.s),
                "engine_prefill")

    def prefill_batch(self, embeds: torch.Tensor, pos3: torch.Tensor, seq_len, rows):
        """several FRESH prompts in one pass over the weights (reference `PromptProcessingBatch`): embeds
        (sum round8(T_g), hidden) bf16 concatenated along the token axis with every sequence padded to a multiple
        of 8 tokens, pos3 (3, sum round8(T_g)) int32 device, sequence g fills pool row rows[g]; the first tokens land
        in the token log in order"""
        seq_len = np.ascontiguousarray(np.asarray(seq_len, dtype=np.int32))
        rows = np.ascontiguousarray(np.asarray(rows, dtype=np.int32))
        T = int(((seq_len + 7) // 8 * 8).sum())     # every sequence padded to a multiple of 8 tokens
        assert embeds.shape[0] == T and pos3.shape[-1] == T and len(rows) == len(seq_len)
        self.ensure_workspace(tokens=T)
        N.check(self.lib.b200_engine_prefill_batch(self.h, embeds.data_ptr(), pos3.data_ptr(), len(seq_len),
                                                   seq_len.ctypes.data, rows.ctypes.data, self.s), "engine_prefill_batch")

    def decode(self, n_steps: int, force_tokens: Optional[np.ndarray] = None):
        fp = 0
        if force_tokens is not None:
            force_tokens = np.ascontiguousarray(force_tokens, dtype=np.int32)
            assert force_tokens.shape[0] >= n_steps
            fp = force_tokens.ctypes.data
        N.check(self.lib.b200_engine_decode(self.h, n_steps, fp, self.s), "engine_decode")
        if force_tokens is not None:
            self.stream.synchronize()  # the H2D copies read `force_tokens` (pageable)

    # -- lock-step batched decode (decode_batch.cu) -----------------------------
    def set_kv_row(self, row: int):
        N.check(self.lib.b200_engine_set_kv_row(self.h, int(row)), "set_kv_row")

    def batch_begin(self, tok, ctx, pos, active):
        a = [np.ascontiguousarray(x, dtype=np.int32) for x in (tok, ctx, pos, active)]
        B = a[0].shape[0]
        assert all(x.shape == (B,) for x in a)
        N.check(self.lib.b200_batch_begin(self.h, B, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data,
                                          a[3].ctypes.data, self.s), "batch_begin")
        self._batch_B = B

    def batch_decode(self, n_steps: int, want_logprobs: bool = False):
        N.check(self.lib.b200_batch_decode(self.h, int(n_steps), int(want_logprobs), self.s), "batch_decode")

    def batch_fetch(self, first_step: int, n_steps: int, tok_host: torch.Tensor, lp_host: Optional[torch.Tensor] = None):
        """async copy of tokens (and their logprobs) of steps [first, first+n) into pinned (n, B) buffers"""
        N.check(self.lib.b200_batch_fetch(self.h, int(first_step), int(n_steps), tok_host.data_ptr(),
                                          N.ptr(lp_host), self.s), "batch_fetch")

    def batch_set_procs(self, state=None, top_k: int = 0):
        """the armed rows' logits processors (`models/cache.py::BatchProcState`, None: none) and top-k logprobs
        (0: none) until the next batch_begin"""
        st = state
        N.check(self.lib.b200_batch_set_procs(
            self.h, N.ptr(st and st.params), N.ptr(st and st.penalties), N.ptr(st and st.bias_ids),
            N.ptr(st and st.bias_vals), st.BIAS_CAP if st else 0, N.ptr(st and st.hist), N.ptr(st and st.hist_len),
            st.HIST_CAP if st else 0, int(top_k)), "batch_set_procs")

    def batch_fetch_topk(self, first_step: int, n_steps: int, ids_host: torch.Tensor, lp_host: torch.Tensor):
        """async copy of the top-k ids / logprobs of steps [first, first+n) into pinned (n, B, 20) buffers"""
        N.check(self.lib.b200_batch_fetch_topk(self.h, int(first_step), int(n_steps), ids_host.data_ptr(),
                                               lp_host.data_ptr(), self.s), "batch_fetch_topk")

    def batch_logits_view(self, which: str = "logits") -> torch.Tensor:
        p = (self.lib.b200_batch_logits if which == "logits" else self.lib.b200_batch_logprobs)(self.h)
        ldv = (self.cfg.vocab + 7) // 8 * 8      # rows are padded to 16-byte multiples (tail = -inf)
        return self._view(p, self._batch_B * ldv, torch.bfloat16).view(self._batch_B, ldv)[:, :self.cfg.vocab]

    BATCH_LOG_STEPS, BATCH_LOG_ROWS = BATCH_LOG_STEPS, 16

    def batch_token_log_view(self) -> torch.Tensor:
        """int32 (steps since the last batch_begin, 16) view of the batched decoder's token log"""
        p = self.lib.b200_batch_token_log(self.h)
        return self._view(p, self.BATCH_LOG_STEPS * self.BATCH_LOG_ROWS, torch.int32).view(self.BATCH_LOG_STEPS,
                                                                                        self.BATCH_LOG_ROWS)

    def kv_copy_row(self, dst, dst_row: int, src, src_row: int, n_tokens: int):
        """the first n_tokens positions of row src_row of `src` into row dst_row of `dst`, two pools of one type and
        layout (KVPool, QuantizedKVPool or BatchKVQPool): every plane set of the pool, byte for byte"""
        for (d, n_layers, bpp), (s, _, _) in zip(dst.plane_sets(), src.plane_sets(), strict=True):
            N.check(self.lib.b200_pool_copy_row(d.data_ptr(), dst.batch, dst.capacity, int(dst_row), s.data_ptr(),
                                                src.batch, src.capacity, int(src_row), n_layers, dst.n_kv, bpp,
                                                int(n_tokens), self.s), "pool_copy_row")

    def set_next(self, token: int, ctx: int, position: int):
        N.check(self.lib.b200_engine_set_next(self.h, int(token), int(ctx), int(position), self.s),
                "set_next")

    def _view(self, p: int, n: int, dtype) -> torch.Tensor:
        """torch view of an engine-owned device buffer (no copy)."""
        esz = torch.empty((), dtype=dtype).element_size()
        iface = {"shape": (n,), "typestr": {2: "<i2", 4: "<i4"}[esz], "data": (p, False),
                 "version": 3}
        holder = type("_Buf", (), {"__cuda_array_interface__": iface})()
        t = torch.as_tensor(holder, device=self.device)
        return t.view(dtype)

    def logits_view(self) -> torch.Tensor:
        return self._view(self.lib.b200_engine_logits(self.h), self.cfg.vocab, torch.bfloat16)

    def logprobs_view(self) -> torch.Tensor:
        return self._view(self.lib.b200_engine_logprobs(self.h), self.cfg.vocab, torch.bfloat16)

    def token_log_view(self) -> torch.Tensor:
        """int32 view of the engine's device token ring (generated ids, index = token number % capacity)."""
        return self._view(self.lib.b200_engine_token_log(self.h), self.token_log_capacity, torch.int32)

    @property
    def token_log_capacity(self) -> int:
        return int(self.lib.b200_engine_token_log_capacity(self.h))

    def snapshot(self, which: str = "logprobs") -> torch.Tensor:
        """Stream-ordered copy of the current step's logits/logprobs vector."""
        src = (self.lib.b200_engine_logprobs if which == "logprobs"
               else self.lib.b200_engine_logits)(self.h)
        out = self.empty((self.cfg.vocab,))
        N.check(self.lib.b200_memcpy_d2d(out.data_ptr(), src, self.cfg.vocab * 2, self.s),
                "memcpy_d2d")
        return out

    def fetch_tokens(self, start: int, n: int, host: torch.Tensor):
        """async copy of generated ids [start, start+n) into pinned `host` (int32)."""
        N.check(self.lib.b200_engine_fetch_tokens(self.h, start, n, host.data_ptr(), self.s),
                "fetch_tokens")

    @property
    def tokens_launched(self) -> int:
        return int(self.lib.b200_engine_tokens_launched(self.h))

    @property
    def launch_count(self) -> int:
        return int(self.lib.b200_engine_launch_count(self.h))

    def last_decode_ms(self) -> float:
        return float(self.lib.b200_engine_last_decode_ms(self.h))

    def set_graph(self, enabled: bool):
        N.check(self.lib.b200_engine_set_graph(self.h, int(enabled)), "set_graph")

    def set_mega(self, enabled):
        """0/False: one kernel per phase; 1/True: k_mega, the persistent decode-step kernel
        (default).  Any other value raises B200Error and leaves the mode unchanged."""
        N.check(self.lib.b200_engine_set_mega(self.h, int(enabled)), "set_mega")

    def debug_buffer(self, name: str, dtype=torch.float32) -> torch.Tensor:
        """Copy of an internal device buffer (tests / debugging only)."""
        ptr, nbytes = C.c_void_p(), C.c_long()
        N.check(self.lib.b200_engine_debug_buffer(self.h, name.encode(), C.byref(ptr), C.byref(nbytes)),
                "debug_buffer")
        out = self.empty((nbytes.value // torch.empty((), dtype=dtype).element_size(),), dtype)
        N.check(self.lib.b200_memcpy_d2d(out.data_ptr(), ptr, nbytes.value, self.s), "memcpy_d2d")
        self.stream.synchronize()
        return out

    def device_error(self) -> int:
        v = C.c_int(0)
        N.check(self.lib.b200_engine_device_error(self.h, C.byref(v)), "device_error")
        return int(v.value)

    def set_pdl(self, enabled: bool):
        N.check(self.lib.b200_engine_set_pdl(self.h, int(enabled)), "set_pdl")

    def set_attn_cluster(self, n: int):
        N.check(self.lib.b200_engine_set_attn_cluster(self.h, int(n)), "set_attn_cluster")
