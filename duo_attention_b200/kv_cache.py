"""Head-major DuoAttention KV cache for H100.

Replaces the reference's token-major caches —

* ``DuoAttentionStaticKVCache``       (duo_attn/patch/static_kv_cache.py:18-315)
* the per-layer tuple cache           (duo_attn/patch/llama.py:168-171,292-301)
* ``DuoAttentionStaticINT4KVCache``   (demo/int4_kv.py:115-492)

— with one layout designed for coalesced 128 B HBM loads and TMA tiles:

    full_k / full_v : [B, n_full,   capacity,                 128]   retrieval heads
    ring_k / ring_v : [B, n_stream, sink + recent + stage_cap, 128]  streaming heads
                      slots [0,sink) sinks | [sink,sink+recent) true ring | staging for the chunk in flight

The streaming cache is a real ring (token ``p`` lives in slot ``sink + (p - sink) % recent``): the
reference's per-step compaction copies (static_kv_cache.py:127-167) become index arithmetic.  The Python
object only owns buffers and three integers per layer; all data movement and math is CUDA
(``csrc/``) reached through the C ABI.  Public methods keep the reference's names and semantics:
``kv_seq_len``, ``clear()``, ``evict_last(n)``, ``memory_usage``; overflow raises ``ValueError``.
"""
from __future__ import annotations

import ctypes as C
import numbers
import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _C


def _count_full(row) -> int:
    return int((np.asarray(row, dtype=np.float64) > 0.5).sum())


def model_geometry(model, full_attention_heads=None) -> dict:
    """The cache geometry of a Hugging Face model, as :class:`DuoKVCache` keyword arguments: ``num_layers``,
    ``num_heads``, ``num_kv_heads``, ``head_dim``, ``dtype`` and ``device`` (those of its first parameter), and given
    the gate matrix ``full_attention_heads``, the retrieval heads per layer ``num_full_kv_head_list``."""
    p = next(model.parameters())
    cfg = model.config
    geo = dict(num_layers=cfg.num_hidden_layers, num_heads=cfg.num_attention_heads,
               num_kv_heads=cfg.num_key_value_heads,
               head_dim=getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads,
               dtype=p.dtype, device=p.device)
    if full_attention_heads is not None:
        geo["num_full_kv_head_list"] = [_count_full(r) for r in full_attention_heads]
    return geo


# ---- ring arithmetic (pure integers; the CUDA side implements the same formulas in duo_common.cuh) ----
def ring_slot(pos: int, sink: int, recent: int) -> int:
    """Slot of token ``pos`` in the streaming cache: sinks map to themselves, the rest into the ring."""
    return pos if pos < sink else sink + (pos - sink) % recent


def ring_advance(total: int, lo: int, n: int, sink: int, recent: int):
    """State after appending ``n`` tokens: the ring keeps the last ``recent`` positions."""
    total += n
    return total, max(lo, total - recent, sink)


def ring_evict(total: int, lo: int, n: int, sink: int):
    """State after ``evict_last(n)`` (static_kv_cache.py:290-297): the newest ``n`` tokens are dropped."""
    total = max(0, total - n)
    return total, max(sink, min(lo, total))


def ring_live_positions(total: int, lo: int, sink: int):
    """Token positions a streaming head can still see (what the reference's compacted cache holds)."""
    return list(range(0, min(total, sink))) + list(range(max(lo, sink), total))


class DuoKVCache:
    pooled = False      # per-row capacities of a DuoRaggedKVCache: the retrieval K/V in one pool per layer
    rows_changed = False  # a row changed on the host since the last DuoDecodeGraph.resync() (ragged caches only)

    def __init__(
        self,
        num_layers: int,
        num_heads: int,
        num_kv_heads: int,
        head_dim: int,
        num_full_kv_head_list: Sequence[int],
        batch_size: int,
        max_size: int,
        sink_size: int,
        recent_size: int,
        dtype: torch.dtype,
        device,
        stage_cap: int = 64,
        kv_format: str = "same",
        growable: bool = False,
        local_full_cap: Optional[int] = None,
        workspace: Optional[torch.Tensor] = None,
    ):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("DuoKVCache lives in GPU memory: the CUDA kernels have no CPU fallback")
        if head_dim != 128:
            raise ValueError(f"head_dim {head_dim} not supported (the kernels are specialised for 128)")
        if dtype not in (torch.bfloat16, torch.float16):
            raise ValueError(f"dtype {dtype} not supported (bf16 / fp16)")
        if kv_format not in ("same", "int4"):
            raise ValueError(f"kv_format {kv_format!r} not supported")
        self.lib = _C.load()
        self.batch_size, self.max_size = int(batch_size), int(max_size)
        self.sink_size, self.recent_size = int(sink_size), int(recent_size)
        self.num_layers, self.num_heads, self.num_kv_heads = num_layers, num_heads, num_kv_heads
        self.num_kv_groups = num_heads // num_kv_heads
        self.head_dim = head_dim
        self.dtype, self.device = dtype, device
        self.kv_format = kv_format
        self.growable = growable
        self.num_full_kv_head_list = [int(n) for n in num_full_kv_head_list]
        self.num_streaming_kv_head_list = [num_kv_heads - n for n in self.num_full_kv_head_list]
        assert len(self.num_full_kv_head_list) == num_layers
        # occupancy, per layer (mirrors kv_seq_len_list / streaming_kv_seq_len_list of the reference)
        self.kv_seq_len_list = [0] * num_layers   # retrieval cache length
        self.total_list = [0] * num_layers        # tokens seen by the streaming heads
        self.lo_list = [self.sink_size] * num_layers
        # rows actually allocated per retrieval head (== max_size unless a subclass shards the positions over ranks)
        self.full_cap_list = [self.max_size if local_full_cap is None else int(local_full_cap)] * num_layers
        self.stage_cap_list = [max(1, int(stage_cap))] * num_layers
        self.tensors: List[Optional[dict]] = [None] * num_layers
        self.handles: List[Optional[int]] = [None] * num_layers
        for l in range(num_layers):
            self._set_layer(l, self.full_cap_list[l], self.stage_cap_list[l])
        self.graph_attached = False  # set by DuoDecodeGraph: buffers must then keep their addresses
        self.dev_state = None        # optional device copy of (full_len, total, lo): see enable_device_state()
        self.launch_count = 0        # kernels of this library enqueued through this cache
        self.profile_events = None   # set to [] to collect (start, end) CUDA events around every duo_attention
        if workspace is None:  # a caller may share one zero-initialised workspace between caches used in turn
            ws = self.lib.duo_workspace_bytes(self.batch_size, num_kv_heads, self.num_kv_groups, _C.DECODE_MAX_Q)
            workspace = torch.zeros(ws, dtype=torch.uint8, device=device)
        self.workspace = workspace

    # ------------------------------------------------------------------------------------------
    @property
    def W(self):
        return self.sink_size + self.recent_size

    @property
    def stage_off(self):
        """First staging slot (duo_b200.h): right after the ring, 64-aligned for INT4 caches."""
        return self.W if self.kv_format == "same" else (self.W + 63) // 64 * 64

    # ---- layer tensors and handles ---------------------------------------------------------------------------
    def _alloc_kv(self, t, name, shape):
        """Allocate K/V tensor ``name`` of ``shape + [head_dim]`` into ``t``: 16-bit, or for INT4 caches packed codes
        ``[.., head_dim / 2]`` plus fp16 ``name_scale`` / ``name_zero`` of ``shape``."""
        if self.kv_format == "same":
            t[name] = torch.zeros(*shape, self.head_dim, dtype=self.dtype, device=self.device)
        else:
            t[name] = torch.zeros(*shape, self.head_dim // 2, dtype=torch.uint8, device=self.device)
            t[name + "_scale"] = torch.zeros(*shape, dtype=torch.float16, device=self.device)
            t[name + "_zero"] = torch.zeros(*shape, dtype=torch.float16, device=self.device)

    def _alloc_layer(self, l, full_cap, stage_cap, old=None):
        """Layer ``l``'s tensors at these capacities.  Given its current tensors ``old``, a retrieval tensor of unchanged
        shape is kept (it may hold GBs); the others are re-allocated and keep the cached rows or the sink + ring slots."""
        nf, ns = self.num_full_kv_head_list[l], self.num_streaming_kv_head_list[l]
        slots = self.stage_off + stage_cap
        if self.kv_format == "int4":
            slots = (slots + 7) // 8 * 8
            full_cap = (full_cap + 63) // 64 * 64
        # pooled: one pool of pool_tokens * n_full rows per retrieval tensor (duo_layer_create_pooled)
        full = (self.pool_tokens * nf,) if self.pooled else (self.batch_size, nf, full_cap)
        ring, n, W = (self.batch_size, ns, slots), self.kv_seq_len_list[l], self.W
        t = {}
        for name, shape, keep in (("full_k", full, n), ("full_v", full, n), ("ring_k", ring, W), ("ring_v", ring, W)):
            if old is not None and name.startswith("full") and tuple(old[name].shape[:-1]) == shape:
                t.update((k, v) for k, v in old.items() if k.startswith(name))
                continue
            self._alloc_kv(t, name, shape)
            if old is not None:
                for k in t:
                    if k.startswith(name):
                        t[k][:, :, :keep].copy_(old[k][:, :, :keep])
        return t

    def _set_layer(self, l, full_cap, stage_cap):
        """(Re-)derive layer ``l`` at these capacities: its tensors (see ``_alloc_layer``) and a new handle over them."""
        self.tensors[l] = self._alloc_layer(l, full_cap, stage_cap, self.tensors[l])
        self.full_cap_list[l], self.stage_cap_list[l] = full_cap, stage_cap
        self._make_handle(l)

    def _make_handle(self, l):
        """Replace layer ``l``'s handle by a new one over its current tensors."""
        h, self.handles[l] = self.handles[l], None
        self._release([h])
        self.handles[l] = self._create_handle(l, self.tensors[l])

    def _create_handle(self, l, t, kv_format=None) -> int:
        """A ``duo_layer`` over the tensors ``t`` of a layer with layer ``l``'s heads (``kv_format="same"``: the 16-bit
        image of an INT4 cache); a pooled cache's handle is a pooled one."""
        kv_format = kv_format or self.kv_format
        d = _C.LayerDesc()
        for key, v in t.items():
            setattr(d, key, v.data_ptr() if v.numel() else None)
        d.full_cap = 0 if self.pooled else t["full_k"].shape[2]
        d.batch = self.batch_size
        d.n_full = self.num_full_kv_head_list[l]
        d.n_stream = self.num_streaming_kv_head_list[l]
        d.group = self.num_kv_groups
        d.head_dim = self.head_dim
        d.sink, d.recent = self.sink_size, self.recent_size
        d.stage_cap = t["ring_k"].shape[2] - (self.W if kv_format == "same" else self.stage_off)
        d.dtype = _C.DT_BF16 if self.dtype == torch.bfloat16 else _C.DT_FP16
        d.kv_format = _C.KV_SAME if kv_format == "same" else _C.KV_INT4
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            if self.pooled:
                _C.check(self.lib.duo_layer_create_pooled(C.byref(d), self.pool_tokens, C.byref(h)))
            else:
                _C.check(self.lib.duo_layer_create(C.byref(d), C.byref(h)))
        return h.value

    def _release(self, handles):
        for h in handles:
            if h is not None:
                self.lib.duo_layer_destroy(h)

    def _owned_handles(self) -> list:
        """Every handle this cache created and still holds: its layers' and those of its 16-bit image."""
        dq = getattr(self, "_dq", None)
        return list(self.handles) + (list(dq["handles"].values()) if dq else [])

    def __del__(self):
        try:
            self._release(self._owned_handles())
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------
    def _room_error(self, l, q_len) -> ValueError:
        # the message of static_kv_cache.py:112-115
        return ValueError(f"Trying to put {q_len} KVs into a cache with max size {self.max_size}, "
                          f"current size: {self.kv_seq_len_list[l]}.")

    def check_room(self, q_len, layers=None):
        """Raise the overflow ``ValueError`` if a layer of ``layers`` (default: all) lacks room for ``q_len`` more tokens
        in its retrieval cache.  The batched ragged step and ``DuoDecodeGraph.step`` check here, and layers without
        retrieval heads are skipped; eager ``attend`` (``_ensure_room``) raises for such a layer too.  The two
        conditions differ on purpose: unifying them would change which calls raise."""
        for l in range(self.num_layers) if layers is None else layers:
            if self.num_full_kv_head_list[l] > 0 and self._rows_needed(l, q_len) > self.full_cap_list[l]:
                raise self._room_error(l, q_len)

    def _ensure_room(self, l, q_len):
        """Grow the staging area (always allowed) and, for growable caches (tuple-path compatibility,
        where the reference simply torch.cat's), the retrieval cache."""
        need_full = self._rows_needed(l, q_len)
        grow_full = need_full > self.full_cap_list[l]
        if grow_full and not self.growable:
            raise self._room_error(l, q_len)
        if grow_full or q_len > self.stage_cap_list[l]:
            self._grow_layer(l, q_len, max(need_full, 2 * self.full_cap_list[l], 256) if grow_full else None)

    def _grow_layer(self, l, q_len, full_cap=None):
        """Layer ``l`` with a staging area for a chunk of ``q_len`` tokens and ``full_cap`` retrieval rows (default: as
        now).  A longer staging area leaves the (possibly multi-GB) retrieval cache where it is."""
        if self.graph_attached:
            raise ValueError("this cache is captured in a DuoDecodeGraph: its buffers cannot be re-allocated "
                             f"(chunk of {q_len} tokens > staging capacity {self.stage_cap_list[l]})")
        self._set_layer(l, full_cap or self.full_cap_list[l], max(self.stage_cap_list[l], q_len))

    def _first_chunk_scratch(self, S):
        sc = getattr(self, "_scratch", None)
        if sc is None or sc.max_size < S:
            sc = DuoKVCache(1, self.num_heads, self.num_kv_heads, self.head_dim, [self.num_kv_heads],
                            self.batch_size, max(S, 64), self.sink_size, self.recent_size, self.dtype, self.device,
                            stage_cap=max(S, 64), kv_format="same")  # no streaming heads: staging costs nothing
            self._scratch = sc
        return sc

    # ---- large chunks (>= 128 tokens) over an INT4 cache: wgmma prefill kernel on a 16-bit image ----------------
    def _dequant_scratch(self, l, S):
        """Image of layer ``l``'s INT4 cache in the activation dtype for ONE attention call of a chunk of >= 128 tokens — what the
        reference does on EVERY call (``get()`` dequantises the whole cache, demo/int4_kv.py:373-436, then
        flash_attn_func runs on it, demo/w8a8kv4_llama.py:239-274).  For such a chunk the O(ctx) dequantisation pass
        is < 1 % of the chunk x ctx attention, and the attention runs on the tensor-core prefill kernel.  Decode and small chunks never
        come here: their kernels dequantise in the K/V load stage.  fp16 layers get K2's fp16 values
        (duo_dequant_int4), bf16 layers bf16_rn(fma(code, scale, zero)) (duo_dequant_int4_bf16).  One flat
        zero-initialised buffer is shared by all layers (they are processed one after the other; rows beyond the
        dequantised range hold zeros or finite leftovers and are masked); a layer handle is created per distinct
        number of retrieval heads, and released with the image."""
        sc = getattr(self, "_dq", None)
        B, D = self.batch_size, self.head_dim
        cap = max(self.full_cap_list)
        slots = self.W + max(max(self.stage_cap_list), S)
        if sc is None or sc["cap"] < cap or sc["slots"] < slots:
            nf_max = max(self.num_full_kv_head_list)
            ns_max = max(self.num_streaming_kv_head_list)
            new = {"cap": cap, "slots": slots, "handles": {},
                   "full": [torch.zeros(B * nf_max * cap * D, dtype=self.dtype, device=self.device) for _ in range(2)],
                   "ring": [torch.zeros(B * ns_max * slots * D, dtype=self.dtype, device=self.device) for _ in range(2)]}
            if sc is not None:
                self._release(sc["handles"].values())
            self._dq = sc = new
        nf, ns = self.num_full_kv_head_list[l], self.num_streaming_kv_head_list[l]
        cap = sc["cap"]  # the image's handles are encoded at its capacity (rows of a pooled cache share one image)
        fk, fv = (t[: B * nf * cap * D].view(B, nf, cap, D) for t in sc["full"])
        rk, rv = (t[: B * ns * slots * D].view(B, ns, slots, D) for t in sc["ring"])
        if nf not in sc["handles"]:
            sc["handles"][nf] = self._create_handle(l, {"full_k": fk, "full_v": fv, "ring_k": rk, "ring_v": rv},
                                                    kv_format="same")
        # dequantise what this call can see: retrieval rows [0, full_len + S) (of a sequence-sharded cache: the rows of
        # the local slice), sink + ring slots, the staged chunk
        t = self.tensors[l]
        stream = torch.cuda.current_stream(self.device).cuda_stream
        n_rows = self._rows_needed(l, S)
        W, so = self.W, self.stage_off
        dequant = self.lib.duo_dequant_int4_bf16 if self.dtype == torch.bfloat16 else self.lib.duo_dequant_int4
        for b in range(B):
            for hh in range(nf):
                for name, dst in (("full_k", fk), ("full_v", fv)):
                    self._launch(dequant, t[name][b, hh].data_ptr(), t[name + "_scale"][b, hh].data_ptr(),
                                 t[name + "_zero"][b, hh].data_ptr(), n_rows, dst[b, hh].data_ptr(), stream)
            for hh in range(ns):
                for name, dst in (("ring_k", rk), ("ring_v", rv)):
                    for src0, dst0, rows in ((0, 0, W), (so, W, S)):
                        self._launch(dequant, t[name][b, hh, src0:].data_ptr(),
                                     t[name + "_scale"][b, hh, src0:].data_ptr(),
                                     t[name + "_zero"][b, hh, src0:].data_ptr(), rows, dst[b, hh, dst0:].data_ptr(),
                                     stream)
        return sc["handles"][nf]

    def state(self, l) -> _C.CacheState:
        ds = self.dev_state.data_ptr() if self.dev_state is not None else None
        return _C.CacheState(self.kv_seq_len_list[l], self.total_list[l], self.lo_list[l], ds)

    def _rows_needed(self, l, q_len) -> int:
        """Rows of the (local) retrieval cache in use after appending ``q_len`` tokens."""
        return self.kv_seq_len_list[l] + q_len

    # ---- device-resident occupancy (CUDA-graph replay of decode steps) ---------------------------------
    def enable_device_state(self):
        """Keep a device copy of (full_len, total, lo) that the decode kernels read at launch, so that a captured
        decode step can be replayed while the context grows.  All layers hold the same occupancy at step
        boundaries, so one copy serves the whole cache."""
        if self.dev_state is None:
            self.dev_state = torch.zeros(4, dtype=torch.int64, device=self.device)
        self.sync_device_state()
        return self

    def sync_device_state(self):
        """Stream-ordered refresh of the device copy: the integers travel as kernel arguments (duo_state_set), so
        back-to-back evict_last()/clear() calls cannot race through a shared staging buffer."""
        if self.dev_state is None:
            return
        l = self.num_layers - 1
        self._launch(self.lib.duo_state_set, self.dev_state.data_ptr(), self.kv_seq_len_list[l], self.total_list[l],
                     self.lo_list[l], torch.cuda.current_stream(self.device).cuda_stream)

    def advance_device(self, n):
        """Enqueue full_len += n, total += n, lo = max(lo, total - recent, sink) on the device copy."""
        self._launch(self.lib.duo_state_advance, self.dev_state.data_ptr(), int(n), self.sink_size, self.recent_size,
                     torch.cuda.current_stream(self.device).cuda_stream)

    def snapshot_state(self):
        """Copy of the host occupancy: lets a caller run throw-away steps (CUDA-graph warm-up / capture) and put it
        back with ``restore_state``."""
        return list(self.kv_seq_len_list), list(self.total_list), list(self.lo_list)

    def restore_state(self, snap):
        self.kv_seq_len_list[:], self.total_list[:], self.lo_list[:] = (list(x) for x in snap)

    def snapshot_ring(self):
        """Copy of the sink+ring slots of every layer (a few hundred KB each): lets a caller run throw-away steps
        (CUDA-graph warm-up / capture) and put the streaming cache back exactly as it was."""
        W = self.W
        return [{k: v[:, :, :W].clone() for k, v in t.items() if k.startswith("ring")} for t in self.tensors]

    def restore_ring(self, snap):
        W = self.W
        for t, sn in zip(self.tensors, snap):
            for k, v in sn.items():
                t[k][:, :, :W].copy_(v)

    def advance_host(self, n):
        """Mirror of advance_device for the host integers (call once per graph replay)."""
        for l in range(self.num_layers):
            self.advance(l, n)

    def advance(self, l, q_len):
        self.kv_seq_len_list[l] += q_len
        self.total_list[l], self.lo_list[l] = ring_advance(self.total_list[l], self.lo_list[l], q_len,
                                                           self.sink_size, self.recent_size)

    # ------------------------------------------------------------------------------------------
    # reference-compatible surface (static_kv_cache.py:100-107, 285-315)
    @property
    def kv_seq_len(self):
        return self.kv_seq_len_list[-1]

    @property
    def streaming_kv_seq_len(self):
        """Rows the reference's compacted streaming cache would hold (sinks + live ring entries)."""
        tot, lo = self.total_list[-1], self.lo_list[-1]
        return min(tot, self.sink_size) + max(0, tot - max(lo, self.sink_size))

    def clear(self):
        for l in range(self.num_layers):
            self.kv_seq_len_list[l] = 0
            self.total_list[l] = 0
            self.lo_list[l] = self.sink_size
        self.sync_device_state()

    def evict_last(self, num_tokens):
        for l in range(self.num_layers):
            self.kv_seq_len_list[l] = max(0, self.kv_seq_len_list[l] - num_tokens)
            self.total_list[l], self.lo_list[l] = ring_evict(self.total_list[l], self.lo_list[l], num_tokens,
                                                             self.sink_size)
        self.sync_device_state()

    @property
    def memory_usage(self):
        tot = 0
        for t in self.tensors:
            for v in t.values():
                tot += v.element_size() * v.numel()
        return tot

    # ------------------------------------------------------------------------------------------
    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """The fused per-layer hot path: RoPE + append, mixed-head attention, ring commit.

        qkv  ``[B, S, (Hq + 2 Hkv) * D]`` (last dim contiguous) — q is rotated in place on the three-launch path,
             left untouched on the one-launch path.
        out  ``[B, S, Hq, D]`` contiguous, written.
        ``fused=False`` forces the three-launch path for decode-sized chunks.  On 16-bit caches both paths leave the
        same bits in the cache and in the streaming-head rows of ``out``; the retrieval-head rows agree to rounding
        only (the one-launch kernel splits the cached keys and attends the new tokens as one extra tile, the
        three-launch kernel tiles cached and new keys together).
        """
        S, scale, cp, sp, stream = self._attend_args(l, qkv, out, cos, sin, scale)
        self._ensure_room(l, S)
        st = self.state(l)
        h = self.handles[l]
        lib = self.lib
        # decode-sized chunks take ONE launch: 16-bit caches up to 16 packed rows, INT4 caches up to 8 (the keys-as-M
        # kernel) — except the very first INT4 call, which attends the raw 16-bit K/V (see below)
        one_launch = (S * self.num_kv_groups <= _C.DECODE_MAX_Q if self.kv_format == "same" else
                      S * self.num_kv_groups <= _C.DECODE_MAX_Q_INT4 and not (st.full_len == 0 and st.total == 0))
        if (one_launch and fused and not force_mma and qkv.stride(1) % 8 == 0 and qkv.data_ptr() % 16 == 0):
            # decode-sized chunk: RoPE + append + attention + ring commit in ONE launch (q is not written back)
            self._launch(lib.duo_decode_fused, h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode & 0xFF,
                         out.data_ptr(), S, float(scale), self.workspace.data_ptr(), self.workspace.numel(), stream,
                         timed=True)
            self.advance(l, S)
            return out
        self._launch(lib.duo_rope_append, h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode, S, stream)
        ah, ast = h, st
        if self.kv_format == "int4" and st.full_len == 0 and st.total == 0:
            # The reference attends the RAW 16-bit K/V on the very first call and only later calls see the
            # quantise->dequantise round trip (demo/w8a8kv4_llama.py:229-238 vs :239-274).  The chunk has just
            # been quantised into the INT4 cache above; attention for this one call runs on a 16-bit scratch layer
            # of the activation dtype
            # (every head is plain causal on the first call, so all heads are "retrieval" there).
            sc = self._first_chunk_scratch(S)
            ah, ast = sc.handles[0], _C.CacheState(0, 0, sc.sink_size)
            self._launch(lib.duo_rope_append, ah, C.byref(ast), qkv.data_ptr(), qkv.stride(1), cp, sp,
                         rope_mode | _C.ROPE_SKIP_Q, S, stream)
        elif self.kv_format == "int4" and S >= 128 and self.W <= 2048 and not force_mma:
            ah, ast = self._dequant_scratch(l, S), _C.CacheState(st.full_len, st.total, st.lo, None)
        self._launch(lib.duo_attention_mma if force_mma else lib.duo_attention, ah, C.byref(ast), qkv.data_ptr(),
                     qkv.stride(1), out.data_ptr(), S, float(scale), self.workspace.data_ptr(), self.workspace.numel(),
                     stream, timed=True)
        # a layer without streaming heads has nothing to commit: no kernel
        self._launch(lib.duo_stream_commit, h, C.byref(st), S, stream,
                     count=1 if self.num_streaming_kv_head_list[l] > 0 else 0)
        self.advance(l, S)
        return out

    def _attend_args(self, l, qkv, out, cos, sin, scale):
        """Checks shared by the ``attend`` methods; returns ``(q_len, scale, cos pointer, sin pointer, stream)``."""
        if not qkv.is_cuda or not out.is_cuda:
            raise RuntimeError("duo_attention_b200 kernels need CUDA tensors (no CPU fallback)")
        B, S, width = qkv.shape
        self._check_chunk(l, S)
        assert B == self.batch_size and width == (self.num_heads + 2 * self.num_kv_heads) * self.head_dim
        assert qkv.stride(2) == 1 and (B == 1 or qkv.stride(0) == S * qkv.stride(1)), "qkv rows must be uniformly strided"
        assert out.is_contiguous() and qkv.dtype == self.dtype and out.dtype == self.dtype
        return (S, self.head_dim ** -0.5 if scale is None else scale, cos.data_ptr() if cos is not None else None,
                sin.data_ptr() if sin is not None else None, torch.cuda.current_stream(self.device).cuda_stream)

    def _check_chunk(self, l, q_len):
        """Raise ``ValueError`` for a chunk of ``q_len`` tokens that ``attend`` does not take (none here)."""

    def _launch(self, fn, *args, count=1, timed=False):
        """Call the C entry point ``fn``, raise on its status and count its ``count`` kernel launches; ``timed``
        launches are bracketed by a CUDA event pair in ``profile_events`` when that is a list."""
        timed = timed and self.profile_events is not None
        if timed:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _C.check(fn(*args))
        if timed:
            e1.record()
            self.profile_events.append((e0, e1))
        self.launch_count += count


class DuoAttentionStaticKVCache(DuoKVCache):
    """Drop-in for the reference class of the same name (static_kv_cache.py:18-98): same constructor
    arguments (plus optional keyword extras), same ``clear`` / ``evict_last`` / ``memory_usage`` /
    ``kv_seq_len`` surface, head-major storage underneath."""

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                 prefilling_chunk_size: int = 64, kv_format: str = "same"):
        super().__init__(
            **model_geometry(model, full_attention_heads),
            batch_size=batch_size,
            max_size=max_size,
            sink_size=sink_size,
            recent_size=recent_size,
            stage_cap=prefilling_chunk_size,
            kv_format=kv_format,
            growable=False,
        )


class DuoSeqShardKVCache(DuoKVCache):
    """Decode-phase cache of the SEQUENCE-SHARDED tensor-parallel layout (scope row f1; ``tp.install_seq_shard``):
    every rank holds all heads of a layer, but of each retrieval head only its block-cyclic slice of the token
    positions (``seqshard.SeqShardPlan``); streaming heads are replicated.  ``kv_seq_len`` keeps counting GLOBAL tokens.

    ``attend`` = duo_rope_append (appends only positions this rank owns) -> duo_attention_seq (slice partials for the
    retrieval heads, streaming heads final) -> duo_seq_merge (peer-memory exchange + merge) -> duo_stream_commit, for
    decode-sized chunks (up to ``max_q`` tokens: group x q_len <= 16).  A longer chunk (the next user turn, an appended
    document) takes duo_prefill_seq instead (the wgmma prefill kernel from 128 tokens, the 64-row mma.sync kernel
    below) and a merge scattered by rows (``SeqComm.merge_scattered``); its partial buffers and the staging area grow
    on demand.  The first prefill runs head-parallel and ``tp.reshard_heads_to_seq`` moves the caches over
    (``load_from_head_parallel``).  Same ``clear`` / ``evict_last`` / ``memory_usage`` surface as the static cache;
    ``DuoDecodeGraph`` can capture its decode steps (not longer chunks)."""

    _KV = "same"                              # the one kv_format of the class
    max_rows = _C.DECODE_MAX_Q                # packed rows (group x q_len) of one decode call
    _attention = "duo_attention_seq"          # C entry points: decode-sized chunk / one fused token
    _fused = "duo_decode_fused_seq"

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size, seq=None):
        from .seqshard import SeqShardPlan

        seq = seq if seq is not None else model._duo_seq
        self.seq = seq
        self.plan = SeqShardPlan(seq.world, seq.block)
        super().__init__(
            **model_geometry(model, full_attention_heads), batch_size=batch_size, max_size=max_size,
            sink_size=sink_size, recent_size=recent_size, stage_cap=self.max_rows, kv_format=self._KV, growable=False,
            local_full_cap=self.plan.capacity(int(max_size)) + 1)
        self.max_q = max(1, self.max_rows // self.num_kv_groups)  # duo_seq_merge checks its row count per call
        self.part_o = torch.zeros(batch_size, self.max_q, self.num_heads, self.head_dim, dtype=torch.float32,
                                  device=self.device)
        self.part_lse = torch.zeros(batch_size, self.max_q, self.num_heads, dtype=torch.float32, device=self.device)

    def state(self, l) -> _C.CacheState:
        st = super().state(l)
        st.seq_rank, st.seq_world, st.seq_block = self.seq.rank, self.seq.world, self.seq.block
        return st

    def _rows_needed(self, l, q_len) -> int:
        return self.plan.local_len(self.seq.rank, self.kv_seq_len_list[l] + q_len)

    def _check_chunk(self, l, q_len):
        if q_len > self.max_q:
            if self.graph_attached:
                raise ValueError(f"this cache is captured in a DuoDecodeGraph, which replays decode steps of <= "
                                 f"{self.max_q} tokens: a chunk of {q_len} tokens would re-allocate its buffers")
            return
        # duo_seq_merge refuses more rows than its communicator holds, but only after this step's append and ring
        # commit have run: refuse here, before any launch, so that a refused call leaves the cache as it was
        nfq = self.num_full_kv_head_list[l] * self.num_kv_groups
        rows = self.batch_size * q_len * nfq
        if rows > self.seq.comm.max_rows:
            raise ValueError(f"layer {l}: a chunk of {q_len} token(s) at batch {self.batch_size} merges {rows} rows "
                             f"({nfq} retrieval q-heads each), more than the communicator's max_rows "
                             f"{self.seq.comm.max_rows}: decode in smaller chunks or raise max_rows "
                             "(install_seq_shard)")

    def partials(self, S):
        """``(part_o, part_lse)`` views ``[B, S, Hq, D]`` / ``[B, S, Hq]`` for a chunk of ``S`` tokens (the kernels index
        ``[batch][q_len][heads]``), the buffers grown first if they are too small."""
        B, H, D = self.batch_size, self.num_heads, self.head_dim
        if S == self.part_o.shape[1]:
            return self.part_o, self.part_lse
        if B * S * H > self.part_lse.numel():
            self.part_o = torch.zeros(B, S, H, D, dtype=torch.float32, device=self.device)
            self.part_lse = torch.zeros(B, S, H, dtype=torch.float32, device=self.device)
            return self.part_o, self.part_lse
        return (self.part_o.view(-1)[: B * S * H * D].view(B, S, H, D), self.part_lse.view(-1)[: B * S * H].view(B, S, H))

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """``fused=False``: one token takes the unfused launches too (RoPE/append, attention, merge, ring commit)."""
        S, scale, cp, sp, stream = self._attend_args(l, qkv, out, cos, sin, scale)
        self._ensure_room(l, S)
        if S > self.max_q:
            return self._attend_chunk(l, qkv, S, scale, cp, sp, rope_mode, out, stream)
        st = self.state(l)
        B, h, lib = self.batch_size, self.handles[l], self.lib
        nfq = self.num_full_kv_head_list[l] * self.num_kv_groups
        po, pl = self.partials(S)
        fused = fused and S == 1 and qkv.stride(1) % 8 == 0 and qkv.data_ptr() % 16 == 0
        if not fused:
            self._launch(lib.duo_rope_append, h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode, S,
                         stream)
        if fused:  # one token: RoPE + owner-only append + slice attention + streaming heads + ring commit, one launch
            self._launch(getattr(lib, self._fused), h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cp, sp,
                         rope_mode & 0xFF, out.data_ptr(), po.data_ptr(), pl.data_ptr(), float(scale),
                         self.workspace.data_ptr(), self.workspace.numel(), stream, timed=True)
        else:
            self._launch(getattr(lib, self._attention), h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out.data_ptr(),
                         po.data_ptr(), pl.data_ptr(), S, float(scale), self.workspace.data_ptr(),
                         self.workspace.numel(), stream, timed=True)
        if nfq:
            self.seq.comm.merge(po, pl, out, B * S, self.num_heads, nfq)
            self.launch_count += 1
        if not fused:
            self._launch(lib.duo_stream_commit, h, C.byref(st), S, stream,
                         count=1 if self.num_streaming_kv_head_list[l] > 0 else 0)
        self.advance(l, S)
        return out

    def _attend_chunk(self, l, qkv, S, scale, cp, sp, rope_mode, out, stream):
        """A chunk longer than ``max_q``: duo_rope_append (owned positions only) -> duo_prefill_seq on the rank's slice
        (INT4 caches: on the 16-bit image of it; chunks of group x q_len <= 16 there take duo_attention_seq) -> the
        row-scattered merge -> duo_stream_commit.  Streaming heads see the ring as it was before the chunk plus the
        whole chunk causally, as on an unsharded cache."""
        st = self.state(l)
        B, h, lib = self.batch_size, self.handles[l], self.lib
        nfq = self.num_full_kv_head_list[l] * self.num_kv_groups
        self._launch(lib.duo_rope_append, h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode, S, stream)
        po, pl = self.partials(S)
        ah, fn = h, lib.duo_prefill_seq
        if self.kv_format == "int4":
            ah = self._dequant_scratch(l, S)
            if S * self.num_kv_groups <= _C.DECODE_MAX_Q:
                fn = lib.duo_attention_seq
        ast = _C.CacheState(st.full_len, st.total, st.lo, None)  # a prefill chunk is sized from the host state
        ast.seq_rank, ast.seq_world, ast.seq_block = st.seq_rank, st.seq_world, st.seq_block
        self._launch(fn, ah, C.byref(ast), qkv.data_ptr(), qkv.stride(1), out.data_ptr(), po.data_ptr(), pl.data_ptr(),
                     S, float(scale), self.workspace.data_ptr(), self.workspace.numel(), stream, timed=True)
        if nfq:
            self.seq.comm.merge_scattered(po, pl, out, B * S, self.num_heads, nfq)
            self.launch_count += 1
        self._launch(lib.duo_stream_commit, h, C.byref(st), S, stream,
                     count=1 if self.num_streaming_kv_head_list[l] > 0 else 0)
        self.advance(l, S)
        return out

    def load_from_head_parallel(self, hp_cache: "DuoKVCache", head_plan, group=None):
        """Take over the contents of a head-parallel cache of the same ``kv_format`` (this rank's heads, all positions —
        what the prefill phase filled) by point-to-point resharding; streaming rings are all-gathered (they are tiny).
        Every tensor of a layer moves: for INT4 caches the codes and the fp16 scale / zero rows."""
        from . import tp

        if hp_cache.kv_format != self.kv_format:
            raise ValueError(f"{type(self).__name__} holds {self.kv_format!r} KV; the head-parallel cache holds "
                             f"{hp_cache.kv_format!r}")
        rank, world = self.seq.rank, self.seq.world
        for l in range(self.num_layers):
            n = hp_cache.kv_seq_len_list[l]
            mask_row = head_plan.mask[l]
            owners = head_plan.owners[l]
            for name, dst in self.tensors[l].items():  # the same order on every rank
                if not dst.numel():
                    continue
                if name.startswith("full"):
                    tp.reshard_heads_to_seq(hp_cache.tensors[l][name], owners, mask_row, rank, world, n, self.seq.block,
                                            dst, group)
                else:
                    tp.all_gather_rings(hp_cache.tensors[l][name], owners, mask_row, rank, world, self.W, dst, group)
            self.kv_seq_len_list[l] = n
            self.total_list[l] = hp_cache.total_list[l]
            self.lo_list[l] = hp_cache.lo_list[l]
        self.sync_device_state()
        return self


class DuoSeqShardINT4KVCache(DuoSeqShardKVCache):
    """:class:`DuoSeqShardKVCache` over the INT4 KV format of :class:`DuoAttentionStaticINT4KVCache` (136 B per retrieval
    head and key instead of 512 B): the layout for contexts whose INT4 cache does not fit one GPU.  Same constructor.

    ``attend`` = duo_rope_append (K1-quantises only the positions this rank owns) -> duo_attention_seq_int4 ->
    duo_seq_merge -> duo_stream_commit, or one duo_decode_fused_seq_int4 launch for one token, for chunks of
    ``group x q_len <= 8`` packed rows.  A longer chunk dequantises the rank's slice into a 16-bit image and attends
    that (duo_prefill_seq, or duo_attention_seq for group x q_len <= 16), then merges scattered by rows.  An INT4 cache's first chunk attends the raw 16-bit K/V, which a sharded decode
    never sees: prefill head-parallel (``DuoAttentionStaticINT4KVCache``) and ``load_from_head_parallel``; ``attend`` on
    an empty layer raises ``ValueError``."""

    _KV = "int4"
    max_rows = _C.DECODE_MAX_Q_INT4
    _attention = "duo_attention_seq_int4"
    _fused = "duo_decode_fused_seq_int4"

    def _check_chunk(self, l, q_len):
        super()._check_chunk(l, q_len)
        if self.kv_seq_len_list[l] == 0 and self.total_list[l] == 0:
            raise ValueError(f"{type(self).__name__}: layer {l} is empty; an INT4 cache's first chunk attends the raw "
                             "K/V: prefill head-parallel and move the caches over with load_from_head_parallel()")


class DuoAttentionStaticINT4KVCache(DuoAttentionStaticKVCache):
    """Drop-in for the demo's INT4 cache (demo/int4_kv.py:115-260): same constructor arguments.  Storage is the
    packed-nibble + fp16 scale/zero format of demo/quantize_int4.cu in head-major order; there is no 16-bit scratch
    copy of the cache and no per-step ``get()`` dequantisation pass — the attention kernel dequantises in its
    K/V load stage.  The model may run in fp16 (as in the demo, run_duo_w8a8kv4.py:41-45) or bf16; with bf16
    activations K, V and q must lie within fp16's finite range (the format's scale / zero are fp16, and the kernels'
    inner loop is fp16)."""

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                 prefilling_chunk_size):
        super().__init__(model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                         prefilling_chunk_size=prefilling_chunk_size, kv_format="int4")


# ---- ragged batches: every batch row has its own occupancy (duo_decode_ragged) ----------------------------------
def ragged_want(batch: int, n_full: int, n_stream: int, sm_count: int = 132, *, ctas_per_sm: int = 2) -> int:
    """Split budget per (row, retrieval head) at equal lengths: ``split_want`` (duo_common.cuh) as ragged_geom
    calls it, ``ctas_per_sm`` CTAs per SM minus the streaming CTAs, capped at 512."""
    budget, stream_ctas = ctas_per_sm * sm_count, batch * n_stream
    want = (budget - stream_ctas if budget - stream_ctas > 0 else 1) // (batch * max(n_full, 1))
    return min(max(want, 1), 512)


def ragged_keys_per_split(n_sum: int, n_max: int, batch: int, want: int, *, tile: int = 64,
                          min_keys: int = 256) -> int:
    """Host twin of duo_common.cuh's ragged_keys_per_split: the decode split policy of ``plan_splits`` (>= ``min_keys``
    keys per split, <= ``want`` and <= 512 splits, ``tile``-key tiles) applied to the mean row length, raised so that
    no row needs more than 512 splits."""
    lbar = -(-n_sum // batch)
    s = min(max(1, -(-lbar // min_keys)), want, 512)
    kps = max(tile, -(-(-(-lbar // s)) // tile) * tile)
    cap = -(-(-(-n_max // 512)) // tile) * tile
    return max(kps, cap)


# The partition policy of duo_decode_ragged_int4 (the keys-as-M INT4 decode kernel): 128-key tiles, >= 1024 keys per
# split, 4 CTAs per SM.  Its rows have full_len + q_len keys (the new tokens are cache rows of the last split).
INT4_RAGGED_POLICY = {"tile": 128, "min_keys": 1024, "ctas_per_sm": 4}


def ragged_partition(lengths: Sequence[int], n_full: int, n_stream: int, sm_count: int = 132, *, tile: int = 64,
                     min_keys: int = 256, ctas_per_sm: int = 2) -> dict:
    """The retrieval-head key partition every CTA of a ragged decode launch derives from the row key counts
    ``lengths``: row ``b`` takes ``splits[b]`` consecutive slots of the ``slots`` grid slots per retrieval head, split
    ``i`` covering keys ``[i * keys_per_split, (i + 1) * keys_per_split)``.  ``slots`` depends on the geometry only.
    The defaults are duo_decode_ragged's policy; ``**INT4_RAGGED_POLICY`` gives duo_decode_ragged_int4's."""
    B = len(lengths)
    want = ragged_want(B, n_full, n_stream, sm_count, ctas_per_sm=ctas_per_sm)
    kps = ragged_keys_per_split(sum(lengths), max(lengths), B, want, tile=tile, min_keys=min_keys)
    splits = [max(1, -(-int(n) // kps)) for n in lengths]
    return {"want": want, "slots": B * (want + 1), "keys_per_split": kps, "splits": splits}


# ---- per-row capacities: one retrieval pool per layer (duo_layer_create_pooled) ------------------------------------
POOL_ALIGN = 128  # a 64-key (16-bit) or 128-key (INT4) tile never crosses into a neighbour's region


def _round_up(n: int, align: int) -> int:
    return -(-int(n) // align) * align


def pool_layout(capacities: Sequence[int], pool_size: Optional[int] = None, align: int = POOL_ALIGN) -> dict:
    """Regions of a pooled ragged cache: row ``b`` owns the pool tokens ``[first[b], first[b] + cap[b])``, ``cap[b]`` its
    capacity rounded up to ``align``, rows laid out in order.  ``pool_tokens`` is the sum of the regions, or
    ``pool_size`` rounded up to ``align`` when that is larger (headroom for :meth:`DuoRaggedKVCache.resize_row`)."""
    caps = [int(c) for c in capacities]
    if not caps or min(caps) < 1:
        raise ValueError(f"per-row capacities must be >= 1 (got {caps})")
    cap = [_round_up(c, align) for c in caps]
    first = [sum(cap[:b]) for b in range(len(cap))]
    pool_tokens = sum(cap)
    if pool_size is not None:
        if _round_up(pool_size, align) < pool_tokens:
            raise ValueError(f"pool_size {pool_size} is smaller than the {pool_tokens} tokens the row capacities need")
        pool_tokens = _round_up(pool_size, align)
    return {"first": first, "cap": cap, "pool_tokens": pool_tokens}


def pool_first_fit(first: Sequence[int], cap: Sequence[int], b: int, capacity: int, pool_tokens: int,
                   align: int = POOL_ALIGN) -> int:
    """First token of the lowest free ``align``-aligned range of the pool that holds ``capacity`` tokens for row ``b``,
    every other row keeping its region ``[first, first + cap)`` (row ``b``'s own region counts as free).
    ``ValueError`` if no range fits."""
    need = _round_up(capacity, align)
    pos = 0
    for lo, hi in sorted((f, f + c) for i, (f, c) in enumerate(zip(first, cap)) if i != b):
        if lo - pos >= need:
            return pos
        pos = max(pos, hi)
    if pool_tokens - pos >= need:
        return pos
    raise ValueError(f"no free range of {need} tokens for row {b} in the pool of {pool_tokens} tokens "
                     f"(regions of the other rows: {sorted((f, c) for i, (f, c) in enumerate(zip(first, cap)) if i != b)})")


def _shared_with_parent(name):
    """Attribute of a row that lives on its parent, shared by every row (see _RaggedRow)."""
    return property(lambda self: getattr(self._parent, name, None), lambda self, v: setattr(self._parent, name, v))


class _RaggedRow(DuoKVCache):
    """Batch-1 view of row ``b`` of a :class:`DuoRaggedKVCache`: its tensors are row ``b`` of the parent's, its layer
    handles are its own, and it owns that row's occupancy.  Every path of a batch-1 cache of the parent's
    ``kv_format`` works on it (wgmma prefill, small chunks, one-launch decode, ``evict_last``, ``clear``; for INT4 also
    the raw first chunk and the dequantised image of chunks >= 128 tokens) with the same bits."""

    # The 16-bit scratch of the INT4 paths (_first_chunk_scratch, _dequant_scratch) serves one attention call at a
    # time, and every row has the same geometry: the rows share one of each, held (and released) by the parent (an
    # image per row would cost ~2 GB per row at 512K capacity with 8 retrieval heads).
    _scratch = _shared_with_parent("_scratch")
    _dq = _shared_with_parent("_dq")

    def __init__(self, parent: "DuoRaggedKVCache", b: int):
        self._parent, self._row = parent, b
        super().__init__(parent.num_layers, parent.num_heads, parent.num_kv_heads, parent.head_dim,
                         parent.num_full_kv_head_list, 1, parent.row_capacities[b], parent.sink_size,
                         parent.recent_size, parent.dtype, parent.device, stage_cap=parent.stage_cap_list[0],
                         kv_format=parent.kv_format, workspace=parent.workspace)

    def _alloc_layer(self, l, full_cap, stage_cap, old=None):
        b, P = self._row, self._parent
        if not P.pooled:
            return {k: v[b : b + 1] for k, v in P.tensors[l].items()}
        # pooled: the row's region of the pool, [1][n_full][cap][..] from pool row first * n_full
        first, cap = P._geom[b]
        nf = self.num_full_kv_head_list[l]
        return {k: (v[first * nf : (first + cap) * nf].view(1, nf, cap, *v.shape[1:]) if k.startswith("full")
                    else v[b : b + 1]) for k, v in P.tensors[l].items()}

    def _owned_handles(self) -> list:
        return list(self.handles)  # the shared 16-bit image is the parent's

    def _ensure_room(self, l, q_len):
        if q_len > self.stage_cap_list[l]:  # a longer staging area is grown for every row of the parent
            self._parent._grow_layer(l, q_len)
        super()._ensure_room(l, q_len)

    def attend(self, l, *args, **kwargs):
        out = super().attend(l, *args, **kwargs)
        self._parent.rows_changed = True
        return out

    def clear(self):
        super().clear()
        self._parent.rows_changed = True
        self._parent.sync_device_state()

    def evict_last(self, num_tokens):
        super().evict_last(num_tokens)
        self._parent.rows_changed = True
        self._parent.sync_device_state()


class DuoRaggedKVCache(DuoKVCache):
    """A batch of sequences of different lengths, decoded together: one ``duo_decode_ragged`` launch per layer and
    step serves every row at its own length, so a batch of requests shares each pass over the weights.

    Same constructor arguments as :class:`DuoAttentionStaticKVCache` (16-bit KV only; INT4 KV:
    :class:`DuoRaggedINT4KVCache`).  Prefill, continue, evict or clear one row through ``cache.row(b)``, a batch-1
    cache that shares row ``b``'s buffers; pass the parent as ``past_key_values`` for batched decode steps
    (``group * q_len <= max_rows``).  ``row_lengths`` / ``lengths`` give the per-row retrieval lengths;
    ``evict_last`` / ``clear`` act on every row.  A finished row can be cleared and refilled with a new prompt while
    the others keep decoding (continuous batching).

    ``max_size`` is one capacity for every row, or a sequence of ``batch_size`` per-row capacities.  The latter selects
    the pooled layout: the retrieval K/V of all rows share one pool per layer, row ``b`` owning a region of its own
    capacity (rounded up to 128 tokens), so a batch of one long and several short rows reserves what the rows need,
    not ``batch_size`` times the longest.  ``pool_size=`` (tokens) reserves headroom beyond the rows' regions, and
    ``resize_row(b, capacity)`` moves an empty row to a region of another size, also while a ``DuoDecodeGraph`` is
    attached.  ``row_capacities`` gives the per-row capacities."""

    _KV = "same"                    # the one kv_format of the class
    max_rows = _C.DECODE_MAX_Q      # packed rows (group x q_len) of one batched step
    _decode = "duo_decode_ragged"   # its C entry point and workspace size
    _ws_bytes = "duo_ragged_workspace_bytes"

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                 prefilling_chunk_size: int = 64, kv_format: str = "same", pool_size: Optional[int] = None):
        self._check_args(batch_size, kv_format)
        self._init_ragged(**model_geometry(model, full_attention_heads), batch_size=batch_size, max_size=max_size,
                          sink_size=sink_size, recent_size=recent_size, stage_cap=prefilling_chunk_size,
                          pool_size=pool_size)

    @classmethod
    def from_geometry(cls, num_layers, num_heads, num_kv_heads, head_dim, num_full_kv_head_list, batch_size, max_size,
                      sink_size, recent_size, dtype, device, stage_cap: int = 64, kv_format: Optional[str] = None,
                      pool_size: Optional[int] = None):
        """Construct from the raw geometry (the argument list of :class:`DuoKVCache`) instead of a model."""
        cls._check_args(batch_size, cls._KV if kv_format is None else kv_format)
        self = cls.__new__(cls)
        self._init_ragged(num_layers, num_heads, num_kv_heads, head_dim, num_full_kv_head_list, batch_size, max_size,
                          sink_size, recent_size, dtype, device, stage_cap, pool_size)
        return self

    @classmethod
    def _check_args(cls, batch_size, kv_format):
        if kv_format != cls._KV:
            raise ValueError(f"{cls.__name__}: kv_format {kv_format!r} is not supported yet ({cls._KV!r} KV only; "
                             "INT4 KV: DuoRaggedINT4KVCache)")
        if not 1 <= int(batch_size) <= _C.RAGGED_MAX_BATCH:
            raise ValueError(f"{cls.__name__}: batch_size {batch_size} outside [1, {_C.RAGGED_MAX_BATCH}]")

    def _init_ragged(self, num_layers, num_heads, num_kv_heads, head_dim, num_full_kv_head_list, batch_size, max_size,
                     sink_size, recent_size, dtype, device, stage_cap, pool_size=None):
        if not isinstance(max_size, numbers.Integral):  # per-row capacities: the pooled layout
            caps = [int(c) for c in max_size]
            if len(caps) != int(batch_size):
                raise ValueError(f"{type(self).__name__}: {len(caps)} row capacities for batch_size {batch_size}")
            lay = pool_layout(caps, pool_size)
            self.pooled = True
            self._row_caps = caps                                   # logical capacities (what rows report / enforce)
            self._geom = [list(x) for x in zip(lay["first"], lay["cap"])]  # {first, cap} per row, 128-aligned tokens
            self.pool_tokens = lay["pool_tokens"]
            max_size = max(caps)
        elif pool_size is not None:
            raise ValueError(f"{type(self).__name__}: pool_size needs per-row capacities (a sequence as max_size)")
        self.rows = []  # the batch-1 views, made once the tensors exist
        super().__init__(num_layers, num_heads, num_kv_heads, head_dim, num_full_kv_head_list, batch_size, max_size,
                         sink_size, recent_size, dtype, device, stage_cap=stage_cap, kv_format=self._KV, growable=False)
        need = getattr(self.lib, self._ws_bytes)(self.batch_size, num_kv_heads)
        if need > self.workspace.numel():
            self.workspace = torch.zeros(need, dtype=torch.uint8, device=self.device)
        self.row_state = torch.zeros(self.batch_size, 4, dtype=torch.int64, device=self.device)  # {full_len, total, lo, 0}
        if self.pooled:  # read by the pooled kernels at launch: resize_row rewrites it without a re-capture
            self.row_geom = torch.tensor(self._geom, dtype=torch.int64, device=self.device)
        self.dev_state = self.row_state  # always device-resident: the driver advances it after every step
        self.rows = [_RaggedRow(self, b) for b in range(self.batch_size)]
        self.sync_device_state()

    # ---- rows ---------------------------------------------------------------------------------------------------
    def row(self, b: int) -> DuoKVCache:
        return self.rows[b]

    @property
    def row_lengths(self) -> List[int]:
        return [r.kv_seq_len for r in self.rows]

    @property
    def row_capacities(self) -> List[int]:
        """Token capacity of every row's retrieval cache."""
        return list(self._row_caps) if self.pooled else [self.max_size] * self.batch_size

    def _set_layer(self, l, full_cap, stage_cap):
        super()._set_layer(l, full_cap, stage_cap)
        for r in self.rows:  # the rows view the new tensors
            r._set_layer(l, r.full_cap_list[l], stage_cap)

    def resize_row(self, b: int, capacity: int):
        """Give the empty row ``b`` a region of ``capacity`` tokens: the first free 128-aligned range of the pool that
        fits (its old region counts as free).  ``ValueError`` if the row holds tokens or no range fits.  The pool is
        never re-allocated and the kernels read the row geometry from device memory, so this is allowed while a
        ``DuoDecodeGraph`` is attached (refill the row through ``row(b)`` afterwards, as after ``clear``)."""
        if not self.pooled:
            raise ValueError(f"{type(self).__name__}: resize_row needs per-row capacities (a sequence as max_size)")
        r = self.rows[b]
        if any(r.kv_seq_len_list) or any(r.total_list):
            raise ValueError(f"{type(self).__name__}: row {b} is not empty (length {r.kv_seq_len}): clear it before "
                             "resize_row")
        capacity = int(capacity)
        if capacity < 1:
            raise ValueError(f"{type(self).__name__}: capacity {capacity} < 1")
        first = pool_first_fit([g[0] for g in self._geom], [g[1] for g in self._geom], b, capacity, self.pool_tokens)
        self._geom[b] = [first, _round_up(capacity, POOL_ALIGN)]
        self._row_caps[b] = capacity
        self.row_geom[b].copy_(torch.tensor(self._geom[b], dtype=torch.int64))  # stream-ordered, like row_state
        r.max_size = capacity
        for l in range(self.num_layers):
            r._set_layer(l, capacity, r.stage_cap_list[l])
        self.rows_changed = True

    @property
    def lengths(self) -> torch.Tensor:
        """Device view of the rows' retrieval lengths (``row_state[:, 0]``)."""
        return self.row_state[:, 0]

    @property
    def kv_seq_len(self):
        """Length of the longest row."""
        return max(self.row_lengths)

    @property
    def streaming_kv_seq_len(self):
        return max(r.streaming_kv_seq_len for r in self.rows)

    def clear(self):
        for r in self.rows:
            DuoKVCache.clear(r)
        self.rows_changed = True
        self.sync_device_state()

    def evict_last(self, num_tokens):
        for r in self.rows:
            DuoKVCache.evict_last(r, num_tokens)
        self.rows_changed = True
        self.sync_device_state()

    def advance(self, l, q_len):
        for r in self.rows:
            r.advance(l, q_len)

    def state(self, l):
        raise TypeError("DuoRaggedKVCache has one occupancy per row: use row(b).state(l) or row_state")

    def snapshot_state(self):
        return [r.snapshot_state() for r in self.rows]

    def restore_state(self, snap):
        for r, s in zip(self.rows, snap):
            r.restore_state(s)

    def check_room(self, q_len, layers=None):
        for r in self.rows:  # every row against its own capacity
            r.check_room(q_len, layers)

    # ---- device-resident occupancy ----------------------------------------------------------------------------------
    def enable_device_state(self):
        self.sync_device_state()
        return self

    def sync_device_state(self, l: Optional[int] = None):
        """row_state := the rows' host occupancy of layer ``l`` (default: the last layer), stream-ordered."""
        l = self.num_layers - 1 if l is None else l
        host = torch.tensor([[r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l], 0] for r in self.rows],
                            dtype=torch.int64)
        self.row_state.copy_(host)

    def advance_device(self, n):
        self._launch(self.lib.duo_ragged_state_advance, self.row_state.data_ptr(), self.batch_size, int(n),
                     self.sink_size, self.recent_size, torch.cuda.current_stream(self.device).cuda_stream)

    # ---- batched decode step -----------------------------------------------------------------------------------------
    def check_rows(self, layers: Sequence[int]):
        """Raise ValueError if a row cannot join a batched step of these layers (16-bit caches: every row can)."""

    def _check_chunk(self, l, q_len):
        if q_len * self.num_kv_groups > self.max_rows:
            raise ValueError(f"{type(self).__name__} decodes chunks of group x q_len <= {self.max_rows} rows (got "
                             f"{q_len} tokens): prefill each row through cache.row(b)")
        self.check_rows([l])

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """One decode-sized chunk for every row, one ``duo_decode_ragged`` launch.  ``qkv`` ``[B, S, (Hq + 2 Hkv) * D]``
        (rows 16-byte aligned), ``cos`` / ``sin`` ``[B, S, D]`` per-row tables (or None with ROPE_NONE), ``out``
        ``[B, S, Hq, D]`` contiguous."""
        S, scale, cp, sp, stream = self._attend_args(l, qkv, out, cos, sin, scale)
        if cos is not None:
            assert cos.shape == (self.batch_size, S, self.head_dim) and cos.is_contiguous() and sin.is_contiguous()
        self.check_room(S, [l])
        if not self.graph_attached:  # eager: the rows' host occupancy is authoritative
            self.sync_device_state(l)
        lens = [r.kv_seq_len_list[l] for r in self.rows]
        if self.pooled:
            min_room = min(c - n for c, n in zip(self._row_caps, lens))
            self._launch(self.lib.duo_decode_ragged_pooled, self.handles[l], self.row_state.data_ptr(),
                         self.row_geom.data_ptr(), min_room, qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode & 0xFF,
                         out.data_ptr(), S, float(scale), self.workspace.data_ptr(), self.workspace.numel(), stream,
                         timed=True)
        else:
            self._launch(getattr(self.lib, self._decode), self.handles[l], self.row_state.data_ptr(), max(lens),
                         qkv.data_ptr(), qkv.stride(1), cp, sp, rope_mode & 0xFF, out.data_ptr(), S, float(scale),
                         self.workspace.data_ptr(), self.workspace.numel(), stream, timed=True)
        self.advance(l, S)
        return out


class DuoRaggedINT4KVCache(DuoRaggedKVCache):
    """:class:`DuoRaggedKVCache` over the INT4 KV format of :class:`DuoAttentionStaticINT4KVCache` (136 B per retrieval
    head and key instead of 512 B at 16 bits): one ``duo_decode_ragged_int4`` launch per layer and step.  Same
    constructor arguments as :class:`DuoAttentionStaticINT4KVCache` (plus ``from_geometry``); fp16 or bf16 models.

    ``row(b)`` is a full batch-1 INT4 cache: a row's first chunk attends the raw 16-bit K/V (as the reference's first
    call does), later chunks of >= 128 tokens attend a dequantised image, small chunks and decode steps the INT4
    kernels.  The rows share one such image and one first-chunk scratch.  Batched steps take ``group x q_len <= 8``
    rows, and every row must have been prefilled through ``row(b)`` first: an empty row's first call must attend its
    raw K/V, which the batched kernel never sees."""

    _KV = "int4"
    max_rows = _C.DECODE_MAX_Q_INT4
    _decode = "duo_decode_ragged_int4"
    _ws_bytes = "duo_ragged_int4_workspace_bytes"

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                 prefilling_chunk_size: int = 64, pool_size: Optional[int] = None):
        super().__init__(model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                         prefilling_chunk_size=prefilling_chunk_size, kv_format="int4", pool_size=pool_size)

    def check_rows(self, layers: Sequence[int]):
        for b, r in enumerate(self.rows):
            for l in layers:
                if r.kv_seq_len_list[l] == 0 and r.total_list[l] == 0:
                    raise ValueError(f"{type(self).__name__}: row {b} is empty; its first chunk attends the raw K/V: "
                                     "prefill it through cache.row(b)")
