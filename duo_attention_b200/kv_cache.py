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
import weakref
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import _C

PREFILL_MAX_WINDOW = 2048  # the most sink + recent slots the wgmma prefill kernel's streaming validity table holds


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


def _refuse_pending(cache, what: str):
    """ValueError while ``cache`` holds a verify chunk awaiting ``accept`` (see DuoKVCache.verify)."""
    S = getattr(cache, "pending_verify", None)
    if S:
        raise ValueError(f"{type(cache).__name__}: a verify chunk of {S} tokens awaits accept(): {what} is refused "
                         "until it is accepted (or the cache cleared)")


class _Call(NamedTuple):
    """One attention call as the C entry points take it (``DuoKVCache._attend_call``); pointers are ints."""
    S: int            # tokens per row
    scale: float
    stream: int
    qkv: tuple        # (pointer, row stride in elements)
    cos_sin: tuple    # RoPE table pointers (None with ROPE_NONE)
    out: int
    ws: tuple         # workspace (pointer, bytes)

    @property
    def aligned(self) -> bool:
        """Whether the qkv rows are 16-byte aligned, as the one-launch kernels load them."""
        return self.qkv[1] % 8 == 0 and self.qkv[0] % 16 == 0


class DuoKVCache:
    pooled = False      # per-row capacities of a DuoRaggedKVCache: the retrieval K/V in one pool per layer
    seq = None          # a DuoSeqShardKVCache's rank, world, block and exchange: state() adds its shard descriptor
    rows_changed = False  # a row changed on the host since the last DuoDecodeGraph.resync() (ragged caches only)
    _verifies = True    # the class takes verify chunks (verify / accept)

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
        self._verify_len = [0] * num_layers      # per layer: tokens of a verify chunk awaiting accept (0: none)
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
    def _dequant_scratch(self, l, S, prefix=None):
        """Image of layer ``l``'s INT4 cache in the activation dtype for ONE attention call of a chunk of >= 128 tokens — what the
        reference does on EVERY call (``get()`` dequantises the whole cache, demo/int4_kv.py:373-436, then
        flash_attn_func runs on it, demo/w8a8kv4_llama.py:239-274).  For such a chunk the O(ctx) dequantisation pass
        is < 1 % of the chunk x ctx attention, and the attention runs on the tensor-core prefill kernel.  Decode and small chunks never
        come here: their kernels dequantise in the K/V load stage.  fp16 layers get K2's fp16 values
        (duo_dequant_int4), bf16 layers bf16_rn(fma(code, scale, zero)) (duo_dequant_int4_bf16).  One flat
        zero-initialised buffer is shared by all layers (they are processed one after the other; rows beyond the
        dequantised range hold zeros or finite leftovers and are masked); a layer handle is created per distinct
        number of retrieval heads, and released with the image.  ``prefix = (tensors, P)`` (a sharer, batch 1): image
        rows ``[0, P)`` are the donor's region rows ``[0, P)`` and the own region's rows follow at image row ``P``, so
        the image is the one of a row holding a copy of the prompt."""
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
        P = prefix[1] if prefix is not None else 0
        # retrieval rows: (source tensors, first image row, rows), the donor's prefix first for a sharer
        parts = ((t, 0, n_rows),) if P == 0 else ((prefix[0], 0, P), (t, P, n_rows - P))
        for b in range(B):
            for hh in range(nf):
                for name, dst in (("full_k", fk), ("full_v", fv)):
                    for src, d0, rows in parts:
                        self._launch(dequant, src[name][b, hh].data_ptr(), src[name + "_scale"][b, hh].data_ptr(),
                                     src[name + "_zero"][b, hh].data_ptr(), rows, dst[b, hh, d0:].data_ptr(), stream)
            for hh in range(ns):
                for name, dst in (("ring_k", rk), ("ring_v", rv)):
                    for src0, dst0, rows in ((0, 0, W), (so, W, S)):
                        self._launch(dequant, t[name][b, hh, src0:].data_ptr(),
                                     t[name + "_scale"][b, hh, src0:].data_ptr(),
                                     t[name + "_zero"][b, hh, src0:].data_ptr(), rows, dst[b, hh, dst0:].data_ptr(),
                                     stream)
        return sc["handles"][nf]

    def state(self, l, host=False, prefix=0) -> _C.CacheState:
        """Layer ``l``'s occupancy as the kernels take it: with ``dev_state`` when it is enabled, unless ``host`` (a
        chunk sized from the host integers), and a sharded cache's shard descriptor.  ``prefix``: the state of the own
        region that follows ``prefix`` shared keys (``full_len - prefix``)."""
        ds = self.dev_state.data_ptr() if self.dev_state is not None and not host else None
        st = _C.CacheState(self.kv_seq_len_list[l] - prefix, self.total_list[l], self.lo_list[l], ds)
        if self.seq is not None:
            st.seq_rank, st.seq_world, st.seq_block = self.seq.rank, self.seq.world, self.seq.block
        return st

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
        self._verify_len = [0] * self.num_layers  # a pending verify chunk is discarded
        self.sync_device_state()

    def evict_last(self, num_tokens):
        _refuse_pending(self, "evict_last")
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
        _refuse_pending(self, "attend")
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        S = call.S
        self._ensure_room(l, S)
        st = self.state(l)
        h = self.handles[l]
        first_int4 = self.kv_format == "int4" and st.full_len == 0 and st.total == 0
        # decode-sized chunks take ONE launch: 16-bit caches up to 16 packed rows, INT4 caches up to 8 (the keys-as-M
        # kernel) — except the very first INT4 call, which attends the raw 16-bit K/V (see below)
        one_launch = (S * self.num_kv_groups <= _C.DECODE_MAX_Q if self.kv_format == "same" else
                      S * self.num_kv_groups <= _C.DECODE_MAX_Q_INT4 and not first_int4)
        if one_launch and fused and not force_mma and call.aligned:
            # decode-sized chunk: RoPE + append + attention + ring commit in ONE launch (q is not written back)
            self._launch(self.lib.duo_decode_fused, h, C.byref(st), *call.qkv, *call.cos_sin, rope_mode & 0xFF,
                         call.out, S, call.scale, *call.ws, call.stream, timed=True)
            self.advance(l, S)
            return out
        self._rope_append(h, call, st, rope_mode)
        ah, ast = h, st
        if first_int4:
            # The reference attends the RAW 16-bit K/V on the very first call and only later calls see the
            # quantise->dequantise round trip (demo/w8a8kv4_llama.py:229-238 vs :239-274).  The chunk has just
            # been quantised into the INT4 cache above; attention for this one call runs on a 16-bit scratch layer
            # of the activation dtype
            # (every head is plain causal on the first call, so all heads are "retrieval" there).
            sc = self._first_chunk_scratch(S)
            ah, ast = sc.handles[0], _C.CacheState(0, 0, sc.sink_size)
            self._rope_append(ah, call, ast, rope_mode | _C.ROPE_SKIP_Q)
        elif self._attends_image(S) and not force_mma:
            ah, ast = self._dequant_scratch(l, S), self.state(l, host=True)
        fn = self.lib.duo_attention_mma if force_mma else self.lib.duo_attention
        return self._attend_commit(l, call, st, out, fn, (ah,), ast)

    def _attends_image(self, S) -> bool:
        """Whether a chunk of ``S`` tokens on this INT4 cache attends its layer's 16-bit image (``_dequant_scratch``)."""
        return self.kv_format == "int4" and S >= 128 and self.W <= PREFILL_MAX_WINDOW

    def _rope_append(self, h, call, st, rope_mode):
        """``duo_rope_append`` of the chunk's K/V into the layer ``h`` at ``st`` (q rotated in place unless
        ``rope_mode`` has ``ROPE_SKIP_Q``)."""
        self._launch(self.lib.duo_rope_append, h, C.byref(st), *call.qkv, *call.cos_sin, rope_mode, call.S, call.stream)

    def _attend_commit(self, l, call, st, out, fn, head, ast, partials=None, scattered=False):
        """The rest of a chunk that ``_rope_append`` placed at ``st``: the attention launch ``fn(*head, ast, ...)``
        (timed), the merge of a sharded cache's slice ``partials``, the ring commit at ``st``, ``advance``."""
        parts = () if partials is None else (partials[0].data_ptr(), partials[1].data_ptr())
        self._launch(fn, *head, C.byref(ast), *call.qkv, call.out, *parts, call.S, call.scale, *call.ws, call.stream,
                     timed=True)
        if partials is not None:
            self._merge(l, out, call.S, *partials, scattered)
        self._commit(l, st, call.S, call.stream)
        self.advance(l, call.S)
        return out

    def _commit(self, l, st, n, stream):
        """``duo_stream_commit`` of ``n`` staged tokens at ``st`` (a layer without streaming heads launches nothing)."""
        self._launch(self.lib.duo_stream_commit, self.handles[l], C.byref(st), n, stream,
                     count=1 if self.num_streaming_kv_head_list[l] > 0 else 0)

    # ---- verifying drafted tokens (speculative decoding, DESIGN §2) -------------------------------------------------
    @property
    def pending_verify(self) -> Optional[int]:
        """Tokens of the verify chunk awaiting ``accept`` (None: none)."""
        return max(getattr(self, "_verify_len", None) or [0]) or None  # (caches built without __init__ hold none)

    def _check_verify(self, l, S, max_rows):
        """ValueError, before anything changes, for a verify chunk of ``S`` tokens on layer ``l`` that this cache does
        not take."""
        name = type(self).__name__
        if self.kv_format != "same":
            raise ValueError(f"{name}: INT4 caches cannot verify drafts")
        if not self._verifies:
            raise ValueError(f"{name}: sequence-sharded caches cannot verify drafts")
        if self.graph_attached:
            raise ValueError(f"{name}: verify chunks are not captured by a DuoDecodeGraph: detach it first")
        if S < 1 or S * self.num_kv_groups > max_rows:
            raise ValueError(f"{name}: a verify chunk takes group x S <= {max_rows} rows (got {S} tokens at group "
                             f"{self.num_kv_groups})")
        if S > self.recent_size:
            raise ValueError(f"{name}: a verify chunk of {S} tokens exceeds recent_size {self.recent_size}")
        pend = self.pending_verify
        if self._verify_len[l] or (pend is not None and pend != S):
            raise ValueError(f"{name}: a verify chunk of {pend} tokens awaits accept(): layer {l} cannot take another")

    def _accept_len(self) -> int:
        """The pending chunk's length: every layer must hold one, of one length."""
        S = self._verify_len[0]
        if not S or any(n != S for n in self._verify_len):
            raise ValueError(f"{type(self).__name__}: accept() needs a verify chunk on every layer (pending per layer: "
                             f"{self._verify_len})")
        return S

    def verify(self, l, qkv, cos, sin, rope_mode, out, scale=None):
        """Attend a chunk of drafts on layer ``l`` without committing it: token t of the chunk gets exactly the keys a
        one-token ``attend`` at its position would see after tokens 0 .. t - 1 (DESIGN §2), the retrieval K/V are
        appended past the current length, the streaming K/V are staged, and no occupancy moves.  ``accept(a)`` keeps
        the first ``a`` tokens.  Arguments as for ``attend``.  group x S <= 16 takes one launch
        (``duo_decode_verify``), up to 64 rows ``duo_rope_append`` + ``duo_attention_verify`` (q rotated in place).
        ``ValueError`` before anything changes for INT4 and sequence-sharded caches, an attached ``DuoDecodeGraph``,
        more rows, S > recent_size, or a layer that already holds a pending chunk.  A growable cache grows first."""
        S = qkv.shape[1]
        self._check_verify(l, S, _C.VERIFY_MAX_ROWS)
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        self._ensure_room(l, S)
        st, h = self.state(l, host=True), self.handles[l]
        if S * self.num_kv_groups <= _C.DECODE_MAX_Q and call.aligned:
            self._launch(self.lib.duo_decode_verify, h, C.byref(st), *call.qkv, *call.cos_sin, rope_mode & 0xFF,
                         call.out, S, call.scale, *call.ws, call.stream, timed=True)
        else:
            self._rope_append(h, call, st, rope_mode)
            self._launch(self.lib.duo_attention_verify, h, C.byref(st), *call.qkv, call.out, S, call.scale, *call.ws,
                         call.stream, timed=True)
        self._verify_len[l] = S
        return out

    def accept(self, a: int):
        """Keep the first ``a`` tokens (0 <= a <= S) of the verify chunk every layer holds: their staged streaming rows
        are committed (``duo_stream_commit``) and length, total and lo advance by ``a``, on the host and in
        ``dev_state``.  The cache bytes are then those of ``a`` one-token steps on the same qkv rows."""
        S = self._accept_len()
        if isinstance(a, bool) or not isinstance(a, numbers.Integral) or not 0 <= int(a) <= S:
            raise ValueError(f"{type(self).__name__}: accept({a!r}) outside [0, {S}]")
        a = int(a)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for l in range(self.num_layers):
            if a:
                self._commit(l, self.state(l, host=True), a, stream)
            self.advance(l, a)
        self._verify_len = [0] * self.num_layers
        self.sync_device_state()

    def _attend_call(self, l, qkv, out, cos, sin, scale) -> _Call:
        """The checked call (``_attend_args``) as the entry points take it."""
        S, scale, cp, sp, stream = self._attend_args(l, qkv, out, cos, sin, scale)
        return _Call(S, float(scale), stream, (qkv.data_ptr(), qkv.stride(1)), (cp, sp), out.data_ptr(),
                     (self.workspace.data_ptr(), self.workspace.numel()))

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
    _verifies = False
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

    def _attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """``attend``: ``fused=False``: one token takes the unfused launches too (RoPE/append, attention, merge, ring
        commit)."""
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        S = call.S
        self._ensure_room(l, S)
        if S > self.max_q:
            return self._attend_chunk(l, call, rope_mode, out)
        st, h = self.state(l), self.handles[l]
        po, pl = self.partials(S)
        if fused and S == 1 and call.aligned:
            # one token: RoPE + owner-only append + slice attention + streaming heads + ring commit, one launch
            self._launch(getattr(self.lib, self._fused), h, C.byref(st), *call.qkv, *call.cos_sin, rope_mode & 0xFF,
                         call.out, po.data_ptr(), pl.data_ptr(), call.scale, *call.ws, call.stream, timed=True)
            self._merge(l, out, S, po, pl)
            self.advance(l, S)
            return out
        self._rope_append(h, call, st, rope_mode)
        return self._attend_commit(l, call, st, out, getattr(self.lib, self._attention), (h,), st, (po, pl))

    def _attend_chunk(self, l, call, rope_mode, out):
        """A chunk longer than ``max_q``: duo_rope_append (owned positions only) -> duo_prefill_seq on the rank's slice
        (INT4 caches: on the 16-bit image of it; chunks of group x q_len <= 16 there take duo_attention_seq) -> the
        row-scattered merge -> duo_stream_commit.  Streaming heads see the ring as it was before the chunk plus the
        whole chunk causally, as on an unsharded cache."""
        st, h = self.state(l), self.handles[l]
        self._rope_append(h, call, st, rope_mode)
        partials = self.partials(call.S)
        ah, fn = h, self.lib.duo_prefill_seq
        if self.kv_format == "int4":
            ah = self._dequant_scratch(l, call.S)
            if call.S * self.num_kv_groups <= _C.DECODE_MAX_Q:
                fn = self.lib.duo_attention_seq
        # a prefill chunk is sized from the host state
        return self._attend_commit(l, call, st, out, fn, (ah,), self.state(l, host=True), partials, scattered=True)

    def _merge(self, l, out, S, po, pl, scattered=False):
        """The exchange that merges every rank's slice partials of the retrieval heads into ``out`` (a layer without
        retrieval heads has none); ``scattered``: by rows, for a prefill-sized chunk."""
        nfq = self.num_full_kv_head_list[l] * self.num_kv_groups
        if nfq:
            merge = self.seq.comm.merge_scattered if scattered else self.seq.comm.merge
            merge(po, pl, out, self.batch_size * S, self.num_heads, nfq)
            self.launch_count += 1

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

    # ---- forks: continuations of this cache's prompt that read its slice in place (DuoSeqShardForkKVCache) --------
    _forks = None  # the live fork caches made from this one (a WeakSet), created by the first fork()

    def _check_no_forks(self, what: str):
        if self._forks:
            raise ValueError(f"{type(self).__name__}: cannot {what} while forks made from this cache are alive "
                             "(clear() them or drop them first)")

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        self._check_no_forks("attend")
        return self._attend(l, qkv, cos, sin, rope_mode, out, scale, force_mma, fused)

    def clear(self):
        self._check_no_forks("clear")
        super().clear()

    def evict_last(self, num_tokens):
        self._check_no_forks("evict_last")
        super().evict_last(num_tokens)

    def fork(self, batch_size: int, max_new_tokens: int) -> "DuoSeqShardForkKVCache":
        """``batch_size`` continuations of this batch-1 cache's prompt, decoded in lockstep (parallel sampling): see
        :class:`DuoSeqShardForkKVCache`.  This cache becomes the donor: it refuses ``attend``, ``evict_last`` and
        ``clear`` while the forks are alive."""
        return DuoSeqShardForkKVCache(self, batch_size, max_new_tokens)


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


def fork_prefix_len(n: int, world: int, block: int) -> int:
    """Positions the forks of an ``n``-token sharded prompt share with it: ``n`` rounded down to whole rounds of
    ``world * block``, so that position ``p >= P`` has the owner of ``p - P`` at local row ``local_index(p) - P / world``
    and every rank holds exactly ``P / world`` prefix rows."""
    rnd = world * block
    return n // rnd * rnd


def fork_tail_plan(n: int, max_new_tokens: int, plan) -> List[dict]:
    """Per rank: what ``fork`` copies into every row's own slice.  ``prefix_rows`` = P / world donor rows stay shared;
    the donor's local rows ``[prefix_rows, prefix_rows + tail_rows)`` (positions ``[P, n)``) move to own rows
    ``[0, tail_rows)``; ``own_cap`` rows hold the positions ``p - P < n - P + max_new_tokens``."""
    P = fork_prefix_len(n, plan.world, plan.block)
    return [{"P": P, "prefix_rows": P // plan.world, "tail_rows": plan.local_len(r, n - P),
             "own_cap": plan.capacity(n - P + max_new_tokens)} for r in range(plan.world)]


class DuoSeqShardForkKVCache(DuoSeqShardKVCache):
    """``batch_size`` continuations of one sequence-sharded prompt (``DuoSeqShardKVCache.fork``): parallel sampling
    (best-of-n, self-consistency) over a prompt whose KV only fits sharded.  The rows move in lockstep and share the
    donor's first ``P = fork_prefix_len(n, world, block)`` positions in place: each rank streams its ``P / world`` prefix
    rows once per step for the packed queries of all rows.  Every row owns a slice of the positions ``p >= P`` alone,
    laid out as a sharded cache of the positions ``p - P`` (the donor's tail ``[P, n)`` is copied there, as are its sink
    and ring slots), with room for ``max_new_tokens`` more (question tokens included).

    ``kv_seq_len`` counts logical tokens, so ``model(input_ids=[B, 1], past_key_values=forks)`` and ``DuoDecodeGraph``
    work unchanged.  One ``duo_decode_fused_seq_shared`` (two launches) per layer and step, then ``duo_seq_merge``.
    Every row may also take a prefill-sized chunk of the same length S (``group x S > 16``), e.g. its own question over a
    shared document: ``model(input_ids=[B, S], past_key_values=forks)``.  Its attention is ``duo_prefill_seq_shared``,
    then the row-scattered merge; the outputs are bit-identical to a batch-B sharded cache holding copies of the prompt.
    Refused with ``ValueError`` before any change: chunks of ``1 < S`` tokens with ``group x S <= 16``, any chunk while
    a ``DuoDecodeGraph`` is attached, with ``P > 0`` a chunk on a block that is not a multiple of 8, ``evict_last``
    below ``P``, forks of forks, and with ``P > 0`` a call that cannot take the forks' launches (``fused=False``,
    ``force_mma=True``, or qkv rows that are not 16-byte aligned: forks have no unfused step).  ``clear()`` releases the donor; the cleared forks
    are a plain sharded cache of their own capacity.  While a ``DuoDecodeGraph`` is attached, ``clear()`` is refused:
    the captured launches read the donor's prefix at a fixed ``P``.  With ``P = 0`` (a prompt shorter than one round)
    nothing is shared and every step is ``DuoSeqShardKVCache``'s."""

    def __init__(self, donor: DuoSeqShardKVCache, batch_size: int, max_new_tokens: int):
        name = type(donor).__name__
        if donor.kv_format != "same":
            raise ValueError(f"{name}: forks of an INT4 cache are not supported (16-bit sequence-sharded caches only)")
        if isinstance(donor, DuoSeqShardForkKVCache):
            raise ValueError(f"{name}: forks of forks are not supported")
        if donor.batch_size != 1:
            raise ValueError(f"{name}: the donor of fork() must be batch 1 (got {donor.batch_size})")
        lens = set(donor.kv_seq_len_list)
        if len(lens) != 1 or len(set(donor.total_list)) != 1 or len(set(donor.lo_list)) != 1:
            raise ValueError(f"{name}: fork() needs every layer at one length (got {sorted(lens)})")
        n = donor.kv_seq_len
        if n == 0:
            raise ValueError(f"{name}: fork() of an empty cache: there is no prompt to share")
        if int(batch_size) < 1 or int(max_new_tokens) < 0:
            raise ValueError(f"{name}: fork() needs batch_size >= 1 and max_new_tokens >= 0")
        B, seq = int(batch_size), donor.seq
        self.seq, self.plan = seq, donor.plan
        tail = fork_tail_plan(n, int(max_new_tokens), self.plan)[seq.rank]
        self.prefix_len, self.donor = tail["P"], donor
        nkv, lib = donor.num_kv_heads, donor.lib
        # the shared step's workspace, and a batch-B DuoSeqShardKVCache's, which holds the 64-row split-KV layout of a
        # prefill-sized chunk (duo_prefill_seq_shared partitions as duo_prefill_seq does) and every step with P = 0
        ws = max(lib.duo_seq_shared_workspace_bytes(B, nkv), lib.duo_workspace_bytes(B, nkv, donor.num_kv_groups,
                                                                                     _C.DECODE_MAX_Q))
        ws = torch.zeros(ws, dtype=torch.uint8, device=donor.device)
        DuoKVCache.__init__(
            self, donor.num_layers, donor.num_heads, nkv, donor.head_dim, donor.num_full_kv_head_list, B,
            n + int(max_new_tokens), donor.sink_size, donor.recent_size, donor.dtype, donor.device,
            stage_cap=self.max_rows, kv_format="same", growable=False, local_full_cap=tail["own_cap"] + 1,
            workspace=ws)  # (one spare row, as DuoSeqShardKVCache allocates)
        self.max_q = 1
        self.part_o = torch.zeros(B, 1, self.num_heads, self.head_dim, dtype=torch.float32, device=self.device)
        self.part_lse = torch.zeros(B, 1, self.num_heads, dtype=torch.float32, device=self.device)
        p0, tr, W = tail["prefix_rows"], tail["tail_rows"], self.W
        for l in range(self.num_layers):
            src, dst = donor.tensors[l], self.tensors[l]
            for name in ("full_k", "full_v"):
                if dst[name].numel() and tr:
                    dst[name][:, :, :tr].copy_(src[name][:, :, p0 : p0 + tr].expand(B, -1, -1, -1))
            for name in ("ring_k", "ring_v"):
                if dst[name].numel():
                    dst[name][:, :, :W].copy_(src[name][:, :, :W].expand(B, -1, -1, -1))
            self.kv_seq_len_list[l], self.total_list[l], self.lo_list[l] = n, donor.total_list[l], donor.lo_list[l]
        if donor._forks is None:
            donor._forks = weakref.WeakSet()
        donor._forks.add(self)

    def fork(self, batch_size: int, max_new_tokens: int):
        raise ValueError(f"{type(self).__name__}: forks of forks are not supported")

    def _rows_needed(self, l, q_len) -> int:
        return self.plan.local_len(self.seq.rank, self.kv_seq_len_list[l] - self.prefix_len + q_len)

    def _check_chunk(self, l, q_len):
        name = type(self).__name__
        if q_len != 1 and q_len * self.num_kv_groups <= _C.DECODE_MAX_Q:
            raise ValueError(f"{name}: forks take one token per row per step, or a prefill-sized chunk of group x q_len "
                             f"> {_C.DECODE_MAX_Q} rows (got a chunk of {q_len} at group {self.num_kv_groups})")
        if q_len != 1 and self.prefix_len and self.plan.block % 8:
            raise ValueError(f"{name}: chunks on forks of a shared prompt need a block that is a multiple of 8 (got block "
                             f"{self.plan.block}): the key tile across the donor's rows is loaded in 8-row pieces")
        super()._check_chunk(l, q_len)

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """One token per row: duo_decode_fused_seq_shared (prefix rows shared, own slices) -> duo_seq_merge; a
        prefill-sized chunk: see ``_attend_shared_chunk``.  With ``P > 0`` there are only these launches:
        ``fused=False``, ``force_mma=True`` and qkv rows that are not 16-byte aligned (``qkv.stride(1) % 8``,
        ``qkv.data_ptr() % 16``) raise ``ValueError`` before any launch."""
        if self.prefix_len == 0:
            return self._attend(l, qkv, cos, sin, rope_mode, out, scale, force_mma, fused)
        if not fused or force_mma:
            raise ValueError(f"{type(self).__name__}: forks of a shared prompt decode through the one-launch step only "
                             "(fused=True, force_mma=False)")
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        if not call.aligned:
            raise ValueError(f"{type(self).__name__}: qkv rows must be 16-byte aligned (row stride a multiple of 8 "
                             "elements): forks have no unfused step")
        self._ensure_room(l, call.S)
        if call.S > 1:
            return self._attend_shared_chunk(l, call, rope_mode, out)
        po, pl = self.partials(1)
        self._launch(self.lib.duo_decode_fused_seq_shared, self.handles[l], self.donor.handles[l], self.prefix_len,
                     C.byref(self.state(l)), *call.qkv, *call.cos_sin, rope_mode & 0xFF, call.out, po.data_ptr(),
                     pl.data_ptr(), call.scale, *call.ws, call.stream, count=2 if self.num_full_kv_head_list[l] else 1,
                     timed=True)
        self._merge(l, out, 1, po, pl)
        self.advance(l, 1)
        return out

    def _attend_shared_chunk(self, l, call, rope_mode, out):
        """A prefill-sized chunk of S tokens on every row (P > 0): duo_rope_append at the own slices (state shifted to
        ``full_len - P``) -> duo_prefill_seq_shared over the donor's prefix rows and the own slices (logical state) ->
        the row-scattered merge -> duo_stream_commit (shifted state, which it reads for the ring only).  A prefill
        chunk is sized from the host state."""
        h, own = self.handles[l], self.state(l, host=True, prefix=self.prefix_len)
        self._rope_append(h, call, own, rope_mode)
        return self._attend_commit(l, call, own, out, self.lib.duo_prefill_seq_shared,
                                   (h, self.donor.handles[l], self.prefix_len), self.state(l, host=True),
                                   self.partials(call.S), scattered=True)

    def evict_last(self, num_tokens):
        left = min(self.kv_seq_len_list) - int(num_tokens)
        if left < self.prefix_len:
            raise ValueError(f"{type(self).__name__}: evict_last({num_tokens}) would evict into the shared prefix "
                             f"({self.prefix_len} positions; the forks hold {self.kv_seq_len})")
        DuoKVCache.evict_last(self, num_tokens)

    def clear(self):
        """Empty the forks and release the donor: the forks are then a plain sharded cache of their own capacity.
        Refused while a ``DuoDecodeGraph`` is attached: its captured launches read the donor's prefix at a fixed ``P``."""
        if self.graph_attached and self.prefix_len > 0:
            raise ValueError(f"{type(self).__name__}: cannot clear() forks captured in a DuoDecodeGraph: the graph reads "
                             f"the donor's first {self.prefix_len} positions; drop the graph and its forks instead")
        if self.donor is not None and self.donor._forks is not None:
            self.donor._forks.discard(self)
        self.donor, self.prefix_len = None, 0
        DuoKVCache.clear(self)


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
                     min_keys: int = 256, ctas_per_sm: int = 2, active: Optional[Sequence[bool]] = None) -> dict:
    """The retrieval-head key partition every CTA of a ragged decode launch derives from the row key counts
    ``lengths``: row ``b`` takes ``splits[b]`` consecutive slots of the ``slots`` grid slots per retrieval head, split
    ``i`` covering keys ``[i * keys_per_split, (i + 1) * keys_per_split)``.  ``slots`` depends on the geometry only.
    The defaults are duo_decode_ragged's policy; ``**INT4_RAGGED_POLICY`` gives duo_decode_ragged_int4's.

    ``active`` (default: every row) marks the rows that take part in the step; an idle row takes 0 splits and the
    active rows are partitioned as a compact batch of just those rows, with that batch's ``want``, unless its splits
    could exceed ``slots``: ``want`` is then clamped to ``slots // n_active - 1`` and ``clamped`` is True (the bits of
    the compact batch are then not promised).  With no active row ``keys_per_split`` is ``tile`` and no slot is used."""
    B = len(lengths)
    act = [True] * B if active is None else [bool(a) for a in active]
    if len(act) != B:
        raise ValueError(f"{len(act)} active flags for {B} rows")
    want = ragged_want(B, n_full, n_stream, sm_count, ctas_per_sm=ctas_per_sm)
    slots = B * (want + 1)
    lens = [int(n) for n, a in zip(lengths, act) if a]
    n_act, step_want, clamped = len(lens), want, False
    if 0 < n_act < B:
        step_want = ragged_want(n_act, n_full, n_stream, sm_count, ctas_per_sm=ctas_per_sm)
        clamped = step_want > slots // n_act - 1
        step_want = min(step_want, slots // n_act - 1)
    kps = ragged_keys_per_split(sum(lens), max(lens), n_act, step_want, tile=tile, min_keys=min_keys) if lens else tile
    splits = [max(1, -(-int(n) // kps)) if a else 0 for n, a in zip(lengths, act)]
    return {"want": want, "slots": slots, "keys_per_split": kps, "splits": splits, "step_want": step_want,
            "clamped": clamped}


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


def shared_prefix_len(length: int, align: int = POOL_ALIGN) -> int:
    """Keys a fork of a row of ``length`` tokens shares with it: the whole ``align``-key blocks, so that no 64-key tile
    straddles the end of the shared prefix."""
    return int(length) // align * align


def share_table(shares: Sequence[Optional[tuple]]) -> List[List[int]]:
    """The ``row_share`` array of duo_decode_ragged_shared from the rows' shares (``(donor, P)`` or None per row): a
    sharer gets ``[donor, P]``, a donor ``[donor, P]`` with the largest ``P`` of its sharers (it joins that group), every
    other row ``[-1, 0]``."""
    table = [[-1, 0] for _ in shares]
    for b, sh in enumerate(shares):
        if sh is not None:
            d, P = sh
            table[b] = [d, P]
            table[d] = [d, max(P, table[d][1])]
    return table


def share_fork_plan(length: int, share: Optional[tuple], src: int, capacity: int) -> dict:
    """What ``share_prefix`` does for a fork of row ``src`` (``length`` tokens, ``share`` its own ``(donor, P)`` or None)
    into a region of ``capacity`` tokens: the donor and shared keys ``P`` (a fork of a sharer shares the same donor
    prefix), the region row ``copy_from`` of src's first own key (a sharer's own keys start its region) and the
    ``n_copy`` tail rows copied into the new region.  ``ValueError`` if they do not fit ``capacity``."""
    donor, P = share if share is not None else (src, shared_prefix_len(length))
    n_copy = int(length) - P
    if n_copy > capacity:
        raise ValueError(f"row {src} holds {n_copy} tokens past its shared prefix of {P}: more than the capacity "
                         f"{capacity} of the new row's region")
    return {"donor": donor, "P": P, "copy_from": 0 if share is not None else P, "n_copy": n_copy}


# ---- batched ragged prefill (duo_prefill_ragged) -------------------------------------------------------------------
PREFILL_TILE = 128  # query rows of one CTA of the wgmma prefill kernel


def ragged_prefill_plan(lengths: Sequence[int], n_tokens: int, batch_size: int, tile: int = PREFILL_TILE) -> dict:
    """How ``duo_prefill_ragged`` lays out the chunks of one call: row ``b``'s ``lengths[b]`` tokens start at packed index
    ``offsets[b]`` (``offsets[batch_size] == n_tokens``), take ``tiles[b]`` query tiles per q-head, and the attention grid
    is ``n_q_heads * max_tiles`` by ``batch_size`` CTAs, the CTAs past a row's own tiles exiting at once.  ``rows`` are the
    rows with a chunk.  ``ValueError`` for a length count other than ``batch_size``, a negative length, or lengths that do
    not add up to ``n_tokens``."""
    lens = [int(n) for n in lengths]
    if len(lens) != int(batch_size):
        raise ValueError(f"chunk_lengths has {len(lens)} entries for a batch of {batch_size} rows")
    if any(n < 0 for n in lens):
        raise ValueError(f"chunk lengths must be >= 0 (got {lens})")
    if sum(lens) != int(n_tokens):
        raise ValueError(f"chunk lengths add up to {sum(lens)}, but {n_tokens} packed tokens were given")
    offsets = [sum(lens[:b]) for b in range(len(lens) + 1)]
    tiles = [-(-n // tile) for n in lens]
    return {"offsets": offsets, "tiles": tiles, "max_tiles": max(tiles, default=0),
            "rows": [b for b, n in enumerate(lens) if n > 0]}


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

    @property
    def pending_verify(self) -> Optional[int]:
        return self._parent.pending_verify  # a verify chunk is the parent's, over all rows

    def verify(self, l, qkv, cos, sin, rope_mode, out, scale=None):
        raise ValueError(f"row {self._row}: the rows of a ragged batch verify drafts together, through the parent cache")

    def accept(self, a):
        raise ValueError(f"row {self._row}: the rows of a ragged batch accept drafts together, through the parent cache")

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        _refuse_pending(self, f"row({self._row}).attend")
        sh = self._parent._share[self._row] if self._parent.pooled else None
        if sh is None:
            out = super().attend(l, qkv, cos, sin, rope_mode, out, scale=scale, force_mma=force_mma, fused=fused)
        else:
            out = self._attend_shared(l, sh, qkv, cos, sin, rope_mode, out, scale, force_mma)
        self._parent.rows_changed = True
        return out

    def _attend_shared(self, l, sh, qkv, cos, sin, rope_mode, out, scale, force_mma):
        """A prefill-sized chunk of a sharer: its keys ``[0, P)`` are the donor's region rows, the rest (and the chunk)
        its own region's rows ``j - P``; ``duo_attention_shared`` reads both with the tiles of a plain row, so the bits
        are those of a row that holds a copy of the prompt.  On INT4, chunks of >= 128 tokens attend the dequantised
        image of both regions instead, as a plain INT4 row's do.  Decode-sized chunks go through the batched step."""
        donor, P = sh
        S = qkv.shape[1]
        int4 = getattr(self, "kv_format", "same") == "int4"
        max_rows = _C.DECODE_MAX_Q_INT4 if int4 else _C.DECODE_MAX_Q
        if S * self.num_kv_groups <= max_rows:
            raise ValueError(f"row {self._row} shares the first {P} keys of row {donor}: decode-sized chunks (group x "
                             f"q_len <= {max_rows}) go through the batched step of the parent cache, not through "
                             "row(b)")
        if force_mma:
            raise ValueError(f"row {self._row} shares the first {P} keys of row {donor}: force_mma is not supported on "
                             "a sharer (its chunks take the kernel duo_attention would choose)")
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        if self._rows_needed(l, S) > self.full_cap_list[l]:  # before _ensure_room may grow the staging area
            raise self._room_error(l, S)
        self._ensure_room(l, S)
        h = self.handles[l]
        own = self.state(l, host=True, prefix=P)  # the own region's rows (the ring commit reads only total and lo)
        self._rope_append(h, call, own, rope_mode)
        dn = self._parent.rows[donor]
        if self._attends_image(S):
            # the dequantised image a copy row would attend (DuoKVCache.attend), built from both regions
            fn, head = self.lib.duo_attention, (self._dequant_scratch(l, S, prefix=(dn.tensors[l], P)),)
        else:
            fn, head = self.lib.duo_attention_shared, (h, dn.handles[l], P)
        return self._attend_commit(l, call, own, out, fn, head, self.state(l, host=True))

    def clear(self):
        P = self._parent
        _refuse_pending(self, f"row({self._row}).clear")
        if P.pooled:
            P._check_not_donor(self._row, "clear")
            P._end_share(self._row)
        super().clear()
        P.rows_changed = True
        P.sync_device_state()

    def evict_last(self, num_tokens):
        if self._parent.pooled:
            self._parent._check_evict(self._row, num_tokens)
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
    attached.  ``row_capacities`` gives the per-row capacities.

    ``share_prefix(src, dst, capacity)`` makes the empty row ``dst`` of a pooled cache a continuation of row ``src``
    (parallel sampling, best-of-n, beam search): ``dst`` reads src's first ``P`` retrieval keys (whole 128-key blocks) in
    place from src's region, and decode steps read that prefix once for all its sharers (``duo_decode_ragged_shared``).
    ``row_prefix`` gives each row's ``(donor, P)``.  While a row's prefix is shared it refuses ``clear``,
    ``resize_row`` and an ``evict_last`` below the prefix.  A sharer takes prefill-sized chunks (``group x q_len > 16``,
    e.g. its own question after the shared document) through ``row(b)`` (``duo_attention_shared``: the same bits as a
    row holding a copy of the prompt) and decodes through the batched step.

    ``set_active(b, False)`` lets row ``b`` sit out batched steps while it is prefilled, evicted, cleared or forked
    through ``row(b)`` (e.g. a long prompt admitted in chunks between decode steps of the other rows); ``row_active``
    gives the flags.

    ``attend_rows(l, qkv, cos, sin, rope_mode, out, lengths)`` prefills many rows in one pass: row ``b`` takes a chunk of
    its own length, the chunks packed back to back, in three launches per layer whatever the batch size
    (``duo_prefill_ragged``); ``model(input_ids=[1, T], past_key_values=cache, chunk_lengths=[...])`` drives it."""

    _KV = "same"                    # the one kv_format of the class
    _share_formats = ("same",)      # the kv_format(s) share_prefix serves on this class
    max_rows = _C.DECODE_MAX_Q      # packed rows (group x q_len) of one batched step
    graph_shared = False            # a DuoDecodeGraph captured the shared-prefix launch (set by DuoDecodeGraph)
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
            self._row_caps = caps                                   # logical capacities of the rows' own regions
            self._geom = [list(x) for x in zip(lay["first"], lay["cap"])]  # {first, cap} per row, 128-aligned tokens
            self.pool_tokens = lay["pool_tokens"]
            max_size = max(caps)
        elif pool_size is not None:
            raise ValueError(f"{type(self).__name__}: pool_size needs per-row capacities (a sequence as max_size)")
        self.rows = []  # the batch-1 views, made once the tensors exist
        self._share = [None] * int(batch_size)  # (donor, P) of a row that shares a donor's first P keys
        self._active = [True] * int(batch_size)  # False: the row sits out batched steps (set_active)
        super().__init__(num_layers, num_heads, num_kv_heads, head_dim, num_full_kv_head_list, batch_size, max_size,
                         sink_size, recent_size, dtype, device, stage_cap=stage_cap, kv_format=self._KV, growable=False)
        need = getattr(self.lib, self._ws_bytes)(self.batch_size, num_kv_heads)
        if need > self.workspace.numel():
            self.workspace = torch.zeros(need, dtype=torch.uint8, device=self.device)
        self.row_state = torch.zeros(self.batch_size, 4, dtype=torch.int64, device=self.device)  # {full_len, total, lo, flags}
        if self.pooled:  # read by the pooled kernels at launch: resize_row rewrites it without a re-capture
            self.row_geom = torch.tensor(self._geom, dtype=torch.int64, device=self.device)
            self.row_share = torch.tensor(share_table(self._share), dtype=torch.int64, device=self.device)
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
        """Token capacity of every row's retrieval cache (a sharer's: its shared prefix plus its own region)."""
        if not self.pooled:
            return [self.max_size] * self.batch_size
        return [c + (sh[1] if sh else 0) for c, sh in zip(self._row_caps, self._share)]

    @property
    def row_active(self) -> List[bool]:
        """Per row, whether it takes part in batched steps (see :meth:`set_active`)."""
        return list(self._active)

    def set_active(self, b: int, active: bool):
        """Let row ``b`` sit out batched steps (``active=False``) or rejoin them.  An idle row is skipped by every
        batched launch: none of its keys or ring slots is read, nothing of it is written (its rows of the attention
        output keep what they held, so the model's logits for it are meaningless), and ``advance``, ``evict_last`` and
        the capacity checks of the parent pass it by.  ``row(b)`` works on it as on any row: prefill it in chunks,
        evict, clear or fork it while the other rows keep decoding, then make it active again.  An idle donor's shared
        prefix is still read by its active sharers.  Rows start active; ``clear`` and ``share_prefix`` leave the flag
        alone.  Stream-ordered, and valid while a ``DuoDecodeGraph`` is attached (the kernels read the flag from
        ``row_state``)."""
        B = self.batch_size
        if isinstance(b, bool) or not isinstance(b, numbers.Integral) or not 0 <= int(b) < B:
            raise ValueError(f"{type(self).__name__}: set_active row {b!r} outside [0, {B})")
        if not isinstance(active, (bool, numbers.Integral)) or int(active) not in (0, 1):
            raise ValueError(f"{type(self).__name__}: set_active needs a bool (got {active!r})")
        _refuse_pending(self, "set_active")
        self._active[int(b)] = bool(active)
        self.rows_changed = True
        self.sync_device_state()

    def _active_rows(self) -> list:
        return [r for r, a in zip(self.rows, self._active) if a]

    @property
    def row_prefix(self) -> List[Optional[tuple]]:
        """Per row, ``(donor, shared tokens)`` of a row made by ``share_prefix``, else None."""
        return list(self._share) if self.pooled else [None] * self.batch_size

    @property
    def sharing(self) -> bool:
        """Whether any row shares a donor's prefix (decode steps then take duo_decode_ragged_shared)."""
        return self.pooled and any(sh is not None for sh in self._share)

    def _donor_floor(self, b: int) -> int:
        """The longest prefix of row ``b`` that other rows share (0 if none)."""
        return max([sh[1] for sh in self._share if sh is not None and sh[0] == b], default=0)

    def _check_not_donor(self, b: int, what: str):
        floor = self._donor_floor(b)
        if floor:
            sharers = [r for r, sh in enumerate(self._share) if sh is not None and sh[0] == b]
            raise ValueError(f"{type(self).__name__}: rows {sharers} share the first {floor} keys of row {b}: {what} "
                             f"of row {b} would change them; clear the sharers first")

    def _check_evict(self, b: int, n: int):
        """ValueError if ``evict_last(n)`` on row ``b`` would cut into keys that are shared: a donor's below the longest
        prefix it lends, a sharer's into its shared prefix."""
        r = self.rows[b]
        left = max(0, min(r.kv_seq_len_list) - int(n))
        floor = self._donor_floor(b)
        if left < floor:
            raise ValueError(f"{type(self).__name__}: evict_last({n}) would cut row {b} to {left} tokens, below the "
                             f"{floor} keys other rows share with it")
        sh = self._share[b]
        if sh is not None and left < sh[1]:
            raise ValueError(f"{type(self).__name__}: evict_last({n}) would cut row {b} to {left} tokens, into the "
                             f"{sh[1]} keys it shares with row {sh[0]}")

    def _sync_share(self):
        self.row_share.copy_(torch.tensor(share_table(self._share), dtype=torch.int64))  # stream-ordered

    def _end_share(self, b: int):
        """Row ``b`` stops sharing (it is being cleared): its capacity is its own region's again."""
        if self._share[b] is None:
            return
        self._share[b] = None
        self._sync_share()
        r = self.rows[b]
        r.max_size = self._row_caps[b]
        for l in range(self.num_layers):
            r._set_layer(l, self._row_caps[b], r.stage_cap_list[l])

    def share_prefix(self, src: int, dst: int, capacity: int):
        """Make the empty row ``dst`` a continuation of row ``src``'s current context, in every layer.  ``dst`` shares
        src's first ``P = floor(len / 128) * 128`` retrieval keys, read in place from src's region (a fork of a sharer
        shares the same donor prefix), and gets a region of ``capacity`` tokens (first fit in the pool) for its own
        keys: src's remaining tail, copied now, and everything it appends later.  Its sink and ring slots and its
        occupancy are copies of src's; ``row_capacities[dst]`` is ``P + capacity``.  ``dst`` takes prefill-sized chunks
        through ``row(dst)`` and decode-sized ones through the batched step, with the rows together.  Both KV formats
        share (an INT4 row's tail copy includes its scale / zero rows).  ``ValueError``, with the cache unchanged, for a
        uniform-capacity cache, a cache class that does not declare its format in ``_share_formats``, a non-empty
        ``dst``, an empty ``src``, a tail longer than ``capacity``, no free range, or an attached ``DuoDecodeGraph``
        captured without the shared launch."""
        name = type(self).__name__
        _refuse_pending(self, "share_prefix")
        if not self.pooled or self.kv_format not in getattr(self, "_share_formats", ("same",)):
            raise ValueError(f"{name}: share_prefix needs a 16-bit cache with per-row capacities (DuoRaggedKVCache "
                             "with a sequence as max_size) or a DuoRaggedINT4KVCache with per-row capacities")
        B = self.batch_size
        src, dst, capacity = int(src), int(dst), int(capacity)
        if not (0 <= src < B and 0 <= dst < B) or src == dst:
            raise ValueError(f"{name}: share_prefix({src}, {dst}) needs two different rows of the {B}")
        s, d = self.rows[src], self.rows[dst]
        if any(d.kv_seq_len_list) or any(d.total_list):
            raise ValueError(f"{name}: row {dst} is not empty (length {d.kv_seq_len}): clear it before share_prefix")
        if not any(s.kv_seq_len_list):
            raise ValueError(f"{name}: row {src} is empty: there is no prefix to share")
        if len(set(s.kv_seq_len_list)) != 1 or len(set(s.total_list)) != 1:
            raise ValueError(f"{name}: row {src}'s layers hold different lengths (mid-step): fork between steps")
        if capacity < 1:
            raise ValueError(f"{name}: capacity {capacity} < 1")
        if self.graph_attached and not self.graph_shared:
            raise ValueError(f"{name}: the attached DuoDecodeGraph was captured without the shared-prefix launch and "
                             "would read the wrong keys: build a new DuoDecodeGraph after share_prefix")
        plan = share_fork_plan(s.kv_seq_len, self._share[src], src, capacity)
        first = pool_first_fit([g[0] for g in self._geom], [g[1] for g in self._geom], dst, capacity, self.pool_tokens)
        need = self.lib.duo_ragged_shared_workspace_bytes(B, self.num_kv_heads)
        if need == 0:
            raise ValueError(f"{name}: no shared-prefix workspace for batch {B} x {self.num_kv_heads} kv heads")
        if need > self.workspace.numel():  # (a graph captured with the shared launch already holds a large one)
            self.workspace = torch.zeros(need, dtype=torch.uint8, device=self.device)
        # ---- checks done: the fork
        P, n = plan["P"], plan["n_copy"]
        self._geom[dst] = [first, _round_up(capacity, POOL_ALIGN)]
        self._row_caps[dst] = capacity
        self.row_geom[dst].copy_(torch.tensor(self._geom[dst], dtype=torch.int64))
        d.max_size = P + capacity
        W, c0 = self.W, plan["copy_from"]
        for l in range(self.num_layers):
            d._set_layer(l, P + capacity, d.stage_cap_list[l])
            for key, t in d.tensors[l].items():
                if key.startswith("full"):
                    t[0, :, :n].copy_(s.tensors[l][key][0, :, c0 : c0 + n])
                else:
                    t[0, :, :W].copy_(s.tensors[l][key][0, :, :W])
        d.restore_state(s.snapshot_state())
        if P > 0:
            self._share[dst] = (plan["donor"], P)
            self._sync_share()
        self.rows_changed = True
        self.sync_device_state()

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
        if self.pooled:  # every share ends
            for b in range(self.batch_size):
                self._end_share(b)
        for r in self.rows:
            DuoKVCache.clear(r)
        self._verify_len = [0] * self.num_layers  # a pending verify chunk is discarded
        self.rows_changed = True
        self.sync_device_state()

    def evict_last(self, num_tokens):
        """``evict_last`` on every active row (idle rows keep their tokens)."""
        _refuse_pending(self, "evict_last")
        if self.pooled:  # refused as a whole, before any row changes
            for b in range(self.batch_size):
                if self._active[b]:
                    self._check_evict(b, num_tokens)
        for r in self._active_rows():
            DuoKVCache.evict_last(r, num_tokens)
        self.rows_changed = True
        self.sync_device_state()

    def advance(self, l, q_len):
        for r in self._active_rows():
            r.advance(l, q_len)

    def state(self, l):
        raise TypeError("DuoRaggedKVCache has one occupancy per row: use row(b).state(l) or row_state")

    def snapshot_state(self):
        return [r.snapshot_state() for r in self.rows]

    def restore_state(self, snap):
        for r, s in zip(self.rows, snap):
            r.restore_state(s)

    def check_room(self, q_len, layers=None):
        for r in self._active_rows():  # every active row against its own capacity
            r.check_room(q_len, layers)

    # ---- device-resident occupancy ----------------------------------------------------------------------------------
    def enable_device_state(self):
        self.sync_device_state()
        return self

    def sync_device_state(self, l: Optional[int] = None):
        """row_state := the rows' host occupancy of layer ``l`` (default: the last layer), stream-ordered."""
        l = self.num_layers - 1 if l is None else l
        host = torch.tensor([[r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l], 0 if a else _C.ROW_IDLE]
                             for r, a in zip(self.rows, self._active)], dtype=torch.int64)
        self.row_state.copy_(host)

    def advance_device(self, n):
        self._launch(self.lib.duo_ragged_state_advance, self.row_state.data_ptr(), self.batch_size, int(n),
                     self.sink_size, self.recent_size, torch.cuda.current_stream(self.device).cuda_stream)

    # ---- batched decode step -----------------------------------------------------------------------------------------
    def check_rows(self, layers: Sequence[int]):
        """Raise ValueError if an active row cannot join a batched step of these layers (16-bit caches: every row
        can)."""

    def _check_chunk(self, l, q_len):
        if q_len * self.num_kv_groups > self.max_rows:
            raise ValueError(f"{type(self).__name__} decodes chunks of group x q_len <= {self.max_rows} rows (got "
                             f"{q_len} tokens): prefill each row through cache.row(b)")
        self.check_rows([l])

    def attend_rows(self, l, qkv, cos, sin, rope_mode, out, lengths, scale=None):
        """A batched prefill of layer ``l``: row ``b`` takes the next ``lengths[b] >= 0`` tokens, packed back to back in
        ``qkv`` ``[1, T, (Hq + 2 Hkv) * D]`` (T = the sum; rows 16-byte aligned, q rotated in place), with per-token RoPE
        tables ``cos`` / ``sin`` ``[T, D]`` (or None with ROPE_NONE); ``out`` ``[1, T, Hq, D]`` contiguous.  Three
        launches whatever the batch size (``duo_prefill_ragged``): RoPE + append, one wgmma attention launch over every
        row's chunk, ring commit.  A row with a chunk of >= 128 tokens gets the bits ``row(b).attend`` gives it (outputs
        and every cache byte; a sharer's as ``duo_attention_shared`` gives them); a shorter chunk, which ``row(b)`` hands
        to the mma.sync kernel, agrees to rounding.  Rows of length 0 are not touched; idle rows (``set_active``) with a
        chunk are prefilled, which is how a row is admitted.  A chunk of a token or two over a long context occupies a
        128-row tile: decode steps belong to ``attend``.  Each row's capacity is checked as ``row(b)`` checks it, before
        anything runs, and the staging area grows as there (refused while a ``DuoDecodeGraph`` is attached).  Then every
        participating row advances by its length and ``row_state`` follows.  16-bit caches with sink + recent <= 2048
        only; all lengths 0 is a no-op."""
        name = type(self).__name__
        _refuse_pending(self, "attend_rows")
        if self.W > PREFILL_MAX_WINDOW:
            raise ValueError(f"{name}: attend_rows needs sink + recent <= {PREFILL_MAX_WINDOW} (got {self.W}): prefill "
                             "each row through cache.row(b)")
        if not qkv.is_cuda or not out.is_cuda:
            raise RuntimeError("duo_attention_b200 kernels need CUDA tensors (no CPU fallback)")
        B, D, Hq = self.batch_size, self.head_dim, self.num_heads
        assert qkv.dim() == 3 and qkv.shape[0] == 1 and qkv.shape[2] == (Hq + 2 * self.num_kv_heads) * D
        T = qkv.shape[1]
        plan = ragged_prefill_plan(lengths, T, B)
        lens = [int(n) for n in lengths]
        for b in plan["rows"]:  # every row's room first: a refusal changes nothing
            self.rows[b].check_room(lens[b], [l])
        if not plan["rows"]:
            return out
        assert qkv.stride(2) == 1 and qkv.dtype == self.dtype and out.dtype == self.dtype
        assert out.shape == (1, T, Hq, D) and out.is_contiguous()
        if cos is not None:
            assert cos.shape == (T, D) and cos.is_contiguous() and sin.is_contiguous()
        if max(lens) > self.stage_cap_list[l]:  # as row(b) grows it (for every row)
            self._grow_layer(l, max(lens))
        self.sync_device_state(l)  # row_state := layer l's host occupancy, which the kernels read
        room = [c - r.kv_seq_len_list[l] for c, r in zip(self.row_capacities, self.rows)]
        stream = torch.cuda.current_stream(self.device).cuda_stream
        self._launch(self.lib.duo_prefill_ragged, self.handles[l], self.row_state.data_ptr(),
                     self.row_geom.data_ptr() if self.pooled else None,
                     self.row_share.data_ptr() if self.pooled else None, (C.c_int32 * B)(*lens),
                     (C.c_int64 * B)(*room), qkv.data_ptr(), qkv.stride(1),
                     cos.data_ptr() if cos is not None else None, sin.data_ptr() if sin is not None else None,
                     rope_mode & 0xFF, out.data_ptr(), float(D ** -0.5 if scale is None else scale),
                     self.workspace.data_ptr(), self.workspace.numel(), stream, timed=True,
                     count=2 + (self.num_streaming_kv_head_list[l] > 0))
        for b in plan["rows"]:
            self.rows[b].advance(l, lens[b])
        self.rows_changed = True
        self.sync_device_state()
        return out

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        """One decode-sized chunk for every row, one ``duo_decode_ragged`` launch.  ``qkv`` ``[B, S, (Hq + 2 Hkv) * D]``
        (rows 16-byte aligned), ``cos`` / ``sin`` ``[B, S, D]`` per-row tables (or None with ROPE_NONE), ``out``
        ``[B, S, Hq, D]`` contiguous.  Idle rows (``set_active``) are skipped: their rows of ``out`` are not written."""
        _refuse_pending(self, "attend")
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        S = call.S
        if cos is not None:
            assert cos.shape == (self.batch_size, S, self.head_dim) and cos.is_contiguous() and sin.is_contiguous()
        self.check_room(S, [l])
        if not self.graph_attached:  # eager: the rows' host occupancy is authoritative
            self.sync_device_state(l)
        h, rs = self.handles[l], self.row_state.data_ptr()
        tail = (*call.qkv, *call.cos_sin, rope_mode & 0xFF, call.out, S, call.scale, *call.ws, call.stream)
        if self.sharing:  # the cascade: each shared prefix once for its rows, then every row's own keys
            self._launch(self.lib.duo_decode_ragged_shared, h, rs, self.row_geom.data_ptr(), self.row_share.data_ptr(),
                         self._min_room(l, S), *tail, timed=True, count=2 if self.num_full_kv_head_list[l] else 1)
        elif self.pooled:
            self._launch(self.lib.duo_decode_ragged_pooled, h, rs, self.row_geom.data_ptr(), self._min_room(l, S),
                         *tail, timed=True)
        else:
            max_len = max((r.kv_seq_len_list[l] for r in self._active_rows()), default=0)
            self._launch(getattr(self.lib, self._decode), h, rs, max_len, *tail, timed=True)
        self.advance(l, S)
        return out

    def _min_room(self, l, S) -> int:
        """The least retrieval room of layer ``l`` over the active rows (``S`` when none is active), which the pooled
        and verify launches check their chunk against."""
        return min((c - r.kv_seq_len_list[l] for c, r, a in zip(self.row_capacities, self.rows, self._active) if a),
                   default=S)

    def verify(self, l, qkv, cos, sin, rope_mode, out, scale=None):
        """A verify chunk (see :meth:`DuoKVCache.verify`) of one length S for every active row, each at its own
        position, in one ``duo_decode_ragged_verify`` launch; arguments as for ``attend``.  Idle rows are skipped.
        Refused with ``ValueError`` before anything changes as there, and for rows that share a prefix and
        group x S > 16."""
        S = qkv.shape[1]
        self._check_verify(l, S, self.max_rows)
        if self.sharing:
            raise ValueError(f"{type(self).__name__}: rows that share a prefix cannot verify drafts")
        call = self._attend_call(l, qkv, out, cos, sin, scale)
        if cos is not None:
            assert cos.shape == (self.batch_size, S, self.head_dim) and cos.is_contiguous() and sin.is_contiguous()
        self.check_room(S, [l])
        if S > self.stage_cap_list[l]:
            self._grow_layer(l, S)
        self.sync_device_state(l)
        self._launch(self.lib.duo_decode_ragged_verify, self.handles[l], self.row_state.data_ptr(),
                     self.row_geom.data_ptr() if self.pooled else None, self._min_room(l, S), *call.qkv,
                     *call.cos_sin, rope_mode & 0xFF, call.out, S, call.scale, *call.ws, call.stream, timed=True)
        self._verify_len[l] = S
        return out

    def accept(self, counts):
        """Keep the first ``counts[b]`` tokens (0 <= counts[b] <= S; 0 for an idle row) of row ``b``'s verify chunk:
        one ``duo_stream_commit_rows`` launch per layer commits the staged streaming rows against each row's own total,
        then every row advances by its count on the host and in ``row_state``."""
        S = self._accept_len()
        name, B = type(self).__name__, self.batch_size
        try:
            ok = len(counts) == B and all(not isinstance(c, bool) and isinstance(c, numbers.Integral) for c in counts)
        except TypeError:
            ok = False
        if not ok:
            raise ValueError(f"{name}: accept() takes one integer count per row ({B}), got {counts!r}")
        counts = [int(c) for c in counts]
        for b, (c, a) in enumerate(zip(counts, self._active)):
            if not 0 <= c <= (S if a else 0):
                raise ValueError(f"{name}: row {b}'s count {c} outside [0, {S if a else 0}]"
                                 + ("" if a else " (an idle row keeps nothing)"))
        arr = (C.c_int32 * B)(*counts)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for l in range(self.num_layers):
            self.sync_device_state(l)  # row_state := the rows' totals the chunk was staged against
            self._launch(self.lib.duo_stream_commit_rows, self.handles[l], self.row_state.data_ptr(), arr, stream,
                         count=1 if any(counts) and self.num_streaming_kv_head_list[l] > 0 else 0)
            for r, c in zip(self.rows, counts):
                r.advance(l, c)
        self._verify_len = [0] * self.num_layers
        self.rows_changed = True
        self.sync_device_state()


class DuoRaggedINT4KVCache(DuoRaggedKVCache):
    """:class:`DuoRaggedKVCache` over the INT4 KV format of :class:`DuoAttentionStaticINT4KVCache` (136 B per retrieval
    head and key instead of 512 B at 16 bits): one ``duo_decode_ragged_int4`` launch per layer and step.  Same
    constructor arguments as :class:`DuoAttentionStaticINT4KVCache` (plus ``from_geometry``); fp16 or bf16 models.

    ``row(b)`` is a full batch-1 INT4 cache: a row's first chunk attends the raw 16-bit K/V (as the reference's first
    call does), later chunks of >= 128 tokens attend a dequantised image, small chunks and decode steps the INT4
    kernels.  The rows share one such image and one first-chunk scratch.  Batched steps take ``group x q_len <= 8``
    rows, and every row must have been prefilled through ``row(b)`` first: an empty row's first call must attend its
    raw K/V, which the batched kernel never sees.

    With per-row capacities, ``share_prefix`` works as on :class:`DuoRaggedKVCache`: forks read the donor's INT4 codes,
    scales and zeros in place, decode steps take ``duo_decode_ragged_shared`` (the prefix streamed once per 64 packed
    rows), and a sharer's chunks through ``row(b)`` give the bits of a row holding a copy: ``group x q_len > 8`` rows
    on the INT4 kernels (``duo_attention_shared``), chunks of >= 128 tokens on the dequantised image of both regions.
    On INT4, sharing trades speed for memory: the prefix pass streams the shared keys far below HBM rate, so below
    about ten forks a step of the sharing rows is slower than the same rows holding copies (DESIGN §5); it is what lets
    several continuations of a prompt fit that copies would not."""

    _KV = "int4"
    _share_formats = ("int4",)
    max_rows = _C.DECODE_MAX_Q_INT4
    _decode = "duo_decode_ragged_int4"
    _ws_bytes = "duo_ragged_int4_workspace_bytes"

    def __init__(self, model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                 prefilling_chunk_size: int = 64, pool_size: Optional[int] = None):
        super().__init__(model, full_attention_heads, batch_size, max_size, sink_size, recent_size,
                         prefilling_chunk_size=prefilling_chunk_size, kv_format="int4", pool_size=pool_size)

    def attend_rows(self, l, qkv, cos, sin, rope_mode, out, lengths, scale=None):
        """Not on INT4 caches: a chunk of >= 128 tokens of an INT4 row attends a dequantised image of that row."""
        raise ValueError(f"{type(self).__name__}: the batched ragged prefill (attend_rows, chunk_lengths=) takes 16-bit "
                         "caches only: prefill each row of an INT4 cache through cache.row(b)")

    def check_rows(self, layers: Sequence[int]):
        for b, r in enumerate(self.rows):
            if not self._active[b]:  # an emptied row may sit idle until it is refilled through row(b)
                continue
            for l in layers:
                if r.kv_seq_len_list[l] == 0 and r.total_list[l] == 0:
                    raise ValueError(f"{type(self).__name__}: row {b} is empty; its first chunk attends the raw K/V: "
                                     "prefill it through cache.row(b)")
