"""CUDA-graph replay of the decode step (scope-table row f3).

A decode step of the patched model is ~32 x (3 GEMMs + 6 of our kernels [+ 2 all-reduces]): at short context and
under tensor parallelism it is bound by launch latency and by the Python driver, not by the GPU.  The kernels
read the cache occupancy from device memory (``duo_cache_state.device_state``) and RoPE positions come from a
device tensor, so ONE captured step can be replayed for every generated token:

    g = DuoDecodeGraph(model, cache)          # cache: DuoKVCache / DuoAttentionStaticKVCache after prefill
    logits = g.step(next_token_tensor)        # [B, 1] int64 on the GPU; returns [B, 1, vocab]

``cache.evict_last`` / ``clear`` keep working between steps (they refresh the device copy).

A ``DuoRaggedKVCache`` is captured the same way: positions are ``[B, 1]`` and advance on the device with the rows.
After a row is evicted, cleared or refilled through ``cache.row(b)``, ``step()`` reloads the positions from the row
lengths (``resync()`` does it explicitly).  A graph captured while rows share a prefix (``share_prefix``) holds the
shared-prefix launch and keeps working across later forks, clears and refills; ``share_prefix`` refuses to fork while
a graph captured without it is attached.  ``cache.set_active(b, ...)`` may be toggled between any two steps: the
kernels read the idle flags from ``row_state``, and an idle row's positions are reloaded when it rejoins.
"""
from __future__ import annotations

import torch

from .kv_cache import DuoRaggedKVCache


class DuoDecodeGraph:
    def __init__(self, model, cache, warmup: int = 2):
        if cache.growable:
            raise ValueError("DuoDecodeGraph needs a pre-allocated cache (DuoAttentionStaticKVCache): a growable "
                             "cache may be re-allocated, which would leave stale pointers in the captured graph")
        self.model, self.cache = model, cache
        self.ragged = isinstance(cache, DuoRaggedKVCache)
        cache.graph_attached = True  # the captured launches hold raw buffer addresses: no re-allocation from now on
        dev = cache.device
        B = cache.batch_size
        cache.enable_device_state()
        self.ids = torch.zeros(B, 1, dtype=torch.long, device=dev)
        self.pos = torch.zeros(B if self.ragged else 1, 1, dtype=torch.long, device=dev)
        self.graph = torch.cuda.CUDAGraph()
        snap = cache.snapshot_state()
        ring = cache.snapshot_ring()  # warm-up steps commit a throw-away token into the ring: undone below

        def restore():
            cache.restore_state(snap)
            cache.sync_device_state()
            self._reload_positions()

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):  # lazy weight fusion, cuBLAS workspaces, cudaFuncSetAttribute ...
                restore()
                self._forward()
            restore()
            torch.cuda.synchronize(dev)
            with torch.cuda.graph(self.graph, stream=side):
                self.logits = self._forward()
            if self.ragged:  # which launch the graph holds: a shared-prefix one serves any later sharing pattern
                cache.graph_shared = cache.sharing
            cache.restore_ring(ring)
        torch.cuda.current_stream(dev).wait_stream(side)
        restore()  # capture itself did not execute anything

    def _forward(self):
        out = self.model(input_ids=self.ids, position_ids=self.pos, past_key_values=self.cache, use_cache=True)
        self.pos.add_(1)
        return out.logits

    def step(self, token: torch.Tensor) -> torch.Tensor:
        """Run one decode step for ``token`` ([B,1] int64, device or pinned host)."""
        c = self.cache
        if c.rows_changed:
            self.resync()
        if self.ragged:  # INT4: an emptied row must be refilled through row(b) first, as in eager decode
            c.check_rows(range(c.num_layers))
        c.check_room(1)  # the capture-time overflow check does not re-run on replay: same error as eager
        self.ids.copy_(token, non_blocking=True)
        self.graph.replay()
        self.cache.advance_host(1)
        return self.logits

    def _reload_positions(self):
        if self.ragged:
            self.pos.copy_(self.cache.row_state[:, :1])
            self.cache.rows_changed = False
        else:
            self.pos.fill_(self.cache.kv_seq_len)

    def resync(self):
        """Call after evict_last()/clear() (or, for a ragged cache, a row refilled through row(b)): positions restart
        from the cache length, per row for a ragged cache."""
        if self.ragged:
            self.cache.sync_device_state()
        self._reload_positions()
