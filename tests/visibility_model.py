"""Which cached positions every query row of a chunk may see: the reference's tuple-cache semantics as pure integers.
TEST INFRASTRUCTURE ONLY (the GPU visibility census, tests/test_gpu_visibility_census.py).

The tuple cache (duo_attn/patch/llama.py:168-301, ``oracle.duo_oracle.tuple_attention_core``) concatenates every chunk
to both caches, attends bottom-right causally, then keeps the sinks plus the last ``recent`` entries of the streaming
cache; ``evict_last(n)`` slices the newest ``n`` entries off both.  A token is named by its absolute position: after
an eviction the next token takes the evicted position again.  The caches are kept as sorted lists of half-open
position intervals, so a million-token context costs a few integers.

``tests/test_visibility_model_host.py`` pins this model to ``tuple_attention_core`` run in fp64 and to
``streaming_visible``.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

Intervals = List[Tuple[int, int]]


def _count(iv: Sequence[Tuple[int, int]]) -> int:
    return sum(b - a for a, b in iv)


def _append(iv: Intervals, a: int, b: int) -> Intervals:
    """``iv`` followed by the positions ``[a, b)``."""
    if a >= b:
        return list(iv)
    if iv and iv[-1][1] == a:
        return iv[:-1] + [(iv[-1][0], b)]
    return iv + [(a, b)]


def _slice(iv: Sequence[Tuple[int, int]], start: int, stop: int) -> Intervals:
    """The entries ``start .. stop - 1`` (by index, not by position) of the interval list ``iv``."""
    out: Intervals = []
    idx = 0
    for a, b in iv:
        n = b - a
        lo, hi = max(start, idx), min(stop, idx + n)
        if lo < hi:
            out = _append(out, a + lo - idx, a + hi - idx)
        idx += n
    return out


def positions(iv: Sequence[Tuple[int, int]]) -> List[int]:
    return [p for a, b in iv for p in range(a, b)]


class Chunk:
    """Visibility of the ``S`` query rows of one chunk whose first token sits at position ``start``: row ``i`` sees the
    retrieval cache before the chunk (``full``) or the streaming cache before the chunk (``stream``), plus the chunk's
    positions ``[start, start + i]``."""

    def __init__(self, start: int, S: int, full: Intervals, stream: Intervals):
        self.start, self.S, self.full, self.stream = start, S, full, stream

    def intervals(self, i: int, retrieval: bool) -> Intervals:
        return _append(self.full if retrieval else self.stream, self.start, self.start + i + 1)

    def visible(self, i: int, retrieval: bool) -> List[int]:
        """Sorted absolute positions query row ``i`` may see."""
        return positions(self.intervals(i, retrieval))


class TupleVisibility:
    """The positions held by the retrieval and the streaming tuple caches of one layer, moved by ``chunk`` and
    ``evict``."""

    def __init__(self, sink: int, recent: int):
        self.sink, self.recent = int(sink), int(recent)
        self.full: Intervals = []
        self.stream: Intervals = []

    @property
    def total(self) -> int:
        """Position of the next token (= the retrieval cache length)."""
        return _count(self.full)

    def chunk(self, S: int) -> Chunk:
        """Attend a chunk of ``S`` tokens: returns what its rows see, then appends it (and compacts the streaming
        cache)."""
        start = self.total
        c = Chunk(start, S, list(self.full), list(self.stream))
        self.full = _append(self.full, start, start + S)
        st = _append(self.stream, start, start + S)
        n = _count(st)
        if n > self.sink + self.recent:
            kept: Intervals = []
            for a, b in _slice(st, 0, self.sink) + _slice(st, n - self.recent, n):
                kept = _append(kept, a, b)
            st = kept
        self.stream = st
        return c

    def evict(self, n: int):
        """``evict_last(n)``: the newest ``n`` entries of both caches go."""
        self.full = _slice(self.full, 0, max(0, _count(self.full) - n))
        self.stream = _slice(self.stream, 0, max(0, _count(self.stream) - n))

    def stream_live(self) -> List[int]:
        """Positions the streaming cache holds now (each in slot ``kv_cache.ring_slot(p)``)."""
        return positions(self.stream)
