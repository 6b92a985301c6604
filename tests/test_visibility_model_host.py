"""The visibility model of the GPU census (tests/visibility_model.py) against the oracle, on the CPU.

``tuple_attention_core`` runs in fp64 with q = k = 0 (uniform attention) and V = one-hot position labels, so the output
row of a query is 1/|visible| on exactly the dimensions of the positions it sees.  Over seeded random schedules of
chunks and ``evict_last`` calls the model must name the same positions for both head classes; before the first
eviction it must also agree with the closed form ``streaming_visible``; and the ring state the product keeps
(``ring_advance`` / ``ring_evict``) must hold the model's streaming positions in distinct slots.
"""
import random

import pytest
import torch

from duo_attention_b200.kv_cache import ring_advance, ring_evict, ring_live_positions, ring_slot
from oracle import duo_oracle as O
from visibility_model import TupleVisibility

SINK_RECENT = [(0, 5), (1, 2), (4, 12), (16, 48), (64, 256), (3, 700)]


def _schedule(rng, sink, recent, max_total):
    """[("chunk", S) | ("evict", n)]: chunks of 1-700 tokens (mostly short), evictions of at most the live ring
    entries (the modelled contract, DESIGN §2)."""
    ops, total, live_ring = [], 0, 0
    while True:
        S = rng.choice([1, 1, 2, 3, rng.randint(1, 40), rng.randint(1, 700)])
        if total + S > max_total:
            return ops
        ops.append(("chunk", S))
        total += S
        live_ring = min(recent, live_ring + S) if total > sink else 0
        live_ring = min(live_ring, total - min(total, sink))
        if live_ring and rng.random() < 0.3:
            n = rng.randint(1, min(live_ring, 5))
            ops.append(("evict", n))
            total -= n
            live_ring -= n


def _oracle_visible(out_row):
    nz = torch.nonzero(out_row).flatten().tolist()
    return nz, out_row[nz]


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("sink,recent", SINK_RECENT)
def test_visibility_model_matches_tuple_oracle(sink, recent, seed):
    rng = random.Random(1000 * seed + 7 * sink + recent)
    max_total = 1800
    P = max_total + 8  # one label dimension per position
    model = TupleVisibility(sink, recent)
    total, lo = 0, sink  # the product's ring state
    past = None
    evicted = False
    for op, n in _schedule(rng, sink, recent, max_total):
        if op == "evict":
            model.evict(n)
            total, lo = ring_evict(total, lo, n, sink)
            fk, sk = past
            past = (fk[:, :, : fk.shape[2] - n].contiguous(), sk[:, :, : sk.shape[2] - n].contiguous())
            evicted = True
        else:
            S = n
            start = model.total
            assert start == total
            q = torch.zeros(1, S, 2, P, dtype=torch.float64)
            k = torch.zeros(1, S, 2, P, dtype=torch.float64)
            v = torch.zeros(1, S, 2, P, dtype=torch.float64)
            for i in range(S):
                v[0, i, :, start + i] = 1.0
            out, past = O.tuple_attention_core(q, k, v, past, 1, 1, sink, recent)
            ch = model.chunk(S)
            for i in range(S):
                for head, retrieval in ((0, True), (1, False)):
                    want = ch.visible(i, retrieval)
                    got, vals = _oracle_visible(out[0, i, head])
                    assert got == want, (op, S, i, retrieval)
                    torch.testing.assert_close(vals, torch.full_like(vals, 1.0 / len(want)), rtol=1e-6, atol=0)
                    if not evicted:
                        closed = [j for j in range(start + i + 1)
                                  if retrieval or O.streaming_visible(start + i, j, start, sink, recent)]
                        assert want == closed, (S, i, retrieval)
            total, lo = ring_advance(total, lo, S, sink, recent)
        assert model.total == total == past[0].shape[2]
        live = model.stream_live()
        assert live == ring_live_positions(total, lo, sink) and len(live) == past[1].shape[2]
        assert len({ring_slot(p, sink, recent) for p in live}) == len(live)
        assert all(ring_slot(p, sink, recent) < sink + recent for p in live)


def test_visibility_model_by_hand():
    m = TupleVisibility(2, 3)
    c = m.chunk(4)  # first call: plain causal
    assert c.visible(3, False) == [0, 1, 2, 3] and c.visible(0, True) == [0]
    c = m.chunk(2)  # 6 positions: sinks 0, 1 + ring 2, 3 before compaction
    assert c.visible(0, False) == [0, 1, 2, 3, 4] and c.visible(1, False) == [0, 1, 2, 3, 4, 5]
    assert m.stream_live() == [0, 1, 3, 4, 5]
    m.evict(2)
    assert m.total == 4 and m.stream_live() == [0, 1, 3]
    c = m.chunk(1)
    assert c.visible(0, True) == [0, 1, 2, 3, 4] and c.visible(0, False) == [0, 1, 3, 4]
    assert ring_slot(4, 2, 3) == 4 and ring_slot(5, 2, 3) == 2
