"""Verify chunks on ragged batches (DuoRaggedKVCache.verify / accept, duo_decode_ragged_verify, duo_stream_commit_rows):
uniform and pooled layouts, rows at different lengths (an unwrapped and a wrapped ring) and an idle row.  Every active
row is checked against a batch-1 twin that takes the row's tokens one per step: parity of its output rows against
fp64 attention over the keys of the twin's steps, and after accept(counts), with its own count per row, its retrieval
rows, sink / ring slots, occupancy and row_state equal the twin's after that many steps.  The idle row's bytes and its
rows of the output are untouched."""
import math

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache, DuoRaggedKVCache
from parity import assert_parity
from verify_ref import D, SequentialTwin, reference, rope_tables, rotate

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
SINK, RECENT, HKV = 8, 24, 2
LENGTHS = [12, 70, 30]  # unwrapped, wrapped, and the idle row
IDLE = 2


def new_ragged(pooled, Hq, n_full, dtype):
    caps = [256, 384, 128] if pooled else 256
    return DuoRaggedKVCache.from_geometry(1, Hq, HKV, D, [n_full], 3, caps, SINK, RECENT, dtype, DEV)


def new_single(Hq, n_full, dtype):
    return DuoKVCache(1, Hq, HKV, D, [n_full], 1, 256, SINK, RECENT, dtype, DEV, stage_cap=64)


@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
@pytest.mark.parametrize("dtype,G,S,rope", [(torch.bfloat16, 4, 4, _C.ROPE_HF), (torch.float16, 1, 7, _C.ROPE_FP32),
                                            (torch.bfloat16, 1, 16, _C.ROPE_NONE), (torch.float16, 4, 2, _C.ROPE_HF)])
def test_ragged_verify_rows_against_batch1_twins(pooled, dtype, G, S, rope):
    Hq, n_full = HKV * G, 1
    width = (Hq + 2 * HKV) * D
    gen = torch.Generator().manual_seed(S * 10 + G)
    count_sets = [[S, 1, 0], [0, math.ceil(S / 2), 0]]
    caches = [new_ragged(pooled, Hq, n_full, dtype) for _ in count_sets]
    prompts = [(torch.randn(1, n, width, generator=gen) * 0.5).to(dtype).to(DEV) for n in LENGTHS]
    need = {(b, cs[b]) for cs in count_sets for b in range(2)} | {(b, S) for b in range(2)}
    twins = {k: new_single(Hq, n_full, dtype) for k in need}
    for b, pq in enumerate(prompts):
        n = pq.shape[1]
        cos, sin = rope_tables(list(range(n)), rope, dtype, DEV)
        targets = [c.row(b) for c in caches] + [t for (bb, _), t in twins.items() if bb == b]
        for c in targets:
            c.attend(0, pq.clone(), cos, sin, rope, torch.empty(1, n, Hq, D, dtype=dtype, device=DEV))
    for c in caches:
        c.set_active(IDLE, False)
    idle_before = {k: v[0].clone() for k, v in caches[0].row(IDLE).tensors[0].items()}

    qkv = (torch.randn(3, S, width, generator=gen) * 0.5).to(dtype).to(DEV)
    pos = [[LENGTHS[b] + t for t in range(S)] for b in range(3)]
    cos, sin = rope_tables(pos, rope, dtype, DEV)
    outs = []
    for c in caches:
        o = torch.full((3, S, Hq, D), 7.0, dtype=dtype, device=DEV)
        c.verify(0, qkv.clone(), cos, sin, rope, o)
        assert c.pending_verify == S and c.row_lengths == LENGTHS
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    out = outs[0]
    assert (out[IDLE] == 7.0).all(), "the idle row's output rows were written"

    for b in range(2):
        rec = SequentialTwin(twins[(b, S)])
        tw_out = torch.empty(1, S, Hq, D, dtype=dtype, device=DEV)
        for t in range(S):
            ct, st = (None, None) if cos is None else (cos[b, t : t + 1], sin[b, t : t + 1])
            rec.step(qkv[b : b + 1, t : t + 1].clone(), ct, st, rope, tw_out[:, t : t + 1])
        for (bb, a), tw in twins.items():
            if bb == b and a < S:
                for t in range(a):
                    ct, st = (None, None) if cos is None else (cos[b, t : t + 1], sin[b, t : t + 1])
                    tw.attend(0, qkv[b : b + 1, t : t + 1].clone(), ct, st, rope,
                              torch.empty(1, 1, Hq, D, dtype=dtype, device=DEV))
        q = qkv[b : b + 1, :, : Hq * D].view(1, S, Hq, D).double()
        if cos is not None:
            q = rotate(q, cos[b][None, :, None], sin[b][None, :, None]).to(dtype).double()
        ref = reference(rec, q, G, D ** -0.5).float()
        assert_parity(tw_out, ref, f"row {b} twin")
        assert_parity(out[b : b + 1], ref, f"row {b}")

    for c, counts in zip(caches, count_sets):
        c.accept(counts)
        assert c.pending_verify is None
        for b in range(2):
            r, tw, n = c.row(b), twins[(b, counts[b])], LENGTHS[b] + counts[b]
            for name in ("full_k", "full_v"):
                assert torch.equal(r.tensors[0][name][:, :, :n], tw.tensors[0][name][:, :, :n]), (b, name)
            for name in ("ring_k", "ring_v"):
                assert torch.equal(r.tensors[0][name][:, :, : c.W], tw.tensors[0][name][:, :, : c.W]), (b, name)
            assert (r.kv_seq_len_list, r.total_list, r.lo_list) == (tw.kv_seq_len_list, tw.total_list, tw.lo_list)
            assert c.row_state[b, :3].tolist() == [tw.kv_seq_len_list[0], tw.total_list[0], tw.lo_list[0]]
        assert c.row_lengths[IDLE] == LENGTHS[IDLE]
        for k, v in c.row(IDLE).tensors[0].items():
            assert torch.equal(v[0], idle_before[k]), f"idle row: {k} changed"


def test_ragged_refusals_change_nothing():
    Hq, dtype = 8, torch.bfloat16
    width = (Hq + 2 * HKV) * D
    c = new_ragged(True, Hq, 1, dtype)
    gen = torch.Generator().manual_seed(1)
    for b, n in enumerate(LENGTHS):
        c.row(b).attend(0, (torch.randn(1, n, width, generator=gen) * 0.5).to(dtype).to(DEV), None, None,
                        _C.ROPE_NONE, torch.empty(1, n, Hq, D, dtype=dtype, device=DEV))
    qkv = (torch.randn(3, 3, width, generator=gen) * 0.5).to(dtype).to(DEV)
    out = torch.empty(3, 3, Hq, D, dtype=dtype, device=DEV)
    big = qkv[:, :1].repeat(1, 5, 1)  # G * S = 20 > 16
    with pytest.raises(ValueError):
        c.verify(0, big, None, None, _C.ROPE_NONE, torch.empty(3, 5, Hq, D, dtype=dtype, device=DEV))
    c.verify(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
    snap = {k: v.clone() for k, v in c.tensors[0].items()}
    rs = c.row_state.clone()
    state = c.snapshot_state()
    for call in (lambda: c.attend(0, qkv[:, :1].clone(), None, None, _C.ROPE_NONE, out[:, :1]),
                 lambda: c.row(0).attend(0, qkv[:1].clone(), None, None, _C.ROPE_NONE, out[:1]),
                 lambda: c.evict_last(1), lambda: c.row(1).evict_last(1), lambda: c.share_prefix(1, 2, 64),
                 lambda: c.accept([1, 1]), lambda: c.accept([4, 0, 0]), lambda: c.accept([1, -1, 0]),
                 lambda: c.set_active(0, False)):
        with pytest.raises(ValueError):
            call()
        assert c.snapshot_state() == state and c.pending_verify == 3 and torch.equal(c.row_state, rs)
        assert all(torch.equal(v, snap[k]) for k, v in c.tensors[0].items())
    c.clear()
    assert c.pending_verify is None
