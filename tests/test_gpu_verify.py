"""Verify chunks on static caches (DuoKVCache.verify / accept, duo_decode_verify, duo_rope_append +
duo_attention_verify).  Each case feeds one chunk of S drafted tokens to verifying caches and the same qkv rows, one
token per step, to sequential twins:

* every row of the verify output passes the parity gate against fp64 attention over the keys the twin's step for that
  token saw (the per-token streaming windows), with the oldest live ring slots and the dead ones holding V = +-64, so
  weight on a slot outside a token's window fails;
* retrieval-head rows are bit-identical to duo_decode_fused / duo_attention on the same chunk (a third cache), and all
  rows are where the chunk masks no ring slot;
* after accept(a) for a in {0, 1, ceil(S / 2), S} the retrieval rows, sink / ring slots, lengths, total, lo and
  dev_state are those of the twin after a steps, and further decode steps give the same bits.
"""
import math

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from parity import assert_parity
from verify_ref import D, SequentialTwin, reference, rope_tables, rotate, slot_valid

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
SINK, RECENT, B, HKV = 8, 24, 2, 2
CONTEXTS = {"unwrapped": ([12], 0), "wrapped": ([40, 30], 0), "evicted": ([40, 30], 9)}


def poison_ring(c, S):
    """V = +-64 in the slots of the S oldest live ring positions (seen by the chunk's first tokens only) and in every
    dead ring slot (seen by none)."""
    n, total, lo = c.kv_seq_len_list[0], c.total_list[0], c.lo_list[0]
    sign = torch.where(torch.arange(D, device=DEV) % 2 == 0, 64.0, -64.0).to(c.dtype)
    for j in range(SINK, c.W):
        pos_live = slot_valid(j, SINK, RECENT, total, lo)
        if pos_live:
            last = total - 1
            p = last - (last - j) % RECENT
            if p >= lo + S:
                continue
        c.tensors[0]["ring_v"][:, :, j] = sign


def feed(caches, chunks, evict, width, dtype, rope, gen):
    pos = 0
    for n in chunks:
        qkv = (torch.randn(B, n, width, generator=gen) * 0.5).to(dtype).to(DEV)
        cos, sin = rope_tables(list(range(pos, pos + n)), rope, dtype, DEV)
        for c in caches:
            c.attend(0, qkv.clone(), cos, sin, rope, torch.empty(B, n, width // D - 2 * HKV, D, dtype=dtype, device=DEV))
        pos += n
    for c in caches:
        if evict:
            c.evict_last(evict)
        c.enable_device_state()


def assert_same_bytes(c, twin, n):
    for name in ("full_k", "full_v"):
        assert torch.equal(c.tensors[0][name][:, :, :n], twin.tensors[0][name][:, :, :n]), name
    for name in ("ring_k", "ring_v"):
        assert torch.equal(c.tensors[0][name][:, :, : c.W], twin.tensors[0][name][:, :, : c.W]), name
    assert (c.kv_seq_len_list, c.total_list, c.lo_list) == (twin.kv_seq_len_list, twin.total_list, twin.lo_list)
    assert torch.equal(c.dev_state, twin.dev_state)


def run_case(dtype, G, rope, n_full, ctx, S, seed):
    Hq = HKV * G
    width = (Hq + 2 * HKV) * D
    gen = torch.Generator().manual_seed(seed)
    mk = lambda: DuoKVCache(1, Hq, HKV, D, [n_full], B, 256, SINK, RECENT, dtype, DEV, stage_cap=64)
    accepts = sorted({0, 1, math.ceil(S / 2), S})
    ver = {a: mk() for a in accepts}
    twins = {a: mk() for a in accepts}
    ctl = mk()
    everyone = [*ver.values(), *twins.values(), ctl]
    chunks, evict = CONTEXTS[ctx]
    feed(everyone, chunks, evict, width, dtype, rope, gen)
    ctl.dev_state = None  # (duo_attention takes device_state only for chunks of <= 16 tokens)
    n, total, lo = ctl.kv_seq_len_list[0], ctl.total_list[0], ctl.lo_list[0]
    for c in everyone:
        poison_ring(c, S)
    qkv = (torch.randn(B, S, width, generator=gen) * 0.5).to(dtype).to(DEV)
    cos, sin = rope_tables(list(range(n, n + S)), rope, dtype, DEV)
    new_out = lambda s: torch.full((B, s, Hq, D), 7.0, dtype=dtype, device=DEV)

    outs = []
    for a, c in ver.items():
        outs.append(c.verify(0, qkv.clone(), cos, sin, rope, new_out(S)))
        assert c.pending_verify == S and c.kv_seq_len_list[0] == n and c.total_list[0] == total
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    out = outs[0]
    out_ctl = ctl.attend(0, qkv.clone(), cos, sin, rope, new_out(S))

    # the twins: twins[S] takes every token and records the keys of each step
    rec = SequentialTwin(twins[S])
    twin_out = new_out(S)
    for t in range(S):
        ct, st = (None, None) if cos is None else (cos[t : t + 1], sin[t : t + 1])
        o_t = new_out(1)
        rec.step(qkv[:, t : t + 1].clone(), ct, st, rope, o_t)
        twin_out[:, t : t + 1] = o_t
    for a, c in twins.items():
        for t in range(a if a < S else 0):
            ct, st = (None, None) if cos is None else (cos[t : t + 1], sin[t : t + 1])
            c.attend(0, qkv[:, t : t + 1].clone(), ct, st, rope, new_out(1))
            c.advance_device(1)

    q = qkv[..., : Hq * D].view(B, S, Hq, D).double()
    if cos is not None:
        q = rotate(q, cos[None, :, None], sin[None, :, None]).to(dtype).double()
    ref = reference(rec, q, G, D ** -0.5).float()
    what = f"{dtype} G{G} rope{rope} n_full{n_full} {ctx} S{S}"
    assert_parity(twin_out, ref, what + " (the sequential twin)")
    assert_parity(out, ref, what)
    nr = n_full * G
    assert torch.equal(out[:, :, :nr], out_ctl[:, :, :nr]), "retrieval rows differ from the plain chunk's"
    if total + S - 1 - RECENT <= lo:  # no ring slot is masked for any token: the chunk rule itself
        assert torch.equal(out, out_ctl)

    for a in accepts:
        ver[a].accept(a)
        assert ver[a].pending_verify is None
        assert_same_bytes(ver[a], twins[a], n + a)
        for _ in range(2):  # decode continues with the same bits
            q1 = (torch.randn(B, 1, width, generator=gen) * 0.5).to(dtype).to(DEV)
            p = ver[a].kv_seq_len_list[0]
            c1, s1 = rope_tables([p], rope, dtype, DEV)
            o1 = ver[a].attend(0, q1.clone(), c1, s1, rope, new_out(1))
            o2 = twins[a].attend(0, q1.clone(), c1, s1, rope, new_out(1))
            ver[a].advance_device(1)
            twins[a].advance_device(1)
            assert torch.equal(o1, o2)
            assert_same_bytes(ver[a], twins[a], p + 1)


# (dtype, G, S): G * S <= 16 takes duo_decode_verify, larger chunks duo_rope_append + duo_attention_verify (16 rows at
# G = 1, the 64-row kernel above)
SHAPES = [(dt, 1, S) for dt in (torch.bfloat16, torch.float16) for S in (2, 16, 20)] + \
         [(dt, 4, S) for dt in (torch.bfloat16, torch.float16) for S in (2, 4, 5, 16)]
ROPES = [_C.ROPE_NONE, _C.ROPE_HF, _C.ROPE_FP32]
HEADS = {"none": 0, "some": 1, "all": 2}


@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("i", range(len(SHAPES)))
def test_verify_shapes(i, ctx):
    dtype, G, S = SHAPES[i]
    run_case(dtype, G, ROPES[i % 3], list(HEADS.values())[(i // 3 + i) % 3], ctx, S, seed=100 + i)


@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("heads", list(HEADS))
@pytest.mark.parametrize("rope", ROPES, ids=["none", "hf", "fp32"])
def test_verify_rope_and_heads(rope, heads, ctx):
    run_case(torch.bfloat16, 4, rope, HEADS[heads], ctx, 5, seed=7 + rope)
    run_case(torch.float16, 1, rope, HEADS[heads], ctx, 9, seed=9 + rope)


def test_pending_state_refusals_change_nothing():
    dtype, Hq = torch.bfloat16, 8
    width = (Hq + 2 * HKV) * D
    c = DuoKVCache(1, Hq, HKV, D, [1], B, 256, SINK, RECENT, dtype, DEV, stage_cap=64)
    gen = torch.Generator().manual_seed(3)
    feed([c], [40], 0, width, dtype, _C.ROPE_NONE, gen)
    qkv = (torch.randn(B, 3, width, generator=gen) * 0.5).to(dtype).to(DEV)
    out = torch.empty(B, 3, Hq, D, dtype=dtype, device=DEV)
    for bad in (qkv[:, :1].repeat(1, RECENT + 1, 1), qkv[:, :1].repeat(1, 17, 1)):  # S > recent, G * S > 64
        with pytest.raises(ValueError):
            c.verify(0, bad, None, None, _C.ROPE_NONE, torch.empty(B, bad.shape[1], Hq, D, dtype=dtype, device=DEV))
    with pytest.raises(ValueError):
        c.accept(0)  # nothing pending
    c.verify(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
    snap = {k: v.clone() for k, v in c.tensors[0].items()}
    state = c.snapshot_state()
    for call in (lambda: c.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, out),
                 lambda: c.verify(0, qkv.clone(), None, None, _C.ROPE_NONE, out),
                 lambda: c.evict_last(1), lambda: c.accept(4), lambda: c.accept(-1), lambda: c.accept(True)):
        with pytest.raises(ValueError):
            call()
        assert c.snapshot_state() == state and c.pending_verify == 3
        assert all(torch.equal(v, snap[k]) for k, v in c.tensors[0].items())
    c.clear()  # discards the chunk
    assert c.pending_verify is None and c.kv_seq_len == 0
