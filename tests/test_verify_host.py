"""Verify chunks without a GPU: the verify entry points and duo_stream_commit_rows refusing bad arguments before any
CUDA call, the cache-side refusals that need no device, and the accept arithmetic against ring_advance."""
import ctypes as C

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import (DuoKVCache, DuoRaggedKVCache, DuoSeqShardKVCache, _refuse_pending,
                                         ring_advance)


def _layer(lib, batch=2, kv_format=_C.KV_SAME, group=4, sink=4, recent=8, stage_cap=64, pool_tokens=0):
    """A handle that needs no tensor map (a 16-bit layer without heads, or an INT4 layer)."""
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, 0, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = sink, recent, stage_cap, _C.DT_BF16, kv_format
    h = C.c_void_p()
    if pool_tokens:
        assert lib.duo_layer_create_pooled(C.byref(d), pool_tokens, C.byref(h)) == _C.DUO_OK, _C.last_error()
    else:
        assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK, _C.last_error()
    return h.value


QKV, OUT, COS, SIN, RS, RG = 0x40000, 0x50000, 0x60000, 0x70000, 0x10000, 0x20000


def _st(seq_world=0, **kw):
    st = _C.CacheState(kw.get("full_len", 10), kw.get("total", 10), kw.get("lo", 4), None)
    if seq_world:
        st.seq_rank, st.seq_world, st.seq_block = 0, seq_world, 64
    return st


def test_verify_entry_points_refuse_before_cuda():
    lib = _C.load()
    L = _layer(lib)
    i4 = _layer(lib, kv_format=_C.KV_INT4)
    small = _layer(lib, stage_cap=2)
    pooled = _layer(lib, pool_tokens=256)
    dec = lambda h, st=None, q_len=2, **kw: lib.duo_decode_verify(
        h, C.byref(st or _st()), kw.get("qkv", QKV), 16 * 128, COS, SIN, _C.ROPE_HF, kw.get("out", OUT), q_len, 0.1,
        None, 0, None)
    att = lambda h, st=None, q_len=2: lib.duo_attention_verify(h, C.byref(st or _st()), QKV, 16 * 128, OUT, q_len, 0.1,
                                                                None, 0, None)
    rag = lambda h, q_len=2, rg=None, rs=RS, room=100: lib.duo_decode_ragged_verify(
        h, rs, rg, room, QKV, 16 * 128, COS, SIN, _C.ROPE_HF, OUT, q_len, 0.1, None, 0, None)
    try:
        inval = {
            "decode: INT4": dec(i4), "decode: sharded": dec(L, _st(seq_world=2)), "decode: G*S > 16": dec(L, q_len=5),
            "decode: S > recent": dec(_layer(lib, group=1), q_len=9), "decode: null out": dec(L, out=None),
            "decode: unaligned qkv": dec(L, qkv=QKV + 8),
            "attention: INT4": att(i4), "attention: sharded": att(L, _st(seq_world=2)),
            "attention: G*S > 64": att(L, q_len=17), "attention: S > recent": att(_layer(lib, group=1), q_len=9),
            "ragged: INT4": rag(i4), "ragged: G*S > 16": rag(L, q_len=5), "ragged: S > recent":
                rag(_layer(lib, group=1), q_len=9), "ragged: null row_state": rag(L, rs=None),
            "ragged: pooled layer without row_geom": rag(pooled), "ragged: row_geom on a uniform layer": rag(L, rg=RG),
        }
        for what, rc in inval.items():
            assert rc == _C.DUO_EINVAL, (what, rc, _C.last_error())
        over = {"decode: S > stage_cap": dec(small, q_len=3), "attention: S > stage_cap": att(small, q_len=3),
                "ragged: S > stage_cap": rag(small, q_len=3)}
        for what, rc in over.items():
            assert rc == _C.DUO_EOVERFLOW, (what, rc, _C.last_error())
        commit = lambda h, counts, rs=RS: lib.duo_stream_commit_rows(h, rs, (C.c_int32 * len(counts))(*counts), None)
        assert commit(L, [1, 0], rs=None) == _C.DUO_EINVAL
        assert lib.duo_stream_commit_rows(L, RS, None, None) == _C.DUO_EINVAL
        assert commit(i4, [1, 0]) == _C.DUO_EINVAL
        assert commit(L, [-1, 0]) == _C.DUO_EINVAL
        assert commit(L, [9, 0]) == _C.DUO_EINVAL  # > recent
        assert commit(small, [3, 0]) == _C.DUO_EOVERFLOW
        assert commit(L, [0, 0]) == _C.DUO_OK  # a layer without streaming heads: nothing to launch
    finally:
        for h in (L, i4, small, pooled):
            lib.duo_layer_destroy(h)


class _Bare:
    """The integers the cache-side checks read, on an object that owns no device memory."""

    def __new__(cls, base, **kw):
        c = object.__new__(base)
        c.kv_format, c.graph_attached, c.num_kv_groups, c.recent_size, c.num_layers = "same", False, 4, 8, 2
        c._verify_len = [0, 0]
        for k, v in kw.items():
            setattr(c, k, v)
        return c


@pytest.mark.parametrize("what,base,kw,S", [
    ("INT4", DuoKVCache, dict(kv_format="int4"), 2),
    ("sequence-sharded", DuoSeqShardKVCache, {}, 2),
    ("graph attached", DuoKVCache, dict(graph_attached=True), 2),
    ("too many rows", DuoKVCache, {}, 17),
    ("S > recent", DuoKVCache, dict(num_kv_groups=1), 9),
    ("layer pending", DuoKVCache, dict(_verify_len=[2, 0]), 2),
    ("other length pending", DuoKVCache, dict(_verify_len=[0, 3]), 2),
])
def test_cache_refuses_verify_chunks(what, base, kw, S):
    c = _Bare(base, **kw)
    before = dict(vars(c))
    with pytest.raises(ValueError):
        c._check_verify(0, S, _C.VERIFY_MAX_ROWS)
    assert vars(c) == before


def test_pending_chunk_refuses_other_calls():
    c = _Bare(DuoKVCache, _verify_len=[3, 3])
    assert c.pending_verify == 3
    for what in ("attend", "evict_last"):
        with pytest.raises(ValueError, match="awaits accept"):
            _refuse_pending(c, what)
    for bad in (4, -1, True, 1.5):
        with pytest.raises(ValueError):
            c.accept(bad)
    assert c._verify_len == [3, 3]
    half = _Bare(DuoKVCache, _verify_len=[3, 0])  # not every layer holds the chunk
    with pytest.raises(ValueError):
        half.accept(1)
    rg = _Bare(DuoRaggedKVCache, _verify_len=[3, 3], batch_size=3, _active=[True, True, False])
    for bad in ([1, 1], [4, 0, 0], [1, -1, 0], [1, 1, 1], "abc", [1.0, 0, 0]):
        with pytest.raises(ValueError):
            rg.accept(bad)


@pytest.mark.parametrize("sink,recent", [(4, 8), (8, 24), (0, 5)])
def test_accept_arithmetic_matches_one_token_steps(sink, recent):
    """accept(a) advances total / lo once by a; a one-token steps advance them a times by 1: the same state, from any
    reachable state (including one after an eviction)."""
    for total0 in range(0, 3 * (sink + recent)):
        for lo_back in (0, 3):
            lo0 = max(sink, total0 - recent)
            lo0 = max(sink, min(lo0, total0 - lo_back)) if total0 >= sink else sink
            for a in range(0, recent + 1):
                t1, l1 = ring_advance(total0, lo0, a, sink, recent)
                t2, l2 = total0, lo0
                for _ in range(a):
                    t2, l2 = ring_advance(t2, l2, 1, sink, recent)
                assert (t1, l1) == (t2, l2)
