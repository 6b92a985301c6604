"""Sequence-sharded decode, host side (no GPU): every argument check of the shard descriptor in the C ABI, and the
capacity check of check_chunk (api.cu) against SeqShardPlan.local_len.  All of these run before any CUDA call, on
layer handles that need no tensor map (a 16-bit layer without heads, or an INT4 layer)."""
import ctypes as C

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.seqshard import SeqShardPlan

QKV, OUT, PO, PL, COS, SIN = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
STRIDE = 16 * 128  # qkv row stride in elements: a multiple of 8


def _layer(lib, group=4, n_full=0, full_cap=0, kv_format=_C.KV_SAME, stage_cap=64):
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = full_cap, 1, n_full, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, stage_cap, _C.DT_BF16, kv_format
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK, _C.last_error()
    return h.value


def _state(full_len=0, rank=0, world=0, block=0):
    st = _C.CacheState(full_len, full_len, 4, None)
    st.seq_rank, st.seq_world, st.seq_block = rank, world, block
    return st


def _calls(lib, h, st, q_len=1):
    """The four entry points that take a shard descriptor, called with valid buffers."""
    return {
        "duo_rope_append": lambda: lib.duo_rope_append(h, C.byref(st), QKV, STRIDE, None, None, _C.ROPE_NONE, q_len,
                                                       None),
        "duo_attention_seq": lambda: lib.duo_attention_seq(h, C.byref(st), QKV, STRIDE, OUT, PO, PL, q_len, 0.1, None, 0,
                                                           None),
        "duo_decode_fused_seq": lambda: lib.duo_decode_fused_seq(h, C.byref(st), QKV, STRIDE, None, None, _C.ROPE_NONE,
                                                                 OUT, PO, PL, 0.1, None, 0, None),
        "duo_stream_commit": lambda: lib.duo_stream_commit(h, C.byref(st), q_len, None),
    }


@pytest.mark.parametrize("rank,world,block", [(0, 1, 16), (0, 9, 16), (-1, 2, 16), (2, 2, 16), (8, 8, 4), (0, 2, 0),
                                              (1, 4, -3), (0, -2, 16)])
def test_bad_shard_descriptor_is_refused(rank, world, block):
    lib = _C.load()
    h = _layer(lib)
    try:
        for name, call in _calls(lib, h, _state(10, rank, world, block)).items():
            assert call() == _C.DUO_EINVAL, name
            assert "bad sequence-shard descriptor" in _C.last_error(), (name, _C.last_error())
    finally:
        lib.duo_layer_destroy(h)


def test_descriptor_and_entry_point_must_agree():
    lib = _C.load()
    h = _layer(lib)
    try:
        sharded, plain = _state(10, 1, 2, 16), _state(10)
        rc = lib.duo_attention(h, C.byref(sharded), QKV, STRIDE, OUT, 1, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "duo_attention_seq" in _C.last_error()
        rc = lib.duo_decode_fused(h, C.byref(sharded), QKV, STRIDE, None, None, _C.ROPE_NONE, OUT, 1, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "unsharded caches" in _C.last_error()
        for name in ("duo_attention_seq", "duo_decode_fused_seq"):
            assert _calls(lib, h, plain)[name]() == _C.DUO_EINVAL, name
            assert "carries no sequence-shard descriptor" in _C.last_error()
        # partial-output buffers are required
        rc = lib.duo_attention_seq(h, C.byref(sharded), QKV, STRIDE, OUT, None, PL, 1, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "null buffer" in _C.last_error()
        rc = lib.duo_decode_fused_seq(h, C.byref(sharded), QKV, STRIDE, None, None, _C.ROPE_NONE, OUT, PO, None, 0.1,
                                      None, 0, None)
        assert rc == _C.DUO_EINVAL and "null buffer" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


def test_packed_rows_and_int4_are_refused():
    lib = _C.load()
    st = _state(10, 0, 2, 16)
    g4, g16, g17 = _layer(lib, group=4), _layer(lib, group=16), _layer(lib, group=17)
    int4 = _layer(lib, n_full=1, full_cap=64, kv_format=_C.KV_INT4)
    try:
        assert _calls(lib, g4, st, q_len=5)["duo_attention_seq"]() == _C.DUO_EINVAL
        assert "group * q_len <= 16" in _C.last_error()
        assert _calls(lib, g16, st, q_len=2)["duo_attention_seq"]() == _C.DUO_EINVAL
        assert _calls(lib, g17, st)["duo_decode_fused_seq"]() == _C.DUO_EINVAL
        assert "group <= 16" in _C.last_error()
        for name in ("duo_attention_seq", "duo_decode_fused_seq"):
            assert _calls(lib, int4, st)[name]() == _C.DUO_EINVAL, name
            assert "16-bit caches" in _C.last_error()
    finally:
        for h in (g4, g16, g17, int4):
            lib.duo_layer_destroy(h)


def _fits(lib, h, full_len, q_len, rank, world, block):
    """True if check_chunk lets the chunk through (duo_attention_seq on an INT4 layer then refuses the KV format, before
    any CUDA call), False on DUO_EOVERFLOW."""
    st = _state(full_len, rank, world, block)
    rc = lib.duo_attention_seq(h, C.byref(st), QKV, STRIDE, OUT, PO, PL, q_len, 0.1, None, 0, None)
    if rc == _C.DUO_EOVERFLOW:
        msg = _C.last_error()
        assert f"Trying to put {q_len} KVs into a cache with max size" in msg, msg
        return False
    assert rc == _C.DUO_EINVAL and "16-bit caches" in _C.last_error(), (rc, _C.last_error())
    return True


@pytest.mark.parametrize("world,block", [(2, 1), (2, 16), (3, 5), (4, 1), (4, 3), (5, 8), (8, 2), (8, 13)])
def test_local_capacity_check_agrees_with_the_plan(world, block):
    """For every rank, chunk size and context length around the capacity: the C ABI reports DUO_EOVERFLOW exactly
    when the rows of the rank's slice after the append (SeqShardPlan.local_len) exceed its capacity."""
    lib = _C.load()
    plan = SeqShardPlan(world, block)
    for cap in (8, 24):
        h = _layer(lib, n_full=1, full_cap=cap, kv_format=_C.KV_INT4, stage_cap=8)
        try:
            for rank in range(world):
                for q_len in (1, 2, 3, 8):
                    n = 0
                    while plan.local_len(rank, n) <= cap:  # every length up to the first one already past capacity
                        want = plan.local_len(rank, n + q_len) <= cap
                        assert _fits(lib, h, n, q_len, rank, world, block) == want, (cap, rank, q_len, n)
                        n += 1
        finally:
            lib.duo_layer_destroy(h)


def test_owner_overflows_at_exactly_the_local_capacity():
    """Every rank holds exactly plan.capacity(n) rows: the owner of position n is refused, the other ranks are not, on
    every entry point that appends or attends."""
    lib = _C.load()
    # (an INT4 layer keeps full_cap a multiple of 8: contexts whose capacity is one)
    for world, block, n in [(2, 16, 64), (2, 16, 72), (4, 1, 32), (3, 8, 48), (8, 1, 64), (5, 8, 80)]:
        plan = SeqShardPlan(world, block)
        cap = plan.capacity(n)
        assert cap % 8 == 0
        h = _layer(lib, n_full=1, full_cap=cap, kv_format=_C.KV_INT4, stage_cap=8)
        try:
            for rank in range(world):
                if plan.owner(n) != rank:  # accepted (the call would go on to launch: check it on the layer's format)
                    assert _fits(lib, h, n, 1, rank, world, block), (world, block, n, rank)
                    continue
                for name, call in _calls(lib, h, _state(n, rank, world, block)).items():
                    assert call() == _C.DUO_EOVERFLOW, (name, world, block, n, rank)
                    assert f"Trying to put 1 KVs into a cache with max size {cap}" in _C.last_error()
        finally:
            lib.duo_layer_destroy(h)
