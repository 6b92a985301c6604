"""The INT4 sequence-sharded entry points (duo_attention_seq_int4, duo_decode_fused_seq_int4), host side (no GPU): every
refusal of the C ABI runs before any CUDA call — a bad or missing shard descriptor, a 16-bit layer, too many packed
rows, null buffers, and the owner's overflow at exactly its local capacity.  The layers need no tensor map (INT4
layers, or a 16-bit layer without heads)."""
import ctypes as C

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.seqshard import SeqShardPlan

QKV, OUT, PO, PL, COS, SIN = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
STRIDE = 16 * 128  # qkv row stride in elements: a multiple of 8
NAMES = ("duo_attention_seq_int4", "duo_decode_fused_seq_int4")


def _layer(lib, group=4, n_full=1, full_cap=64, kv_format=_C.KV_INT4, stage_cap=8):
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


def _call(lib, name, h, st, q_len=1, out=OUT, po=PO, pl=PL):
    if name == "duo_attention_seq_int4":
        return lib.duo_attention_seq_int4(h, C.byref(st), QKV, STRIDE, out, po, pl, q_len, 0.1, None, 0, None)
    return lib.duo_decode_fused_seq_int4(h, C.byref(st), QKV, STRIDE, None, None, _C.ROPE_NONE, out, po, pl, 0.1,
                                         None, 0, None)


@pytest.mark.parametrize("rank,world,block", [(0, 1, 16), (0, 9, 16), (-1, 2, 16), (2, 2, 16), (8, 8, 4), (0, 2, 0),
                                              (1, 4, -3), (0, -2, 16)])
def test_bad_shard_descriptor_is_refused(rank, world, block):
    lib = _C.load()
    h = _layer(lib)
    try:
        for name in NAMES:
            assert _call(lib, name, h, _state(10, rank, world, block)) == _C.DUO_EINVAL, name
            assert "bad sequence-shard descriptor" in _C.last_error(), (name, _C.last_error())
    finally:
        lib.duo_layer_destroy(h)


def test_missing_descriptor_16bit_layer_and_null_buffers_are_refused():
    lib = _C.load()
    int4, same = _layer(lib), _layer(lib, n_full=0, full_cap=0, kv_format=_C.KV_SAME)
    sharded = _state(10, 1, 2, 16)
    try:
        for name in NAMES:
            assert _call(lib, name, int4, _state(10)) == _C.DUO_EINVAL, name
            assert "carries no sequence-shard descriptor" in _C.last_error()
            assert _call(lib, name, same, sharded) == _C.DUO_EINVAL, name
            assert "INT4 caches only" in _C.last_error()
            for bufs in ({"out": None}, {"po": None}, {"pl": None}):
                assert _call(lib, name, int4, sharded, **bufs) == _C.DUO_EINVAL, (name, bufs)
                assert "null buffer" in _C.last_error()
        # the 16-bit entry points keep refusing INT4 layers, and name their INT4 twins
        rc = lib.duo_attention_seq(int4, C.byref(sharded), QKV, STRIDE, OUT, PO, PL, 1, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "16-bit caches" in _C.last_error() and NAMES[0] in _C.last_error()
        rc = lib.duo_decode_fused_seq(int4, C.byref(sharded), QKV, STRIDE, None, None, _C.ROPE_NONE, OUT, PO, PL, 0.1,
                                      None, 0, None)
        assert rc == _C.DUO_EINVAL and "16-bit caches" in _C.last_error() and NAMES[1] in _C.last_error()
    finally:
        for h in (int4, same):
            lib.duo_layer_destroy(h)


def test_packed_rows_are_limited_to_the_int4_decode_kernel():
    lib = _C.load()
    st = _state(10, 0, 2, 16)
    g4, g8, g16 = _layer(lib, group=4), _layer(lib, group=8), _layer(lib, group=16)
    try:
        for h, q_len in ((g4, 3), (g8, 2)):
            assert _call(lib, "duo_attention_seq_int4", h, st, q_len=q_len) == _C.DUO_EINVAL
            assert f"group * q_len <= {_C.DECODE_MAX_Q_INT4}" in _C.last_error()
        for name in NAMES:
            assert _call(lib, name, g16, st) == _C.DUO_EINVAL, name
            assert f"group * q_len <= {_C.DECODE_MAX_Q_INT4}" in _C.last_error()
    finally:
        for h in (g4, g8, g16):
            lib.duo_layer_destroy(h)


def test_owner_overflows_at_exactly_the_local_capacity():
    """Every rank holds exactly plan.capacity(n) rows: the owner of position n is refused (DUO_EOVERFLOW) by both
    entry points; the other ranks pass the capacity check (and stop at the packed-row limit of a group-16 layer, the
    last check before the launch)."""
    lib = _C.load()
    for world, block, n in [(2, 16, 64), (2, 16, 72), (4, 1, 32), (3, 8, 48), (8, 1, 64), (5, 8, 80)]:
        plan = SeqShardPlan(world, block)
        cap = plan.capacity(n)
        assert cap % 8 == 0
        h = _layer(lib, group=16, full_cap=cap)
        try:
            for rank in range(world):
                st = _state(n, rank, world, block)
                for name in NAMES:
                    rc = _call(lib, name, h, st)
                    if plan.owner(n) == rank:
                        assert rc == _C.DUO_EOVERFLOW, (name, world, block, n, rank)
                        assert f"Trying to put 1 KVs into a cache with max size {cap}" in _C.last_error()
                    else:
                        assert rc == _C.DUO_EINVAL and "group * q_len" in _C.last_error(), (name, rank, _C.last_error())
        finally:
            lib.duo_layer_destroy(h)
