"""duo_prefill_seq, host side (no GPU): the symbol is exported and declared, and every refusal fires before any CUDA
call (on layer handles that need no tensor map: a 16-bit layer without heads, or an INT4 layer)."""
import ctypes as C
import os
import re

import pytest

from duo_attention_b200 import _C

QKV, OUT, PO, PL = 0x10000, 0x20000, 0x30000, 0x40000
STRIDE = 16 * 128
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "duo_b200.h")


def _layer(lib, group=4, n_full=0, full_cap=0, kv_format=_C.KV_SAME, stage_cap=4096):
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = full_cap, 1, n_full, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, stage_cap, _C.DT_BF16, kv_format
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK, _C.last_error()
    return h.value


def _state(full_len=0, rank=0, world=0, block=0, device_state=None):
    st = _C.CacheState(full_len, full_len, 4, device_state)
    st.seq_rank, st.seq_world, st.seq_block = rank, world, block
    return st


def _prefill(lib, h, st, q_len, q=QKV, out=OUT, po=PO, pl=PL):
    return lib.duo_prefill_seq(h, C.byref(st), q, STRIDE, out, po, pl, q_len, 0.1, None, 0, None)


def test_symbol_is_exported_and_declared():
    lib = _C.load()
    assert "duo_prefill_seq" in _C.SYMBOLS
    getattr(lib, "duo_prefill_seq")
    with open(HEADER) as f:
        assert re.search(r"DUO_API int duo_prefill_seq\(", f.read())


@pytest.fixture
def lib():
    return _C.load()


def test_state_without_shard_descriptor_is_refused(lib):
    h = _layer(lib)
    try:
        assert _prefill(lib, h, _state(10), 200) == _C.DUO_EINVAL
        assert "carries no sequence-shard descriptor" in _C.last_error()
        assert _prefill(lib, h, _state(10, 0, 9, 16), 200) == _C.DUO_EINVAL
        assert "bad sequence-shard descriptor" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


def test_int4_layer_is_refused(lib):
    h = _layer(lib, n_full=1, full_cap=4096, kv_format=_C.KV_INT4)
    try:
        assert _prefill(lib, h, _state(10, 1, 2, 16), 200) == _C.DUO_EINVAL
        assert "16-bit caches only" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


@pytest.mark.parametrize("which", ["q", "out", "po", "pl"])
def test_null_buffers_are_refused(lib, which):
    h = _layer(lib)
    try:
        rc = _prefill(lib, h, _state(10, 0, 2, 16), 200, **{which: None})
        assert rc == _C.DUO_EINVAL and "null buffer" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


@pytest.mark.parametrize("group,q_len", [(4, 1), (4, 4), (16, 1), (1, 16), (2, 8)])
def test_decode_sized_chunks_are_refused(lib, group, q_len):
    h = _layer(lib, group=group)
    try:
        assert _prefill(lib, h, _state(10, 0, 2, 16), q_len) == _C.DUO_EINVAL
        msg = _C.last_error()
        assert "group * q_len > 16" in msg and "duo_attention_seq" in msg, msg
    finally:
        lib.duo_layer_destroy(h)


def test_device_state_is_refused(lib):
    h = _layer(lib)
    try:
        assert _prefill(lib, h, _state(10, 0, 2, 16, device_state=0x70000), 200) == _C.DUO_EINVAL
        assert "device_state" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


def test_existing_entry_points_keep_their_row_limits(lib):
    """duo_prefill_seq is a separate entry point: duo_attention_seq still refuses group * q_len > 16."""
    h = _layer(lib)
    try:
        st = _state(10, 0, 2, 16)
        rc = lib.duo_attention_seq(h, C.byref(st), QKV, STRIDE, OUT, PO, PL, 5, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "group * q_len <= 16" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h)


@pytest.mark.parametrize("world,block", [(2, 16), (3, 5), (8, 1024)])
def test_overflow_of_the_local_slice_is_refused(lib, world, block):
    """The rank whose slice lacks room for the chunk's positions gets DUO_EOVERFLOW with the reference's message, the
    staging capacity is checked too; a chunk that fits reaches the KV-format check (the INT4 layer stops it there)."""
    from duo_attention_b200.seqshard import SeqShardPlan

    plan = SeqShardPlan(world, block)
    cap = 64
    h = _layer(lib, n_full=1, full_cap=cap, kv_format=_C.KV_INT4, stage_cap=512)
    try:
        for rank in range(world):
            for n, q_len in [(0, 100), (40, 300), (100, 17), (cap * world, 200)]:
                rc = _prefill(lib, h, _state(n, rank, world, block), q_len)
                if plan.local_len(rank, n + q_len) > cap:
                    assert rc == _C.DUO_EOVERFLOW and f"Trying to put {q_len} KVs" in _C.last_error()
                else:
                    assert rc == _C.DUO_EINVAL and "16-bit caches only" in _C.last_error()
            assert _prefill(lib, h, _state(0, rank, world, block), 513) in (_C.DUO_EOVERFLOW,)
    finally:
        lib.duo_layer_destroy(h)
