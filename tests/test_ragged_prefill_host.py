"""The batched ragged prefill without a GPU: duo_prefill_ragged rejecting bad arguments before any CUDA call, the packed
offsets and tile counts of ragged_prefill_plan, and the refusals of attend_rows that need no device."""
import ctypes as C

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import (PREFILL_MAX_WINDOW, DuoRaggedINT4KVCache, DuoRaggedKVCache,
                                         ragged_prefill_plan)


def _layer(lib, batch=3, kv_format=_C.KV_SAME, sink=4, recent=8, stage_cap=64, pool_tokens=0):
    """A handle that needs no tensor map (a 16-bit layer without heads, or an INT4 layer), as the other ABI tests use."""
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, 0, 0, 4, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = sink, recent, stage_cap, _C.DT_BF16, kv_format
    h = C.c_void_p()
    if pool_tokens:
        assert lib.duo_layer_create_pooled(C.byref(d), pool_tokens, C.byref(h)) == _C.DUO_OK, _C.last_error()
    else:
        assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK, _C.last_error()
    return h.value


RS, RG, RSH, QKV, OUT, COS, SIN = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000, 0x70000


def _call(lib, layer, lengths=(5, 0, 7), room=(100, 100, 100), rs=RS, rg=None, rsh=None, qkv=QKV, out=OUT,
          rope_mode=_C.ROPE_HF, cos=COS, sin=SIN, stride=16 * 128):
    lens = (C.c_int32 * len(lengths))(*lengths) if lengths is not None else None
    rooms = (C.c_int64 * len(room))(*room) if room is not None else None
    return lib.duo_prefill_ragged(layer, rs, rg, rsh, lens, rooms, qkv, stride, cos, sin, rope_mode, out, 0.1, None, 0,
                                  None)


def test_entry_point_rejects_bad_arguments_before_cuda():
    lib = _C.load()
    L = _layer(lib)
    bad = {"int4": _layer(lib, kv_format=_C.KV_INT4), "wide": _layer(lib, sink=64, recent=2000),
           "batch65": _layer(lib, batch=65), "pooled": _layer(lib, pool_tokens=256)}
    try:
        inval = {
            "null layer": _call(lib, None), "null row_state": _call(lib, L, rs=None),
            "null lengths": _call(lib, L, lengths=None), "null room": _call(lib, L, room=None),
            "null qkv": _call(lib, L, qkv=None), "null out": _call(lib, L, out=None),
            "null cos": _call(lib, L, cos=None), "null sin": _call(lib, L, sin=None),
            "bad rope_mode": _call(lib, L, rope_mode=7), "skip-q flag": _call(lib, L, rope_mode=_C.ROPE_HF | _C.ROPE_SKIP_Q),
            "unaligned rows": _call(lib, L, stride=16 * 128 + 4), "unaligned qkv": _call(lib, L, qkv=QKV + 8),
            "int4": _call(lib, bad["int4"]), "sink + recent > 2048": _call(lib, bad["wide"]),
            "batch > max": _call(lib, bad["batch65"], lengths=[1] * 65, room=[9] * 65),
            "negative length": _call(lib, L, lengths=(5, -1, 7)),
            "row_geom on a uniform layer": _call(lib, L, rg=RG),
            "row_share on a uniform layer": _call(lib, L, rsh=RSH),
            "pooled without row_geom": _call(lib, bad["pooled"]),
        }
        for what, rc in inval.items():
            assert rc == _C.DUO_EINVAL, (what, rc, _C.last_error())
        # the room of a row counts only for layers with retrieval heads (these have none), staging for every layer
        over = {"chunk > staging": _call(lib, L, lengths=(65, 0, 0))}
        for what, rc in over.items():
            assert rc == _C.DUO_EOVERFLOW, (what, rc, _C.last_error())
        assert "staging capacity" in _C.last_error()
        # nothing to do: every length 0 returns before any CUDA call too
        assert _call(lib, L, lengths=(0, 0, 0)) == _C.DUO_OK
        assert _call(lib, bad["pooled"], rg=RG, rsh=RSH, lengths=(0, 0, 0)) == _C.DUO_OK
        assert _call(lib, L, lengths=(0, 0, 0), rope_mode=_C.ROPE_NONE, cos=None, sin=None) == _C.DUO_OK
    finally:
        for h in [L, *bad.values()]:
            lib.duo_layer_destroy(h)


def test_no_room_is_overflow_on_layers_with_retrieval_heads():
    """A row without room is DUO_EOVERFLOW before any CUDA call; needs a layer with retrieval heads, so a pooled one
    (its pool map is encoded at creation over a fake address, which needs no device)."""
    lib = _C.load()
    d = _C.LayerDesc()
    d.full_k, d.full_v, d.ring_k, d.ring_v = 0x100000, 0x200000, None, None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, 2, 1, 0, 4, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, 64, _C.DT_BF16, _C.KV_SAME
    h = C.c_void_p()
    rc = lib.duo_layer_create_pooled(C.byref(d), 256, C.byref(h))
    if rc != _C.DUO_OK:  # the tensor-map encoder is a driver entry point: absent without a driver
        pytest.skip(f"no CUDA driver to encode a tensor map: {_C.last_error()}")
    try:
        rc = _call(lib, h.value, lengths=(3, 9), room=(3, 8), rg=RG)
        assert rc == _C.DUO_EOVERFLOW and "room for 8 more" in _C.last_error()
    finally:
        lib.duo_layer_destroy(h.value)


@pytest.mark.parametrize("lengths", [[128], [0, 0, 0], [1, 3, 17, 64, 127], [128, 0, 129, 300, 4097, 0], [0, 256, 0]])
def test_plan_packs_rows_back_to_back(lengths):
    T = sum(lengths)
    plan = ragged_prefill_plan(lengths, T, len(lengths))
    off = plan["offsets"]
    assert off[0] == 0 and off[-1] == T and len(off) == len(lengths) + 1
    for b, n in enumerate(lengths):
        assert off[b + 1] - off[b] == n
        assert plan["tiles"][b] == -(-n // 128) and (plan["tiles"][b] - 1) * 128 < n <= plan["tiles"][b] * 128 or n == 0
    assert plan["max_tiles"] == max(plan["tiles"])
    assert plan["rows"] == [b for b, n in enumerate(lengths) if n]
    # every packed token belongs to exactly one row (the kernels' ragged_chunk_row: the last row with off <= token)
    for t in range(0, T, 37):
        b = max(r for r in range(len(lengths)) if off[r] <= t)
        assert off[b] <= t < off[b + 1] and lengths[b] > 0


def test_plan_refusals():
    with pytest.raises(ValueError, match="entries for a batch of 3"):
        ragged_prefill_plan([1, 2], 3, 3)
    with pytest.raises(ValueError, match=">= 0"):
        ragged_prefill_plan([4, -1, 0], 3, 3)
    with pytest.raises(ValueError, match="add up to 5"):
        ragged_prefill_plan([2, 3, 0], 6, 3)


class _Rows:
    """The host state attend_rows reads before it touches a device: a stand-in row with a capacity check."""

    def __init__(self, room):
        self.room = room

    def check_room(self, q_len, layers=None):
        if q_len > self.room:
            raise ValueError(f"Trying to put {q_len} KVs into a cache with max size {self.room}, current size: 0.")


def _host_cache(cls, W=12, rooms=(100, 100, 100)):
    c = cls.__new__(cls)
    c.sink_size, c.recent_size = 4, W - 4
    c.batch_size, c.head_dim, c.num_heads, c.num_kv_heads = len(rooms), 128, 4, 1
    c.rows = [_Rows(r) for r in rooms]
    return c


class _FakeCuda:
    is_cuda = True

    def __init__(self, shape):
        self.shape = shape

    def dim(self):
        return len(self.shape)


def test_attend_rows_refusals():
    width = (4 + 2) * 128
    qkv, out = _FakeCuda((1, 12, width)), _FakeCuda((1, 12, 4, 128))
    with pytest.raises(ValueError, match="16-bit caches only"):
        DuoRaggedINT4KVCache.attend_rows(_host_cache(DuoRaggedINT4KVCache), 0, qkv, None, None, _C.ROPE_NONE, out,
                                         [4, 4, 4])
    with pytest.raises(ValueError, match=f"sink \\+ recent <= {PREFILL_MAX_WINDOW}"):
        _host_cache(DuoRaggedKVCache, W=2049).attend_rows(0, qkv, None, None, _C.ROPE_NONE, out, [4, 4, 4])
    c = _host_cache(DuoRaggedKVCache, rooms=(100, 3, 100))
    with pytest.raises(ValueError, match="entries for a batch of 3"):
        c.attend_rows(0, qkv, None, None, _C.ROPE_NONE, out, [6, 6])
    with pytest.raises(ValueError, match="add up to 11"):
        c.attend_rows(0, qkv, None, None, _C.ROPE_NONE, out, [4, 3, 4])
    with pytest.raises(ValueError, match="Trying to put 4 KVs"):
        c.attend_rows(0, qkv, None, None, _C.ROPE_NONE, out, [4, 4, 4])


def test_symbol_bound():
    lib = _C.load()
    assert "duo_prefill_ragged" in _C.SYMBOLS and hasattr(lib, "duo_prefill_ragged")
