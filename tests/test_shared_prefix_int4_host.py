"""Shared prefixes on the INT4 cache, host side: the C entry points take INT4 layers and refuse bad arguments before any
CUDA call (INT4 layer handles are created without one), the workspace bound covers the INT4 cascade, and
share_prefix serves the formats a cache class declares."""
import ctypes as C
import types

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache, DuoRaggedKVCache


def _layer(lib, kv_format=_C.KV_INT4, pool_tokens=0, group=4, n_full=2, n_stream=6, full_cap=1024, batch=1):
    d = _C.LayerDesc()
    for k in ("full_k", "full_v", "ring_k", "ring_v", "full_k_scale", "full_k_zero", "full_v_scale", "full_v_zero",
              "ring_k_scale", "ring_k_zero", "ring_v_scale", "ring_v_zero"):
        if hasattr(d, k):
            setattr(d, k, 0x10000)
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = full_cap, batch, n_full, n_stream, group, 128
    d.sink, d.recent, d.stage_cap = 16, 48, 64
    d.dtype, d.kv_format = _C.DT_BF16, kv_format
    h = C.c_void_p()
    if pool_tokens:
        _C.check(lib.duo_layer_create_pooled(C.byref(d), pool_tokens, C.byref(h)))
    else:
        _C.check(lib.duo_layer_create(C.byref(d), C.byref(h)))
    return h.value


def test_attention_shared_takes_int4_and_refuses_before_cuda():
    lib = _C.load()
    own, pre = _layer(lib, full_cap=512), _layer(lib, full_cap=1024)
    try:
        st = _C.CacheState(600, 600, 16, None)
        call = lambda layer, prefix, P, q_len: lib.duo_attention_shared(  # noqa: E731
            layer, prefix, P, C.byref(st), 0x1000, 1536, 0x2000, q_len, 0.1, None, 0, None)
        # decode-sized chunks of an INT4 sharer (group 4 x 2 = 8 rows) go through the batched step
        assert call(own, pre, 512, 2) == _C.DUO_EINVAL and "group * q_len > 8" in _C.last_error()
        # a bad prefix length
        assert call(own, pre, 500, 3) == _C.DUO_EINVAL and "multiple of 128" in _C.last_error()
        # the own region holds 600 - 512 + q_len rows: 512 rows of capacity take 424 more, not 425
        assert call(own, pre, 512, 425) == _C.DUO_EOVERFLOW
        # the two handles must be of one KV format
        same = _layer(lib, kv_format=_C.KV_SAME, n_full=0, n_stream=0)  # no tensor maps: no CUDA call
        try:
            assert call(own, same, 512, 3) == _C.DUO_EINVAL and "one KV format" in _C.last_error()
        finally:
            lib.duo_layer_destroy(same)
    finally:
        lib.duo_layer_destroy(own)
        lib.duo_layer_destroy(pre)


def test_decode_ragged_shared_takes_int4_and_refuses_before_cuda():
    lib = _C.load()
    pooled, flat = _layer(lib, pool_tokens=4096, batch=4), _layer(lib, batch=4)
    try:
        call = lambda layer, q_len, min_room: lib.duo_decode_ragged_shared(  # noqa: E731
            layer, 0x1000, 0x1000, 0x1000, min_room, 0x1000, 1536, None, None, _C.ROPE_NONE, 0x2000, q_len, 0.1,
            None, 0, None)
        assert call(pooled, 3, 100) == _C.DUO_EINVAL and "group * q_len <= 8" in _C.last_error()
        assert call(flat, 1, 100) == _C.DUO_EINVAL and "no retrieval pool" in _C.last_error()
        assert call(pooled, 2, 1) == _C.DUO_EOVERFLOW
    finally:
        lib.duo_layer_destroy(pooled)
        lib.duo_layer_destroy(flat)


def test_shared_workspace_bound_covers_the_int4_cascade():
    lib = _C.load()
    for B in (1, 2, 17, 64):
        for n_kv in (1, 8):
            ws = lib.duo_ragged_shared_workspace_bytes(B, n_kv)
            assert 0 < ws < 1 << 34
            # at least the INT4 prefix partials: batch x 8 packed rows x n_kv heads of 129 fp32
            assert ws > B * _C.DECODE_MAX_Q_INT4 * n_kv * 129 * 4


def test_share_prefix_serves_the_declared_formats():
    assert DuoRaggedKVCache._share_formats == ("same",) and DuoRaggedINT4KVCache._share_formats == ("int4",)
    assert DuoRaggedINT4KVCache.share_prefix is DuoRaggedKVCache.share_prefix
    # a pooled INT4 cache gets past the format check (and on to the argument checks); a uniform one does not
    rows = [types.SimpleNamespace(kv_seq_len_list=[n], total_list=[n], kv_seq_len=n) for n in (300, 0)]
    stub = types.SimpleNamespace(pooled=True, kv_format="int4", _share_formats=("int4",), rows=rows,
                                 _share=[None, None], batch_size=2, graph_attached=False, graph_shared=False)
    with pytest.raises(ValueError, match="two different rows"):
        DuoRaggedKVCache.share_prefix(stub, 0, 0, 100)
    stub.pooled = False
    with pytest.raises(ValueError, match="needs a 16-bit cache with per-row capacities"):
        DuoRaggedKVCache.share_prefix(stub, 0, 1, 100)
