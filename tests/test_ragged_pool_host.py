"""Ragged batches with per-row capacities, host side (no GPU): the pool planner, the C-ABI symbols and every argument
rejection of duo_layer_create_pooled / duo_decode_ragged_pooled that happens before any CUDA call."""
import ctypes as C
import os
import re
import types

import pytest
import torch

from duo_attention_b200.kv_cache import (POOL_ALIGN, DuoRaggedINT4KVCache, DuoRaggedKVCache, pool_first_fit,
                                         pool_layout)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _disjoint_aligned_inside(lay):
    regs = sorted(zip(lay["first"], lay["cap"]))
    for (f, c), (f2, _) in zip(regs, regs[1:]):
        assert f + c <= f2
    for f, c in regs:
        assert f % POOL_ALIGN == 0 and c % POOL_ALIGN == 0 and 0 <= f and f + c <= lay["pool_tokens"]


@pytest.mark.parametrize("caps", [[1], [524288 + 64] + [32768 + 64] * 7, [1, 127, 128, 129, 1000, 1048576], [300] * 5])
def test_pool_layout_regions_disjoint_aligned_inside(caps):
    lay = pool_layout(caps)
    _disjoint_aligned_inside(lay)
    assert all(c >= want for c, want in zip(lay["cap"], caps))
    assert lay["pool_tokens"] == sum(-(-c // 128) * 128 for c in caps)


def test_equal_capacities_give_the_uniform_layout():
    """first_b = b * cap: the pool is [B][n_full][cap][128] byte for byte (row b, head h, key j at b*nf*cap + h*cap + j)."""
    for cap in (128, 4096, 70016):
        lay = pool_layout([cap] * 6)
        assert lay["first"] == [b * cap for b in range(6)] and lay["cap"] == [cap] * 6
        assert lay["pool_tokens"] == 6 * cap
        nf = 3
        pool_row = lambda b, h, j: lay["first"][b] * nf + h * lay["cap"][b] + j
        assert all(pool_row(b, h, j) == (b * nf + h) * cap + j for b in (0, 5) for h in range(nf) for j in (0, cap - 1))


def test_pool_size_headroom_and_rejections():
    assert pool_layout([100, 200], pool_size=1000)["pool_tokens"] == 1024
    assert pool_layout([100, 200], pool_size=384)["pool_tokens"] == 384
    with pytest.raises(ValueError, match="smaller than"):
        pool_layout([100, 200], pool_size=256)
    with pytest.raises(ValueError, match=">= 1"):
        pool_layout([100, 0])


def test_first_fit_reuses_freed_space_and_raises_when_full():
    lay = pool_layout([256, 512, 128], pool_size=1024 + 256)   # regions [0,256) [256,768) [768,896), free [896,1280)
    first, cap, P = lay["first"], lay["cap"], lay["pool_tokens"]
    assert pool_first_fit(first, cap, 1, 512, P) == 256          # its own region counts as free
    assert pool_first_fit(first, cap, 1, 384, P) == 256          # ... also for a smaller region
    assert pool_first_fit(first, cap, 2, 384, P) == 768          # own region + headroom
    assert pool_first_fit(first, cap, 0, 300, P) == 896          # first fit: the hole at 0 is 256 tokens, too small
    assert pool_first_fit(first, cap, 0, 1, P) == 0
    with pytest.raises(ValueError, match="no free range of 512 tokens for row 0"):
        pool_first_fit(first, cap, 0, 500, P)
    # moving row 0 into the headroom frees [0,256) for a later row
    first[0], cap[0] = 896, 384
    _disjoint_aligned_inside({"first": first, "cap": cap, "pool_tokens": P})
    assert pool_first_fit(first, cap, 2, 256, P) == 0


def test_resize_row_refuses_a_row_with_tokens_and_uniform_caches():
    row = types.SimpleNamespace(kv_seq_len_list=[0, 5], total_list=[0, 5], kv_seq_len=5)
    stub = types.SimpleNamespace(pooled=True, rows=[row])
    with pytest.raises(ValueError, match="row 0 is not empty"):
        DuoRaggedKVCache.resize_row(stub, 0, 256)
    row.kv_seq_len_list, row.total_list = [0, 0], [0, 3]  # streaming tokens only: still not empty
    with pytest.raises(ValueError, match="not empty"):
        DuoRaggedKVCache.resize_row(stub, 0, 256)
    with pytest.raises(ValueError, match="per-row capacities"):
        DuoRaggedKVCache.resize_row(types.SimpleNamespace(pooled=False), 0, 256)


def test_cache_argument_rejections_before_cuda():
    geo = (2, 8, 2, 128, [1, 1])
    with pytest.raises(ValueError, match="3 row capacities for batch_size 4"):
        DuoRaggedKVCache.from_geometry(*geo, 4, [256, 256, 256], 4, 8, torch.bfloat16, "cpu")
    with pytest.raises(ValueError, match="pool_size needs per-row capacities"):
        DuoRaggedINT4KVCache.from_geometry(*geo, 4, 256, 4, 8, torch.float16, "cpu", pool_size=4096)
    with pytest.raises(ValueError, match="smaller than"):
        DuoRaggedKVCache.from_geometry(*geo, 2, [256, 256], 4, 8, torch.bfloat16, "cpu", pool_size=128)
    with pytest.raises(RuntimeError, match="GPU memory"):  # valid arguments: the base class refuses a CPU device
        DuoRaggedKVCache.from_geometry(*geo, 2, [256, 1000], 4, 8, torch.bfloat16, "cpu", pool_size=4096)


def test_symbols_in_header_binding_and_exports():
    from duo_attention_b200 import _C

    lib = _C.load()
    header = open(os.path.join(ROOT, "include", "duo_b200.h")).read()
    for name in ("duo_layer_create_pooled", "duo_decode_ragged_pooled"):
        assert name in _C.SYMBOLS and hasattr(lib, name)
        assert re.search(r"DUO_API int " + name + r"\(", header)


def _desc(_C, batch=4, n_full=1, n_stream=0, kv_format=None):
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, n_full, n_stream, 4, 128
    d.sink, d.recent, d.stage_cap, d.dtype = 4, 8, 8, _C.DT_BF16
    d.kv_format = _C.KV_SAME if kv_format is None else kv_format
    return d


def _create(lib, _C, d, pool_tokens):
    h = C.c_void_p()
    rc = lib.duo_layer_create_pooled(C.byref(d), pool_tokens, C.byref(h))
    return rc, h.value


def test_layer_create_pooled_rejections_before_cuda():
    from duo_attention_b200 import _C

    lib = _C.load()
    for bad in (0, -128, 100, 129):
        rc, h = _create(lib, _C, _desc(_C), bad)
        assert rc == _C.DUO_EINVAL and h is None and "not a positive multiple of 128" in _C.last_error()
    rc, h = _create(lib, _C, _desc(_C, n_full=8), (1 << 28))  # 2^31 pool rows: past the int32 TMA coordinate
    assert rc == _C.DUO_EINVAL and "32-bit TMA row coordinate" in _C.last_error()
    assert lib.duo_layer_create_pooled(None, 128, C.byref(C.c_void_p())) == _C.DUO_EINVAL


def _pooled_layer(lib, _C, batch=4, kv_format=None):
    # no tensor maps to encode (INT4 layers have none; the 16-bit layer has no heads that need one), so creation
    # stays on the host
    d = _desc(_C, batch=batch, n_full=1 if kv_format == _C.KV_INT4 else 0, n_stream=0, kv_format=kv_format)
    rc, h = _create(lib, _C, d, 1024)
    assert rc == _C.DUO_OK, _C.last_error()
    return h


def test_decode_ragged_pooled_rejections_before_cuda():
    from duo_attention_b200 import _C

    lib = _C.load()
    args = lambda h, room=10, q=1, rg=0x3000, qkv=0x1000, stride=640 * 2, out=0x2000: (
        h, 0x1000, rg, room, qkv, stride, None, None, _C.ROPE_NONE, out, q, 0.1, None, 0, None)
    fn = lib.duo_decode_ragged_pooled
    int4 = _pooled_layer(lib, _C, kv_format=_C.KV_INT4)
    # null / misaligned buffers
    assert fn(None, *args(int4)[1:]) == _C.DUO_EINVAL and "null argument" in _C.last_error()
    assert fn(*args(int4, rg=None)) == _C.DUO_EINVAL and "null argument" in _C.last_error()
    assert fn(*args(int4, out=None)) == _C.DUO_EINVAL and "null buffer" in _C.last_error()
    assert fn(*args(int4, qkv=0x1008)) == _C.DUO_EINVAL and "16-byte aligned" in _C.last_error()
    assert fn(*args(int4, stride=644)) == _C.DUO_EINVAL and "16-byte aligned" in _C.last_error()
    # too many packed rows: 8 on INT4 KV (group 4 x q_len 3 = 12), 16 on 16-bit KV (group 4 x 5 = 20)
    assert fn(*args(int4, q=3)) == _C.DUO_EINVAL and "group * q_len <= 8" in _C.last_error()
    # overflow: q_len > min_b (cap_b - full_len_b)
    assert fn(*args(int4, room=1, q=2)) == _C.DUO_EOVERFLOW
    assert "Trying to put 2 KVs into a cache row with room for 1 more" in _C.last_error()
    # the other ragged entry points refuse a pooled handle and name the new one
    for name in ("duo_decode_ragged", "duo_decode_ragged_int4"):
        rc = getattr(lib, name)(int4, 0x1000, 0, 0x1000, 640 * 2, None, None, _C.ROPE_NONE, 0x2000, 1, 0.1, None, 0, None)
        assert rc == _C.DUO_EINVAL and "duo_decode_ragged_pooled" in _C.last_error()
    # ... and so do the batch-1 entry points (the rows have handles of their own)
    st = _C.CacheState(0, 0, 4, None)
    assert lib.duo_attention(int4, C.byref(st), 0x1000, 640, 0x2000, 1, 0.1, None, 0, None) == _C.DUO_EINVAL
    assert "duo_decode_ragged_pooled" in _C.last_error()
    lib.duo_layer_destroy(int4)
    same = _pooled_layer(lib, _C)
    assert fn(*args(same, q=5)) == _C.DUO_EINVAL and "group * q_len <= 16" in _C.last_error()
    lib.duo_layer_destroy(same)
    big = _pooled_layer(lib, _C, batch=65)
    assert fn(*args(big)) == _C.DUO_EINVAL and "batch 65" in _C.last_error()
    lib.duo_layer_destroy(big)
    # a handle from duo_layer_create is not pooled
    d = _desc(_C)
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK
    assert fn(*args(h.value)) == _C.DUO_EINVAL and "duo_layer_create_pooled" in _C.last_error()
    lib.duo_layer_destroy(h.value)
