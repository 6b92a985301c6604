"""Host-side logic of ragged INT4 batches (duo_decode_ragged_int4 / DuoRaggedINT4KVCache): the key partition every CTA
of the keys-as-M INT4 decode kernel derives from the row lengths, the workspace size, the C-ABI rejections and the
cache's argument checks.  No GPU needed."""
import ctypes as C

import pytest
import torch

from duo_attention_b200.kv_cache import (INT4_RAGGED_POLICY, DuoRaggedINT4KVCache, DuoRaggedKVCache,
                                         ragged_partition)

SMS = 132


def dec8_partition(nkeys, batch, n_full, n_stream, sm_count=SMS):
    """plan_splits (duo_common.cuh) as launch_i4_dec8 (attn_int4.cu) calls it: 4 CTAs per SM, 128-key tiles, >= 1024
    keys per split, nkeys = full_len + q_len, every row at the same length."""
    budget, stream_ctas = 4 * sm_count, batch * n_stream
    want = max(1, (budget - stream_ctas if budget - stream_ctas > 0 else 1) // (batch * n_full))
    splits = min(want, max(1, -(-nkeys // 1024)), 512)
    kps = max(128, -(-(-(-nkeys // splits)) // 128) * 128)
    return kps, max(1, -(-nkeys // kps))


def check_cover(nkeys, n_full, n_stream):
    part = ragged_partition(nkeys, n_full, n_stream, SMS, **INT4_RAGGED_POLICY)
    kps, splits = part["keys_per_split"], part["splits"]
    assert kps % 128 == 0 and kps >= 128
    assert sum(splits) <= part["slots"], (sum(splits), part["slots"])
    for n, s in zip(nkeys, splits):
        assert 1 <= s <= 512
        ranges = [(i * kps, max(i * kps, min(n, (i + 1) * kps))) for i in range(s)]
        assert ranges[0][0] == 0 and ranges[-1][1] == n  # every key exactly once, in order, no empty split
        assert all(ranges[i][1] == ranges[i + 1][0] for i in range(s - 1))
        assert all(b > a for a, b in ranges)
    return part


@pytest.mark.parametrize("n_full,n_stream", [(1, 7), (4, 4), (8, 0), (2, 6), (3, 5)])
@pytest.mark.parametrize("seed", range(6))
def test_int4_partition_covers_every_key_once(n_full, n_stream, seed):
    g = torch.Generator().manual_seed(100 + seed)
    for B in (1, 2, 7, 8, 33, 64):
        for q_len in (1, 2):
            lengths = torch.randint(0, 1 << (8 + 2 * seed), (B,), generator=g).tolist()
            check_cover([n + q_len for n in lengths], n_full, n_stream)
            check_cover([q_len] * B, n_full, n_stream)
            check_cover([(1 << 20) + q_len] * B, n_full, n_stream)


@pytest.mark.parametrize("B", [1, 2, 4, 8, 16, 64])
@pytest.mark.parametrize("n_full,n_stream", [(1, 7), (4, 4), (8, 0), (1, 0)])
def test_int4_equal_lengths_match_dec8_partition(B, n_full, n_stream):
    for L in (0, 1, 1023, 1024, 1025, 4097, 131072, 1 << 20):
        for q_len in (1, 2):
            part = ragged_partition([L + q_len] * B, n_full, n_stream, SMS, **INT4_RAGGED_POLICY)
            kps, splits = dec8_partition(L + q_len, B, n_full, n_stream)
            assert part["keys_per_split"] == kps, (L, q_len, B)
            assert part["splits"] == [splits] * B


def test_default_policy_is_unchanged():
    """The keyword parameters default to the 16-bit kernel's policy."""
    lengths = [524288] + [32768] * 7
    assert ragged_partition(lengths, 4, 4) == ragged_partition(lengths, 4, 4, SMS, tile=64, min_keys=256, ctas_per_sm=2)


def test_int4_workspace_bytes_finite_for_every_geometry():
    from duo_attention_b200 import _C

    lib = _C.load()
    assert "duo_ragged_int4_workspace_bytes" in _C.SYMBOLS and "duo_decode_ragged_int4" in _C.SYMBOLS
    for B in range(1, 65):
        for n_kv in range(1, 9):
            ws = lib.duo_ragged_int4_workspace_bytes(B, n_kv)
            assert 0 < ws < 1 << 32, (B, n_kv, ws)
    assert lib.duo_ragged_int4_workspace_bytes(0, 8) == 0 and lib.duo_ragged_int4_workspace_bytes(65, 8) == 0
    assert lib.duo_ragged_int4_workspace_bytes(8, 0) == 0


def _layer(lib, _C, batch, kv_format, group=4, full_cap=0):
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    # no streaming heads and INT4 (or no capacity): no tensor maps to encode, so creation stays on the host
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = full_cap, batch, 1, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, 8, _C.DT_FP16, kv_format
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK
    return h.value


def test_decode_ragged_int4_rejections_before_cuda():
    from duo_attention_b200 import _C

    lib = _C.load()
    f = lib.duo_decode_ragged_int4

    def args(h, ml=0, q=1, qkv=0x1000, stride=640 * 2, out=0x2000, rope=_C.ROPE_NONE, cos=None):
        return (h, 0x1000, ml, qkv, stride, cos, cos, rope, out, q, 0.1, None, 0, None)

    h = _layer(lib, _C, 8, _C.KV_SAME)
    assert f(*args(h)) == _C.DUO_EINVAL and "INT4 caches only" in _C.last_error()
    lib.duo_layer_destroy(h)
    h = _layer(lib, _C, 65, _C.KV_INT4)
    assert f(*args(h)) == _C.DUO_EINVAL and "batch 65" in _C.last_error()
    lib.duo_layer_destroy(h)
    h = _layer(lib, _C, 8, _C.KV_INT4)
    assert f(*args(h, q=3)) == _C.DUO_EINVAL and "<= 8" in _C.last_error()  # group 4 x 3 rows > 8
    assert f(*args(h, q=0)) == _C.DUO_EINVAL
    assert f(*args(h, ml=-1)) == _C.DUO_EINVAL
    assert f(None, *args(h)[1:]) == _C.DUO_EINVAL
    assert f(*((h, None) + args(h)[2:])) == _C.DUO_EINVAL  # no row_state
    assert f(*args(h, out=None)) == _C.DUO_EINVAL and "null buffer" in _C.last_error()
    assert f(*args(h, qkv=0x1008)) == _C.DUO_EINVAL and "16-byte" in _C.last_error()
    assert f(*args(h, stride=644)) == _C.DUO_EINVAL and "16-byte" in _C.last_error()
    assert f(*args(h, rope=_C.ROPE_HF)) == _C.DUO_EINVAL  # RoPE without tables
    assert f(*args(h, rope=7, cos=0x3000)) == _C.DUO_EINVAL and "rope_mode" in _C.last_error()
    assert f(*args(h)) == _C.DUO_EOVERFLOW
    assert "Trying to put 1 KVs into a cache with max size 0, current size: 0." in _C.last_error()
    lib.duo_layer_destroy(h)
    h = _layer(lib, _C, 8, _C.KV_INT4, group=1, full_cap=64)
    assert f(*args(h, q=9)) == _C.DUO_EINVAL  # MHA: 9 rows > 8
    assert f(*args(h, ml=60, q=8)) == _C.DUO_EOVERFLOW
    assert "Trying to put 8 KVs into a cache with max size 64, current size: 60." in _C.last_error()
    lib.duo_layer_destroy(h)


def test_decode_ragged_points_int4_layers_to_the_new_entry_point():
    from duo_attention_b200 import _C

    lib = _C.load()
    h = _layer(lib, _C, 8, _C.KV_INT4)
    rc = lib.duo_decode_ragged(h, 0x1000, 0, 0x1000, 640 * 2, None, None, _C.ROPE_NONE, 0x2000, 1, 0.1, None, 0, None)
    assert rc == _C.DUO_EINVAL and "INT4" in _C.last_error() and "duo_decode_ragged_int4" in _C.last_error()
    lib.duo_layer_destroy(h)


def test_int4_cache_rejects_cpu_and_oversize_batch():
    geo = (2, 8, 2, 128, [1, 1])
    with pytest.raises(ValueError, match="batch_size 65"):
        DuoRaggedINT4KVCache.from_geometry(*geo, 65, 256, 4, 8, torch.float16, "cpu")
    with pytest.raises(RuntimeError, match="GPU memory"):
        DuoRaggedINT4KVCache.from_geometry(*geo, 4, 256, 4, 8, torch.float16, "cpu")
    with pytest.raises(ValueError, match="not supported yet"):
        DuoRaggedINT4KVCache.from_geometry(*geo, 4, 256, 4, 8, torch.float16, "cpu", kv_format="same")
    with pytest.raises(ValueError, match="DuoRaggedINT4KVCache"):  # the 16-bit class points to the INT4 one
        DuoRaggedKVCache.from_geometry(*geo, 4, 256, 4, 8, torch.float16, "cpu", kv_format="int4")
    assert DuoRaggedINT4KVCache.max_rows == 8 and DuoRaggedKVCache.max_rows == 16
