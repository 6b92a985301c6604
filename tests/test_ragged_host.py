"""Host-side logic of ragged batches (duo_decode_ragged / DuoRaggedKVCache): the key partition every CTA derives from
the row lengths, per-row ring arithmetic, the C-ABI surface and argument rejections.  No GPU needed."""
import ctypes as C

import pytest
import torch

from duo_attention_b200.kv_cache import (DuoRaggedKVCache, ragged_keys_per_split, ragged_partition, ragged_want,
                                         ring_advance, ring_evict, ring_live_positions)

SMS = 132


def fused_partition(L, batch, n_full, n_stream, sm_count=SMS):
    """plan_splits (duo_common.cuh) as launch_variant (attn_mma.cu) calls it for a decode-sized chunk at batch
    ``batch``, every row at L."""
    budget, base, stream_ctas = 2 * sm_count, batch * n_full, batch * n_stream
    want = max(1, (budget - stream_ctas if budget - stream_ctas > 0 else 1) // base)
    splits = min(want, max(1, -(-L // 256)))
    splits = min(splits, 512)
    kps = -(-L // splits)
    kps = max(64, -(-kps // 64) * 64)
    return kps, max(1, -(-L // kps))


def check_cover(lengths, n_full, n_stream, sm_count=SMS):
    part = ragged_partition(lengths, n_full, n_stream, sm_count)
    kps, splits = part["keys_per_split"], part["splits"]
    assert kps % 64 == 0 and kps >= 64
    assert sum(splits) <= part["slots"], (sum(splits), part["slots"])  # the CTAs used never exceed the grid
    for n, s in zip(lengths, splits):
        assert 1 <= s <= 512
        covered = []
        for i in range(s):  # each split's key range, as the kernel computes it
            a0, a1 = i * kps, min(n, (i + 1) * kps)
            covered.append((a0, max(a0, a1)))
        assert covered[0][0] == 0 and covered[-1][1] == n  # every key exactly once, in order
        assert all(covered[i][1] == covered[i + 1][0] for i in range(s - 1))
        assert all(b > a for a, b in covered) or n == 0
    return part


@pytest.mark.parametrize("n_full,n_stream", [(1, 7), (4, 4), (8, 0), (2, 6), (8, 8)])
@pytest.mark.parametrize("seed", range(6))
def test_partition_covers_every_key_once(n_full, n_stream, seed):
    g = torch.Generator().manual_seed(seed)
    for B in (1, 2, 7, 8, 33, 64):
        lengths = torch.randint(0, 1 << (8 + 2 * seed), (B,), generator=g).tolist()
        check_cover(lengths, n_full, n_stream)
        check_cover([0] * B, n_full, n_stream)
        check_cover([1 << 20] * B, n_full, n_stream)


@pytest.mark.parametrize("B", [1, 2, 4, 8, 16, 64])
@pytest.mark.parametrize("n_full,n_stream", [(1, 7), (4, 4), (8, 0), (1, 0)])
def test_equal_lengths_match_fused_partition(B, n_full, n_stream):
    for L in (0, 1, 63, 64, 255, 256, 257, 4097, 20000, 131072, 524288, 1 << 20):
        part = ragged_partition([L] * B, n_full, n_stream)
        kps, splits = fused_partition(L, B, n_full, n_stream)
        assert part["keys_per_split"] == kps, (L, B)
        assert part["splits"] == [splits] * B


def test_skewed_batches_stay_balanced():
    # one 512K row next to seven 32K rows (Llama-3-8B at sparsity 0.5: 4 retrieval + 4 streaming kv heads)
    lengths = [524288] + [32768] * 7
    part = check_cover(lengths, 4, 4)
    uniform = check_cover([sum(lengths) // 8] * 8, 4, 4)
    assert part["splits"][0] >= 32  # the long row is spread over most of the grid, not 1/8 of it
    # the slowest CTA streams at most ~one split of keys: within 5% of the equal-length batch's
    assert part["keys_per_split"] <= 1.05 * uniform["keys_per_split"]
    assert sum(part["splits"]) <= part["slots"] and sum(part["splits"]) >= 0.9 * sum(uniform["splits"])
    # 1M tokens next to 63 one-token rows
    lengths = [1 << 20] + [1] * 63
    part = check_cover(lengths, 4, 4)
    assert part["splits"][0] >= 60 and part["splits"][1:] == [1] * 63
    assert part["keys_per_split"] * part["splits"][0] <= (1 << 20) + part["keys_per_split"]


def test_keys_per_split_caps_splits_per_row():
    for B, want in ((64, 512), (2, 512), (64, 1)):
        kps = ragged_keys_per_split((1 << 22) + B, 1 << 22, B, want)
        assert -(-(1 << 22) // kps) <= 512
    assert ragged_want(8, 4, 4) == 7 and ragged_want(64, 4, 4) == 1 and ragged_want(1, 1, 0) == 264


def test_per_row_ring_arithmetic_under_evict_and_clear():
    sink, recent = 4, 6
    rows = [(0, sink), (0, sink), (0, sink)]
    steps = [(3, 0), (1, 2), (20, 1), (1, 0)]
    hist = [[], [], []]
    for b, (n, ev) in enumerate(steps[:3]):
        t, lo = rows[b]
        t, lo = ring_advance(t, lo, n * (b + 1), sink, recent)
        t, lo = ring_evict(t, lo, ev, sink)
        rows[b] = (t, lo)
    for b, (t, lo) in enumerate(rows):  # rows stay independent: the live set is that of a lone sequence
        live = ring_live_positions(t, lo, sink)
        assert len(live) <= sink + recent and live == sorted(set(live))
        hist[b] = live
    assert hist[0] == [0, 1, 2]
    t, lo = rows[2]
    assert hist[2] == list(range(4)) + list(range(max(lo, sink), t)) and t == 59
    rows[1] = (0, sink)  # clear() of one row: the others keep their state
    assert ring_live_positions(*rows[1], sink) == [] and hist[2] == ring_live_positions(*rows[2], sink)


def test_symbols_exported_and_bound():
    from duo_attention_b200 import _C

    lib = _C.load()
    for name in ("duo_decode_ragged", "duo_ragged_workspace_bytes", "duo_ragged_state_advance"):
        assert name in _C.SYMBOLS and hasattr(lib, name)
    assert lib.duo_ragged_workspace_bytes(0, 8) == 0 and lib.duo_ragged_workspace_bytes(65, 8) == 0
    ws = lib.duo_ragged_workspace_bytes(8, 8)
    assert ws > 0 and lib.duo_ragged_workspace_bytes(64, 8) >= lib.duo_ragged_workspace_bytes(64, 1)


def _layer(lib, _C, batch, kv_format):
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    # no retrieval capacity and no streaming heads: no tensor maps to encode, so creation stays on the host
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, 1, 0, 4, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, 8, _C.DT_BF16, kv_format
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK
    return h.value


def test_decode_ragged_rejections_before_cuda():
    from duo_attention_b200 import _C

    lib = _C.load()
    args = lambda h, ml=0, q=1: (h, 0x1000, ml, 0x1000, 640 * 2, None, None, _C.ROPE_NONE, 0x2000, q, 0.1, None, 0, None)
    h = _layer(lib, _C, 65, _C.KV_SAME)
    assert lib.duo_decode_ragged(*args(h)) == _C.DUO_EINVAL and "batch 65" in _C.last_error()
    lib.duo_layer_destroy(h)
    h = _layer(lib, _C, 8, _C.KV_INT4)
    assert lib.duo_decode_ragged(*args(h)) == _C.DUO_EINVAL and "INT4" in _C.last_error()
    lib.duo_layer_destroy(h)
    h = _layer(lib, _C, 8, _C.KV_SAME)
    assert lib.duo_decode_ragged(*args(h, q=5)) == _C.DUO_EINVAL  # group 4 x 5 rows > 16
    assert lib.duo_decode_ragged(*args(h)) == _C.DUO_EOVERFLOW
    assert "Trying to put 1 KVs into a cache with max size 0, current size: 0." in _C.last_error()
    assert lib.duo_decode_ragged(None, *args(h)[1:]) == _C.DUO_EINVAL
    lib.duo_layer_destroy(h)
    assert lib.duo_ragged_state_advance(None, 8, 1, 4, 8, None) == _C.DUO_EINVAL
    assert lib.duo_ragged_state_advance(0x1000, 65, 1, 4, 8, None) == _C.DUO_EINVAL


def test_cache_rejects_int4_and_oversize_batch_before_cuda():
    geo = (2, 8, 2, 128, [1, 1])
    with pytest.raises(ValueError, match="not supported yet"):
        DuoRaggedKVCache.from_geometry(*geo, 4, 256, 4, 8, torch.bfloat16, "cpu", kv_format="int4")
    with pytest.raises(ValueError, match="batch_size 65"):
        DuoRaggedKVCache.from_geometry(*geo, 65, 256, 4, 8, torch.bfloat16, "cpu")
    with pytest.raises(RuntimeError, match="GPU memory"):  # a CPU device is refused by the base class
        DuoRaggedKVCache.from_geometry(*geo, 4, 256, 4, 8, torch.bfloat16, "cpu")
