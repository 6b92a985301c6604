"""Shared prefixes of a pooled ragged cache, host side: the alignment of the shared prefix, the row_share table, the
fork plan (capacity accounting, forking from a sharer) and the refusals that happen before any device work."""
import types

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import (POOL_ALIGN, DuoRaggedINT4KVCache, DuoRaggedKVCache, pool_first_fit,
                                         share_fork_plan, share_table, shared_prefix_len)


def test_prefix_is_whole_128_key_blocks():
    assert POOL_ALIGN == 128
    for n, P in ((0, 0), (1, 0), (127, 0), (128, 128), (129, 128), (255, 128), (256, 256), (524288 + 77, 524288)):
        assert shared_prefix_len(n) == P
        assert P % 64 == 0  # no 64-key tile straddles the end of the prefix


def test_fork_plan_capacity_and_fork_of_a_sharer():
    p = share_fork_plan(300, None, 0, 100)  # 256 shared, the 44-token tail copied from region row 256 of the donor
    assert p == {"donor": 0, "P": 256, "copy_from": 256, "n_copy": 44}
    p = share_fork_plan(100, None, 2, 100)  # below 128: nothing shared, everything copied
    assert p == {"donor": 2, "P": 0, "copy_from": 0, "n_copy": 100}
    # a sharer of row 0 (P = 256) that has grown to 400 tokens: the fork shares the same donor prefix and copies the
    # sharer's own 144 rows, which start its region
    p = share_fork_plan(400, (0, 256), 1, 144)
    assert p == {"donor": 0, "P": 256, "copy_from": 0, "n_copy": 144}
    with pytest.raises(ValueError, match="144 tokens past its shared prefix of 256"):
        share_fork_plan(400, (0, 256), 1, 143)
    with pytest.raises(ValueError, match="capacity 40"):
        share_fork_plan(300, None, 0, 40)


def test_share_table_groups():
    assert share_table([None, None]) == [[-1, 0], [-1, 0]]
    # rows 1, 2 share 256 keys of row 0, row 4 shares 512 keys of row 0, row 5 shares 128 keys of row 3
    t = share_table([None, (0, 256), (0, 256), None, (0, 512), (3, 128)])
    assert t == [[0, 512], [0, 256], [0, 256], [3, 128], [0, 512], [3, 128]]


def test_own_region_is_first_fit_and_capacity_reports_the_prefix():
    # the new row's region holds only its own keys: first fit of `capacity`, not of P + capacity
    first = pool_first_fit([0, 0, 1024], [1024, 0, 256], 1, 100, 4096)
    assert first == 1280
    row = types.SimpleNamespace()
    stub = types.SimpleNamespace(pooled=True, _row_caps=[1024, 100], _share=[None, (0, 896)], batch_size=2, rows=[row])
    assert DuoRaggedKVCache.row_capacities.fget(stub) == [1024, 996]
    assert DuoRaggedKVCache.row_prefix.fget(stub) == [None, (0, 896)]
    assert DuoRaggedKVCache.sharing.fget(stub)


def _stub(lengths, shares):
    rows = [types.SimpleNamespace(kv_seq_len_list=[n, n], total_list=[n, n], kv_seq_len=n) for n in lengths]
    stub = types.SimpleNamespace(pooled=True, kv_format="same", rows=rows, _share=list(shares), batch_size=len(lengths),
                                 graph_attached=False, graph_shared=False)
    for name in ("_donor_floor", "_check_not_donor", "_check_evict"):
        setattr(stub, name, getattr(DuoRaggedKVCache, name).__get__(stub))
    return stub


def test_refusals_protect_the_donor_and_the_sharers_prefix():
    s = _stub([300, 300, 0], [None, (0, 256), None])
    assert s._donor_floor(0) == 256 and s._donor_floor(1) == 0
    s._check_evict(0, 44)  # down to exactly P
    with pytest.raises(ValueError, match="below the 256 keys other rows share"):
        s._check_evict(0, 45)
    s._check_evict(1, 44)
    with pytest.raises(ValueError, match="into the 256 keys it shares with row 0"):
        s._check_evict(1, 45)
    with pytest.raises(ValueError, match=r"rows \[1\] share the first 256 keys of row 0: clear of row 0"):
        s._check_not_donor(0, "clear")
    s._check_not_donor(1, "clear")
    s._check_not_donor(2, "clear")


def test_share_prefix_refusals_before_any_change():
    s = _stub([300, 0, 5], [None, None, None])
    sp = DuoRaggedKVCache.share_prefix
    with pytest.raises(ValueError, match="not empty"):
        sp(s, 0, 2, 100)
    s.rows[2].kv_seq_len_list, s.rows[2].total_list = [0, 0], [0, 0]
    with pytest.raises(ValueError, match="row 1 is empty"):
        sp(s, 1, 2, 100)
    with pytest.raises(ValueError, match="two different rows"):
        sp(s, 0, 0, 100)
    with pytest.raises(ValueError, match="two different rows"):
        sp(s, 0, 3, 100)
    with pytest.raises(ValueError, match="capacity 0"):
        sp(s, 0, 1, 0)
    s.rows[0].kv_seq_len_list = [300, 299]
    with pytest.raises(ValueError, match="different lengths"):
        sp(s, 0, 1, 100)
    s.rows[0].kv_seq_len_list = [300, 300]
    s.graph_attached = True
    with pytest.raises(ValueError, match="build a new DuoDecodeGraph"):
        sp(s, 0, 1, 100)
    assert s._share == [None, None, None]  # nothing changed


def test_share_prefix_refuses_int4_and_uniform_caches():
    for kw in (dict(pooled=False, kv_format="same"), dict(pooled=True, kv_format="int4"),
               dict(pooled=False, kv_format="int4")):
        with pytest.raises(ValueError, match="needs a 16-bit cache with per-row capacities"):
            DuoRaggedKVCache.share_prefix(types.SimpleNamespace(**kw), 0, 1, 100)
    assert DuoRaggedINT4KVCache.share_prefix is DuoRaggedKVCache.share_prefix  # the INT4 class refuses through it


def test_abi_entry_refuses_null_arguments_before_cuda():
    lib = _C.load()
    for name in ("duo_decode_ragged_shared", "duo_ragged_shared_workspace_bytes"):
        assert name in _C.SYMBOLS
    rc = lib.duo_decode_ragged_shared(None, None, None, None, 0, None, 0, None, None, 0, None, 1, 1.0, None, 0, None)
    assert rc == _C.DUO_EINVAL and "duo_decode_ragged_shared: null argument" in _C.last_error()
    assert lib.duo_ragged_shared_workspace_bytes(0, 8) == 0 and lib.duo_ragged_shared_workspace_bytes(65, 8) == 0
