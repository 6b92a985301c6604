"""Idle rows of a ragged batch, host side: the active-row partition of the host twin (compact-batch partition, the
clamp that keeps it inside the launch's slots), and the parent cache's batched paths (advance, evict_last, check_room,
the min_room / max_full_len passed to the kernels, the INT4 row check) passing idle rows by.  No GPU needed."""
import types

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import (INT4_RAGGED_POLICY, DuoKVCache, DuoRaggedINT4KVCache, DuoRaggedKVCache,
                                         ragged_partition, ragged_want)

SMS = 132
POLICIES = [{}, INT4_RAGGED_POLICY]


@pytest.mark.parametrize("policy", POLICIES, ids=["bf16", "int4"])
@pytest.mark.parametrize("n_full,n_stream", [(1, 7), (4, 4), (8, 0), (2, 6)])
@pytest.mark.parametrize("seed", range(4))
def test_active_subset_is_the_compact_batch(policy, n_full, n_stream, seed):
    g = torch.Generator().manual_seed(seed)
    for B in (2, 3, 8, 17, 64):
        lengths = torch.randint(0, 1 << (10 + 2 * seed), (B,), generator=g).tolist()
        active = (torch.rand(B, generator=g) < 0.6).tolist()
        part = ragged_partition(lengths, n_full, n_stream, SMS, active=active, **policy)
        full = ragged_partition(lengths, n_full, n_stream, SMS, **policy)
        assert part["slots"] == full["slots"] and part["want"] == full["want"]  # the grid is the geometry's
        assert all(s == 0 for s, a in zip(part["splits"], active) if not a)
        assert sum(part["splits"]) <= part["slots"]
        comp = [n for n, a in zip(lengths, active) if a]
        if not comp:
            assert part["splits"] == [0] * B
            continue
        compact = ragged_partition(comp, n_full, n_stream, SMS, **policy)
        if not part["clamped"]:  # the active rows get the compact batch's partition, in row order
            assert part["keys_per_split"] == compact["keys_per_split"]
            assert [s for s, a in zip(part["splits"], active) if a] == compact["splits"]
            assert part["step_want"] == compact["want"]
        else:
            assert part["step_want"] == part["slots"] // len(comp) - 1 < compact["want"]


def test_all_active_is_todays_partition():
    for lengths in ([5, 70000, 3, 1 << 20], [0] * 8, [4096] * 64):
        for nf, ns in ((1, 7), (4, 4)):
            for policy in POLICIES:
                a = ragged_partition(lengths, nf, ns, SMS, **policy)
                b = ragged_partition(lengths, nf, ns, SMS, active=[True] * len(lengths), **policy)
                assert a == b and not a["clamped"] and a["step_want"] == a["want"]


def test_clamp_binds_and_stays_inside_the_slots():
    # n_full 1, n_stream 7, B 2, one row active, 132 SMs: the compact batch wants 257 splits, the grid has 2 x 126
    assert ragged_want(1, 1, 7, SMS) == 257 and ragged_want(2, 1, 7, SMS) == 125
    part = ragged_partition([1 << 20, 1 << 20], 1, 7, SMS, active=[True, False])
    assert part["clamped"] and part["slots"] == 252 and part["step_want"] == 251
    assert part["splits"][1] == 0 and part["splits"][0] <= part["slots"]
    for B in (2, 3, 5, 8):
        for n_act in range(1, B):
            for L in (1, 300, 65536, 1 << 20, 1 << 22):
                lengths = [L] * B
                active = [b < n_act for b in range(B)]
                for policy in POLICIES:
                    p = ragged_partition(lengths, 1, 7, SMS, active=active, **policy)
                    assert sum(p["splits"]) <= p["slots"] and max(p["splits"]) <= 512
                    assert p["step_want"] * n_act + n_act <= p["slots"]


def test_partition_flag_count_checked():
    with pytest.raises(ValueError, match="2 active flags for 3 rows"):
        ragged_partition([1, 2, 3], 1, 7, active=[True, False])


# ---- the parent cache's batched paths, on a host-only cache (no handles, no device) --------------------------------
def _row(n, cap, sink=4, recent=8, layers=2):
    r = DuoKVCache.__new__(DuoKVCache)
    r.num_layers, r.sink_size, r.recent_size, r.max_size = layers, sink, recent, cap
    r.kv_seq_len_list, r.total_list, r.lo_list = [n] * layers, [n] * layers, [max(sink, n - recent)] * layers
    r.num_full_kv_head_list, r.full_cap_list, r.dev_state = [1] * layers, [cap] * layers, None
    return r


def _cache(lengths, caps, cls=DuoRaggedKVCache, pooled=True):
    c = cls.__new__(cls)
    B = len(lengths)
    c.batch_size, c.num_layers, c.pooled, c.kv_format = B, 2, pooled, cls._KV
    c.rows = [_row(n, cap) for n, cap in zip(lengths, caps)]
    c._active, c._share, c._row_caps = [True] * B, [None] * B, list(caps)
    c.row_state = torch.zeros(B, 4, dtype=torch.int64)
    c.rows_changed, c.graph_attached = False, False
    c.num_full_kv_head_list, c.num_kv_groups, c.max_rows = [1, 1], 4, cls.max_rows
    return c


def test_set_active_flags_row_state_and_range_checks():
    c = _cache([10, 20, 30], [64, 64, 64])
    assert c.row_active == [True, True, True] and c.row_state[:, 3].tolist() == [0, 0, 0]
    c.set_active(1, False)
    assert c.row_active == [True, False, True] and c.rows_changed
    assert c.row_state[:, 3].tolist() == [0, _C.ROW_IDLE, 0] and c.row_state[:, 0].tolist() == [10, 20, 30]
    c.set_active(1, True)
    assert c.row_state[:, 3].tolist() == [0, 0, 0]
    for b in (-1, 3, 1.0, True, "0", None):
        with pytest.raises(ValueError, match="set_active row"):
            c.set_active(b, False)
    for a in (2, "no", None, 0.5):
        with pytest.raises(ValueError, match="needs a bool"):
            c.set_active(0, a)
    assert c.row_active == [True, True, True]


def test_advance_and_evict_skip_idle_rows():
    c = _cache([10, 20, 30], [64, 64, 64])
    c.set_active(1, False)
    before = c.rows[1].snapshot_state()
    DuoKVCache.advance_host(c, 3)  # one replayed step of 3 tokens
    c.advance(0, 1)
    assert c.rows[1].snapshot_state() == before
    assert [r.kv_seq_len_list for r in c.rows] == [[14, 13], [20, 20], [34, 33]]
    c.evict_last(2)
    assert c.rows[1].snapshot_state() == before and c.row_lengths == [11, 20, 31]
    assert c.row_state[:, 0].tolist() == [11, 20, 31] and c.row_state[1, 3] == _C.ROW_IDLE


def test_a_full_idle_row_no_longer_blocks_a_step():
    c = _cache([64, 20, 30], [64, 64, 64])
    with pytest.raises(ValueError, match="max size 64"):
        c.check_room(1)
    c.set_active(0, False)
    c.check_room(1)
    c.check_room(34)
    with pytest.raises(ValueError, match="max size 64"):
        c.check_room(35)


def _launches(c, S=1):
    """attend() of one batched step with the launch recorded instead of run: {entry point: args}."""
    seen = {}
    lib = types.SimpleNamespace(**{n: n for n in ("duo_decode_ragged", "duo_decode_ragged_int4",
                                                  "duo_decode_ragged_pooled", "duo_decode_ragged_shared")})
    c.lib, c.handles = lib, [0, 0]
    c.row_geom = c.row_share = c.workspace = torch.zeros(1, dtype=torch.int64)

    def attend_args(l, qkv, out, cos, sin, scale):
        c._check_chunk(l, S)
        return S, 0.1, None, None, None

    c._attend_args = attend_args
    c._launch = lambda fn, *args, **kw: seen.setdefault(fn, args)
    t = torch.zeros(1, S, 8)
    c.attend(0, t, None, None, _C.ROPE_NONE, t)
    return seen


def test_min_room_and_max_len_passed_to_the_kernels_skip_idle_rows():
    c = _cache([60, 10, 30], [64, 40, 64])
    c.set_active(0, False)
    args = _launches(c)["duo_decode_ragged_pooled"]
    assert args[3] == min(40 - 10, 64 - 30)
    assert [r.kv_seq_len_list[0] for r in c.rows] == [60, 11, 31]  # the idle row did not advance
    u = _cache([60, 10, 30], [64, 64, 64], pooled=False)
    u.set_active(0, False)
    assert _launches(u)["duo_decode_ragged"][2] == 30  # max_full_len over the active rows (the idle one holds 60)
    for b in range(3):
        u.set_active(b, False)
    assert _launches(u)["duo_decode_ragged"][2] == 0  # every row idle: the launch writes nothing
    c.set_active(1, False)
    c.set_active(2, False)
    assert _launches(c, S=2)["duo_decode_ragged_pooled"][3] == 2


def test_int4_empty_row_may_sit_idle():
    c = _cache([0, 100, 50], [256] * 3, cls=DuoRaggedINT4KVCache)
    with pytest.raises(ValueError, match="row 0 is empty"):
        c.check_rows([0, 1])
    c.set_active(0, False)
    c.check_rows([0, 1])
    assert "duo_decode_ragged_pooled" in _launches(c)
    c.set_active(0, True)
    with pytest.raises(ValueError, match="row 0 is empty"):
        _launches(c)
