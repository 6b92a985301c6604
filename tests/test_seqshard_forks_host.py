"""Forks of a sequence-sharded prompt without a GPU: the shared-prefix arithmetic and the per-rank tail copy against
SeqShardPlan, and duo_decode_fused_seq_shared rejecting bad arguments before any CUDA call."""
import ctypes as C

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import fork_prefix_len, fork_tail_plan
from duo_attention_b200.seqshard import SeqShardPlan


@pytest.mark.parametrize("world,block", [(1, 7), (2, 16), (3, 5), (8, 4), (8, 1024)])
def test_prefix_and_tail_plan_match_the_shard_plan(world, block):
    plan = SeqShardPlan(world, block)
    rnd = world * block
    for n in sorted({1, block - 1, rnd - 1, rnd, rnd + 1, 2 * rnd + block + 3, 5 * rnd - 1, 7 * rnd}):
        P = fork_prefix_len(n, world, block)
        assert P % rnd == 0 and P <= n < P + rnd
        for new in (0, 1, 3 * block + 2):
            rows = fork_tail_plan(n, new, plan)
            for r, t in enumerate(rows):
                assert t["P"] == P and t["prefix_rows"] == P // world == plan.local_len(r, P)
                assert t["prefix_rows"] + t["tail_rows"] == plan.local_len(r, n)
                # position p >= P: same owner as p - P, local row shifted by P / world
                for p in range(P, n + new):
                    assert plan.owner(p) == plan.owner(p - P)
                    if plan.owner(p) == r:
                        own = plan.local_index(p) - t["prefix_rows"]
                        assert own == plan.local_index(p - P) < t["own_cap"]
                        if p < n:
                            assert own < t["tail_rows"]
                assert t["own_cap"] == plan.capacity(n - P + new)


def _layer(lib, batch=1, group=4, kv_format=_C.KV_SAME):
    """A handle that needs no tensor map (a 16-bit layer without heads, or an INT4 layer), as the other ABI tests use."""
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, 0, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, 64, _C.DT_BF16, kv_format
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(d), C.byref(h)) == _C.DUO_OK, _C.last_error()
    return h.value


def _state(full_len, rank=0, world=2, block=16):
    st = _C.CacheState(full_len, full_len, 4, None)
    st.seq_rank, st.seq_world, st.seq_block = rank, world, block
    return st


QKV, OUT, PO, PL = 0x10000, 0x20000, 0x30000, 0x40000


def test_entry_point_rejects_bad_arguments_before_cuda():
    lib = _C.load()
    assert lib.duo_seq_shared_workspace_bytes(0, 8) == 0 and lib.duo_seq_shared_workspace_bytes(4, 0) == 0
    forks, donor = _layer(lib, batch=3), _layer(lib)
    bad = {"int4": _layer(lib, kv_format=_C.KV_INT4), "batch2": _layer(lib, batch=2), "group2": _layer(lib, group=2)}

    def call(layer=forks, prefix=donor, prefix_len=64, st=_state(70), qkv=QKV, out=OUT, po=PO, pl=PL):
        return lib.duo_decode_fused_seq_shared(layer, prefix, prefix_len, C.byref(st) if st else None, qkv, 16 * 128,
                                               None, None, _C.ROPE_NONE, out, po, pl, 0.1, None, 0, None)

    try:
        cases = {
            "null layer": call(layer=None), "null prefix": call(prefix=None), "null state": call(st=None),
            "null qkv": call(qkv=None), "null out": call(out=None), "null out_o": call(po=None),
            "null out_lse": call(pl=None),
            "int4 forks": call(layer=bad["int4"]), "int4 prefix": call(prefix=bad["int4"]),
            "prefix batch 2": call(prefix=bad["batch2"]), "group mismatch": call(prefix=bad["group2"]),
            "no descriptor": call(st=_state(70, 0, 0, 0)), "world 1": call(st=_state(70, 0, 1, 16)),
            "bad rank": call(st=_state(70, 2, 2, 16)),
            "prefix_len 0": call(prefix_len=0), "prefix_len off the round": call(prefix_len=48),
            "prefix_len > full_len": call(prefix_len=96, st=_state(70)),
        }
        for what, rc in cases.items():
            assert rc == _C.DUO_EINVAL, (what, rc, _C.last_error())
    finally:
        for h in [forks, donor, *bad.values()]:
            lib.duo_layer_destroy(h)


def test_symbols_present():
    lib = _C.load()
    for s in ("duo_decode_fused_seq_shared", "duo_seq_shared_workspace_bytes"):
        assert s in _C.SYMBOLS and hasattr(lib, s)
