"""Prefill-sized chunks on forks of a sequence-sharded prompt without a GPU: duo_prefill_seq_shared rejects bad
arguments before any CUDA call, and DuoSeqShardForkKVCache refuses the chunks it does not take before any launch."""
import ctypes as C
import types

import pytest

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoSeqShardForkKVCache
from duo_attention_b200.seqshard import SeqShardPlan


def _layer(lib, batch=1, group=4, kv_format=_C.KV_SAME, pool=0, stage_cap=64):
    """A handle that needs no tensor map (a 16-bit layer without heads, or an INT4 layer), as the other ABI tests use."""
    d = _C.LayerDesc()
    d.full_k = d.full_v = d.ring_k = d.ring_v = None
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 0, batch, 0, 0, group, 128
    d.sink, d.recent, d.stage_cap, d.dtype, d.kv_format = 4, 8, stage_cap, _C.DT_BF16, kv_format
    h = C.c_void_p()
    rc = lib.duo_layer_create_pooled(C.byref(d), pool, C.byref(h)) if pool else lib.duo_layer_create(C.byref(d),
                                                                                                      C.byref(h))
    assert rc == _C.DUO_OK, _C.last_error()
    return h.value


def _state(full_len, rank=0, world=2, block=16, device_state=None):
    st = _C.CacheState(full_len, full_len, 4, device_state)
    st.seq_rank, st.seq_world, st.seq_block = rank, world, block
    return st


Q, OUT, PO, PL = 0x10000, 0x20000, 0x30000, 0x40000


def test_entry_point_rejects_bad_arguments_before_cuda():
    lib = _C.load()
    forks, donor = _layer(lib, batch=3), _layer(lib)
    bad = {"int4": _layer(lib, kv_format=_C.KV_INT4), "pooled": _layer(lib, pool=128),
           "batch2": _layer(lib, batch=2), "group2": _layer(lib, group=2),
           "small stage": _layer(lib, batch=3, stage_cap=16)}

    def call(layer=forks, prefix=donor, prefix_len=64, st=None, q=Q, out=OUT, po=PO, pl=PL, q_len=24):
        st = _state(70) if st is None else st
        return lib.duo_prefill_seq_shared(layer, prefix, prefix_len, C.byref(st) if st != "null" else None, q,
                                          16 * 128, out, po, pl, q_len, 0.1, None, 0, None)

    try:
        einval = {
            "null layer": call(layer=None), "null prefix": call(prefix=None), "null state": call(st="null"),
            "null q": call(q=None), "null out": call(out=None), "null out_o": call(po=None),
            "null out_lse": call(pl=None),
            "int4 forks": call(layer=bad["int4"]), "int4 prefix": call(prefix=bad["int4"]),
            "pooled forks": call(layer=bad["pooled"]), "pooled prefix": call(prefix=bad["pooled"]),
            "prefix batch 2": call(prefix=bad["batch2"]), "group mismatch": call(prefix=bad["group2"]),
            "no descriptor": call(st=_state(70, 0, 0, 0)), "world 1": call(st=_state(70, 0, 1, 16)),
            "world 9": call(st=_state(70, 0, 9, 16)), "bad rank": call(st=_state(70, 2, 2, 16)),
            "block 0": call(st=_state(70, 0, 2, 0)), "device_state": call(st=_state(70, device_state=0x5000)),
            "q_len 0": call(q_len=0),
            "prefix_len 0": call(prefix_len=0), "prefix_len off the round": call(prefix_len=48),
            "prefix_len > full_len": call(prefix_len=96, st=_state(70)),
            # block 4 at world 2: P = 8 is a whole round, but its 4 local rows are not a multiple of 8
            "prefix rows not a multiple of 8": call(prefix_len=8, st=_state(70, 0, 2, 4)),
        }
        for what, rc in einval.items():
            assert rc == _C.DUO_EINVAL, (what, rc, _C.last_error())
        # decode-sized chunks point to the one-token step
        for q_len in (1, 2, 4):
            assert call(q_len=q_len) == _C.DUO_EINVAL
            assert "duo_decode_fused_seq_shared" in _C.last_error()
        assert call(prefix_len=8, st=_state(70, 0, 2, 4)) == _C.DUO_EINVAL and "multiple of 8" in _C.last_error()
        # own-slice room (the staging area here; the retrieval rows are checked with full_len - P the same way)
        assert call(layer=bad["small stage"], q_len=17) == _C.DUO_EOVERFLOW
    finally:
        for h in [forks, donor, *bad.values()]:
            lib.duo_layer_destroy(h)


def test_symbol_present():
    lib = _C.load()
    assert "duo_prefill_seq_shared" in _C.SYMBOLS and hasattr(lib, "duo_prefill_seq_shared")


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _forks(group, block, P, graph=False):
    """A stub of forks at world 2 sharing P positions; nothing behind it may be launched."""
    f = DuoSeqShardForkKVCache.__new__(DuoSeqShardForkKVCache)
    f.num_kv_groups, f.prefix_len, f.plan, f.max_q = group, P, SeqShardPlan(2, block), 1
    f.graph_attached, f.batch_size, f.num_full_kv_head_list = graph, 3, [2]
    f.seq = types.SimpleNamespace(comm=types.SimpleNamespace(max_rows=1 << 20), rank=0, world=2, block=block)
    f.lib, f.launch_count = _NoLaunch(), 0
    return f


@pytest.mark.parametrize("group", [1, 4])
def test_forks_refuse_decode_sized_chunks(group):
    f = _forks(group, 16, 64)
    for S in range(2, 16 // group + 1):
        with pytest.raises(ValueError, match="one token"):
            f._check_chunk(0, S)
    f._check_chunk(0, 1)
    f._check_chunk(0, 16 // group + 1)  # the smallest prefill-sized chunk
    assert f.launch_count == 0


def test_forks_refuse_chunks_on_blocks_they_cannot_load():
    for block in (4, 12, 20):
        with pytest.raises(ValueError, match=f"block {block}"):
            _forks(4, block, 4 * block)._check_chunk(0, 100)
        _forks(4, block, 0)._check_chunk(0, 100)  # nothing shared: DuoSeqShardKVCache's chunk path
        _forks(4, block, 4 * block)._check_chunk(0, 1)  # one-token steps are unaffected
    for block in (8, 16, 24, 1024):
        _forks(4, block, 4 * block)._check_chunk(0, 100)


def test_forks_refuse_chunks_under_a_graph():
    f = _forks(4, 16, 64, graph=True)
    with pytest.raises(ValueError, match="DuoDecodeGraph"):
        f._check_chunk(0, 100)
    f._check_chunk(0, 1)
