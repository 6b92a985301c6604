"""The batched ragged prefill (``DuoRaggedKVCache.attend_rows``, ``duo_prefill_ragged``) against ``row(b).attend``.

* chunks of >= 128 tokens: outputs and every byte of the cache (pool headroom, the rows of rows without a chunk, sink,
  ring and staging slots), ``row_state`` and host occupancy bit-identical to a control cache that takes the same chunks
  one row at a time, across dtypes, head mixes, uniform and pooled layouts, rows at occupancy 0 / below the sink /
  mid-ring / many wraps / 9,000 tokens, donors and sharers (a fork of a sharer too) in one call, and idle rows;
* short chunks (1, 3, 17, 64, 127 tokens), which ``row(b)`` hands to the mma.sync kernel: fp64 attention through both
  gates of ``tests/parity.py``, with poison (V = 1024) in region slack past each row's length, in free pool rows and in
  the donor's rows past P, and a write census: no byte outside each row's new rows, its ring and its staging changes;
* refusals change no byte.
"""
import copy
import ctypes as C

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedKVCache
from oracle import duo_oracle as O
from parity import assert_parity
from test_gpu_attention import Fa2Shadow, split_qkv

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def _snap(c):
    return {k: v.clone() for k, v in c.tensors[0].items()}


def _same_cache(S, Cc, what):
    for k, v in S.tensors[0].items():
        assert torch.equal(v, Cc.tensors[0][k]), f"{what}: {k} differs from the row-by-row control"
    Cc.sync_device_state()  # row(b).attend leaves the parent's device copy to the next batched step
    assert torch.equal(S.row_state, Cc.row_state), f"{what}: row_state"
    assert S.snapshot_state() == Cc.snapshot_state(), f"{what}: host occupancy"


def _batched(S, lens, xs, cs, ss, Hq):
    """One attend_rows call on the packed chunks ``xs`` (per row, None for 0 tokens); returns the per-row outputs."""
    parts = [x for x in xs if x is not None]
    qkv = torch.cat(parts, 1).contiguous()
    cos = torch.cat([c for c in cs if c is not None], 0).contiguous()
    sin = torch.cat([s for s in ss if s is not None], 0).contiguous()
    out = torch.empty(1, qkv.shape[1], Hq, D, dtype=qkv.dtype, device=DEV)
    S.attend_rows(0, qkv, cos, sin, _C.ROPE_HF, out, lens)
    outs, o = [], 0
    for n in lens:
        outs.append(out[:, o : o + n])
        o += n
    return outs


def _row_by_row(Cc, lens, xs, cs, ss, Hq):
    outs = []
    for b, n in enumerate(lens):
        if n == 0:
            outs.append(None)
            continue
        o = torch.empty(1, n, Hq, D, dtype=xs[b].dtype, device=DEV)
        Cc.row(b).attend(0, xs[b].clone(), cs[b], ss[b], _C.ROPE_HF, o)
        outs.append(o)
    return outs


# ---- 1. bit identity with row(b).attend ---------------------------------------------------------------------------
HEADS = [(32, 8, 0), (32, 8, 1), (32, 8, 4), (32, 8, 8), (8, 8, 4)]


@pytest.mark.parametrize("layout", ["uniform", "pooled"])
@pytest.mark.parametrize("Hq,Hkv,n_full", HEADS, ids=["g4_0of8", "g4_1of8", "g4_4of8", "g4_8of8", "mha_4of8"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_chunks_of_128_and_more_are_bit_identical_to_row_by_row(dtype, Hq, Hkv, n_full, layout):
    """Rows start at 0, 10 (below the sink of 16), 40 (mid-ring of W = 64), 700 (many wraps) and 9,000 tokens; row 5 is
    idle.  Three rounds of chunks mixed with zeros; on the pooled layout rows 6 and 7 are forks of row 3 and of row 6
    (a fork of a sharer), taking chunks in the same calls as their donor."""
    sink, recent = 16, 48
    pooled = layout == "pooled"
    starts = [0, 10, 40, 700, 9000, 128]
    rounds = [[300, 128, 0, 129, 4097, 128], [128, 0, 256, 300, 129, 0], [4097, 129, 128, 0, 128, 300]]
    B = len(starts) + (2 if pooled else 0)
    if pooled:
        rounds = [r + [0, 0] for r in rounds[:1]] + [r + [129, 300] for r in rounds[1:]]
        caps = [n + 8800 for n in starts] + [8800, 8800]
        mk = lambda: DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV,
                                                    stage_cap=4224, pool_size=sum(caps) + 4096)
    else:
        mk = lambda: DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, 18000, sink, recent, dtype, DEV,
                                                    stage_cap=4224)
    S, Cc = mk(), mk()
    g = torch.Generator().manual_seed(7 * n_full + Hq + pooled)
    for c in (S, Cc):  # the same finite poison everywhere nothing was written yet (both layouts, rings included)
        for k, t in c.tensors[0].items():
            t.copy_((torch.rand(t.shape, generator=torch.Generator().manual_seed(len(k))) * 8 - 4).to(dtype))
    width = (Hq + 2 * Hkv) * D
    x = lambda n: torch.randn(1, n, width, generator=g).to(dtype).to(DEV)
    tab = lambda n: (torch.rand(n, D, generator=g) * 2 - 1).to(dtype).to(DEV)
    for b, n in enumerate(starts):  # history, identical in both caches, through row(b)
        for c0 in range(0, n, 4096):
            xb, cb, sb = x(min(4096, n - c0)), tab(min(4096, n - c0)), tab(min(4096, n - c0))
            for c in (S, Cc):
                o = torch.empty(1, xb.shape[1], Hq, D, dtype=dtype, device=DEV)
                c.row(b).attend(0, xb.clone(), cb, sb, _C.ROPE_HF, o)
    for c in (S, Cc):
        c.set_active(5, False)
    _same_cache(S, Cc, "history")
    for k, lens in enumerate(rounds):
        if pooled and k == 1:
            for c in (S, Cc):
                c.share_prefix(3, 6, 8800)
                c.share_prefix(6, 7, 8800)
            assert S.row_prefix[6] == S.row_prefix[7] == (3, S.row_lengths[3] // 128 * 128)
        xs = [x(n) if n else None for n in lens]
        cs = [tab(n) if n else None for n in lens]
        ss = [tab(n) if n else None for n in lens]
        got = _batched(S, lens, [t.clone() if t is not None else None for t in xs], cs, ss, Hq)
        want = _row_by_row(Cc, lens, xs, cs, ss, Hq)
        for b, n in enumerate(lens):
            if n:
                assert torch.equal(got[b], want[b]), f"round {k}: row {b}, chunk of {n}"
        torch.cuda.synchronize()
        _same_cache(S, Cc, f"round {k}")
    assert S.row_lengths[4] > 9000


# ---- 2. short chunks against fp64, poison and a write census --------------------------------------------------------
POISON_V = 1024.0


def _census(before, after, S, lens, rows_own0):
    """Every byte that changed lies in a participating row's new retrieval rows, its ring + staging slots."""
    W = S.W
    nf = S.num_full_kv_head_list[0]
    for k in before:
        changed = (before[k] != after[k])
        changed = changed.reshape(changed.shape[0], -1).any(-1) if k.startswith("full") else changed.any(-1)
        allowed = torch.zeros_like(changed)
        for b, n in enumerate(lens):
            if not n:
                continue
            if k.startswith("full"):
                first, cap = S._geom[b]
                for h in range(nf):
                    r0 = first * nf + h * cap + rows_own0[b]
                    allowed[r0 : r0 + n] = True
            else:
                allowed[b, :, : W + n] = True
        bad = changed & ~allowed
        assert not bad.any(), f"{k}: {int(bad.sum())} rows written outside the rows' new keys, rings and staging"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_short_chunks_match_fp64_and_write_nothing_else(dtype):
    """Rows: 0 a donor of 300 tokens, 1 and 2 its forks (P = 256), 3 a plain row of 150 tokens, 4 an empty row, 5 a row
    of 40.  After the forks the donor appends 100 tokens the forks must not see.  Poison (K = 0, V = 1024) fills the pool
    before any write: region slack, free rows, and the donor's rows past P from the forks' view."""
    Hq, Hkv, n_full, sink, recent = 32, 8, 3, 16, 48
    G = Hq // Hkv
    B = 6
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, [600, 300, 300, 400, 300, 300], sink, recent, dtype,
                                       DEV, stage_cap=256, pool_size=4096)
    t = S.tensors[0]
    t["full_k"].zero_()
    t["full_v"].fill_(POISON_V)
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(11)
    x = lambda n: torch.randn(1, n, width, generator=g).to(dtype)
    hist = {}
    for b, n in ((0, 300), (3, 150), (5, 40)):
        hist[b] = x(n)
        o = torch.empty(1, n, Hq, D, dtype=dtype, device=DEV)
        S.row(b).attend(0, hist[b].to(DEV), None, None, _C.ROPE_NONE, o)
    S.share_prefix(0, 1, 300)
    S.share_prefix(0, 2, 300)
    hist[1] = hist[2] = hist[0]
    more = x(100)
    o = torch.empty(1, 100, Hq, D, dtype=dtype, device=DEV)
    S.row(0).attend(0, more.to(DEV), None, None, _C.ROPE_NONE, o)
    hist[0] = torch.cat([hist[0], more], 1)
    hist[4] = None
    for lens in ([17, 1, 127, 3, 64, 0], [128, 64, 3, 1, 17, 127]):
        xs = [x(n) if n else None for n in lens]
        qkv = torch.cat([v for v in xs if v is not None], 1)
        out = torch.empty(1, qkv.shape[1], Hq, D, dtype=dtype, device=DEV)
        own0 = [S.row_lengths[b] - (S.row_prefix[b][1] if S.row_prefix[b] else 0) for b in range(B)]
        before = _snap(S)
        S.attend_rows(0, qkv.to(DEV), None, None, _C.ROPE_NONE, out, lens)
        torch.cuda.synchronize()
        _census(before, _snap(S), S, lens, own0)
        o = 0
        for b, n in enumerate(lens):
            if not n:
                continue
            past = None
            shadow = Fa2Shadow(n_full, G, sink, recent)
            if hist[b] is not None:
                q, k, v = split_qkv(hist[b], Hq, Hkv)
                _, past = O.tuple_attention_core(q.double(), k.double(), v.double(), None, n_full, G, sink, recent)
                shadow.step(q, k, v)
            q, k, v = split_qkv(xs[b], Hq, Hkv)
            ref, _ = O.tuple_attention_core(q.double(), k.double(), v.double(), past, n_full, G, sink, recent)
            fa2, truth = copy.copy(shadow).step(q, k, v)
            got = out[:, o : o + n].float().cpu()
            assert got.abs().max() < POISON_V / 2, f"row {b}: poison reached the output"
            assert_parity(got, ref, f"row {b}: chunk of {n} after {S.row_lengths[b] - n} keys", fa2=fa2, truth=truth)
            hist[b] = xs[b] if hist[b] is None else torch.cat([hist[b], xs[b]], 1)
            o += n


# ---- 3. refusals change nothing ---------------------------------------------------------------------------------------
def test_refusals_change_no_byte():
    from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache

    Hq, Hkv, n_full, dtype = 32, 8, 4, torch.bfloat16
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], 3, [300, 200, 300], 16, 48, dtype, DEV,
                                       stage_cap=256)
    width = (Hq + 2 * Hkv) * D
    x = lambda n: torch.randn(1, n, width, dtype=dtype, device=DEV)
    o = torch.empty(1, 150, Hq, D, dtype=dtype, device=DEV)
    S.row(1).attend(0, x(150), None, None, _C.ROPE_NONE, o)
    before, st, rs = _snap(S), S.snapshot_state(), S.row_state.clone()

    def unchanged(what):
        torch.cuda.synchronize()
        for k, v in before.items():
            assert torch.equal(v, S.tensors[0][k]), f"{what}: {k} changed"
        assert S.snapshot_state() == st and torch.equal(S.row_state, rs), f"{what}: occupancy changed"

    out = torch.empty(1, 200, Hq, D, dtype=dtype, device=DEV)
    for lens, match in (([100, 100, 0], "room"), ([100, 100], "entries"), ([100, 50, 0], "add up"),
                        ([300, 0, -100], ">= 0")):
        with pytest.raises(ValueError, match=match if match != "room" else "Trying to put 100 KVs"):
            S.attend_rows(0, x(200), None, None, _C.ROPE_NONE, out, lens)
        unchanged(str(lens))
    # the C entry point's own check of a row without room (the host checks first on the way through attend_rows)
    lens, room = (C.c_int32 * 3)(0, 51, 0), (C.c_int64 * 3)(300, 50, 300)
    q = x(51)
    rc = S.lib.duo_prefill_ragged(S.handles[0], S.row_state.data_ptr(), S.row_geom.data_ptr(), S.row_share.data_ptr(),
                                  lens, room, q.data_ptr(), q.stride(1), None, None, _C.ROPE_NONE, out.data_ptr(),
                                  0.1, None, 0, None)
    assert rc == _C.DUO_EOVERFLOW and "room for 50 more" in _C.last_error()
    unchanged("C no room")
    # INT4 caches refuse the method
    I = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], 2, 256, 16, 48, dtype, DEV)
    with pytest.raises(ValueError, match="16-bit caches only"):
        I.attend_rows(0, x(128), None, None, _C.ROPE_NONE, torch.empty(1, 128, Hq, D, dtype=dtype, device=DEV), [128, 0])
    # all lengths 0: a no-op
    S.attend_rows(0, x(0), None, None, _C.ROPE_NONE, torch.empty(1, 0, Hq, D, dtype=dtype, device=DEV), [0, 0, 0])
    unchanged("all zero")
