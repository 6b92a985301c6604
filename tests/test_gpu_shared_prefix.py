"""Shared prefixes on the GPU: duo_decode_ragged_shared through DuoRaggedKVCache.share_prefix, the patched model and
DuoDecodeGraph.

* against a control cache in which every row holds its own copy of the prompt: outputs and cache bytes;
* no sharing: the same bits as duo_decode_ragged_pooled;
* model level (greedy tokens of forks against independent rows) and graph replay across forks, clears and evictions;
* refusals leave the cache bytes unchanged.
"""

import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedKVCache

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
TOL = {torch.bfloat16: dict(rtol=1.6e-2, atol=1.6e-2), torch.float16: dict(rtol=2e-3, atol=2e-3)}


def _prefill(caches_rows, L, width, dtype, Hq, g):
    for c0 in range(0, L, 4096):
        S = min(4096, L - c0)
        qkv = torch.randn(1, S, width, generator=g).to(dtype).to(DEV)
        for r in caches_rows:
            r.attend(0, qkv, None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))


def _cache_bytes(c):
    return [{k: v.clone() for k, v in t.items()} for t in c.tensors]


# ---- 1. against an unshared control cache ----------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 8), (8, 8, 1), (8, 8, 8)])
@pytest.mark.parametrize("q_len", [1, 2, 4])
@pytest.mark.parametrize("LA,LB", [(300, 1024), (256, 100), (4097, 640)])
def test_sharers_match_control(LA, LB, q_len, Hq, Hkv, n_full, dtype):
    """Rows: 0 donor of prompt A, 1 forked from 0, 2 forked from 1 (a fork of a sharer), 3 donor of prompt B, 4 forked
    from 3, 5 a plain row.  The control holds every prompt in every row that reads it."""
    sink, recent, B = 16, 48, 6
    steps = 5
    room = 128 + steps * q_len
    caps_s = [LA + room, room, room, LB + room, room, 700 + room]
    caps_c = [LA + room, LA + room, LA + room, LB + room, LB + room, 700 + room]
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps_s, sink, recent, dtype, DEV, stage_cap=64)
    C = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps_c, sink, recent, dtype, DEV, stage_cap=64)
    g = torch.Generator().manual_seed(LA + 7 * q_len + 13 * n_full + Hq)
    width = (Hq + 2 * Hkv) * D
    _prefill([S.row(0), C.row(0), C.row(1), C.row(2)], LA, width, dtype, Hq, g)
    _prefill([S.row(3), C.row(3), C.row(4)], LB, width, dtype, Hq, g)
    _prefill([S.row(5), C.row(5)], 700, width, dtype, Hq, g)
    S.share_prefix(0, 1, room)
    S.share_prefix(1, 2, room)
    S.share_prefix(3, 4, room)
    PA, PB = LA // 128 * 128, LB // 128 * 128
    exp = [None, (0, PA), (0, PA), None, (3, PB), None]
    assert S.row_prefix == [e if e and e[1] else None for e in exp]
    assert S.row_capacities[1] == (PA if PA else 0) + room
    for step in range(steps):
        qkv = torch.randn(B, q_len, width, generator=g).to(dtype).to(DEV)
        os_, oc = (torch.empty(B, q_len, Hq, D, dtype=dtype, device=DEV) for _ in range(2))
        S.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, os_)
        C.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, oc)
        torch.testing.assert_close(os_.float(), oc.float(), **TOL[dtype], msg=lambda m: f"step {step}: {m}")
        if not S.sharing:  # nothing shared (prompts below 128 keys): the pooled launch, the same bits
            assert torch.equal(os_, oc)
    torch.cuda.synchronize()
    assert S.row_lengths == C.row_lengths
    W = S.W
    for b in range(B):
        P = S.row_prefix[b][1] if S.row_prefix[b] else 0
        n = S.row_lengths[b]
        for name, t in S.row(b).tensors[0].items():
            mine, theirs = t[0], C.row(b).tensors[0][name][0]
            if name.startswith("full"):
                mine, theirs = mine[:, : n - P], theirs[:, P:n]
            else:
                mine, theirs = mine[:, :W], theirs[:, :W]
            assert torch.equal(mine, theirs), f"row {b}: {name} differs from the control's"


# ---- 2. no sharing: the pooled launch's bits ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 4), (8, 8, 8)])
def test_no_sharing_is_bit_identical_to_pooled(Hq, Hkv, n_full, dtype):
    sink, recent = 16, 48
    lengths = [0, 1, 129, 700, 5000]
    B = len(lengths)
    caps = [L + 64 + 37 * b for b, L in enumerate(lengths)]
    A, Bc = (DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64)
             for _ in range(2))
    g = torch.Generator().manual_seed(5 + n_full)
    width = (Hq + 2 * Hkv) * D
    for b, L in enumerate(lengths):
        _prefill([A.row(b), Bc.row(b)], L, width, dtype, Hq, g)
    lib = _C.load()
    ws = torch.zeros(lib.duo_ragged_shared_workspace_bytes(B, Hkv), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    for step, S in enumerate([1, 2, 1, 4, 1]):
        if Hq // Hkv * S > 16:
            continue
        qkv = torch.randn(B, S, width, generator=g).to(dtype).to(DEV)
        oa, ob = (torch.empty(B, S, Hq, D, dtype=dtype, device=DEV) for _ in range(2))
        A.attend(0, qkv, None, None, _C.ROPE_NONE, oa)
        Bc.check_room(S, [0])
        Bc.sync_device_state(0)
        min_room = min(c - n for c, n in zip(Bc.row_capacities, Bc.row_lengths))
        _C.check(lib.duo_decode_ragged_shared(Bc.handles[0], Bc.row_state.data_ptr(), Bc.row_geom.data_ptr(),
                                              Bc.row_share.data_ptr(), min_room, qkv.data_ptr(), qkv.stride(1), None,
                                              None, _C.ROPE_NONE, ob.data_ptr(), S, D ** -0.5, ws.data_ptr(),
                                              ws.numel(), stream))
        Bc.advance(0, S)
        assert torch.equal(oa, ob), f"step {step}: duo_decode_ragged_shared differs from duo_decode_ragged_pooled"
    torch.cuda.synchronize()
    for name in A.tensors[0]:
        assert torch.equal(A.tensors[0][name], Bc.tensors[0][name]), f"{name} differs"


# ---- model level ---------------------------------------------------------------------------------------------------
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])


def _patched(seed, sink, recent):
    from transformers import LlamaConfig, LlamaForCausalLM

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                      intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                      attn_implementation="eager")
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda()


@pytest.mark.parametrize("L", [300, 640, 90])
def test_model_forks_decode_like_independent_rows(L):
    """One row prefilled, forked into 3 more rows; greedy decoding equals that of independent rows that each prefilled
    the prompt (a control cache), token for token, and the logits agree."""
    sink, recent = 4, 12
    model = _patched(21, sink, recent)
    S = DuoRaggedKVCache(model, GATES, 4, [L + 64, 160, 160, 160], sink, recent)
    C = DuoRaggedKVCache(model, GATES, 4, [L + 64] * 4, sink, recent)
    ids = torch.randint(0, 512, (1, L), generator=torch.Generator().manual_seed(L))
    with torch.no_grad():
        first = model(input_ids=ids.cuda(), past_key_values=S.row(0), use_cache=True).logits[:, -1:].argmax(-1)
        for b in range(4):
            model(input_ids=ids.cuda(), past_key_values=C.row(b), use_cache=True)
        for b in (1, 2, 3):
            S.share_prefix(0 if b < 3 else 2, b, 160)
        assert S.sharing == (L >= 128)
        # rows continue from different tokens, so the forks diverge
        tok = torch.cat([first, (first + 1) % 512, (first + 2) % 512, (first + 3) % 512], 0)
        ts, tc = tok.clone(), tok.clone()
        for step in range(12):
            ls = model(input_ids=ts, past_key_values=S, use_cache=True).logits
            lc = model(input_ids=tc, past_key_values=C, use_cache=True).logits
            torch.testing.assert_close(ls.float(), lc.float(), rtol=5e-2, atol=5e-2)
            ts, tc = ls.argmax(-1), lc.argmax(-1)
            assert torch.equal(ts, tc), f"step {step}: greedy tokens differ"
    assert S.row_lengths == C.row_lengths


def test_graph_replay_across_forks_clears_and_evictions():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 6
    model = _patched(23, sink, recent)
    caps = [400, 96, 96, 200]
    ca = DuoRaggedKVCache(model, GATES, 4, caps, sink, recent, pool_size=2048)
    cb = DuoRaggedKVCache(model, GATES, 4, caps, sink, recent, pool_size=2048)
    g = torch.Generator().manual_seed(8)
    prompt = torch.randint(0, 512, (1, 300), generator=g)
    with torch.no_grad():
        for c in (ca, cb):
            model(input_ids=prompt.cuda(), past_key_values=c.row(0), use_cache=True)
            model(input_ids=prompt[:, :40].cuda(), past_key_values=c.row(3), use_cache=True)
            c.share_prefix(0, 1, 96)
        graph = DuoDecodeGraph(model, cb)
        assert cb.graph_shared
        captured = graph.graph
        tok = torch.randint(0, 512, (4, 1), generator=g).cuda()
        for c in (ca, cb):  # a fork made while the graph is attached
            c.share_prefix(0, 2, 96)
        for step in range(10):
            le = model(input_ids=tok, past_key_values=ca, use_cache=True).logits
            lg = graph.step(tok)
            assert torch.equal(le, lg), f"step {step}: graph replay differs from eager decode"
            tok = le.argmax(-1)
            if step == 3:  # a sharer finishes: cleared and refilled through row(b) with a new request
                ids = torch.randint(0, 512, (1, 30), generator=g)
                for c in (ca, cb):
                    c.row(1).clear()
                    model(input_ids=ids.cuda(), past_key_values=c.row(1), use_cache=True)
            if step == 6:  # a fork made while the graph is attached
                for c in (ca, cb):
                    c.row(2).clear()
                    c.share_prefix(1, 2, 96)
            if step >= 7:
                for c in (ca, cb):
                    c.evict_last(1)
            assert ca.row_lengths == cb.row_lengths and ca.row_prefix == cb.row_prefix
        assert graph.graph is captured
        assert torch.equal(ca.row_state, cb.row_state) and torch.equal(ca.row_share, cb.row_share)


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_cache_unchanged():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 12
    model = _patched(25, sink, recent)
    c = DuoRaggedKVCache(model, GATES, 3, [400, 64, 64], sink, recent)
    with torch.no_grad():
        model(input_ids=torch.randint(0, 512, (1, 300)).cuda(), past_key_values=c.row(0), use_cache=True)
        c.share_prefix(0, 1, 64)
        torch.cuda.synchronize()
        before = (_cache_bytes(c), c.row_state.clone(), c.row_geom.clone(), c.row_share.clone(), c.row_prefix,
                  c.row_capacities, c.row_lengths, c.launch_count)

        def unchanged():
            torch.cuda.synchronize()
            now = _cache_bytes(c)
            for t0, t1 in zip(before[0], now):
                for k in t0:
                    assert torch.equal(t0[k], t1[k]), k
            assert torch.equal(before[1], c.row_state) and torch.equal(before[2], c.row_geom)
            assert torch.equal(before[3], c.row_share)
            assert before[4:] == (c.row_prefix, c.row_capacities, c.row_lengths, c.launch_count)

        for call, match in ((lambda: c.row(0).clear(), "share the first 256 keys of row 0"),
                            (lambda: c.row(0).evict_last(45), "below the 256 keys"),
                            (lambda: c.evict_last(45), "below the 256 keys"),
                            (lambda: c.row(1).evict_last(45), "into the 256 keys"),
                            (lambda: c.resize_row(0, 500), "not empty"),
                            (lambda: c.share_prefix(0, 1, 64), "row 1 is not empty"),
                            (lambda: c.share_prefix(2, 1, 64), "row 1 is not empty"),
                            (lambda: c.share_prefix(0, 2, 40), "capacity 40"),
                            (lambda: model(input_ids=torch.zeros(1, 1, dtype=torch.long).cuda(),
                                           past_key_values=c.row(1), use_cache=True), "batched step")):
            with pytest.raises(ValueError, match=match):
                call()
            unchanged()
        # a graph captured without the shared launch: forking would make it read wrong keys
        c2 = DuoRaggedKVCache(model, GATES, 2, [400, 64], sink, recent)
        model(input_ids=torch.randint(0, 512, (1, 300)).cuda(), past_key_values=c2.row(0), use_cache=True)
        model(input_ids=torch.randint(0, 512, (1, 3)).cuda(), past_key_values=c2.row(1), use_cache=True)
        DuoDecodeGraph(model, c2)
        c2.row(1).clear()
        snap = _cache_bytes(c2)
        with pytest.raises(ValueError, match="build a new DuoDecodeGraph"):
            c2.share_prefix(0, 1, 64)
        torch.cuda.synchronize()
        for t0, t1 in zip(snap, _cache_bytes(c2)):
            for k in t0:
                assert torch.equal(t0[k], t1[k]), k
        assert c2.row_prefix == [None, None]
        # the parent's clear ends every share
        c.clear()
        assert c.row_prefix == [None, None, None] and c.row_capacities == [400, 64, 64] and not c.sharing
