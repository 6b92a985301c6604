"""Shared prefixes on the INT4 KV cache, on the GPU: DuoRaggedINT4KVCache.share_prefix, the INT4 cascade of
duo_decode_ragged_shared, a sharer's chunks (duo_attention_shared on INT4 handles, or the dequantised image), the patched
model and DuoDecodeGraph.

* decode against a control cache in which every row holds its own copy of the prompt: outputs within the 16-bit
  shared-prefix test's tolerance, own retrieval rows (codes, scales, zeros), sinks and rings bit-identical; the free
  rows of every region hold poison, which a kernel reading past a row's keys would carry into the outputs;
* no sharing: the bits of duo_decode_ragged_pooled;
* a sharer's chunks bit-identical to the same chunks on a row holding a copy, for forks made before and after a question;
* idle donors and wholly idle groups; graph replay; model level; refusals leave every byte unchanged.
"""

import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
TOL = {torch.bfloat16: dict(rtol=1.6e-2, atol=1.6e-2), torch.float16: dict(rtol=2e-3, atol=2e-3)}


def _cache(Hq, Hkv, n_full, caps, sink, recent, dtype, stage_cap=64):
    return DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], len(caps), caps, sink, recent, dtype, DEV,
                                              stage_cap=stage_cap)


def _prefill(rows, L, width, dtype, Hq, g, chunk=4096):
    for c0 in range(0, L, chunk):
        S = min(chunk, L - c0)
        qkv = (torch.randn(1, S, width, generator=g) * 0.5).to(dtype).to(DEV)
        for r in rows:
            r.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))


def _cache_bytes(c):
    return [{k: v.clone() for k, v in t.items()} for t in c.tensors]


def _poison_free_rows(c, b):
    """Codes 0xff with scale and zero 1000 in the rows of row b's region past its keys: a weight on any of them would
    move the output far outside the tolerance."""
    r = c.row(b)
    n_own = r.kv_seq_len - (c.row_prefix[b][1] if c.row_prefix[b] else 0)
    for k, t in r.tensors[0].items():
        if k.startswith("full"):
            t[0, :, n_own:] = 0xFF if t.dtype == torch.uint8 else 1000.0


def _own_rows_equal(S, C, b):
    P = S.row_prefix[b][1] if S.row_prefix[b] else 0
    n, W = S.row_lengths[b], S.W
    for name, t in S.row(b).tensors[0].items():
        mine, theirs = t[0], C.row(b).tensors[0][name][0]
        if name.startswith("full"):
            mine, theirs = mine[:, : n - P], theirs[:, P:n]
        else:
            mine, theirs = mine[:, :W], theirs[:, :W]
        assert torch.equal(mine, theirs), f"row {b}: {name} differs from the control's"


# ---- 1. decode against a control that holds copies ------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 8), (8, 8, 1), (8, 8, 8)])
@pytest.mark.parametrize("q_len", [1, 2, 8])
@pytest.mark.parametrize("LA,LB", [(300, 1024), (256, 100), (4097, 640), (9000, 300)])
def test_sharers_match_control(LA, LB, q_len, Hq, Hkv, n_full, dtype):
    """Rows: 0 donor of prompt A, 1 forked from 0, 2 forked from 1 (a fork of a sharer), 3 donor of prompt B, 4 forked
    from 3, 5 a plain row.  LA = 9000: the prefix launch splits its 8960 keys."""
    if Hq // Hkv * q_len > _C.DECODE_MAX_Q_INT4:
        pytest.skip("decode steps of an INT4 cache take group x q_len <= 8 rows")
    sink, recent, B, steps = 16, 48, 6, 4
    room = 128 + steps * q_len
    caps_s = [LA + room, room, room, LB + room, room, 700 + room]
    caps_c = [LA + room, LA + room, LA + room, LB + room, LB + room, 700 + room]
    S, C = _cache(Hq, Hkv, n_full, caps_s, sink, recent, dtype), _cache(Hq, Hkv, n_full, caps_c, sink, recent, dtype)
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
    S.check_rows([0])  # a sharer is not empty
    for b in (1, 2, 4):
        _own_rows_equal(S, C, b)  # the fork's tail copy: codes, scales and zeros
        _poison_free_rows(S, b)
    for step in range(steps):
        qkv = (torch.randn(B, q_len, width, generator=g) * 0.5).to(dtype).to(DEV)
        os_, oc = (torch.empty(B, q_len, Hq, D, dtype=dtype, device=DEV) for _ in range(2))
        S.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, os_)
        C.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, oc)
        torch.testing.assert_close(os_.float(), oc.float(), **TOL[dtype], msg=lambda m: f"step {step}: {m}")
        if not S.sharing:  # nothing shared: the pooled launch, the same bits
            assert torch.equal(os_, oc)
    torch.cuda.synchronize()
    assert S.row_lengths == C.row_lengths
    for b in range(B):
        _own_rows_equal(S, C, b)


# ---- 2. no sharing: the pooled launch's bits ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 4), (8, 8, 8)])
def test_no_sharing_is_bit_identical_to_pooled(Hq, Hkv, n_full, dtype):
    sink, recent = 16, 48
    lengths = [1, 129, 700, 5000]
    B = len(lengths)
    caps = [L + 64 + 37 * b for b, L in enumerate(lengths)]
    A, Bc = (_cache(Hq, Hkv, n_full, caps, sink, recent, dtype) for _ in range(2))
    g = torch.Generator().manual_seed(5 + n_full)
    width = (Hq + 2 * Hkv) * D
    for b, L in enumerate(lengths):
        _prefill([A.row(b), Bc.row(b)], L, width, dtype, Hq, g)
    lib = _C.load()
    ws = torch.zeros(lib.duo_ragged_shared_workspace_bytes(B, Hkv), dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    for step, S in enumerate([1, 2, 1, 8, 1]):
        if Hq // Hkv * S > 8:
            continue
        qkv = (torch.randn(B, S, width, generator=g) * 0.5).to(dtype).to(DEV)
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


# ---- 3. a sharer's chunks: the bits of a row holding a copy ---------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n_full", [1, 8])
@pytest.mark.parametrize("recent", [48, 2544], ids=["W64", "W2560"])
@pytest.mark.parametrize("chunk", [3, 4, 9, 100, 128, 700, 4097])
def test_sharer_chunks_bit_identical_to_copy(chunk, recent, n_full, dtype):
    """Row 1 forks row 0's prompt and takes a question chunk; row 2 forks row 1 after that question and takes another.
    The control's rows 1 and 2 prefilled the same tokens themselves.  Chunks of 3 and 4 tokens (12 and 16 rows) take
    the 16-row INT4 kernel, 9 and 100 the 64-row one, >= 128 the dequantised image at W = 64 and the 64-row INT4 kernel
    at W = 2560."""
    Hq, Hkv, sink, L = 32, 8, 16, 1000
    room = 2 * chunk + 256
    caps_s, caps_c = [L + room, room, room], [L + room] * 3
    S = _cache(Hq, Hkv, n_full, caps_s, sink, recent, dtype)
    C = _cache(Hq, Hkv, n_full, caps_c, sink, recent, dtype)
    g = torch.Generator().manual_seed(chunk + recent + n_full)
    width = (Hq + 2 * Hkv) * D
    _prefill([S.row(0), C.row(0), C.row(1), C.row(2)], L, width, dtype, Hq, g)
    S.share_prefix(0, 1, room)
    q1 = (torch.randn(1, chunk, width, generator=g) * 0.5).to(dtype).to(DEV)
    q2 = (torch.randn(1, chunk, width, generator=g) * 0.5).to(dtype).to(DEV)
    o = [torch.empty(1, chunk, Hq, D, dtype=dtype, device=DEV) for _ in range(4)]
    S.row(1).attend(0, q1.clone(), None, None, _C.ROPE_NONE, o[0])
    C.row(1).attend(0, q1.clone(), None, None, _C.ROPE_NONE, o[1])
    C.row(2).attend(0, q1.clone(), None, None, _C.ROPE_NONE, torch.empty_like(o[1]))
    assert torch.equal(o[0], o[1]), "fork before the question: the chunk differs from a copy row's"
    S.share_prefix(1, 2, room)  # a fork after the question: it copies row 1's own rows, question included
    S.row(2).attend(0, q2.clone(), None, None, _C.ROPE_NONE, o[2])
    C.row(2).attend(0, q2.clone(), None, None, _C.ROPE_NONE, o[3])
    assert torch.equal(o[2], o[3]), "fork after the question: the chunk differs from a copy row's"
    torch.cuda.synchronize()
    for b in (1, 2):
        _own_rows_equal(S, C, b)


# ---- 4. idle donors and idle groups --------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_idle_donor_and_idle_group(dtype):
    """Rows 0 (donor A), 1, 2 (sharers of A), 3 (donor B), 4 (sharer of B).  Row 0 idle while 1, 2 decode; then rows 3
    and 4 (a whole group) idle.  The control holds copies and the same flags; idle rows are not written."""
    Hq, Hkv, n_full, sink, recent, B = 32, 8, 4, 16, 48, 5
    room = 256
    caps_s = [2000 + room, room, room, 700 + room, room]
    caps_c = [2000 + room] * 3 + [700 + room] * 2
    S, C = _cache(Hq, Hkv, n_full, caps_s, sink, recent, dtype), _cache(Hq, Hkv, n_full, caps_c, sink, recent, dtype)
    g = torch.Generator().manual_seed(3)
    width = (Hq + 2 * Hkv) * D
    _prefill([S.row(0), C.row(0), C.row(1), C.row(2)], 2000, width, dtype, Hq, g)
    _prefill([S.row(3), C.row(3), C.row(4)], 700, width, dtype, Hq, g)
    S.share_prefix(0, 1, room)
    S.share_prefix(0, 2, room)
    S.share_prefix(3, 4, room)
    for idle in ([0], [3, 4], [0, 3, 4], []):
        for c in (S, C):
            for b in range(B):
                c.set_active(b, b not in idle)
        for step in range(2):
            qkv = (torch.randn(B, 2, width, generator=g) * 0.5).to(dtype).to(DEV)
            os_ = torch.full((B, 2, Hq, D), 7.0, dtype=dtype, device=DEV)
            oc = os_.clone()
            S.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, os_)
            C.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, oc)
            act = [b for b in range(B) if b not in idle]
            torch.testing.assert_close(os_[act].float(), oc[act].float(), **TOL[dtype])
            for b in idle:
                assert bool((os_[b] == 7.0).all()), f"idle row {b} was written"
        assert S.row_lengths == C.row_lengths
    torch.cuda.synchronize()
    for b in range(B):
        _own_rows_equal(S, C, b)


# ---- model level ---------------------------------------------------------------------------------------------------
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])


def _patched(seed, sink, recent, dtype=torch.bfloat16, arch="llama"):
    import transformers

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    Config, Model = ((transformers.LlamaConfig, transformers.LlamaForCausalLM) if arch == "llama" else
                     (transformers.MistralConfig, transformers.MistralForCausalLM))
    cfg = Config(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                 intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                 attn_implementation="eager")
    model = Model(cfg).to(dtype).eval()
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda()


def _agree_where_decided(ls, lc, step):
    """Greedy tokens of the forks equal the control's wherever the control's top two logits are > 0.1 apart."""
    top2 = lc.float().topk(2, dim=-1).values
    decided = (top2[..., 0] - top2[..., 1]) > 0.1
    ts, tc = ls.argmax(-1), lc.argmax(-1)
    assert torch.equal(ts[decided], tc[decided]), f"step {step}: greedy tokens differ"
    return tc


@pytest.mark.parametrize("arch,dtype", [("llama", torch.bfloat16), ("mistral", torch.float16)],
                         ids=["llama-bf16", "mistral-fp16"])
@pytest.mark.parametrize("L", [300, 640])
def test_model_forks_decode_and_take_questions_like_independent_rows(L, arch, dtype):
    """Row 0 prefilled, forked into 3 rows; rows 1 and 2 then take their own questions through row(b); all decode
    greedily against a control whose rows prefilled the prompt (and the questions) themselves."""
    sink, recent = 4, 12
    model = _patched(21, sink, recent, dtype, arch)
    S = DuoRaggedINT4KVCache(model, GATES, 4, [L + 96, 160, 160, 160], sink, recent)
    C = DuoRaggedINT4KVCache(model, GATES, 4, [L + 96 + 40] * 4, sink, recent)
    gen = torch.Generator().manual_seed(L)
    ids = torch.randint(0, 512, (1, L), generator=gen)
    qs = {1: torch.randint(0, 512, (1, 9), generator=gen), 2: torch.randint(0, 512, (1, 30), generator=gen)}
    with torch.no_grad():
        first = model(input_ids=ids.cuda(), past_key_values=S.row(0), use_cache=True).logits[:, -1:].argmax(-1)
        for b in range(4):
            model(input_ids=ids.cuda(), past_key_values=C.row(b), use_cache=True)
        for b in (1, 2, 3):
            S.share_prefix(0 if b < 3 else 2, b, 160)
        assert S.sharing
        last = {}
        for b, q in qs.items():  # each fork's own question (9 tokens: the INT4 kernels; 30: too)
            ls = model(input_ids=q.cuda(), past_key_values=S.row(b), use_cache=True).logits[:, -1:]
            lc = model(input_ids=q.cuda(), past_key_values=C.row(b), use_cache=True).logits[:, -1:]
            assert torch.equal(ls, lc), f"row {b}: the question's logits differ from a copy row's"
            last[b] = lc.argmax(-1)
        tok = torch.cat([first, last[1], last[2], (first + 3) % 512], 0)
        ts, tc = tok.clone(), tok.clone()
        for step in range(10):
            ls = model(input_ids=ts, past_key_values=S, use_cache=True).logits
            lc = model(input_ids=tc, past_key_values=C, use_cache=True).logits
            ts = tc = _agree_where_decided(ls, lc, step)
    assert S.row_lengths == C.row_lengths


def test_graph_replay_across_forks_clears_and_evictions():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 6
    model = _patched(23, sink, recent)
    caps = [400, 96, 96, 200]
    ca = DuoRaggedINT4KVCache(model, GATES, 4, caps, sink, recent, pool_size=2048)
    cb = DuoRaggedINT4KVCache(model, GATES, 4, caps, sink, recent, pool_size=2048)
    g = torch.Generator().manual_seed(8)
    prompt = torch.randint(0, 512, (1, 300), generator=g)
    with torch.no_grad():
        for c in (ca, cb):
            model(input_ids=prompt.cuda(), past_key_values=c.row(0), use_cache=True)
            model(input_ids=prompt[:, :40].cuda(), past_key_values=c.row(3), use_cache=True)
            c.share_prefix(0, 1, 96)
            c.share_prefix(0, 2, 96)
        graph = DuoDecodeGraph(model, cb)
        assert cb.graph_shared
        captured = graph.graph
        tok = torch.randint(0, 512, (4, 1), generator=g).cuda()
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
                    c.share_prefix(0, 2, 96)
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
    c = DuoRaggedINT4KVCache(model, GATES, 3, [400, 64, 64], sink, recent)
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

        qkv = torch.zeros(1, 9, (4 + 2 * 2) * 128, dtype=torch.bfloat16, device=DEV)
        for call, match in ((lambda: c.row(0).clear(), "share the first 256 keys of row 0"),
                            (lambda: c.row(0).evict_last(45), "below the 256 keys"),
                            (lambda: c.evict_last(45), "below the 256 keys"),
                            (lambda: c.row(1).evict_last(45), "into the 256 keys"),
                            (lambda: c.share_prefix(0, 1, 64), "row 1 is not empty"),
                            (lambda: c.row(1).attend(0, qkv, None, None, _C.ROPE_NONE,
                                                     torch.empty(1, 9, 4, 128, dtype=torch.bfloat16, device=DEV),
                                                     force_mma=True), "force_mma"),
                            (lambda: model(input_ids=torch.zeros(1, 2, dtype=torch.long).cuda(),
                                           past_key_values=c.row(1), use_cache=True), "batched step")):
            with pytest.raises(ValueError, match=match):
                call()
            unchanged()
        # a graph captured without the shared launch: forking would make it read wrong keys
        c2 = DuoRaggedINT4KVCache(model, GATES, 2, [400, 64], sink, recent)
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
        # a uniform-capacity INT4 cache does not share
        c3 = DuoRaggedINT4KVCache(model, GATES, 2, 400, sink, recent)
        model(input_ids=torch.randint(0, 512, (1, 300)).cuda(), past_key_values=c3.row(0), use_cache=True)
        snap = _cache_bytes(c3)
        with pytest.raises(ValueError, match="needs a 16-bit cache with per-row capacities"):
            c3.share_prefix(0, 1, 64)
        torch.cuda.synchronize()
        for t0, t1 in zip(snap, _cache_bytes(c3)):
            for k in t0:
                assert torch.equal(t0[k], t1[k]), k
        # the parent's clear ends every share
        c.clear()
        assert c.row_prefix == [None, None, None] and c.row_capacities == [400, 64, 64] and not c.sharing
