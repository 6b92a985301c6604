"""Prefill-sized chunks on rows that share a prompt (``row(b).attend`` on a sharer, ``duo_attention_shared``).

* bit identity with a control row that holds a copy of the prompt: outputs, own-region bytes and ring bytes, across
  dtypes, head mixes, prompts on and off a 128-key boundary, chunks on both kernels and windows that force the
  mma.sync kernel at every length; each run forks a sharer, lets the donor append after the fork and interleaves
  chunks with batched decode steps;
* fp64 attention through ``assert_parity`` (both gates), rows taking chunks of different lengths;
* a visibility census (every key has logit 0 and a one-hot value by where it lives, every row a sharer must not read
  holds poison) on both kernels, and a write census (only the sharer's own new rows and its ring / staging slots change);
* model level: questions of 9 and 700 tokens on two forks of a 300-token prompt, then greedy steps together, against
  rows that prefilled prompt and question themselves, against ``OracleModel`` and under ``DuoDecodeGraph`` replay;
* refusals leave the cache unchanged.
"""
import copy

import numpy as np
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
TOL = {torch.bfloat16: dict(rtol=1.6e-2, atol=1.6e-2), torch.float16: dict(rtol=2e-3, atol=2e-3)}


def _attend(rows, qkv, Hq):
    """The same chunk on every row of ``rows``; returns their outputs."""
    outs = []
    for r in rows:
        o = torch.empty(1, qkv.shape[1], Hq, D, dtype=qkv.dtype, device=DEV)
        r.attend(0, qkv, None, None, _C.ROPE_NONE, o)
        outs.append(o)
    return outs


def _same_row_bytes(S, C, b):
    """Row b of S holds exactly what row b of the control C holds: retrieval keys (a sharer's own ones at region rows
    j - P) and the sink + ring slots."""
    P = S.row_prefix[b][1] if S.row_prefix[b] else 0
    n, W = S.row_lengths[b], S.W
    for name, t in S.row(b).tensors[0].items():
        mine, theirs = t[0], C.row(b).tensors[0][name][0]
        if name.startswith("full"):
            mine, theirs = mine[:, : n - P], theirs[:, P:n]
        else:
            mine, theirs = mine[:, :W], theirs[:, :W]
        assert torch.equal(mine, theirs), f"row {b}: {name} differs from the control's"


# ---- 1. bit identity with a physical copy of the prompt -------------------------------------------------------------
CHUNKS = [5, 64, 127, 128, 129, 1000, 4096]


@pytest.mark.parametrize("sink,recent", [(16, 48), (64, 256), (1024, 1536)], ids=["w64", "w320", "w2560"])
@pytest.mark.parametrize("L", [256, 300, 4097])
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 8), (8, 8, 1), (8, 8, 8)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_sharer_chunks_are_bit_identical_to_a_copy(dtype, Hq, Hkv, n_full, L, sink, recent):
    """Rows: 0 the donor, 1 a fork of 0, 2 a fork of 1 made after row 1's first question.  Row 1 takes the chunks
    5 (17 at MHA: a decode-sized 5 is the batched step's), 127, 129, 4096 and row 2 takes 64, 128, 1000, with two
    batched decode steps before each later turn; the donor appends 200 tokens after the first fork.  The control cache
    holds the prompt in every row and gets the same calls."""
    G = Hq // Hkv
    lens = [17 if n * G <= 16 else n for n in CHUNKS]
    turns1, turns2 = lens[0::2], lens[1::2]
    steps = 2
    P = L // 128 * 128
    own = L - P + sum(lens) + 8 * steps + 16
    caps_s = [L + 200 + 8 * steps + 16, own, own]
    caps_c = [L + own] * 3
    mk = lambda caps: DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], 3, caps, sink, recent, dtype, DEV,
                                                     stage_cap=4096)
    S, C = mk(caps_s), mk(caps_c)
    g = torch.Generator().manual_seed(L + 17 * n_full + Hq + sink)
    width = (Hq + 2 * Hkv) * D
    x = lambda n, B=1: torch.randn(B, n, width, generator=g).to(dtype).to(DEV)

    for c0 in range(0, L, 4096):
        _attend([S.row(0), C.row(0), C.row(1), C.row(2)], x(min(4096, L - c0)), Hq)
    S.share_prefix(0, 1, own)
    assert S.row_prefix[1] == (0, P) and S.row_capacities[1] == P + own

    def turn(b, n, what):
        q = x(n)
        got, want = _attend([S.row(b), C.row(b)], q, Hq)
        assert torch.equal(got, want), f"{what}: row {b}, chunk of {n} after {S.row_lengths[b] - n} keys"
        return q

    q = turn(1, turns1[0], "first question")
    _attend([S.row(0), C.row(0)], x(200), Hq)  # the donor keeps appending past P after the fork
    S.share_prefix(1, 2, own)  # a fork of a sharer: the same donor prefix, row 1's own rows copied
    _attend([C.row(2)], q, Hq)
    assert S.row_prefix[2] == (0, P)
    for k in range(1, len(turns1)):
        for step in range(steps):
            d = x(1, 3)
            os_, oc = (torch.empty(3, 1, Hq, D, dtype=dtype, device=DEV) for _ in range(2))
            S.attend(0, d, None, None, _C.ROPE_NONE, os_)
            C.attend(0, d, None, None, _C.ROPE_NONE, oc)
            torch.testing.assert_close(os_.float(), oc.float(), **TOL[dtype], msg=lambda m: f"turn {k}: {m}")
        turn(1, turns1[k], f"turn {k}")
        turn(2, turns2[k - 1], f"turn {k}")
    torch.cuda.synchronize()
    assert S.row_lengths == C.row_lengths
    for b in range(3):
        _same_row_bytes(S, C, b)


# ---- 2. fp64 attention ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full,L,chunks", [
    (32, 8, 3, 700, [129, 40, 1000]),   # wgmma, mma.sync (160 packed rows), wgmma over several tiles
    (32, 8, 8, 4097, [300, 17]),
    (8, 8, 5, 300, [64, 256, 130]),     # MHA
])
def test_sharers_match_fp64_attention(Hq, Hkv, n_full, L, chunks, dtype):
    """Row 0 holds the prompt; rows 1.. are forks of it and each takes a question of its own length."""
    sink, recent = 16, 48
    G, B = Hq // Hkv, len(chunks) + 1
    own = max(chunks) + 128
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, [L + 64] + [own] * (B - 1), sink, recent, dtype, DEV,
                                       stage_cap=1024)
    g = torch.Generator().manual_seed(L + n_full)
    width = (Hq + 2 * Hkv) * D
    prompt = torch.randn(1, L, width, generator=g).to(dtype)
    for c0 in range(0, L, 1024):
        _attend([S.row(0)], prompt[:, c0 : c0 + 1024].to(DEV), Hq)
    q, k, v = split_qkv(prompt, Hq, Hkv)
    _, past = O.tuple_attention_core(q.double(), k.double(), v.double(), None, n_full, G, sink, recent)
    shadow = Fa2Shadow(n_full, G, sink, recent)
    shadow.step(q, k, v)
    for b in range(1, B):
        S.share_prefix(0, b, own)
    for b, n in enumerate(chunks, start=1):
        x = torch.randn(1, n, width, generator=g).to(dtype)
        (got,) = _attend([S.row(b)], x.to(DEV), Hq)
        q, k, v = split_qkv(x, Hq, Hkv)
        ref, _ = O.tuple_attention_core(q.double(), k.double(), v.double(), past, n_full, G, sink, recent)
        fa2, truth = copy.copy(shadow).step(q, k, v)
        assert_parity(got.float().cpu(), ref, f"row {b}: chunk of {n} after {L} shared keys", fa2=fa2, truth=truth)


# ---- 3. visibility and write census -----------------------------------------------------------------------------------
POISON = 127


@pytest.mark.parametrize("sink,recent", [(16, 48), (1024, 1536)], ids=["wgmma", "mma"])
def test_visibility_and_write_census(sink, recent):
    """Rows: 0 a donor of 300 keys (256 shared), 1 its fork, 2 a plain row of 500 keys.  Keys have logit 0; values are
    one-hot: dim 0 / 1 the donor's shared part / tail, 4 row 2's prompt, 5 what the donor appends after the fork, 10 + i
    the sharer's i-th chunk.  Every other row of the pool (region slack, headroom) lights POISON.  Chunks of 200 and then
    40 tokens (160 packed rows) take the wgmma and the mma.sync kernel, or both the mma.sync kernel when W > 2048.
    Retrieval q-heads are checked exactly; the write census checks that the sharer's chunks change nothing but its own
    rows [n - P, n - P + S) and its ring / staging slots."""
    Hq, Hkv, n_full, dtype = 32, 8, 4, torch.bfloat16
    G = Hq // Hkv
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], 3, [400, 300, 564], sink, recent, dtype, DEV,
                                       stage_cap=256, pool_size=4096)
    t = S.tensors[0]
    t["full_k"].zero_()
    t["full_v"].zero_()
    t["full_v"][:, POISON] = 1
    onehot = lambda n, dim: torch.nn.functional.one_hot(torch.full((n,), dim), D).to(dtype).to(DEV)
    for b, parts, n in ((0, [(0, 256, 0), (256, 300, 1)], 300), (2, [(0, 500, 4)], 500)):
        r = S.row(b)
        for lo, hi, dim in parts:
            r.tensors[0]["full_v"][0, :, lo:hi] = onehot(hi - lo, dim)
        r.kv_seq_len_list[0] = r.total_list[0] = n
        r.lo_list[0] = max(sink, n - recent)
    S.sync_device_state()
    S.share_prefix(0, 1, 300)
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(4)

    def chunk(n, dim):
        x = torch.zeros(1, n, width, dtype=dtype)
        x[..., : Hq * D] = torch.randn(1, n, Hq * D, generator=g).to(dtype)  # any q: every key has logit 0
        x[0, :, (Hq + Hkv) * D :].view(n, Hkv, D)[:, :, dim] = 1
        return x.to(DEV)

    _attend([S.row(0)], chunk(100, 5), Hq)  # the donor appends after the fork: rows [300, 400) must stay unseen
    first, cap = S._geom[1]
    seen = {0: 256, 1: 44}
    for i, n in enumerate((200, 40)):
        before = {k: v.clone() for k, v in S.tensors[0].items()}
        n0 = S.row_lengths[1]
        (out,) = _attend([S.row(1)], chunk(n, 10 + i), Hq)
        torch.cuda.synchronize()
        got = out[0, :, : n_full * G].double().cpu()  # the retrieval q-heads
        for tok in range(n):
            cnt = dict(seen)
            cnt[10 + i] = tok + 1
            exp = torch.zeros(D, dtype=torch.float64)
            for dim, c in cnt.items():
                exp[dim] = c / sum(cnt.values())
            lit = exp > 0
            row = got[tok]
            assert torch.all(row[:, ~lit] == 0), f"chunk {i} token {tok}: sees keys it must not"
            assert torch.all((row[:, lit] - exp[lit]).abs() <= exp[lit] * 2 ** -8), f"chunk {i} token {tok}"
        seen[10 + i] = n
        # write census: the pool changed only in the sharer's own rows [n0 - 256, n0 - 256 + n) of every head
        for name in ("full_k", "full_v"):
            changed = torch.zeros(t[name].shape[0], dtype=torch.bool, device=DEV)
            for h in range(n_full):
                base = first * n_full + h * cap + n0 - 256
                changed[base : base + n] = True
            diff = (S.tensors[0][name] != before[name]).any(-1)
            assert not diff[~changed].any(), f"chunk {i}: {name} changed outside the sharer's new rows"
        for name in ("ring_k", "ring_v"):
            diff = (S.tensors[0][name] != before[name]).any(-1)
            assert not diff[[0, 2]].any(), f"chunk {i}: {name} of another row changed"
    assert S.row_lengths == [400, 540, 500]


# ---- 4. model level ---------------------------------------------------------------------------------------------------
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])


def _models(seed, sink, recent):
    from transformers import LlamaConfig, LlamaForCausalLM

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                      intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                      attn_implementation="eager")
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    oracle = O.OracleModel(copy.deepcopy(model), GATES, sink, recent)
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda(), oracle


def test_model_questions_on_forks():
    """A 300-token prompt in row 0, forks 1 and 2 take questions of 9 and 700 tokens, then the three rows decode 8 greedy
    steps together: against a control whose rows prefilled prompt and question themselves (question logits
    bit-identical; in the steps, where the shared-prefix cascade and the control's launch round differently, logits
    within tolerance and the same greedy token wherever the control's top two logits are further apart than that),
    against OracleModel per row, and DuoDecodeGraph replay against eager.  Both caches are fed the sharers' tokens."""
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 12
    model, oracle = _models(31, sink, recent)
    g = torch.Generator().manual_seed(9)
    prompt, q1, q2 = (torch.randint(0, 512, (1, n), generator=g) for n in (300, 9, 700))
    questions = {1: q1, 2: q2}
    caps = [300 + 64, 800, 800]
    ce, cg = (DuoRaggedKVCache(model, GATES, 3, caps, sink, recent) for _ in range(2))
    C = DuoRaggedKVCache(model, GATES, 3, [300 + 800] * 3, sink, recent)
    run = lambda ids, past: model(input_ids=ids.cuda(), past_key_values=past, use_cache=True).logits
    with torch.no_grad():
        logits = {}
        for c in (ce, cg):
            logits[0] = run(prompt, c.row(0))
            c.share_prefix(0, 1, 800)
            c.share_prefix(0, 2, 800)
            for b, qb in questions.items():
                logits[b] = run(qb, c.row(b))
        assert ce.row_prefix == [None, (0, 256), (0, 256)]
        lo, past0 = oracle(prompt, None)
        pasts = [past0] * 3
        torch.testing.assert_close(logits[0].cpu(), lo, rtol=5e-2, atol=5e-2)
        for b in range(3):
            want = run(prompt, C.row(b))
            if b:
                want = run(questions[b], C.row(b))
                lo, pasts[b] = oracle(questions[b], pasts[b])
                torch.testing.assert_close(logits[b].cpu(), lo, rtol=5e-2, atol=5e-2)
            assert torch.equal(logits[b], want), f"row {b}: question logits differ from the control's"
        tok = torch.cat([logits[b][:, -1:].argmax(-1) for b in range(3)], 0)
        graph = DuoDecodeGraph(model, cg)
        te = tok.clone()
        for step in range(8):
            le = run(te, ce)
            lg = graph.step(te)
            lc = run(te, C)
            assert torch.equal(le, lg), f"step {step}: graph replay differs from eager decode"
            torch.testing.assert_close(le.float(), lc.float(), rtol=5e-2, atol=5e-2)
            for b in range(3):
                lo, pasts[b] = oracle(te[b : b + 1].cpu(), pasts[b])
                torch.testing.assert_close(le[b : b + 1].cpu(), lo, rtol=5e-2, atol=5e-2)
            top2 = lc.float().topk(2, -1).values
            clear = top2[..., 0] - top2[..., 1] > 0.1
            assert torch.equal(le.argmax(-1)[clear], lc.argmax(-1)[clear]), f"step {step}: greedy tokens differ"
            te = le.argmax(-1)
    assert ce.row_lengths == C.row_lengths == [308, 317, 1008]


# ---- 5. refusals --------------------------------------------------------------------------------------------------
def _cache_bytes(c):
    return [{k: v.clone() for k, v in t.items()} for t in c.tensors]


def test_refusals_leave_the_cache_unchanged():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 12
    model, _ = _models(33, sink, recent)
    c = DuoRaggedKVCache(model, GATES, 3, [400, 400, 64], sink, recent)
    run = lambda n, b: model(input_ids=torch.randint(0, 512, (1, n)).cuda(), past_key_values=c.row(b), use_cache=True)
    with torch.no_grad():
        run(300, 0)
        run(5, 2)
        c.share_prefix(0, 1, 400)  # row 1: 300 keys, 256 of them shared, room for 356 more; staging of 300 rows

        def snapshot():
            torch.cuda.synchronize()
            return (_cache_bytes(c), c.row_state.clone(), c.row_geom.clone(), c.row_share.clone(), c.row_prefix,
                    c.row_capacities, c.row_lengths, c.launch_count, c.stage_cap_list)

        def unchanged(before):
            now = snapshot()
            for t0, t1 in zip(before[0], now[0]):
                for k in t0:
                    assert torch.equal(t0[k], t1[k]), k
            for a, b in zip(before[1:4], now[1:4]):
                assert torch.equal(a, b)
            assert before[4:] == now[4:]

        width = (model.config.num_attention_heads + 2 * model.config.num_key_value_heads) * D
        qkv = torch.zeros(1, 40, width, dtype=torch.bfloat16, device=DEV)
        out = torch.empty(1, 40, model.config.num_attention_heads, D, dtype=torch.bfloat16, device=DEV)
        before = snapshot()
        for call, match in ((lambda: run(1, 1), "batched step"),
                            (lambda: run(8, 1), "batched step"),  # group 2 x 8 tokens = 16 rows
                            (lambda: c.row(1).attend(0, qkv, None, None, _C.ROPE_NONE, out, force_mma=True),
                             "force_mma"),
                            (lambda: run(357, 1), "Trying to put 357 KVs")):
            with pytest.raises(ValueError, match=match):
                call()
            unchanged(before)
        DuoDecodeGraph(model, c)
        before = snapshot()
        with pytest.raises(ValueError, match="captured in a DuoDecodeGraph"):
            run(320, 1)  # > the staging capacity of 300 (the prompt's chunk): the staging area would have to grow
        unchanged(before)
