"""Ragged batches with per-row capacities on the GPU: duo_decode_ragged_pooled through DuoRaggedKVCache /
DuoRaggedINT4KVCache built with a sequence of capacities, the patched model and DuoDecodeGraph.

* bit-identity with the uniform-capacity ragged launch at the same lengths and K/V (16-bit and INT4, bf16 and fp16);
* per-row oracle parity and batch-1 cache identity, and no row writing outside its region;
* full size: a 1M-token region next to short ones;
* model level (including a row resized and refilled), graph replay across resize_row, and the error paths.
"""
import copy

import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache, DuoRaggedINT4KVCache, DuoRaggedKVCache, ragged_partition
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
HEADS = pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 4), (32, 8, 8), (8, 8, 3)])


def split_qkv(qkv, Hq, Hkv):
    B, S, _ = qkv.shape
    return (qkv[..., : Hq * D].reshape(B, S, Hq, D), qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D),
            qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D))


def prefill(caches, b, L, width, dtype, Hq, g):
    for c0 in range(0, L, 4096):
        S = min(4096, L - c0)
        qkv = torch.randn(1, S, width, generator=g).to(dtype).to(DEV)
        for c in caches:
            c.row(b).attend(0, qkv, None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))


def assert_row_equal(P, U, b):
    """Row b's retrieval rows in use, sink and ring slots: pooled cache P against uniform cache U."""
    n, W = P.row_lengths[b], P.W
    for name, t in P.row(b).tensors[0].items():
        mine, theirs = t[0], U.tensors[0][name][b]
        if name.startswith("full"):
            mine, theirs = mine[:, :n], theirs[:, :n]
        else:
            mine, theirs = mine[:, :W], theirs[:, :W]
        assert torch.equal(mine, theirs), f"row {b}: {name} differs from the uniform-capacity cache"


def assert_pool_untouched_outside_rows(P):
    """Pool rows no row holds a token in are still zero: no row wrote into a neighbour's region or the headroom."""
    for l, t in enumerate(P.tensors):
        nf = P.num_full_kv_head_list[l]
        for name, v in t.items():
            if not name.startswith("full") or nf == 0:
                continue
            used = torch.zeros(v.shape[0], dtype=torch.bool, device=DEV)
            for b, (first, cap) in enumerate(P._geom):
                n = P.row(b).kv_seq_len_list[l]
                idx = first * nf + torch.arange(nf, device=DEV)[:, None] * cap + torch.arange(n, device=DEV)[None]
                used[idx.flatten()] = True
            assert not v[~used].any(), f"layer {l}: {name} has bytes outside the rows' tokens"


# ---- 1. bit-identity with the uniform-capacity ragged launch -------------------------------------------------------
def _bit_identity(cls, lengths, steps, Hq, Hkv, n_full, dtype, seed):
    sink, recent, B = 16, 48, len(lengths)
    grow = sum(steps)
    # rows 0 and 3 end exactly at their capacity, the others keep room; all capacities differ
    caps = [L + grow if b in (0, 3) else L + grow + 37 * (b + 1) for b, L in enumerate(lengths)]
    U = cls.from_geometry(1, Hq, Hkv, D, [n_full], B, max(caps), sink, recent, dtype, DEV, stage_cap=64)
    P = cls.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64)
    assert P.row_capacities == caps and [r.max_size for r in P.rows] == caps
    g = torch.Generator().manual_seed(seed)
    width = (Hq + 2 * Hkv) * D
    for b, L in enumerate(lengths):
        prefill((U, P), b, L, width, dtype, Hq, g)
    for step, S in enumerate(steps):
        qkv = torch.randn(B, S, width, generator=g).to(dtype).to(DEV)
        ou, op = (torch.empty(B, S, Hq, D, dtype=dtype, device=DEV) for _ in range(2))
        U.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, ou)
        P.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, op)
        assert torch.equal(ou, op), f"step {step}: pooled output differs from the uniform-capacity launch"
    torch.cuda.synchronize()
    assert P.row_lengths == U.row_lengths
    assert [P.row_lengths[b] for b in (0, 3)] == [caps[0], caps[3]]  # filled exactly to capacity
    for b in range(B):
        assert_row_equal(P, U, b)
    assert_pool_untouched_outside_rows(P)


@DTYPES
@HEADS
def test_pooled_bit_identical_to_uniform_ragged(Hq, Hkv, n_full, dtype):
    _bit_identity(DuoRaggedKVCache, [0, 1, 63, 129, 320, 4097, 9000], [1, 2, 1, 3, 1, 1], Hq, Hkv, n_full, dtype,
                  11 * n_full + Hq)


@DTYPES
@HEADS
def test_pooled_int4_bit_identical_to_uniform_ragged(Hq, Hkv, n_full, dtype):
    _bit_identity(DuoRaggedINT4KVCache, [1, 64, 127, 129, 1500, 5000], [1, 2, 1, 2, 1], Hq, Hkv, n_full, dtype,
                  13 * n_full + Hq)


# ---- 2. per-row oracle parity, batch-1 cache identity, per-row eviction --------------------------------------------
LENGTHS = [0, 1, 63, 129, 320, 4097, 20000]


@DTYPES
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 4), (8, 8, 3)])
def test_pooled_rows_match_oracle_and_batch1_caches(Hq, Hkv, n_full, dtype):
    sink, recent = 16, 48
    B = len(LENGTHS)
    caps = [L + 16 + 50 * b for b, L in enumerate(LENGTHS)]
    g = torch.Generator().manual_seed(7 * n_full + Hq)
    R = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64)
    singles = [DuoKVCache(1, Hq, Hkv, D, [n_full], 1, caps[b], sink, recent, dtype, DEV, stage_cap=64) for b in range(B)]
    width = (Hq + 2 * Hkv) * D
    pasts = []
    for b, L in enumerate(LENGTHS):
        ks, vs = [], []
        for c0 in range(0, L, 4096):
            S = min(4096, L - c0)
            qkv = torch.randn(1, S, width, generator=g).to(dtype)
            for cache in (R.row(b), singles[b]):
                cache.attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))
            _, k, v = split_qkv(qkv, Hq, Hkv)
            ks.append(k)
            vs.append(v)
        if L:
            k, v = torch.cat(ks, 1), torch.cat(vs, 1)
            fk, fv, sk, sv = k[:, :, :n_full], v[:, :, :n_full], k[:, :, n_full:], v[:, :, n_full:]
            if sk.shape[1] > sink + recent:
                sk, sv = (torch.cat([t[:, :sink], t[:, -recent:]], 1) for t in (sk, sv))
            pasts.append((torch.cat([fk, fv], 0).transpose(1, 2).contiguous(),
                          torch.cat([sk, sv], 0).transpose(1, 2).contiguous()))
        else:
            pasts.append(None)
    for step, S in enumerate([1, 1, 2, 1, 1, 1, 3, 1]):
        qkv = torch.randn(B, S, width, generator=g).to(dtype)
        out = torch.empty(B, S, Hq, D, dtype=dtype, device=DEV)
        R.attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, out)
        got = out.float().cpu()
        for b in range(B):
            singles[b].attend(0, qkv[b : b + 1].to(DEV), None, None, _C.ROPE_NONE,
                              torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))
            q, k, v = split_qkv(qkv[b : b + 1], Hq, Hkv)
            ref, pasts[b] = O.tuple_attention_core(q, k, v, pasts[b], n_full, Hq // Hkv, sink, recent)
            assert_parity(got[b : b + 1], ref, f"step {step} row {b}")
        if step == 2:
            for b, n in ((2, 2), (5, 1)):
                R.row(b).evict_last(n)
                singles[b].evict_last(n)
                pasts[b] = tuple(t[:, :, : t.shape[2] - n].contiguous() for t in pasts[b])
    torch.cuda.synchronize()
    W = R.W
    for b in range(B):
        n = R.row_lengths[b]
        assert n == singles[b].kv_seq_len
        for name, t in R.row(b).tensors[0].items():
            mine, theirs = t[0], singles[b].tensors[0][name][0]
            mine, theirs = (mine[:, :n], theirs[:, :n]) if name.startswith("full") else (mine[:, :W], theirs[:, :W])
            assert torch.equal(mine, theirs), f"row {b}: {name} differs from the batch-1 cache"
    assert_pool_untouched_outside_rows(R)  # (the evicted rows were written again by the later steps)


# ---- 3. full size -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", [DuoRaggedKVCache, DuoRaggedINT4KVCache], ids=["bf16", "int4"])
def test_full_size_pooled_region_next_to_short_rows(cls):
    """A 1,048,576-token region next to short ones.  The uniform-capacity cache gives the expected bits (same K/V,
    same lengths); one-hot keys at the long row's tile, split and region boundaries; memory ~ the sum of capacities."""
    N = 1048576
    Hq, Hkv, n_full, sink, recent = 32, 8, 4, 64, 256
    lengths = [N - 8, 100, 5000, 1]
    caps = [N, 300, 5200, 200]
    B = len(lengths)
    dtype = torch.bfloat16
    P = cls.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV)
    U = cls.from_geometry(1, Hq, Hkv, D, [n_full], B, N, sink, recent, dtype, DEV)
    per_tok = (2 * D * 2) if cls is DuoRaggedKVCache else 2 * (D // 2 + 4)
    assert P.memory_usage < (sum(caps) + 4 * 128) * n_full * per_tok + U.memory_usage // 20
    assert U.memory_usage > B * N * n_full * per_tok
    g = torch.Generator(device=DEV).manual_seed(3)
    for name, t in U.tensors[0].items():
        if t.dtype == torch.uint8:
            t.random_(0, 256, generator=g)
        elif name.endswith("_scale"):
            t.uniform_(0.002, 0.02, generator=g)
        elif name.endswith("_zero"):
            t.uniform_(-0.1, 0.1, generator=g)
        else:
            t.normal_(generator=g)
    for b in range(B):
        for name, t in P.row(b).tensors[0].items():
            n = caps[b] if name.startswith("full") else t.shape[2]
            t[0, :, :n].copy_(U.tensors[0][name][b, :, :n])
    qkv = (torch.randn(B, 1, (Hq + 2 * Hkv) * D, generator=g, device=DEV) * 0.5).to(dtype)
    for c in (P, U):
        for r, L in zip(c.rows, lengths):
            r.kv_seq_len_list[0], r.total_list[0], r.lo_list[0] = L, L, max(sink, L - recent)

    def decode(c, x):
        out = torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV)
        saved = [(list(r.kv_seq_len_list), list(r.total_list), list(r.lo_list)) for r in c.rows]
        c.attend(0, x.clone(), None, None, _C.ROPE_NONE, out)
        for r, s in zip(c.rows, saved):  # every call attends the same lengths
            r.kv_seq_len_list[:], r.total_list[:], r.lo_list[:] = s
        return out

    assert torch.equal(decode(P, qkv), decode(U, qkv))
    if cls is DuoRaggedKVCache:
        policy = {}
    else:
        from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY as policy
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    kps = ragged_partition([L + (0 if cls is DuoRaggedKVCache else 1) for L in lengths], n_full, Hkv - n_full, sms,
                           **policy)["keys_per_split"]
    assert kps < N
    if cls is DuoRaggedKVCache:
        kvh = 3  # last retrieval head of the long row: its keys end at the region's last token
        t = P.row(0).tensors[0]
        qrow = qkv[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D].float()
        for pos in sorted({0, 63, 64, kps - 1, kps, 2 * kps, N // 2 + 17, N - 9}):
            saved = t["full_k"][0, kvh, pos].clone()
            t["full_k"][0, kvh, pos] = (qrow / qrow.norm() * 40.0).to(dtype)
            o = decode(P, qkv).float()
            torch.testing.assert_close(o[0, 0, kvh * 4], t["full_v"][0, kvh, pos].float(), rtol=1e-2, atol=1e-3)
            t["full_k"][0, kvh, pos] = saved
        # the neighbour's first key (the row after the long one starts right at its region's end)
        t1 = P.row(1).tensors[0]
        q1 = qkv[1, 0, 0:D].float()
        t1["full_k"][0, 0, 0] = (q1 / q1.norm() * 40.0).to(dtype)
        o = decode(P, qkv).float()
        torch.testing.assert_close(o[1, 0, 0], t1["full_v"][0, 0, 0].float(), rtol=1e-2, atol=1e-3)
    # the new token went to each row's own region, right after its keys
    for b, L in enumerate(lengths):
        assert torch.equal(P.row(b).tensors[0]["full_v"][0, :, L], U.tensors[0]["full_v"][b, :, L])


# ---- 4. model level -------------------------------------------------------------------------------------------------
def tiny_model(kind, seed=0):
    torch.manual_seed(seed)
    if kind == "llama":
        from transformers import LlamaConfig, LlamaForCausalLM as M

        cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                          intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                          attn_implementation="eager")
    else:
        from transformers import MistralConfig, MistralForCausalLM as M

        cfg = MistralConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                            intermediate_size=1024, vocab_size=512, head_dim=128, max_position_embeddings=8192,
                            rope_theta=10000.0, sliding_window=None, attn_implementation="eager")
    return M(cfg).to(torch.bfloat16).eval()


GATES = np.array([[0.9, 0.1], [0.2, 0.8]])


def _patched(kind, seed, sink, recent):
    from duo_attn.patch import enable_duo_attention_eval

    model = tiny_model(kind, seed)
    oracle = O.OracleModel(copy.deepcopy(model), GATES, sink, recent)
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda(), oracle


@pytest.mark.parametrize("kind", ["llama", "mistral"])
def test_model_pooled_decode_matches_oracle_per_row(kind):
    sink, recent = 4, 12
    model, oracle = _patched(kind, 11, sink, recent)
    cache = DuoRaggedKVCache(model, GATES, 3, [60, 150, 20], sink, recent, pool_size=1024)
    g = torch.Generator().manual_seed(5)
    pasts, toks = [None] * 3, [None] * 3
    tol = dict(rtol=5e-2, atol=5e-2)

    def prefill(b, n):
        ids = torch.randint(0, 512, (1, n), generator=g)
        lo, pasts[b] = oracle(ids, None)
        out = model(input_ids=ids.cuda(), past_key_values=cache.row(b), use_cache=True)
        torch.testing.assert_close(out.logits.cpu(), lo, **tol)
        toks[b] = lo.argmax(-1)

    with torch.no_grad():
        for b, n in enumerate([45, 130, 7]):
            prefill(b, n)
        for step in range(10):
            out = model(input_ids=torch.cat(toks, 0).cuda(), past_key_values=cache, use_cache=True)
            assert out.logits.shape == (3, 1, 512)
            for b in range(3):
                lo, pasts[b] = oracle(toks[b], pasts[b])
                torch.testing.assert_close(out.logits[b : b + 1].cpu(), lo, **tol)
                toks[b] = lo.argmax(-1)
            if step == 4:  # row 2 finished; a longer request takes its place in a larger region
                cache.row(2).clear()
                cache.resize_row(2, 400)
                assert cache.row_capacities == [60, 150, 400] and cache.row(2).max_size == 400
                prefill(2, 300)
            assert cache.row_lengths == [p[0][0].shape[2] for p in pasts]
    assert_pool_untouched_outside_rows(cache)


# ---- 5. graph replay across resize_row ----------------------------------------------------------------------------
def test_graph_replay_across_resize_matches_eager():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 6
    model, _ = _patched("llama", 13, sink, recent)
    ca = DuoRaggedKVCache(model, GATES, 3, [64, 40, 100], sink, recent, pool_size=1024)
    cb = DuoRaggedKVCache(model, GATES, 3, [64, 40, 100], sink, recent, pool_size=1024)
    g = torch.Generator().manual_seed(6)

    def prefill(b, ids):
        for c in (ca, cb):
            model(input_ids=ids.cuda(), past_key_values=c.row(b), use_cache=True)

    with torch.no_grad():
        for b, n in enumerate([37, 9, 70]):
            prefill(b, torch.randint(0, 512, (1, n), generator=g))
        graph = DuoDecodeGraph(model, cb)
        captured = graph.graph
        tok = torch.randint(0, 512, (3, 1), generator=g).cuda()
        for step in range(16):
            le = model(input_ids=tok, past_key_values=ca, use_cache=True).logits
            lg = graph.step(tok)
            assert torch.equal(le, lg), f"step {step}: graph replay differs from eager pooled decode"
            tok = le.argmax(-1)
            if step == 5:  # row 1 finished: a larger request moves into the headroom, no re-capture
                ids = torch.randint(0, 512, (1, 60), generator=g)  # <= the staging capacity: no re-allocation
                for c in (ca, cb):
                    c.row(1).clear()
                    c.resize_row(1, 300)
                assert cb._geom[1][0] >= 256 and cb.row_capacities[1] == 300
                prefill(1, ids)
            assert ca.row_lengths == cb.row_lengths
        assert graph.graph is captured
        assert torch.equal(ca.row_state, cb.row_state) and torch.equal(ca.row_geom, cb.row_geom)


# ---- 6. error paths ----------------------------------------------------------------------------------------------
def test_errors_overflow_resize_and_empty_int4_row():
    sink, recent = 4, 12
    model, _ = _patched("llama", 17, sink, recent)
    cache = DuoRaggedKVCache(model, GATES, 2, [50, 300], sink, recent)
    with torch.no_grad():
        model(input_ids=torch.zeros(1, 49, dtype=torch.long).cuda(), past_key_values=cache.row(0), use_cache=True)
        model(input_ids=torch.zeros(1, 5, dtype=torch.long).cuda(), past_key_values=cache.row(1), use_cache=True)
        model(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [50, 6]
        with pytest.raises(ValueError, match=r"Trying to put 1 KVs into a cache with max size 50, current size: 50\."):
            model(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [50, 6]  # nothing was appended to either row
        with pytest.raises(ValueError, match="max size 50"):
            model(input_ids=torch.zeros(1, 2, dtype=torch.long).cuda(), past_key_values=cache.row(0), use_cache=True)
        # row 1 keeps its own, larger capacity
        model(input_ids=torch.zeros(1, 290, dtype=torch.long).cuda(), past_key_values=cache.row(1), use_cache=True)
        assert cache.row_lengths == [50, 296]
        with pytest.raises(ValueError, match="row 0 is not empty"):
            cache.resize_row(0, 64)
        cache.row(0).clear()
        with pytest.raises(ValueError, match="no free range"):  # the pool holds 128 + 384 tokens, row 1 keeps 384
            cache.resize_row(0, 200)
        cache.resize_row(0, 100)  # fits its old region
        assert cache.row_capacities == [100, 300]
    ci = DuoRaggedINT4KVCache.from_geometry(1, 8, 2, D, [1], 2, [256, 512], sink, recent, torch.float16, DEV)
    x = torch.randn(1, 20, 12 * D, dtype=torch.float16, device=DEV)
    ci.row(0).attend(0, x, None, None, _C.ROPE_NONE, torch.empty(1, 20, 8, D, dtype=torch.float16, device=DEV))
    with pytest.raises(ValueError, match="row 1 is empty"):
        ci.attend(0, torch.randn(2, 1, 12 * D, dtype=torch.float16, device=DEV), None, None, _C.ROPE_NONE,
                  torch.empty(2, 1, 8, D, dtype=torch.float16, device=DEV))
