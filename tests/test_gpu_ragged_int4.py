"""Ragged batches on the INT4 KV cache: duo_decode_ragged_int4 through DuoRaggedINT4KVCache, the patched model and
DuoDecodeGraph, for fp16 and bf16 activations.

* kernel parity: rows at different lengths decoded in one launch, every row against the INT4 oracle run on that row
  alone, and every row's codes / scales / zeros against a batch-1 INT4 cache that ran the same schedule;
* equal lengths: bit-identical to duo_decode_fused on a batch-4 INT4 cache;
* full size: one long row (128K / 1M) next to short rows, size-independent properties of the dequantised values;
* model level, graph replay, the error paths and the shared 16-bit scratch.
"""
import copy

import numpy as np
import pytest
import torch

import int4_bf16_oracle as H
from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY, DuoKVCache, DuoRaggedINT4KVCache, ragged_partition
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


def split_qkv(qkv, Hq, Hkv):
    B, S, _ = qkv.shape
    return (qkv[..., : Hq * D].reshape(B, S, Hq, D), qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D),
            qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D))


def int4_core(dtype):
    return O.int4_attention_core if dtype == torch.float16 else H.int4_attention_core


def oracle_past(k, v, n_full, sink, recent):
    """The INT4 oracle's tuple cache after all of k / v ([1, N, Hkv, D]): the K1 -> K2 round trip of every retrieval
    token, of the sinks and of the last ``recent`` streaming tokens."""
    k, v = H.int4_roundtrip(k), H.int4_roundtrip(v)
    fk, fv, sk, sv = k[:, :, :n_full], v[:, :, :n_full], k[:, :, n_full:], v[:, :, n_full:]
    if sk.shape[1] > sink + recent:
        sk, sv = (torch.cat([t[:, :sink], t[:, -recent:]], 1) for t in (sk, sv))
    return (torch.cat([fk, fv], 0).transpose(1, 2).contiguous(), torch.cat([sk, sv], 0).transpose(1, 2).contiguous())


def evict_past(past, n):
    return tuple(t[:, :, : t.shape[2] - n].contiguous() for t in past)


def assert_same_cache(ragged, b, single):
    """Codes, scales and zeros of the retrieval rows and of the sink + ring slots (the staging area behind the ring
    is per-call scratch)."""
    W = ragged.W
    for name, t in ragged.tensors[0].items():
        mine, theirs = t[b], single.tensors[0][name][0]
        if name.startswith("ring"):
            mine, theirs = mine[:, :W], theirs[:, :W]
        assert torch.equal(mine, theirs), f"row {b}: {name} differs from the batch-1 INT4 cache"


def dequant(packed, scale, zero):
    """float32 values of stored INT4 rows: code * scale + zero (element 2i is the high nibble of byte i)."""
    codes = torch.stack([(packed >> 4), (packed & 15)], -1).flatten(-2).float()
    return codes * scale.float()[..., None] + zero.float()[..., None]


def pack(codes):
    """[..., 128] codes 0..15 -> [..., 64] packed bytes."""
    c = codes.to(torch.uint8)
    return (c[..., 0::2] << 4) | c[..., 1::2]


LENGTHS = [1, 63, 129, 320, 4097, 20000]
G4_STEPS, MHA_STEPS = [1, 1, 2, 1, 1, 1, 2, 1], [1, 1, 8, 1, 1, 1, 3, 1]


@DTYPES
@pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 4), (32, 8, 8), (8, 8, 3)])
def test_ragged_int4_rows_match_oracle_and_batch1_caches(Hq, Hkv, n_full, dtype):
    sink, recent = 16, 48
    B = len(LENGTHS)
    g = torch.Generator().manual_seed(7 * n_full + Hq + (dtype == torch.float16))
    cap = max(LENGTHS) + 32
    R = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, cap, sink, recent, dtype, DEV, stage_cap=64)
    singles = [DuoKVCache(1, Hq, Hkv, D, [n_full], 1, cap, sink, recent, dtype, DEV, stage_cap=64, kv_format="int4")
               for _ in range(B)]
    width = (Hq + 2 * Hkv) * D
    pasts = []
    for b, L in enumerate(LENGTHS):  # prefill through the batch-1 views: a raw first chunk, then chunks >= 128 tokens
        ks, vs = [], []
        for c0 in range(0, L, 4096):
            S = min(4096, L - c0)
            qkv = torch.randn(1, S, width, generator=g).to(dtype)
            for cache in (R.row(b), singles[b]):
                out = torch.empty(1, S, Hq, D, dtype=dtype, device=DEV)
                cache.attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, out)
            _, k, v = split_qkv(qkv, Hq, Hkv)
            ks.append(k)
            vs.append(v)
        pasts.append(oracle_past(torch.cat(ks, 1), torch.cat(vs, 1), n_full, sink, recent))
    assert R.row_lengths == LENGTHS
    core = int4_core(dtype)
    for step, S in enumerate(MHA_STEPS if Hq == Hkv else G4_STEPS):
        qkv = torch.randn(B, S, width, generator=g).to(dtype)
        out = torch.empty(B, S, Hq, D, dtype=dtype, device=DEV)
        launches = R.launch_count
        R.attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, out)
        assert R.launch_count == launches + 1  # one launch for the whole batch
        got = out.float().cpu()
        for b in range(B):
            o1 = torch.empty(1, S, Hq, D, dtype=dtype, device=DEV)
            singles[b].attend(0, qkv[b : b + 1].to(DEV), None, None, _C.ROPE_NONE, o1)
            q, k, v = split_qkv(qkv[b : b + 1], Hq, Hkv)
            ref, pasts[b] = core(q, k, v, pasts[b], n_full, Hq // Hkv, sink, recent)
            assert_parity(got[b : b + 1], ref.float(), f"step {step} row {b} (len {R.row_lengths[b] - S})")
        if step == 2:  # per-row eviction: rows 2 and 5 drop their newest tokens
            for b, n in ((2, 2), (5, 1)):
                R.row(b).evict_last(n)
                singles[b].evict_last(n)
                pasts[b] = evict_past(pasts[b], n)
        if step == 5:  # eviction of every row
            R.evict_last(1)
            for b in range(B):
                singles[b].evict_last(1)
                pasts[b] = evict_past(pasts[b], 1)
        assert R.row_lengths == [c.kv_seq_len for c in singles]
    torch.cuda.synchronize()
    for b in range(B):
        assert_same_cache(R, b, singles[b])


def _random_int4(t, g):
    """Random codes; K scale / zero keep |k| <= 0.375, V's keep v in [-1, 0.875]."""
    for name in ("full_k", "full_v", "ring_k", "ring_v"):
        t[name].copy_(torch.randint(0, 256, t[name].shape, generator=g, device=DEV, dtype=torch.uint8))
        t[name + "_scale"].fill_(0.05 if name.endswith("k") else 0.125)
        t[name + "_zero"].fill_(-0.375 if name.endswith("k") else -1.0)


@DTYPES
@pytest.mark.parametrize("Hq,Hkv,n_full,rope", [(32, 8, 4, _C.ROPE_HF), (32, 8, 1, _C.ROPE_FP32), (8, 8, 3, _C.ROPE_HF),
                                                (32, 8, 8, _C.ROPE_NONE)])
@pytest.mark.parametrize("L", [300, 5000, 70000])
def test_equal_lengths_bit_identical_to_decode_fused(Hq, Hkv, n_full, rope, L, dtype):
    sink, recent, B = 16, 48, 4
    g = torch.Generator(device=DEV).manual_seed(L + n_full)
    F = DuoKVCache(1, Hq, Hkv, D, [n_full], B, L + 32, sink, recent, dtype, DEV, kv_format="int4")
    R = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, L + 32, sink, recent, dtype, DEV)
    _random_int4(F.tensors[0], g)
    for name, t in F.tensors[0].items():
        R.tensors[0][name].copy_(t)
    F.kv_seq_len_list[0], F.total_list[0], F.lo_list[0] = L, L, L - recent
    for r in R.rows:
        r.kv_seq_len_list[0], r.total_list[0], r.lo_list[0] = L, L, L - recent
    width = (Hq + 2 * Hkv) * D
    tdt = torch.float32 if rope == _C.ROPE_FP32 else dtype
    G = Hq // Hkv
    for step, S in enumerate([1, 1, 8 // G, 1, 2]):
        qkv = torch.randn(B, S, width, generator=g, device=DEV).to(dtype)
        cos = sin = cb = sb = None
        if rope != _C.ROPE_NONE:
            cos, sin = (torch.rand(S, D, generator=g, device=DEV).to(tdt) for _ in range(2))
            cb, sb = cos[None].repeat(B, 1, 1).contiguous(), sin[None].repeat(B, 1, 1).contiguous()
        of = torch.empty(B, S, Hq, D, dtype=dtype, device=DEV)
        orr = torch.empty_like(of)
        F.attend(0, qkv.clone(), cos, sin, rope, of)
        R.attend(0, qkv.clone(), cb, sb, rope, orr)
        assert torch.equal(of, orr), f"step {step}: output differs from duo_decode_fused"
    torch.cuda.synchronize()
    for name, t in F.tensors[0].items():
        assert torch.equal(t, R.tensors[0][name]), f"{name} differs from duo_decode_fused's cache"


@DTYPES
@pytest.mark.parametrize("N", [131072, 1048576])
def test_full_size_skewed_int4_decode_properties(N, dtype):
    """One long row next to short ones, properties that hold at any size: constant V, q = 0 (uniform attention over
    the dequantised V), one-hot keys at the long row's split boundaries."""
    Hq, Hkv, n_full, sink, recent = 32, 8, 4, 64, 256
    lengths = [N, 100, 5000, 1]
    B = len(lengths)
    R = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, N + 8, sink, recent, dtype, DEV)
    t = R.tensors[0]
    g = torch.Generator(device=DEV).manual_seed(3)
    _random_int4(t, g)
    qkv = torch.randn(B, 1, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    out = torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV)

    def decode(x):
        for r, L in zip(R.rows, lengths):
            r.kv_seq_len_list[0], r.total_list[0], r.lo_list[0] = L, L, max(sink, L - recent)
        R.attend(0, x.clone(), None, None, _C.ROPE_NONE, out)
        return out.float()

    # (1) every V row holds c = 0.125 * (d % 16) - 1 (exact in INT4, and K1 of c gives it back) -> every output is c
    pattern = torch.arange(D, device=DEV) % 16
    c = (0.125 * pattern - 1.0).to(dtype)
    for name in ("full_v", "ring_v"):
        t[name][:] = pack(pattern)
    xc = qkv.clone()
    xc[..., (Hq + Hkv) * D :] = c.repeat(Hkv)
    o = decode(xc)
    torch.testing.assert_close(o, c.float().expand_as(o), rtol=1e-2, atol=1e-3)
    # (2) q == 0 -> the mean of each row's visible dequantised V (the new token's after its K1 round trip)
    for name in ("full_v", "ring_v"):
        t[name].copy_(torch.randint(0, 256, t[name].shape, generator=g, device=DEV, dtype=torch.uint8))
    xz = qkv.clone()
    xz[..., : Hq * D] = 0
    vnew = H.int4_roundtrip(xz[:, 0, (Hq + Hkv) * D :].view(B, Hkv, D).cpu()).float().to(DEV)
    means = []
    for b, L in enumerate(lengths):
        live = [p for p in range(L) if p < sink or p >= max(sink, L - recent)]
        slots = torch.tensor([p if p < sink else sink + (p - sink) % recent for p in live], device=DEV, dtype=torch.long)
        row = []
        for kvh in range(Hkv):
            if kvh < n_full:
                v = dequant(t["full_v"][b, kvh, :L], t["full_v_scale"][b, kvh, :L], t["full_v_zero"][b, kvh, :L])
            else:
                h = kvh - n_full
                v = dequant(t["ring_v"][b, h][slots], t["ring_v_scale"][b, h][slots], t["ring_v_zero"][b, h][slots])
            row.append((v.sum(0) + vnew[b, kvh]) / (v.shape[0] + 1))
        means.append(row)
    o = decode(xz)
    for b in range(B):
        for h in range(Hq):
            torch.testing.assert_close(o[b, 0, h], means[b][h // 4], rtol=1e-2, atol=2e-3)
    # (3) one key with an overwhelming logit in the long row, at the split boundaries of the host twin's partition
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    kps = ragged_partition([L + 1 for L in lengths], n_full, Hkv - n_full, sms, **INT4_RAGGED_POLICY)["keys_per_split"]
    assert kps < N
    kvh = 1
    qrow = qkv[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D].float()
    for pos in sorted({0, kps - 1, kps, 2 * kps, N // 2 + 17, N - 1}):
        saved = [t[n][0, kvh, pos].clone() for n in ("full_k", "full_k_scale", "full_k_zero")]
        t["full_k"][0, kvh, pos] = pack(torch.where(qrow > 0, 15, 0))  # k = +-7.5 along the signs of q
        t["full_k_scale"][0, kvh, pos] = 1.0
        t["full_k_zero"][0, kvh, pos] = -7.5
        o = decode(qkv)
        want = dequant(t["full_v"][0, kvh, pos], t["full_v_scale"][0, kvh, pos], t["full_v_zero"][0, kvh, pos])
        torch.testing.assert_close(o[0, 0, kvh * 4], want, rtol=1e-2, atol=1e-2)
        for n, s in zip(("full_k", "full_k_scale", "full_k_zero"), saved):
            t[n][0, kvh, pos] = s


# ---- model level ---------------------------------------------------------------------------------------------------
def tiny_model(kind, seed, dtype):
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
    return M(cfg).to(dtype).eval()


GATES = np.array([[0.9, 0.1], [0.2, 0.8]])


def _patched(kind, seed, sink, recent, dtype=torch.bfloat16):
    from duo_attn.patch import enable_duo_attention_eval

    model = tiny_model(kind, seed, dtype)
    oracle = O.OracleModel(copy.deepcopy(model), GATES, sink, recent, kv_format="int4")
    oracle.core = int4_core(dtype)
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda(), oracle


@pytest.mark.parametrize("kind,dtype", [("llama", torch.bfloat16), ("mistral", torch.float16)])
def test_model_ragged_int4_decode_matches_oracle_per_row(kind, dtype):
    sink, recent = 4, 12
    model, oracle = _patched(kind, 11, sink, recent, dtype)
    cache = DuoRaggedINT4KVCache(model, GATES, 3, 256, sink, recent)
    g = torch.Generator().manual_seed(5)
    pasts, toks = [None] * 3, [None] * 3
    tol = dict(rtol=5e-2, atol=5e-2)

    def prefill(b, n):
        ids = torch.randint(0, 512, (1, n), generator=g)
        lo, pasts[b] = oracle(ids, pasts[b])
        out = model(input_ids=ids.cuda(), past_key_values=cache.row(b), use_cache=True)
        torch.testing.assert_close(out.logits.float().cpu(), lo.float(), **tol)
        toks[b] = lo[:, -1:].argmax(-1)

    with torch.no_grad():
        for b, chunks in enumerate([[45], [20, 130], [7]]):  # row 1: raw first chunk, then the dequantised image
            for n in chunks:
                prefill(b, n)
        for step in range(10):
            ids = torch.cat(toks, 0)
            out = model(input_ids=ids.cuda(), past_key_values=cache, use_cache=True)
            assert out.logits.shape == (3, 1, 512) and out.past_key_values is cache
            for b in range(3):
                lo, pasts[b] = oracle(toks[b], pasts[b])
                torch.testing.assert_close(out.logits[b : b + 1].float().cpu(), lo.float(), **tol)
                toks[b] = lo.argmax(-1)
            if step in (2, 6):  # per-row eviction of the newest token
                b = 0 if step == 2 else 2
                cache.row(b).evict_last(1)
                pasts[b] = tuple(evict_past(p, 1) for p in pasts[b])
            if step == 4:  # continuous batching: row 1 finished, a new prompt takes its place
                cache.row(1).clear()
                pasts[1] = None
                prefill(1, 33)
            assert cache.row_lengths == [p[0][0].shape[2] for p in pasts]


@DTYPES
def test_graph_replay_matches_eager_ragged_int4_decode(dtype):
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 6
    model, _ = _patched("llama", 13, sink, recent, dtype)
    ca = DuoRaggedINT4KVCache(model, GATES, 3, 256, sink, recent)
    cb = DuoRaggedINT4KVCache(model, GATES, 3, 256, sink, recent)
    g = torch.Generator().manual_seed(6)

    def prefill(b, ids):
        for c in (ca, cb):
            model(input_ids=ids.cuda(), past_key_values=c.row(b), use_cache=True)

    with torch.no_grad():
        for b, n in enumerate([37, 9, 70]):
            prefill(b, torch.randint(0, 512, (1, n), generator=g))
        graph = DuoDecodeGraph(model, cb)
        tok = torch.randint(0, 512, (3, 1), generator=g).cuda()
        for step in range(14):  # several ring wraps (recent 6)
            le = model(input_ids=tok, past_key_values=ca, use_cache=True).logits
            lg = graph.step(tok)
            assert torch.equal(le, lg), f"step {step}: graph replay differs from eager ragged INT4 decode"
            tok = le.argmax(-1)
            if step == 3:
                for c in (ca, cb):
                    c.row(1).evict_last(2)
            if step == 7:
                ids = torch.randint(0, 512, (1, 21), generator=g)
                for c in (ca, cb):
                    c.row(2).clear()
                prefill(2, ids)
                graph.resync()
            assert ca.row_lengths == cb.row_lengths
        assert torch.equal(ca.row_state, cb.row_state)
        # an emptied row cannot join a replayed step either
        cb.row(0).clear()
        with pytest.raises(ValueError, match="row 0 is empty.*prefill it through cache.row"):
            graph.step(tok)


def test_errors_empty_row_chunk_limit_and_overflow():
    sink, recent = 4, 12
    model, _ = _patched("llama", 17, sink, recent)
    cache = DuoRaggedINT4KVCache(model, GATES, 2, 50, sink, recent)
    with torch.no_grad():
        model(input_ids=torch.zeros(1, 49, dtype=torch.long).cuda(), past_key_values=cache.row(0), use_cache=True)
        with pytest.raises(ValueError, match="row 1 is empty.*prefill it through cache.row"):
            model(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [49, 0]
        model(input_ids=torch.zeros(1, 5, dtype=torch.long).cuda(), past_key_values=cache.row(1), use_cache=True)
        with pytest.raises(ValueError, match="prefill each row"):  # group 2 x 5 tokens = 10 rows > 8
            model(input_ids=torch.zeros(2, 5, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [49, 5]
        model(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [50, 6]
        with pytest.raises(ValueError, match="Trying to put 1 KVs into a cache with max size 50, current size: 50."):
            model(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)
        assert cache.row_lengths == [50, 6] and cache.memory_usage > 0


def test_rows_share_one_dequantised_image():
    """Chunks of >= 128 tokens on several rows use the parent's one 16-bit image (and one first-chunk scratch)."""
    Hq, Hkv, n_full, cap, B = 32, 8, 8, 8192, 4
    R = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, cap, 16, 48, torch.float16, DEV)
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator(device=DEV).manual_seed(1)

    def chunk(b, S):
        out = torch.empty(1, S, Hq, D, dtype=torch.float16, device=DEV)
        R.row(b).attend(0, torch.randn(1, S, width, generator=g, device=DEV).half(), None, None, _C.ROPE_NONE, out)

    for b in range(B):
        chunk(b, 200)  # raw first chunks (and a longer staging area for every row)
    assert all(R.row(b)._scratch is R.row(0)._scratch for b in range(B))
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated(DEV)
    chunk(0, 200)
    torch.cuda.synchronize()
    m1 = torch.cuda.memory_allocated(DEV)
    image = 2 * n_full * cap * D * 2  # K and V of the retrieval heads in fp16
    assert m1 - m0 >= image
    for b in range(1, B):
        chunk(b, 200)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) - m1 < image // 8, "a row allocated its own dequantised image"
    assert all(R.row(b)._dq is R.row(0)._dq for b in range(B))
