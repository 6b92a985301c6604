"""Parity of the CUDA hot path (through the C ABI) against the CPU oracle on identical seeded inputs.

Tolerance: north_star's bf16 bar, rtol=1e-2 / atol=1e-3, on the attention output.
Every test drives ``DuoKVCache.attend`` = duo_rope_append -> duo_attention -> duo_stream_commit.
"""
import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
RTOL, ATOL = 1e-2, 1e-3


def split_qkv(qkv, Hq, Hkv):
    B, S, _ = qkv.shape
    q = qkv[..., : Hq * D].reshape(B, S, Hq, D)
    k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D)
    v = qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D)
    return q, k, v


class Fa2Shadow:
    """The reference forward's attention core (llama.py:225-290) with the INSTALLED flash_attn_func on token-major GPU
    caches, fed the same chunks as the product: gives every parity assertion FlashAttention-2's own deviation from
    the oracle on the same inputs (tests/parity.py).  None when flash_attn is not importable."""

    def __init__(self, n_full, groups, sink, recent):
        try:
            from flash_attn import flash_attn_func
        except Exception:
            flash_attn_func = None
        self.fa = flash_attn_func
        self.n_full, self.G, self.sink, self.recent = n_full, groups, sink, recent
        self.kv = None

    @staticmethod
    def exact(q, k, v):
        """fp64 bottom-right-causal GQA attention on the GPU (row-blocked): no rounding anywhere."""
        B, Sq, Hq, Dh = q.shape
        Sk, Hkv = k.shape[1], k.shape[2]
        G = Hq // Hkv
        out = torch.empty(B, Sq, Hq, Dh, dtype=torch.float64, device=q.device)
        kd, vd = k.double(), v.double()
        jj = torch.arange(Sk, device=q.device)[None, :]
        for r0 in range(0, Sq, 512):
            r1 = min(Sq, r0 + 512)
            ii = torch.arange(r0, r1, device=q.device)[:, None] + (Sk - Sq)
            for h in range(Hq):
                s = torch.einsum("bqd,bkd->bqk", q[:, r0:r1, h].double(), kd[:, :, h // G]) / Dh ** 0.5
                s = s.masked_fill((jj > ii)[None], float("-inf"))
                out[:, r0:r1, h] = torch.einsum("bqk,bkd->bqd", torch.softmax(s, -1), vd[:, :, h // G])
        return out

    def step(self, q, k, v):
        """-> (flash_attn_func output, exact fp64 output) of this chunk, both fp32 on the CPU."""
        if self.fa is None:
            return None, None
        nf, G = self.n_full, self.G
        q, k, v = q.cuda(), k.cuda(), v.cuda()
        if self.kv is None:
            out = self.fa(q, k, v, causal=True)
            truth = self.exact(q, k, v)
            fk, fv, sk, sv = k[:, :, :nf], v[:, :, :nf], k[:, :, nf:], v[:, :, nf:]
        else:
            fk, fv, sk, sv = self.kv
            fk, fv = torch.cat([fk, k[:, :, :nf]], 1), torch.cat([fv, v[:, :, :nf]], 1)
            sk, sv = torch.cat([sk, k[:, :, nf:]], 1), torch.cat([sv, v[:, :, nf:]], 1)
            parts, tparts = [], []
            if nf > 0:
                parts.append(self.fa(q[:, :, : nf * G], fk, fv, causal=True))
                tparts.append(self.exact(q[:, :, : nf * G], fk, fv))
            if nf * G < q.shape[2]:
                parts.append(self.fa(q[:, :, nf * G :], sk, sv, causal=True))
                tparts.append(self.exact(q[:, :, nf * G :], sk, sv))
            out = torch.cat(parts, dim=2)
            truth = torch.cat(tparts, dim=2)
        if sk.shape[1] > self.sink + self.recent:
            sk = torch.cat([sk[:, : self.sink], sk[:, sk.shape[1] - self.recent :]], 1)
            sv = torch.cat([sv[:, : self.sink], sv[:, sv.shape[1] - self.recent :]], 1)
        self.kv = (fk, fv, sk, sv)
        return out.float().cpu(), truth.float().cpu()

    def evict(self, n):
        if self.kv is not None:
            self.kv = tuple(t[:, : t.shape[1] - n] for t in self.kv)


def run_schedule(Hq, Hkv, n_full, sink, recent, chunks, B=1, dtype=torch.bfloat16, seed=0, evict_after=None,
                 force_mma=False, max_size=None, stage_cap=8, check=True, qscale=1.0):
    dev = torch.device("cuda:0")
    shadow = Fa2Shadow(n_full, Hq // Hkv, sink, recent) if check else None
    g = torch.Generator().manual_seed(seed)
    total = sum(chunks)
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], B, max_size or total + 8, sink, recent, dtype, dev,
                       stage_cap=stage_cap)
    past = None
    worst = 0.0
    outs = []
    for i, S in enumerate(chunks):
        qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(dtype)
        qkv[..., : Hq * D] *= qscale
        out = torch.empty(B, S, Hq, D, dtype=dtype, device=dev)
        cache.attend(0, qkv.to(dev), None, None, _C.ROPE_NONE, out, force_mma=force_mma)
        q, k, v = split_qkv(qkv, Hq, Hkv)
        ref, past = O.tuple_attention_core(q, k, v, past, n_full, Hq // Hkv, sink, recent)
        got = out.float().cpu()
        outs.append(got)
        if check:
            fa2, truth = shadow.step(q, k, v)
            assert_parity(got, ref, f"chunk {i} (len {S}, past {cache.kv_seq_len - S})", fa2=fa2, truth=truth)
        worst = max(worst, (got - ref.float()).abs().max().item())
        ev = (evict_after or {}).get(i, 0)
        if ev:
            cache.evict_last(ev)
            if shadow is not None:
                shadow.evict(ev)
            fk, sk = past
            past = (fk[:, :, : fk.shape[2] - ev].contiguous(), sk[:, :, : sk.shape[2] - ev].contiguous())
        assert cache.kv_seq_len == past[0].shape[2]
        assert cache.streaming_kv_seq_len == past[1].shape[2]
    torch.cuda.synchronize()
    return worst, outs


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_full", [0, 1, 4, 7, 8])
def test_head_mix_gqa4(n_full):
    run_schedule(32, 8, n_full, 16, 48, [70, 1, 1, 5, 30, 1, 90, 1, 2], seed=n_full)


@pytest.mark.parametrize("n_full", [0, 3, 8])
def test_head_mix_mha(n_full):
    run_schedule(8, 8, n_full, 8, 24, [40, 1, 16, 1, 33, 1], seed=10 + n_full)


@pytest.mark.parametrize("q_len", [1, 2, 3, 4, 5, 8, 15, 16, 17, 31, 64, 65])
def test_continuation_chunk_lengths(q_len):
    run_schedule(8, 2, 1, 8, 24, [50, q_len, 1, q_len], seed=100 + q_len)


@pytest.mark.parametrize("sink,recent", [(64, 256), (128, 256), (16, 64), (1, 2), (0, 5)])
def test_sink_recent_configs(sink, recent):
    W = sink + recent
    chunks = [max(1, sink // 2), 1, max(1, recent // 2), W + 3, 1, 1, 2 * W + 5, 1, 7, 1]
    run_schedule(8, 2, 1, sink, recent, chunks, seed=sink * 7 + recent)


@pytest.mark.parametrize("first", [1, 63, 129, 320, 321, 1025])
def test_first_prefill_lengths_then_decode(first):
    # first call: every head is plain causal (llama.py:225-233); then decode steps
    run_schedule(8, 2, 1, 64, 256, [first, 1, 1, 1], seed=first)


def test_ring_wraps_many_times():
    run_schedule(4, 2, 1, 2, 5, [3] + [1] * 40 + [4, 1, 9, 1, 1], seed=5)


def test_decode_only_from_empty_cache():
    run_schedule(8, 2, 1, 4, 4, [1] * 20, seed=6)


def test_batch2():
    run_schedule(8, 2, 1, 4, 12, [20, 1, 1, 9, 1, 33, 1], B=2, seed=7)


def test_fp16():
    run_schedule(8, 2, 1, 16, 48, [70, 1, 1, 5, 30, 1], dtype=torch.float16, seed=8)


def test_evict_last_like_the_benchmark():
    # benchmark_static.py:96-103: decode one token, evict_last(1), repeat
    chunks = [300, 40] + [1] * 6
    run_schedule(8, 2, 1, 16, 64, chunks, evict_after={i: 1 for i in range(2, 8)}, seed=9)


def test_split_kv_long_context_decode():
    # one retrieval kv head, 20k keys: ~150+ key splits merged by the last CTA in the same launch
    run_schedule(4, 1, 1, 64, 256, [20000, 1, 1, 3, 1], seed=11, stage_cap=20000)


def test_split_kv_with_streaming_heads_long():
    run_schedule(16, 4, 2, 64, 256, [9000, 1, 2, 1], seed=12, stage_cap=9000)


def test_sharp_softmax_large_logits():
    # large |q| makes the softmax nearly one-hot: exercises running-max rescaling across tiles/splits
    run_schedule(8, 2, 1, 8, 24, [700, 1, 1, 5], seed=13, qscale=6.0)


def test_overflow_raises_value_error_like_reference():
    dev = torch.device("cuda:0")
    cache = DuoKVCache(1, 8, 2, D, [1], 1, 16, 4, 4, torch.bfloat16, dev)
    qkv = torch.zeros(1, 17, 12 * D, dtype=torch.bfloat16, device=dev)
    out = torch.empty(1, 17, 8, D, dtype=torch.bfloat16, device=dev)
    with pytest.raises(ValueError, match="Trying to put 17 KVs into a cache with max size 16"):
        cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        cache.attend(0, qkv.cpu(), None, None, _C.ROPE_NONE, out)


def test_growable_cache_matches_static():
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    Hq, Hkv = 8, 2
    a = DuoKVCache(1, Hq, Hkv, D, [1], 1, 2048, 4, 12, torch.bfloat16, dev, stage_cap=512)
    b = DuoKVCache(1, Hq, Hkv, D, [1], 1, 16, 4, 12, torch.bfloat16, dev, stage_cap=1, growable=True)
    for S in [100, 1, 300, 1, 1, 500, 1]:
        qkv = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(torch.bfloat16).to(dev)
        oa = torch.empty(1, S, Hq, D, dtype=torch.bfloat16, device=dev)
        ob = torch.empty_like(oa)
        a.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, oa)
        b.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, ob)
        assert torch.equal(oa, ob)


# ------------------------------------------------------------------------------------------------
# size-independent properties at the benchmark's full context length (1M tokens, one layer)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [131072, 1048576])
def test_full_size_decode_properties(N):
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent = 32, 8, 4, 64, 256
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, N + 8, sink, recent, torch.bfloat16, dev)
    t = cache.tensors[0]
    W = sink + recent
    g = torch.Generator(device=dev).manual_seed(1)
    # synthetic resident cache, as the benchmark fills it
    t["full_k"].normal_(generator=g)
    t["ring_k"].normal_(generator=g)
    cache.kv_seq_len_list[0] = N
    cache.total_list[0] = N
    cache.lo_list[0] = N - recent
    qkv = torch.randn(1, 1, (Hq + 2 * Hkv) * D, generator=g, device=dev, dtype=torch.float32).to(torch.bfloat16)
    out = torch.empty(1, 1, Hq, D, dtype=torch.bfloat16, device=dev)

    def decode():
        cache.kv_seq_len_list[0] = N
        cache.total_list[0] = N
        cache.lo_list[0] = N - recent
        cache.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
        return out.float().clone()

    # (1) all V rows equal a constant vector c  ->  output == c for every head (softmax sums to 1)
    c = torch.linspace(-1, 1, D, device=dev).to(torch.bfloat16)
    t["full_v"][:] = c
    t["ring_v"][:] = c
    q_c = qkv.clone()
    q_c[..., (Hq + Hkv) * D :] = c.repeat(Hkv)
    qkv_backup = qkv.clone()
    qkv.copy_(q_c)
    o = decode()
    torch.testing.assert_close(o, c.float().expand_as(o), rtol=1e-2, atol=1e-3)
    qkv.copy_(qkv_backup)

    # (2) q == 0 -> uniform attention -> output == mean of the visible V rows
    t["full_v"].normal_(generator=g)
    t["ring_v"].normal_(generator=g)
    qz = qkv.clone()
    qz[..., : Hq * D] = 0
    qkv.copy_(qz)
    vnew = qz[0, 0, (Hq + Hkv) * D :].view(Hkv, D).float()
    # expected means are taken BEFORE the call: the ring commit that follows the attention overwrites one slot
    means = []
    for kvh in range(Hkv):
        if kvh < n_full:
            means.append((t["full_v"][0, kvh, :N].float().sum(0) + vnew[kvh]) / (N + 1))
        else:
            means.append((t["ring_v"][0, kvh - n_full, :W].float().sum(0) + vnew[kvh]) / (W + 1))
    o = decode()[0, 0]
    for h in range(Hq):
        torch.testing.assert_close(o[h], means[h // 4], rtol=1e-2, atol=1e-3)
    qkv.copy_(qkv_backup)

    # (3) one key with an overwhelming logit -> output == that key's V row, wherever it sits
    #     (first key, tile/split boundaries, last cached key)
    for pos in [0, 63, 64, 4095, N // 2 + 17, N - 1]:
        kvh = 1
        qrow = qkv[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D].float()
        saved = t["full_k"][0, kvh, pos].clone()
        t["full_k"][0, kvh, pos] = (qrow / qrow.norm() * 40.0).to(torch.bfloat16)
        qs = qkv.clone()
        qs[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D] = (qrow / qrow.norm() * 40.0).to(torch.bfloat16)
        qkv.copy_(qs)
        o = decode()[0, 0, kvh * 4]
        torch.testing.assert_close(o, t["full_v"][0, kvh, pos].float(), rtol=1e-2, atol=2e-3)
        t["full_k"][0, kvh, pos] = saved
        qkv.copy_(qkv_backup)


# ------------------------------------------------------------------------------------------------
# wgmma prefill kernel (chunks >= 128 tokens) — shapes beyond the plain bf16 / B=1 / GQA-4 case, each
# cross-checked against the oracle AND against the mma.sync kernel family on the same inputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    dict(Hq=8, Hkv=2, n_full=1, sink=16, recent=48, chunks=[200, 128, 1, 333], B=2),             # batch 2
    dict(Hq=8, Hkv=2, n_full=1, sink=16, recent=48, chunks=[256, 1, 130], dtype=torch.float16),  # fp16
    dict(Hq=3, Hkv=3, n_full=1, sink=8, recent=24, chunks=[384, 129, 1, 257]),                   # MHA: token-tile pairs, odd tile counts
    dict(Hq=8, Hkv=2, n_full=0, sink=64, recent=256, chunks=[500, 400, 1, 128]),                 # streaming heads only
    dict(Hq=8, Hkv=2, n_full=2, sink=64, recent=256, chunks=[129, 1, 640]),                      # retrieval heads only
    dict(Hq=12, Hkv=2, n_full=1, sink=4, recent=4, chunks=[128, 128, 128, 1, 128]),              # G=6, tiny window
])
def test_tc_prefill_shapes(kw):
    kw = dict(kw)
    run_schedule(seed=77, stage_cap=max(kw["chunks"]), **kw)
    _, a = run_schedule(seed=78, stage_cap=max(kw["chunks"]), check=False, **kw)
    _, b = run_schedule(seed=78, stage_cap=max(kw["chunks"]), check=False, force_mma=True, **kw)
    for x, y in zip(a, b):
        assert_parity(x, y, "wgmma vs mma.sync kernel family")


def test_tc_prefill_sharp_softmax_rescales():
    # growing logits force a running-max update (and O rescale) on many tiles of the wgmma prefill kernel
    run_schedule(8, 2, 1, 8, 24, [900, 300], seed=14, qscale=8.0, stage_cap=900)
