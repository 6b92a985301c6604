"""Shared prefixes on the GPU, checked against exact references rather than against the library itself.

* fp64 attention (the oracle's tuple-cache attention) for every row of batches that share prompts, including groups of
  more than 64 packed rows, which the prefix kernel serves in several 64-row blocks;
* a visibility census: all keys get the same logit and carry one-hot values by where they live, and every cache row a
  row must not see (the pool's slack and headroom, other groups' regions, the donor's rows appended after the fork)
  holds poison that lights dimension 127, so each output is an exact histogram of the keys that row attends;
* graph replay against eager steps with ``evict_last(1)`` after every step, forks while the graph is attached and a
  sharer cleared and refilled.
"""
import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedKVCache
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def split_qkv(qkv, Hq, Hkv):
    B, S, _ = qkv.shape
    return (qkv[..., : Hq * D].reshape(B, S, Hq, D), qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D),
            qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D))


# ---- fp64 attention, groups of one to several 64-row blocks ---------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full,B,q_len,L", [
    (32, 8, 3, 18, 1, 700),    # donor + 17 sharers at G = 4: 72 packed rows, two blocks
    (32, 8, 8, 6, 4, 1000),    # G * q_len = 16: 6 members, 96 packed rows, two blocks
    (32, 8, 2, 4, 2, 4097),    # one block, a prompt one past a tile boundary
    (8, 8, 5, 5, 1, 300),      # MHA
])
def test_shared_rows_match_fp64_attention(Hq, Hkv, n_full, B, q_len, L, dtype):
    sink, recent = 16, 48
    G = Hq // Hkv
    steps = 4
    own = 128 + steps * q_len
    caps = [L + own] + [own] * (B - 1)
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64)
    g = torch.Generator().manual_seed(B * 31 + q_len + L)
    width = (Hq + 2 * Hkv) * D
    qkv = torch.randn(1, L, width, generator=g).to(dtype)
    for c0 in range(0, L, 4096):
        n = min(4096, L - c0)
        S.row(0).attend(0, qkv[:, c0 : c0 + n].to(DEV), None, None, _C.ROPE_NONE,
                        torch.empty(1, n, Hq, D, dtype=dtype, device=DEV))
    q, k, v = split_qkv(qkv.double(), Hq, Hkv)
    _, past = O.tuple_attention_core(q, k, v, None, n_full, G, sink, recent)
    for b in range(1, B):  # forks of the donor and of sharers
        S.share_prefix(0 if b % 2 else b - 1, b, own)
    P = L // 128 * 128
    assert all(S.row_prefix[b] == (0, P) for b in range(1, B))
    pasts = [past] * B
    for step in range(steps):
        x = torch.randn(B, q_len, width, generator=g).to(dtype)
        out = torch.empty(B, q_len, Hq, D, dtype=dtype, device=DEV)
        S.attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        got = out.float().cpu()
        for b in range(B):
            qb, kb, vb = split_qkv(x[b : b + 1].double(), Hq, Hkv)
            ref, pasts[b] = O.tuple_attention_core(qb, kb, vb, pasts[b], n_full, G, sink, recent)
            assert_parity(got[b : b + 1], ref, f"step {step} row {b}")


# ---- visibility census ----------------------------------------------------------------------------------------------
POISON = 127


def _onehot(n, dim, dtype):
    v = torch.zeros(n, D, dtype=dtype, device=DEV)
    v[:, dim] = 1
    return v


def test_visibility_census_two_groups_and_plain_rows():
    """Rows: 0 donor of prompt A (300 keys, 256 shared), 1 forked from 0, 2 forked from 1, 3 donor of prompt B (700 keys,
    640 shared), 4 forked from 3, 5 a plain row of 500 keys.  Value dimensions: 0 / 1 prompt A's shared part / tail,
    2 / 3 prompt B's, 4 row 5's prompt, 10 + b row b's decoded tokens (the donors keep appending after the fork)."""
    Hq, Hkv, n_full, dtype = 32, 8, 8, torch.bfloat16
    B, steps = 6, 5
    lengths = [300, 0, 0, 700, 0, 500]
    caps = [300 + 64, 200, 200, 700 + 64, 200, 500 + 64]
    S = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, 16, 48, dtype, DEV, stage_cap=64,
                                       pool_size=4096)
    for name in ("full_k", "full_v"):  # the whole pool is poison until written
        S.tensors[0][name].zero_()
    S.tensors[0]["full_v"][:, POISON] = 1
    layout = {0: [(0, 256, 0), (256, 300, 1)], 3: [(0, 640, 2), (640, 700, 3)], 5: [(0, 500, 4)]}
    for b, parts in layout.items():
        r = S.row(b)
        for lo, hi, dim in parts:
            r.tensors[0]["full_v"][0, :, lo:hi] = _onehot(hi - lo, dim, dtype)
        r.tensors[0]["full_v"][0, :, lengths[b]:, POISON] = 1  # (already poison: the region's slack)
        r.kv_seq_len_list[0] = r.total_list[0] = lengths[b]
    S.sync_device_state()
    S.share_prefix(0, 1, 200)
    S.share_prefix(1, 2, 200)
    S.share_prefix(3, 4, 200)
    base = {0: {0: 256, 1: 44}, 1: {0: 256, 1: 44}, 2: {0: 256, 1: 44}, 3: {2: 640, 3: 60}, 4: {2: 640, 3: 60},
            5: {4: 500}}
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(3)
    for step in range(steps):
        x = torch.zeros(B, 1, width, dtype=dtype)
        x[..., : Hq * D] = torch.randn(B, 1, Hq * D, generator=g).to(dtype)  # any q: every key has logit 0
        for b in range(B):
            x[b, 0, (Hq + Hkv) * D :].view(Hkv, D)[:, 10 + b] = 1
        out = torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV)
        S.attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        got = out.float().cpu()[:, 0]
        for b in range(B):
            cnt = dict(base[b])
            cnt[10 + b] = step + 1
            n = sum(cnt.values())
            exp = torch.zeros(D, dtype=torch.float64)
            for dim, c in cnt.items():
                exp[dim] = c / n
            for h in range(Hq):
                row = got[b, h].double()
                lit = exp > 0
                assert torch.all(row[~lit] == 0), f"step {step} row {b} head {h}: sees keys it must not " \
                                                  f"(dims {torch.nonzero(row * ~lit).flatten().tolist()})"
                assert torch.all((row[lit] - exp[lit]).abs() <= exp[lit] * 2 ** -8), \
                    f"step {step} row {b} head {h}: {row[lit].tolist()} != {exp[lit].tolist()}"


# ---- graph replay with evict_last(1) after every step ----------------------------------------------------------------
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


def test_graph_replay_with_eviction_after_every_step():
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 6
    model = _patched(29, sink, recent)
    caps = [400, 96, 96, 200]
    ca, cb = (DuoRaggedKVCache(model, GATES, 4, caps, sink, recent, pool_size=2048) for _ in range(2))
    g = torch.Generator().manual_seed(9)
    prompt = torch.randint(0, 512, (1, 300), generator=g)
    with torch.no_grad():
        for c in (ca, cb):
            model(input_ids=prompt.cuda(), past_key_values=c.row(0), use_cache=True)
            model(input_ids=prompt[:, :40].cuda(), past_key_values=c.row(3), use_cache=True)
            c.share_prefix(0, 1, 96)
        graph = DuoDecodeGraph(model, cb)
        captured = graph.graph
        for c in (ca, cb):  # a fork made while the graph is attached
            c.share_prefix(1, 2, 96)
        tok = torch.randint(0, 512, (4, 1), generator=g).cuda()
        for step in range(12):
            le = model(input_ids=tok, past_key_values=ca, use_cache=True).logits
            lg = graph.step(tok)
            assert torch.equal(le, lg), f"step {step}: graph replay differs from eager decode"
            for c in (ca, cb):
                c.evict_last(1)  # every step is taken back: the next one decodes at the same positions
            tok = le.argmax(-1)
            if step == 5:  # a sharer finishes, is cleared and refilled through row(b)
                ids = torch.randint(0, 512, (1, 30), generator=g)
                for c in (ca, cb):
                    c.row(2).clear()
                    model(input_ids=ids.cuda(), past_key_values=c.row(2), use_cache=True)
            assert ca.row_lengths == cb.row_lengths and ca.row_prefix == cb.row_prefix
        assert graph.graph is captured
        assert ca.row_lengths == [300, 300, 30, 40]
        assert torch.equal(ca.row_state, cb.row_state) and torch.equal(ca.row_share, cb.row_share)
