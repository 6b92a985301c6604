"""The batched ragged prefill at model level: ``model(input_ids=[1, T], past_key_values=ragged, chunk_lengths=[...])``.

* one forward takes new prompts on empty rows and the forks' questions on a shared prompt, against per-row forwards
  through ``row(b)`` (logits within tolerance, the same greedy token wherever the control's top two logits are more than
  0.1 apart: the GEMMs run on other shapes, so the bits are not promised) and against ``OracleModel``; then the rows
  decode together, identically;
* batched prefills between ``DuoDecodeGraph`` replays give what eager decode gives over the same schedule, bit for bit;
  a chunk longer than the staging area is refused while the graph is attached, and changes nothing.
"""
import copy

import numpy as np
import pytest
import torch

from duo_attention_b200.kv_cache import DuoRaggedKVCache
from oracle import duo_oracle as O

pytestmark = pytest.mark.gpu
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])
TOL = dict(rtol=5e-2, atol=5e-2)


def _models(kind, seed, sink, recent):
    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    if kind == "llama":
        from transformers import LlamaConfig, LlamaForCausalLM as M

        cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                          intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                          attn_implementation="eager")
        dtype = torch.bfloat16
    else:
        from transformers import MistralConfig, MistralForCausalLM as M

        cfg = MistralConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                            intermediate_size=1024, vocab_size=512, head_dim=128, max_position_embeddings=8192,
                            rope_theta=10000.0, sliding_window=None, attn_implementation="eager")
        dtype = torch.float16
    model = M(cfg).to(dtype).eval()
    oracle = O.OracleModel(copy.deepcopy(model), GATES, sink, recent)
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda(), oracle


def _check_greedy(le, lc, what):
    torch.testing.assert_close(le.float(), lc.float(), **TOL, msg=lambda m: f"{what}: {m}")
    top2 = lc.float().topk(2, -1).values
    clear = top2[..., 0] - top2[..., 1] > 0.1
    assert torch.equal(le.argmax(-1)[clear], lc.argmax(-1)[clear]), f"{what}: greedy tokens differ"


@pytest.mark.parametrize("kind", ["llama", "mistral"])
def test_one_forward_admits_prompts_and_questions(kind):
    """Row 0 holds a 300-token prompt, rows 1 and 2 are its forks; one forward gives row 1 a question of 40 tokens, row 2
    one of 130, and the empty rows 3 and 4 new prompts of 200 and 9; row 0 takes nothing.  The control's rows take the
    same tokens through row(b)."""
    sink, recent = 4, 12
    model, oracle = _models(kind, 51, sink, recent)
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, 512, (1, 300), generator=g)
    chunks = {1: 40, 2: 130, 3: 200, 4: 9}
    ids = {b: torch.randint(0, 512, (1, n), generator=g) for b, n in chunks.items()}
    caps = [364, 400, 400, 400, 400]
    X, Cc = (DuoRaggedKVCache(model, GATES, 5, caps, sink, recent, prefilling_chunk_size=256) for _ in range(2))
    run = lambda i, past, **kw: model(input_ids=i.cuda(), past_key_values=past, use_cache=True, **kw).logits
    with torch.no_grad():
        for c in (X, Cc):
            run(prompt, c.row(0))
            c.share_prefix(0, 1, 400)
            c.share_prefix(0, 2, 400)
        lens = [0] + [chunks[b] for b in range(1, 5)]
        packed = torch.cat([ids[b] for b in range(1, 5)], 1)
        lx = run(packed, X, chunk_lengths=lens)
        assert lx.shape == (5, 1, 512)
        lo0, past0 = oracle(prompt, None)
        pasts = {0: past0, 1: past0, 2: past0, 3: None, 4: None}
        for b in range(1, 5):
            lc = run(ids[b], Cc.row(b))[:, -1:]
            _check_greedy(lx[b : b + 1], lc, f"row {b}'s chunk of {chunks[b]}")
            lo, pasts[b] = oracle(ids[b], pasts[b])
            torch.testing.assert_close(lx[b : b + 1].float().cpu(), lo.float(), **TOL)
        assert X.row_lengths == Cc.row_lengths == [300, 340, 430, 200, 9]
        Cc.sync_device_state()  # row(b) leaves the parent's device copy to the next batched step
        assert torch.equal(X.row_state, Cc.row_state)
        te = torch.cat([lx[b : b + 1, -1:].argmax(-1) for b in range(5)], 0)
        for step in range(6):  # the rows decode together, in both caches, on the same tokens
            le, lc = run(te, X), run(te, Cc)
            _check_greedy(le, lc, f"step {step}")
            for b in range(1, 5):
                lo, pasts[b] = oracle(te[b : b + 1].cpu(), pasts[b])
                torch.testing.assert_close(le[b : b + 1].float().cpu(), lo.float(), **TOL)
            te = lc.argmax(-1)
        assert X.row_lengths == Cc.row_lengths


def test_batched_prefills_between_graph_replays_equal_eager():
    """Rows 0 and 1 are admitted in one forward and decode in a DuoDecodeGraph; rows 2 and 3 sit idle until a second
    forward admits them (row 2 with 150 tokens, row 3 with 20) and row 0 takes a follow-up of 130 in the same call; then
    all four decode.  An eager twin takes every call; the graph's logits equal it bit for bit, and a chunk longer than
    the staging area (which the first forward grew to 300 rows) is refused under the graph without changing anything."""
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 12
    model, _ = _models("llama", 61, sink, recent)
    g = torch.Generator().manual_seed(8)
    caps = [700, 400, 400, 400]
    Xe, Xg = (DuoRaggedKVCache(model, GATES, 4, caps, sink, recent, prefilling_chunk_size=256) for _ in range(2))
    run = lambda i, past, **kw: model(input_ids=i.cuda(), past_key_values=past, use_cache=True, **kw).logits
    with torch.no_grad():
        first = torch.randint(0, 512, (1, 300 + 128), generator=g)
        for c in (Xe, Xg):
            c.set_active(2, False)
            c.set_active(3, False)
            lf = run(first, c, chunk_lengths=[300, 128, 0, 0])
        graph = DuoDecodeGraph(model, Xg)
        te = lf.argmax(-1)

        def steps(n, what):
            nonlocal te
            for s in range(n):
                le, lg = run(te, Xe), graph.step(te)
                act = [b for b in range(4) if Xe.row_active[b]]
                assert torch.equal(le[act], lg[act]), f"{what} step {s}: graph replay differs from eager"
                te = le.argmax(-1)

        steps(3, "rows 0 and 1")
        width_before = [t.clone() for t in Xg.tensors[0].values()]
        rs_before = Xg.row_state.clone()
        with pytest.raises(ValueError, match="DuoDecodeGraph"):
            run(torch.randint(0, 512, (1, 400), generator=g), Xg, chunk_lengths=[0, 0, 400, 0])
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(width_before, Xg.tensors[0].values()))
        assert torch.equal(rs_before, Xg.row_state)
        second = torch.randint(0, 512, (1, 130 + 150 + 20), generator=g)
        for c in (Xe, Xg):
            ls = run(second, c, chunk_lengths=[130, 0, 150, 20])
            c.set_active(2, True)
            c.set_active(3, True)
        nxt = ls.argmax(-1)
        te = torch.stack([nxt[0], te[1], nxt[2], nxt[3]])
        steps(4, "all four rows")
        assert Xe.row_lengths == Xg.row_lengths == [300 + 3 + 130 + 4, 128 + 3 + 4, 154, 24]
        assert torch.equal(Xe.row_state, Xg.row_state)
