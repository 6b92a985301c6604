"""Idle rows at model level: a row admitted in chunks through ``row(b)`` while the other rows decode in a captured
``DuoDecodeGraph``, on a pooled 16-bit cache and on an INT4 cache (where the admitted row was emptied first and sits
idle until it is refilled).

* the decoding rows against an uninterrupted control cache of just those rows: logits within tolerance and the same
  greedy token wherever the control's top two logits are more than 0.1 apart (the controls decode in a batch of
  another size, whose GEMMs may round differently);
* a decoding row toggled idle for two steps and back, in both caches, while the graph keeps replaying: its position
  drifts in the graph while it is idle and is reloaded when it rejoins;
* the admitted row's chunks and later decode against a batch-1 cache fed the same tokens;
* graph replay against an eager twin cache that takes the same calls: active rows' logits bit-identical.
"""
import numpy as np
import pytest
import torch

from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache, DuoRaggedKVCache

pytestmark = pytest.mark.gpu
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])
TOL = dict(rtol=5e-2, atol=5e-2)


def _model(seed, sink, recent):
    from transformers import LlamaConfig, LlamaForCausalLM

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                      intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                      attn_implementation="eager")
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    enable_duo_attention_eval(model, GATES, sink, recent)
    return model.cuda()


def _check_greedy(le, lc, what):
    torch.testing.assert_close(le.float(), lc.float(), **TOL)
    top2 = lc.float().topk(2, -1).values
    clear = top2[..., 0] - top2[..., 1] > 0.1
    assert torch.equal(le.argmax(-1)[clear], lc.argmax(-1)[clear]), f"{what}: greedy tokens differ"


@pytest.mark.parametrize("kind", ["bf16_pooled", "int4"])
def test_admit_a_row_in_chunks_while_the_others_decode_in_a_graph(kind):
    from duo_attention_b200.graph import DuoDecodeGraph

    sink, recent = 4, 12
    model = _model(41, sink, recent)
    int4 = kind == "int4"
    cls = DuoRaggedINT4KVCache if int4 else DuoRaggedKVCache
    caps4 = 600 if int4 else [300, 260, 400, 600]
    Xe, Xg = (cls(model, GATES, 4, caps4, sink, recent) for _ in range(2))  # eager twin, graph
    C = cls(model, GATES, 3, 600 if int4 else [300, 260, 400], sink, recent)  # rows 0-2, never interrupted
    R = cls(model, GATES, 1, 600 if int4 else [600], sink, recent)  # batch-1 control of the admitted row
    run = lambda ids, past: model(input_ids=ids.cuda(), past_key_values=past, use_cache=True).logits
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        last = []
        for b, n in enumerate((45, 130, 7)):
            ids = torch.randint(0, 512, (1, n), generator=g)
            for c in (Xe, Xg):
                run(ids, c.row(b))
            last.append(run(ids, C.row(b))[:, -1:])
        old = torch.randint(0, 512, (1, 20), generator=g)  # row 3's first request
        for c in (Xe, Xg):
            run(old, c.row(3))
        graph = DuoDecodeGraph(model, Xg)
        captured = graph.graph
        tc = torch.cat(last, 0).argmax(-1)  # the control's greedy tokens for rows 0-2
        t3 = torch.zeros(1, 1, dtype=torch.long)

        def step(what, active3):
            """One batched step of the four rows; rows 0-2 take the control's tokens.  Returns row 3's logits."""
            nonlocal tc
            te = torch.cat([tc.cpu(), t3], 0).cuda()
            le = run(te, Xe)
            lg = graph.step(te)
            act = [b for b in range(4) if Xe.row_active[b]]
            assert Xg.row_active == Xe.row_active
            assert torch.equal(le[act], lg[act]), f"{what}: graph replay differs from eager"
            crow = [b for b in act if b < 3]
            lc = run(tc, C)
            _check_greedy(le[crow], lc[crow], what)
            nxt = lc.argmax(-1)
            tc = torch.stack([nxt[b] if b in act else tc[b].to(nxt.device) for b in range(3)])  # idle: token kept
            return le[3:4] if active3 else None

        for s in range(2):  # row 3's first request decodes with the others
            step(f"step {s}", True)
        # row 3 finished: it is emptied and sits idle (INT4: an empty active row would stop the batch)
        for c in (Xe, Xg):
            c.row(3).clear()
            c.set_active(3, False)
        assert Xg.row_active == [True, True, True, False]
        prompt = torch.randint(0, 512, (1, 200), generator=g)
        for k, c0 in enumerate(range(0, 200, 50)):  # admitted in chunks of 50, two steps of the others between
            chunk = prompt[:, c0 : c0 + 50]
            lr = run(chunk, R.row(0))
            for c in (Xe, Xg):
                torch.testing.assert_close(run(chunk, c.row(3)).float(), lr.float(), **TOL)
            if k == 1:  # row 1 sits out two steps, in the control too, then rejoins
                for c in (Xe, Xg, C):
                    c.set_active(1, False)
            for s in range(2):
                step(f"chunk {k} step {s}", False)
            if k == 1:
                for c in (Xe, Xg, C):
                    c.set_active(1, True)
        assert Xe.row_lengths[3] == Xg.row_lengths[3] == 200
        for c in (Xe, Xg):
            c.set_active(3, True)
        t3 = lr[:, -1:].argmax(-1).cpu()
        for s in range(6):  # the admitted row decodes with the others, against its batch-1 control
            l3 = step(f"admitted step {s}", True)
            lr = run(t3, R)
            _check_greedy(l3, lr, f"admitted row, step {s}")
            t3 = lr.argmax(-1).cpu()
        assert graph.graph is captured
        assert Xe.row_lengths == Xg.row_lengths
        assert Xe.row_lengths[:3] == C.row_lengths and Xe.row_lengths[3] == R.row_lengths[0] == 206
        assert torch.equal(Xe.row_state, Xg.row_state)
