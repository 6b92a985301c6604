"""Prefill-sized chunks on forks of a sequence-sharded prompt at model level, ranks emulated on one GPU: a small random
bf16 Llama and an fp16 Mistral run prompt -> ``fork(B)`` -> ``model(input_ids=[B, S])`` with a different question per
row -> decode, eagerly and under ``DuoDecodeGraph``.

``RankGroup`` and the prompt's placement are tests/test_gpu_seqshard_forks_model.py's.  The control is a batch-B
DuoSeqShardKVCache per rank whose rows each hold the prompt.  The question's logits must be bit-identical to the
control's (duo_prefill_seq_shared runs duo_prefill_seq's tiles on the same slice); decode steps take the forks' cascade,
so the greedy tokens must agree wherever the control's top two logits are more than 0.1 apart, and graph replay must
equal eager decode bit for bit."""
import pytest
import torch

from duo_attention_b200.kv_cache import DuoAttentionStaticKVCache
from test_gpu_seqshard_forks_model import GATES, RECENT, SINK, RankGroup, _model, _sharded

pytestmark = pytest.mark.gpu


def _mistral(seed):
    from transformers import MistralConfig, MistralForCausalLM

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    cfg = MistralConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                        intermediate_size=1024, vocab_size=512, head_dim=128, max_position_embeddings=8192,
                        rope_theta=10000.0, sliding_window=None, attn_implementation="eager")
    model = MistralForCausalLM(cfg).to(torch.float16).eval()
    enable_duo_attention_eval(model, GATES, SINK, RECENT)
    return model.cuda()


def _ranks(model, src, W, block, B, max_size):
    ranks = _sharded(model, src, W, block, B, max_size)
    comm = ranks[0].seq.comm  # one LocalSeqComm: its stacked merge serves prefill-sized chunks too
    comm.merge_scattered = comm.merge
    return ranks


@pytest.mark.parametrize("arch,W,block,n,S", [("llama", 2, 16, 300, 24), ("llama", 3, 8, 230, 300),
                                              ("mistral", 2, 8, 250, 300), ("mistral", 3, 16, 330, 24)])
def test_model_takes_questions_on_forks_like_the_control(arch, W, block, n, S):
    from duo_attention_b200.graph import DuoDecodeGraph

    model = _model(43 + W) if arch == "llama" else _mistral(47 + W)
    B, steps = 4, 10
    g = torch.Generator().manual_seed(W + S)
    prompt = torch.randint(0, 512, (1, n), generator=g).cuda()
    run = lambda ids, past: model(input_ids=ids, past_key_values=past, use_cache=True).logits
    cap = n + S + steps + 8
    with torch.no_grad():
        src = DuoAttentionStaticKVCache(model, GATES, 1, n + 8, SINK, RECENT, prefilling_chunk_size=n)
        run(prompt, src)
        donors, donors_g = _ranks(model, src, W, block, 1, cap), _ranks(model, src, W, block, 1, cap)
        control = RankGroup(_ranks(model, src, W, block, B, cap))
        forks = RankGroup([d.fork(B, S + steps + 4) for d in donors])
        forks_g = RankGroup([d.fork(B, S + steps + 4) for d in donors_g])
        P = forks.ranks[0].prefix_len
        assert P == n // (W * block) * (W * block) > 0 and (P // W) % 64 != 0  # a key tile across the donor's rows
        questions = torch.randint(0, 512, (B, S), generator=g).cuda()  # a different question per fork
        lf, lfg, lc = run(questions, forks), run(questions, forks_g), run(questions, control)
        assert torch.equal(lf, lc), "the question's logits differ from the control's"
        assert torch.equal(lfg, lf)
        assert forks.kv_seq_len == control.kv_seq_len == n + S
        graph = DuoDecodeGraph(model, forks_g)
        tok = lf[:, -1:].argmax(-1).contiguous()
        compared = 0
        for step in range(steps):
            le = run(tok, forks)
            lg = graph.step(tok)
            lc = run(tok, control)
            assert torch.equal(le, lg), f"step {step}: DuoDecodeGraph replay differs from eager decode"
            torch.testing.assert_close(le.float(), lc.float(), rtol=5e-2, atol=5e-2)
            top2 = lc.float().topk(2, -1).values
            clear = top2[..., 0] - top2[..., 1] > 0.1
            assert torch.equal(le.argmax(-1)[clear], lc.argmax(-1)[clear]), f"step {step}: greedy tokens differ"
            compared += int(clear.sum())
            tok = le[:, -1:].argmax(-1)
        assert compared >= B * steps // 4
        assert forks.kv_seq_len == forks_g.kv_seq_len == control.kv_seq_len == n + S + steps
