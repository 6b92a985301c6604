"""Greedy speculative decoding through model(..., verify=True): a random bf16 Llama and an fp16 Mistral, on a static
batch-1 cache and a ragged batch-3 cache.  The drafts are a plain greedy run's tokens, corrupted at chosen positions so
that the accepted length varies by row and step.  The emitted tokens equal plain greedy decoding up to the first
position where its top two logits are within 0.1 of each other, and the verify logits at accepted positions match the
plain steps' logits."""
import numpy as np
import pytest
import torch

from duo_attention_b200.kv_cache import DuoAttentionStaticKVCache, DuoRaggedKVCache

pytestmark = pytest.mark.gpu
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])
SINK, RECENT, K = 4, 12, 4  # K drafts per step
TOL = dict(rtol=5e-2, atol=5e-2)


def tiny_model(kind, seed):
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
    from duo_attn.patch import enable_duo_attention_eval

    model = M(cfg).to(dtype).eval()
    enable_duo_attention_eval(model, GATES, SINK, RECENT)
    return model.cuda()


def plain_greedy(model, make_cache, prompts, steps):
    """Per row: the greedy tokens, the logits that chose them and their top-two margins (one-token steps)."""
    B = len(prompts)
    cache = make_cache()
    toks, logits = [[] for _ in range(B)], [[] for _ in range(B)]
    last = prefill(model, cache, prompts)
    for _ in range(steps):
        ids = torch.stack([lo.argmax(-1) for lo in last])[:, None]
        for b in range(B):
            toks[b].append(int(ids[b]))
        out = model(input_ids=ids.cuda(), past_key_values=cache, use_cache=True).logits[:, -1].float().cpu()
        last = list(out)
        for b in range(B):
            logits[b].append(out[b])
    return toks, logits


def prefill(model, cache, prompts):
    if isinstance(cache, DuoRaggedKVCache):
        return [model(input_ids=p.cuda(), past_key_values=cache.row(b), use_cache=True).logits[0, -1].float().cpu()
                for b, p in enumerate(prompts)]
    return list(model(input_ids=torch.cat(prompts).cuda(), past_key_values=cache, use_cache=True).logits[:, -1]
                .float().cpu())


def margin(lo):
    top = lo.topk(2).values
    return float(top[0] - top[1])


@pytest.mark.parametrize("layout", ["static", "ragged"])
@pytest.mark.parametrize("kind", ["llama", "mistral"])
def test_greedy_speculative_decoding_matches_plain_greedy(kind, layout):
    model = tiny_model(kind, 21)
    g = torch.Generator().manual_seed(4)
    B = 1 if layout == "static" else 3
    lens = [37] if B == 1 else [37, 70, 9]
    prompts = [torch.randint(0, 512, (1, n), generator=g) for n in lens]
    if layout == "static":
        make = lambda: DuoAttentionStaticKVCache(model, GATES, 1, 512, SINK, RECENT)
    else:
        make = lambda: DuoRaggedKVCache(model, GATES, 3, 512, SINK, RECENT)
    steps = 24
    with torch.no_grad():
        ref_toks, ref_logits = plain_greedy(model, make, prompts, steps * (K + 1) + K + 2)
        cache = make()
        last = prefill(model, cache, prompts)
        emitted = [[int(lo.argmax())] for lo in last]  # the next token of each row, not yet in the cache
        vlogits = [[] for _ in range(B)]
        rnd = np.random.default_rng(7)
        seen = set()
        for step in range(steps):
            ids = []
            for b in range(B):
                pos = len(emitted[b])  # drafts are plain greedy's tokens at the next positions, some corrupted
                drafts = list(ref_toks[b][pos : pos + K])
                drafts += [0] * (K - len(drafts))
                for i in range(K):
                    if rnd.random() < 0.3:
                        drafts[i] = (drafts[i] + 1 + b) % 512
                ids.append([emitted[b][-1]] + drafts)
            out = model(input_ids=torch.tensor(ids).cuda(), past_key_values=cache, use_cache=True, verify=True)
            assert out.logits.shape == (B, K + 1, 512)
            lo = out.logits.float().cpu()
            counts = []
            for b in range(B):
                a = 1
                while a <= K and ids[b][a] == int(lo[b, a - 1].argmax()):
                    a += 1
                vlogits[b] += list(lo[b, :a])
                emitted[b] += ids[b][1:a] + [int(lo[b, a - 1].argmax())]
                counts.append(a)
            cache.accept(counts[0] if layout == "static" else counts)
            seen.update(counts)
        assert len(seen) > 1, "the corrupted drafts should give different accepted lengths"
        for b in range(B):
            n = len(emitted[b])
            firm = next((i for i in range(n) if margin(ref_logits[b][i - 1] if i else last[b]) <= 0.1), n)
            assert emitted[b][:firm] == ref_toks[b][:firm], f"row {b}: greedy tokens differ before position {firm}"
            upto = min(firm, len(vlogits[b]))
            if upto:
                torch.testing.assert_close(torch.stack(vlogits[b][:upto]), torch.stack(ref_logits[b][:upto]), **TOL)
            n_now = cache.row_lengths[b] if layout == "ragged" else cache.kv_seq_len
            assert n_now == lens[b] + len(vlogits[b])
