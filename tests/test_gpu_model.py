"""Model-level parity: random-init HF Llama / Mistral patched through the drop-in API
(enable_duo_attention_eval) vs (a) the CPU oracle model that restates the reference driver
(tuple_kv_cache.py:241-490 + llama.py:146-306) and (b) unpatched HF eager attention when every head is a
retrieval head (weight-reorder invariance)."""
import copy

import numpy as np
import pytest
import torch

from duo_attn.patch import DuoAttentionStaticKVCache, enable_duo_attention_eval
from duo_attn.patch import enable_llama_duo_attention_static_kv_cache_eval
from oracle import duo_oracle as O

pytestmark = pytest.mark.gpu


def tiny_model(kind="llama", layers=2, n_heads=4, n_kv=2, hidden=512, seed=0):
    torch.manual_seed(seed)
    if kind == "llama":
        from transformers import LlamaConfig, LlamaForCausalLM as M

        cfg = LlamaConfig(hidden_size=hidden, num_attention_heads=n_heads, num_key_value_heads=n_kv,
                          num_hidden_layers=layers, intermediate_size=1024, vocab_size=512,
                          max_position_embeddings=8192, rope_theta=10000.0, attn_implementation="eager")
    else:
        from transformers import MistralConfig, MistralForCausalLM as M

        cfg = MistralConfig(hidden_size=hidden, num_attention_heads=n_heads, num_key_value_heads=n_kv,
                            num_hidden_layers=layers, intermediate_size=1024, vocab_size=512, head_dim=128,
                            max_position_embeddings=8192, rope_theta=10000.0, sliding_window=None,
                            attn_implementation="eager")
    model = M(cfg).to(torch.bfloat16).eval()
    return model


SCHEDULE = [45, 1, 1, 30, 1, 1, 1, 20, 1, 1]


@pytest.mark.parametrize("kind", ["llama", "mistral"])
def test_patched_model_matches_oracle_model(kind):
    model = tiny_model(kind)
    gates = np.array([[0.9, 0.1], [0.2, 0.8]])
    sink, recent = 4, 12
    oracle = O.OracleModel(copy.deepcopy(model), gates, sink, recent)
    enable_duo_attention_eval(model, gates, sink, recent)
    model.cuda()
    g = torch.Generator().manual_seed(1)
    past_o, past_g = None, None
    with torch.no_grad():
        for S in SCHEDULE:
            ids = torch.randint(0, 512, (1, S), generator=g)
            lo, past_o = oracle(ids, past_o)
            out = model(input_ids=ids.cuda(), past_key_values=past_g, use_cache=True)
            past_g = out.past_key_values
            assert out.logits.shape == (1, 1, 512) and out.logits.dtype == torch.float32
            torch.testing.assert_close(out.logits.cpu(), lo, rtol=5e-2, atol=5e-2)
            assert past_g.kv_seq_len == past_o[0][0].shape[2]


def test_all_full_heads_equals_unpatched_hf():
    model = tiny_model("llama", seed=3)
    ref = copy.deepcopy(model).cuda()
    gates = np.ones((2, 2))
    enable_duo_attention_eval(model, gates, 4, 12)
    model.cuda()
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, 512, (1, 80), generator=g).cuda()
    with torch.no_grad():
        want = ref(input_ids=ids).logits[:, -1:, :].float()
        got = model(input_ids=ids, past_key_values=None, use_cache=True).logits
    torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-2)


def test_static_cache_protocol_like_benchmark_static():
    model = tiny_model("llama", seed=5)
    gates = np.array([[1.0, 0.0], [0.0, 1.0]])
    sink, recent = 8, 16
    oracle = O.OracleModel(copy.deepcopy(model), gates, sink, recent)
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    cache = DuoAttentionStaticKVCache(model, gates, 1, 200, sink, recent)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 512, (1, 150), generator=g)
    with torch.no_grad():
        past_o = None
        for i in range(0, 150, 64):  # chunked prefill, benchmark_static.py:68-77
            chunk = ids[:, i : i + 64]
            lo, past_o = oracle(chunk, past_o)
            out = model(input_ids=chunk.cuda(), past_key_values=cache, use_cache=True)
        assert out.logits.dtype == torch.bfloat16  # llama static eval keeps bf16 logits
        torch.testing.assert_close(out.logits.float().cpu(), lo, rtol=5e-2, atol=5e-2)
        tok = lo.argmax(-1)
        # decode + evict_last(1), benchmark_static.py:96-103.  The first step still sees the token that the
        # eviction then drops out of the recent window, so step 1 differs from steps 2.. in the reference too;
        # from step 2 on every repetition is identical.
        lo1, past1 = oracle(tok, past_o)
        outs = []
        for _ in range(4):
            out = model(input_ids=tok.cuda(), past_key_values=cache, use_cache=True)
            cache.evict_last(1)
            outs.append(out.logits.clone())
        torch.testing.assert_close(outs[0].float().cpu(), lo1, rtol=5e-2, atol=5e-2)
        past2 = tuple((f[:, :, :-1].contiguous(), s_[:, :, :-1].contiguous()) for f, s_ in past1)  # evict_last(1)
        lo2, _ = oracle(tok, past2)
        torch.testing.assert_close(outs[1].float().cpu(), lo2, rtol=5e-2, atol=5e-2)
        assert torch.equal(outs[1], outs[2]) and torch.equal(outs[2], outs[3])
        assert cache.kv_seq_len == 150
        assert cache.memory_usage > 0
        cache.clear()
        assert cache.kv_seq_len == 0
        with pytest.raises(ValueError, match="max size 200"):
            model(input_ids=torch.zeros(1, 201, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)


def test_cuda_graph_decode_matches_eager_decode():
    """DuoDecodeGraph (one captured step, device-resident cache occupancy) == the eager driver, token by token,
    across ring wrap-around and an evict_last in the middle."""
    from duo_attention_b200.graph import DuoDecodeGraph

    model = tiny_model("llama", seed=7)
    gates = np.array([[1.0, 0.0], [0.0, 1.0]])
    sink, recent = 4, 6
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    ca = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent)
    cb = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent)
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 512, (1, 37), generator=g).cuda()
    with torch.no_grad():
        model(input_ids=ids, past_key_values=ca, use_cache=True)
        model(input_ids=ids, past_key_values=cb, use_cache=True)
        graph = DuoDecodeGraph(model, cb)
        toks = torch.randint(0, 512, (20, 1, 1), generator=g).cuda()
        for i in range(20):
            want = model(input_ids=toks[i], past_key_values=ca, use_cache=True).logits
            got = graph.step(toks[i])
            torch.testing.assert_close(got.float(), want.float(), rtol=0, atol=0, msg=lambda m: f"step {i}: {m}")
            assert ca.kv_seq_len == cb.kv_seq_len
            if i == 9:
                ca.evict_last(1)
                cb.evict_last(1)
                graph.resync()


def test_int4_cuda_graph_decode_matches_eager():
    """Device-resident occupancy (dstate) path of the INT4 decode kernels: graph replay == eager, token by token."""
    from duo_attention_b200.graph import DuoDecodeGraph

    model = tiny_model("llama", seed=7).to(torch.float16)
    gates = np.array([[1.0, 0.0], [0.0, 1.0]])
    sink, recent = 4, 6
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    ca = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent, kv_format="int4")
    cb = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent, kv_format="int4")
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 512, (1, 37), generator=g).cuda()
    with torch.no_grad():
        model(input_ids=ids, past_key_values=ca, use_cache=True)
        model(input_ids=ids, past_key_values=cb, use_cache=True)
        graph = DuoDecodeGraph(model, cb)
        toks = torch.randint(0, 512, (20, 1, 1), generator=g).cuda()
        for i in range(20):
            want = model(input_ids=toks[i], past_key_values=ca, use_cache=True).logits
            got = graph.step(toks[i])
            torch.testing.assert_close(got.float(), want.float(), rtol=0, atol=0, msg=lambda m: f"step {i}: {m}")
            if i == 9:
                ca.evict_last(1)
                cb.evict_last(1)
                graph.resync()


def test_int4_model_through_the_drop_in_cache_class():
    """Model level, INT4 KV: enable_*_static_kv_cache_eval + DuoAttentionStaticINT4KVCache (the demo's class name and
    constructor, demo/int4_kv.py:115-260) vs the oracle model whose attention core restates
    demo/w8a8kv4_llama.py:215-278 (first call raw fp16, later calls the quantise->dequantise round trip)."""
    from duo_attn.patch import DuoAttentionStaticINT4KVCache

    model = tiny_model("llama", seed=11).to(torch.float16)
    gates = np.array([[1.0, 0.0], [1.0, 1.0]])
    sink, recent = 8, 16
    oracle = O.OracleModel(copy.deepcopy(model), gates, sink, recent, kv_format="int4")
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    cache = DuoAttentionStaticINT4KVCache(model, gates, 1, 512, sink, recent, 160)
    g = torch.Generator().manual_seed(5)
    past_o = None
    with torch.no_grad():
        for S in [150, 1, 1, 140, 1, 33, 1, 1]:  # 140: a >= 128-token chunk over an INT4 cache (wgmma prefill kernel on the fp16 image)
            ids = torch.randint(0, 512, (1, S), generator=g)
            lo, past_o = oracle(ids, past_o)
            out = model(input_ids=ids.cuda(), past_key_values=cache, use_cache=True)
            torch.testing.assert_close(out.logits.float().cpu(), lo, rtol=5e-2, atol=5e-2)
            assert cache.kv_seq_len == past_o[0][0].shape[2]
    assert cache.memory_usage > 0


def test_graph_step_raises_when_the_cache_is_full():
    """Replaying the captured step past the capacity must raise the reference's ValueError (static_kv_cache.py:112-115),
    not write past the allocation."""
    from duo_attention_b200.graph import DuoDecodeGraph

    model = tiny_model("llama", seed=9)
    gates = np.array([[1.0, 0.0], [0.0, 1.0]])
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    cache = DuoAttentionStaticKVCache(model, gates, 1, 40, 4, 6, prefilling_chunk_size=37)
    ids = torch.randint(0, 512, (1, 37)).cuda()
    with torch.no_grad():
        model(input_ids=ids, past_key_values=cache, use_cache=True)
        graph = DuoDecodeGraph(model, cache)
        tok = torch.zeros(1, 1, dtype=torch.long, device="cuda")
        for _ in range(3):
            graph.step(tok)
        assert cache.kv_seq_len == 40
        with pytest.raises(ValueError, match="Trying to put 1 KVs into a cache with max size 40"):
            graph.step(tok)
        cache.clear()
        with pytest.raises(ValueError, match="captured in a DuoDecodeGraph"):  # 39 tokens > staging capacity 37
            model(input_ids=torch.zeros(1, 39, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)


@pytest.mark.parametrize("kind", ["llama", "mistral"])
def test_static_path_with_flashinfer_rope_matches_reference_run_logits(kind):
    """enable_*_static_kv_cache_eval(..., rope="flashinfer") against the logits the REFERENCE's static driver produced
    (tests/golden/model_{llama,mistral}_static.npz: static_kv_cache.py:318-805 + flashinfer-style fp32 RoPE, run in fp32
    by tests/golden/make_golden.py) — product (bf16, GPU) vs reference directly, without the oracle in between."""
    import os

    import golden_cases as GC
    from duo_attn.patch import enable_mistral_duo_attention_static_kv_cache_eval

    case = next(c for c in GC.MODEL_CASES if c["name"] == f"{kind}_static")
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", f"model_{kind}_static.npz"))
    model, ids, _ = GC.make_tiny_model(case)
    model = model.to(torch.bfloat16)
    gates = np.array(case["gates"])
    enable = (enable_llama_duo_attention_static_kv_cache_eval if kind == "llama"
              else enable_mistral_duo_attention_static_kv_cache_eval)
    enable(model, gates, rope="flashinfer")
    model.cuda()
    cache = DuoAttentionStaticKVCache(model, gates, 1, case["max_size"], case["sink"], case["recent"],
                                      prefilling_chunk_size=max(case["chunks"]))
    with torch.no_grad():
        for i, x in enumerate(ids):
            out = model(input_ids=x.cuda(), past_key_values=cache, use_cache=True)
            # bf16 weights/activations on the GPU vs the reference run in fp32 (logits up to ~5): bf16-level agreement
            torch.testing.assert_close(out.logits.float().cpu()[0, 0], torch.from_numpy(gold["logits"][0, i]),
                                       rtol=5e-2, atol=1.2e-1)
            ev = case.get("evict_after", {}).get(i, 0)
            if ev:
                cache.evict_last(ev)
            assert cache.kv_seq_len == int(gold["lens"][i][0])
