"""Efficiency benchmark with the reference's protocol and output format (scope-table row f4).

Mirrors ``eval/efficiency/benchmark_static.py`` of mit-han-lab/duo-attention step by step (reference lines cited
inline): load a DuoAttention pattern, sparsify it, patch the model for the static KV cache, then time
  * the chunked pre-filling of ``max_length - 1`` tokens  (10 timed runs after 3 warm-ups, :58-75) and
  * one decoding step followed by ``evict_last(1)``       (100 timed runs after 50 warm-ups, :96-105)
with CUDA events, and write the same nine lines to ``<output_dir>/benchmark_result.txt`` (:107-119).

Differences, all additive: ``--random_init ARCH`` builds a random-weight model of a named architecture (there is no
network for checkpoints or tokenizers here; timing does not depend on the weights), ``--kv_format int4`` selects the
INT4 cache of demo/int4_kv.py, ``--dtype {fp16,bf16}`` the activation dtype (default fp16 for the INT4 cache, as in the
reference's INT4 demo, bf16 otherwise), ``--cuda_graph`` replays the decode step from a CUDA graph (DuoDecodeGraph).

    python eval/efficiency/benchmark_static.py --random_init llama3-8b-1048k \\
        --attn_load_dir attn_patterns/Llama-3-8B-Instruct-Gradient-1048k/lr=0.02-reg=0.05-ctx=1000_32000-multi_passkey10 \\
        --sparsity 0.5 --max_length 100000 --prefilling_chunk_size 32000 --output_dir outputs/bench
"""
from __future__ import annotations

import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARCHS = {  # the four models of the reference's efficiency figures (BASELINE.md), HF config values
    "llama3-8b-1048k": dict(kind="llama", hidden_size=4096, num_attention_heads=32, num_key_value_heads=8,
                            num_hidden_layers=32, intermediate_size=14336, vocab_size=128256, rope_theta=3580165449.0,
                            max_position_embeddings=1048576),
    "llama3-8b-4194k": dict(kind="llama", hidden_size=4096, num_attention_heads=32, num_key_value_heads=8,
                            num_hidden_layers=32, intermediate_size=14336, vocab_size=128256, rope_theta=45775831080.0,
                            max_position_embeddings=4194304),
    "llama2-7b-32k": dict(kind="llama", hidden_size=4096, num_attention_heads=32, num_key_value_heads=32,
                          num_hidden_layers=32, intermediate_size=11008, vocab_size=32000, rope_theta=10000.0,
                          max_position_embeddings=32768),
    "mistral-7b-v0.3": dict(kind="mistral", hidden_size=4096, num_attention_heads=32, num_key_value_heads=8,
                            num_hidden_layers=32, intermediate_size=14336, vocab_size=32768, rope_theta=1000000.0,
                            max_position_embeddings=32768),
}


def parse_args(argv=None):
    """The subset of duo_attn/utils.py:parse_args this script reads (same names and defaults), plus the additions."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--model_name", type=str, default=None)
    ap.add_argument("--attn_load_dir", type=str, default=None)
    ap.add_argument("--threshold", type=float, default=0.5)
    ap.add_argument("--sparsity", type=float, default=None)
    ap.add_argument("--max_length", type=int, default=4096)
    ap.add_argument("--prefilling_chunk_size", type=int, default=4096)
    ap.add_argument("--device", type=str, default="0")
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--output_dir", type=str, default="outputs")
    ap.add_argument("--random_init", type=str, default=None, choices=sorted(ARCHS))
    ap.add_argument("--num_layers", type=int, default=None, help="truncate the random-init model (smoke runs)")
    ap.add_argument("--kv_format", type=str, default="same", choices=["same", "int4"])
    ap.add_argument("--dtype", type=str, default=None, choices=["fp16", "bf16"],
                    help="activation dtype (default: fp16 with --kv_format int4, as in the reference's INT4 demo, "
                         "else bf16)")
    ap.add_argument("--cuda_graph", action="store_true")
    ap.add_argument("--ctx_steps", type=int, default=10)
    ap.add_argument("--gen_steps", type=int, default=100)
    args = ap.parse_args(argv)
    if (args.model_name is None) == (args.random_init is None):
        ap.error("give exactly one of --model_name (local checkpoint) and --random_init ARCH")
    return args


def format_result(gen_latency, gen_memory, ctx_latency, ctx_memory, model_name, max_length, sparsity,
                  prefilling_chunk_size, kv_cache_memory_usage):
    """The nine lines of benchmark_result.txt, in the reference's order and wording (benchmark_static.py:110-118)."""
    return "\n".join([
        f"Average generation time: {gen_latency:.4f} ms",
        f"Peak generation memory usage: {gen_memory:.4f} MB",
        f"Average context time: {ctx_latency:.4f} ms",
        f"Peak context memory usage: {ctx_memory:.4f} MB",
        f"Model name: {model_name}",
        f"Context length: {max_length}",
        f"Sparsity: {sparsity}",
        f"Prefilling chunk size: {prefilling_chunk_size}",
        f"KV cache memory usage: {kv_cache_memory_usage:.4f} MB",
    ]) + "\n"


def bench_func(func, num_steps=100, num_warmup_steps=5):
    """eval/efficiency/utils.py:8-30: warm up, reset the peak-memory counter, time num_steps calls between two CUDA
    events -> (average ms, peak MB)."""
    import torch

    for _ in range(num_warmup_steps):
        func()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(num_steps):
        func()
    end.record()
    torch.cuda.synchronize()
    avg = start.elapsed_time(end) / num_steps
    peak = torch.cuda.max_memory_allocated() / 1024 / 1024
    print(f"Average latency: {avg:.2f} ms")
    print(f"Peak memory usage: {peak:.2f} MB")
    return avg, peak


def build_model(args, dtype):
    import torch
    import transformers

    if args.model_name is not None:  # a local checkpoint directory (duo_attn/utils.py:get_model)
        return transformers.AutoModelForCausalLM.from_pretrained(args.model_name, torch_dtype=dtype,
                                                                 low_cpu_mem_usage=True, attn_implementation="eager")
    a = dict(ARCHS[args.random_init])
    kind = a.pop("kind")
    if args.num_layers:
        a["num_hidden_layers"] = args.num_layers
    cfg_cls, model_cls = ((transformers.LlamaConfig, transformers.LlamaForCausalLM) if kind == "llama" else
                          (transformers.MistralConfig, transformers.MistralForCausalLM))
    cfg = cfg_cls(head_dim=128, attn_implementation="eager", **a)
    with torch.device("meta"):
        model = model_cls(cfg)
    model = model.to(dtype).to_empty(device="cuda")
    g = torch.Generator(device="cuda").manual_seed(1234)
    with torch.no_grad():
        for _, prm in model.named_parameters():
            if prm.dim() == 1:
                prm.fill_(1.0)
            else:
                prm.normal_(0.0, 0.02, generator=g)
    rot = type(model.model.rotary_emb)
    model.model.rotary_emb = rot(config=cfg, device="cuda")  # buffers are not materialised by to_empty
    return model


def main(argv=None):
    args = parse_args(argv)
    import torch

    from duo_attn.patch import (DuoAttentionStaticKVCache, enable_llama_duo_attention_static_kv_cache_eval,
                                enable_mistral_duo_attention_static_kv_cache_eval)
    from duo_attn.utils import load_attn_pattern, seed_everything, sparsify_attention_heads

    if not torch.cuda.is_available():
        raise RuntimeError("benchmark_static needs a CUDA device (the CUDA kernels have no CPU fallback)")
    if args.seed is not None:
        seed_everything(args.seed)
    torch.cuda.set_device(int(args.device))
    dtype = torch.float16 if (args.dtype or ("fp16" if args.kv_format == "int4" else "bf16")) == "fp16" else torch.bfloat16
    with torch.no_grad():
        model = build_model(args, dtype)
    model.eval().cuda()

    sparsity = None
    if args.attn_load_dir is None:
        raise SystemExit("--attn_load_dir is required (the static cache is built from a DuoAttention pattern)")
    full_attention_heads, sink_size, recent_size = load_attn_pattern(args.attn_load_dir)
    full_attention_heads, sparsity = sparsify_attention_heads(full_attention_heads, None, args.sparsity)
    print(f"True Sparsity: {sparsity}")
    n_layers = model.config.num_hidden_layers
    full_attention_heads = full_attention_heads[:n_layers]
    if "llama" in model.config.model_type:  # benchmark_static.py:43
        enable_llama_duo_attention_static_kv_cache_eval(model, full_attention_heads)
    else:
        enable_mistral_duo_attention_static_kv_cache_eval(model, full_attention_heads)

    # the reference tokenises "a\n\n" * max_length and keeps max_length - 1 ids (:45-49); without a tokenizer the ids
    # are random (latency does not depend on them)
    g = torch.Generator().manual_seed(args.seed or 0)
    input_ids = torch.randint(0, model.config.vocab_size, (1, args.max_length - 1), generator=g).cuda()
    print(input_ids.shape)
    max_size = input_ids.size(1) + 5
    chunk = args.prefilling_chunk_size
    print(f"Max size: {max_size}, Prefilling chunk size: {chunk}")
    kv_cache = DuoAttentionStaticKVCache(model, full_attention_heads, 1, max_size, sink_size, recent_size,
                                         prefilling_chunk_size=chunk, kv_format=args.kv_format)

    def prefill():
        out = None
        with torch.no_grad():
            for i in range(0, input_ids.size(1), chunk):
                out = model(input_ids=input_ids[:, i: i + chunk], past_key_values=kv_cache, use_cache=True)
        return out

    def func1():
        prefill()
        kv_cache.clear()

    ctx_latency, ctx_memory = bench_func(func1, num_steps=args.ctx_steps, num_warmup_steps=3)
    kv_cache.clear()
    outputs = prefill()
    print(f"Peak memory usage in the pre-filling stage: {torch.cuda.max_memory_allocated() / 1024 / 1024:.2f} MB")
    pred_token_idx = outputs.logits[:, -1, :].argmax(dim=-1).unsqueeze(1)

    if args.cuda_graph:
        from duo_attention_b200.graph import DuoDecodeGraph

        graph = DuoDecodeGraph(model, kv_cache)

        def func2():
            graph.step(pred_token_idx)
            kv_cache.evict_last(1)
            graph.resync()
    else:
        def func2():
            with torch.no_grad():
                model(input_ids=pred_token_idx, past_key_values=kv_cache, use_cache=True)
            kv_cache.evict_last(1)

    gen_latency, gen_memory = bench_func(func2, num_steps=args.gen_steps, num_warmup_steps=max(5, args.gen_steps // 2))
    kv_mb = kv_cache.memory_usage / 1024 / 1024
    text = format_result(gen_latency, gen_memory, ctx_latency, ctx_memory, args.model_name or args.random_init,
                         args.max_length, sparsity, chunk, kv_mb)
    print(text, end="")
    if args.output_dir is not None:
        os.makedirs(args.output_dir, exist_ok=True)
        with open(os.path.join(args.output_dir, "benchmark_result.txt"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
