"""Verify chunks of drafted tokens against one-token decode steps, on bench.py's workload.

Workload: the Llama-3-8B-Instruct-Gradient-1048k architecture (32 layers, 32 q / 8 kv heads, bf16), its DuoAttention
pattern at sparsity 0.5, sink 64 / recent 256, batch 1, 512K context (seeded random K/V: attention time does not depend
on the values).

* attention: the 32 layers' attention launches of one step, captured per arm in a CUDA graph.  Arms: the one-token
  step (duo_decode_fused) and verify chunks of S in {2, 4, 8, 16} tokens (S <= 4: duo_decode_verify, one launch per
  layer; S >= 8 at group 4: duo_rope_append + duo_attention_verify on the 64-row kernel).  The graphs are replayed
  alternately over --rounds rounds of --reps replays each, timed with CUDA events; every replay writes the same rows
  (nothing advances).  GB per step are the K/V bytes bench.py counts for one decode step at this context.
* model: one whole step with random weights, model(input_ids=[1, S], verify=True) against a plain decode step
  (--no-model skips it); each call is undone (accept(0) / evict_last(1)) so every repeat sees the same context.

tok/s at a mean accepted length m is DERIVED from the measured step times (m / step time): this bench has no drafter,
so acceptance is not measured.  The card's name and power limit are printed with the numbers.

  python eval/efficiency/bench_verify.py [--ctx 524288] [--rounds 5] [--reps 20] [--no-model] [--json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the flagship benchmark's head pattern, model and cache fill)
from duo_attention_b200 import _C  # noqa: E402
from duo_attention_b200.kv_cache import DuoAttentionStaticKVCache, DuoKVCache  # noqa: E402

HQ, HKV, D, LAYERS, SINK, RECENT = 32, 8, 128, 32, 64, 256
G = HQ // HKV
WIDTH = (HQ + 2 * HKV) * D
ARMS = [1, 2, 4, 8, 16]  # 1 = the one-token decode step


def gpu_info():
    import subprocess

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def attention_step(cache, S, qkv, cos, sin, out):
    """Enqueue the 32 layers' attention launches of one step of S tokens at the cache's (fixed) state."""
    lib, stream = cache.lib, torch.cuda.current_stream().cuda_stream
    ws = (cache.workspace.data_ptr(), cache.workspace.numel())
    for l in range(cache.num_layers):
        st = _C.CacheState(cache.kv_seq_len_list[l], cache.total_list[l], cache.lo_list[l], None)
        h, args = cache.handles[l], (qkv.data_ptr(), qkv.stride(1), cos.data_ptr(), sin.data_ptr(), _C.ROPE_HF)
        if S == 1:
            _C.check(lib.duo_decode_fused(h, C.byref(st), *args, out.data_ptr(), 1, D ** -0.5, *ws, stream))
        elif S * G <= _C.DECODE_MAX_Q:
            _C.check(lib.duo_decode_verify(h, C.byref(st), *args, out.data_ptr(), S, D ** -0.5, *ws, stream))
        else:
            _C.check(lib.duo_rope_append(h, C.byref(st), *args, S, stream))
            _C.check(lib.duo_attention_verify(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out.data_ptr(), S,
                                              D ** -0.5, *ws, stream))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def bench_attention(args, mask):
    dev = torch.device("cuda:0")
    nf = [int(x) for x in mask.sum(1)]
    cache = DuoKVCache(LAYERS, HQ, HKV, D, nf, 1, args.ctx + 64, SINK, RECENT, torch.bfloat16, dev, stage_cap=64)
    bench.fill_cache_synthetic(cache, args.ctx)
    g = torch.Generator(device=dev).manual_seed(3)
    graphs = {}
    for S in ARMS:
        qkv = torch.randn(1, S, WIDTH, generator=g, device=dev).to(torch.bfloat16)
        cos, sin = (torch.randn(S, D, generator=g, device=dev).to(torch.bfloat16) for _ in range(2))
        out = torch.empty(1, S, HQ, D, dtype=torch.bfloat16, device=dev)
        attention_step(cache, S, qkv, cos, sin, out)  # warm-up: kernel attributes, modules
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            attention_step(cache, S, qkv, cos, sin, out)
        graphs[S] = (gr, qkv, cos, sin, out)
    for S in ARMS:
        timed(graphs[S][0].replay, 3)
    ms = {S: [] for S in ARMS}
    for _ in range(args.rounds):
        for S in ARMS:
            ms[S].append(timed(graphs[S][0].replay, args.reps))
    del graphs, cache
    torch.cuda.empty_cache()
    return ms


def bench_model(args, mask):
    dev = torch.device("cuda:0")
    margs = types.SimpleNamespace(arch="llama3-8b-1048k", layers=LAYERS, kv_format="bf16")
    model, local_mask, _ = bench.build_model(margs, mask, 0, 1, dev)
    cache = DuoAttentionStaticKVCache(model, local_mask, 1, args.ctx + 64, SINK, RECENT)
    bench.fill_cache_synthetic(cache, args.ctx)
    g = torch.Generator(device=dev).manual_seed(5)
    ids = {S: torch.randint(0, 1000, (1, S), generator=g, device=dev) for S in ARMS}

    def step(S):
        if S == 1:
            model(input_ids=ids[1], past_key_values=cache, use_cache=True)
            cache.evict_last(1)
        else:
            model(input_ids=ids[S], past_key_values=cache, use_cache=True, verify=True)
            cache.accept(0)

    ms = {S: [] for S in ARMS}
    with torch.no_grad():
        for S in ARMS:
            timed(lambda: step(S), 2)
        for _ in range(args.rounds):
            for S in ARMS:
                ms[S].append(timed(lambda: step(S), args.model_reps))
    del model, cache
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctx", type=int, default=524288)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--model-reps", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_verify.py measures on a GPU; none is visible")
    name, power = gpu_info()
    mask, sparsity = bench.head_pattern()
    gb = bench.decode_bytes_per_token(mask, args.ctx) / 1e9
    res = {"gpu": name, "power_limit_w": power, "ctx": args.ctx, "sparsity": sparsity, "gb_per_step": gb,
           "attention": bench_attention(args, mask)}
    if not args.no_model:
        res["model"] = bench_model(args, mask)
    print(f"{name}, power limit {power} W; ctx {args.ctx}, sparsity {sparsity:.2f}, {gb:.2f} GB K/V per step")
    for part in ("attention", "model"):
        if part not in res:
            continue
        base = min(res[part][1])
        print(f"-- {part}: ms per step (min / median over {args.rounds} rounds)"
              + (", TB/s of the K/V bytes" if part == "attention" else ""))
        for S in ARMS:
            v = sorted(res[part][S])
            line = f"  S={S:2d}: {v[0]:8.3f} / {v[len(v) // 2]:8.3f} ms  x{v[0] / base:5.3f} of S=1"
            if part == "attention":
                line += f"  {gb / v[0]:5.2f} TB/s"
            if S > 1:  # derived, not measured: this bench has no drafter
                line += "  derived tok/s at mean accepted m: " + ", ".join(
                    f"m={m:g}: {m / v[0] * 1e3:7.1f}" for m in (1, 1.5, 2, 3, 4, 6) if m <= S)
            else:
                line += f"  (plain decode: {1e3 / v[0]:7.1f} tok/s)"
            print(line)
    if args.json:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
