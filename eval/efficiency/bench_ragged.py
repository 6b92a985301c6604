"""Ragged-batch decode on one GPU: a batch of rows at different lengths decoded together (DuoRaggedKVCache, one
duo_decode_ragged launch per layer, CUDA-graph replay) against the same rows decoded one at a time at batch 1.
With --kv int4 the caches hold the INT4 format (DuoRaggedINT4KVCache, one duo_decode_ragged_int4 launch per layer;
batch 1: DuoAttentionStaticINT4KVCache), 136 B per (head, key) instead of 512 B, and the uniform batch is also
decoded through a batch-8 DuoAttentionStaticINT4KVCache (duo_decode_fused): at equal lengths that launch makes the
same partition and does the same work, so the difference is the cost of the ragged kernel's row search.

Workload: the Llama-3-8B-Instruct-Gradient-1048k architecture (random init, bf16), its DuoAttention pattern at
sparsity 0.5, sink 64 / recent 256.  Two batches of 8 rows with the same total tokens:
  skewed : one 524288-token row and seven 32768-token rows
  uniform: eight 94208-token rows
With --capacity uniform (the default) the cache keeps one capacity for every row ([batch][heads][capacity][128]), so
the skewed batch reserves 8 x 512K rows per retrieval head: a full 32-layer model of it does not fit in 80 GB.  With
--capacity per-row every row gets a region of its own length plus the step padding in one retrieval pool per layer
(duo_decode_ragged_pooled), so the batches reserve what they hold.  The script decodes the first --layers layers of
the architecture (default: as many as fit next to the skewed batch at that capacity) for every configuration, so the
numbers compare like with like.  The caches are filled with seeded random K/V through the row views: decode time
does not depend on the values.

Reported per configuration: graph-replayed step time and tokens/s; the summed CUDA-event time of the attention
launches of one (eager) step and the attention bandwidth (algorithmic K+V bytes / that time); for the batches, the
same rows decoded one at a time at batch 1 (sum of their step times).  The card's name and power limit are part of
the output.

--ab-runs R replaces all of the above by a cost comparison at identical lengths (the skewed batch) and layer count:
the pooled launch (per-row capacities) against the uniform-capacity ragged launch, the two arms alternating R times
each in this one process.  Per run it reports the graph-replayed step time and the attention time of one eager step
averaged over 10 steps; then per arm the mean and the spread (max - min) over the runs, and the pooled / uniform ratio.

  python eval/efficiency/bench_ragged.py [--kv {bf16,int4}] [--capacity {uniform,per-row}] [--steps 20] [--warmup 3]
                                         [--layers N] [--skip-batch1] [--ab-runs R]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the flagship benchmark's model builder and head pattern)
from duo_attention_b200.graph import DuoDecodeGraph  # noqa: E402
from duo_attention_b200.kv_cache import (DuoAttentionStaticINT4KVCache, DuoAttentionStaticKVCache,  # noqa: E402
                                         DuoRaggedINT4KVCache, DuoRaggedKVCache)

SKEWED = [524288] + [32768] * 7
UNIFORM = [sum(SKEWED) // 8] * 8
# K + V of one token of one head: bf16, or INT4 (2 x (64 B codes + fp16 scale + fp16 zero))
ROW_BYTES = {"bf16": 128 * 2 * 2, "int4": 2 * (64 + 2 + 2)}


def gpu_info(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def attention_bytes(mask, lengths, sink, recent, row_bytes):
    """Algorithmic K+V bytes of one decode step: retrieval heads read len + 1 rows, streaming heads
    min(len, sink + recent) + 1."""
    tot = 0
    for row in mask:
        nf = int((row > 0.5).sum())
        ns = len(row) - nf
        for L in lengths:
            tot += (nf * (L + 1) + ns * (min(L, sink + recent) + 1)) * row_bytes
    return tot


def fill(cache_rows, tensors, lengths, sink, recent, seed=7):
    g = torch.Generator(device=tensors[0]["full_k"].device).manual_seed(seed)
    for t in tensors:
        for v in t.values():
            if v.numel():
                if v.dtype == torch.uint8:  # INT4 codes
                    v.random_(0, 256, generator=g)
                else:
                    v.normal_(generator=g)
    for r, L in zip(cache_rows, lengths):
        for l in range(r.num_layers):
            r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l] = L, L, max(sink, L - recent)


def time_steps(model, cache, B, steps, warmup, eager=3, attn_steps=1):
    """(ms per graph-replayed step, summed ms of the attention launches of one eager step, averaged over the last
    ``attn_steps`` of ``eager`` eager steps)."""
    tok = torch.zeros(B, 1, dtype=torch.long, device=cache.device)
    snap = cache.snapshot_state() if isinstance(cache, DuoRaggedKVCache) else None
    with torch.no_grad():
        cache.profile_events = []
        for _ in range(eager):  # eager steps: the attention launches are bracketed by CUDA events
            model(input_ids=tok, past_key_values=cache, use_cache=True)
            cache.evict_last(1)
        torch.cuda.synchronize()
        n = cache.num_layers
        attn_ms = sum(a.elapsed_time(b) for a, b in cache.profile_events[-n * attn_steps:]) / attn_steps
        cache.profile_events = None
        graph = DuoDecodeGraph(model, cache)
        for _ in range(warmup):
            graph.step(tok)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            graph.step(tok)
        e1.record()
        torch.cuda.synchronize()
    del graph
    if snap is not None:
        cache.restore_state(snap)
    return e0.elapsed_time(e1) / steps, attn_ms


def fit_layers(mask, caps, budget_bytes, row_bytes):
    """Layers whose caches fit in ``budget_bytes`` when the 8 rows reserve ``caps`` tokens per retrieval head."""
    per = [int((row > 0.5).sum()) * sum(caps) * row_bytes + 8 * 8 * (bench.SINK + bench.RECENT + 64) * row_bytes
           for row in mask]
    n, used = 0, 0
    while n < len(per) and used + per[n] <= budget_bytes:
        used += per[n]
        n += 1
    return max(1, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--kv", choices=["bf16", "int4"], default="bf16")
    ap.add_argument("--capacity", choices=["uniform", "per-row"], default="uniform")
    ap.add_argument("--skip-batch1", action="store_true", help="skip the rows-one-at-a-time comparison")
    ap.add_argument("--ab-runs", type=int, default=0, help="pooled vs uniform-capacity cost comparison, R runs per arm")
    args = ap.parse_args()
    per_row = args.capacity == "per-row"
    int4 = args.kv == "int4"
    row_bytes = ROW_BYTES[args.kv]
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    name, power = gpu_info(dev)
    sink, recent = bench.SINK, bench.RECENT
    mask_all, sparsity = bench.head_pattern()
    pad = args.steps + args.warmup + 64
    # tokens each row reserves per retrieval head: the longest row's for one capacity, its own with per-row capacities
    # (the A/B comparison holds the uniform-capacity arm, whatever --capacity says)
    caps = [L + pad for L in SKEWED] if per_row and not args.ab_runs else [max(SKEWED) + pad] * len(SKEWED)
    if args.layers is None:
        free = torch.cuda.mem_get_info(dev)[0]
        # uniform: weights of a few layers, embeddings, head; per-row: room for all 32 layers' weights (~16 GB bf16)
        args.layers = fit_layers(mask_all, caps, free - (20 if per_row else 12) * 2 ** 30, row_bytes)
    mask = mask_all[: args.layers]
    margs = types.SimpleNamespace(arch="llama3-8b-1048k", layers=args.layers, kv_format="bf16")
    model, mask, _ = bench.build_model(margs, mask, 0, 1, dev)
    results = {"gpu": name, "power_limit_w": power, "kv": args.kv, "capacity": args.capacity, "layers": args.layers,
               "sparsity": sparsity, "sink": sink, "recent": recent, "steps": args.steps}
    ragged_cls = DuoRaggedINT4KVCache if int4 else DuoRaggedKVCache

    def ragged_cache(lengths, pooled):
        size = [L + pad for L in lengths] if pooled else max(lengths) + pad
        c = ragged_cls(model, mask, len(lengths), size, sink, recent)
        fill(c.rows, c.tensors, lengths, sink, recent)
        c.sync_device_state()
        return c

    if args.ab_runs:
        runs = {"pooled": [], "uniform": []}
        for i in range(2 * args.ab_runs):  # alternate the arms: pooled, uniform, pooled, ...
            arm = "pooled" if i % 2 == 0 else "uniform"
            cache = ragged_cache(SKEWED, arm == "pooled")
            ms, attn_ms = time_steps(model, cache, len(SKEWED), args.steps, args.warmup, eager=12, attn_steps=10)
            del cache
            gc.collect()
            torch.cuda.empty_cache()
            runs[arm].append({"step_ms": round(ms, 4), "attn_ms": round(attn_ms, 4)})
            print(f"[ab {arm}] {json.dumps(runs[arm][-1])}", file=sys.stderr)
        for arm, rs in runs.items():
            for k in ("step_ms", "attn_ms"):
                v = [r[k] for r in rs]
                results[f"{arm}_{k}"] = {"runs": v, "mean": round(sum(v) / len(v), 4), "spread": round(max(v) - min(v), 4)}
        for k in ("step_ms", "attn_ms"):
            results[f"pooled_vs_uniform_{k}"] = round(results[f"pooled_{k}"]["mean"] / results[f"uniform_{k}"]["mean"], 4)
        results["lengths"] = SKEWED
        print(json.dumps(results))
        return

    def static_cache(batch, size):
        if int4:
            return DuoAttentionStaticINT4KVCache(model, mask, batch, size, sink, recent, 64)
        return DuoAttentionStaticKVCache(model, mask, batch, size, sink, recent)

    def timed_static(batch, L):
        """(ms per step, attention ms) of a batch of `batch` rows at L through the static cache."""
        c = static_cache(batch, L + pad)
        fill([c], c.tensors, [L], sink, recent)
        c.sync_device_state()
        out = time_steps(model, c, batch, args.steps, args.warmup)
        del c
        gc.collect()
        torch.cuda.empty_cache()
        return out

    for label, lengths in (("skewed", SKEWED), ("uniform", UNIFORM)):
        B = len(lengths)
        cache = ragged_cache(lengths, per_row)
        pool_gb = round(sum(v.numel() * v.element_size() for t in cache.tensors for k, v in t.items()
                            if k.startswith("full")) / 1e9, 2)
        ms, attn_ms = time_steps(model, cache, B, args.steps, args.warmup)
        del cache
        gc.collect()  # the rows and the parent reference each other
        torch.cuda.empty_cache()
        byts = attention_bytes(mask, lengths, sink, recent, row_bytes)
        results[label] = {
            "lengths": lengths, "step_ms": round(ms, 3), "tok_s": round(B / ms * 1e3, 1),
            "attn_ms": round(attn_ms, 3), "attn_GBps": round(byts / (attn_ms * 1e-3) / 1e9, 1),
            "kv_GB": round(byts / 1e9, 2), "retrieval_reserved_GB": pool_gb,
        }
        if not args.skip_batch1:
            seq_ms = 0.0
            for L in sorted(set(lengths)):  # the same rows one at a time at batch 1
                ms1, _ = timed_static(1, L)
                seq_ms += ms1 * lengths.count(L)
            results[label].update({"batch1_sum_step_ms": round(seq_ms, 3), "batch1_tok_s": round(B / seq_ms * 1e3, 1)})
        if int4 and len(set(lengths)) == 1:  # the same batch through duo_decode_fused
            fms, fattn_ms = timed_static(B, lengths[0])
            results[label].update({"fused_step_ms": round(fms, 3), "fused_attn_ms": round(fattn_ms, 3),
                                   "fused_attn_GBps": round(byts / (fattn_ms * 1e-3) / 1e9, 1)})
        print(f"[{label}] {json.dumps(results[label])}", file=sys.stderr)
    results["skewed_vs_uniform_attn_bw"] = round(results["skewed"]["attn_GBps"] / results["uniform"]["attn_GBps"], 3)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
