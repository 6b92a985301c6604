"""Per-rank attention of a follow-up chunk (the next user turn) on a sequence-sharded cache, on one GPU.

In the sequence-sharded layout (DuoSeqShardKVCache, DuoSeqShardINT4KVCache) every rank holds 1/world of every retrieval
head's positions (block-cyclic, block 1024) and the streaming heads in full.  A chunk longer than a decode step runs,
per layer and rank, duo_prefill_seq over the rank's slice (the wgmma prefill kernel's sequence-shard mode; INT4 caches
first dequantise the slice into a 16-bit image), then the row-scattered merge of the (O, log-sum-exp) partials.  The
per-rank attention is measured here by giving one H100 rank 0's slice; for INT4 the image dequantisation is part of
the timed launches.  The exchange cannot be measured on one GPU: its bytes per rank are computed, its time is "not
measured".  The reference line is the unsharded wgmma prefill kernel (duo_attention) on the same chunk over a
16-bit context that fits one GPU.

Workload: the Llama-3-8B-Instruct-Gradient-4194k architecture (32 layers, 32 q / 8 kv heads), its DuoAttention pattern
at sparsity 0.5, sink 64 / recent 256, bf16 activations, batch 1; chunks of 4,096 and 32,768 tokens; global contexts
of 1,048,576 (bf16 and INT4 at world 2, 4, 8) and 4,194,304 (INT4 at world 4, 8).  Cache contents are seeded random.

Per run: ms per chunk (CUDA events around the 32 layers' attention launches, after warm-up, averaged over --steps),
FLOP = 4 * 128 * (visible (query, key) pairs of rank 0: retrieval rows see local_len(0, ctx + t + 1) keys, streaming
rows sink + recent + t + 1), TFLOP/s, and the exchange bytes per rank (all_to_all of 516-byte partial rows out and in,
all_gather of 256-byte merged rows in).  The card's name and power limit are part of the output.

  python eval/efficiency/bench_seqshard_prefill.py [--steps 2] [--warmup 1] [--chunks 4096 32768] [--json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import gc
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402  (head pattern, sink / recent of the flagship benchmark)
from bench_ragged import gpu_info  # noqa: E402
from duo_attention_b200 import _C, tp  # noqa: E402
from duo_attention_b200.kv_cache import DuoKVCache, DuoSeqShardINT4KVCache, DuoSeqShardKVCache  # noqa: E402
from duo_attention_b200.seqshard import SeqShardPlan  # noqa: E402

PATTERN = "Llama-3-8B-Instruct-Gradient-4194k"
HQ, HKV, D, LAYERS = 32, 8, 128, 32
BLOCK = 1024
M1, M4 = 1 << 20, 1 << 22
# (kv format, world, global context); world 1: the unsharded wgmma kernel on a context that fits one GPU
RUNS = ([("same", 1, 1 << 17), ("same", 1, 1 << 19)] + [("same", w, M1) for w in (2, 4, 8)]
        + [("int4", w, M1) for w in (2, 4, 8)] + [("int4", w, M4) for w in (4, 8)])


class _Geometry(torch.nn.Module):
    """What the caches read from a model: one parameter (dtype, device) and the config."""

    def __init__(self, dev):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=torch.bfloat16, device=dev), requires_grad=False)
        self.config = types.SimpleNamespace(num_hidden_layers=LAYERS, num_attention_heads=HQ, num_key_value_heads=HKV,
                                            head_dim=D, hidden_size=HQ * D)


class _NoComm:
    """The merge is not part of the per-rank attention measured here."""

    max_rows = 1 << 30

    def merge(self, *args):
        raise AssertionError("not used")


def visible_pairs(world, ctx, S, mask):
    """(query, key) pairs rank 0 attends over the 32 layers for a chunk of S tokens after ctx tokens."""
    plan = SeqShardPlan(world, BLOCK) if world > 1 else None
    per_tok = sum(plan.local_len(0, ctx + t + 1) if plan else ctx + t + 1 for t in range(S))
    stream = sum(min(bench.SINK + bench.RECENT, ctx) + t + 1 for t in range(S))
    n_f = mask.sum(1)
    return float((n_f * 4 * per_tok + (HKV - n_f) * 4 * stream).sum())


def exchange_bytes(world, S, mask):
    """Bytes rank 0 sends + receives in the row-scattered merge of one chunk (32 layers)."""
    if world == 1:
        return 0.0
    tot = 0.0
    for nf in mask.sum(1):
        rows = int(nf) * 4 * S
        share = tp.scatter_counts(rows, world)
        tot += (rows - share[0]) * 516 + (world - 1) * share[0] * 516  # all_to_all out, in
        tot += (world - 1) * share[0] * 2 * D                         # all_gather in (bf16 rows)
    return tot


def run(fmt, world, ctx, S, mask, dev, steps, warmup):
    nf_list = [int((row > 0.5).sum()) for row in mask]
    if world == 1:
        cache = DuoKVCache(LAYERS, HQ, HKV, D, nf_list, 1, ctx + S, bench.SINK, bench.RECENT, torch.bfloat16, dev,
                           stage_cap=S)
    else:
        cls = DuoSeqShardKVCache if fmt == "same" else DuoSeqShardINT4KVCache
        cache = cls(_Geometry(dev), mask.tolist(), 1, ctx + S, bench.SINK, bench.RECENT,
                    seq=tp.SeqShardContext(0, world, BLOCK, _NoComm()))
        for l in range(LAYERS):
            cache._grow_layer(l, S)
    g = torch.Generator(device=dev).manual_seed(world * 7 + ctx % 97 + S)
    for t in cache.tensors:
        for name, v in t.items():
            if v.dtype == torch.uint8:
                v.random_(0, 256, generator=g)
            elif name.endswith("_scale"):
                v.uniform_(0.05, 0.25, generator=g)
            elif name.endswith("_zero"):
                v.uniform_(-2.0, -0.5, generator=g)
            else:
                v.normal_(generator=g)
    for l in range(LAYERS):
        cache.kv_seq_len_list[l], cache.total_list[l], cache.lo_list[l] = ctx, ctx, ctx - bench.RECENT
    qkv = (torch.randn(1, S, (HQ + 2 * HKV) * D, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    out = torch.empty(1, S, HQ, D, dtype=torch.bfloat16, device=dev)
    lib, stream, ws = cache.lib, torch.cuda.current_stream(dev).cuda_stream, cache.workspace
    if world > 1:
        po, pl = cache.partials(S)
        states = []
        for l in range(LAYERS):
            st = cache.state(l)
            st.device_state = None
            states.append(st)
    else:
        states = [cache.state(l) for l in range(LAYERS)]

    def step():
        for l in range(LAYERS):
            st = C.byref(states[l])
            if world == 1:
                _C.check(lib.duo_attention(cache.handles[l], st, qkv.data_ptr(), qkv.stride(1), out.data_ptr(), S,
                                           D ** -0.5, ws.data_ptr(), ws.numel(), stream))
                continue
            h = cache._dequant_scratch(l, S) if fmt == "int4" else cache.handles[l]
            _C.check(lib.duo_prefill_seq(h, st, qkv.data_ptr(), qkv.stride(1), out.data_ptr(), po.data_ptr(),
                                         pl.data_ptr(), S, D ** -0.5, ws.data_ptr(), ws.numel(), stream))

    for _ in range(warmup):
        step()
    torch.cuda.synchronize(dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for e0, e1 in ev:
        e0.record()
        step()
        e1.record()
    torch.cuda.synchronize(dev)
    times = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
    ms = sum(times) / steps
    flop = 4 * D * visible_pairs(world, ctx, S, mask)
    local = SeqShardPlan(world, BLOCK).local_len(0, ctx) if world > 1 else ctx
    res = dict(fmt=fmt, world=world, ctx=ctx, chunk=S, local_keys=local, ms=ms, ms_min=times[0], ms_max=times[-1],
               flop=flop, tflops=flop / (ms * 1e-3) / 1e12, exchange_mb=exchange_bytes(world, S, mask) / 1e6)
    del cache
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chunks", type=int, nargs="+", default=[4096, 32768])
    ap.add_argument("--json", action="store_true", help="also print one JSON line with every run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seqshard_prefill measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    name, power = gpu_info(dev)
    mask, sparsity = bench.head_pattern(PATTERN, 0.5)
    print(f"card: {name}, power limit: {power} W")
    print(f"workload: {PATTERN} architecture, sparsity {sparsity:.2f} (sum n_full = {int(mask.sum())}), "
          f"sink {bench.SINK} / recent {bench.RECENT}, bf16, batch 1, block {BLOCK}; rank 0's attention launches of "
          f"one follow-up chunk (32 layers), {args.steps} steps after {args.warmup} warm-up", flush=True)
    rows = []
    for S in args.chunks:
        for fmt, world, ctx in RUNS:
            r = run(fmt, world, ctx, S, mask, dev, args.steps, args.warmup)
            gc.collect()  # the run's cache (tens of GB) goes before the next one is allocated
            torch.cuda.empty_cache()
            rows.append(r)
            print(f"{r['fmt']:>5} world {r['world']} ctx {r['ctx']:>8} chunk {r['chunk']:>6}: {r['ms']:9.2f} ms "
                  f"({r['ms_min']:.2f} .. {r['ms_max']:.2f}), {r['tflops']:6.1f} TFLOP/s, local keys {r['local_keys']}, "
                  f"exchange {r['exchange_mb']:.1f} MB/rank", flush=True)
    print("exchange time and multi-GPU chunk time: not measured (one GPU)")
    if args.json:
        print(json.dumps(dict(card=name, power_limit_w=power, runs=rows)))


if __name__ == "__main__":
    main()
