"""Per-rank attention of a sequence-sharded decode step over an INT4 KV cache, on one GPU.

In the sequence-sharded layout (DuoSeqShardINT4KVCache) every rank holds 1/world of every retrieval head's positions
(block-cyclic, block 1024) and the streaming heads in full; a decode step is one duo_decode_fused_seq_int4 launch per
layer on each rank, then one exchange of the (O, log-sum-exp) partials.  The per-rank part is measured here by giving
one H100 rank 0's slice (rank 0 also owns the new position: it quantises and appends it).  The exchange and the
multi-GPU step time cannot be measured on one GPU: they are reported as "not measured".

Workload: the Llama-3-8B-Instruct-Gradient-4194k architecture (32 layers, 32 q / 8 kv heads), its DuoAttention pattern
at sparsity 0.5, sink 64 / recent 256, bf16 activations, batch 1.  The INT4 codes, scales and zeros are seeded random
values (decode time does not depend on them).  Runs: world 2, 4, 8 at global contexts 1,048,576 and 4,194,304; world 1
(the unsharded duo_decode_fused on an INT4 cache) at 1,048,576 — at 4,194,304 one GPU would need 73 GB of INT4 KV next
to 16 GB of weights, which does not fit in 80 GB.

Per run: ms per step (CUDA events around the 32 layers' attention launches, after warm-up, averaged over --steps
steps), the per-rank algorithmic bytes sum_l (n_f * local_len + n_s * (sink + recent + 1)) * 136 B (local_len: the rows
of rank 0's slice the step reads, the new one included), GB/s, and the ratio of the per-rank time to world 1 at the same
context.  The card's name and power limit are part of the output.

  python eval/efficiency/bench_seqshard_int4.py [--steps 50] [--warmup 10] [--json]
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
from duo_attention_b200.kv_cache import DuoKVCache, DuoSeqShardINT4KVCache  # noqa: E402
from duo_attention_b200.seqshard import SeqShardPlan  # noqa: E402

PATTERN = "Llama-3-8B-Instruct-Gradient-4194k"
HQ, HKV, D, LAYERS = 32, 8, 128, 32
BLOCK = 1024
ROW_BYTES = 2 * (64 + 2 + 2)  # K + V of one INT4 row: codes + fp16 scale + fp16 zero
RUNS = [(1, 1 << 20)] + [(w, ctx) for ctx in (1 << 20, 1 << 22) for w in (2, 4, 8)]


class _Geometry(torch.nn.Module):
    """What the caches read from a model: one parameter (dtype, device) and the config."""

    def __init__(self, dev):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=torch.bfloat16, device=dev), requires_grad=False)
        self.config = types.SimpleNamespace(num_hidden_layers=LAYERS, num_attention_heads=HQ, num_key_value_heads=HKV,
                                            head_dim=D, hidden_size=HQ * D)


class _NoComm:
    """The merge is not part of the per-rank attention measured here."""

    def merge(self, *args):
        raise AssertionError("not used")


def make_cache(world, ctx, mask, dev):
    nf_list = [int((row > 0.5).sum()) for row in mask]
    if world == 1:
        return DuoKVCache(LAYERS, HQ, HKV, D, nf_list, 1, ctx + 8, bench.SINK, bench.RECENT, torch.bfloat16, dev,
                          stage_cap=8, kv_format="int4")
    return DuoSeqShardINT4KVCache(_Geometry(dev), mask.tolist(), 1, ctx + 8, bench.SINK, bench.RECENT,
                                  seq=tp.SeqShardContext(0, world, BLOCK, _NoComm()))


def run(world, ctx, mask, dev, steps, warmup):
    cache = make_cache(world, ctx, mask, dev)
    g = torch.Generator(device=dev).manual_seed(world * 7 + ctx % 97)
    for t in cache.tensors:
        for name, v in t.items():
            if v.dtype == torch.uint8:
                v.random_(0, 256, generator=g)
            elif name.endswith("_scale"):
                v.uniform_(0.05, 0.25, generator=g)
            else:
                v.uniform_(-2.0, -0.5, generator=g)
    for l in range(LAYERS):
        cache.kv_seq_len_list[l], cache.total_list[l], cache.lo_list[l] = ctx, ctx, ctx - bench.RECENT
    width = (HQ + 2 * HKV) * D
    qkv = (torch.randn(1, 1, width, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    ang = ctx * torch.pow(torch.tensor(500000.0, device=dev), -torch.arange(0, D, 2, device=dev) / D)
    cos = torch.cat([ang.cos(), ang.cos()])[None].to(torch.bfloat16).contiguous()
    sin = torch.cat([ang.sin(), ang.sin()])[None].to(torch.bfloat16).contiguous()
    out = torch.empty(1, 1, HQ, D, dtype=torch.bfloat16, device=dev)
    lib, stream = cache.lib, torch.cuda.current_stream(dev).cuda_stream
    ws = cache.workspace
    states = [cache.state(l) for l in range(LAYERS)]  # the same occupancy every step: rank 0 rewrites its new row
    if world > 1:
        po, pl = cache.part_o[:, :1], cache.part_lse[:, :1]

    def step():
        for l in range(LAYERS):
            h, st = cache.handles[l], C.byref(states[l])
            if world == 1:
                _C.check(lib.duo_decode_fused(h, st, qkv.data_ptr(), qkv.stride(1), cos.data_ptr(), sin.data_ptr(),
                                              _C.ROPE_HF, out.data_ptr(), 1, D ** -0.5, ws.data_ptr(), ws.numel(),
                                              stream))
            else:
                _C.check(lib.duo_decode_fused_seq_int4(h, st, qkv.data_ptr(), qkv.stride(1), cos.data_ptr(),
                                                       sin.data_ptr(), _C.ROPE_HF, out.data_ptr(), po.data_ptr(),
                                                       pl.data_ptr(), D ** -0.5, ws.data_ptr(), ws.numel(), stream))

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
    plan = SeqShardPlan(max(world, 1), BLOCK)
    local = plan.local_len(0, ctx + 1) if world > 1 else ctx + 1
    n_f = mask.sum(1)
    n_s = mask.shape[1] - n_f
    nbytes = float(((n_f * local + n_s * (bench.SINK + bench.RECENT + 1)) * ROW_BYTES).sum())
    kv_gb = cache.memory_usage / 1e9
    return dict(world=world, ctx=ctx, local_len=local, ms=ms, ms_min=times[0], ms_max=times[-1], bytes=nbytes,
                gbps=nbytes / (ms * 1e-3) / 1e9, kv_gb=kv_gb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", action="store_true", help="also print one JSON line with every run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seqshard_int4 measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    name, power = gpu_info(dev)
    mask, sparsity = bench.head_pattern(PATTERN, 0.5)
    print(f"card: {name}, power limit: {power} W")
    print(f"workload: {PATTERN} architecture, sparsity {sparsity:.2f} (sum n_full = {int(mask.sum())}), "
          f"sink {bench.SINK} / recent {bench.RECENT}, bf16, batch 1, block {BLOCK}; per-rank attention of one decode "
          f"step (32 layers), {args.steps} steps after {args.warmup} warm-up")
    rows = []
    base = {}
    for world, ctx in RUNS:
        r = run(world, ctx, mask, dev, args.steps, args.warmup)
        gc.collect()  # the run's cache (tens of GB) goes before the next one is allocated
        torch.cuda.empty_cache()
        if world == 1:
            base[ctx] = r["ms"]
        r["vs_world1"] = r["ms"] / base[ctx] if ctx in base else None
        rows.append(r)
    print(f"{'world':>5} {'context':>9} {'local keys':>10} {'ms/step':>8} {'min':>7} {'max':>7} {'MB/rank':>9} "
          f"{'GB/s':>7} {'KV GB/rank':>10} {'vs world 1':>10}")
    for r in rows:
        ratio = f"{r['vs_world1']:.3f}" if r["vs_world1"] is not None else "-"
        print(f"{r['world']:>5} {r['ctx']:>9} {r['local_len']:>10} {r['ms']:>8.3f} {r['ms_min']:>7.3f} "
              f"{r['ms_max']:>7.3f} {r['bytes'] / 1e6:>9.1f} {r['gbps']:>7.0f} {r['kv_gb']:>10.2f} {ratio:>10}")
    print(f"world 1 at {1 << 22}: not run (one GPU would hold "
          f"{float((mask.sum(1) * (1 << 22)).sum()) * ROW_BYTES / 1e9:.1f} GB of INT4 retrieval KV)")
    print("NVLink exchange of the partials and multi-GPU step time: not measured (one GPU)")
    if args.json:
        print(json.dumps(dict(card=name, power_limit_w=power, runs=rows)))


if __name__ == "__main__":
    main()
