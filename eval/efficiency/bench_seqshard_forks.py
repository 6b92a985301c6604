"""Parallel sampling over a 1M-token prompt on sequence-sharded caches: rank 0 of world 8, on one GPU.

B forks of one prompt (DuoSeqShardKVCache.fork) read the donor's slice of the prompt in place: one
duo_decode_fused_seq_shared (two launches) per layer and step.  The alternative is a batch-B DuoSeqShardKVCache holding
B copies of the prompt (duo_decode_fused_seq).  Both are measured here as rank 0 of world 8 (131,072 local prompt
positions; rank 0 owns the new position, so it also appends).  The exchange (duo_seq_merge) is not part of either
arm and cannot be measured on one GPU: "not measured".

Workload: Llama-3-8B-Instruct-Gradient-1048k attention (32 layers, 32 q / 8 kv heads), its DuoAttention pattern at
sparsity 0.5, sink / recent of the flagship benchmark, bf16, seeded random K/V (decode time does not depend on them).
Timing: the 32 layers' launches of one step captured in a CUDA graph per arm; the arms are replayed alternately,
--steps replays each per round over --rounds rounds, CUDA events around every replay.  B copies of the prompt need
B x 8.6 GB per rank; where that does not fit next to the donor, the copies arm runs on fewer layers and its time and
bytes are scaled to 32 (marked "scaled").

  python eval/efficiency/bench_seqshard_forks.py [--steps 20] [--warmup 5] [--rounds 3] [--json]
"""
from __future__ import annotations

import argparse
import ctypes as C
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
from duo_attention_b200.kv_cache import DuoSeqShardKVCache  # noqa: E402
from duo_attention_b200.seqshard import SeqShardPlan  # noqa: E402

PATTERN = "Llama-3-8B-Instruct-Gradient-1048k"
HQ, HKV, D, LAYERS = 32, 8, 128, 32
WORLD, BLOCK, CTX = 8, 1024, 1 << 20
ROW_BYTES = 2 * D * 2  # K + V of one 16-bit row
BATCHES = [1, 2, 4, 8, 16, 17, 32]
COPY_BUDGET = 40e9  # bytes of prompt copies the copies arm may hold next to the donor


class _Geometry(torch.nn.Module):
    def __init__(self, dev, layers):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=torch.bfloat16, device=dev), requires_grad=False)
        self.config = types.SimpleNamespace(num_hidden_layers=layers, num_attention_heads=HQ,
                                            num_key_value_heads=HKV, head_dim=D, hidden_size=HQ * D)


class _NoComm:
    max_rows = 1 << 20

    def merge(self, *args):
        raise AssertionError("not used")


def filled(mask, batch, dev, g):
    c = DuoSeqShardKVCache(_Geometry(dev, len(mask)), mask.tolist(), batch, CTX + 64, bench.SINK, bench.RECENT,
                           seq=tp.SeqShardContext(0, WORLD, BLOCK, _NoComm()))
    for t in c.tensors:
        for v in t.values():
            v.normal_(generator=g)
    for l in range(c.num_layers):
        c.kv_seq_len_list[l], c.total_list[l], c.lo_list[l] = CTX, CTX, CTX - bench.RECENT
    return c


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def step_fn(cache, B, dev, g, donor=None):
    """The per-layer launches of one step at a fixed occupancy (rank 0 rewrites its new row every replay)."""
    width = (HQ + 2 * HKV) * D
    qkv = (torch.randn(B, 1, width, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    ang = CTX * torch.pow(torch.tensor(500000.0, device=dev), -torch.arange(0, D, 2, device=dev) / D)
    cos = torch.cat([ang.cos(), ang.cos()])[None].to(torch.bfloat16).contiguous()
    sin = torch.cat([ang.sin(), ang.sin()])[None].to(torch.bfloat16).contiguous()
    out = torch.empty(B, 1, HQ, D, dtype=torch.bfloat16, device=dev)
    po, pl = cache.partials(1)
    lib, ws = cache.lib, cache.workspace
    states = [cache.state(l) for l in range(cache.num_layers)]
    keep = (qkv, cos, sin, out, po, pl, states)

    def fn():
        stream = torch.cuda.current_stream(dev).cuda_stream
        for l in range(cache.num_layers):
            a = (C.byref(states[l]), qkv.data_ptr(), qkv.stride(1), cos.data_ptr(), sin.data_ptr(), _C.ROPE_HF,
                 out.data_ptr(), po.data_ptr(), pl.data_ptr(), D ** -0.5, ws.data_ptr(), ws.numel(), stream)
            if donor is None:
                _C.check(lib.duo_decode_fused_seq(cache.handles[l], *a))
            else:
                _C.check(lib.duo_decode_fused_seq_shared(cache.handles[l], donor.handles[l], cache.prefix_len, *a))
    fn.keep = keep
    return fn


def timed(graph, n):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for e0, e1 in ev:
        e0.record()
        graph.replay()
        e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=str, default=",".join(map(str, BATCHES)))
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seqshard_forks measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    name, power = gpu_info(dev)
    mask, sparsity = bench.head_pattern(PATTERN, 0.5)
    n_f = mask.sum(1)
    n_s = mask.shape[1] - n_f
    plan = SeqShardPlan(WORLD, BLOCK)
    local = plan.local_len(0, CTX)
    print(f"card: {name}, power limit: {power} W")
    print(f"workload: {PATTERN} attention, sparsity {sparsity:.2f}, sink {bench.SINK} / recent {bench.RECENT}, bf16, "
          f"rank 0 of world {WORLD} (block {BLOCK}): {local} local prompt positions of {CTX}")
    g = torch.Generator(device=dev).manual_seed(1)
    donor = filled(mask, 1, dev, g)
    stream_bytes = float((n_s * (bench.SINK + bench.RECENT + 1) * ROW_BYTES).sum())
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        forks = donor.fork(B, 64)
        blocks = (B * (HQ // HKV) + 63) // 64  # 64-row blocks of the prefix launch: each streams the prefix once
        fb = float((n_f * local * ROW_BYTES).sum()) * blocks + B * stream_bytes + B * float((n_f * ROW_BYTES).sum())
        per_copy = float((n_f * (local + 1) * ROW_BYTES).sum())
        layers = min(LAYERS, int(COPY_BUDGET / (B * per_copy / LAYERS)))
        fg = capture(step_fn(forks, B, dev, g, donor))
        copies = filled(mask[:layers], B, dev, g) if layers > 0 else None
        cg = capture(step_fn(copies, B, dev, g)) if copies is not None else None
        timed(fg, args.warmup)
        if cg:
            timed(cg, args.warmup)
        ft, ct = [], []
        for _ in range(args.rounds):  # arms alternated
            ft += timed(fg, args.steps)
            if cg:
                ct += timed(cg, args.steps)
        f_ms = sum(ft) / len(ft)
        row = dict(B=B, forks_ms=f_ms, forks_ms_min=min(ft), forks_ms_max=max(ft), forks_tok_s=B / (f_ms * 1e-3),
                   forks_gb=fb / 1e9, forks_tbps=fb / (f_ms * 1e-3) / 1e12,
                   forks_reserved_gb=(donor.memory_usage + forks.memory_usage) / 1e9)
        if cg:
            scale = LAYERS / layers
            c_ms = sum(ct) / len(ct) * scale
            cb = float((n_f[:layers] * (local + 1) * ROW_BYTES).sum() * B + B * stream_bytes * layers / LAYERS) * scale
            row.update(copies_layers=layers, copies_ms=c_ms, copies_tok_s=B / (c_ms * 1e-3), copies_gb=cb / 1e9,
                       copies_tbps=cb / (c_ms * 1e-3) / 1e12, copies_reserved_gb=B * per_copy / 1e9,
                       speedup=c_ms / f_ms)
        rows.append(row)
        c_txt = (f"copies {row['copies_ms']:.2f} ms{' (scaled from %d layers)' % layers if layers < LAYERS else ''}, "
                 f"{row['copies_gb']:.1f} GB, {row['copies_tbps']:.2f} TB/s, x{row['speedup']:.2f}") if cg else \
            "copies do not fit"
        print(f"B={B:3d}: forks {f_ms:.2f} ms (min {min(ft):.2f}, max {max(ft):.2f}), {row['forks_tok_s']:.0f} tok/s "
              f"per rank, {fb / 1e9:.2f} GB/step, {row['forks_tbps']:.2f} TB/s, reserved {row['forks_reserved_gb']:.1f}"
              f" GB | {c_txt}")
        del fg, cg, copies, forks
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    print("exchange (duo_seq_merge over NVLink): not measured (one GPU)")
    if args.json:
        print(json.dumps(dict(card=name, power_w=power, pattern=PATTERN, world=WORLD, ctx=CTX, rows=rows)))


if __name__ == "__main__":
    main()
