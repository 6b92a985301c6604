"""Questions on forks of a 1M-token prompt on sequence-sharded caches: rank 0 of world 8, on one GPU.

B forks of one prompt (DuoSeqShardKVCache.fork) each take a question of S tokens over the donor's slice of the prompt
in place: one duo_prefill_seq_shared per layer.  The alternative is a batch-B DuoSeqShardKVCache holding B copies of
the prompt (duo_prefill_seq).  Both run the same tiles on the same slice, so the ratio of their times isolates the
cost of reading the prefix rows from the donor's tensors.  Both arms are measured as rank 0 of world 8 (131,072 local
prompt positions).  Only the attention launch is timed (the append and ring commit are the same in both arms); the
row-scattered exchange (merge_scattered) is not part of either arm and cannot be measured on one GPU: "not measured".

Workload: Llama-3-8B-Instruct-Gradient-1048k attention (32 layers, 32 q / 8 kv heads), its DuoAttention pattern at
sparsity 0.5, sink / recent of the flagship benchmark, bf16, seeded random K/V and q.  Timing: the 32 layers' launches
captured in a CUDA graph per arm; the arms are replayed alternately, --steps replays each per round over --rounds
rounds, CUDA events around every replay.  B copies of the prompt need B x 8.6 GB per rank; where that does not fit next
to the donor, the copies arm runs on fewer layers and its time is scaled to 32 (marked "scaled").  Attention FLOP/s
count 4 x 128 FLOPs per (q head, token, visible key) of rank 0, from the shapes.

  python eval/efficiency/bench_seqshard_fork_chunks.py [--steps 5] [--warmup 2] [--rounds 3] [--json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402  (head pattern, sink / recent of the flagship benchmark)
from bench_ragged import gpu_info  # noqa: E402
from bench_seqshard_forks import (BLOCK, CTX, D, HKV, HQ, LAYERS, PATTERN, ROW_BYTES, WORLD, _Geometry, _NoComm,  # noqa: E402
                                  capture, timed)
from duo_attention_b200 import _C, tp  # noqa: E402
from duo_attention_b200.kv_cache import DuoSeqShardKVCache  # noqa: E402
from duo_attention_b200.seqshard import SeqShardPlan  # noqa: E402

BATCHES = [2, 4, 8]
QUESTIONS = [128, 512, 2048]
COPY_BUDGET = 40e9  # bytes of prompt copies the copies arm may hold next to the donor


def filled(mask, batch, room, dev, g):
    """Rank 0's cache of the prompt (random K/V) with room for `room` more tokens and a staging area that takes them."""
    c = DuoSeqShardKVCache(_Geometry(dev, len(mask)), mask.tolist(), batch, CTX + room, bench.SINK, bench.RECENT,
                           seq=tp.SeqShardContext(0, WORLD, BLOCK, _NoComm()))
    for t in c.tensors:
        for v in t.values():
            v.normal_(generator=g)
    for l in range(c.num_layers):
        c.kv_seq_len_list[l], c.total_list[l], c.lo_list[l] = CTX, CTX, CTX - bench.RECENT
    return c


def attn_flops(n_f, n_s, plan, S):
    """FLOPs of rank 0's attention for one row's chunk of S tokens after CTX: retrieval q-heads see the local rows of
    the positions <= CTX + t, streaming q-heads the sink + ring slots and the chunk causally."""
    G = HQ // HKV
    keys_f = sum(plan.local_len(0, CTX + t + 1) for t in range(S))
    keys_s = sum(min(CTX, bench.SINK + bench.RECENT) + t + 1 for t in range(S))
    return 4 * D * G * (float(n_f.sum()) * keys_f + float(n_s.sum()) * keys_s)


def chunk_fn(cache, B, S, dev, g, donor=None):
    """The per-layer attention launches of one chunk of S tokens on every row, at the prompt's occupancy."""
    width = (HQ + 2 * HKV) * D
    qkv = (torch.randn(B, S, width, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    out = torch.empty(B, S, HQ, D, dtype=torch.bfloat16, device=dev)
    po, pl = cache.partials(S)
    lib, ws = cache.lib, cache.workspace
    states = []
    for l in range(cache.num_layers):
        cache._ensure_room(l, S)  # the staging area of a chunk of S tokens
        st = cache.state(l)
        s = _C.CacheState(st.full_len, st.total, st.lo, None)
        s.seq_rank, s.seq_world, s.seq_block = st.seq_rank, st.seq_world, st.seq_block
        states.append(s)
    keep = (qkv, out, po, pl, states)

    def fn():
        stream = torch.cuda.current_stream(dev).cuda_stream
        for l in range(cache.num_layers):
            a = (C.byref(states[l]), qkv.data_ptr(), qkv.stride(1), out.data_ptr(), po.data_ptr(), pl.data_ptr(), S,
                 D ** -0.5, ws.data_ptr(), ws.numel(), stream)
            if donor is None:
                _C.check(lib.duo_prefill_seq(cache.handles[l], *a))
            else:
                _C.check(lib.duo_prefill_seq_shared(cache.handles[l], donor.handles[l], cache.prefix_len, *a))
    fn.keep = keep
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=str, default=",".join(map(str, BATCHES)))
    ap.add_argument("--questions", type=str, default=",".join(map(str, QUESTIONS)))
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seqshard_fork_chunks measures on a CUDA device; none is visible")
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
    donor = filled(mask, 1, 0, dev, g)
    per_copy = float((n_f * (local + 1) * ROW_BYTES).sum())
    rows = []
    for B in [int(b) for b in args.batches.split(",")]:
        for S in [int(s) for s in args.questions.split(",")]:
            forks = donor.fork(B, S + 64)
            layers = min(LAYERS, int(COPY_BUDGET / (B * per_copy / LAYERS)))
            fg = capture(chunk_fn(forks, B, S, dev, g, donor))
            copies = filled(mask[:layers], B, S, dev, g) if layers > 0 else None
            cg = capture(chunk_fn(copies, B, S, dev, g)) if copies is not None else None
            timed(fg, args.warmup)
            if cg:
                timed(cg, args.warmup)
            ft, ct = [], []
            for _ in range(args.rounds):  # arms alternated
                ft += timed(fg, args.steps)
                if cg:
                    ct += timed(cg, args.steps)
            f_ms = sum(ft) / len(ft)
            flops = B * attn_flops(n_f, n_s, plan, S)
            row = dict(B=B, S=S, forks_ms=f_ms, forks_ms_min=min(ft), forks_ms_max=max(ft),
                       forks_tflops=flops / (f_ms * 1e-3) / 1e12,
                       forks_retrieval_kv_gb=(float((n_f * donor.full_cap_list[0]).sum()) +
                                              B * float((n_f * forks.full_cap_list[0]).sum())) * ROW_BYTES / 1e9)
            if cg:
                c_flops = B * attn_flops(n_f[:layers], n_s[:layers], plan, S)
                c_ms = sum(ct) / len(ct) * LAYERS / layers
                row.update(copies_layers=layers, copies_ms=c_ms, copies_tflops=c_flops / (sum(ct) / len(ct) * 1e-3) / 1e12,
                           copies_retrieval_kv_gb=B * per_copy / 1e9, ratio=f_ms / c_ms)
            rows.append(row)
            c_txt = (f"copies {row['copies_ms']:.2f} ms{' (scaled from %d layers)' % layers if layers < LAYERS else ''}"
                     f", {row['copies_tflops']:.0f} TFLOP/s, {row['copies_retrieval_kv_gb']:.1f} GB | forks / copies "
                     f"{row['ratio']:.3f}") if cg else "copies do not fit"
            print(f"B={B} S={S:5d}: forks {f_ms:.2f} ms (min {min(ft):.2f}, max {max(ft):.2f}), "
                  f"{row['forks_tflops']:.0f} TFLOP/s, retrieval KV {row['forks_retrieval_kv_gb']:.1f} GB | {c_txt}")
            del fg, cg, copies, forks
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    print("exchange (merge_scattered): not measured (one GPU)")
    if args.json:
        print(json.dumps(dict(card=name, power_w=power, pattern=PATTERN, world=WORLD, ctx=CTX, rows=rows)))


if __name__ == "__main__":
    main()
