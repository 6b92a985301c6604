"""Admitting a long prompt into a ragged batch that keeps decoding (DuoRaggedKVCache.set_active), on one GPU.

Workload: the Llama-3-8B-Instruct-Gradient-1048k architecture (random init, bf16), its DuoAttention pattern at sparsity
0.5, sink 64 / recent 256, a pooled cache (per-row capacities), graph-replayed decode steps.

1. Admission (``--part admission``, 16-bit cache): eight rows decode at 32,768 tokens each while a ninth row admits a
   131,072-token prompt through ``row(8)`` in 8,192-token chunks, the ninth row idle meanwhile.  Two schedules:
     sequential : every chunk, then decoding resumes (what a batch that must step every row has to do);
     interleaved: a chunk, then k decode steps of the eight rows, repeated (k from --k).
   Reported per schedule: the admission wall time (first chunk to last chunk done), the longest gap between two
   tokens of a decoding row (CUDA events after every step and chunk), and the decoding rows' tokens/s during the
   admission.  The schedules alternate --runs times.
2. Idle cost (``--part idle``, bf16 and INT4): the graph-replayed step of B rows with k of them idle against a compact
   cache of the B - k active rows at the same lengths, the two arms alternated --runs times in this process.
The card's name and power limit are part of the output.  The caches are filled with seeded random K/V.

  python eval/efficiency/bench_admission.py [--part {admission,idle,all}] [--k 1,4] [--runs 2] [--steps 20]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
from bench_ragged import fill, gpu_info  # noqa: E402
from duo_attention_b200.graph import DuoDecodeGraph  # noqa: E402
from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache, DuoRaggedKVCache  # noqa: E402

DECODE_LEN, N_DECODE, PROMPT, CHUNK = 32768, 8, 131072, 8192


def _spread(v):
    return {"runs": [round(x, 3) for x in v], "mean": round(sum(v) / len(v), 3), "spread": round(max(v) - min(v), 3)}


def admission(model, mask, ks, runs, dev):
    sink, recent = bench.SINK, bench.RECENT
    pad = 16 * max(ks) * runs + 256
    caps = [DECODE_LEN + pad] * N_DECODE + [PROMPT + 64]
    cache = DuoRaggedKVCache(model, mask, N_DECODE + 1, caps, sink, recent, prefilling_chunk_size=CHUNK)
    fill(cache.rows[:N_DECODE], cache.tensors, [DECODE_LEN] * N_DECODE, sink, recent)
    cache.set_active(N_DECODE, False)
    cache.sync_device_state()
    snap = cache.snapshot_state()
    tok = torch.zeros(N_DECODE + 1, 1, dtype=torch.long, device=dev)
    prompt = torch.randint(0, 32000, (1, PROMPT), generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        graph = DuoDecodeGraph(model, cache)
        for _ in range(3):
            graph.step(tok)
        # warm the chunk path at the chunk size (kernels, cuBLAS algorithms), then empty the row again
        model(input_ids=prompt[:, :CHUNK], past_key_values=cache.row(N_DECODE), use_cache=True)
        torch.cuda.synchronize()

        def reset():
            cache.row(N_DECODE).clear()
            cache.restore_state(snap)
            cache.set_active(N_DECODE, False)  # also re-syncs row_state and reloads the graph's positions
            torch.cuda.synchronize()

        def ev():
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            return e

        def schedule(k):
            """k = 0: sequential.  Returns (admission ms, longest token gap ms, decoding rows' tok/s during it)."""
            reset()
            graph.step(tok)  # the token before the admission starts
            marks, steps = [ev()], 0
            for c0 in range(0, PROMPT, CHUNK):
                model(input_ids=prompt[:, c0 : c0 + CHUNK], past_key_values=cache.row(N_DECODE), use_cache=True)
                chunk_done = ev()
                for _ in range(k):
                    graph.step(tok)
                    marks.append(ev())
                    steps += 1
            end = chunk_done if k == 0 else marks[-1]
            graph.step(tok)  # decoding resumes
            marks.append(ev())
            torch.cuda.synchronize()
            assert cache.row_lengths[N_DECODE] == PROMPT
            adm = marks[0].elapsed_time(end)
            gap = max(a.elapsed_time(b) for a, b in zip(marks, marks[1:]))
            return adm, gap, N_DECODE * steps / (adm / 1e3)

        res = {}
        names = ["sequential"] + [f"interleaved_k{k}" for k in ks]
        for _ in range(runs):
            for name, k in zip(names, [0] + list(ks)):
                adm, gap, tps = schedule(k)
                r = res.setdefault(name, {"admission_ms": [], "longest_gap_ms": [], "decode_tok_s": []})
                r["admission_ms"].append(adm)
                r["longest_gap_ms"].append(gap)
                r["decode_tok_s"].append(tps)
                print(f"[admission {name}] {adm:.1f} ms, gap {gap:.1f} ms, {tps:.1f} tok/s", file=sys.stderr)
        # the steady step of the eight rows with the admitted row idle, for reference
        reset()
        e0 = ev()
        for _ in range(20):
            graph.step(tok)
        e1 = ev()
        torch.cuda.synchronize()
        out = {n: {m: _spread(v) for m, v in r.items()} for n, r in res.items()}
        out["step_ms_8_rows"] = round(e0.elapsed_time(e1) / 20, 3)
    del graph, cache
    gc.collect()
    torch.cuda.empty_cache()
    return out


def graph_ms(model, cache, B, steps, warmup):
    tok = torch.zeros(B, 1, dtype=torch.long, device=cache.device)
    snap = cache.snapshot_state()
    with torch.no_grad():
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
    cache.restore_state(snap)
    cache.sync_device_state()
    return e0.elapsed_time(e1) / steps


def idle_cost(model, mask, kv, B, n_idle, runs, steps, warmup):
    sink, recent = bench.SINK, bench.RECENT
    cls = DuoRaggedINT4KVCache if kv == "int4" else DuoRaggedKVCache
    lengths = [DECODE_LEN] * B
    cap = DECODE_LEN + steps + warmup + 64
    ms = {"idle": [], "compact": []}
    for i in range(2 * runs):  # alternate the arms
        arm = "idle" if i % 2 == 0 else "compact"
        n = B if arm == "idle" else B - n_idle
        c = cls(model, mask, n, [cap] * n, sink, recent)
        fill(c.rows, c.tensors, lengths[:n], sink, recent)
        if arm == "idle":
            for b in range(B - n_idle, B):
                c.set_active(b, False)
        c.sync_device_state()
        ms[arm].append(graph_ms(model, c, n, steps, warmup))
        del c
        gc.collect()
        torch.cuda.empty_cache()
        print(f"[idle {kv} {arm}] {ms[arm][-1]:.3f} ms", file=sys.stderr)
    out = {arm: _spread(v) for arm, v in ms.items()}
    out["idle_over_compact"] = round(out["idle"]["mean"] / out["compact"]["mean"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=["admission", "idle", "all"], default="all")
    ap.add_argument("--k", default="1,4", help="decode steps between two chunks in the interleaved schedules")
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32, help="debug only: a run with fewer layers is not a valid number")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    name, power = gpu_info(dev)
    mask, sparsity = bench.head_pattern()
    mask = mask[: args.layers]
    margs = types.SimpleNamespace(arch="llama3-8b-1048k", layers=args.layers, kv_format="bf16")
    model, mask, _ = bench.build_model(margs, mask, 0, 1, dev)
    res = {"gpu": name, "power_limit_w": power, "layers": args.layers, "sparsity": sparsity, "sink": bench.SINK,
           "recent": bench.RECENT}
    t0 = time.time()
    if args.part in ("admission", "all"):
        res["admission"] = admission(model, mask, [int(k) for k in args.k.split(",")], args.runs, dev)
        res["admission"]["setup"] = (f"{N_DECODE} rows decoding at {DECODE_LEN} tokens, a {PROMPT}-token prompt "
                                     f"admitted in {CHUNK}-token chunks, bf16 pooled cache")
    if args.part in ("idle", "all"):
        res["idle_cost"] = {}
        for kv in ("bf16", "int4"):
            for B, k in ((8, 2), (8, 6)):
                res["idle_cost"][f"{kv}_B{B}_idle{k}"] = idle_cost(model, mask, kv, B, k, args.runs, args.steps,
                                                                   args.warmup)
    res["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
