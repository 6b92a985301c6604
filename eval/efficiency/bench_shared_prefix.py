"""Several continuations of one long prompt, decoded together: rows that share the prompt's retrieval KV
(DuoRaggedKVCache.share_prefix, one duo_decode_ragged_shared cascade per layer) against rows that each hold a copy.

Workload: the attention of the Llama-3-8B-Instruct-Gradient-1048k architecture (32 layers, 32 q / 8 kv heads, bf16),
its DuoAttention pattern at sparsity 0.5 (128 retrieval kv heads in all), sink 64 / recent 256.  One step is the 32
layers' attention launches for a batch of one-token chunks, captured once in a CUDA graph and replayed; the weights
and GEMMs of the model are not part of it, so the step times are attention-only.  The caches are filled with seeded
random K/V: decode time does not depend on the values.

  shared : one 524288-token prompt; row 0 holds it, rows 1..B-1 fork it (share_prefix), and every row then holds 4096
           tokens of its own.  B in {1, 2, 4, 8, 16, 17, 32}.  At group 4 one 64-row block of the prefix kernel holds
           16 rows: B = 17 and 32 take two blocks, each of which streams the prefix again.
  compare: a 65536-token prompt at B = 8, shared against 8 rows that each prefilled a copy, alternated in this process.

--kv int4 runs the same on DuoRaggedINT4KVCache (136 B per retrieval head and key instead of 512 B): the default prompt
is then 1048576 tokens (18.3 GB of retrieval KV at this pattern, which B copies would multiply), and the bytes per step
count 136 B per (head, key).  The INT4 prefix launch is the 64-row INT4 kernel, the suffix launch the pooled ragged
keys-as-M decode kernel.

Per configuration: graph-replayed step time (min-max over --repeats), aggregate tokens/s (B / step), the retrieval
bytes the cascade must read per step (the prefix once per 64-row block, every row's own keys, the streaming heads'
sink + ring slots), and that over the step time (attention bandwidth: the step is attention only).  The card's name
and power limit are printed with the numbers.

  python eval/efficiency/bench_shared_prefix.py [--kv {bf16,int4}] [--steps 20] [--warmup 3] [--repeats 3]
      [--batches 1,2,4,8,16,17,32] [--prompt N] [--compare-prompt N]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the flagship benchmark's head pattern)
from duo_attention_b200 import _C  # noqa: E402
from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache, DuoRaggedKVCache  # noqa: E402

HQ, HKV, D, LAYERS, SINK, RECENT = 32, 8, 128, 32, 64, 256
OWN = 4096
ROW_BYTES = {"bf16": 2 * D * 2, "int4": 2 * (D // 2 + 4)}  # K + V of one token of one head (INT4: codes + fp16 scale, zero)
CACHE = {"bf16": DuoRaggedKVCache, "int4": DuoRaggedINT4KVCache}


def gpu_info():
    import subprocess

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def step_bytes(n_full, n_stream, prompt, B, shared, kv="bf16"):
    """Retrieval + streaming K/V bytes one step reads.  Shared (B > 1): the prefix once per 64-row block of the group
    (4 rows per member at group 4), then every row's own keys; otherwise every row's whole context."""
    ctx = prompt + OWN
    if shared and B > 1:
        P = prompt // 128 * 128
        retr = (-(-B * (HQ // HKV) // 64) * P + B * (ctx - P)) * sum(n_full)
    else:
        retr = B * ctx * sum(n_full)
    return (retr + sum(n_stream) * B * (SINK + RECENT + 1)) * ROW_BYTES[kv]


def build(mask, prompt, B, shared, dev, kv="bf16"):
    nf = [int((r > 0.5).sum()) for r in mask]
    if shared:
        caps = [prompt + OWN + 64] + [OWN + 64 + 128] * (B - 1)
    else:
        caps = [prompt + OWN + 64] * B
    c = CACHE[kv].from_geometry(LAYERS, HQ, HKV, D, nf, B, caps, SINK, RECENT, torch.bfloat16, dev)
    g = torch.Generator(device=dev).manual_seed(7)
    for t in c.tensors:
        for k, v in t.items():
            if not v.numel():
                continue
            if v.dtype == torch.uint8:  # INT4 codes
                v.random_(0, 256, generator=g)
            elif k.endswith("_scale"):  # INT4 scale / zero: K / V of unit size
                v.uniform_(0.0, 0.2, generator=g)
            elif k.endswith("_zero"):
                v.uniform_(-1.5, 0.0, generator=g)
            else:
                v.normal_(generator=g)
    lens = [prompt] + ([0] * (B - 1) if shared else [prompt] * (B - 1))
    for r, L in zip(c.rows, lens):
        for l in range(LAYERS):
            r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l] = L, L, max(SINK, L - RECENT)
    if shared:
        for b in range(1, B):
            c.share_prefix(0, b, OWN + 64 + 128)
    for r in c.rows:  # every row then holds OWN tokens of its own (random K/V already in place)
        for l in range(LAYERS):
            L = r.kv_seq_len_list[l] + OWN
            r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l] = L, L, max(SINK, L - RECENT)
    c.sync_device_state()
    return c


def capture(c, B, dev):
    width = (HQ + 2 * HKV) * D
    qkv = (torch.randn(B, 1, width, device=dev) * 0.5).to(torch.bfloat16)
    out = torch.empty(B, 1, HQ, D, dtype=torch.bfloat16, device=dev)
    snap = c.snapshot_state()
    c.graph_attached = True  # the occupancy stays in row_state: no host-to-device copy inside the capture
    c.graph_shared = c.sharing

    def step():
        for l in range(LAYERS):
            c.attend(l, qkv, None, None, _C.ROPE_NONE, out)

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            c.restore_state(snap)
            step()
        c.restore_state(snap)
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    c.restore_state(snap)  # every replay appends at the same rows: the lengths stay put
    return g


def time_graph(g, steps, warmup):
    for _ in range(warmup):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1,2,4,8,16,17,32")
    ap.add_argument("--kv", choices=("bf16", "int4"), default="bf16")
    ap.add_argument("--prompt", type=int, default=None, help="default 524288 (bf16), 1048576 (int4)")
    ap.add_argument("--compare-prompt", type=int, default=65536)
    args = ap.parse_args()
    kv = args.kv
    prompt = args.prompt or (1048576 if kv == "int4" else 524288)
    if not torch.cuda.is_available():
        raise SystemExit("bench_shared_prefix.py measures on a GPU: no CUDA device found")
    dev = torch.device("cuda:0")
    mask, _ = bench.head_pattern()
    nf = [int((r > 0.5).sum()) for r in mask]
    ns = [HKV - n for n in nf]
    name, power = gpu_info()
    print(f"# {name}, power limit {power} W; {kv} KV, attention-only steps of {LAYERS} layers, sum n_full = {sum(nf)}")
    rows = []

    def record(kind, prompt, B, shared, ms):
        by = step_bytes(nf, ns, prompt, B, shared, kv)
        r = {"kind": kind, "kv": kv, "prompt": prompt, "B": B, "shared": shared, "ms_min": min(ms), "ms_max": max(ms),
             "tok_s": B / (min(ms) / 1e3), "bytes_GB": by / 1e9, "TB_s": by / (min(ms) / 1e3) / 1e12}
        rows.append(r)
        print(json.dumps(r), flush=True)

    # shared against unshared copies, alternated
    caches = {s: build(mask, args.compare_prompt, 8, s, dev, kv) for s in (True, False)}
    graphs = {s: capture(caches[s], 8, dev) for s in (True, False)}
    ms = {True: [], False: []}
    for _ in range(args.repeats):
        for s in (True, False):
            ms[s].append(time_graph(graphs[s], args.steps, args.warmup))
    for s in (True, False):
        record("compare", args.compare_prompt, 8, s, ms[s])
    del caches, graphs
    gc.collect()
    torch.cuda.empty_cache()

    for B in [int(x) for x in args.batches.split(",")]:
        c = build(mask, prompt, B, True, dev, kv)
        g = capture(c, B, dev)
        record("shared", prompt, B, True, [time_graph(g, args.steps, args.warmup) for _ in range(args.repeats)])
        del c, g
        gc.collect()
        torch.cuda.empty_cache()
    out = os.environ.get("BENCH_OUT")  # optional JSON copy of the rows
    if out:
        with open(out, "w") as fh:
            json.dump({"gpu": name, "power_limit_W": power, "kv": kv, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
