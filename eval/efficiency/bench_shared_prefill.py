"""A question on a fork of one long prompt: the chunk on a row that shares the prompt's retrieval KV
(DuoRaggedKVCache.share_prefix, then row(b).attend -> duo_attention_shared) against the same chunk on a row that holds a
copy of the prompt (duo_attention).

Workload: the attention of the Llama-3-8B-Instruct-Gradient-1048k architecture (32 layers, 32 q / 8 kv heads, bf16),
its DuoAttention pattern at sparsity 0.5 (128 retrieval kv heads in all), sink 64 / recent 256.  One pass is the 32
layers' duo_rope_append + duo_attention[_shared] + duo_stream_commit for one question chunk; the weights and GEMMs of
the model are not part of it.  The caches hold seeded random K/V (attention time does not depend on the values); the
copy row's retrieval region is a byte copy of the donor's.  Chunks of 512 and 4096 tokens over prompts of 131072 and
262144 tokens; both arms run at the same length and are alternated in one process, timed with CUDA events.

Per configuration: ms per pass (min-max over --repeats), FLOP = 4 * 128 per visible (query, key) pair per q-head
(both head classes) and TFLOP/s, the sharer / copy time ratio, and the retrieval KV that 8 forks of the prompt reserve
with and without sharing (each fork's own region holding the question).  The card's name and power limit are printed
with the numbers.

  python eval/efficiency/bench_shared_prefill.py [--repeats 3] [--warmup 1] [--json]
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
from duo_attention_b200.kv_cache import DuoRaggedKVCache  # noqa: E402

HQ, HKV, D, LAYERS, SINK, RECENT = 32, 8, 128, 32, 64, 256
G = HQ // HKV
ROW_BYTES = 2 * D * 2  # K + V of one token of one head, bf16
FORKS = 8


def gpu_info():
    import subprocess

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def pass_flop(nf, prompt, S):
    """4 * 128 FLOP per visible (query, key) pair per q-head: retrieval q-heads see the prompt and the chunk causally,
    streaming q-heads the sink + ring slots the prompt left plus the chunk causally."""
    causal = S * (S + 1) // 2
    retr = G * sum(nf) * (S * prompt + causal)
    strm = G * sum(HKV - n for n in nf) * (S * min(prompt, SINK + RECENT) + causal)
    return 4 * D * (retr + strm)


def reserved_gb(nf, prompt, S, shared):
    """Retrieval KV of FORKS forks of the prompt, each holding the question: the prompt once plus every fork's own
    region, or the prompt in every fork."""
    own = -(-S // 128) * 128
    tokens = prompt + FORKS * own if shared else FORKS * (prompt + own)
    return tokens * sum(nf) * ROW_BYTES / 1e9


def build(nf, prompt, S, dev):
    """Row 0 holds the prompt, row 1 forks it (share_prefix), row 2 holds a byte copy of it."""
    caps = [prompt + 128, S + 128, prompt + S + 128]
    c = DuoRaggedKVCache.from_geometry(LAYERS, HQ, HKV, D, nf, 3, caps, SINK, RECENT, torch.bfloat16, dev,
                                       stage_cap=S)
    g = torch.Generator(device=dev).manual_seed(7)
    for t in c.tensors:
        for v in t.values():
            if v.numel():
                v.normal_(generator=g)
    for b in (0, 2):
        r = c.row(b)
        for l in range(LAYERS):
            r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l] = prompt, prompt, max(SINK, prompt - RECENT)
    for l in range(LAYERS):
        for key in c.row(0).tensors[l]:
            c.row(2).tensors[l][key][0, :, : prompt if key.startswith("full") else SINK + RECENT].copy_(
                c.row(0).tensors[l][key][0, :, : prompt if key.startswith("full") else SINK + RECENT])
    c.sync_device_state()
    c.share_prefix(0, 1, S + 128)
    return c


def time_pass(row, qkv, out, warmup):
    """One 32-layer pass of the chunk on `row`, timed with CUDA events; the row's occupancy is put back after it."""
    snap = row.snapshot_state()
    for _ in range(warmup):
        for l in range(LAYERS):
            row.attend(l, qkv, None, None, _C.ROPE_NONE, out)
        row.restore_state(snap)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for l in range(LAYERS):
        row.attend(l, qkv, None, None, _C.ROPE_NONE, out)
    e1.record()
    torch.cuda.synchronize()
    row.restore_state(snap)
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--prompts", default="131072,262144")
    ap.add_argument("--chunks", default="512,4096")
    ap.add_argument("--json", action="store_true", help="print one JSON document with every row at the end")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shared_prefill.py measures on a GPU: no CUDA device found")
    dev = torch.device("cuda:0")
    mask, _ = bench.head_pattern()
    nf = [int((r > 0.5).sum()) for r in mask]
    name, power = gpu_info()
    print(f"# {name}, power limit {power} W; attention-only passes of {LAYERS} layers, sum n_full = {sum(nf)}")
    print("# prompt  chunk  arm     ms(min-max)        TFLOP  TFLOP/s  sharer/copy  reserved GB for 8 forks")
    rows = []
    for prompt in [int(x) for x in args.prompts.split(",")]:
        for S in [int(x) for x in args.chunks.split(",")]:
            c = build(nf, prompt, S, dev)
            qkv = (torch.randn(1, S, (HQ + 2 * HKV) * D, device=dev) * 0.5).to(torch.bfloat16)
            out = torch.empty(1, S, HQ, D, dtype=torch.bfloat16, device=dev)
            arms = {"sharer": c.row(1), "copy": c.row(2)}
            assert c.row_prefix[1] == (0, prompt) and c.row_lengths[1] == c.row_lengths[2] == prompt
            ms = {a: [] for a in arms}
            for a, r in arms.items():  # warm-up
                time_pass(r, qkv, out, args.warmup)
            for _ in range(args.repeats):
                for a, r in arms.items():
                    ms[a].append(time_pass(r, qkv, out, 0))
            flop = pass_flop(nf, prompt, S)
            for a in arms:
                rec = {"prompt": prompt, "chunk": S, "arm": a, "ms_min": min(ms[a]), "ms_max": max(ms[a]),
                       "TFLOP": flop / 1e12, "TFLOP_s": flop / (min(ms[a]) / 1e3) / 1e12,
                       "ratio_sharer_copy": min(ms["sharer"]) / min(ms["copy"]),
                       "reserved_GB_8_forks": reserved_gb(nf, prompt, S, a == "sharer")}
                rows.append(rec)
                print(f"  {prompt:7d} {S:6d}  {a:6s}  {rec['ms_min']:8.2f}-{rec['ms_max']:8.2f}  {rec['TFLOP']:7.2f}  "
                      f"{rec['TFLOP_s']:7.1f}  {rec['ratio_sharer_copy']:11.3f}  {rec['reserved_GB_8_forks']:8.1f}",
                      flush=True)
            del c, arms, qkv, out
            gc.collect()
            torch.cuda.empty_cache()
    if args.json:
        print(json.dumps({"gpu": name, "power_limit_W": power, "rows": rows}))


if __name__ == "__main__":
    main()
