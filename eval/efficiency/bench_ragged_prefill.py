"""Many rows' chunks in one batched ragged prefill (DuoRaggedKVCache.attend_rows, duo_prefill_ragged) against the same
chunks one row at a time (row(b).attend).

Workload: the Llama-3-8B-Instruct-Gradient-1048k architecture (32 layers, 32 q / 8 kv heads, bf16), its DuoAttention
pattern at sparsity 0.5 (128 retrieval kv heads in all), sink 64 / recent 256, random weights and seeded random K/V
(attention time does not depend on the values).

* forks: row 0 holds a prompt of --prompt tokens (131072), rows 1..B share it (share_prefix) and each takes a question
  of S tokens, B in {2, 4, 8, 16} and S in {128, 512, 2048}.  Attention pass: the 32 layers' append + attention + commit
  of all B questions, batched (3 launches per layer) or row by row (3 launches per row and layer); FLOP = 4 * 128 per
  visible (query, key) pair per q-head, as in bench_shared_prefill.py.  Model: one whole forward of the B questions
  (model(..., chunk_lengths=)) against B per-row forwards (--no-model skips it).
* admission: 8 new prompts of 512 tokens on empty rows, batched against one at a time (attention pass and model).

Both arms of a configuration run in one process, alternated, timed with CUDA events; every call is undone (the rows'
occupancy is put back) so each repeat sees the same state.  Reported: ms per pass (min-max over --repeats), TFLOP/s of
the attention pass, and the row-by-row / batched time ratio.  The card's name and power limit are printed with them.

  python eval/efficiency/bench_ragged_prefill.py [--repeats 3] [--warmup 1] [--no-model] [--json]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the flagship benchmark's head pattern and model)
from duo_attention_b200 import _C  # noqa: E402
from duo_attention_b200.kv_cache import DuoRaggedKVCache  # noqa: E402

HQ, HKV, D, LAYERS, SINK, RECENT = 32, 8, 128, 32, 64, 256
G = HQ // HKV
WIDTH = (HQ + 2 * HKV) * D


def gpu_info():
    import subprocess

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def chunk_flop(nf, ctx, S):
    """4 * 128 FLOP per visible (query, key) pair per q-head for one chunk of S tokens after ctx tokens."""
    causal = S * (S + 1) // 2
    retr = G * sum(nf) * (S * ctx + causal)
    strm = G * sum(HKV - n for n in nf) * (S * min(ctx, SINK + RECENT) + causal)
    return 4 * D * (retr + strm)


def build_cache(nf, prompt, B, S, dev, model=None):
    """Row 0 holds `prompt` random tokens (0: no donor, every row empty); rows 1..B fork it and have room for S more."""
    caps = [max(prompt, 1) + 128] + [S + 128] * B
    if model is not None:
        c = DuoRaggedKVCache(model, model._bench_mask, B + 1, caps, SINK, RECENT, prefilling_chunk_size=S)
    else:
        c = DuoRaggedKVCache.from_geometry(LAYERS, HQ, HKV, D, nf, B + 1, caps, SINK, RECENT, torch.bfloat16, dev,
                                           stage_cap=S)
    g = torch.Generator(device=dev).manual_seed(7)
    for t in c.tensors:
        for v in t.values():
            if v.numel():
                v.normal_(generator=g)
    if prompt:
        r = c.row(0)
        for l in range(LAYERS):
            r.kv_seq_len_list[l], r.total_list[l], r.lo_list[l] = prompt, prompt, max(SINK, prompt - RECENT)
        c.sync_device_state()
        for b in range(1, B + 1):
            c.share_prefix(0, b, S + 128)
    return c


def timed(c, fn, warmup):
    """fn() once per warm-up and once timed, the rows' occupancy put back after each; returns ms."""
    snap = c.snapshot_state()
    for _ in range(warmup):
        fn()
        c.restore_state(snap)
        c.sync_device_state()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    c.restore_state(snap)
    c.sync_device_state()
    return e0.elapsed_time(e1)


def attention_arms(c, B, S, dev):
    qkv = (torch.randn(1, B * S, WIDTH, device=dev) * 0.5).to(torch.bfloat16)
    out = torch.empty(1, B * S, HQ, D, dtype=torch.bfloat16, device=dev)
    lens = [0] + [S] * B

    def batched():
        for l in range(LAYERS):
            c.attend_rows(l, qkv, None, None, _C.ROPE_NONE, out, lens)

    def row_by_row():
        for l in range(LAYERS):
            for b in range(1, B + 1):
                c.row(b).attend(l, qkv[:, (b - 1) * S : b * S], None, None, _C.ROPE_NONE, out[:, (b - 1) * S : b * S])

    return {"batched": batched, "row_by_row": row_by_row}


def model_arms(model, c, B, S, dev):
    ids = torch.randint(0, model.config.vocab_size, (1, B * S), device=dev)
    lens = [0] + [S] * B

    def batched():
        model(input_ids=ids, past_key_values=c, use_cache=True, chunk_lengths=lens)

    def row_by_row():
        for b in range(1, B + 1):
            model(input_ids=ids[:, (b - 1) * S : b * S], past_key_values=c.row(b), use_cache=True)

    return {"batched": batched, "row_by_row": row_by_row}


def run(c, arms, repeats, warmup):
    ms = {a: [] for a in arms}
    for fn in arms.values():
        timed(c, fn, warmup)
    for _ in range(repeats):
        for a, fn in arms.items():
            ms[a].append(timed(c, fn, 0))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--prompt", type=int, default=131072)
    ap.add_argument("--forks", default="2,4,8,16")
    ap.add_argument("--chunks", default="128,512,2048")
    ap.add_argument("--no-model", action="store_true", help="attention passes only")
    ap.add_argument("--json", action="store_true", help="print one JSON document with every row at the end")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_prefill.py measures on a GPU: no CUDA device found")
    dev = torch.device("cuda:0")
    mask, _ = bench.head_pattern()
    nf = [int((r > 0.5).sum()) for r in mask]
    model = None
    if not args.no_model:
        margs = types.SimpleNamespace(arch="llama3-8b-1048k", layers=LAYERS, kv_format="bf16")
        model, _, _ = bench.build_model(margs, mask, 0, 1, dev)
        model._bench_mask = mask
    name, power = gpu_info()
    print(f"# {name}, power limit {power} W; {LAYERS} layers, sum n_full = {sum(nf)}, prompt {args.prompt}")
    print("# case       B  chunk  what   arm         ms(min-max)          TFLOP/s  row_by_row/batched")
    rows = []
    cases = [("forks", args.prompt, int(B), int(S)) for B in args.forks.split(",") for S in args.chunks.split(",")]
    cases.append(("admission", 0, 8, 512))
    with torch.no_grad():
        for case, prompt, B, S in cases:
            c = build_cache(nf, prompt, B, S, dev, model)
            results = {"attention": run(c, attention_arms(c, B, S, dev), args.repeats, args.warmup)}
            if model is not None:
                results["model"] = run(c, model_arms(model, c, B, S, dev), args.repeats, args.warmup)
            flop = B * chunk_flop(nf, prompt, S)
            for what, ms in results.items():
                for a in ms:
                    rec = {"case": case, "B": B, "chunk": S, "prompt": prompt, "what": what, "arm": a,
                           "ms_min": min(ms[a]), "ms_max": max(ms[a]),
                           "ratio": min(ms["row_by_row"]) / min(ms["batched"])}
                    if what == "attention":
                        rec["TFLOP_s"] = flop / (min(ms[a]) / 1e3) / 1e12
                    rows.append(rec)
                    tf = f"{rec['TFLOP_s']:7.1f}" if "TFLOP_s" in rec else "      -"
                    print(f"  {case:9s} {B:3d} {S:6d}  {what:6s} {a:10s} {rec['ms_min']:9.2f}-{rec['ms_max']:9.2f}  "
                          f"{tf}  {rec['ratio']:6.2f}", flush=True)
            del c
            gc.collect()
            torch.cuda.empty_cache()
    if args.json:
        print(json.dumps({"gpu": name, "power_limit_W": power, "rows": rows}))


if __name__ == "__main__":
    main()
