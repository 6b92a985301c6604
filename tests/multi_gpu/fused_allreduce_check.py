"""Multi-GPU check of the EXPERIMENTAL fused all-reduce + residual add + RMSNorm kernel (csrc/comm.cu), run under
torchrun on a multi-GPU node with a hard timeout, e.g.

   timeout 120 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 \
       --master-addr 127.0.0.1 --master-port 29517 tests/multi_gpu/fused_allreduce_check.py

Kernel level: FusedAllReduce.add_rmsnorm == NCCL all-reduce followed by duo_add_rmsnorm, for 1..16 rows, many
back-to-back calls (epoch / double-buffer protocol), eagerly and replayed from a CUDA graph; bit-identical results on
every rank.  Prints FUSED_AR_OK and per-call latencies (CUDA events) of both variants.
Model level: run tests/multi_gpu/tp_check.py with DUO_FUSED_ALLREDUCE=1 in the environment (install_allreduce then
routes the small exchanges through the fused kernel) — it must still reproduce the single-GPU logits."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from duo_attention_b200 import ops, tp  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    hidden, eps = 4096, 1e-5
    comm = tp.FusedAllReduce(None, hidden, torch.bfloat16, dev, max_rows=16)
    g = torch.Generator(device="cpu").manual_seed(100 + rank)
    w = (torch.rand(hidden, generator=g) + 0.5).to(torch.bfloat16).to(dev)
    dist.broadcast(w, 0)
    worst = 0.0
    for it, rows in enumerate([1, 1, 1, 2, 16, 1, 5, 1, 1, 16, 16, 1] * 4):
        part = torch.randn(rows, hidden, generator=g).to(torch.bfloat16).to(dev)
        res = torch.randn(rows, hidden, generator=torch.Generator().manual_seed(it)).to(torch.bfloat16).to(dev)
        ref_sum = part.clone()
        dist.all_reduce(ref_sum)
        ref_out, ref_h = ops.add_rmsnorm(ref_sum, res.clone(), w, eps)
        out, h = comm.add_rmsnorm(part, res.clone(), w, eps)
        # NCCL may round partial sums differently (bf16 ring): compare with a tolerance, and ranks with each other exactly
        torch.testing.assert_close(h.float(), ref_h.float(), rtol=2e-2, atol=2e-2)
        torch.testing.assert_close(out.float(), ref_out.float(), rtol=3e-2, atol=3e-2)
        worst = max(worst, (h.float() - ref_h.float()).abs().max().item())
        gathered = [torch.empty_like(h) for _ in range(world)]
        dist.all_gather(gathered, h)
        assert all(torch.equal(gathered[0], t) for t in gathered), "ranks disagree on the reduced residual stream"
    assert not comm.error(), "a peer timed out"

    # graph replay: 8 back-to-back calls per replay, replayed 20 times
    part = torch.randn(1, hidden, generator=g).to(torch.bfloat16).to(dev)
    res = torch.zeros(1, hidden, dtype=torch.bfloat16, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for _ in range(8):
                comm.add_rmsnorm(part, res, w, eps)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    dist.barrier()
    graph = torch.cuda.CUDAGraph()
    res.zero_()
    with torch.cuda.graph(graph):
        for _ in range(8):
            out_g, _ = comm.add_rmsnorm(part, res, w, eps)
    res.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    dist.barrier()
    e0.record()
    for _ in range(20):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    fused_us = e0.elapsed_time(e1) * 1e3 / 160
    tot = part.clone()
    dist.all_reduce(tot)
    # after 160 accumulations the residual holds 160 * sum(part) up to bf16 rounding of the running sum: check it moved
    assert torch.isfinite(res.float()).all() and res.float().abs().sum() > 0
    assert not comm.error(), "a peer timed out during graph replay"

    # NCCL + add_rmsnorm latency for comparison (eager launches)
    x = part.clone()
    torch.cuda.synchronize()
    dist.barrier()
    e0.record()
    for _ in range(160):
        dist.all_reduce(x)
        ops.add_rmsnorm(x, res, w, eps)
    e1.record()
    torch.cuda.synchronize()
    nccl_us = e0.elapsed_time(e1) * 1e3 / 160
    if rank == 0:
        print(f"FUSED_AR_OK world={world} max|dh|={worst:.4f} fused={fused_us:.1f}us/call (graph) "
              f"nccl+norm={nccl_us:.1f}us/call (eager)")
    dist.barrier()
    os._exit(0)


if __name__ == "__main__":
    main()
