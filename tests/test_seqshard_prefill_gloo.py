"""World-size-2 and -4 gloo (CPU) tests of the row-scattered cross-rank merge of a prefill-sized chunk on the
sequence-sharded layout (tp.merge_scattered): every rank contributes its (O, log-sum-exp) partials of every
(token, retrieval head) row; all_to_all_single hands each rank a share of the rows, the rank merges its share, and
all_gather_into_tensor collects the merged rows.  With a CPU restatement of duo_merge_partials as the merge function,
every rank's output must equal stacking all ranks' partials and merging them in rank order, bit for bit, and the
streaming-head rows of `out` must stay untouched.  Covered: shares of unequal size (tokens x heads not divisible by
the world), fewer rows than ranks, and rows that see no key on some ranks (lse = -inf)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from duo_attention_b200 import tp

D = 128
# (batch, tokens, heads_total, heads_used): rows = batch * tokens * heads_used
SHAPES = [(2, 17, 8, 3), (1, 5, 4, 4), (1, 1, 4, 1), (3, 129, 12, 5), (2, 100, 32, 16)]


def merge_cpu(o_parts, lse_parts, out):
    """duo_merge_partials restated: out = sum_p 2^(lse_p - max) o_p / sum_p 2^(lse_p - max), parts in order, fp32."""
    mx = lse_parts.max(0).values
    acc = torch.zeros(o_parts.shape[1:], dtype=torch.float32)
    wsum = torch.zeros(lse_parts.shape[1:], dtype=torch.float32)
    for q in range(o_parts.shape[0]):
        seen = lse_parts[q] != float("-inf")
        w = torch.where(seen, torch.exp2(lse_parts[q] - mx), torch.zeros_like(mx))
        acc = acc + w[:, None] * o_parts[q]
        wsum = wsum + w
    out.copy_(torch.where(wsum[:, None] > 0, acc / wsum[:, None], torch.zeros_like(acc)).to(out.dtype))


def _partials(rank, shape, g_seed):
    """Rank `rank`'s partials of one chunk: fp32 O, log2-domain lse with some rows -inf (no key on this rank)."""
    B, S, H, _ = shape
    g = torch.Generator().manual_seed(g_seed * 101 + rank)
    po = torch.randn(B, S, H, D, generator=g)
    pl = torch.randn(B, S, H, generator=g) * 8
    empty = torch.rand(B, S, H, generator=g) < 0.2
    pl[empty] = float("-inf")
    po[empty] = 0.0
    return po, pl


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ok = True
        for i, shape in enumerate(SHAPES):
            B, S, H, used = shape
            for dtype in (torch.bfloat16, torch.float16):
                po, pl = _partials(rank, shape, i)
                out = torch.full((B, S, H, D), 7.0, dtype=dtype)  # streaming-head rows must keep this
                tp.merge_scattered(po, pl, out, B * S, H, used, merge_fn=merge_cpu)
                parts = [_partials(r, shape, i) for r in range(world)]
                o_all = torch.stack([p[0].reshape(B * S, H, D)[:, :used].reshape(-1, D) for p in parts])
                l_all = torch.stack([p[1].reshape(B * S, H)[:, :used].reshape(-1) for p in parts])
                want = torch.empty(B * S * used, D, dtype=dtype)
                merge_cpu(o_all, l_all, want)
                ok = ok and torch.equal(out[:, :, :used].reshape(-1, D), want)
                ok = ok and bool((out[:, :, used:] == 7.0).all())
        counts = tp.scatter_counts(7, world)
        ok = ok and sum(counts) == 7 and max(counts) - min(counts) <= 1 and counts == sorted(counts, reverse=True)
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_scattered_merge_equals_the_stacked_merge(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 35500 + (os.getpid() % 2000) + world
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {r: True for r in range(world)}
