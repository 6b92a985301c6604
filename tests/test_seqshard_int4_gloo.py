"""World-size-2 and -4 gloo (CPU) tests of moving an INT4 cache from the head-parallel prefill layout to the
sequence-sharded decode layout (DuoSeqShardINT4KVCache.load_from_head_parallel): tp.reshard_heads_to_seq on the packed
codes ([B, n, N, 64] uint8) and the fp16 scale / zero rows ([B, n, N]), and tp.all_gather_rings on INT4-shaped
streaming rings.  Every rank's result must equal the source rows bit for bit."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from duo_attention_b200 import tp

MASK = np.array([[1.0, 0.0, 1.0, 1.0], [0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 1.0], [0.0, 1.0, 0.0, 0.0]])


def _int4_tensors(shape, g):
    """Random INT4 cache tensors of [B, heads, rows]: codes, scale, zero (fp16 with every bit pattern but NaN / inf)."""
    codes = torch.randint(0, 256, shape + (64,), generator=g, dtype=torch.uint8)
    halves = [torch.randint(0, 0x7C00, shape, generator=g, dtype=torch.int16) for _ in range(2)]
    sign = [torch.randint(0, 2, shape, generator=g, dtype=torch.int16) << 15 for _ in range(2)]
    scale, zero = ((h | s).view(torch.float16) for h, s in zip(halves, sign))
    return {"": codes, "_scale": scale, "_zero": zero}


def _same_bits(a, b):
    if a.dtype == torch.float16:
        a, b = a.view(torch.int16), b.view(torch.int16)
    return torch.equal(a, b)


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from duo_attention_b200.seqshard import SeqShardPlan

        g = torch.Generator().manual_seed(0)  # the same "global" cache on every rank
        n_tok, cap, block, B, W, slots = 77, 96, 8, 2, 12, 24
        plan = tp.plan_heads(MASK, world)
        sp = SeqShardPlan(world, block)
        ok = True
        for l in range(MASK.shape[0]):
            full_ids = [h for h in range(4) if MASK[l][h] > 0.5]
            stream_ids = [h for h in range(4) if MASK[l][h] <= 0.5]
            glob_full = _int4_tensors((B, 4, cap), g)     # [B, original head id, position, ...]
            glob_ring = _int4_tensors((B, 4, slots), g)
            mine_f = [h for h in plan.owners[l][rank] if MASK[l][h] > 0.5]
            mine_s = [h for h in plan.owners[l][rank] if MASK[l][h] <= 0.5]
            pos = sp.positions(rank, n_tok)
            for sfx, glob in glob_full.items():
                src = glob[:, mine_f].contiguous()
                dst = torch.zeros((B, len(full_ids), sp.capacity(cap) + 1) + tuple(glob.shape[3:]), dtype=glob.dtype)
                tp.reshard_heads_to_seq(src, plan.owners[l], MASK[l], rank, world, n_tok, block, dst)
                ok = ok and _same_bits(dst[:, :, : len(pos)], glob[:, full_ids][:, :, pos])
                ok = ok and bool((dst[:, :, len(pos):] == 0).all())
            for sfx, glob in glob_ring.items():
                src = glob[:, mine_s].contiguous()
                dst = torch.zeros((B, len(stream_ids), slots) + tuple(glob.shape[3:]), dtype=glob.dtype)
                tp.all_gather_rings(src, plan.owners[l], MASK[l], rank, world, W, dst)
                ok = ok and _same_bits(dst[:, :, :W], glob[:, stream_ids][:, :, :W])
                ok = ok and bool((dst[:, :, W:] == 0).all())  # staging slots are not moved
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_int4_cache_moves_to_the_sequence_sharded_layout(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 33500 + (os.getpid() % 2000) + world
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {r: True for r in range(world)}
