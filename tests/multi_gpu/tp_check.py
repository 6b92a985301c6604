"""Multi-GPU check (run under torchrun on a multi-GPU node, e.g.
   python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
       --master-port 29511 tests/multi_gpu/tp_check.py):
the head-parallel shards (NCCL all-reduce per layer) reproduce the single-GPU patched model."""
import copy
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from duo_attention_b200 import tp  # noqa: E402
from duo_attn.patch import enable_duo_attention_eval  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(0)
    cfg = LlamaConfig(hidden_size=1024, num_attention_heads=8, num_key_value_heads=8 if world > 4 else 4, head_dim=128,
                      num_hidden_layers=3, intermediate_size=2048, vocab_size=512, max_position_embeddings=8192,
                      rope_theta=10000.0, attn_implementation="eager")
    full = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    n_kv = cfg.num_key_value_heads
    rng = np.random.RandomState(1)
    gates = (rng.rand(3, n_kv) > 0.5).astype(float)
    sink, recent = 4, 12
    shard, local_mask = tp.shard_model(full, gates, rank, world)
    enable_duo_attention_eval(shard, local_mask, sink, recent)
    shard.to(dev)
    tp.install_allreduce(shard)
    shard._duo_tp_pipeline_rows, shard._duo_tp_pipeline_blocks = 128, 3  # chunks of >= 128 rows: pipelined exchange
    single = copy.deepcopy(full)
    enable_duo_attention_eval(single, gates, sink, recent)
    single.to(dev)
    g = torch.Generator().manual_seed(2)
    pa = pb = None
    worst = 0.0
    with torch.no_grad():
        for S in [150, 1, 1, 40, 1, 130, 1]:
            ids = torch.randint(0, 512, (1, S), generator=g).to(dev)
            oa = shard(input_ids=ids, past_key_values=pa, use_cache=True)
            ob = single(input_ids=ids, past_key_values=pb, use_cache=True)
            pa, pb = oa.past_key_values, ob.past_key_values
            err = (oa.logits - ob.logits).abs().max().item()
            worst = max(worst, err)
            torch.testing.assert_close(oa.logits, ob.logits, rtol=5e-2, atol=5e-2)
    t = torch.tensor([worst], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(f"TP_CHECK_OK world={world} max|dlogit|={t.item():.4f}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
