"""Multi-GPU check of prefill-sized chunks on the sequence-sharded layout, run under torchrun on a multi-GPU node
(tests/test_gpu_multi_seqshard_prefill.py):

  head-parallel prefill (tp.shard_model + NCCL)  ->  tp.reshard_heads_to_seq (DuoSeqShardKVCache.load_from_head_parallel)
  ->  decode steps  ->  a second turn of 1,000 tokens on the sharded cache (duo_prefill_seq + the row-scattered merge,
      NCCL all_to_all_single / all_gather_into_tensor)  ->  decode steps again

must reproduce the logits of the single-GPU patched model token by token (the whole second turn included), and every
rank must hold bit-identical logits."""
import copy
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from duo_attention_b200 import tp  # noqa: E402
from duo_attention_b200.kv_cache import DuoSeqShardKVCache  # noqa: E402
from duo_attn.patch import enable_duo_attention_eval  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(0)
    n_kv = 8 if world > 4 else 4
    cfg = LlamaConfig(hidden_size=1024, num_attention_heads=2 * n_kv, num_key_value_heads=n_kv, head_dim=128,
                      num_hidden_layers=3, intermediate_size=2048, vocab_size=512, max_position_embeddings=8192,
                      rope_theta=10000.0, attn_implementation="eager")
    full = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    rng = np.random.RandomState(1)
    gates = (rng.rand(3, n_kv) > 0.5).astype(float)
    gates[1] = 0.0          # a layer without retrieval heads
    gates[2, :] = 1.0       # a layer without streaming heads
    sink, recent, block = 4, 12, 16

    single = copy.deepcopy(full)
    enable_duo_attention_eval(single, gates, sink, recent)
    single.to(dev)
    hp, local_mask = tp.shard_model(full, gates, rank, world)
    enable_duo_attention_eval(hp, local_mask, sink, recent)
    hp.to(dev)
    tp.install_allreduce(hp)
    plan = tp.plan_heads(gates, world)
    sp = tp.shard_model_seq(full, rank, world)
    enable_duo_attention_eval(sp, gates, sink, recent)
    sp.to(dev)
    tp.install_seq_shard(sp, block=block)

    g = torch.Generator().manual_seed(2)
    worst = 0.0
    with torch.no_grad():
        pa = pb = None
        for S in [150, 1, 40, 130]:  # first turn: head-parallel prefill
            ids = torch.randint(0, 512, (1, S), generator=g).to(dev)
            oa = hp(input_ids=ids, past_key_values=pa, use_cache=True)
            ob = single(input_ids=ids, past_key_values=pb, use_cache=True)
            pa, pb = oa.past_key_values, ob.past_key_values
        cache = DuoSeqShardKVCache(sp, gates, 1, 2048, sink, recent).load_from_head_parallel(pa, plan)
        assert cache.kv_seq_len == pb.kv_seq_len == 321

        def check(ids, logits_sp):
            nonlocal worst
            want = single(input_ids=ids, past_key_values=pb, use_cache=True).logits
            worst = max(worst, (logits_sp.float() - want.float()).abs().max().item())
            torch.testing.assert_close(logits_sp.float(), want.float(), rtol=5e-2, atol=5e-2)
            gathered = [torch.empty_like(logits_sp) for _ in range(world)]
            dist.all_gather(gathered, logits_sp.contiguous())
            assert all(torch.equal(gathered[0], t) for t in gathered), "ranks disagree on the logits"

        def decode(n):
            for _ in range(n):
                tok = torch.randint(0, 512, (1, 1), generator=g).to(dev)
                check(tok, sp(input_ids=tok, past_key_values=cache, use_cache=True).logits)

        decode(8)
        turn = torch.randint(0, 512, (1, 1000), generator=g).to(dev)  # the second user turn, in one chunk
        check(turn, sp(input_ids=turn, past_key_values=cache, use_cache=True).logits)
        decode(8)
        assert cache.kv_seq_len == pb.kv_seq_len == 321 + 8 + 1000 + 8
    assert not sp._duo_seq.comm.error() and not sp._duo_comm.error(), "a peer timed out"
    t = torch.tensor([worst], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(f"SEQSHARD_PREFILL_OK world={world} max|dlogit|={t.item():.4f}")
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
