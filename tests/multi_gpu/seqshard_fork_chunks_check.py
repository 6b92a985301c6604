"""Multi-GPU check of prefill-sized chunks on forks of a sequence-sharded prompt, run under torchrun on a multi-GPU node
(tests/test_gpu_multi_seqshard_fork_chunks.py):

  head-parallel prefill of one prompt (tp.shard_model + NCCL)  ->  DuoSeqShardKVCache.load_from_head_parallel (batch 1,
  the donor)  ->  donor.fork(B)  ->  a different 300-token question per row (duo_prefill_seq_shared + the scattered
  merge)  ->  B rows decode in lockstep, eagerly and replayed by DuoDecodeGraph

must match the single-GPU patched model taking the same questions and tokens on a batch-B cache that holds the prompt
in every row (logits within tolerance, greedy tokens equal wherever its top two logits are more than 0.1 apart), graph
replay must equal eager decode bit for bit, and every rank must hold bit-identical logits."""
import copy
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from duo_attention_b200 import tp  # noqa: E402
from duo_attention_b200.graph import DuoDecodeGraph  # noqa: E402
from duo_attention_b200.kv_cache import DuoAttentionStaticKVCache, DuoSeqShardKVCache  # noqa: E402
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
    sink, recent, block, B, steps, n, S = 4, 12, 16, 4, 10, 700, 300

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
    worst, compared = 0.0, 0
    with torch.no_grad():
        prompt = torch.randint(0, 512, (1, n), generator=g).to(dev)
        pa = hp(input_ids=prompt, past_key_values=None, use_cache=True).past_key_values
        ctl = DuoAttentionStaticKVCache(single, gates, B, n + S + steps + 8, sink, recent, prefilling_chunk_size=n)
        single(input_ids=prompt.expand(B, n), past_key_values=ctl, use_cache=True)
        donor = DuoSeqShardKVCache(sp, gates, 1, n + 8, sink, recent).load_from_head_parallel(pa, plan)
        donor_g = DuoSeqShardKVCache(sp, gates, 1, n + 8, sink, recent).load_from_head_parallel(pa, plan)
        forks, forks_g = donor.fork(B, S + steps + 4), donor_g.fork(B, S + steps + 4)
        assert forks.prefix_len == n // (world * block) * (world * block) > 0
        questions = torch.randint(0, 512, (B, S), generator=g).to(dev)  # a different question per fork
        lf = sp(input_ids=questions, past_key_values=forks, use_cache=True).logits
        lfg = sp(input_ids=questions, past_key_values=forks_g, use_cache=True).logits
        lc = single(input_ids=questions, past_key_values=ctl, use_cache=True).logits
        assert torch.equal(lf, lfg)
        worst = (lf.float() - lc.float()).abs().max().item()
        torch.testing.assert_close(lf.float(), lc.float(), rtol=5e-2, atol=5e-2)
        graph = DuoDecodeGraph(sp, forks_g)
        tok = lf[:, -1:].argmax(-1).contiguous()
        for step in range(steps):
            lf = sp(input_ids=tok, past_key_values=forks, use_cache=True).logits
            lg = graph.step(tok)
            lc = single(input_ids=tok, past_key_values=ctl, use_cache=True).logits
            assert torch.equal(lf, lg), f"step {step}: graph replay differs from eager decode"
            worst = max(worst, (lf.float() - lc.float()).abs().max().item())
            torch.testing.assert_close(lf.float(), lc.float(), rtol=5e-2, atol=5e-2)
            top2 = lc.float().topk(2, -1).values
            clear = top2[..., 0] - top2[..., 1] > 0.1
            assert torch.equal(lf.argmax(-1)[clear], lc.argmax(-1)[clear]), f"step {step}: greedy tokens differ"
            compared += int(clear.sum())
            gathered = [torch.empty_like(lf) for _ in range(world)]
            dist.all_gather(gathered, lf.contiguous())
            assert all(torch.equal(gathered[0], t) for t in gathered), "ranks disagree on the logits"
            tok = lf[:, -1:].argmax(-1)
        assert forks.kv_seq_len == ctl.kv_seq_len == n + S + steps
    assert not sp._duo_seq.comm.error() and not sp._duo_comm.error(), "a peer timed out"
    t = torch.tensor([worst], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(f"SEQSHARD_FORK_CHUNKS_OK world={world} max|dlogit|={t.item():.4f} compared={compared}")
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
