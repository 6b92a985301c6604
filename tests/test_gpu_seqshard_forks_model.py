"""Forks of a sequence-sharded prompt at model level, ranks emulated on one GPU: a small random Llama decodes B
continuations of one prompt through ``model(input_ids=[B, 1], past_key_values=...)`` and through ``DuoDecodeGraph``.

``RankGroup`` is the one cache the model sees.  Its ``attend(l, ...)`` runs the attend of every emulated rank's cache in
rank order on the same qkv, and LocalSeqComm merges the W partials at the last rank's call, so one forward of the model
drives all W ranks layer by layer; every other cache call goes to every rank.  The prompt is prefilled on one GPU and
scattered into the ranks as load_from_head_parallel places it.  The control is a batch-B DuoSeqShardKVCache per rank
whose rows each hold the prompt.  Both are fed the forks' greedy tokens; the greedy tokens must agree wherever the
control's top two logits are more than 0.1 apart, and graph replay must equal eager decode bit for bit."""
import numpy as np
import pytest
import torch

from duo_attention_b200 import tp
from duo_attention_b200.kv_cache import DuoAttentionStaticKVCache, DuoKVCache, DuoSeqShardKVCache
from duo_attention_b200.seqshard import SeqShardPlan
from test_gpu_seqshard_decode import LocalSeqComm

pytestmark = pytest.mark.gpu
GATES = np.array([[0.9, 0.1], [0.2, 0.8]])
SINK, RECENT = 4, 12


class RankGroup(DuoKVCache):
    """W emulated rank caches behind one DuoKVCache: attend runs every rank, the rest is forwarded to every rank (and
    read from rank 0).  Rank 0's output is what the model continues with; the merge gives every rank the same bits."""

    def __init__(self, ranks):  # no DuoKVCache.__init__: the ranks hold everything
        object.__setattr__(self, "ranks", ranks)

    def __getattr__(self, name):
        return getattr(self.ranks[0], name)

    def __setattr__(self, name, value):
        for c in self.ranks:
            setattr(c, name, value)

    def attend(self, l, qkv, cos, sin, rope_mode, out, scale=None, force_mma=False, fused=True):
        outs = [out] + [torch.empty_like(out) for _ in self.ranks[1:]]
        for c, o in zip(self.ranks, outs):
            c.attend(l, qkv, cos, sin, rope_mode, o, scale, force_mma, fused)
        return out

    def _each(name):
        def f(self, *args):
            return [getattr(c, name)(*args) for c in self.ranks][0]
        f.__name__ = name
        return f

    for _n in ("enable_device_state", "sync_device_state", "advance_device", "advance_host", "check_room",
               "evict_last", "clear", "snapshot_state", "restore_state"):  # (every rank holds the same occupancy)
        locals()[_n] = _each(_n)
    del _n, _each

    def snapshot_ring(self):
        return [c.snapshot_ring() for c in self.ranks]

    def restore_ring(self, snaps):
        for c, s in zip(self.ranks, snaps):
            c.restore_ring(s)

    def __del__(self):  # the ranks own their handles
        pass

    @property
    def kv_seq_len(self):
        return self.ranks[0].kv_seq_len

    @property
    def memory_usage(self):
        return sum(c.memory_usage for c in self.ranks)


def _model(seed):
    from transformers import LlamaConfig, LlamaForCausalLM

    from duo_attn.patch import enable_duo_attention_eval

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                      intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                      attn_implementation="eager")
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    enable_duo_attention_eval(model, GATES, SINK, RECENT)
    return model.cuda()


def _sharded(model, src, W, block, B, max_size):
    """W rank caches of batch B holding src's prompt in every row (load_from_head_parallel's placement)."""
    plan, comm = SeqShardPlan(W, block), LocalSeqComm(W)
    ranks = [DuoSeqShardKVCache(model, GATES, B, max_size, SINK, RECENT, seq=tp.SeqShardContext(r, W, block, comm))
             for r in range(W)]
    n, Wr = src.kv_seq_len, src.W
    for r, c in enumerate(ranks):
        pos = plan.positions(r, n).cuda()
        for l in range(c.num_layers):
            for name, t in c.tensors[l].items():
                s = src.tensors[l][name]
                if not t.numel():
                    continue
                if name.startswith("full"):
                    t[:, :, : len(pos)] = s[:, :, pos]
                else:
                    t[:, :, :Wr] = s[:, :, :Wr]
            c.kv_seq_len_list[l], c.total_list[l], c.lo_list[l] = n, src.total_list[l], src.lo_list[l]
        c.sync_device_state()
    return ranks


@pytest.mark.parametrize("W,block,n", [(2, 16, 300), (3, 8, 200)])
def test_model_decodes_forks_like_the_control(W, block, n):
    from duo_attention_b200.graph import DuoDecodeGraph

    model = _model(41 + W)
    B, steps = 5, 12
    g = torch.Generator().manual_seed(W)
    prompt = torch.randint(0, 512, (1, n), generator=g).cuda()
    run = lambda ids, past: model(input_ids=ids, past_key_values=past, use_cache=True).logits
    with torch.no_grad():
        src = DuoAttentionStaticKVCache(model, GATES, 1, n + 8, SINK, RECENT, prefilling_chunk_size=n)
        first = run(prompt, src)
        donors = _sharded(model, src, W, block, 1, n + steps + 8)
        donors_g = _sharded(model, src, W, block, 1, n + steps + 8)
        control = RankGroup(_sharded(model, src, W, block, B, n + steps + 8))
        forks = RankGroup([d.fork(B, steps + 4) for d in donors])
        forks_g = RankGroup([d.fork(B, steps + 4) for d in donors_g])
        P = forks.ranks[0].prefix_len
        assert P == n // (W * block) * (W * block) > 0
        graph = DuoDecodeGraph(model, forks_g)
        # every fork starts from the prompt's greedy token, then they diverge through different sampled tokens
        tok = first[:, -1:].argmax(-1).expand(B, 1).contiguous()
        tok[1:, 0] = torch.randint(0, 512, (B - 1,), generator=g).cuda()
        compared = 0
        for step in range(steps):
            lf = run(tok, forks)
            lg = graph.step(tok)
            lc = run(tok, control)
            assert torch.equal(lf, lg), f"step {step}: DuoDecodeGraph replay differs from eager decode"
            torch.testing.assert_close(lf.float(), lc.float(), rtol=5e-2, atol=5e-2)
            top2 = lc.float().topk(2, -1).values
            clear = top2[..., 0] - top2[..., 1] > 0.1
            assert torch.equal(lf.argmax(-1)[clear], lc.argmax(-1)[clear]), f"step {step}: greedy tokens differ"
            compared += int(clear.sum())
            tok = lf[:, -1:].argmax(-1)
        assert compared >= B * steps // 4
        assert forks.kv_seq_len == forks_g.kv_seq_len == control.kv_seq_len == n + steps
        # the captured forks refuse clear(): the graph reads the donors' prefix at a fixed P
        before = [[{k: v.clone() for k, v in t.items()} for t in c.tensors] for c in forks_g.ranks]
        with pytest.raises(ValueError, match="DuoDecodeGraph"):
            forks_g.clear()
        torch.cuda.synchronize()
        for c, b in zip(forks_g.ranks, before):
            assert c.kv_seq_len == n + steps and c.prefix_len == P
            for t, bt in zip(c.tensors, b):
                assert all(torch.equal(t[k], bt[k]) for k in bt)
