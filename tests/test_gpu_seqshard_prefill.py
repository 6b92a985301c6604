"""Prefill-sized chunks on sequence-sharded caches, on one GPU: W ranks of DuoSeqShardKVCache /
DuoSeqShardINT4KVCache emulated on one device, the way tests/test_gpu_seqshard_decode.py does for decode steps.

Every rank is a real sharded cache fed its own clone of the same qkv; a local stand-in for tp.SeqComm stacks the W
partials in rank order and merges them with duo_merge_partials (what tp.merge_scattered computes, row by row; the
scattered exchange itself is tests/test_seqshard_prefill_gloo.py).  The state is an unsharded cache of the same format
(the control), scattered the way load_from_head_parallel does.  Schedules mix decode steps, chunks of 3 .. 4096 tokens
and evict_last.  After every call:

* cache bytes: every rank's slice equals the control's rows at plan.positions, bit for bit; the rows past the slice
  still hold the sentinel; the rings equal the control's;
* streaming-head rows of `out` are bit-identical to the control's where the control runs the same kernel (16-bit
  caches; INT4 caches on decode steps and on chunks the control also attends through its 16-bit image), else within
  parity of fp64 attention over the rank's 16-bit image of the ring and the chunk; every rank's merged `out` is
  bit-identical to every other rank's;
* the merged retrieval rows are within parity of fp64 attention over what the kernels attend (the 16-bit cache, the
  16-bit image of an INT4 slice for chunks longer than max_q, exact code * scale + zero for INT4 decode steps), and of
  the control's rows where it runs the same kernel;
* per rank: part_lse within 1e-3 of the fp64 log2-domain log-sum-exp over exactly the keys the token may see on that
  rank, part_o within parity of the fp64 slice output, lse = -inf / O = 0 for rows that see no key.

test_slice_visibility_is_exact checks the visibility of the two kernels of duo_prefill_seq exactly, with probe keys
(tests/test_gpu_visibility_census.py's technique) and poison in every row a call may not see.
"""
import ctypes as C

import pytest
import torch

from duo_attention_b200 import _C, tp
from duo_attention_b200.kv_cache import DuoKVCache, DuoSeqShardINT4KVCache, DuoSeqShardKVCache, ring_slot
from duo_attention_b200.seqshard import SeqShardPlan
from parity import assert_parity
from test_gpu_seqshard_decode import LocalSeqComm, _Model, host_rope_q, rope_tables
from test_gpu_seqshard_int4_decode import SENT_CODE, SENT_HALF, dequant, same_bits
from visibility_model import TupleVisibility

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
LOG2E = 1.4426950408889634
BF16, FP16 = torch.bfloat16, torch.float16
NONE, HF, FP32 = _C.ROPE_NONE, _C.ROPE_HF, _C.ROPE_FP32


class LocalComm(LocalSeqComm):
    """LocalSeqComm (rank order, duo_merge_partials) for both exchanges: the merge of a prefill-sized chunk gives every
    row the same bits as the stacked merge."""

    merge_scattered = LocalSeqComm.merge


def attn64(q, k, v, vis, scale, tok_chunk=512):
    """fp64 attention, chunked over tokens.  q [B,S,nf,G,D], k/v [B,nf,N,D], vis [S,N] -> (O, natural-log lse);
    rows that see no key get O = 0, lse = -inf."""
    os, ls = [], []
    for t0 in range(0, q.shape[1], tok_chunk):
        s = torch.einsum("bsngd,bnjd->bsngj", q[:, t0 : t0 + tok_chunk], k) * scale
        s = s.masked_fill(~vis[None, t0 : t0 + tok_chunk, None, None, :], float("-inf"))
        lse = torch.logsumexp(s, -1)
        p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
        os.append(torch.einsum("bsngj,bnjd->bsngd", p, v))
        ls.append(lse)
    return torch.cat(os, 1), torch.cat(ls, 1)


class Rig:
    """W sequence-shard rank caches of one KV format and the unsharded control of the same geometry."""

    def __init__(self, fmt, W, block, Hq, Hkv, n_full, B, dtype, max_size, sink, recent):
        self.fmt, self.W, self.block, self.Hq, self.Hkv, self.nf, self.B, self.dtype = fmt, W, block, Hq, Hkv, n_full, B, dtype
        self.sink, self.recent = sink, recent
        self.G = Hq // Hkv
        self.nfq = n_full * self.G
        self.plan = SeqShardPlan(W, block)
        self.control = DuoKVCache(1, Hq, Hkv, D, [n_full], B, max_size, sink, recent, dtype, DEV, stage_cap=16,
                                  kv_format=fmt)
        self.comm = LocalComm(W)
        cls = DuoSeqShardKVCache if fmt == "same" else DuoSeqShardINT4KVCache
        model, gates = _Model(Hq, Hkv, dtype), [[1.0] * n_full + [0.0] * (Hkv - n_full)]
        self.ranks = [cls(model, gates, B, max_size, sink, recent, seq=tp.SeqShardContext(r, W, block, self.comm))
                      for r in range(W)]
        self.high = [0] * W
        self.width = (Hq + 2 * Hkv) * D
        self.vis = TupleVisibility(sink, recent)

    def prefill(self, n, g):
        x = torch.randn(self.B, n, self.width, generator=g, device=DEV).to(self.dtype)
        self.control.attend(0, x, None, None, NONE, torch.empty(self.B, n, self.Hq, D, dtype=self.dtype, device=DEV))
        self.vis.chunk(n)

    def scatter(self):
        c, W_ = self.control, self.control.W
        n = c.kv_seq_len
        for r, rc in enumerate(self.ranks):
            pos = self.plan.positions(r, n).to(DEV)
            for name, x in rc.tensors[0].items():
                if name.startswith("full"):
                    x.fill_(SENT_CODE if x.dtype == torch.uint8 else SENT_HALF)
                    x[:, :, : len(pos)] = c.tensors[0][name][:, :, pos]
                else:
                    x[:, :, :W_] = c.tensors[0][name][:, :, :W_]
            rc.kv_seq_len_list[0], rc.total_list[0], rc.lo_list[0] = n, c.total_list[0], c.lo_list[0]
            self.high[r] = len(pos)

    def evict(self, k):
        for c in [self.control] + self.ranks:
            c.evict_last(k)
        self.vis.evict(k)

    def step(self, S, rope, g):
        c = self.control
        n = c.kv_seq_len
        qkv = torch.randn(self.B, S, self.width, generator=g, device=DEV).to(self.dtype)
        cos, sin = rope_tables(rope, n, S, self.dtype)
        oc = torch.full((self.B, S, self.Hq, D), float("nan"), dtype=self.dtype, device=DEV)
        c.attend(0, qkv.clone(), cos, sin, rope, oc, fused=(S == 1))
        outs = []
        for rc in self.ranks:
            o = torch.full_like(oc, float("nan"))
            rc.attend(0, qkv.clone(), cos, sin, rope, o)
            outs.append(o)
        torch.cuda.synchronize()
        chunk = self.vis.chunk(S)
        long_chunk = S > self.ranks[0].max_q
        what = f"n={n} S={S}"
        self.check_cache(what)
        # the control attends an INT4 chunk > max_q through its 16-bit image only for >= 128 tokens and W <= 2048
        same_kernel = self.fmt == "same" or not long_chunk or (S >= 128 and self.sink + self.recent <= 2048)
        for r, o in enumerate(outs):
            assert torch.equal(o, outs[0]), f"{what}: rank {r}'s merged output differs from rank 0's"
        if same_kernel:
            assert torch.equal(outs[0][:, :, self.nfq :], oc[:, :, self.nfq :]), f"{what}: streaming rows"
        q = host_rope_q(qkv[..., : self.Hq * D].view(self.B, S, self.Hq, D), rope, cos, sin)
        if not same_kernel and self.nfq < self.Hq:
            assert_parity(outs[0][:, :, self.nfq :], self.stream_truth(q, chunk, S), f"{what}: streaming rows vs fp64")
        if self.nfq:
            kv = [self.slice_kv(rc, long_chunk) for rc in self.ranks]
            truth, _ = self.truth(q, n, S, kv, None)
            assert_parity(outs[0][:, :, : self.nfq], truth, f"{what}: merged retrieval rows vs fp64")
            if same_kernel:
                assert_parity(outs[0][:, :, : self.nfq], oc[:, :, : self.nfq], f"{what}: merged rows vs control")
            self.check_partials(q, n, S, kv, chunk, what)

    def stream_truth(self, q, chunk, S):
        """fp64 output of the streaming q-heads over rank 0's 16-bit image of the ring and the staged chunk (what its
        kernel attended), visibility from the model: the streaming cache before the chunk plus the chunk causally."""
        dq, ns, Wr = self.ranks[0]._dq, self.Hkv - self.nf, self.sink + self.recent
        k, v = (x[: self.B * ns * dq["slots"] * D].view(self.B, ns, dq["slots"], D)[:, :, : Wr + S].double()
                for x in dq["ring"])
        vis = torch.zeros(S, Wr + S, dtype=torch.bool, device=DEV)
        vis[:, [ring_slot(p, self.sink, self.recent) for a, b in chunk.stream for p in range(a, b)]] = True
        vis[:, Wr:] = torch.ones(S, S, dtype=torch.bool, device=DEV).tril()
        qq = q.double().view(self.B, S, self.Hkv, self.G, D)[:, :, self.nf :]
        return attn64(qq, k, v, vis, D ** -0.5)[0].reshape(self.B, S, ns * self.G, D)

    def check_cache(self, what):
        n, W_ = self.ranks[0].kv_seq_len, self.control.W
        for r, rc in enumerate(self.ranks):
            loc = self.plan.local_len(r, n)
            assert rc.kv_seq_len == n
            self.high[r] = max(self.high[r], loc)
            pos = self.plan.positions(r, n).to(DEV)
            for name, x in rc.tensors[0].items():
                if name.startswith("full"):
                    assert same_bits(x[:, :, :loc], self.control.tensors[0][name][:, :, pos]), f"{what}: rank {r} {name}"
                    sent = SENT_CODE if x.dtype == torch.uint8 else SENT_HALF
                    assert (x[:, :, self.high[r] :] == sent).all(), f"{what}: rank {r} {name} written past its slice"
                else:
                    assert same_bits(x[:, :, :W_], self.control.tensors[0][name][:, :, :W_]), f"{what}: rank {r} {name}"

    def slice_kv(self, rc, image):
        """fp64 K, V of rank rc's slice as its kernel attended them: the 16-bit cache, the 16-bit image of an INT4 slice
        (chunks longer than max_q), or exact code * scale + zero (INT4 decode steps)."""
        t, rows = rc.tensors[0], rc.plan.local_len(rc.seq.rank, rc.kv_seq_len)
        if self.fmt == "same":
            return tuple(t[k][:, :, :rows].double() for k in ("full_k", "full_v"))
        if image:
            cap = rc._dq["cap"]
            return tuple(x[: self.B * self.nf * cap * D].view(self.B, self.nf, cap, D)[:, :, :rows].double()
                         for x in rc._dq["full"])
        return tuple(dequant(t[k][:, :, :rows], t[k + "_scale"][:, :, :rows], t[k + "_zero"][:, :, :rows])
                     for k in ("full_k", "full_v"))

    def truth(self, q, n, S, kv, rank):
        qq = q.double().view(self.B, S, self.Hkv, self.G, D)[:, :, : self.nf]
        tok = torch.arange(n, n + S, device=DEV)[:, None]
        if rank is None:
            k = torch.empty(self.B, self.nf, n + S, D, dtype=torch.float64, device=DEV)
            v = torch.empty_like(k)
            for r in range(self.W):
                p = self.plan.positions(r, n + S).to(DEV)
                k[:, :, p], v[:, :, p] = kv[r]
            pos = torch.arange(n + S, device=DEV)
        else:
            pos = self.plan.positions(rank, n + S).to(DEV)
            k, v = kv[rank]
        o, lse = attn64(qq, k, v, pos[None, :] <= tok, D ** -0.5)
        return o.reshape(self.B, S, self.nfq, D), lse.reshape(self.B, S, self.nfq)

    def check_partials(self, q, n, S, kv, chunk, what):
        # the visibility model: retrieval row i sees the positions [0, n + i] (one interval), so on rank r it sees the
        # plan.local_len(r, n + i + 1) first rows of the slice
        assert chunk.intervals(0, True) == [(0, n + 1)] and chunk.intervals(S - 1, True) == [(0, n + S)], what
        for r, rc in enumerate(self.ranks):
            seen = torch.tensor([self.plan.local_len(r, n + i + 1) for i in range(S)], device=DEV)
            po, pl = rc.partials(S)
            po, pl = po[:, :, : self.nfq], pl[:, :, : self.nfq]
            o64, lse = self.truth(q, n, S, kv, r)
            lse2 = lse * LOG2E
            empty = torch.isneginf(lse2)
            assert torch.equal(empty, (seen == 0)[None, :, None].expand_as(empty)), f"{what}: rank {r} visibility model"
            assert torch.equal(torch.isneginf(pl), empty), f"{what}: rank {r} lse == -inf exactly where no key is seen"
            assert (po[empty] == 0).all(), f"{what}: rank {r} part_o of rows without keys"
            if (~empty).any():
                err = (pl[~empty].double() - lse2[~empty]).abs().max().item()
                assert err <= 1e-3, f"{what}: rank {r} part_lse off by {err}"
                assert_parity(po[~empty], o64[~empty], f"{what}: rank {r} part_o vs fp64")


# id: (fmt, W, block, Hq, Hkv, n_full, B, dtype, rope, context, schedule, sink, recent); "e<k>" = evict_last(k)
CASES = {
    # every chunk size around the two kernels' boundaries, a block of 16 (a chunk spans many blocks), a ring that wraps
    "same_w2_b16_bf16": ("same", 2, 16, 16, 4, 2, 2, BF16, NONE, 40,
                         [1, 17, 1, 100, 2, 127, 128, "e3", 129, 1, 1000], 8, 24),
    # block 1024 from a short context: ranks 1, 2 see no key for the first tokens of the 1000-token chunk
    "same_w3_b1024_fp16_hf": ("same", 3, 1024, 8, 2, 1, 2, FP16, HF, 40, [1, 1000, 1, "e5", 4096, 1, 129], 8, 24),
    # eight ranks, every head a retrieval head, fp32 RoPE
    "same_w8_b16_allfull_fp32": ("same", 8, 16, 8, 2, 2, 2, BF16, FP32, 300, [127, 1, 128, 129, 1], 8, 24),
    # no retrieval heads: nothing to merge
    "same_w2_b16_nofull": ("same", 2, 16, 8, 2, 0, 2, BF16, HF, 100, [200, 1, 17], 8, 24),
    # sink + recent > 2048: the 64-row mma.sync kernel also for chunks of >= 128 tokens
    "same_w3_b16_bigring": ("same", 3, 16, 8, 2, 1, 2, FP16, NONE, 2500, [1, 200, 1, 129, "e1", 1000], 64, 2048),
    # INT4: 3- and 4-token chunks (group 4: duo_attention_seq on the image), chunks around 128, a decode step between
    "int4_w2_b16_bf16": ("int4", 2, 16, 16, 4, 2, 2, BF16, NONE, 300,
                         [1, 3, 4, 2, 17, 1, 127, 128, "e2", 129, 1000], 8, 24),
    "int4_w3_b1024_fp16_hf": ("int4", 3, 1024, 8, 2, 1, 2, FP16, HF, 2000, [1, 4096, 2, 100], 8, 24),
    "int4_w8_b16_fp32_bigring": ("int4", 8, 16, 8, 2, 2, 2, FP16, FP32, 2200, [200, 1, 129], 64, 2048),
}


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_sharded_prefill_matches_fp64(case):
    fmt, W, block, Hq, Hkv, nf, B, dtype, rope, n0, sched, sink, recent = CASES[case]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    steps = sum(s for s in sched if isinstance(s, int))
    rig = Rig(fmt, W, block, Hq, Hkv, nf, B, dtype, n0 + steps + 8, sink, recent)
    rig.prefill(n0, g)
    rig.scatter()
    rig.check_cache("after the scatter")
    for s in sched:
        if isinstance(s, str):
            rig.evict(int(s[1:]))
        else:
            rig.step(s, rope, g)
    assert rig.comm.calls == (sum(isinstance(s, int) for s in sched) if nf else 0)


def test_long_chunk_is_refused_while_a_graph_is_attached():
    rig = Rig("same", 2, 16, 8, 2, 1, 1, BF16, 300, 8, 24)
    rig.ranks[0].graph_attached = True
    qkv = torch.zeros(1, 17, rig.width, dtype=BF16, device=DEV)
    with pytest.raises(ValueError, match="DuoDecodeGraph"):
        rig.ranks[0].attend(0, qkv, None, None, NONE, torch.empty(1, 17, 8, D, dtype=BF16, device=DEV))
    assert rig.ranks[0].kv_seq_len == 0


# ---- exact visibility: probe keys --------------------------------------------------------------------------------
POISON = 127


@pytest.mark.parametrize("W,block,n,S,big_ring", [
    (2, 16, 100, 127, False), (2, 16, 100, 128, False), (2, 16, 96, 129, False), (3, 128, 250, 256, False),
    (3, 128, 0, 300, False), (4, 16, 1024, 128, True), (2, 128, 127, 129, True), (8, 16, 16, 255, False)])
def test_slice_visibility_is_exact(W, block, n, S, big_ring):
    """Every key of a rank's slice gets the same logit and a one-hot value on a dimension chosen from its position,
    rows past the slice are poison (same logit, value on dimension 127), so a row's part_o is the histogram of the keys
    it sees divided by their number and part_lse = logit * scale * log2(e) + log2(count).  Both are checked exactly for
    every rank, row and retrieval q-head, against plan.positions(rank, n + t + 1).  The wgmma kernel serves chunks of
    >= 128 tokens, the 64-row mma.sync kernel the others and every chunk when sink + recent > 2048 (big_ring)."""
    Hq, Hkv, B, dtype = 8, 2, 2, BF16
    sink, recent = (64, 2048) if big_ring else (4, 12)
    plan = SeqShardPlan(W, block)
    cap = plan.capacity(n + S) + 64
    lib = _C.load()
    scale = D ** -0.5
    u = torch.where(torch.arange(D, device=DEV) % 3 == 0, -1.0, 1.0)
    for rank in range(W):
        c = DuoKVCache(1, Hq, Hkv, D, [Hkv], B, cap, sink, recent, dtype, DEV, stage_cap=S)
        t = c.tensors[0]
        rows = plan.local_len(rank, n + S)
        pos = plan.positions(rank, n + S).to(DEV)
        t["full_k"][:] = u.to(dtype)  # every row, poison included, has the probe logit
        t["full_v"].zero_()
        t["full_v"][..., POISON] = 1.0
        t["full_v"][:, :, :rows] = 0.0
        t["full_v"][:, :, torch.arange(rows, device=DEV), pos % 120] = 1.0
        q = u.to(dtype).expand(B, S, Hq, D).contiguous()
        out = torch.empty(B, S, Hq, D, dtype=dtype, device=DEV)
        po = torch.full((B, S, Hq, D), float("nan"), device=DEV)
        pl = torch.full((B, S, Hq), float("nan"), device=DEV)
        st = _C.CacheState(n, n, max(sink, n - recent), None)
        st.seq_rank, st.seq_world, st.seq_block = rank, W, block
        _C.check(lib.duo_prefill_seq(c.handles[0], C.byref(st), q.data_ptr(), Hq * D, out.data_ptr(), po.data_ptr(),
                                     pl.data_ptr(), S, scale, c.workspace.data_ptr(), c.workspace.numel(),
                                     torch.cuda.current_stream(DEV).cuda_stream))
        torch.cuda.synchronize()
        exp_o = torch.zeros(S, D, dtype=torch.float64)
        cnt = torch.zeros(S, dtype=torch.float64)
        for i in range(S):
            p = plan.positions(rank, n + i + 1)
            cnt[i] = len(p)
            if len(p):
                exp_o[i] = torch.bincount(p % 120, minlength=D).double() / len(p)
        logit2 = float(u @ u) * scale * LOG2E
        exp_l = torch.where(cnt > 0, logit2 + torch.log2(cnt.clamp_min(1)), torch.full_like(cnt, float("-inf")))
        what = f"rank {rank}"
        for h in range(Hq):
            got_o, got_l = po[:, :, h].double().cpu(), pl[:, :, h].double().cpu()
            assert (got_o[..., POISON] == 0).all(), f"{what} head {h}: a poison row was attended"
            assert torch.allclose(got_o, exp_o.expand_as(got_o), rtol=0, atol=1e-6), f"{what} head {h}: key set"
            assert torch.equal(torch.isneginf(got_l), torch.isneginf(exp_l).expand_as(got_l)), f"{what} head {h}"
            fin = ~torch.isneginf(exp_l).expand_as(got_l)
            assert torch.allclose(got_l[fin], exp_l.expand_as(got_l)[fin], rtol=0, atol=1e-4), f"{what} head {h}: lse"
