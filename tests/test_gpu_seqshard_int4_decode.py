"""Sequence-sharded decode on an INT4 cache, on one GPU: W ranks of DuoSeqShardINT4KVCache emulated on one device, the
way tests/test_gpu_seqshard_decode.py does for 16-bit caches (its LocalSeqComm merges the W partials in rank order with
duo_merge_partials, the algebra and order of duo_seq_merge).

The control is an unsharded INT4 DuoKVCache of the same geometry, scattered to the ranks the way
load_from_head_parallel does.  After every step:

* cache bytes: every rank's slice of codes, scale and zero equals the control's rows at plan.positions, bit for bit;
  the rows past the slice still hold the sentinel (a huge logit if it were ever attended); the rings equal the
  control's;
* streaming-head rows of `out` are bit-identical to the control's, and all ranks' merged `out` are bit-identical;
* the merged retrieval rows, and the control's, are within parity of fp64 attention over the dequantised values the
  kernels attend: code * scale + zero, exact (the decode kernels apply scale and zero algebraically to the logits and
  outputs, so the fp16 rounding of a dequantised element, K2 in tests/int4_bf16_oracle.py, never happens);
* per-rank partials: part_lse within 1e-3 of the fp64 log2-domain log-sum-exp over the keys the token sees on that
  rank, part_o within parity, -inf / 0 for rows that see no key on the rank.  The INT4 kernels form a logit as
  s * (Q . (1024 + c) - 1024 sum(Q)) + z sum(Q) in fp32, whose absolute error grows with |q|: a case with q scaled by
  k (the sharp-softmax cases) is held to k * 1e-3.
"""
import ctypes as C

import pytest
import torch

from duo_attention_b200 import _C, tp
from duo_attention_b200.kv_cache import DuoKVCache, DuoSeqShardINT4KVCache
from duo_attention_b200.seqshard import SeqShardPlan
from parity import assert_parity
from test_gpu_seqshard_decode import LocalSeqComm, _Model, attn64, host_rope_q, partials, rope_tables

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
LOG2E = 1.4426950408889634
SINK, RECENT = 8, 24
SENT_CODE, SENT_HALF = 0xFF, 64.0  # dequantises to 15 * 64 + 64 per element: a huge logit if ever attended
SFX = ("", "_scale", "_zero")
BF16, FP16 = torch.bfloat16, torch.float16
NONE, HF, FP32 = _C.ROPE_NONE, _C.ROPE_HF, _C.ROPE_FP32


def dequant(codes, scale, zero):
    """INT4 rows as fp64: code * scale + zero (exact); codes [..., 64] (high nibble first), scale / zero [...]."""
    c = torch.stack([codes >> 4, codes & 15], -1).flatten(-2).double()
    return c * scale.double()[..., None] + zero.double()[..., None]


def same_bits(a, b):
    if a.dtype == torch.float16:
        a, b = a.view(torch.int16), b.view(torch.int16)
    return torch.equal(a, b)


def fill_random(t, names, g, kscale=1.0):
    for n in names:
        t[n].random_(0, 256, generator=g)
        s = kscale if n.endswith("_k") else 1.0
        t[n + "_scale"].uniform_(0.05 * s, 0.25 * s, generator=g)
        t[n + "_zero"].uniform_(-2.0 * s, -0.5 * s, generator=g)


class Rig:
    """W INT4 sequence-shard rank caches and the unsharded INT4 control of the same geometry."""

    def __init__(self, W, block, Hq, Hkv, n_full, B, dtype, max_size):
        self.W, self.block, self.Hq, self.Hkv, self.nf, self.B, self.dtype = W, block, Hq, Hkv, n_full, B, dtype
        self.G = Hq // Hkv
        self.nfq = n_full * self.G
        self.plan = SeqShardPlan(W, block)
        self.control = DuoKVCache(1, Hq, Hkv, D, [n_full], B, max_size, SINK, RECENT, dtype, DEV, stage_cap=8,
                                  kv_format="int4")
        self.ranks = self.make_ranks(max_size)
        self.width = (Hq + 2 * Hkv) * D

    def make_ranks(self, max_size):
        self.comm = LocalSeqComm(self.W)
        model = _Model(self.Hq, self.Hkv, self.dtype)
        gates = [[1.0] * self.nf + [0.0] * (self.Hkv - self.nf)]
        ranks = [DuoSeqShardINT4KVCache(model, gates, self.B, max_size, SINK, RECENT,
                                        seq=tp.SeqShardContext(r, self.W, self.block, self.comm)) for r in range(self.W)]
        self.high = [0] * self.W
        return ranks

    def prefill(self, n, g):
        c = self.control
        if n <= 2048:  # the first chunk attends its raw K/V and quantises them into the cache
            x = torch.randn(self.B, n, self.width, generator=g, device=DEV).to(self.dtype)
            c.attend(0, x, None, None, NONE, torch.empty(self.B, n, self.Hq, D, dtype=self.dtype, device=DEV))
            return
        fill_random(c.tensors[0], ("full_k", "full_v", "ring_k", "ring_v"), g)
        c.kv_seq_len_list[0], c.total_list[0], c.lo_list[0] = n, n, max(SINK, n - RECENT)

    def scatter(self, ranks=None):
        """load_from_head_parallel without torch.distributed: rank r takes the control's rows at plan.positions(r, n)."""
        c, W_ = self.control, self.control.W
        n = c.kv_seq_len
        for r, rc in enumerate(ranks or self.ranks):
            t = rc.tensors[0]
            pos = self.plan.positions(r, n).to(DEV)
            for name, x in t.items():
                if name.startswith("full"):
                    x.fill_(SENT_CODE if x.dtype == torch.uint8 else SENT_HALF)
                    x[:, :, : len(pos)] = c.tensors[0][name][:, :, pos]
                else:
                    x[:, :, :W_] = c.tensors[0][name][:, :, :W_]
            rc.kv_seq_len_list[0], rc.total_list[0], rc.lo_list[0] = n, c.total_list[0], c.lo_list[0]
            rc.sync_device_state()
            self.high[r] = len(pos)

    def evict(self, k):
        for c in [self.control] + self.ranks:
            c.evict_last(k)

    def inputs(self, S, g, qscale=1.0):
        x = torch.randn(self.B, S, self.width, generator=g, device=DEV)
        x[..., : self.Hq * D] *= qscale
        return x.to(self.dtype)

    def step(self, S, rope, g, qscale=1.0, fused=True):
        c = self.control
        n = c.kv_seq_len
        qkv = self.inputs(S, g, qscale)
        cos, sin = rope_tables(rope, n, S, self.dtype)
        oc = torch.full((self.B, S, self.Hq, D), float("nan"), dtype=self.dtype, device=DEV)
        c.attend(0, qkv.clone(), cos, sin, rope, oc, fused=fused and S == 1)  # the kernel family of the sharded step
        outs = []
        for rc in self.ranks:
            o = torch.full_like(oc, float("nan"))
            rc.attend(0, qkv.clone(), cos, sin, rope, o, fused=fused)
            outs.append(o)
        torch.cuda.synchronize()
        what = f"n={n} S={S} fused={fused}"
        self.check_cache(what)
        for r, o in enumerate(outs):
            assert torch.equal(o[:, :, self.nfq :], oc[:, :, self.nfq :]), f"{what}: rank {r} streaming rows"
            assert torch.equal(o, outs[0]), f"{what}: rank {r}'s merged output differs from rank 0's"
        q = host_rope_q(qkv[..., : self.Hq * D].view(self.B, S, self.Hq, D), rope, cos, sin)
        if self.nfq:
            truth, _ = self.truth(q, n, S, None)
            assert_parity(outs[0][:, :, : self.nfq], truth, f"{what}: merged retrieval rows vs fp64")
            assert_parity(oc[:, :, : self.nfq], truth, f"{what}: control vs fp64")
            self.check_partials(q, n, S, what, lse_tol=1e-3 * qscale)
        return outs[0]

    # ---- checks ----------------------------------------------------------------------------------------------------
    def check_cache(self, what, ranks=None, ref=None):
        n = (ranks or self.ranks)[0].kv_seq_len
        W_ = self.control.W
        for r, rc in enumerate(ranks or self.ranks):
            t = rc.tensors[0]
            loc = self.plan.local_len(r, n)
            assert rc.kv_seq_len == n
            self.high[r] = max(self.high[r], loc)
            pos = self.plan.positions(r, n).to(DEV)
            for name, x in t.items():
                if name.startswith("full"):
                    want = self.control.tensors[0][name][:, :, pos] if ref is None else ref[r].tensors[0][name][:, :, :loc]
                    assert same_bits(x[:, :, :loc], want), f"{what}: rank {r} {name} slice"
                    sent = SENT_CODE if x.dtype == torch.uint8 else SENT_HALF
                    assert (x[:, :, self.high[r] :] == sent).all(), f"{what}: rank {r} {name} written past its slice"
                else:
                    src = self.control if ref is None else ref[r]
                    assert same_bits(x[:, :, :W_], src.tensors[0][name][:, :, :W_]), f"{what}: rank {r} {name}"

    def slice_kv(self, rc, rows):
        t = rc.tensors[0]
        return tuple(dequant(t[k][:, :, :rows], t[k + "_scale"][:, :, :rows], t[k + "_zero"][:, :, :rows])
                     for k in ("full_k", "full_v"))

    def truth(self, q, n, S, rank, ranks=None):
        """fp64 attention of the chunk's retrieval rows over all positions (rank None) or over `rank`'s slice."""
        ranks = ranks or self.ranks
        qq = q.double().view(self.B, S, self.Hkv, self.G, D)[:, :, : self.nf]
        tok = torch.arange(n, n + S, device=DEV)[:, None]
        if rank is None:
            k = torch.empty(self.B, self.nf, n + S, D, dtype=torch.float64, device=DEV)
            v = torch.empty_like(k)
            for r, rc in enumerate(ranks):
                p = self.plan.positions(r, n + S).to(DEV)
                k[:, :, p], v[:, :, p] = self.slice_kv(rc, len(p))
            pos = torch.arange(n + S, device=DEV)
        else:
            pos = self.plan.positions(rank, n + S).to(DEV)
            k, v = self.slice_kv(ranks[rank], len(pos))
        o, lse = attn64(qq, k, v, pos[None, :] <= tok, D ** -0.5)
        return o.reshape(self.B, S, self.nfq, D), lse.reshape(self.B, S, self.nfq)

    def check_partials(self, q, n, S, what, ranks=None, lse_tol=1e-3):
        for r, rc in enumerate(ranks or self.ranks):
            po, pl = partials(rc, S)
            po, pl = po[:, :, : self.nfq], pl[:, :, : self.nfq]
            o64, lse = self.truth(q, n, S, r, ranks)
            lse2 = lse * LOG2E
            empty = torch.isneginf(lse2)
            assert torch.equal(torch.isneginf(pl), empty), f"{what}: rank {r} lse == -inf exactly where no key is seen"
            assert (po[empty] == 0).all(), f"{what}: rank {r} part_o of rows without keys"
            if (~empty).any():
                err = (pl[~empty].double() - lse2[~empty]).abs().max().item()
                assert err <= lse_tol, f"{what}: rank {r} part_lse off by {err}"
                assert_parity(po[~empty], o64[~empty], f"{what}: rank {r} part_o vs fp64")


# id: (W, block, Hq, Hkv, n_full, B, dtype, rope, context, schedule, qscale); "e<k>" in a schedule = evict_last(k)
CASES = {
    # ranks 1.. start empty (3 tokens, block 16); fused tokens and 2-token chunks open rank 1's first block and cross
    # the round boundary 32
    "w2b16_g4_from_empty": (2, 16, 32, 8, 4, 1, BF16, NONE, 3, [1, 2, 2, 1, 2, 2, 1, 1, 2, 2, 2, 1, 2, 2, 1, 2, 1], 1),
    # group 8 (one token per step): evict_last(1) takes back the token that opened rank 1's first block, evict_last(2)
    # goes back across the round boundary 15
    "w3b5_g8_fp16_hf_evict": (3, 5, 32, 4, 2, 2, FP16, HF, 4, [1, 1, "e1", 1, 1, 1, 1, 1, 1, 1, 1, 1, "e2", 1, 1], 1),
    # round-robin ownership, MHA chunks of up to 8 tokens that touch every rank, no streaming heads
    "w4b1_mha_allfull_fp32": (4, 1, 8, 8, 8, 1, BF16, FP32, 3, [8, 5, 1, 1, 4, "e2", 3, 8], 1),
    # no retrieval heads: nothing to merge
    "w8b64_nofull": (8, 64, 32, 8, 0, 2, BF16, NONE, 500, [1, 2, 1, 2], 1),
    # the next token is the last of a round; then the first of the next round
    "w8b64_g4_fp16_hf_round": (8, 64, 32, 8, 3, 1, FP16, HF, 1023, [1, 1, 1, 2, "e2", 2, 1], 1),
    # a block that does not divide the 128-key tile
    "w2b100_g4_round": (2, 100, 32, 8, 2, 2, BF16, NONE, 199, [1, 1, 2, 2, 1, "e1", 2], 1),
    "w2b100_g4_fp16_fp32_block": (2, 100, 32, 8, 5, 1, FP16, FP32, 97, [2, 1, 2, 1, 2, 1], 1),
    # ~40K keys per slice: many split-KV CTAs per slice and the in-launch hierarchical merge
    "w2b1024_40k": (2, 1024, 32, 8, 4, 1, BF16, NONE, 80000, [1, 2, 1, 2, "e1", 1], 1),
    "w4b1024_fp16_hf_40k": (4, 1024, 32, 8, 2, 1, FP16, HF, 160000, [1, 2, "e1", 1], 1),
    # sharp softmax (logit std 8): the largest logit sits on one rank
    "w4b16_sharp": (4, 16, 32, 8, 4, 2, BF16, NONE, 300, [1, 2, 1, 2, 1], 8),
    "w3b64_fp16_sharp_hf": (3, 64, 32, 8, 8, 1, FP16, HF, 700, [1, 2, 1, 1], 8),
}


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_sharded_int4_decode_matches_fp64(case):
    W, block, Hq, Hkv, nf, B, dtype, rope, n0, sched, qscale = CASES[case]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    steps = sum(s for s in sched if isinstance(s, int))
    rig = Rig(W, block, Hq, Hkv, nf, B, dtype, n0 + steps + 8)
    rig.prefill(n0, g)
    rig.scatter()
    rig.check_cache("after the scatter")
    for s in sched:
        if isinstance(s, str):
            rig.evict(int(s[1:]))
        else:
            rig.step(s, rope, g, qscale)
    assert rig.comm.calls == (sum(isinstance(s, int) for s in sched) if nf else 0)


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_fused_and_unfused_single_token_leave_the_same_cache(dtype):
    """At q_len 1 the fused launch (duo_decode_fused_seq_int4) and the unfused chain (duo_rope_append,
    duo_attention_seq_int4, merge, duo_stream_commit) write the same cache bytes on every rank; both are held to fp64."""
    W, block, Hq, Hkv, nf, B, rope = 3, 5, 32, 8, 3, 2, HF
    fz, uf = (Rig(W, block, Hq, Hkv, nf, B, dtype, 300) for _ in range(2))
    for rig in (fz, uf):  # the same prefill: the same cache bytes
        rig.prefill(200, torch.Generator(device=DEV).manual_seed(11))
        rig.scatter()
    fz.check_cache("after the scatter", ranks=uf.ranks, ref=fz.ranks)
    for i in range(2 * block * W + 2):  # every rank owns a few new tokens
        fz.step(1, rope, torch.Generator(device=DEV).manual_seed(100 + i), fused=True)
        uf.step(1, rope, torch.Generator(device=DEV).manual_seed(100 + i), fused=False)
        uf.check_cache(f"step {i}: unfused vs fused", ranks=uf.ranks, ref=fz.ranks)


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_exact_local_capacity(dtype):
    """Every rank holds exactly plan.capacity(n0 + 1) rows (a multiple of 64, so the INT4 allocation is exact): the
    step at n0 fills the owner's last row; at n0 + 1 the owner refuses the next token — ValueError from the cache,
    DUO_EOVERFLOW from each C entry point — and the other ranks take the same step."""
    W, block, Hq, Hkv, nf, B = 2, 100, 32, 8, 4, 2
    n0 = 227  # positions 200..299 are rank 0's second block
    rig = Rig(W, block, Hq, Hkv, nf, B, dtype, n0 + 16)
    g = torch.Generator(device=DEV).manual_seed(5)
    cap = rig.plan.capacity(n0 + 1)
    assert cap == 128 and rig.plan.local_len(0, n0 + 1) == cap and rig.plan.owner(n0) == 0
    for rc in rig.ranks:
        rc._set_layer(0, cap, rc.stage_cap_list[0])
        assert rc.tensors[0]["full_k"].shape[2] == cap
    rig.prefill(n0, g)
    rig.scatter()
    rig.step(1, HF, g)
    n = n0 + 1
    owner = rig.plan.owner(n)
    assert owner == 0
    qkv = rig.inputs(1, g)
    cos, sin = rope_tables(HF, n, 1, dtype)
    out = torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV)
    own = rig.ranks[owner]
    with pytest.raises(ValueError, match="Trying to put 1 KVs into a cache with max size"):
        own.attend(0, qkv.clone(), cos, sin, HF, out)
    lib, st, stream = own.lib, own.state(0), torch.cuda.current_stream(DEV).cuda_stream
    po, pl = partials(own, 1)
    h, ws = own.handles[0], own.workspace
    rcs = {
        "duo_decode_fused_seq_int4": lib.duo_decode_fused_seq_int4(
            h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cos.data_ptr(), sin.data_ptr(), HF, out.data_ptr(),
            po.data_ptr(), pl.data_ptr(), D ** -0.5, ws.data_ptr(), ws.numel(), stream),
        "duo_rope_append": lib.duo_rope_append(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cos.data_ptr(),
                                               sin.data_ptr(), HF, 1, stream),
        "duo_attention_seq_int4": lib.duo_attention_seq_int4(
            h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out.data_ptr(), po.data_ptr(), pl.data_ptr(), 1, D ** -0.5,
            ws.data_ptr(), ws.numel(), stream),
    }
    for name, rc in rcs.items():
        assert rc == _C.DUO_EOVERFLOW, (name, rc, _C.last_error())
    assert own.kv_seq_len == n
    for r, rc in enumerate(rig.ranks):
        if r != owner:
            rc.attend(0, qkv.clone(), cos, sin, HF, torch.empty_like(out))
            assert rc.kv_seq_len == n + 1
    torch.cuda.synchronize()
    for r, rc in enumerate(rig.ranks):  # nothing written past the slices; the refused owner is untouched
        for name, x in rc.tensors[0].items():
            if name.startswith("full"):
                sent = SENT_CODE if x.dtype == torch.uint8 else SENT_HALF
                assert (x[:, :, rig.plan.local_len(r, n) :] == sent).all(), (r, name)


def test_empty_cache_is_refused():
    model = _Model(32, 8, BF16)
    c = DuoSeqShardINT4KVCache(model, [[1.0] * 4 + [0.0] * 4], 1, 256, SINK, RECENT,
                               seq=tp.SeqShardContext(0, 2, 16, LocalSeqComm(2)))
    qkv = torch.zeros(1, 1, 48 * D, dtype=BF16, device=DEV)
    with pytest.raises(ValueError, match="is empty"):
        c.attend(0, qkv, None, None, NONE, torch.empty(1, 1, 32, D, dtype=BF16, device=DEV))
    assert c.launch_count == 0


def test_graph_replay_of_the_fused_step():
    """One captured q_len = 1 step of all W ranks (per-rank duo_decode_fused_seq_int4, the merge, advance_device)
    replayed while ownership changes hands many times, with an evict_last + sync in the middle: parity with fp64 after
    every replay, and at the end cache bytes bit-exact with an eager twin fed the same tokens."""
    W, block, Hq, Hkv, nf, B, dtype, rope = 3, 4, 32, 8, 4, 2, BF16, HF
    n0, T = 7000, 3 * block * W + 6
    rig = Rig(W, block, Hq, Hkv, nf, B, dtype, n0 + T + 8)
    g = torch.Generator(device=DEV).manual_seed(9)
    rig.prefill(n0, g)
    eager = rig.ranks
    graphed = rig.make_ranks(n0 + T + 8)
    eager_comm, graph_comm = eager[0].seq.comm, rig.comm
    rig.scatter(eager)
    high_e = list(rig.high)
    rig.scatter(graphed)
    rig.ranks = graphed

    qkv_s = [torch.zeros(B, 1, rig.width, dtype=dtype, device=DEV) for _ in range(W)]
    out_s = [torch.zeros(B, 1, Hq, D, dtype=dtype, device=DEV) for _ in range(W)]
    cos_s, sin_s = (torch.zeros(1, D, dtype=dtype, device=DEV) for _ in range(2))
    for c in graphed:
        c.enable_device_state()
        c.graph_attached = True
    # the capture freezes each slice's split count: with > 2048 keys per slice (>= 1024 keys per split) it is > 1
    assert min(rig.plan.local_len(r, n0) for r in range(W)) >= 2 * 1024
    snap = [(list(c.kv_seq_len_list), list(c.total_list), list(c.lo_list)) for c in graphed]
    rings = [c.snapshot_ring() for c in graphed]

    def restore():
        for c, s, ring in zip(graphed, snap, rings):
            c.kv_seq_len_list[:], c.total_list[:], c.lo_list[:] = (list(x) for x in s)
            c.restore_ring(ring)
            c.sync_device_state()

    for r, c in enumerate(graphed):  # warm-up (kernel attributes) outside the capture, then undo it
        c.attend(0, qkv_s[r], cos_s, sin_s, rope, out_s[r])
    restore()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for r, c in enumerate(graphed):
            c.attend(0, qkv_s[r], cos_s, sin_s, rope, out_s[r])
        for c in graphed:
            c.advance_device(1)
    restore()

    for i in range(T):
        if i == T // 2:
            for c in graphed + eager:
                c.evict_last(2)  # (refreshes the device copy of the graphed ranks)
        n = graphed[0].kv_seq_len
        qkv = rig.inputs(1, g)
        cos, sin = rope_tables(rope, n, 1, dtype)
        for r in range(W):
            qkv_s[r].copy_(qkv)
        cos_s.copy_(cos)
        sin_s.copy_(sin)
        graph.replay()
        for c in graphed:
            c.advance_host(1)
        oe = [torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV) for _ in range(W)]
        for r, c in enumerate(eager):
            c.attend(0, qkv.clone(), cos, sin, rope, oe[r])
        torch.cuda.synchronize()
        what = f"replay {i} (n={n})"
        for r in range(W):
            assert torch.equal(out_s[r], out_s[0]), f"{what}: rank {r}"
        q = host_rope_q(qkv[..., : Hq * D].view(B, 1, Hq, D), rope, cos, sin)
        truth, _ = rig.truth(q, n, 1, None)
        assert_parity(out_s[0][:, :, : rig.nfq], truth, f"{what}: replayed merged rows vs fp64")
        assert_parity(oe[0][:, :, : rig.nfq], truth, f"{what}: eager merged rows vs fp64")
        assert torch.equal(out_s[0][:, :, rig.nfq :], oe[0][:, :, rig.nfq :]), f"{what}: streaming rows"
        rig.check_partials(q, n, 1, what)
    assert graph_comm.calls == 1 + 1 and eager_comm.calls == T  # warm-up + capture; eager steps
    assert [c.kv_seq_len for c in graphed] == [c.kv_seq_len for c in eager] == [n0 + T - 2] * W
    rig.high = [max(a, b) for a, b in zip(rig.high, high_e)]
    rig.check_cache("end of replay", ranks=graphed, ref=eager)


def test_full_size_properties_at_1m_tokens():
    """1,048,576 tokens at world 4 (262,144 keys per slice; sink 64 / recent 256), one fused step of every rank and the
    merge: (1) every V row dequantises to the same vector c -> output == c; (2) q == 0 -> output == the mean of all
    visible V rows; (3) one key with an overwhelming logit -> output == that key's V row, with the key on a non-zero
    rank at the start of its slice, at a split boundary of its slice, and as the last cached key."""
    N, W, block, Hq, Hkv, nf, sink, recent, dtype = 1 << 20, 4, 1024, 32, 8, 4, 64, 256, FP16
    plan = SeqShardPlan(W, block)
    comm = LocalSeqComm(W)
    model = _Model(Hq, Hkv, dtype)
    gates = [[1.0] * nf + [0.0] * (Hkv - nf)]
    ranks = [DuoSeqShardINT4KVCache(model, gates, 1, N + 8, sink, recent, seq=tp.SeqShardContext(r, W, block, comm))
             for r in range(W)]
    g = torch.Generator(device=DEV).manual_seed(2)
    for rc in ranks:  # each rank its own slice; the streaming rings are replicated
        fill_random(rc.tensors[0], ("full_k", "full_v", "ring_k", "ring_v"), g)
        for name, x in rc.tensors[0].items():
            if name.startswith("ring"):
                x.copy_(ranks[0].tensors[0][name])
    loc = [plan.local_len(r, N) for r in range(W)]
    assert loc == [N // W] * W
    G = Hq // Hkv
    qkv0 = (torch.randn(1, 1, (Hq + 2 * Hkv) * D, generator=g, device=DEV) * 0.5).to(dtype)

    def decode(qkv):
        outs = []
        for rc in ranks:
            rc.kv_seq_len_list[0], rc.total_list[0], rc.lo_list[0] = N, N, N - recent
            o = torch.empty(1, 1, Hq, D, dtype=dtype, device=DEV)
            rc.attend(0, qkv.clone(), None, None, NONE, o)
            outs.append(o)
        torch.cuda.synchronize()
        for o in outs:
            assert torch.equal(o, outs[0])
        return outs[0][0, 0, : nf * G].float()

    def v_rows(rc, kvh, rows):
        t = rc.tensors[0]
        return dequant(t["full_v"][0, kvh, rows], t["full_v_scale"][0, kvh, rows], t["full_v_zero"][0, kvh, rows])

    # (1) constant V: codes d % 16, scale 0.125, zero -1 on every row; the new token's V quantises to c exactly
    codes = (torch.arange(D, device=DEV) % 16).to(torch.uint8)
    c = codes.float() * 0.125 - 1.0
    for rc in ranks:
        for n_ in ("full_v", "ring_v"):
            rc.tensors[0][n_][:] = (codes[0::2] << 4) | codes[1::2]
            rc.tensors[0][n_ + "_scale"].fill_(0.125)
            rc.tensors[0][n_ + "_zero"].fill_(-1.0)
    q1 = qkv0.clone()
    q1[..., (Hq + Hkv) * D :] = c.to(dtype).repeat(Hkv)
    o = decode(q1)
    torch.testing.assert_close(o, c.expand_as(o), rtol=1e-2, atol=1e-3)

    # (2) q == 0: uniform attention over the N cached rows and the new one (written by rank plan.owner(N))
    for rc in ranks:
        fill_random(rc.tensors[0], ("full_v",), g)
    q2 = qkv0.clone()
    q2[..., : Hq * D] = 0
    sums = torch.zeros(nf, D, dtype=torch.float64, device=DEV)
    for r, rc in enumerate(ranks):
        for kvh in range(nf):
            sums[kvh] += v_rows(rc, kvh, slice(0, loc[r])).sum(0)
    o = decode(q2)
    own = ranks[plan.owner(N)]
    new_row = plan.local_len(plan.owner(N), N)
    for kvh in range(nf):
        mean = (sums[kvh] + v_rows(own, kvh, slice(new_row, new_row + 1))[0]) / (N + 1)
        for j in range(G):
            torch.testing.assert_close(o[kvh * G + j], mean.float(), rtol=1e-2, atol=1e-3)

    # (3) one overwhelming key of kv head 1 on a non-zero rank
    kvh = 1
    qrow = qkv0[0, 0, kvh * G * D : (kvh * G + 1) * D].float()
    big = (qrow / qrow.norm() * 40.0).to(dtype)
    kp = torch.empty(1, 64, dtype=torch.uint8, device=DEV)
    ks = torch.empty(1, dtype=torch.float16, device=DEV)
    kz = torch.empty(1, dtype=torch.float16, device=DEV)
    _C.check(ranks[0].lib.duo_quant_int4(big.data_ptr(), D, 1, kp.data_ptr(), ks.data_ptr(), kz.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream))
    q3 = qkv0.clone()
    q3[0, 0, kvh * G * D : (kvh * G + 1) * D] = big
    # the split plan of a slice: 128-key tiles, >= 1024 keys per split, about 4 CTAs per SM
    # (rank 1 does not own position N: its key range is its loc[1] cached rows)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    splits = min(max(1, 4 * sms - (Hkv - nf)) // nf, -(-loc[1] // 1024), 512)
    kps = -(-(-(-loc[1] // splits)) // 128) * 128
    assert 1024 <= kps < loc[1]
    for pos in [block, plan.positions(1, N)[kps].item(), N - 1]:
        r = plan.owner(pos)
        assert r != 0
        row = plan.local_len(r, pos)
        t = ranks[r].tensors[0]
        saved = [t["full_k" + s][0, kvh, row].clone() for s in SFX]
        t["full_k"][0, kvh, row], t["full_k_scale"][0, kvh, row], t["full_k_zero"][0, kvh, row] = kp[0], ks[0], kz[0]
        want = v_rows(ranks[r], kvh, slice(row, row + 1))[0].float()
        o = decode(q3)[kvh * G]
        torch.testing.assert_close(o, want, rtol=1e-2, atol=2e-3)
        for s, x in zip(SFX, saved):
            t["full_k" + s][0, kvh, row] = x
