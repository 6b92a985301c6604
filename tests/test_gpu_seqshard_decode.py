"""Sequence-sharded decode on one GPU: W ranks of DuoSeqShardKVCache emulated on one device.

Every rank is a real DuoSeqShardKVCache (its host logic runs: the fused / unfused choice, the part_o views, the
capacity check), fed its own clone of the same qkv; a local stand-in for tp.SeqComm merges the W partials in rank
order with duo_merge_partials, the algebra and order of duo_seq_merge, so the merged output is what W GPUs would
compute (only the peer-memory exchange is left out: tests/multi_gpu/seqshard_check.py; tests/test_gpu_comm_emulated.py
runs duo_seq_merge itself for emulated ranks and holds the two kernels bit-identical).  The state is an unsharded
DuoKVCache (the control) scattered the way load_from_head_parallel does.  After every step:

* cache bytes: every rank's slice equals the control's rows at plan.positions, bit for bit; the rows past the slice
  still hold a finite sentinel (a huge logit if it were ever attended); the rings equal the control's;
* streaming-head rows of `out` are bit-identical to the control's (same kernel family, replicated heads);
* retrieval-head rows of the merged `out` are within parity of fp64 attention over the cache contents (and of the
  oracle for RoPE-free cases);
* per-rank partials: part_lse within 1e-3 of the fp64 log2-domain log-sum-exp over exactly the keys the token may see
  on that rank, part_o within parity of the fp64 slice output, -inf / 0 for rows that see no key on the rank.
"""
import ctypes as C
import types

import pytest
import torch

from duo_attention_b200 import _C, tp
from duo_attention_b200.kv_cache import DuoKVCache, DuoSeqShardKVCache, ring_live_positions, ring_slot
from duo_attention_b200.seqshard import SeqShardPlan
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
SENTINEL = 64.0
LOG2E = 1.4426950408889634
SINK, RECENT = 8, 24
ORACLE_MAX_KEYS = 8192  # the CPU oracle runs up to this context; fp64 truth runs everywhere


class LocalSeqComm:
    """tp.SeqComm's merge() for W ranks stepped in order 0..W-1 on one device: each rank registers (part_o, part_lse,
    out); the last rank's call stacks the W partials in rank order and merges them into every rank's `out`.  Works
    eagerly and inside a CUDA-graph capture."""

    max_rows = 1 << 20

    def __init__(self, world):
        self.world, self.pending, self.calls, self.keep = world, [], 0, None

    def merge(self, part_o, part_lse, out, tokens, heads_total, heads_used):
        self.pending.append((part_o, part_lse, out))
        if len(self.pending) < self.world:
            return
        parts, self.pending = self.pending, []
        po = torch.stack([p[0] for p in parts]).contiguous()
        pl = torch.stack([p[1] for p in parts]).contiguous()
        self.keep = (po, pl)  # a captured graph keeps reading these
        dt = _C.DT_BF16 if out.dtype == torch.bfloat16 else _C.DT_FP16
        stream = torch.cuda.current_stream(out.device).cuda_stream
        for _, _, o in parts:
            _C.check(_C.load().duo_merge_partials(po.data_ptr(), pl.data_ptr(), self.world, tokens, heads_total,
                                                  heads_used, o.data_ptr(), dt, stream))
        self.calls += 1


class _Model(torch.nn.Module):
    """What DuoSeqShardKVCache reads from a model: one parameter (dtype, device) and the config."""

    def __init__(self, Hq, Hkv, dtype):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, dtype=dtype, device=DEV), requires_grad=False)
        self.config = types.SimpleNamespace(num_hidden_layers=1, num_attention_heads=Hq, num_key_value_heads=Hkv,
                                            head_dim=D, hidden_size=Hq * D)


def set_local_capacity(c, cap):
    """Re-allocate a cache's retrieval rows to exactly `cap` (DuoSeqShardKVCache keeps one spare row)."""
    c._set_layer(0, cap, c.stage_cap_list[0])


def partials(c, S):
    """The part_o / part_lse views the kernels wrote for a chunk of S tokens (DuoSeqShardKVCache.attend)."""
    B, H = c.batch_size, c.num_heads
    if S == c.max_q:
        return c.part_o, c.part_lse
    return c.part_o.view(-1)[: B * S * H * D].view(B, S, H, D), c.part_lse.view(-1)[: B * S * H].view(B, S, H)


def rope_tables(rope, n, S, dtype):
    """Tables of positions n..n+S-1 ([S][128]: the kernels' layout), fp32 for ROPE_FP32."""
    if rope == _C.ROPE_NONE:
        return None, None
    pos = torch.arange(n, n + S)[None]
    cos, sin = O.hf_cos_sin(pos, D, 10000.0, torch.float32 if rope == _C.ROPE_FP32 else dtype)
    return cos[0].to(DEV).contiguous(), sin[0].to(DEV).contiguous()


def host_rope_q(q, rope, cos, sin):
    """q [B,S,H,D] rotated on the host with the kernels' arithmetic (HF: torch's ops, bit-exact; FP32: fma(rot, s, x c))."""
    if rope == _C.ROPE_NONE:
        return q
    B = q.shape[0]
    if rope == _C.ROPE_HF:
        c, s = cos[None].expand(B, -1, -1), sin[None].expand(B, -1, -1)
        return O.apply_rotary_pos_emb_hf(q, q, c, s, unsqueeze_dim=2)[0]
    x = q.float()
    xc = x * cos[None, :, None]  # rounded to fp32; then rot * s + xc with one rounding (exact in fp64, rounded once)
    return (O.rotate_half(x).double() * sin[None, :, None].double() + xc.double()).float().to(q.dtype)


def attn64(q, k, v, vis, scale):
    """fp64 attention.  q [B,S,nf,G,D], k/v [B,nf,N,D], vis [S,N] -> (O [B,S,nf,G,D], natural-log lse [B,S,nf,G]);
    rows that see no key get O = 0, lse = -inf."""
    s = torch.einsum("bsngd,bnjd->bsngj", q, k) * scale
    s = s.masked_fill(~vis[None, :, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    return torch.einsum("bsngj,bnjd->bsngd", p, v), lse


class Rig:
    """W sequence-shard rank caches and the unsharded control of the same geometry."""

    def __init__(self, W, block, Hq, Hkv, n_full, B, dtype, max_size):
        self.W, self.block, self.Hq, self.Hkv, self.nf, self.B, self.dtype = W, block, Hq, Hkv, n_full, B, dtype
        self.G = Hq // Hkv
        self.nfq = n_full * self.G
        self.plan = SeqShardPlan(W, block)
        self.control = DuoKVCache(1, Hq, Hkv, D, [n_full], B, max_size, SINK, RECENT, dtype, DEV, stage_cap=16)
        self.ranks = self.make_ranks(max_size)
        self.width = (Hq + 2 * Hkv) * D

    def make_ranks(self, max_size):
        self.comm = LocalSeqComm(self.W)
        model = _Model(self.Hq, self.Hkv, self.dtype)
        gates = [[1.0] * self.nf + [0.0] * (self.Hkv - self.nf)]
        ranks = [DuoSeqShardKVCache(model, gates, self.B, max_size, SINK, RECENT,
                                    seq=tp.SeqShardContext(r, self.W, self.block, self.comm)) for r in range(self.W)]
        self.high = [0] * self.W  # rows of each slice ever written: the rows from there on hold the sentinel
        return ranks

    # ---- state set-up --------------------------------------------------------------------------------------------
    def prefill(self, n, g, kscale=1.0):
        c = self.control
        if n == 0:
            return
        if n <= 2048:
            x = torch.randn(self.B, n, self.width, generator=g, device=DEV)
            x[..., self.Hq * D : (self.Hq + self.Hkv) * D] *= kscale
            c.attend(0, x.to(self.dtype), None, None, _C.ROPE_NONE,
                     torch.empty(self.B, n, self.Hq, D, dtype=self.dtype, device=DEV))
            return
        for name, t in c.tensors[0].items():  # long contexts: random contents, lengths set directly
            t.normal_(generator=g)
            if name.endswith("_k"):
                t.mul_(kscale)
        c.kv_seq_len_list[0], c.total_list[0], c.lo_list[0] = n, n, max(SINK, n - RECENT)

    def scatter(self, ranks=None):
        """load_from_head_parallel without torch.distributed: rank r takes the control's rows at plan.positions(r, n)."""
        c, W_ = self.control, self.control.W
        n = c.kv_seq_len
        for r, rc in enumerate(ranks or self.ranks):
            t = rc.tensors[0]
            t["full_k"].fill_(SENTINEL)
            t["full_v"].fill_(SENTINEL)
            pos = self.plan.positions(r, n).to(DEV)
            for name in ("full_k", "full_v"):
                t[name][:, :, : len(pos)] = c.tensors[0][name][:, :, pos]
            for name in ("ring_k", "ring_v"):
                t[name][:, :, :W_] = c.tensors[0][name][:, :, :W_]
            rc.kv_seq_len_list[0], rc.total_list[0], rc.lo_list[0] = n, c.total_list[0], c.lo_list[0]
            rc.sync_device_state()
            self.high[r] = len(pos)

    def evict(self, k):
        for c in [self.control] + self.ranks:
            c.evict_last(k)

    # ---- one step --------------------------------------------------------------------------------------------------
    def inputs(self, S, g, qscale=1.0, kscale=1.0):
        x = torch.randn(self.B, S, self.width, generator=g, device=DEV)
        x[..., : self.Hq * D] *= qscale
        x[..., self.Hq * D : (self.Hq + self.Hkv) * D] *= kscale
        return x.to(self.dtype)

    def step(self, S, rope, g, qscale=1.0, kscale=1.0):
        c = self.control
        n = c.kv_seq_len
        qkv = self.inputs(S, g, qscale, kscale)
        cos, sin = rope_tables(rope, n, S, self.dtype)
        past = self.control_past() if rope == _C.ROPE_NONE and n + S <= ORACLE_MAX_KEYS else False
        oc = torch.full((self.B, S, self.Hq, D), float("nan"), dtype=self.dtype, device=DEV)
        c.attend(0, qkv.clone(), cos, sin, rope, oc, fused=(S == 1))  # the kernel family of the sharded step
        outs = []
        for rc in self.ranks:
            o = torch.full_like(oc, float("nan"))
            rc.attend(0, qkv.clone(), cos, sin, rope, o)
            outs.append(o)
        torch.cuda.synchronize()
        what = f"n={n} S={S}"
        self.check_cache(what)
        for r, o in enumerate(outs):
            assert torch.equal(o[:, :, self.nfq :], oc[:, :, self.nfq :]), f"{what}: rank {r} streaming rows"
            assert torch.equal(o, outs[0]), f"{what}: rank {r}'s merged output differs from rank 0's"
        q = host_rope_q(qkv[..., : self.Hq * D].view(self.B, S, self.Hq, D), rope, cos, sin)
        if self.nfq:
            truth, _ = self.truth(q, n, S, None)
            assert_parity(outs[0][:, :, : self.nfq], truth, f"{what}: merged retrieval rows vs fp64")
            assert_parity(oc[:, :, : self.nfq], truth, f"{what}: control (unfused={S > 1}) vs fp64")
            self.check_partials(q, n, S, what)
        if past is not False:
            k = qkv[..., self.Hq * D : (self.Hq + self.Hkv) * D].view(self.B, S, self.Hkv, D)
            v = qkv[..., (self.Hq + self.Hkv) * D :].view(self.B, S, self.Hkv, D)
            ref, _ = O.tuple_attention_core(q.cpu(), k.cpu(), v.cpu(), past, self.nf, self.G, SINK, RECENT)
            assert_parity(oc.cpu(), ref, f"{what}: control vs oracle")
            if self.nfq:
                assert_parity(outs[0][:, :, : self.nfq].cpu(), ref[:, :, : self.nfq], f"{what}: merged vs oracle")
        return outs[0]

    def control_past(self):
        """The control's contents in the oracle's tuple layout (None before the first token)."""
        c = self.control
        n, t = c.kv_seq_len, c.tensors[0]
        if n == 0 and c.total_list[0] == 0:
            return None
        slots = [ring_slot(p, SINK, RECENT) for p in ring_live_positions(c.total_list[0], c.lo_list[0], SINK)]
        fk, fv = t["full_k"][:, :, :n], t["full_v"][:, :, :n]
        sk, sv = t["ring_k"][:, :, slots], t["ring_v"][:, :, slots]
        return torch.cat([fk, fv], 0).cpu(), torch.cat([sk, sv], 0).cpu()

    # ---- checks ----------------------------------------------------------------------------------------------------
    def check_cache(self, what, ranks=None, ref=None):
        """Each rank's slice == the reference cache's rows at plan.positions (bit-exact), sentinel past the rows ever
        written, rings equal.  `ref` defaults to the control; with a rank list, it is that list's twin."""
        n = self.ranks[0].kv_seq_len if ranks is None else ranks[0].kv_seq_len
        W_ = self.control.W
        for r, rc in enumerate(ranks or self.ranks):
            t = rc.tensors[0]
            loc = self.plan.local_len(r, n)
            assert rc.kv_seq_len == n
            self.high[r] = max(self.high[r], loc)
            if ref is None:
                pos = self.plan.positions(r, n).to(DEV)
                want = {k: self.control.tensors[0][k][:, :, pos] for k in ("full_k", "full_v")}
            else:
                want = {k: ref[r].tensors[0][k][:, :, :loc] for k in ("full_k", "full_v")}
            for name in ("full_k", "full_v"):
                assert torch.equal(t[name][:, :, :loc], want[name]), f"{what}: rank {r} {name} slice"
                assert (t[name][:, :, self.high[r] :] == SENTINEL).all(), f"{what}: rank {r} {name} written past its slice"
            src = self.control if ref is None else ref[r]
            for name in ("ring_k", "ring_v"):
                assert torch.equal(t[name][:, :, :W_], src.tensors[0][name][:, :, :W_]), f"{what}: rank {r} {name}"

    def gathered(self, n, ranks=None):
        """[B, nf, n, D] K and V of positions [0, n), put together from the rank slices."""
        k = torch.empty(self.B, self.nf, n, D, dtype=torch.float64, device=DEV)
        v = torch.empty_like(k)
        for r, rc in enumerate(ranks or self.ranks):
            pos = self.plan.positions(r, n).to(DEV)
            k[:, :, pos] = rc.tensors[0]["full_k"][:, :, : len(pos)].double()
            v[:, :, pos] = rc.tensors[0]["full_v"][:, :, : len(pos)].double()
        return k, v

    def truth(self, q, n, S, rank, ranks=None):
        """fp64 attention of the chunk's retrieval rows over all positions (rank None) or over `rank`'s slice."""
        qq = q.double().view(self.B, S, self.Hkv, self.G, D)[:, :, : self.nf]
        tok = torch.arange(n, n + S, device=DEV)[:, None]
        if rank is None:
            k, v = self.gathered(n + S, ranks)
            pos = torch.arange(n + S, device=DEV)
        else:
            pos = self.plan.positions(rank, n + S).to(DEV)
            t = (ranks or self.ranks)[rank].tensors[0]
            k, v = t["full_k"][:, :, : len(pos)].double(), t["full_v"][:, :, : len(pos)].double()
        o, lse = attn64(qq, k, v, pos[None, :] <= tok, D ** -0.5)
        return o.reshape(self.B, S, self.nfq, D), lse.reshape(self.B, S, self.nfq)

    def check_partials(self, q, n, S, what, ranks=None):
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
                assert err <= 1e-3, f"{what}: rank {r} part_lse off by {err}"
                assert_parity(po[~empty], o64[~empty], f"{what}: rank {r} part_o vs fp64")


BF16, FP16 = torch.bfloat16, torch.float16
NONE, HF, FP32 = _C.ROPE_NONE, _C.ROPE_HF, _C.ROPE_FP32
# id: (W, block, Hq, Hkv, n_full, B, dtype, rope, context, schedule, qscale, kscale); "e<k>" in a schedule = evict_last(k)
CASES = {
    # ranks 1.. start empty; a fused token and an unfused chunk each open rank 1's first block; a chunk crosses the
    # round boundary 32
    "w2b16_g4_from_empty": (2, 16, 32, 8, 4, 1, BF16, NONE, 0, [1, 2, 4, 4, 3, 1, 1, 2, 1, 4, 4, 4, 4, 1, 1], 1, 1),
    # group 8: the next token lands just before the block boundary 5; evict_last(1) takes back the token that opened
    # rank 1's first block, evict_last(2) goes back across the round boundary 15
    "w3b5_g8_fp16_hf_evict": (3, 5, 32, 4, 2, 2, FP16, HF, 4,
                              [1, 1, "e1", 1, 2, 2, 2, 2, 1, 1, "e2", 2, 1, 2], 1, 1),
    # round-robin ownership, MHA chunks of up to 16 tokens that touch every rank, no streaming heads
    "w4b1_mha_allfull_fp32": (4, 1, 8, 8, 8, 1, BF16, FP32, 3, [16, 5, 1, 1, 4, "e2", 3, 16], 1, 1),
    # no retrieval heads: nothing to merge
    "w8b64_nofull": (8, 64, 32, 8, 0, 2, BF16, NONE, 500, [1, 4, 1, 2], 1, 1),
    # the next token is the last of a round; then the first of the next round
    "w8b64_g4_fp16_hf_round": (8, 64, 32, 8, 3, 1, FP16, HF, 1023, [1, 1, 1, 4, "e2", 2, 1], 1, 1),
    # a block that does not divide the 64-key tile
    "w2b100_g4_round": (2, 100, 32, 8, 2, 2, BF16, NONE, 199, [1, 1, 3, 4, 1, "e1", 2], 1, 1),
    "w2b100_g4_fp16_fp32_block": (2, 100, 32, 8, 5, 1, FP16, FP32, 97, [2, 1, 4, 1, 3], 1, 1),
    # ~20K keys per slice: many split-KV CTAs per slice and the in-launch hierarchical merge
    "w2b1024_40k": (2, 1024, 32, 8, 4, 1, BF16, NONE, 40000, [1, 4, 1, 2, "e1", 1], 1, 1),
    # group 16: one token per step
    "w2b16_g16_hf": (2, 16, 32, 2, 1, 2, BF16, HF, 31, [1, 1, 1, 1, "e1", 1, 1], 1, 1),
    # sharp softmax (logit std 8): the largest logit sits on one rank
    "w4b16_sharp": (4, 16, 32, 8, 4, 2, BF16, NONE, 300, [1, 2, 1, 4, 1], 8, 1),
    # log-sum-exps far above 2^128 in the log2 domain: the cross-rank merge must rescale by the max before exp2
    "w3b16_huge_lse": (3, 16, 32, 8, 8, 1, BF16, NONE, 200, [1, 3, 1, 2], 8, 6),
}


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_sharded_decode_matches_fp64(case):
    W, block, Hq, Hkv, nf, B, dtype, rope, n0, sched, qscale, kscale = CASES[case]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    steps = sum(s for s in sched if isinstance(s, int))
    rig = Rig(W, block, Hq, Hkv, nf, B, dtype, n0 + steps + 8)
    rig.prefill(n0, g, kscale)
    rig.scatter()
    rig.check_cache("after the scatter")
    for s in sched:
        if isinstance(s, str):
            rig.evict(int(s[1:]))
        else:
            rig.step(s, rope, g, qscale, kscale)
    assert rig.comm.calls == (sum(isinstance(s, int) for s in sched) if nf else 0)


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_exact_local_capacity(dtype):
    """Every rank holds exactly plan.capacity(n + 1) rows: the step at n fills the owner's last row; at n + 1 (every
    rank at plan.capacity(n)) the owner refuses the next token — ValueError from the cache, DUO_EOVERFLOW from each C
    entry point — and the other ranks take the same step."""
    W, block, Hq, Hkv, nf, B = 3, 5, 32, 8, 4, 2
    n0 = 33  # positions 30..34 are rank 0's third block
    rig = Rig(W, block, Hq, Hkv, nf, B, dtype, n0 + 16)
    g = torch.Generator(device=DEV).manual_seed(5)
    cap = rig.plan.capacity(n0 + 1)
    assert rig.plan.local_len(0, n0 + 1) == cap and rig.plan.owner(n0) == 0
    for rc in rig.ranks:
        set_local_capacity(rc, cap)
    rig.prefill(n0, g)
    rig.scatter()
    rig.step(1, HF, g)
    n = n0 + 1
    assert all(rc.full_cap_list[0] == rig.plan.capacity(n) for rc in rig.ranks)
    owner = rig.plan.owner(n)
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
        "duo_decode_fused_seq": lib.duo_decode_fused_seq(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cos.data_ptr(),
                                                         sin.data_ptr(), HF, out.data_ptr(), po.data_ptr(), pl.data_ptr(),
                                                         D ** -0.5, ws.data_ptr(), ws.numel(), stream),
        "duo_rope_append": lib.duo_rope_append(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), cos.data_ptr(),
                                               sin.data_ptr(), HF, 1, stream),
        "duo_attention_seq": lib.duo_attention_seq(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out.data_ptr(),
                                                   po.data_ptr(), pl.data_ptr(), 1, D ** -0.5, ws.data_ptr(), ws.numel(),
                                                   stream),
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
        for name in ("full_k", "full_v"):
            assert (rc.tensors[0][name][:, :, rig.plan.local_len(r, n) :] == SENTINEL).all()


def test_graph_replay_of_the_fused_step():
    """One captured q_len = 1 step of all W ranks (per-rank duo_decode_fused_seq, the merge, advance_device) replayed
    while ownership changes hands many times, with an evict_last + sync in the middle: parity with fp64 after every
    replay, and at the end cache bytes bit-exact with an eager twin fed the same tokens."""
    W, block, Hq, Hkv, nf, B, dtype, rope = 3, 4, 32, 8, 4, 2, BF16, HF
    n0, T = 3200, 3 * block * W + 6
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
    # the capture freezes each slice's split count: with ~1000 keys per slice (>= 256 keys per split) it is > 1
    assert min(rig.plan.local_len(r, n0) for r in range(W)) >= 4 * 256
    # warm-up (kernel attributes) outside the capture, then undo it
    snap = [(list(c.kv_seq_len_list), list(c.total_list), list(c.lo_list)) for c in graphed]
    rings = [c.snapshot_ring() for c in graphed]

    def restore():
        for c, s, ring in zip(graphed, snap, rings):
            c.kv_seq_len_list[:], c.total_list[:], c.lo_list[:] = (list(x) for x in s)
            c.restore_ring(ring)
            c.sync_device_state()

    for r, c in enumerate(graphed):
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


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
def test_fused_and_unfused_decode_on_16bit_cache(dtype):
    """DuoKVCache.attend(fused=True) (one launch) against fused=False (RoPE/append, the 4-key-warp decode kernel, ring
    commit) on the same 16-bit cache state: the caches stay bit-identical and so do the streaming rows; the retrieval
    rows are not expected to (the fused kernel plans its splits over the cached keys and attends the new tokens as an
    extra tile, the unfused one tiles all of them), so both are held to fp64 and to the oracle."""
    Hq, Hkv, nf, B, rope = 32, 8, 3, 2, HF
    g = torch.Generator(device=DEV).manual_seed(17)
    width = (Hq + 2 * Hkv) * D
    fz, uf = (DuoKVCache(1, Hq, Hkv, D, [nf], B, 9000, SINK, RECENT, dtype, DEV, stage_cap=16) for _ in range(2))
    x = torch.randn(B, 700, width, generator=g, device=DEV).to(dtype)
    for c in (fz, uf):
        c.attend(0, x.clone(), None, None, _C.ROPE_NONE, torch.empty(B, 700, Hq, D, dtype=dtype, device=DEV))
    nfq, G = nf * (Hq // Hkv), Hq // Hkv
    for S, n_jump in [(1, 0), (2, 0), (4, 0), (1, 7000), (3, 0), (1, 0)]:
        if n_jump:  # a long context: many split-KV CTAs per head (contents beyond the prefill are random)
            for name in ("full_k", "full_v"):
                t = torch.randn(B, nf, n_jump, D, generator=g, device=DEV).to(dtype)
                for c in (fz, uf):
                    c.tensors[0][name][:, :, c.kv_seq_len : c.kv_seq_len + n_jump] = t
            for c in (fz, uf):
                c.kv_seq_len_list[0] += n_jump
        n = fz.kv_seq_len
        qkv = torch.randn(B, S, width, generator=g, device=DEV).to(dtype)
        cos, sin = rope_tables(rope, n, S, dtype)
        of, ou = (torch.full((B, S, Hq, D), float("nan"), dtype=dtype, device=DEV) for _ in range(2))
        fz.attend(0, qkv.clone(), cos, sin, rope, of, fused=True)
        uf.attend(0, qkv.clone(), cos, sin, rope, ou, fused=False)
        torch.cuda.synchronize()
        what = f"n={n} S={S}"
        for name in ("full_k", "full_v"):
            assert torch.equal(fz.tensors[0][name][:, :, : n + S], uf.tensors[0][name][:, :, : n + S]), f"{what}: {name}"
        for name in ("ring_k", "ring_v"):
            assert torch.equal(fz.tensors[0][name][:, :, : fz.W], uf.tensors[0][name][:, :, : fz.W]), f"{what}: {name}"
        assert torch.equal(of[:, :, nfq:], ou[:, :, nfq:]), f"{what}: streaming rows"
        q = host_rope_q(qkv[..., : Hq * D].view(B, S, Hq, D), rope, cos, sin).double().view(B, S, Hkv, G, D)[:, :, :nf]
        k, v = (fz.tensors[0][name][:, :, : n + S].double() for name in ("full_k", "full_v"))
        vis = torch.arange(n + S, device=DEV)[None, :] <= torch.arange(n, n + S, device=DEV)[:, None]
        truth = attn64(q, k, v, vis, D ** -0.5)[0].reshape(B, S, nfq, D)
        assert_parity(of[:, :, :nfq], truth, f"{what}: fused vs fp64")
        assert_parity(ou[:, :, :nfq], truth, f"{what}: unfused vs fp64")
        assert_parity(ou[:, :, :nfq], of[:, :, :nfq], f"{what}: unfused vs fused")
