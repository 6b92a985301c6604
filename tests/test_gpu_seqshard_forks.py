"""Forks of a sequence-sharded prompt on one GPU (DuoSeqShardKVCache.fork, duo_decode_fused_seq_shared): W ranks
emulated on one device, as tests/test_gpu_seqshard_decode.py does.

The control is a batch-B DuoSeqShardKVCache whose rows each hold the whole prompt; the forks share the donor's first
P positions and own the rest.  Both are fed the same tokens.  After every step, per rank:

* bytes: the forks' own slices equal the control's local rows of the positions >= P, bit for bit; the rings are
  identical; the streaming-head rows of `out` are bit-identical (with P = 0, everything is);
* accuracy: the merged retrieval rows pass both parity gates against fp64 attention over the whole context, and each
  rank's partial (prefix slice and own slice together) is within parity of fp64 over that rank's positions;
* visibility: the donor's rows past P / world and the own rows past the own length hold K = 0 and V = 1024.  K = 0
  gives such a row the logit 0 on every query row, a weight comparable to a real key's whatever the sign of q, so any
  weight on it moves the output by ~1024 / n, far outside parity; and the output of every retrieval row and partial,
  a convex combination of the visible V, must stay within their largest magnitude (an explicit mass bound).
"""
import pytest
import torch

from duo_attention_b200 import _C, tp
from duo_attention_b200.kv_cache import DuoSeqShardForkKVCache, DuoSeqShardKVCache, fork_prefix_len
from duo_attention_b200.seqshard import SeqShardPlan
from parity import assert_parity
from test_gpu_comm_emulated import PeerSeqComm, capture_step, same_bits
from test_gpu_seqshard_decode import LocalSeqComm, _Model, attn64, host_rope_q, rope_tables

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
SINK, RECENT = 8, 24
POISON_V = 1024.0  # the V of a poisoned row (its K is 0)
LOG2E = 1.4426950408889634
BF16, FP16 = torch.bfloat16, torch.float16
NONE, HF, FP32 = _C.ROPE_NONE, _C.ROPE_HF, _C.ROPE_FP32


class ForkRig:
    """W donors (batch 1) and their forks, and W control ranks (batch B, the prompt copied into every row)."""

    def __init__(self, W, block, G, nf, B, dtype, n, new, g, comm=LocalSeqComm):
        self.W, self.block, self.G, self.nf, self.B, self.dtype, self.n = W, block, G, nf, B, dtype, n
        self.Hkv = 8 if G > 1 else 4
        self.Hq = self.Hkv * G
        self.nfq = nf * G
        self.width = (self.Hq + 2 * self.Hkv) * D
        self.plan = SeqShardPlan(W, block)
        self.P = fork_prefix_len(n, W, block)
        model = _Model(self.Hq, self.Hkv, dtype)
        gates = [[1.0] * nf + [0.0] * (self.Hkv - nf)]
        self.comm, self.ccomm = comm(W), LocalSeqComm(W)
        mk = lambda b, r, c: DuoSeqShardKVCache(model, gates, b, n + new, SINK, RECENT,
                                                seq=tp.SeqShardContext(r, W, block, c))
        self.donors = [mk(1, r, self.comm) for r in range(W)]
        self.control = [mk(B, r, self.ccomm) for r in range(W)]
        # the prompt: random K/V of every position and a random ring, scattered as load_from_head_parallel does
        kv = {k: torch.randn(1, nf, n, D, generator=g, device=DEV).to(dtype) for k in ("full_k", "full_v")}
        ring = {k: torch.randn(1, self.Hkv - nf, SINK + RECENT, D, generator=g, device=DEV).to(dtype)
                for k in ("ring_k", "ring_v")}
        for r in range(W):
            pos = self.plan.positions(r, n).to(DEV)
            for c in (self.donors[r], self.control[r]):
                t = c.tensors[0]
                for k in ("full_k", "full_v"):
                    t[k].fill_(0.0 if k == "full_k" else POISON_V)
                    t[k][:, :, : len(pos)] = kv[k][:, :, pos]
                for k in ("ring_k", "ring_v"):
                    if t[k].numel():
                        t[k][:, :, : SINK + RECENT] = ring[k]
                c.kv_seq_len_list[0], c.total_list[0], c.lo_list[0] = n, n, max(SINK, n - RECENT)
                c.sync_device_state()
        self.forks = [d.fork(B, new) for d in self.donors]
        # poison the donor's rows past the shared prefix (copied into the own slices above): the forks must never
        # read them; nor the own rows past the copied tail
        for d in self.donors:
            for k in ("full_k", "full_v"):
                d.tensors[0][k][:, :, self.P // W :] = 0.0 if k == "full_k" else POISON_V
        for f in self.forks:
            loc = self.plan.local_len(f.seq.rank, n - self.P)
            for k in ("full_k", "full_v"):
                f.tensors[0][k][:, :, loc:] = 0.0 if k == "full_k" else POISON_V
        self.vmax = kv["full_v"].abs().max().item() if nf else 0.0

    def inputs(self, g):
        return torch.randn(self.B, 1, self.width, generator=g, device=DEV).to(self.dtype)

    def step(self, g, rope):
        n = self.control[0].kv_seq_len
        qkv = self.inputs(g)
        cos, sin = rope_tables(rope, n, 1, self.dtype)
        oc = [torch.full((self.B, 1, self.Hq, D), float("nan"), dtype=self.dtype, device=DEV) for _ in range(self.W)]
        of = [torch.full_like(o, float("nan")) for o in oc]
        for r in range(self.W):
            self.control[r].attend(0, qkv.clone(), cos, sin, rope, oc[r])
        for r in range(self.W):
            self.forks[r].attend(0, qkv.clone(), cos, sin, rope, of[r])
        torch.cuda.synchronize()
        self.check(qkv, n, rope, cos, sin, oc, of)
        return of

    def check(self, qkv, n, rope, cos, sin, oc, of):
        what = f"n={n}"
        self.check_bytes(what)
        for r in range(self.W):
            assert torch.equal(of[r][:, :, self.nfq :], oc[r][:, :, self.nfq :]), f"{what}: rank {r} streaming rows"
            assert same_bits(of[r], of[0]), f"{what}: rank {r}'s merged output differs from rank 0's"
        if self.P == 0:
            for r in range(self.W):
                assert same_bits(of[r], oc[r]), f"{what}: P = 0: rank {r} differs from the control"
                po, pl = self.control[r].partials(1)
                assert same_bits(self.forks[r].part_o, po) and same_bits(self.forks[r].part_lse, pl)
        if not self.nfq:
            return
        q = host_rope_q(qkv[..., : self.Hq * D].view(self.B, 1, self.Hq, D), rope, cos, sin)
        qq = q.double().view(self.B, 1, self.Hkv, self.G, D)[:, :, : self.nf]
        tok = torch.tensor([[n]], device=DEV)
        # fp64 over the control's contents (which the byte checks tie to the forks')
        k = torch.empty(self.B, self.nf, n + 1, D, dtype=torch.float64, device=DEV)
        v = torch.empty_like(k)
        for r, c in enumerate(self.control):
            pos = self.plan.positions(r, n + 1).to(DEV)
            k[:, :, pos] = c.tensors[0]["full_k"][:, :, : len(pos)].double()
            v[:, :, pos] = c.tensors[0]["full_v"][:, :, : len(pos)].double()
        o64, _ = attn64(qq, k, v, torch.arange(n + 1, device=DEV)[None, :] <= tok, D ** -0.5)
        # mass bound: every visible V (prompt and new tokens) is below vmax; a poisoned row would add ~1024 x its weight
        vmax = max(self.vmax, qkv[..., (self.Hq + self.Hkv) * D :].abs().max().item()) * 1.01 + 1e-2
        assert of[0][:, :, : self.nfq].abs().max().item() <= vmax, f"{what}: weight on a poisoned row"
        for f in self.forks:
            assert f.part_o[:, :1, : self.nfq].abs().max().item() <= vmax, f"{what}: weight on a poisoned row"
        assert_parity(of[0][:, :, : self.nfq], o64.reshape(self.B, 1, self.nfq, D), f"{what}: merged forks vs fp64")
        for r, (c, f) in enumerate(zip(self.control, self.forks)):
            pos = self.plan.positions(r, n + 1).to(DEV)
            ko, vo = c.tensors[0]["full_k"][:, :, : len(pos)].double(), c.tensors[0]["full_v"][:, :, : len(pos)].double()
            o_r, lse = attn64(qq, ko, vo, pos[None, :] <= tok, D ** -0.5)
            o_r, lse2 = o_r.reshape(self.B, 1, self.nfq, D), (lse * LOG2E).reshape(self.B, 1, self.nfq)
            po, pl = f.part_o[:, :1, : self.nfq], f.part_lse[:, :1, : self.nfq]
            empty = torch.isneginf(lse2)
            assert torch.equal(torch.isneginf(pl), empty), f"{what}: rank {r} lse == -inf exactly where no key is seen"
            if (~empty).any():
                err = (pl[~empty].double() - lse2[~empty]).abs().max().item()
                assert err <= 1e-3, f"{what}: rank {r} combined lse off by {err}"
                assert_parity(po[~empty], o_r[~empty], f"{what}: rank {r} combined partial vs fp64")

    def check_bytes(self, what):
        n, P, W_ = self.forks[0].kv_seq_len, self.P, SINK + RECENT
        for r, (c, f) in enumerate(zip(self.control, self.forks)):
            assert c.kv_seq_len == f.kv_seq_len == n
            loc, own = self.plan.local_len(r, n), self.plan.local_len(r, n - P)
            assert loc == P // self.W + own
            for k in ("full_k", "full_v"):
                assert torch.equal(f.tensors[0][k][:, :, :own], c.tensors[0][k][:, :, P // self.W : loc]), \
                    f"{what}: rank {r} {k} own slice"
            for k in ("ring_k", "ring_v"):
                assert torch.equal(f.tensors[0][k][:, :, :W_], c.tensors[0][k][:, :, :W_]), f"{what}: rank {r} {k}"

    def evict(self, k):
        for c in self.control + self.forks:
            c.evict_last(k)


# id: (W, block, G, n_full, B, dtype, rope, prompt); prompt "on" = 2 rounds of W * block, "off" = 2 rounds + 7,
# "below" = one round - 3 (P = 0)
def _n(W, block, kind):
    return {"on": 2 * W * block, "off": 2 * W * block + 7, "below": W * block - 3, "long": 40 * W * block + 5,
            "split": 3 * W * block - 48}[kind]


CASES = {
    "w2b16_g4_b5_bf16_on": (2, 16, 4, 4, 5, BF16, NONE, "on"),
    "w2b16_g4_b17_fp16_off_hf": (2, 16, 4, 2, 17, FP16, HF, "off"),
    "w3b5_g1_b16_bf16_off_fp32": (3, 5, 1, 4, 16, BF16, FP32, "off"),
    "w3b5_g4_b2_fp16_below": (3, 5, 4, 3, 2, FP16, HF, "below"),
    "w8b4_g4_b1_bf16_off": (8, 4, 4, 1, 1, BF16, NONE, "off"),
    "w8b4_g1_b17_fp16_on": (8, 4, 1, 4, 17, FP16, NONE, "on"),
    "w8b4_g4_b16_bf16_nofull": (8, 4, 4, 0, 16, BF16, HF, "off"),
    "w2b64_g4_b16_bf16_long": (2, 64, 4, 8, 16, BF16, HF, "long"),
    "w3b16_g1_b5_fp16_allfull_below": (3, 16, 1, 4, 5, FP16, FP32, "below"),
    "w2b16_g4_b17_bf16_allfull_long": (2, 16, 4, 8, 17, BF16, NONE, "long"),
    # a tail of almost one round: the own slices hold 512 / 1024 local rows, so the suffix launch splits its keys and
    # folds the prefix partial in split_kv_finish
    "w2b512_g1_b17_fp16_split": (2, 512, 1, 4, 17, FP16, NONE, "split"),
    "w2b1024_g4_b5_bf16_split": (2, 1024, 4, 4, 5, BF16, HF, "split"),
}
SCHED = [1, 1, "e1", 1, 1, 1, "e2", 1, 1]


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_forks_match_the_control(case):
    W, block, G, nf, B, dtype, rope, kind = CASES[case]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    n = _n(W, block, kind)
    rig = ForkRig(W, block, G, nf, B, dtype, n, 16, g)
    assert rig.P == (0 if kind == "below" else (n // (W * block)) * W * block)
    rig.check_bytes("after fork")
    for s in SCHED:
        if isinstance(s, str):
            rig.evict(int(s[1:]))
        else:
            rig.step(g, rope)
    assert rig.forks[0].kv_seq_len == n + 4


def test_forks_through_duo_seq_merge():
    """The forks' partials through the real exchange (duo_seq_merge of emulated ranks) equal the duo_merge_partials
    path bit for bit."""
    W, block, G, nf, B, dtype, rope = 3, 8, 4, 4, 5, BF16, HF
    n = 5 * W * block + 11
    rigs = [ForkRig(W, block, G, nf, B, dtype, n, 8, torch.Generator(device=DEV).manual_seed(3), comm=c)
            for c in (LocalSeqComm, lambda w: PeerSeqComm(w, 128))]
    g = torch.Generator(device=DEV).manual_seed(4)
    for i in range(4):
        state = g.get_state()
        outs = []
        for rig in rigs:
            g.set_state(state)
            outs.append(rig.step(g, rope))
        for r in range(W):
            assert same_bits(outs[0][r], outs[1][r]), f"step {i}: rank {r} differs between the exchanges"
            assert same_bits(rigs[0].forks[r].part_o, rigs[1].forks[r].part_o)
            assert same_bits(rigs[0].forks[r].part_lse, rigs[1].forks[r].part_lse)
    assert rigs[1].comm.calls == 4


def test_graph_replay_of_the_forks():
    """One captured step of all ranks' forks, replayed over more than two ring wraps with evict_last(1) between
    steps, is bit-identical to eager steps on a twin set of forks."""
    W, block, G, nf, B, dtype, rope = 2, 16, 4, 4, 5, BF16, HF
    n = 3 * W * block + 9
    T = 3 * RECENT  # tokens committed to the ring: three wraps
    seed = torch.Generator(device=DEV).manual_seed(5)
    graph_rig = ForkRig(W, block, G, nf, B, dtype, n, T + 4, seed)
    eager_rig = ForkRig(W, block, G, nf, B, dtype, n, T + 4, torch.Generator(device=DEV).manual_seed(5))
    gr, qs, outs, cs, ss = capture_step(graph_rig.forks, rope, dtype, graph_rig.width)
    g = torch.Generator(device=DEV).manual_seed(6)
    for i in range(T):
        if i % 4 == 3:
            for f in graph_rig.forks + eager_rig.forks:
                f.evict_last(1)
        n_now = graph_rig.forks[0].kv_seq_len
        qkv = graph_rig.inputs(g)
        cos, sin = rope_tables(rope, n_now, 1, dtype)
        for q in qs:
            q.copy_(qkv)
        cs.copy_(cos)
        ss.copy_(sin)
        gr.replay()
        for f in graph_rig.forks:
            f.advance_host(1)
        eo = [torch.empty_like(outs[0]) for _ in range(W)]
        for r, f in enumerate(eager_rig.forks):
            f.attend(0, qkv.clone(), cos, sin, rope, eo[r])
        torch.cuda.synchronize()
        for r in range(W):
            assert same_bits(outs[r], eo[r]), f"replay {i}: rank {r} output"
            for k, x in graph_rig.forks[r].tensors[0].items():
                assert same_bits(x, eager_rig.forks[r].tensors[0][k]), f"replay {i}: rank {r} {k}"
        assert graph_rig.forks[0].kv_seq_len == eager_rig.forks[0].kv_seq_len
    assert graph_rig.forks[0].kv_seq_len == n + T - T // 4


def _snapshot(caches):
    return [([x.clone() for x in c.tensors[0].values()], list(c.kv_seq_len_list), list(c.total_list),
             list(c.lo_list)) for c in caches]


def _same(a, b):
    return all(all(same_bits(x, y) for x, y in zip(p[0], q[0])) and p[1:] == q[1:] for p, q in zip(a, b))


def test_refusals_leave_every_byte_unchanged():
    W, block, G, nf, B, dtype = 2, 16, 4, 4, 3, BF16
    n = 2 * W * block + 5
    rig = ForkRig(W, block, G, nf, B, dtype, n, 8, torch.Generator(device=DEV).manual_seed(7))
    d, f = rig.donors[0], rig.forks[0]
    qkv1 = torch.zeros(1, 1, rig.width, dtype=dtype, device=DEV)
    out1 = torch.zeros(1, 1, rig.Hq, D, dtype=dtype, device=DEV)
    qkv2 = torch.zeros(B, 2, rig.width, dtype=dtype, device=DEV)
    out2 = torch.zeros(B, 2, rig.Hq, D, dtype=dtype, device=DEV)
    before = _snapshot(rig.donors + rig.forks)
    with pytest.raises(ValueError, match="forks"):
        d.attend(0, qkv1, None, None, NONE, out1)
    with pytest.raises(ValueError, match="forks"):
        d.evict_last(1)
    with pytest.raises(ValueError, match="forks"):
        d.clear()
    with pytest.raises(ValueError, match="one token"):
        f.attend(0, qkv2, None, None, NONE, out2)
    with pytest.raises(ValueError, match="shared prefix"):
        f.evict_last(n - rig.P + 1)
    with pytest.raises(ValueError, match="forks of forks"):
        f.fork(2, 4)
    # forks have no unfused step: fused=False, force_mma and unaligned qkv rows are refused before any launch
    qkv = torch.zeros(B, 1, rig.width, dtype=dtype, device=DEV)
    out = torch.zeros(B, 1, rig.Hq, D, dtype=dtype, device=DEV)
    with pytest.raises(ValueError, match="one-launch"):
        f.attend(0, qkv, None, None, NONE, out, fused=False)
    with pytest.raises(ValueError, match="one-launch"):
        f.attend(0, qkv, None, None, NONE, out, force_mma=True)
    unaligned = torch.zeros(B, 1, rig.width + 8, dtype=dtype, device=DEV)[..., 1 : rig.width + 1]
    with pytest.raises(ValueError, match="aligned"):
        f.attend(0, unaligned, None, None, NONE, out)
    torch.cuda.synchronize()
    assert _same(before, _snapshot(rig.donors + rig.forks))
    assert f.launch_count == 0
    # captured in a graph, the forks refuse clear(): the graph reads the donor's prefix at a fixed P
    capture_step(rig.forks, NONE, dtype, rig.width)
    torch.cuda.synchronize()
    before = _snapshot(rig.donors + rig.forks)
    with pytest.raises(ValueError, match="DuoDecodeGraph"):
        f.clear()
    torch.cuda.synchronize()
    assert _same(before, _snapshot(rig.donors + rig.forks)) and f.prefix_len == rig.P and f.donor is d
    for x in rig.forks:
        x.graph_attached = False  # the graph is dropped
    # fork() refusals: INT4, batch > 1, empty, layers at different lengths
    model = _Model(rig.Hq, rig.Hkv, dtype)
    gates = [[1.0] * nf + [0.0] * (rig.Hkv - nf)]
    ctx = tp.SeqShardContext(0, W, block, LocalSeqComm(W))
    from duo_attention_b200.kv_cache import DuoSeqShardINT4KVCache
    i4 = DuoSeqShardINT4KVCache(model, gates, 1, 256, SINK, RECENT, seq=ctx)
    i4.kv_seq_len_list[0] = i4.total_list[0] = 100
    with pytest.raises(ValueError, match="INT4"):
        i4.fork(2, 4)
    with pytest.raises(ValueError, match="batch 1"):
        rig.control[0].fork(2, 4)
    empty = DuoSeqShardKVCache(model, gates, 1, 256, SINK, RECENT, seq=ctx)
    with pytest.raises(ValueError, match="empty"):
        empty.fork(2, 4)
    model2 = _Model(rig.Hq, rig.Hkv, dtype)
    model2.config.num_hidden_layers = 2
    two = DuoSeqShardKVCache(model2, gates * 2, 1, 256, SINK, RECENT, seq=ctx)
    two.kv_seq_len_list[:] = [40, 41]
    two.total_list[:] = [40, 41]
    with pytest.raises(ValueError, match="one length"):
        two.fork(2, 4)
    # clear() releases the donor
    for x in rig.forks:
        x.clear()
    d.evict_last(1)
    assert d.kv_seq_len == n - 1 and f.kv_seq_len == 0 and f.prefix_len == 0
