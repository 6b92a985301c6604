"""Prefill-sized chunks on forks of a sequence-sharded prompt (DuoSeqShardForkKVCache, duo_prefill_seq_shared): W ranks
emulated on one device, with tests/test_gpu_seqshard_forks.py's ForkRig.

Every fork takes its own chunk (a different question per row) of one length S.  The control is a batch-B
DuoSeqShardKVCache whose rows each hold the whole prompt; both are fed the same tokens.  A rank's logical slice of a
fork is the donor's local rows [0, P / world) followed by the fork's own slice, which is exactly the control's slice,
and the two kernels of duo_prefill_seq_shared run duo_prefill_seq's tiles on it.  So after every chunk, per rank:

* bit identity with the control: the merged `out` (retrieval and streaming rows), the rank's (O, lse) partials, the
  own-slice bytes (against the control's local rows >= P / world) and the rings;
* accuracy: the merged retrieval rows pass both parity gates against fp64 attention over the whole context;
* visibility: the donor's rows past P / world and the own rows past the own length hold K = 0 and V = 1024 (ForkRig's
  poison); the output of every retrieval row and partial must stay within the largest visible |V| (a mass bound).

One-token steps between chunks take duo_decode_fused_seq_shared and are checked for bytes, streaming rows and parity
(with P = 0 for bit identity as well).  Cases cover a block of 8 or 16, where one 64- and one 128-key tile straddles
P / world and is loaded in 8-row pieces, and a block of 1024, where none does; sink + recent > 2048, which sends chunks
of >= 128 tokens to the mma.sync kernel; and own slices long enough that the mma.sync launch splits its keys.
"""
import pytest
import torch

import test_gpu_seqshard_forks as tf
from parity import assert_parity
from test_gpu_comm_emulated import capture_step, same_bits
from test_gpu_seqshard_decode import LocalSeqComm, host_rope_q, rope_tables
from test_gpu_seqshard_forks import BF16, FP16, FP32, HF, NONE, ForkRig, _same, _snapshot
from test_gpu_seqshard_prefill import attn64

pytestmark = pytest.mark.gpu
D = 128
DEV = tf.DEV


class LocalComm(LocalSeqComm):
    """LocalSeqComm for both exchanges: the merge of a prefill-sized chunk gives every row the stacked merge's bits."""

    merge_scattered = LocalSeqComm.merge


class ChunkRig(ForkRig):
    """ForkRig whose forks and control take chunks of any length through the rank-order merge."""

    def __init__(self, *args, **kw):
        super().__init__(*args, comm=LocalComm, **kw)
        self.ccomm.merge_scattered = self.ccomm.merge

    def call(self, g, rope, S):
        """One call of S tokens on every row of every rank (S = 1: a decode step), then every check."""
        n, B = self.control[0].kv_seq_len, self.B
        qkv = torch.randn(B, S, self.width, generator=g, device=DEV).to(self.dtype)
        cos, sin = rope_tables(rope, n, S, self.dtype)
        oc = [torch.full((B, S, self.Hq, D), float("nan"), dtype=self.dtype, device=DEV) for _ in range(self.W)]
        of = [torch.full_like(o, float("nan")) for o in oc]
        for r in range(self.W):
            self.control[r].attend(0, qkv.clone(), cos, sin, rope, oc[r])
        for r in range(self.W):
            self.forks[r].attend(0, qkv.clone(), cos, sin, rope, of[r])
        torch.cuda.synchronize()
        self.vmax = max(self.vmax, qkv[..., (self.Hq + self.Hkv) * D :].abs().max().item())
        what = f"n={n} S={S}"
        self.check_bytes(what)
        for r in range(self.W):
            assert torch.equal(of[r][:, :, self.nfq :], oc[r][:, :, self.nfq :]), f"{what}: rank {r} streaming rows"
            assert same_bits(of[r], of[0]), f"{what}: rank {r}'s merged output differs from rank 0's"
            if S > 1 or self.P == 0:  # chunks, and every call with nothing shared: the control's launches and bits
                assert same_bits(of[r], oc[r]), f"{what}: rank {r} merged output differs from the control"
                (fo, fl), (co, cl) = self.forks[r].partials(S), self.control[r].partials(S)
                assert same_bits(fo[:, :, : self.nfq], co[:, :, : self.nfq]), f"{what}: rank {r} part_o"
                assert same_bits(fl[:, :, : self.nfq], cl[:, :, : self.nfq]), f"{what}: rank {r} part_lse"
        if not self.nfq:
            return
        vmax = self.vmax * 1.01 + 1e-2  # a poisoned row would add ~1024 x its weight
        assert of[0][:, :, : self.nfq].abs().max().item() <= vmax, f"{what}: weight on a poisoned row"
        for f in self.forks:
            po = f.partials(S)[0][:, :, : self.nfq]
            assert po.abs().max().item() <= vmax, f"{what}: weight on a poisoned row in a partial"
        q = host_rope_q(qkv[..., : self.Hq * D].view(B, S, self.Hq, D), rope, cos, sin)
        qq = q.double().view(B, S, self.Hkv, self.G, D)[:, :, : self.nf]
        k = torch.empty(B, self.nf, n + S, D, dtype=torch.float64, device=DEV)
        v = torch.empty_like(k)
        for r, c in enumerate(self.control):  # the control's contents, which the byte checks tie to the forks'
            pos = self.plan.positions(r, n + S).to(DEV)
            k[:, :, pos] = c.tensors[0]["full_k"][:, :, : len(pos)].double()
            v[:, :, pos] = c.tensors[0]["full_v"][:, :, : len(pos)].double()
        vis = torch.arange(n + S, device=DEV)[None, :] <= n + torch.arange(S, device=DEV)[:, None]
        o64, _ = attn64(qq, k, v, vis, D ** -0.5)
        assert_parity(of[0][:, :, : self.nfq], o64.reshape(B, S, self.nfq, D), f"{what}: merged forks vs fp64")


# id: (W, block, G, n_full, B, dtype, rope, prompt n, schedule of call lengths, recent)
# c = P / W: 104, 80, 72 straddle a 64- and a 128-key tile (c % 64 != 0); 1024 straddles none; "on" prompts end on a
# round, so the first chunk starts an empty own slice; P = 0 prompts are shorter than one round
CASES = {
    "w2b8_g4_bf16_hf_straddle": (2, 8, 4, 4, 5, BF16, HF, 2 * 8 * 13 + 3, [5, 1, 100, 1, 128, 1], 24),
    "w3b16_g1_fp16_fp32_straddle": (3, 16, 1, 2, 4, FP16, FP32, 3 * 16 * 5 + 7, [1, 1, 17, 1, 700, 1], 24),
    "w8b8_g4_bf16_allfull": (8, 8, 4, 8, 3, BF16, NONE, 8 * 8 * 9 + 5, [128, 1, 5, 1], 24),
    "w8b16_g1_fp16_nofull": (8, 16, 1, 0, 3, FP16, HF, 8 * 16 * 3 + 1, [17, 1, 100, 1], 24),
    "w2b8_g1_bf16_fp32_on": (2, 8, 1, 2, 4, BF16, FP32, 2 * 2 * 8 * 5, [17, 1, 128, 1], 24),
    # own slices of ~1,000 local rows and more: the mma.sync launch splits its keys
    "w2b1024_g4_bf16_hf_split": (2, 1024, 4, 4, 2, BF16, HF, 2 * 1024 + 5, [100, 1, 4097, 1], 24),
    "w3b1024_g1_fp16_fp32_split": (3, 1024, 1, 4, 5, FP16, FP32, 3 * 1024 + 9, [17, 1, 700, 1], 24),
    # sink + recent > 2048: chunks of >= 128 tokens take the mma.sync kernel too
    "w2b16_g4_bf16_hf_window": (2, 16, 4, 4, 3, BF16, HF, 2 * 16 * 7 + 9, [128, 1, 300, 1], 2100),
    # P = 0: the chunks take DuoSeqShardKVCache's path
    "w3b16_g4_fp16_hf_below": (3, 16, 4, 4, 3, FP16, HF, 3 * 16 - 3, [5, 1, 128, 1], 24),
    "w2b1024_g1_bf16_none_below": (2, 1024, 1, 2, 4, BF16, NONE, 1500, [17, 1, 700, 1], 24),
}


@pytest.mark.parametrize("case", list(CASES), ids=list(CASES))
def test_fork_chunks_match_the_control(case, monkeypatch):
    W, block, G, nf, B, dtype, rope, n, sched, recent = CASES[case]
    monkeypatch.setattr(tf, "RECENT", recent)  # ForkRig's ring geometry
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    rig = ChunkRig(W, block, G, nf, B, dtype, n, sum(sched) + 8, g)
    assert rig.P == n // (W * block) * W * block
    c = rig.P // W
    if block < 64 and c:
        assert c % 64 != 0, "the case must put a tile across the donor's rows"
    for S in sched:
        rig.call(g, rope, S)
    assert rig.forks[0].kv_seq_len == n + sum(sched)


def test_refusals_leave_every_byte_unchanged():
    W, G, nf, B, dtype = 2, 4, 4, 3, BF16
    g = torch.Generator(device=DEV).manual_seed(11)
    rig = ChunkRig(W, 16, G, nf, B, dtype, 2 * 16 * 3 + 5, 40, g)
    odd = ChunkRig(W, 4, G, nf, B, dtype, 2 * 4 * 5 + 1, 200, g)  # block 4: P / W = 20 is not a multiple of 8
    caches = rig.donors + rig.forks + odd.donors + odd.forks

    def chunk(f, S):
        f.attend(0, torch.zeros(B, S, rig.width, dtype=dtype, device=DEV), None, None, NONE,
                 torch.zeros(B, S, rig.Hq, D, dtype=dtype, device=DEV))

    before = _snapshot(caches)
    for S in (2, 3, 4):  # decode-sized multi-token chunks
        with pytest.raises(ValueError, match="one token"):
            chunk(rig.forks[0], S)
    with pytest.raises(ValueError, match="Trying to put"):  # past the own capacity
        chunk(rig.forks[0], 100)
    with pytest.raises(ValueError, match="block 4"):
        chunk(odd.forks[0], 100)
    torch.cuda.synchronize()
    assert _same(before, _snapshot(caches))
    assert all(f.launch_count == 0 for f in rig.forks + odd.forks)
    # one-token steps on the block-4 forks are unaffected
    odd.call(g, NONE, 1)
    # with a DuoDecodeGraph attached, any chunk is refused
    capture_step(rig.forks, NONE, dtype, rig.width)
    torch.cuda.synchronize()
    before, counts = _snapshot(caches), [f.launch_count for f in rig.forks]
    with pytest.raises(ValueError, match="DuoDecodeGraph"):
        chunk(rig.forks[0], 20)
    torch.cuda.synchronize()
    assert _same(before, _snapshot(caches)) and counts == [f.launch_count for f in rig.forks]
