"""The peer-memory exchange kernels of comm.cu (duo_seq_merge, duo_allreduce_add_rmsnorm) on one GPU: W ranks emulated
on one device, each with its own receive buffer, flag words and call epochs, every kernel the real one.

The rig.  Rank r's buffer is allocated as tp._symmetric_buffer does it: data_bytes + flag_bytes, zeroed, the flags at
data + data_bytes, followed here by a guard tail filled with a canary.  Each rank has its own local_state (int32
[max_rows + 1]: per-row epochs, then the error word).  The W handles are built with data[q] / flags[q] = rank q's
buffer.  One call of the collective launches the kernels of ranks 0 .. W-1 in that order on one stream.  A kernel
waits until every sender's flag holds the current epoch, so before rank r runs, the rig stages what every sender
s > r would have pushed into rank r's buffer, at the layout the header and comm.cu document (independently of the
kernel): the payload rows, and the flag word [row * W + s] set to the epoch.  Senders s < r have pushed for real, so
the last rank reads nothing but real pushes and the first reads mostly staged rows: a staged layout that disagrees
with the kernel's makes the ranks' outputs differ.

  seq merge  : float [2 slots][W senders][max_rows][132]; floats 0..127 = part_o[tok][h], 128 = part_lse[tok][h],
               row = tok * heads_used + h
  all-reduce : T [2 slots][W senders][max_rows][hidden]
  both       : epoch = state[row] + 1, slot = epoch & 1

Eager calls stage the current slot only, so the other slot must still hold the previous call's payload (a parity
bug shows).  A captured collective stages with device ops captured ahead of each launch: the flag is state + 1
computed on the device, and the payload goes into both slots, because the parity changes with every replay.  After
every call the rig checks every rank's whole receive buffer against a mirror of what the pushes and the staging
wrote, the flags and state against the per-row call counts, the flag padding and the canary.

Safety rules, kept by every test here:
* ranks never run concurrently on several streams: nothing guarantees that W spinning grids are co-resident;
* in eager mode, before each launch, the host asserts that every flag word the kernel will wait on already holds its
  epoch, and does not launch if one does not;
* the bounded (~3 s) wait must never be reached: every call is followed by a check that every rank's error word is 0;
* no misaligned or out-of-range pointer is handed to a kernel (row counts stay within max_rows, buffers are whole
  torch allocations).
"""
import ctypes as C

import pytest
import torch

import test_gpu_seqshard_decode as S16
import test_gpu_seqshard_int4_decode as S4
from duo_attention_b200 import _C, tp
from parity import assert_parity

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
D = 128
SEQ_ROW = 132  # floats per pushed seq-merge row: 128 outputs, the log-sum-exp, padding
GUARD, CANARY = 4096, 0xA5
SENT = -3.5  # exact in bf16 and fp16
BF16, FP16 = torch.bfloat16, torch.float16
SINK, RECENT = S16.SINK, S16.RECENT


def dt_code(dtype):
    return _C.DT_BF16 if dtype == BF16 else _C.DT_FP16


def bits(x):
    return x.contiguous().view(torch.uint8)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def ulp(x, dtype):
    """Spacing of `dtype` at |x| (x fp64): 2^(floor(log2|x|) - mantissa bits), the subnormal spacing below the normal
    range."""
    p = {BF16: 7, FP16: 10}[dtype]
    _, e = torch.frexp(x.abs().clamp_min(torch.finfo(dtype).tiny))
    return torch.exp2((e - 1 - p).double())


def stream():
    return torch.cuda.current_stream(DEV).cuda_stream


class PeerRig:
    """W ranks' receive buffers, flags and epochs on one device; `run` is one call of the collective."""

    def __init__(self, W, max_rows, data_bytes, flag_bytes, elt, width):
        self.W, self.max_rows, self.db, self.fb = W, max_rows, data_bytes, flag_bytes
        assert data_bytes % 16 == 0 and flag_bytes % 256 == 0 and flag_bytes >= 4 * W * max_rows
        self.bufs = []
        for _ in range(W):
            b = torch.zeros(data_bytes + flag_bytes + GUARD, dtype=torch.uint8, device=DEV)
            b[data_bytes + flag_bytes :] = CANARY
            self.bufs.append(b)
        self.state = [torch.zeros(max_rows + 1, dtype=torch.int32, device=DEV) for _ in range(W)]
        self.data = [b[:data_bytes].view(elt).view(2, W, max_rows, width) for b in self.bufs]
        self.flags = [b[data_bytes : data_bytes + 4 * W * max_rows].view(torch.int32).view(max_rows, W)
                      for b in self.bufs]
        self.mirror = [torch.zeros(data_bytes, dtype=torch.uint8, device=DEV) for _ in range(W)]
        self.mirror_v = [m.view(elt).view(2, W, max_rows, width) for m in self.mirror]
        self.count = torch.zeros(max_rows, dtype=torch.int32)  # calls that touched each row (host)

    def fill_desc(self, d, r):
        for q in range(self.W):
            d.data[q] = self.bufs[q].data_ptr()
            d.flags[q] = self.bufs[q].data_ptr() + self.db
        d.local_state = self.state[r].data_ptr()
        d.rank, d.world, d.max_rows = r, self.W, self.max_rows

    def _slots(self, R):
        epoch = self.count[:R] + 1
        return epoch, (epoch & 1).to(DEV, torch.long), torch.arange(R, device=DEV)

    def run(self, R, payload, launch):
        """One collective over rows [0, R): `payload(s)` is sender s's [R, n] pushed rows, `launch(r)` calls rank r's
        C entry point.  Eagerly, or inside a CUDA-graph capture."""
        if R == 0:  # the entry points return before any launch
            for r in range(self.W):
                launch(r)
            return
        assert R <= self.max_rows
        if torch.cuda.is_current_stream_capturing():
            for r in range(self.W):
                for s in range(r + 1, self.W):
                    p = payload(s)
                    self.data[r][:, s, :R, : p.shape[1]] = p  # both slots: the parity changes with every replay
                    self.flags[r][:R, s].copy_(self.state[r][:R]).add_(1)
                launch(r)
            return
        epoch, slot, rows = self._slots(R)
        ep = epoch.to(DEV)
        for r in range(self.W):
            for s in range(r + 1, self.W):
                p = payload(s)
                self.data[r][:, s][slot, rows, : p.shape[1]] = p
                self.flags[r][:R, s] = ep
        for r in range(self.W):
            torch.cuda.synchronize()
            want = epoch[:, None].repeat(1, self.W)
            want[:, r] -= 1  # its own word: the kernel sets it
            got = self.flags[r][:R].cpu()
            if not torch.equal(got, want):
                raise AssertionError(f"rank {r} would wait on a flag that does not hold its epoch: not launched")
            launch(r)
        torch.cuda.synchronize()

    def record(self, R, payload, staged_both):
        """Book the call just made: the mirror of every receive buffer and the per-row call counts."""
        if R == 0:
            return
        _, slot, rows = self._slots(R)
        for r in range(self.W):
            for s in range(self.W):
                p = payload(s)
                self.mirror_v[r][:, s][slot, rows, : p.shape[1]] = p
                if staged_both and s > r:
                    self.mirror_v[r][:, s][1 - slot, rows, : p.shape[1]] = p
        self.count[:R] += 1

    def verify(self, what):
        torch.cuda.synchronize()
        cnt = self.count.to(DEV)
        nf = 4 * self.W * self.max_rows
        for r in range(self.W):
            st, b = self.state[r], self.bufs[r]
            assert st[self.max_rows].item() == 0, f"{what}: rank {r}'s error word is set (a wait timed out)"
            assert torch.equal(st[: self.max_rows], cnt), f"{what}: rank {r}'s epochs != per-row call counts"
            assert torch.equal(self.flags[r], cnt[:, None].expand(-1, self.W)), f"{what}: rank {r}'s flags"
            assert (b[self.db + nf : self.db + self.fb] == 0).all(), f"{what}: rank {r}'s flag padding written"
            assert (b[self.db + self.fb :] == CANARY).all(), f"{what}: rank {r}'s guard canary overwritten"
            assert torch.equal(b[: self.db], self.mirror[r]), f"{what}: rank {r}'s receive slots != the pushes"

    def states_agree(self):
        return all(torch.equal(s, self.state[0]) for s in self.state)


class SeqPeers(PeerRig):
    """duo_seq_merge handles of W emulated ranks."""

    def __init__(self, W, max_rows):
        lib = _C.load()
        super().__init__(W, max_rows, lib.duo_seqcomm_data_bytes(W, max_rows), lib.duo_seqcomm_flag_bytes(W, max_rows),
                         torch.float32, SEQ_ROW)
        self.handles = []
        for r in range(W):
            d = _C.SeqCommDesc()
            self.fill_desc(d, r)
            h = C.c_void_p()
            _C.check(lib.duo_seqcomm_create(C.byref(d), C.byref(h)))
            self.handles.append(h)

    def merge(self, po, pl, outs, tokens, heads_total, heads_used):
        """Rank r merges po[r] [tokens, heads_total, 128] / pl[r] [tokens, heads_total] into outs[r]; returns the payload
        function of the call."""
        lib, R, dt = _C.load(), tokens * heads_used, dt_code(outs[0].dtype)

        def payload(s):
            return torch.cat([po[s][..., :heads_used, :].reshape(R, D), pl[s][..., :heads_used].reshape(R, 1)], 1)

        def launch(r):
            _C.check(lib.duo_seq_merge(self.handles[r], po[r].data_ptr(), pl[r].data_ptr(), outs[r].data_ptr(), tokens,
                                       heads_total, heads_used, dt, stream()))

        self.run(R, payload, launch)
        return payload

    def __del__(self):
        for h in getattr(self, "handles", []):
            _C.load().duo_seqcomm_destroy(h)


class ArPeers(PeerRig):
    """duo_allreduce_add_rmsnorm handles of W emulated ranks."""

    def __init__(self, W, hidden, dtype, max_rows=64):
        lib, dt = _C.load(), dt_code(dtype)
        super().__init__(W, max_rows, lib.duo_comm_data_bytes(W, hidden, max_rows, dt),
                         lib.duo_comm_flag_bytes(W, max_rows), dtype, hidden)
        self.hidden, self.handles = hidden, []
        for r in range(W):
            d = _C.CommDesc()
            self.fill_desc(d, r)
            d.hidden, d.dtype = hidden, dt
            h = C.c_void_p()
            _C.check(lib.duo_comm_create(C.byref(d), C.byref(h)))
            self.handles.append(h)

    def allreduce(self, partials, residuals, weight, out_norm, out_res, rows, eps):
        lib = _C.load()

        def ptr(t):
            return None if t is None else t.data_ptr()

        def launch(r):
            _C.check(lib.duo_allreduce_add_rmsnorm(self.handles[r], partials[r].data_ptr(), ptr(residuals[r]),
                                                   weight.data_ptr(), out_norm[r].data_ptr(), ptr(out_res[r]), rows,
                                                   float(eps), stream()))

        def payload(s):
            return partials[s]

        self.run(rows, payload, launch)
        return payload

    def __del__(self):
        for h in getattr(self, "handles", []):
            _C.load().duo_comm_destroy(h)


# ---- duo_seq_merge ----------------------------------------------------------------------------------------------------
def seq_inputs(W, tokens, ht, pattern, g):
    """Per-rank fp32 partials [tokens, ht, 128] and log2-domain log-sum-exps [tokens, ht] of one lse pattern."""
    po = [torch.randn(tokens, ht, D, generator=g, device=DEV) for _ in range(W)]
    shape = (W, tokens, ht)
    if pattern == "finite":
        pl = torch.randn(shape, generator=g, device=DEV) * 4
    elif pattern == "some_ninf":  # rows where every rank is -inf occur too
        pl = torch.randn(shape, generator=g, device=DEV) * 4
        pl[torch.rand(shape, generator=g, device=DEV) < 0.4] = float("-inf")
    elif pattern == "all_ninf":
        pl = torch.full(shape, float("-inf"), device=DEV)
    elif pattern == "spread":  # +-200 apart: the far weights flush to 0
        pick = torch.randint(0, 3, shape, generator=g, device=DEV).float()
        pl = (pick - 1) * 200 + torch.randn(shape, generator=g, device=DEV) * 0.5
    elif pattern == "equal":
        pl = (torch.randn(tokens, ht, generator=g, device=DEV) * 4).expand(shape).clone()
    else:  # "huge": 2^lse overflows fp32 unless the merge rescales by the max first
        pl = 150 + torch.randn(shape, generator=g, device=DEV) * 3
    for o, l in zip(po, pl):  # a rank that saw no key adds nothing, whatever its o holds: skipped, not weighted by 0
        o[torch.isneginf(l)] = float("nan")
    return po, list(pl.unbind(0))


def check_seq_merge(po, pl, outs, tokens, ht, hu, what):
    """Ranks bit-identical; == duo_merge_partials on the stacked partials; fp64 merge within
    ulp_T(|ref|) + 2^-20 sum_s w_s |o_s| / sum_s w_s; rows of heads >= heads_used untouched."""
    W, dtype = len(po), outs[0].dtype
    for r in range(1, W):
        assert same_bits(outs[r], outs[0]), f"{what}: rank {r}'s output differs from rank 0's"
    assert (outs[0][:, hu:] == SENT).all(), f"{what}: rows of heads >= heads_used written"
    other = torch.full_like(outs[0], SENT)
    sp, sl = torch.stack(po), torch.stack(pl)  # held until the kernel has run
    _C.check(_C.load().duo_merge_partials(sp.data_ptr(), sl.data_ptr(), W, tokens, ht, hu, other.data_ptr(),
                                          dt_code(dtype), stream()))
    torch.cuda.synchronize()
    assert same_bits(outs[0], other), f"{what}: duo_seq_merge != duo_merge_partials on the same partials"
    if hu == 0:
        return
    lse = torch.stack(pl)[:, :, :hu].double()
    o = torch.stack(po)[:, :, :hu].double().masked_fill(torch.isneginf(lse)[..., None], 0.0)
    m = lse.max(0).values
    empty = torch.isneginf(m)
    w = torch.exp2(lse - m.masked_fill(empty, 0.0))
    ws = w.sum(0).clamp_min(1e-300)[..., None]
    ref = (w[..., None] * o).sum(0) / ws
    mag = (w[..., None] * o.abs()).sum(0) / ws
    got = outs[0][:, :hu].double()
    assert (got[empty] == 0).all(), f"{what}: rows that every rank saw no key of must be exactly 0"
    err, bound = (got - ref).abs(), ulp(ref, dtype) + 2.0 ** -20 * mag
    bad = (err > bound) & ~empty[..., None]
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off the fp64 merge, worst {(err / bound).max().item():.3g}x"


# (tokens, heads_total, heads_used, lse pattern): row counts vary, so the per-row epochs diverge
SEQ_CALLS = [
    (1, 32, 32, "finite"), (16, 32, 32, "finite"), (4, 32, 8, "some_ninf"), (3, 8, 1, "all_ninf"),
    (2, 16, 0, "finite"), (8, 40, 40, "spread"), (64, 8, 8, "equal"), (5, 3, 3, "huge"), (1, 1, 1, "some_ninf"),
    (128, 4, 4, "finite"), (7, 12, 5, "spread"), (2, 64, 64, "huge"), (16, 32, 32, "some_ninf"),
    (1, 32, 12, "all_ninf"), (9, 10, 7, "equal"), (512, 1, 1, "finite"), (3, 32, 32, "huge"), (11, 6, 2, "some_ninf"),
    (6, 16, 16, "spread"), (1, 8, 8, "finite"), (32, 16, 16, "some_ninf"), (2, 2, 1, "equal"), (4, 8, 8, "all_ninf"),
]
SEQ_MAX_ROWS = 512


def seq_call(peers, W, dtype, tokens, ht, hu, pattern, g, what):
    po, pl = seq_inputs(W, tokens, ht, pattern, g)
    outs = [torch.full((tokens, ht, D), SENT, dtype=dtype, device=DEV) for _ in range(W)]
    payload = peers.merge(po, pl, outs, tokens, ht, hu)
    peers.record(tokens * hu, payload, staged_both=False)
    peers.verify(what)
    check_seq_merge(po, pl, outs, tokens, ht, hu, what)


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("W", [2, 3, 4, 5, 8])
def test_seq_merge_matches_fp64_and_merge_partials(W, dtype):
    assert max(t * hu for t, _, hu, _ in SEQ_CALLS) == SEQ_MAX_ROWS
    peers = SeqPeers(W, SEQ_MAX_ROWS)
    g = torch.Generator(device=DEV).manual_seed(W)
    for i, (tokens, ht, hu, pattern) in enumerate(SEQ_CALLS):
        seq_call(peers, W, dtype, tokens, ht, hu, pattern, g, f"call {i} ({tokens}x{hu}/{ht}, {pattern})")
    assert len(set(peers.count.tolist())) > 3  # the per-row epochs diverged


@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("W", [2, 5, 8])
def test_seq_merge_graph_replay(W, dtype):
    """One captured collective replayed 12 times, new partials copied into the captured inputs between replays; the
    eager calls before the capture leave the rows at different epochs."""
    peers = SeqPeers(W, 64)
    g = torch.Generator(device=DEV).manual_seed(100 + W)
    for i, (tokens, ht, hu) in enumerate([(3, 8, 8), (1, 8, 5), (2, 8, 3)]):
        seq_call(peers, W, dtype, tokens, ht, hu, "finite", g, f"eager call {i}")
    tokens, ht, hu = 4, 8, 6
    po = [torch.zeros(tokens, ht, D, device=DEV) for _ in range(W)]
    pl = [torch.zeros(tokens, ht, device=DEV) for _ in range(W)]
    outs = [torch.full((tokens, ht, D), SENT, dtype=dtype, device=DEV) for _ in range(W)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        payload = peers.merge(po, pl, outs, tokens, ht, hu)
    patterns = ["finite", "some_ninf", "spread", "huge", "equal", "all_ninf"]
    for i in range(12):
        npo, npl = seq_inputs(W, tokens, ht, patterns[i % len(patterns)], g)
        for r in range(W):
            po[r].copy_(npo[r])
            pl[r].copy_(npl[r])
            outs[r].fill_(SENT)
        torch.cuda.synchronize()
        assert peers.states_agree()  # the captured flags are state + 1: the ranks must agree on the epochs
        graph.replay()
        peers.record(tokens * hu, payload, staged_both=True)
        what = f"replay {i} ({patterns[i % len(patterns)]})"
        peers.verify(what)
        check_seq_merge(po, pl, outs, tokens, ht, hu, what)


# ---- duo_allreduce_add_rmsnorm ------------------------------------------------------------------------------------------
# residual given or NULL x out_res aliasing the residual (as FusedAllReduce passes it), separate or NULL
AR_MODES = {"alias": (True, "alias"), "separate": (True, "separate"), "res_only": (True, None),
            "out_only": (False, "separate"), "neither": (False, None)}
# (rows, mode, eps, zero row)
AR_CALLS = [
    (1, "alias", 1e-5, False), (5, "separate", 1e-6, True), (16, "out_only", 1e-5, False), (64, "alias", 1e-5, True),
    (5, "res_only", 0.5, False), (1, "neither", 1e-5, False), (16, "alias", 1e-6, False), (64, "separate", 1e-2, False),
    (5, "out_only", 1e-5, True), (16, "res_only", 1e-5, False), (1, "separate", 0.5, False), (64, "neither", 1e-6, True),
    (5, "alias", 1e-5, False), (16, "separate", 1e-5, True),
]


def ar_weight(hidden, dtype, g):
    """+-2^k, k in {-1, 0, 1}: the product with the weight is exact, so the ulp bounds below are theorems (with a
    general weight the norm's rounding flip between two kernels can grow to 2 ulp in the product)."""
    sign = torch.randint(0, 2, (hidden,), generator=g, device=DEV) * 2 - 1
    return (sign * torch.exp2(torch.randint(-1, 2, (hidden,), generator=g, device=DEV).float())).to(dtype)


def ar_inputs(W, rows, hidden, dtype, zero, g):
    partials = [torch.randn(rows, hidden, generator=g, device=DEV).to(dtype) for _ in range(W)]
    residual = (torch.randn(rows, hidden, generator=g, device=DEV) * 2).to(dtype)
    if zero:
        for p in partials + [residual]:
            p[rows // 2] = 0
    return partials, residual


def check_allreduce(partials, res_before, weight, out_norm, out_res, rows, eps, what):
    """out_res bit-exact against the rank-order fp32 sum rounded to T (+ residual, rounded); out_norm within 2 ulp_T of
    weight * T(h * rsqrt(mean h^2 + eps)) in fp64 and within 1 ulp_T of duo_add_rmsnorm on the same sum; ranks
    bit-identical."""
    W, dtype, hidden = len(partials), weight.dtype, weight.numel()
    acc = torch.zeros(rows, hidden, dtype=torch.float32, device=DEV)
    for p in partials:  # rank order, fp32, one rounding per add
        acc = acc + p.float()
    a = acc.to(dtype)
    h = a if res_before is None else (res_before.float() + a.float()).to(dtype)
    for r in range(W):
        assert same_bits(out_norm[r], out_norm[0]), f"{what}: rank {r}'s out_norm differs from rank 0's"
        if out_res[r] is not None:
            assert same_bits(out_res[r], h), f"{what}: rank {r}'s out_res != T(T(sum_s p_s) + residual)"
    hd = h.double()
    n = (hd * torch.rsqrt(hd.square().mean(-1, keepdim=True) + eps)).to(dtype)
    ref = weight.double() * n.double()
    got = out_norm[0].double()
    err, bound = (got - ref).abs(), 2 * ulp(ref, dtype)
    assert (err <= bound).all(), f"{what}: out_norm off the fp64 RMSNorm by {(err / bound).max().item():.3g} x 2 ulp"
    o2, h2 = torch.empty_like(a), torch.empty_like(a)
    _C.check(_C.load().duo_add_rmsnorm(a.data_ptr(), None if res_before is None else res_before.data_ptr(),
                                       weight.data_ptr(), o2.data_ptr(), h2.data_ptr(), rows, hidden, float(eps),
                                       dt_code(dtype), stream()))
    torch.cuda.synchronize()
    if res_before is not None:
        assert same_bits(h2, h), f"{what}: duo_add_rmsnorm's residual stream differs"
    d = (got - o2.double()).abs()
    lim = ulp(torch.maximum(got.abs(), o2.double().abs()), dtype)
    assert (d <= lim).all(), f"{what}: out_norm vs duo_add_rmsnorm: {(d / lim).max().item():.3g} ulp"


def ar_call(peers, W, dtype, rows, mode, eps, zero, weight, g, what):
    hidden = peers.hidden
    partials, residual = ar_inputs(W, rows, hidden, dtype, zero, g)
    has_res, out_kind = AR_MODES[mode]
    residuals = [residual.clone() if has_res else None for _ in range(W)]
    out_norm = [torch.full((rows, hidden), SENT, dtype=dtype, device=DEV) for _ in range(W)]
    out_res = [residuals[r] if out_kind == "alias" else
               torch.full((rows, hidden), SENT, dtype=dtype, device=DEV) if out_kind == "separate" else None
               for r in range(W)]
    payload = peers.allreduce(partials, residuals, weight, out_norm, out_res, rows, eps)
    peers.record(rows, payload, staged_both=False)
    peers.verify(what)
    if has_res and out_kind != "alias":
        for r in range(W):
            assert same_bits(residuals[r], residual), f"{what}: rank {r}'s residual written"
    check_allreduce(partials, residual if has_res else None, weight, out_norm, out_res, rows, eps, what)


AR_HIDDEN = [8, 520, 4096, 8192, 12288, 12296, 16384]  # 12296: the first size over 48 KB of shared memory


@pytest.mark.parametrize("hidden", AR_HIDDEN)
@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("W", [2, 4, 8])
def test_allreduce_add_rmsnorm_matches_host_sum_and_fp64(W, dtype, hidden):
    peers = ArPeers(W, hidden, dtype)
    g = torch.Generator(device=DEV).manual_seed(W * 100003 + hidden)
    weight = ar_weight(hidden, dtype, g)
    for i, (rows, mode, eps, zero) in enumerate(AR_CALLS):
        ar_call(peers, W, dtype, rows, mode, eps, zero, weight, g, f"call {i} ({rows} rows, {mode}, eps {eps})")
    assert len(set(peers.count.tolist())) > 2  # the per-row epochs diverged


@pytest.mark.parametrize("hidden", [520, 16384])
@pytest.mark.parametrize("dtype", [BF16, FP16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("W", [2, 4, 8])
def test_allreduce_graph_replay(W, dtype, hidden):
    """FusedAllReduce's use: the residual updated in place, one captured collective of 16 rows replayed 10 times with
    new partials and residuals copied into the captured inputs."""
    peers = ArPeers(W, hidden, dtype)
    g = torch.Generator(device=DEV).manual_seed(7 * W + hidden)
    weight = ar_weight(hidden, dtype, g)
    for i, rows in enumerate([5, 1, 64, 3]):  # the rows reach the capture at different epochs
        ar_call(peers, W, dtype, rows, "alias", 1e-5, False, weight, g, f"eager call {i}")
    rows, eps = 16, 1e-5
    partials = [torch.zeros(rows, hidden, dtype=dtype, device=DEV) for _ in range(W)]
    residuals = [torch.zeros(rows, hidden, dtype=dtype, device=DEV) for _ in range(W)]
    out_norm = [torch.zeros(rows, hidden, dtype=dtype, device=DEV) for _ in range(W)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        payload = peers.allreduce(partials, residuals, weight, out_norm, residuals, rows, eps)
    for i in range(10):
        np_, res = ar_inputs(W, rows, hidden, dtype, i % 3 == 0, g)
        for r in range(W):
            partials[r].copy_(np_[r])
            residuals[r].copy_(res)
            out_norm[r].fill_(SENT)
        torch.cuda.synchronize()
        assert peers.states_agree()
        graph.replay()
        peers.record(rows, payload, staged_both=True)
        what = f"replay {i}"
        peers.verify(what)
        check_allreduce(np_, res, weight, out_norm, residuals, rows, eps, what)


# ---- the sequence-sharded decode through the real exchange ---------------------------------------------------------------
class PeerSeqComm:
    """LocalSeqComm's merge() over SeqPeers: each rank registers (part_o, part_lse, out) in rank order; the last
    rank's call runs the collective (duo_seq_merge of every rank).  Like tp.SeqComm, whose C entry point checks every
    call, it refuses a merge of more than max_rows rows at each rank's call: duo_seq_merge's DUO_EOVERFLOW, raised by
    _C.check as ValueError, nothing launched.  Eager calls are verified at once; after a replay of a captured step,
    call after_replay()."""

    def __init__(self, world, max_rows=128):
        self.world, self.max_rows = world, max_rows
        self.peers = SeqPeers(world, max_rows)
        self.pending, self.calls, self.captured = [], 0, None

    def merge(self, part_o, part_lse, out, tokens, heads_total, heads_used):
        if tokens * heads_used > self.max_rows:
            r, self.pending = len(self.pending), []
            _C.check(_C.load().duo_seq_merge(self.peers.handles[r], part_o.data_ptr(), part_lse.data_ptr(),
                                             out.data_ptr(), tokens, heads_total, heads_used, dt_code(out.dtype),
                                             stream()))
            raise AssertionError("duo_seq_merge accepted more rows than its max_rows")
        self.pending.append((part_o, part_lse, out))
        if len(self.pending) < self.world:
            return
        parts, self.pending = self.pending, []
        po, pl, outs = ([p[i] for p in parts] for i in range(3))
        payload = self.peers.merge(po, pl, outs, tokens, heads_total, heads_used)
        R = tokens * heads_used
        if torch.cuda.is_current_stream_capturing():
            self.captured = (R, payload)
        else:
            self.peers.record(R, payload, staged_both=False)
            self.peers.verify(f"merge {self.calls}")
        self.calls += 1

    def before_replay(self):
        assert self.peers.states_agree()

    def after_replay(self, what):
        self.peers.record(*self.captured, staged_both=True)
        self.peers.verify(what)


class TwinRig:
    """A sequence-shard Rig whose ranks merge through PeerSeqComm, and a twin set of ranks on LocalSeqComm
    (duo_merge_partials) fed the same steps: outputs, caches, partials and lengths must stay bit-identical, on top of
    the Rig's own checks against the unsharded control and fp64."""

    def __init__(self, *args, budget=128):
        self.budget = budget
        super().__init__(*args)

    def make_ranks(self, max_size):
        self.twin = super().make_ranks(max_size)
        self.twin_comm = self.comm
        self.comm = PeerSeqComm(self.W, self.budget)
        cls = type(self.twin[0])
        model = S16._Model(self.Hq, self.Hkv, self.dtype)
        gates = [[1.0] * self.nf + [0.0] * (self.Hkv - self.nf)]
        return [cls(model, gates, self.B, max_size, SINK, RECENT, seq=tp.SeqShardContext(r, self.W, self.block, self.comm))
                for r in range(self.W)]

    def scatter(self, ranks=None):
        if ranks is None:
            super().scatter(self.twin)
        super().scatter(ranks)

    def evict(self, k):
        super().evict(k)
        for c in self.twin:
            c.evict_last(k)

    def inputs(self, *args):
        self.last_qkv = super().inputs(*args)
        return self.last_qkv

    def step(self, S, rope, g, *args, fused=True):
        n = self.control.kv_seq_len
        out = super().step(S, rope, g, *args, **({} if isinstance(self, S16.Rig) else {"fused": fused}))
        cos, sin = S16.rope_tables(rope, n, S, self.dtype)
        outs = [torch.full_like(out, float("nan")) for _ in self.twin]
        for t, o in zip(self.twin, outs):  # LocalSeqComm merges at the last rank's call
            t.attend(0, self.last_qkv.clone(), cos, sin, rope, o, fused=fused)
        torch.cuda.synchronize()
        for r, o in enumerate(outs):
            assert same_bits(o, out), f"n={n} S={S}: rank {r}'s output differs between the exchanges"
        self.check_twins(f"n={n} S={S}")
        return out

    def check_twins(self, what, ranks=None, twin=None):
        for r, (rc, t) in enumerate(zip(ranks or self.ranks, twin or self.twin)):
            assert same_bits(rc.part_o, t.part_o) and same_bits(rc.part_lse, t.part_lse), f"{what}: rank {r} partials"
            for name, x in rc.tensors[0].items():
                assert same_bits(x, t.tensors[0][name]), f"{what}: rank {r} {name}"
            assert (rc.kv_seq_len_list, rc.total_list, rc.lo_list) == (t.kv_seq_len_list, t.total_list, t.lo_list)


class Twin16(TwinRig, S16.Rig):
    pass


class Twin4(TwinRig, S4.Rig):
    pass


KINDS = {"16bit": (Twin16, S16), "int4": (Twin4, S4)}
# W = 2 / 4 / 8; block 100 and 1; batch 2; RoPE none / fp32 / HF; evict_last in every schedule
EMULATED = ["w2b100_g4_round", "w4b1_mha_allfull_fp32", "w8b64_g4_fp16_hf_round"]


@pytest.mark.parametrize("case", EMULATED)
@pytest.mark.parametrize("kind", list(KINDS))
def test_sharded_decode_through_duo_seq_merge(kind, case):
    cls, mod = KINDS[kind]
    W, block, Hq, Hkv, nf, B, dtype, rope, n0, sched, *scales = mod.CASES[case]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, case)))
    steps = sum(s for s in sched if isinstance(s, int))
    rig = cls(W, block, Hq, Hkv, nf, B, dtype, n0 + steps + 8)
    rig.prefill(n0, g, *scales[1:])
    rig.scatter()
    rig.check_cache("after the scatter")
    for s in sched:
        if isinstance(s, str):
            rig.evict(int(s[1:]))
        else:
            rig.step(s, rope, g, *scales)
    n_merges = sum(isinstance(s, int) for s in sched)
    assert rig.comm.calls == rig.twin_comm.calls == n_merges


def capture_step(ranks, rope, dtype, width):
    """Warm up, then capture one q_len = 1 step of all ranks (attend + advance_device); the cache state is restored
    after each.  Returns the graph and its input / output tensors."""
    B, Hq = ranks[0].batch_size, ranks[0].num_heads
    qkv = [torch.zeros(B, 1, width, dtype=dtype, device=DEV) for _ in ranks]
    out = [torch.zeros(B, 1, Hq, D, dtype=dtype, device=DEV) for _ in ranks]
    cos, sin = (torch.zeros(1, D, dtype=dtype, device=DEV) for _ in range(2))
    for c in ranks:
        c.enable_device_state()
        c.graph_attached = True
    snap = [(list(c.kv_seq_len_list), list(c.total_list), list(c.lo_list)) for c in ranks]
    rings = [c.snapshot_ring() for c in ranks]

    def restore():
        for c, s, ring in zip(ranks, snap, rings):
            c.kv_seq_len_list[:], c.total_list[:], c.lo_list[:] = (list(x) for x in s)
            c.restore_ring(ring)
            c.sync_device_state()

    for r, c in enumerate(ranks):
        c.attend(0, qkv[r], cos, sin, rope, out[r])
    restore()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for r, c in enumerate(ranks):
            c.attend(0, qkv[r], cos, sin, rope, out[r])
        for c in ranks:
            c.advance_device(1)
    restore()
    return graph, qkv, out, cos, sin


@pytest.mark.parametrize("kind", list(KINDS))
def test_graph_replay_through_duo_seq_merge(kind):
    """One captured q_len = 1 step of all ranks through the real exchange, and the same capture on LocalSeqComm,
    replayed while ownership changes hands, with an evict_last in the middle: outputs and partials bit-identical after
    every replay, merged rows within parity of fp64, caches bit-identical at the end."""
    cls, _ = KINDS[kind]
    W, block, Hq, Hkv, nf, B, dtype, rope = 3, 4, 32, 8, 4, 2, BF16, S16.HF
    n0, T = (3200 if kind == "16bit" else 7000), 2 * 4 * 3 + 4
    rig = cls(W, block, Hq, Hkv, nf, B, dtype, n0 + T + 8)
    g = torch.Generator(device=DEV).manual_seed(9)
    rig.prefill(n0, g)
    rig.scatter()
    gp = capture_step(rig.ranks, rope, dtype, rig.width)
    gl = capture_step(rig.twin, rope, dtype, rig.width)
    for i in range(T):
        if i == T // 2:
            for c in rig.ranks + rig.twin:
                c.evict_last(2)
        n = rig.ranks[0].kv_seq_len
        qkv = rig.inputs(1, g)
        cos, sin = S16.rope_tables(rope, n, 1, dtype)
        for graph, qs, _, cs, ss in (gp, gl):
            for q in qs:
                q.copy_(qkv)
            cs.copy_(cos)
            ss.copy_(sin)
        rig.comm.before_replay()
        gp[0].replay()
        gl[0].replay()
        for c in rig.ranks + rig.twin:
            c.advance_host(1)
        torch.cuda.synchronize()
        what = f"replay {i} (n={n})"
        rig.comm.after_replay(what)
        for r in range(W):
            assert same_bits(gp[2][r], gp[2][0]), f"{what}: rank {r}"
            assert same_bits(gp[2][r], gl[2][r]), f"{what}: rank {r}'s output differs between the exchanges"
        rig.check_twins(what)
        q = S16.host_rope_q(qkv[..., : Hq * D].view(B, 1, Hq, D), rope, cos, sin)
        truth, _ = rig.truth(q, n, 1, None)
        assert_parity(gp[2][0][:, :, : rig.nfq], truth, f"{what}: replayed merged rows vs fp64")
        rig.check_partials(q, n, 1, what)
    assert [c.kv_seq_len for c in rig.ranks] == [n0 + T - 2] * W
    rig.check_cache("end of replay", ranks=rig.ranks, ref=rig.twin)


# ---- the merge's row budget is checked before any launch ------------------------------------------------------------------
def cache_snapshot(c):
    return ([bits(x).clone() for x in c.tensors[0].values()], list(c.kv_seq_len_list), list(c.total_list),
            list(c.lo_list), c.launch_count)


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_over_budget_merge_is_refused_before_any_launch(kind, path):
    """A step whose merge needs more rows than the communicator holds (batch x q_len x retrieval q-heads > max_rows)
    raises ValueError at every rank's call and leaves every rank's slice (sentinel rows included), rings, lengths and
    launch count as they were; the next in-budget step still matches fp64.  Fused: one token, 2 x 1 x 12 = 24 rows
    over a budget of 16; the in-budget step then runs on a communicator of 128 rows.  Unfused: a 2-token chunk,
    2 x 2 x 8 = 32 rows; the in-budget step is one token, exactly 16 rows, on the same communicator."""
    cls, _ = KINDS[kind]
    W, block, Hq, Hkv, B, dtype, rope = 2, 16, 32, 8, 2, BF16, S16.HF
    nf, S = (3, 1) if path == "fused" else (2, 2)
    rows = B * S * nf * (Hq // Hkv)
    rig = cls(W, block, Hq, Hkv, nf, B, dtype, 120, budget=16)
    g = torch.Generator(device=DEV).manual_seed(21)
    rig.prefill(40, g)
    rig.scatter()
    n = rig.control.kv_seq_len
    before = [cache_snapshot(c) for c in rig.ranks]
    qkv = rig.inputs(S, g)
    cos, sin = S16.rope_tables(rope, n, S, dtype)
    for r, c in enumerate(rig.ranks):
        with pytest.raises(ValueError, match=f"{rows} rows.*max_rows 16"):
            c.attend(0, qkv.clone(), cos, sin, rope, torch.empty(B, S, Hq, D, dtype=dtype, device=DEV),
                     fused=path == "fused")
    torch.cuda.synchronize()
    for r, (c, b) in enumerate(zip(rig.ranks, before)):
        a = cache_snapshot(c)
        for name, x, y in zip(c.tensors[0], a[0], b[0]):
            assert torch.equal(x, y), f"rank {r}: {name} changed by the refused call"
        assert a[1:] == b[1:], f"rank {r}: lengths or launch count changed by the refused call"
    if path == "fused":
        comm = PeerSeqComm(W, 128)
        for c in rig.ranks:
            c.seq.comm = comm
        rig.comm = comm
    rig.step(1, rope, g)
    assert rig.comm.calls == 1
