"""Idle rows of a ragged batch on the GPU (row_state flags bit 0, DuoRaggedKVCache.set_active): duo_decode_ragged,
duo_decode_ragged_pooled (16-bit and INT4), duo_decode_ragged_int4 and the shared-prefix cascade.

* the active rows' outputs and cache bytes are bit-identical to a compact cache of just those rows, wherever the
  host twin says the clamp does not bind (within tolerance where it does);
* idle rows: their regions, rings and row_state are unchanged byte for byte, their rows of `out` keep a poison
  pattern, and poisoning their K/V changes no active output; an all-idle step writes nothing;
* shared cascade: an idle donor with active sharers, idle sharers and an all-idle group against a compact control
  cache whose rows hold a copy of the prompt.
"""
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY, DuoRaggedINT4KVCache, DuoRaggedKVCache, ragged_partition

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
POISON = -3.0  # written into `out` before a step: an idle row's rows must still hold it


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _prefill(pairs, L, width, dtype, Hq, g):
    """The same chunks into row b of each (cache, b) pair."""
    for c0 in range(0, L, 4096):
        S = min(4096, L - c0)
        qkv = torch.randn(1, S, width, generator=g).to(dtype).to(DEV)
        for c, b in pairs:
            c.row(b).attend(0, qkv, None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))


def _row_bytes(c, b):
    """Row b's whole region (pooled) or [n_full][cap] slab, and its sink + ring slots, as a dict of clones."""
    return {k: v.clone() for k, v in c.row(b).tensors[0].items()}


def _poison_row(c, b):
    for k, v in c.row(b).tensors[0].items():
        if v.dtype in (torch.bfloat16, torch.float16):
            v.fill_(1e4)
        else:
            v.fill_(0x5A)


def _equal_used(x, y, n, W, shift=0):
    """Row tensors of two caches: retrieval rows [shift, n) of x against [0, n - shift) of y, and the W slots."""
    for k in x:
        a, b = x[k][0], y[k][0]
        if k.startswith("full"):
            a, b = a[:, shift:n], b[:, : n - shift]
        else:
            a, b = a[:, :W], b[:, :W]
        assert torch.equal(a, b), k


def _idle_vs_compact(cls, pooled, lengths, active, steps, Hq, Hkv, n_full, dtype, seed, poison_idle=True):
    sink, recent, B = 16, 48, len(lengths)
    act = [b for b in range(B) if active[b]]
    grow = sum(steps)
    caps = [L + grow + 64 * (b + 1) for b, L in enumerate(lengths)]
    X = cls.from_geometry(1, Hq, Hkv, D, [n_full], B, caps if pooled else max(caps), sink, recent, dtype, DEV,
                          stage_cap=64)
    C = cls.from_geometry(1, Hq, Hkv, D, [n_full], len(act), [caps[b] for b in act] if pooled else max(caps), sink,
                          recent, dtype, DEV, stage_cap=64) if act else None
    g = torch.Generator().manual_seed(seed)
    width = (Hq + 2 * Hkv) * D
    for b, L in enumerate(lengths):
        _prefill([(X, b)] + ([(C, act.index(b))] if b in act else []), L, width, dtype, Hq, g)
    for b in range(B):
        if not active[b]:
            X.set_active(b, False)
            if poison_idle:
                _poison_row(X, b)
    torch.cuda.synchronize()
    idle_bytes = {b: _row_bytes(X, b) for b in range(B) if not active[b]}
    idle_state = X.row_state[[b for b in range(B) if not active[b]]].clone()
    int4 = cls is DuoRaggedINT4KVCache
    for step, S in enumerate(steps):
        keys = [X.row_lengths[b] + (S if int4 else 0) for b in range(B)]
        part = ragged_partition(keys, n_full, Hkv - n_full, _sms(), active=active,
                                **(INT4_RAGGED_POLICY if int4 else {}))
        qkv = torch.randn(B, S, width, generator=g).to(dtype).to(DEV)
        ox = torch.full((B, S, Hq, D), POISON, dtype=dtype, device=DEV)
        X.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, ox)
        X.advance_device(S)  # as the driver does: the device advance must pass the idle rows by
        if C is not None:
            oc = torch.empty(len(act), S, Hq, D, dtype=dtype, device=DEV)
            C.attend(0, qkv[act].contiguous(), None, None, _C.ROPE_NONE, oc)
            if part["clamped"] and n_full > 0:
                torch.testing.assert_close(ox[act].float(), oc.float(), rtol=2e-2, atol=2e-2 if int4 else 4e-3)
            else:
                assert torch.equal(ox[act], oc), f"step {step}: active rows differ from the compact batch"
        for b in range(B):
            if not active[b]:
                assert (ox[b] == POISON).all(), f"step {step}: idle row {b}'s output was written"
    torch.cuda.synchronize()
    assert torch.equal(X.row_state[[b for b in range(B) if not active[b]]], idle_state)
    assert X.row_state[act, 0].tolist() == [X.row_lengths[b] for b in act]  # the active rows moved on the device
    for b, snap in idle_bytes.items():
        now = _row_bytes(X, b)
        for k in snap:
            assert torch.equal(now[k], snap[k]), f"idle row {b}: {k} changed"
    for i, b in enumerate(act):
        assert X.row_lengths[b] == C.row_lengths[i]
        _equal_used(_row_bytes(X, b), _row_bytes(C, i), X.row_lengths[b], X.W)


DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
HEADS = pytest.mark.parametrize("Hq,Hkv,n_full", [(32, 8, 0), (32, 8, 1), (32, 8, 4)])
PATTERNS = pytest.mark.parametrize("active", [
    [True, False, True, True, False, True],
    [False, True, True, True, True, True],
    [True, True, True, True, True, False],
    [False, False, False, True, False, False],
], ids=["two_idle", "first_idle", "last_idle", "one_active"])
LENGTHS16 = [4097, 1, 20000, 320, 9000, 129]
LENGTHS4 = [5000, 64, 20000, 320, 9000, 1500]


@DTYPES
@HEADS
@PATTERNS
@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
def test_idle_rows_16bit(pooled, active, Hq, Hkv, n_full, dtype):
    _idle_vs_compact(DuoRaggedKVCache, pooled, LENGTHS16, active, [1, 2, 1], Hq, Hkv, n_full, dtype, 5 + n_full)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@HEADS
@PATTERNS
@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
def test_idle_rows_int4(pooled, active, Hq, Hkv, n_full, dtype):
    lengths = list(LENGTHS4)
    for b, a in enumerate(active):  # an idle INT4 row may be empty: it is never attended
        if not a and b == 1:
            lengths[b] = 0
    _idle_vs_compact(DuoRaggedINT4KVCache, pooled, lengths, active, [1, 2, 1], Hq, Hkv, n_full, dtype, 7 + n_full)


@pytest.mark.parametrize("cls", [DuoRaggedKVCache, DuoRaggedINT4KVCache], ids=["bf16", "int4"])
def test_clamp_case_stays_close_to_the_compact_batch(cls):
    """n_full 1, n_stream 7, B 2 with one row active: the compact batch wants more splits than the grid's slots."""
    int4 = cls is DuoRaggedINT4KVCache
    L = 300000
    part = ragged_partition([L + (1 if int4 else 0)] * 2, 1, 7, _sms(), active=[True, False],
                            **(INT4_RAGGED_POLICY if int4 else {}))
    if _sms() == 132:  # 16-bit: 257 wanted, 251 fit; INT4 (4 CTAs/SM): 512 wanted, 515 fit
        assert part["clamped"] == (not int4)
    _idle_vs_compact(cls, True, [L, 5000], [True, False], [1, 1], 32, 8, 1, torch.bfloat16, 3)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_clamp_case_matches_fp64_attention(dtype):
    """The 16-bit clamp case (n_full 1, n_stream 7, B 2, row 1 idle: 251 of the 257 wanted splits fit) against fp64
    attention through both parity gates, at a length where the clamp changes keys-per-split."""
    from oracle import duo_oracle as O
    from parity import assert_parity

    Hq, Hkv, n_full, sink, recent, L = 32, 8, 1, 16, 48, 64320  # 251 splits of 320 keys, not 252 of 256
    part = ragged_partition([L, 700], n_full, Hkv - n_full, _sms(), active=[True, False])
    if _sms() == 132:
        assert part["clamped"] and part["keys_per_split"] != ragged_partition([L], n_full, Hkv - n_full)["keys_per_split"]
    X = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], 2, [L + 64, 1024], sink, recent, dtype, DEV,
                                       stage_cap=64)
    g = torch.Generator().manual_seed(23)
    width = (Hq + 2 * Hkv) * D
    ks, vs = [], []
    for c0 in range(0, L, 4096):
        S = min(4096, L - c0)
        qkv = torch.randn(1, S, width, generator=g).to(dtype)
        X.row(0).attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dtype, device=DEV))
        k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(1, S, Hkv, D)
        v = qkv[..., (Hq + Hkv) * D :].reshape(1, S, Hkv, D)
        ks.append(k)
        vs.append(v)
    _prefill([(X, 1)], 700, width, dtype, Hq, g)
    X.set_active(1, False)
    k, v = torch.cat(ks, 1), torch.cat(vs, 1)
    sk, sv = (torch.cat([t[:, :sink, n_full:], t[:, -recent:, n_full:]], 1) for t in (k, v))
    past = (torch.cat([k[:, :, :n_full], v[:, :, :n_full]], 0).transpose(1, 2).contiguous(),
            torch.cat([sk, sv], 0).transpose(1, 2).contiguous())
    del ks, vs, k, v
    for step in range(3):
        qkv = torch.randn(2, 1, width, generator=g).to(dtype)
        out = torch.full((2, 1, Hq, D), POISON, dtype=dtype, device=DEV)
        X.attend(0, qkv.to(DEV), None, None, _C.ROPE_NONE, out)
        q = qkv[:1, :, : Hq * D].reshape(1, 1, Hq, D)
        kn = qkv[:1, :, Hq * D : (Hq + Hkv) * D].reshape(1, 1, Hkv, D)
        vn = qkv[:1, :, (Hq + Hkv) * D :].reshape(1, 1, Hkv, D)
        ref, past = O.tuple_attention_core(q, kn, vn, past, n_full, Hq // Hkv, sink, recent)
        assert_parity(out[:1].float().cpu(), ref, f"clamp case, step {step}")
        assert (out[1] == POISON).all()


@pytest.mark.parametrize("cls", [DuoRaggedKVCache, DuoRaggedINT4KVCache], ids=["bf16", "int4"])
@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
def test_all_idle_step_writes_nothing(cls, pooled):
    B, Hq, Hkv, dtype = 3, 32, 8, torch.bfloat16
    caps = [2048, 3000, 4000]
    X = cls.from_geometry(1, Hq, Hkv, D, [4], B, caps if pooled else 4000, 16, 48, dtype, DEV, stage_cap=64)
    g = torch.Generator().manual_seed(1)
    for b, L in enumerate((700, 1500, 2000)):
        _prefill([(X, b)], L, (Hq + 2 * Hkv) * D, dtype, Hq, g)
    for b in range(B):
        X.set_active(b, False)
    torch.cuda.synchronize()
    snap = [{k: v.clone() for k, v in t.items()} for t in X.tensors]
    state, ws = X.row_state.clone(), X.workspace.clone()
    out = torch.full((B, 1, Hq, D), POISON, dtype=dtype, device=DEV)
    X.attend(0, torch.randn(B, 1, (Hq + 2 * Hkv) * D, generator=g).to(dtype).to(DEV), None, None, _C.ROPE_NONE, out)
    X.advance_device(1)
    torch.cuda.synchronize()
    assert (out == POISON).all() and torch.equal(X.row_state, state) and torch.equal(X.workspace, ws)
    for t, s in zip(X.tensors, snap):
        for k in s:
            assert torch.equal(t[k], s[k]), k
    assert X.row_lengths == [700, 1500, 2000]


def test_state_advance_skips_idle_rows():
    X = DuoRaggedKVCache.from_geometry(1, 32, 8, D, [4], 4, 1024, 4, 8, torch.bfloat16, DEV, stage_cap=64)
    X.row_state.copy_(torch.tensor([[5, 5, 4, 0], [9, 9, 4, 1], [0, 0, 4, 0], [20, 20, 12, 1]]))
    X.advance_device(3)
    torch.cuda.synchronize()
    assert X.row_state.tolist() == [[8, 8, 4, 0], [9, 9, 4, 1], [3, 3, 4, 0], [20, 20, 12, 1]]


# ---- shared cascade ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("n_full", [1, 4])
@pytest.mark.parametrize("idle", [[0], [1], [0, 2], [0, 1, 2], [3]],
                         ids=["idle_donor", "idle_sharer", "donor_and_sharer", "whole_group", "plain_row"])
def test_shared_cascade_idle_rows_against_copy_control(idle, n_full, dtype):
    """Rows 1 and 2 share row 0's prompt, row 3 is plain.  The control holds the active rows only, each sharer as a row
    with a copy of the prompt: outputs within tolerance, own regions and rings byte-identical."""
    Hq, Hkv, sink, recent, L = 32, 8, 16, 48, 9000
    width = (Hq + 2 * Hkv) * D
    caps = [L + 64, 1024, 1024, 3000]
    X = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], 4, caps, sink, recent, dtype, DEV, stage_cap=64)
    act = [b for b in range(4) if b not in idle]
    ccaps = [L + 1024 if b in (1, 2) else caps[b] for b in act]
    C = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [n_full], len(act), ccaps, sink, recent, dtype, DEV,
                                       stage_cap=64) if act else None
    g = torch.Generator().manual_seed(17 + n_full)
    prompt_rows = [(X, 0)] + [(C, i) for i, b in enumerate(act) if b in (0, 1, 2)]
    _prefill(prompt_rows, L, width, dtype, Hq, g)
    _prefill([(X, 3)] + ([(C, act.index(3))] if 3 in act else []), 2000, width, dtype, Hq, g)
    X.share_prefix(0, 1, 1024)
    X.share_prefix(0, 2, 1024)
    P = X.row_prefix[1][1]
    for b in idle:
        X.set_active(b, False)
    for b in idle:  # poison what an idle row owns, except the donor's lent prefix
        if b == 0:
            for k, v in X.row(0).tensors[0].items():
                if k.startswith("full"):
                    v[:, :, P:].fill_(1e4)
                else:
                    v.fill_(1e4)
        else:
            _poison_row(X, b)
    torch.cuda.synchronize()
    snaps = {b: _row_bytes(X, b) for b in idle}
    for step in range(3):
        qkv = torch.randn(4, 1, width, generator=g).to(dtype).to(DEV)
        ox = torch.full((4, 1, Hq, D), POISON, dtype=dtype, device=DEV)
        X.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, ox)
        if C is not None:
            oc = torch.empty(len(act), 1, Hq, D, dtype=dtype, device=DEV)
            C.attend(0, qkv[act].contiguous(), None, None, _C.ROPE_NONE, oc)
            torch.testing.assert_close(ox[act].float(), oc.float(), rtol=1e-2, atol=4e-3)
        for b in idle:
            assert (ox[b] == POISON).all(), f"idle row {b}'s output was written"
    torch.cuda.synchronize()
    for b, snap in snaps.items():
        now = _row_bytes(X, b)
        for k in snap:
            assert torch.equal(now[k], snap[k]), f"idle row {b}: {k} changed"
    for i, b in enumerate(act):
        n = X.row_lengths[b]
        assert n == C.row_lengths[i]
        x, c = _row_bytes(X, b), _row_bytes(C, i)
        if b in (1, 2):  # a sharer's own region row r holds key P + r
            for k in x:
                if k.startswith("full"):
                    assert torch.equal(x[k][0][:, : n - P], c[k][0][:, P:n]), (b, k)
                else:
                    assert torch.equal(x[k][0][:, : X.W], c[k][0][:, : X.W]), (b, k)
        else:
            _equal_used(x, c, n, X.W)
