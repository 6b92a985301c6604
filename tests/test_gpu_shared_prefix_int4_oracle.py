"""Shared prefixes on the INT4 cache, checked against exact references rather than against the library itself.

* fp64 attention over the dequantised values (``code x scale + zero``) for every retrieval row of a batch that shares
  prompts, through both launches of duo_decode_ragged_shared and through a sharer's chunks on duo_attention_shared,
  held to the forward-error bound of tests/softmax_bound.py.  Every cache row a reader must not see holds poison
  (K = 0, V = 1000: a logit inside the data's range and a value whose weight, however small, leaves the bound): the
  pool's slack and headroom, other rows' regions past their lengths.  The donor's rows >= P, which its sharers must
  not see but the donor does, hold V around 100;
* a visibility census: every key has logit 0 and carries a one-hot value by where it lives, every row a reader must
  not see lights dimension 127, so each output is an exact histogram of the keys that row attends (a prefix launch
  that read one key past P, a suffix launch that read a donor's tail, would show up as a count off by one).
"""
import math

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoRaggedINT4KVCache
from softmax_bound import LOG2E, bound_terms, worst_ratio

pytestmark = pytest.mark.gpu
D = 128
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def _deq(t, name, h, lo, hi):
    """(s c + z, s c, s) in fp64 of rows [lo, hi) of head h of a batch-1 row view ``t`` (high nibble = even dim)."""
    pk = t[name][0, h, lo:hi].long()
    c = torch.stack([pk >> 4, pk & 15], -1).reshape(pk.shape[0], D).double()
    s = t[name + "_scale"][0, h, lo:hi].double()[:, None]
    z = t[name + "_zero"][0, h, lo:hi].double()[:, None]
    return c * s + z, c * s, s[:, 0]


def _fill(t, name, lo, hi, g, big_v=False):
    """Ordinary INT4 rows [lo, hi) of every head of row view ``t``: random codes, K in about [-1, 1.2], V likewise or
    (big_v) around 100."""
    n = hi - lo
    if n <= 0:
        return
    shape = t[name][0, :, lo:hi].shape
    t[name][0, :, lo:hi] = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).to(DEV)
    sc = torch.rand(shape[:2], generator=g, dtype=torch.float64) * 0.1 + 0.05
    zr = -torch.rand(shape[:2], generator=g, dtype=torch.float64)
    if big_v:
        sc, zr = sc * 10, zr + 100
    t[name + "_scale"][0, :, lo:hi] = sc.half().to(DEV)
    t[name + "_zero"][0, :, lo:hi] = zr.half().to(DEV)


def _poison_pool(S):
    t = S.tensors[0]
    for k in ("full_k", "full_k_scale", "full_k_zero", "full_v", "full_v_scale"):
        t[k].zero_()
    t["full_v_zero"].fill_(1000.0)


def _set_len(r, n, sink, recent):
    r.kv_seq_len_list[0] = r.total_list[0] = n
    r.lo_list[0] = max(sink, n - recent)


def _check_rows(row, got, q, n_before, prefix, dtype, G, n_full, what):
    """``got`` [S_tok, Hq, D] of batch-1 row view ``row``, ``q`` [S_tok, Hq, D] its query rows; ``n_before`` the row's
    logical length before the call; ``prefix`` = (donor row view, P) or None.  Every retrieval head against fp64."""
    donor, pre = prefix if prefix is not None else (None, None)
    worst = 0.0
    S_tok = q.shape[0]
    for h in range(n_full):
        parts = []
        if pre is not None:  # the donor's rows [0, P), then the own rows from logical key P
            parts.append(_deq_all(donor, h, 0, pre))
        P = pre or 0
        parts.append(_deq_all(row, h, 0, n_before - P + S_tok))
        k, v, rr, sv = (torch.cat(x) for x in zip(*parts))
        n_keys = k.shape[0]
        keys = torch.arange(n_keys)
        vis = keys[None] < (n_before + 1 + torch.arange(S_tok))[:, None]          # [S_tok, n]
        mask = vis.repeat_interleave(G, 0)
        qh = q[:, h * G : (h + 1) * G].reshape(S_tok * G, D).double()
        l2 = ((qh @ k.T) * (D ** -0.5 * LOG2E)).masked_fill(~mask, -math.inf)
        want, bound, _ = bound_terms(l2, v, torch.float16, dtype, rr, sv)
        g_ = got[:, h * G : (h + 1) * G].reshape(S_tok * G, D).double()
        worst = max(worst, worst_ratio(g_, want, bound))
    assert worst <= 1.0, f"{what}: worst err / bound {worst:.3f}"


def _deq_all(r, h, lo, hi):
    t = r.tensors[0]
    k = _deq(t, "full_k", h, lo, hi)[0]
    v, rr, sv = _deq(t, "full_v", h, lo, hi)
    return k.cpu(), v.cpu(), rr.cpu(), sv.cpu()


# ---- fp64 attention: both launches of the cascade and a sharer's chunks -----------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("Hq,Hkv,n_full,q_len", [(16, 4, 3, 2), (4, 4, 3, 8), (32, 8, 8, 1)])
@pytest.mark.parametrize("LA", [700, 4097])
def test_shared_rows_match_fp64_attention(LA, Hq, Hkv, n_full, q_len, dtype):
    """Rows: 0 donor of prompt A (its tail past P holds V ~ 100), 1 forked from 0, 2 forked from 1, 3 a plain row,
    4 donor of a 300-key prompt, 5 forked from 4.  Decode steps through duo_decode_ragged_shared, then chunks of 3 and
    9 tokens on row 1 through duo_attention_shared (the 16- and 64-row INT4 kernels; 3 tokens only where they make
    more than 8 rows).  The prefix launch splits its keys at both prompt lengths."""
    G = Hq // Hkv
    sink, recent, B, steps = 16, 48, 6, 3
    own = 256 + steps * q_len + 16
    lengths = [LA, 0, 0, 500, 300, 0]
    caps = [LA + own, own, own, 500 + own, 300 + own, own]
    S = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64,
                                           pool_size=4096 + sum(caps))
    g = torch.Generator().manual_seed(LA + Hq + q_len)
    _poison_pool(S)
    PA = LA // 128 * 128
    for b, n in enumerate(lengths):
        r = S.row(b)
        for name in ("full_k", "full_v"):
            _fill(r.tensors[0], name, 0, n, g)
        _set_len(r, n, sink, recent)
    _fill(S.row(0).tensors[0], "full_v", PA, LA, g, big_v=True)  # the donor sees its tail; its sharers must not
    S.sync_device_state()
    S.share_prefix(0, 1, own)
    for name in ("full_k", "full_v"):  # row 1's own tail: ordinary values, unlike the donor's rows it was copied from
        _fill(S.row(1).tensors[0], name, 0, LA - PA, g)
    S.share_prefix(1, 2, own)
    S.share_prefix(4, 5, own)
    assert S.row_prefix == [None, (0, PA), (0, PA), None, None, (4, 256)]
    prefix_of = {b: (S.row(sh[0]), sh[1]) if sh else None for b, sh in enumerate(S.row_prefix)}
    width = (Hq + 2 * Hkv) * D
    for step in range(steps):
        x = (torch.randn(B, q_len, width, generator=g) * 0.5).to(dtype)
        n_before = S.row_lengths
        out = torch.empty(B, q_len, Hq, D, dtype=dtype, device=DEV)
        S.attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        torch.cuda.synchronize()
        got = out.float().cpu()
        for b in range(B):
            _check_rows(S.row(b), got[b], x[b, :, : Hq * D].view(q_len, Hq, D), n_before[b], prefix_of[b], dtype, G,
                        n_full, f"step {step} row {b}")
    for S_tok in (3, 9):
        if S_tok * G <= _C.DECODE_MAX_Q_INT4:
            continue
        x = (torch.randn(1, S_tok, width, generator=g) * 0.5).to(dtype)
        n_before = S.row(1).kv_seq_len
        out = torch.empty(1, S_tok, Hq, D, dtype=dtype, device=DEV)
        S.row(1).attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        torch.cuda.synchronize()
        _check_rows(S.row(1), out.float().cpu()[0], x[0, :, : Hq * D].view(S_tok, Hq, D), n_before, prefix_of[1],
                    dtype, G, n_full, f"chunk of {S_tok} on row 1")


# ---- visibility census ------------------------------------------------------------------------------------------------
POISON = 127


def _onehot_codes(n, dim):
    c = torch.zeros(n, D // 2, dtype=torch.uint8)
    c[:, dim // 2] = 0xF0 if dim % 2 == 0 else 0x0F
    return c.to(DEV)


def _set_v(t, lo, hi, dim):
    """V = one-hot at ``dim`` (code 15, scale 1/15, zero 0) in rows [lo, hi) of every head of row view ``t``."""
    t["full_v"][0, :, lo:hi] = _onehot_codes(hi - lo, dim)
    t["full_v_scale"][0, :, lo:hi] = 1.0 / 15
    t["full_v_zero"][0, :, lo:hi] = 0.0


def test_visibility_census_two_groups_and_plain_rows():
    """Rows: 0 donor of prompt A (300 keys, 256 shared), 1 forked from 0, 2 forked from 1, 3 donor of prompt B (700 keys,
    640 shared), 4 forked from 3, 5 a plain row of 500 keys.  Value dimensions: 0 / 1 prompt A's shared part / tail,
    2 / 3 prompt B's, 4 row 5's prompt, 10 + b row b's decoded tokens (the donors keep appending after the fork), 20 + t
    token t of a chunk on row 1 (duo_attention_shared, 9 tokens: the 64-row kernel; 3: the 16-row kernel)."""
    Hq, Hkv, n_full, dtype = 32, 8, 8, torch.bfloat16
    B, steps, sink, recent = 6, 5, 16, 48
    lengths = [300, 0, 0, 700, 0, 500]
    caps = [300 + 64, 200, 200, 700 + 64, 200, 500 + 64]
    S = DuoRaggedINT4KVCache.from_geometry(1, Hq, Hkv, D, [n_full], B, caps, sink, recent, dtype, DEV, stage_cap=64,
                                           pool_size=4096)
    t = S.tensors[0]  # the whole pool is poison until written: K = 0 (logit 0 like every key), V lights POISON
    for k in ("full_k", "full_k_scale", "full_k_zero", "full_v_zero"):
        t[k].zero_()
    t["full_v"].zero_()
    t["full_v"][..., POISON // 2] = 0x0F
    t["full_v_scale"].fill_(1.0 / 15)
    layout = {0: [(0, 256, 0), (256, 300, 1)], 3: [(0, 640, 2), (640, 700, 3)], 5: [(0, 500, 4)]}
    for b, parts in layout.items():
        r = S.row(b)
        for lo, hi, dim in parts:
            _set_v(r.tensors[0], lo, hi, dim)
        _set_len(r, lengths[b], sink, recent)
    S.sync_device_state()
    S.share_prefix(0, 1, 200)
    S.share_prefix(1, 2, 200)
    S.share_prefix(3, 4, 200)
    cnt = {0: {0: 256, 1: 44}, 1: {0: 256, 1: 44}, 2: {0: 256, 1: 44}, 3: {2: 640, 3: 60}, 4: {2: 640, 3: 60},
           5: {4: 500}}
    width = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(3)

    def check(got, c, what):  # got [Hq, D]
        n = sum(c.values())
        exp = torch.zeros(D, dtype=torch.float64)
        for dim, k in c.items():
            exp[dim] = k / n
        lit = exp > 0
        for h in range(Hq):
            row = got[h].double()
            assert torch.all(row[~lit] == 0), f"{what} head {h}: sees keys it must not " \
                                              f"(dims {torch.nonzero(row * ~lit).flatten().tolist()})"
            assert torch.all((row[lit] - exp[lit]).abs() <= exp[lit] * 2 ** -8), \
                f"{what} head {h}: {row[lit].tolist()} != {exp[lit].tolist()}"

    for step in range(steps):
        x = torch.zeros(B, 1, width, dtype=dtype)
        x[..., : Hq * D] = torch.randn(B, 1, Hq * D, generator=g).to(dtype)  # any q: every key has logit 0
        for b in range(B):
            x[b, 0, (Hq + Hkv) * D :].view(Hkv, D)[:, 10 + b] = 1
        out = torch.empty(B, 1, Hq, D, dtype=dtype, device=DEV)
        S.attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        got = out.float().cpu()[:, 0]
        for b in range(B):
            cnt[b][10 + b] = step + 1
            check(got[b], cnt[b], f"step {step} row {b}")
    for S_tok in (3, 9):  # a sharer's chunks: causal among the new tokens
        x = torch.zeros(1, S_tok, width, dtype=dtype)
        x[..., : Hq * D] = torch.randn(1, S_tok, Hq * D, generator=g).to(dtype)
        for tk in range(S_tok):
            x[0, tk, (Hq + Hkv) * D :].view(Hkv, D)[:, 20 + tk] = 1
        out = torch.empty(1, S_tok, Hq, D, dtype=dtype, device=DEV)
        S.row(1).attend(0, x.to(DEV), None, None, _C.ROPE_NONE, out)
        got = out.float().cpu()[0]
        for tk in range(S_tok):
            cnt[1][20 + tk] = cnt[1].get(20 + tk, 0) + 1
            check(got[tk], cnt[1], f"chunk of {S_tok}, token {tk}")  # (the next chunk sees these keys too)
