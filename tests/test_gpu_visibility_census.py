"""Key visibility of every attention kernel, checked exactly: a probe-key census with poisoned stale rows.

Random-data parity (tests/parity.py) cannot see one key too many or too few at long context: it changes a row by about
|v - o| / N.  Here the inputs are designed so that every output can be read exactly (ROPE_NONE):

* probe keys: K = A u_h (u_h a fixed +-1 pattern per KV head), V = e_c(p), one-hot on a dimension chosen from the
  position p; every probe of a head gets the same logit, so a row's output is the histogram of the probes it sees
  divided by their number.  At most ~32 probes share a dimension, so one missing or extra probe moves a lit
  dimension by >= 3 %, several ulps;
* fillers: K = 0, V = 0.  The probe logit exceeds theirs by > 150 in the log2 domain: their weight is exactly 0;
* poison: every row a call must not attend (retrieval rows past the chunk, ring slots that are not live, staging rows
  past the chunk, evicted tokens, rows of the 16-bit image of an INT4 cache past what a call dequantises) holds
  K = A u_h, V = e_127.  Dimension 127 of every output must be exactly 0.

Batch rows use disjoint dimension ranges, so a row that reads its neighbour's keys lights dimensions that must be 0.
The expected output comes in fp64 from the visibility model of tests/visibility_model.py (pinned to the oracle on the
CPU by tests/test_visibility_model_host.py).  Per call: unlit dimensions exactly 0, lit dimensions within 1 ulp of
the output dtype (2 ulp on INT4 caches, where scale and zero are applied in fp32), a NaN canary past ``out`` intact,
and a write census: every cache row the call may not write (anything but the new retrieval rows, the staging rows
and the ring slots of the new positions) is bit-identical before and after the call.
"""
import random

import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import (DuoKVCache, DuoRaggedINT4KVCache, DuoRaggedKVCache, ragged_partition,
                                         ring_slot)
from oracle import int4_oracle as Q
from visibility_model import TupleVisibility
import int4_bf16_oracle as QB

pytestmark = pytest.mark.gpu
D = 128
A = 4.0            # probe amplitude: logit A^2 sqrt(128) = 181 (261 in the log2 domain) over fillers' 0
POISON = 127       # the dimension only poison rows light
PER_DIM = 32       # probes per dimension and batch row at most
DTYPES = [torch.bfloat16, torch.float16]


def _u(Hkv, dev):
    """Walsh rows: u_h[d] = (-1)^popcount(h & d)."""
    h = torch.arange(Hkv)[:, None]
    d = torch.arange(D)[None, :]
    bits = torch.zeros(Hkv, D, dtype=torch.int64)
    x = h & d
    while x.any():
        bits += x & 1
        x = x >> 1
    return (1 - 2 * (bits % 2)).to(torch.float32).to(dev)


def _labels(B, npos, must=None, seed=0):
    """[B, npos] int64: the dimension of the probe at each position, -1 for a filler.  Every position is a probe when
    the per-dimension budget allows, otherwise the positions ``must`` plus seeded random ones up to the budget.
    Row b owns the dimensions [b nd, (b + 1) nd), nd = 127 // B."""
    nd = POISON // B
    budget = nd * PER_DIM
    lab = torch.full((B, npos), -1, dtype=torch.int64)
    for b in range(B):
        if npos <= budget:
            probes = list(range(npos))
        else:
            rng = random.Random(seed * 31 + b)
            sel = sorted({p for p in (must or []) if 0 <= p < npos})
            assert len(sel) <= budget, (len(sel), budget)
            rest = budget - len(sel)
            extra = set()
            while len(extra) < rest // 2:
                extra.add(rng.randrange(npos))
            probes = sorted(set(sel) | extra)
        idx = torch.tensor(probes, dtype=torch.int64)
        lab[b, idx] = b * nd + (torch.arange(len(probes)) + 7 * b) % nd
    return lab


def _ulp(x, dtype):
    bits = 7 if dtype == torch.bfloat16 else 10
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -24)))
    return torch.pow(2.0, e - bits).clamp_min(2.0 ** -24)


class Census:
    """A DuoKVCache (``ragged``: a DuoRaggedKVCache / DuoRaggedINT4KVCache, ``cap`` a sequence: pooled) filled and
    checked for the census.  ``lab`` [B, npos] labels every position (``_labels``); every batch row has its own
    visibility model, so ragged rows may sit at different lengths.  Optional, for unequal logits
    (tests/test_gpu_softmax_mass.py): ``level`` [B, npos] puts probe keys at K = level_p u_h instead of A u_h, ``qamp``
    [Hq] puts query head i at q = qamp_i u_h instead of A u_h."""

    def __init__(self, Hq, Hkv, nf_list, B, cap, sink, recent, dtype, lab, kv_format="same", stage_cap=64,
                 ragged=False, pool_size=None, level=None, qamp=None):
        self.dev = torch.device("cuda:0")
        self.B, self.Hq, self.Hkv, self.G = B, Hq, Hkv, Hq // Hkv
        self.dtype, self.int4, self.ragged = dtype, kv_format == "int4", ragged
        self.sink, self.recent = sink, recent
        if ragged:
            cls = DuoRaggedINT4KVCache if self.int4 else DuoRaggedKVCache
            self.cache = cls.from_geometry(len(nf_list), Hq, Hkv, D, nf_list, B, cap, sink, recent, dtype, self.dev,
                                           stage_cap=stage_cap, pool_size=pool_size)
        else:
            self.cache = DuoKVCache(len(nf_list), Hq, Hkv, D, nf_list, B, cap, sink, recent, dtype, self.dev,
                                    stage_cap=stage_cap, kv_format=kv_format)
        self.models = [[TupleVisibility(sink, recent) for _ in range(B)] for _ in nf_list]
        self.lab = lab.to(self.dev)
        self.level = None if level is None else level.to(self.dev, torch.float32)
        self.qamp = torch.full((Hq,), A) if qamp is None else qamp
        self.u = _u(Hkv, self.dev)
        self.calls = 0
        for l in range(len(nf_list)):
            if self.cache.pooled:  # the whole pool, headroom included, as one region
                self._poison_region(l, 0, self.cache.pool_tokens)
            for b in range(B):
                self._poison_dead(l, b)

    # ---- rows ------------------------------------------------------------------------------------------------
    def _view(self, tensors, l, b):
        """Batch row b of layer l's ``tensors`` (the cache's, or a snapshot of them) as [1, heads, rows, ..] views:
        a pooled row's retrieval region is pool rows [first_b n_full, (first_b + cap_b) n_full) (DESIGN §2)."""
        c = self.cache
        if not c.pooled:
            return {k: v[b : b + 1] for k, v in tensors.items()}
        first, cap = c._geom[b]
        nf = c.num_full_kv_head_list[l]
        return {k: (v[first * nf : (first + cap) * nf].view(1, nf, cap, *v.shape[1:]) if k.startswith("full")
                    else v[b : b + 1]) for k, v in tensors.items()}

    def _state(self, l, b):
        """(full_len, total, lo) of batch row b in layer l."""
        rc = self.cache.row(b) if self.ragged else self.cache
        return rc.kv_seq_len_list[l], rc.total_list[l], rc.lo_list[l]

    def _rows(self, kind, h, lev=None):
        """16-bit K and V rows for labels ``kind`` [n] (>= 0 probe dimension, -1 filler, -2 poison) of KV head h;
        ``lev`` [n]: the probes' K levels (default A; poison stays at A)."""
        n = kind.numel()
        k = torch.zeros(n, D, device=self.dev)
        v = torch.zeros(n, D, device=self.dev)
        hot = kind != -1
        amp = torch.full((n,), A, device=self.dev)
        if lev is not None:
            amp = torch.where(kind >= 0, lev, amp)
        k[hot] = amp[hot, None] * self.u[h]
        dim = torch.where(kind == -2, POISON, kind).clamp_min(0)
        v[hot, dim[hot]] = 1.0
        return k, v

    def _store(self, t, name, h, slots, rows):
        """Rows (fp32 values exact in fp16 and bf16) into ``slots`` of head h of the [1, heads, rows, ..] view
        ``t[name]`` (INT4: K1-quantised by duo_quant_int4)."""
        if not self.int4:
            t[name][0, h, slots] = rows.to(self.dtype)
            return
        n = rows.shape[0]
        r16 = rows.to(torch.float16).contiguous()
        p = torch.empty(n, D // 2, dtype=torch.uint8, device=self.dev)
        s = torch.empty(n, dtype=torch.float16, device=self.dev)
        z = torch.empty(n, dtype=torch.float16, device=self.dev)
        _C.check(self.cache.lib.duo_quant_int4(r16.data_ptr(), D, n, p.data_ptr(), s.data_ptr(), z.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
        t[name][0, h, slots] = p
        t[name + "_scale"][0, h, slots] = s
        t[name + "_zero"][0, h, slots] = z

    def _fill(self, t, l, name_k, h, slots, kind, lev=None):
        """K/V rows of labels ``kind`` (levels ``lev``) into ``slots`` of head h of the view ``t[name_k]`` (full_k: KV
        head h; ring_k: KV head n_full + h)."""
        if slots.numel():
            kvh = h if name_k == "full_k" else self.cache.num_full_kv_head_list[l] + h
            k, v = self._rows(kind, kvh, lev)
            self._store(t, name_k, h, slots, k)
            self._store(t, name_k.replace("_k", "_v"), h, slots, v)

    def _poison_region(self, l, first, cap):
        """Poison pool tokens [first, first + cap) of layer l laid out as a row region [n_full][cap] (per-head
        poison K, so that a head reading there by mistake sees the probe logit)."""
        t = self.cache.tensors[l]
        nf = self.cache.num_full_kv_head_list[l]
        view = {k: v[first * nf : (first + cap) * nf].view(1, nf, cap, *v.shape[1:])
                for k, v in t.items() if k.startswith("full")}
        rows = torch.arange(cap, device=self.dev)
        for h in range(nf):
            self._fill(view, l, "full_k", h, rows, torch.full_like(rows, -2))

    def _poison_dead(self, l, b):
        """Poison every row batch row b's next call in layer l may not see: retrieval rows >= full_len, ring slots that
        hold no live position, all staging rows."""
        t = self._view(self.cache.tensors[l], l, b)
        nf = self.cache.num_full_kv_head_list[l]
        n = self._state(l, b)[0]
        live = {ring_slot(p, self.sink, self.recent) for p in self.models[l][b].stream_live()}
        dead = torch.tensor([s for s in range(t["ring_k"].shape[2]) if s not in live], dtype=torch.int64,
                            device=self.dev)
        rows = torch.arange(n, t["full_k"].shape[2], device=self.dev)
        for h in range(nf):
            self._fill(t, l, "full_k", h, rows, torch.full_like(rows, -2))
        for h in range(self.Hkv - nf):
            self._fill(t, l, "ring_k", h, dead, torch.full_like(dead, -2))

    def fill(self, l, N, rows=None):
        """Put N positions into layer l of the batch rows ``rows`` (default: all) directly, the state of one N-token
        chunk, as the benchmark fills its cache."""
        c = self.cache
        nf = c.num_full_kv_head_list[l]
        for b in range(self.B) if rows is None else rows:
            m = self.models[l][b]
            assert m.total == 0 and self._state(l, b)[0] == 0
            m.chunk(N)
            live = torch.tensor(m.stream_live(), dtype=torch.int64, device=self.dev)
            slots = torch.tensor([ring_slot(p, self.sink, self.recent) for p in m.stream_live()], dtype=torch.int64,
                                 device=self.dev)
            t = self._view(c.tensors[l], l, b)
            pos = torch.arange(N, device=self.dev)
            lev = self.level[b] if self.level is not None else None
            for h in range(nf):
                self._fill(t, l, "full_k", h, pos, self.lab[b, pos], None if lev is None else lev[pos])
            for h in range(self.Hkv - nf):
                self._fill(t, l, "ring_k", h, slots, self.lab[b, live], None if lev is None else lev[live])
            rc = c.row(b) if self.ragged else c
            rc.kv_seq_len_list[l] = N
            rc.total_list[l] = N
            rc.lo_list[l] = max(self.sink, N - self.recent)
            self._poison_dead(l, b)
        if self.ragged:
            c.rows_changed = True
        c.sync_device_state()

    # ---- one call ----------------------------------------------------------------------------------------------
    def _qkv(self, rows, starts, S):
        Hq, Hkv, G = self.Hq, self.Hkv, self.G
        qkv = torch.zeros(len(rows), S, Hq + 2 * Hkv, D, device=self.dev)
        qkv[:, :, :Hq] = self.qamp.to(self.dev)[:, None] * self.u.repeat_interleave(G, 0)
        for i, b in enumerate(rows):
            kind = self.lab[b, starts[i] : starts[i] + S]
            lev = None if self.level is None else self.level[b, starts[i] : starts[i] + S]
            for h in range(Hkv):
                k, v = self._rows(kind, h, lev)
                qkv[i, :, Hq + h] = k
                qkv[i, :, Hq + Hkv + h] = v
        return qkv.view(len(rows), S, -1).to(self.dtype).contiguous()

    def _lit(self, S, first, force_mma):
        """Value of a lit probe dimension as the kernel attends it: 1 in 16 bits and on an INT4 cache's first call
        (raw K/V); else K2's fp16 value of code 15, or for bf16 chunks of >= 128 tokens the bf16 image value."""
        if not self.int4 or first:
            return 1.0
        e = np.zeros((1, D), dtype=np.float16)
        e[0, 0] = 1
        p, s, z = Q.quantize_int4(e)
        if self.dtype == torch.bfloat16 and S >= 128 and self.cache.W <= 2048 and not force_mma:
            return float(QB.dequantize_int4_bf16(p, s, z)[0, 0])
        return float(Q.dequantize_int4(p, s, z)[0, 0])

    def _expected(self, b, ch, lit):
        """[2, S, 128] fp64 (class 0 retrieval, 1 streaming) for batch row b from the histogram of the visible
        probes."""
        S, P = ch.S, ch.start
        out = torch.empty(2, S, D, dtype=torch.float64, device=self.dev)
        lab = self.lab[b, : P + S]
        oh = torch.zeros(P + S + 1, D, dtype=torch.float64, device=self.dev)
        pr = torch.nonzero(lab >= 0).flatten()
        oh[pr + 1, lab[pr]] = 1.0
        cum = oh.cumsum_(0)
        for cls, before in ((0, ch.full), (1, ch.stream)):
            base = torch.zeros(D, dtype=torch.float64, device=self.dev)
            for a, e in before:
                base += cum[e] - cum[a]
            cnt = base + cum[P + 1 : P + S + 1] - cum[P]
            tot = cnt.sum(-1, keepdim=True)
            assert (tot > 0).all(), "every row must see at least one probe"
            out[cls] = cnt * lit / tot
        return out

    def chunk(self, l, S, force_mma=False, fused=True, image_poison=False, row=None, graph=None, what=""):
        """One call of S tokens on layer l: ``cache.attend``, ``cache.row(row).attend`` for one row of a ragged cache,
        or ``graph`` = (DuoDecodeGraph, its qkv buffer, its out buffer) replayed once for one token."""
        c = self.cache
        rows = list(range(self.B)) if row is None else [row]
        for b in rows:
            self._poison_dead(l, b)
        states = [self._state(l, b) for b in rows]
        starts = [self.models[l][b].total for b in rows]
        for (full_len, total, _), start in zip(states, starts):
            assert start == full_len == total
        first = all(st[0] == 0 and st[1] == 0 for st in states)
        if image_poison:
            self._poison_image(l, S)
        qkv = self._qkv(rows, starts, S)
        before = [{k: v.clone() for k, v in t.items()} for t in c.tensors]
        n = len(rows) * S * self.Hq * D
        if graph is None:
            buf = torch.full((n + 256,), float("nan"), dtype=self.dtype, device=self.dev)
            out = buf[:n].view(len(rows), S, self.Hq, D)
            target = c if row is None else c.row(row)
            target.attend(l, qkv, None, None, _C.ROPE_NONE, out, force_mma=force_mma, fused=fused)
        else:
            g, qkv_buf, buf = graph
            assert S == 1 and row is None and c.num_layers == 1
            qkv_buf.copy_(qkv)
            g.step(torch.zeros(self.B, 1, dtype=torch.long, device=self.dev))
            out = buf[:n].view(len(rows), S, self.Hq, D)
        chs = [self.models[l][b].chunk(S) for b in rows]
        for b, ch in zip(rows, chs):
            assert self._state(l, b)[0] == ch.start + S
        ctx = (f"{what} call {self.calls} layer {l}: S={S} past={starts} rows={rows} force_mma={force_mma} "
               f"fused={fused}")
        self.calls += 1
        assert torch.isnan(buf[n:]).all(), f"{ctx}: canary past out overwritten"
        self._check(out, rows, chs, l, S, first, force_mma, ctx)
        self._write_census(l, before, rows, states, S, ctx)
        return out

    def _check(self, out, rows, chs, l, S, first, force_mma, ctx):
        """``out`` [rows, S, Hq, 128] of one call against the probe histogram."""
        lit = self._lit(S, first, force_mma)
        for i, (b, ch) in enumerate(zip(rows, chs)):
            self._check_out(out[i], self._expected(b, ch, lit), b, l, ctx)

    def evict(self, n, row=None):
        """``evict_last(n)`` on the cache, or on ``cache.row(row)`` only."""
        (self.cache if row is None else self.cache.row(row)).evict_last(n)
        for ms in self.models:
            for b, m in enumerate(ms):
                if row is None or b == row:
                    m.evict(n)

    def clear_and_resize(self, b, capacity):
        """Empty row b of a pooled cache, move it to a region of ``capacity`` tokens and poison the region it left."""
        c = self.cache
        c.row(b).clear()
        old = list(c._geom[b])
        c.resize_row(b, capacity)
        for l in range(c.num_layers):
            self._poison_region(l, *old)
            self.models[l][b] = TupleVisibility(self.sink, self.recent)
            self._poison_dead(l, b)

    # ---- checks ------------------------------------------------------------------------------------------------
    def _check_out(self, out, exp, b, l, ctx):
        """``out`` [S, Hq, 128] of batch row b against ``exp`` [2, S, 128]."""
        nf = self.cache.num_full_kv_head_list[l]
        ulps = 2 if self.int4 else 1
        for h in range(self.Hkv):
            got = out[:, h * self.G : (h + 1) * self.G].double()          # [S, G, D]
            e = exp[0 if h < nf else 1][:, None].expand_as(got)
            kind = "retrieval" if h < nf else "streaming"
            dark = e == 0
            bad = dark & (got != 0)
            if bad.any():
                t, g, d = torch.nonzero(bad)[0].tolist()
                what = "POISON" if d == POISON else "another batch row's" if d // (POISON // self.B) != b else "unlit"
                raise AssertionError(f"{ctx}: kv head {h} ({kind}) row {t} of batch row {b} lights dimension {d} "
                                     f"({what}) = {got[t, g, d].item():.6g}; {int(bad.sum())} such elements")
            err = (got - e).abs()
            tol = ulps * _ulp(e, self.dtype)
            worse = ~dark & ~(err <= tol)
            if worse.any():
                t, g, d = torch.nonzero(worse)[0].tolist()
                raise AssertionError(f"{ctx}: kv head {h} ({kind}) row {t} of batch row {b}, dimension {d}: got "
                                     f"{got[t, g, d].item():.8g}, expected {e[t, g, d].item():.8g} (> {ulps} ulp); "
                                     f"{int(worse.sum())} such elements")

    def _write_census(self, l, before, rows, states, S, ctx):
        """Every layer's tensors must equal the snapshot ``before`` except, in layer l, the rows the call may write
        for the batch rows ``rows``: retrieval rows [full_len, full_len + S), the staging rows and the ring slots of
        the new positions.  Those are copied into the snapshot first, through the same row views."""
        c = self.cache
        for b, (full_len, total, _) in zip(rows, states):
            old, new = self._view(before[l], l, b), self._view(c.tensors[l], l, b)
            ring_ok = torch.zeros(new["ring_k"].shape[2], dtype=torch.bool, device=self.dev)
            ring_ok[c.stage_off :] = True
            if c.num_streaming_kv_head_list[l]:
                ring_ok[[ring_slot(p, self.sink, self.recent) for p in range(total, total + S)]] = True
            for name in old:
                if name.startswith("full"):
                    old[name][:, :, full_len : full_len + S] = new[name][:, :, full_len : full_len + S]
                else:
                    old[name][:, :, ring_ok] = new[name][:, :, ring_ok]
        for ll, snap in enumerate(before):
            for name, old in snap.items():
                same = (c.tensors[ll][name] == old).reshape(-1)
                if not bool(same.all()):
                    raise AssertionError(f"{ctx}: the call wrote layer {ll} {name} rows it may not write "
                                         f"({int((~same).sum())} elements differ)")

    def _poison_image(self, l, S):
        """Poison, in layer l's view, every row of the shared 16-bit image of an INT4 cache: the dequantisation of
        this call overwrites what it may see, whatever another layer left must stay invisible."""
        sc = self.cache._dq
        B = self.B
        nf, ns = self.cache.num_full_kv_head_list[l], self.cache.num_streaming_kv_head_list[l]
        cap = sc["cap"]
        slots = self.cache.W + max(max(self.cache.stage_cap_list), S)
        fk, fv = (x[: B * nf * cap * D].view(B, nf, cap, D) for x in sc["full"])
        rk, rv = (x[: B * ns * slots * D].view(B, ns, slots, D) for x in sc["ring"])
        for h in range(self.Hkv):
            k, v = self._rows(torch.tensor([-2], device=self.dev), h)
            if h < nf:
                fk[:, h] = k.to(self.dtype)
                fv[:, h] = v.to(self.dtype)
            else:
                rk[:, h - nf] = k.to(self.dtype)
                rv[:, h - nf] = v.to(self.dtype)


def _schedule_must(ops, sink, recent):
    """Probe positions where a schedule's visibility changes: sinks, the first / last keys of every call, lo - 1 / lo /
    lo + 1 and the ring wrap, cache tiles of 64 and 128 keys near the end, the chunk diagonal at every 64-row
    boundary of a query tile."""
    must, total = list(range(sink + 2)), 0
    for op, n in ops:
        if op == "evict":
            total -= n
            continue
        P = total
        lo = P - recent
        must += [P - 2, P - 1, P, P + 1, lo - 1, lo, lo + 1]
        w = sink + (lo - sink) // recent * recent if lo > sink else sink
        must += [w - 1, w, w + recent - 1, w + recent]
        for e in range(max(0, P - 256) // 64 * 64, P + 1, 64):
            must += [e - 1, e, e + 1]
        for r in range(64, n + 1, 64):
            must += [P + r - 1, P + r, P + r + 1]
        must += [P + n - 1]
        total += n
    return must


def _run(ops, Hq=8, Hkv=2, nf=1, B=1, sink=4, recent=12, dtype=torch.bfloat16, kv_format="same", must=None,
         force_mma=False, fused=True, stage_cap=64, npos=None, what=""):
    """ops: ("chunk", S) | ("fill", N) | ("evict", n), on a one-layer cache."""
    total = mx = 0
    for op, n in ops:
        total = total + n if op != "evict" else total - n
        mx = max(mx, total)
    npos = npos or mx
    lab = _labels(B, npos, must if must is not None else _schedule_must(ops, sink, recent))
    cen = Census(Hq, Hkv, [nf], B, mx + 8, sink, recent, dtype, lab, kv_format=kv_format, stage_cap=stage_cap)
    for op, n in ops:
        if op == "chunk":
            cen.chunk(0, n, force_mma=force_mma, fused=fused, what=what)
        elif op == "fill":
            cen.fill(0, n)
        else:
            cen.evict(n)
    torch.cuda.synchronize()
    return cen


# ------------------------------------------------------------------------------------------------------------------
# wgmma prefill (chunks >= 128, W <= 2048) and the same schedules on duo_attention_mma (force_mma)
# ------------------------------------------------------------------------------------------------------------------
_GEOMS = [  # (Hq, Hkv, n_full, sink, recent): G 1 / 4 / 6, n_full none / some / all, W 5 / 320 / 2048
    (4, 4, 2, 1, 4), (16, 4, 0, 64, 256), (12, 2, 2, 64, 1984), (8, 2, 1, 64, 256), (6, 1, 1, 1, 4),
    (8, 8, 8, 64, 256),
]


@pytest.mark.parametrize("force_mma", [False, True], ids=["wgmma", "mma"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [128, 129, 255, 383])
def test_first_chunk(S, dtype, force_mma):
    Hq, Hkv, nf, sink, recent = _GEOMS[[128, 129, 255, 383].index(S)]
    _run([("chunk", S), ("chunk", 1)], Hq, Hkv, nf, sink=sink, recent=recent, dtype=dtype, force_mma=force_mma,
         stage_cap=S, what="first chunk")


@pytest.mark.parametrize("force_mma", [False, True], ids=["wgmma", "mma"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("past", [127, 128, 129, 4097])
@pytest.mark.parametrize("S", [128, 200, 256, 1000])
def test_continuation_chunk(S, past, dtype, force_mma):
    i = [128, 200, 256, 1000].index(S) + [127, 128, 129, 4097].index(past)
    Hq, Hkv, nf, sink, recent = _GEOMS[i % len(_GEOMS)]
    ops = [("chunk", past), ("chunk", S)] if past < 4097 else [("fill", past), ("chunk", S)]
    _run(ops, Hq, Hkv, nf, sink=sink, recent=recent, dtype=dtype, force_mma=force_mma, stage_cap=max(S, past),
         what="continuation")


@pytest.mark.parametrize("force_mma", [False, True], ids=["wgmma", "mma"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("sink,recent", [(1, 4), (64, 256), (64, 1984)], ids=["W5", "W320", "W2048"])
def test_streaming_states_batch2(sink, recent, dtype, force_mma):
    """B = 2 on disjoint dimension ranges through every ring state: total < sink, sink <= total < W, wrapped
    (lo != sink), right after evict_last(1) and evict_last(3)."""
    W = sink + recent
    ops = [("chunk", 130) if W > 130 else ("chunk", 1), ("chunk", 128), ("chunk", max(130, W - 200)),
           ("chunk", W + 5), ("chunk", 1), ("evict", 1), ("chunk", 128), ("chunk", 1), ("evict", 3), ("chunk", 200),
           ("chunk", 2)]
    if sink >= 64:
        ops = [("chunk", sink // 2)] + ops[1:]  # total < sink on the next (wgmma) call
    _run(ops, 16, 4, 2, B=2, sink=sink, recent=recent, dtype=dtype, force_mma=force_mma, stage_cap=max(W + 5, 200),
         what="streaming states")


def _bench_must(past, S, sink, recent):
    must = list(range(0, sink + 2)) + [past - 1, past, past + S - 1]
    lo = past - recent
    must += [lo - 1, lo, lo + 1]
    for e in range(0, past, 4096):          # tile edges along the cache (sampled)
        must += [e - 1, e, e + 1]
    for e in range(past - 1024, past + 1, 64):
        must += [e - 1, e, e + 1]
    for r in range(0, S + 1, 64):           # the chunk diagonal at every 64-row boundary of the query tiles
        must += [past + r - 1, past + r, past + r + 1]
    return must


def test_benchmarked_shape():
    """The last 32,768-token chunk of the 128K prefill over 98,304 cached tokens, n_full = 4 of 8 (bf16)."""
    past, S, sink, recent = 98304, 32768, 64, 256
    _run([("fill", past), ("chunk", S)], 32, 8, 4, sink=sink, recent=recent, must=_bench_must(past, S, sink, recent),
         stage_cap=S, what="benchmarked shape")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [128, 300])
def test_wide_window_mma_fallback(S, dtype):
    """W = 2049 > TC_MAX_W: a chunk of >= 128 tokens takes duo_attn_mma_kernel<T,1> over a ring of > 2048 slots."""
    _run([("chunk", 700), ("chunk", 1500), ("chunk", S), ("chunk", 1), ("evict", 1), ("chunk", S)], 8, 2, 1,
         sink=64, recent=1985, dtype=dtype, stage_cap=1500, what="W 2049")


# ------------------------------------------------------------------------------------------------------------------
# decode-sized and small chunks: duo_attn_mma_kernel<T,1> / <T,4> unfused, duo_decode_fused
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S,Hq", [(5, 8), (17, 8), (64, 8), (127, 8), (2, 8), (4, 8), (16, 2)])
def test_small_chunks_unfused(S, Hq, dtype):
    _run([("chunk", 300), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S)], Hq, 2, 1,
         sink=16, recent=48, dtype=dtype, fused=False, stage_cap=300, what="unfused")


def _split_contexts(target, nf, ns, B=1):
    """Three contexts whose retrieval key range ends at, one before and one after a split boundary of the
    fused decode partition (equal lengths: ragged_partition)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    out = []
    n = target
    for _ in range(8):
        kps = ragged_partition([n] * B, nf, ns, sm)["keys_per_split"]
        n2 = max(1, round(target / kps)) * kps
        if n2 == n:
            break
        n = n2
    kps = ragged_partition([n] * B, nf, ns, sm)["keys_per_split"]
    for d in (0, -1, 1):
        if ragged_partition([n + d] * B, nf, ns, sm)["keys_per_split"] == kps:
            out.append(n + d)
    return out, kps


def _decode_must(N, kps, sink, recent):
    must = list(range(0, sink + 2)) + [N - 2, N - 1, N]
    lo = N - recent
    must += [lo - 1, lo, lo + 1]
    for e in range(0, N + 1, kps):
        must += [e - 1, e, e + 1]
    for e in range(max(0, N - 512), N + 1, 64):
        must += [e - 1, e, e + 1]
    return must


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S,Hq", [(1, 8), (2, 8), (4, 8), (16, 2)])
def test_fused_decode_small_context(S, Hq, dtype):
    _run([("chunk", 5), ("chunk", S), ("chunk", 200), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S),
          ("evict", 3), ("chunk", S)], Hq, 2, 1, sink=16, recent=48, dtype=dtype, stage_cap=200, what="fused")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("target", [20000, 131072])
def test_fused_decode_at_split_boundaries(target, dtype):
    Hq, Hkv, nf, sink, recent = 16, 4, 2, 64, 256
    ctxs, kps = _split_contexts(target, nf, Hkv - nf)
    assert len(ctxs) >= 2, ctxs
    for N in ctxs:
        S = 1 if N % 2 else 4
        _run([("fill", N), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S)], Hq, Hkv, nf, sink=sink,
             recent=recent, dtype=dtype, must=_decode_must(N, kps, sink, recent), npos=N + 3 * S,
             what=f"fused decode N={N} kps={kps}")


# ------------------------------------------------------------------------------------------------------------------
# INT4 caches: dec8 (G S <= 8), <4> (8 < G S <= 16), <1> (17-127, and W > 2048 with S >= 128), the >= 128 image path
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [1, 2, 3, 4, 17, 64])
def test_int4_small_chunks(S, dtype):
    _run([("chunk", 300), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S), ("chunk", 130), ("chunk", S)],
         8, 2, 1, sink=16, recent=48, dtype=dtype, kv_format="int4", stage_cap=300, what="int4")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_int4_decode_at_split_boundaries(dtype):
    Hq, Hkv, nf, sink, recent = 8, 2, 1, 64, 256
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY
    n = 20000
    kps = ragged_partition([n + 1], nf, Hkv - nf, sm, **INT4_RAGGED_POLICY)["keys_per_split"]
    N0 = round(n / kps) * kps - 1  # full_len + q_len keys end at a boundary for one token
    for N in (N0, N0 - 1, N0 + 1):
        _run([("fill", N), ("chunk", 1), ("chunk", 2), ("evict", 1), ("chunk", 1)], Hq, Hkv, nf, sink=sink,
             recent=recent, dtype=dtype, kv_format="int4", must=_decode_must(N, kps, sink, recent),
             what=f"int4 dec8 N={N} kps={kps}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [128, 300])
def test_int4_wide_window_takes_int4_kernel(S, dtype):
    _run([("chunk", 700), ("chunk", 1500), ("chunk", S), ("chunk", 1), ("evict", 1), ("chunk", S)], 8, 2, 1,
         sink=64, recent=1985, dtype=dtype, kv_format="int4", stage_cap=1500, what="int4 W 2049")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_int4_image_two_layers(dtype):
    """Chunks >= 128 over an INT4 cache attend a 16-bit image shared by all layers: two layers with different n_full
    and lengths, every image row poisoned before a call, so rows past a call's range (another layer's leftovers)
    must stay invisible."""
    Hq, Hkv, sink, recent = 8, 4, 16, 240
    lab = _labels(1, 3000)
    cen = Census(Hq, Hkv, [3, 1], 1, 3000, sink, recent, dtype, lab, kv_format="int4", stage_cap=1200)
    cen.chunk(0, 1200, what="image")   # first call: raw K/V
    cen.chunk(1, 300, what="image")
    cen.chunk(0, 600, what="image")    # layer 0's rows now fill the image to 1800
    cen.chunk(1, 200, image_poison=True, what="image")
    cen.chunk(1, 1, what="image")
    cen.evict(3)
    cen.chunk(0, 128, image_poison=True, what="image")
    cen.chunk(1, 129, image_poison=True, what="image")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# ragged batches: duo_decode_ragged, duo_decode_ragged_int4, duo_decode_ragged_pooled (both formats)
# ------------------------------------------------------------------------------------------------------------------
def _ragged_must(lengths, nf, ns, int4, sink, recent, S):
    """Probe positions of every row: sinks, ends, lo +- 1 and the split edges of the ragged partition of these
    lengths (16-bit: full_len keys per row; INT4: full_len + q_len)."""
    from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    keys = [n + S for n in lengths] if int4 else list(lengths)
    kps = ragged_partition(keys, nf, ns, sm, **(INT4_RAGGED_POLICY if int4 else {}))["keys_per_split"]
    must = []
    for N in lengths:
        must += _decode_must(N, kps, sink, recent)
    return must


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
@pytest.mark.parametrize("kv_format", ["same", "int4"])
@pytest.mark.parametrize("S", [1, 2])
def test_ragged_decode(S, kv_format, pooled, dtype):
    """Rows at different lengths on their own dimension ranges (a neighbour's dimensions must read 0); pooled: the
    rows' regions, the pool headroom and the region a resize_row frees are poisoned and must stay unread and
    unwritten."""
    Hq, Hkv, nf, sink, recent = 8, 4, 2, 16, 48
    int4 = kv_format == "int4"
    lengths = [6000, 0, 700]       # row 1 is prefilled through row(1).attend
    caps = [6100, 400, 800]
    lab = _labels(3, 6200, _ragged_must([6000, 130, 700], nf, Hkv - nf, int4, sink, recent, S))
    cen = Census(Hq, Hkv, [nf], 3, caps if pooled else max(caps), sink, recent, dtype, lab, kv_format=kv_format,
                 stage_cap=130, ragged=True, pool_size=sum(caps) + 2048 if pooled else None)
    for b, N in enumerate(lengths):
        if N:
            cen.fill(0, N, rows=[b])
    cen.chunk(0, 130, row=1, what="ragged prefill")
    for _ in range(2):
        cen.chunk(0, S, what="ragged")
    cen.evict(1)
    cen.chunk(0, S, what="ragged after evict_last(1)")
    cen.evict(3, row=2)
    cen.chunk(0, S, what="ragged after row(2).evict_last(3)")
    if pooled:
        cen.clear_and_resize(1, 900)
        cen.fill(0, 600, rows=[1])
        cen.chunk(0, S, what="ragged after resize_row")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# DuoDecodeGraph replay: the occupancy comes from device memory
# ------------------------------------------------------------------------------------------------------------------
class _AttentionOnly:
    """Stands in for the patched model under DuoDecodeGraph: every layer attends the one token of ``qkv`` (refilled
    before each replay) into ``out``, then the device occupancy advances, as the model driver does."""

    def __init__(self, cache):
        B, Hq, Hkv = cache.batch_size, cache.num_heads, cache.num_kv_heads
        n = B * Hq * D
        self.qkv = torch.zeros(B, 1, (Hq + 2 * Hkv) * D, dtype=cache.dtype, device=cache.device)
        self.buf = torch.full((n + 256,), float("nan"), dtype=cache.dtype, device=cache.device)
        self.out = self.buf[:n].view(B, 1, Hq, D)

    def __call__(self, input_ids, position_ids, past_key_values, use_cache):
        from types import SimpleNamespace

        c = past_key_values
        for l in range(c.num_layers):
            c.attend(l, self.qkv, None, None, _C.ROPE_NONE, self.out)
        c.advance_device(1)
        return SimpleNamespace(logits=self.out)


def _graph_schedule(cen, what):
    from duo_attention_b200.graph import DuoDecodeGraph

    m = _AttentionOnly(cen.cache)
    g = DuoDecodeGraph(m, cen.cache)
    run = (g, m.qkv, m.buf)
    for _ in range(3):
        cen.chunk(0, 1, graph=run, what=what)
    cen.evict(1)
    cen.chunk(0, 1, graph=run, what=what + " after evict_last(1)")
    cen.chunk(0, 1, graph=run, what=what)
    cen.evict(3)
    cen.chunk(0, 1, graph=run, what=what + " after evict_last(3)")
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_graph_replay_fused_decode(dtype):
    Hq, Hkv, nf, sink, recent = 16, 4, 2, 16, 48
    N = 9000
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    kps = ragged_partition([N], nf, Hkv - nf, sm)["keys_per_split"]
    lab = _labels(1, N + 16, _decode_must(N, kps, sink, recent))
    cen = Census(Hq, Hkv, [nf], 1, N + 16, sink, recent, dtype, lab)
    cen.fill(0, N)
    _graph_schedule(cen, "graph fused")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_graph_replay_ragged_int4(dtype):
    Hq, Hkv, nf, sink, recent = 8, 4, 2, 16, 48
    lengths = [5000, 300]
    lab = _labels(2, 5100, _ragged_must(lengths, nf, Hkv - nf, True, sink, recent, 1))
    cen = Census(Hq, Hkv, [nf], 2, 5100, sink, recent, dtype, lab, kv_format="int4", ragged=True)
    for b, N in enumerate(lengths):
        cen.fill(0, N, rows=[b])
    _graph_schedule(cen, "graph ragged int4")
