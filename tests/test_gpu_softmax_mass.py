"""How much weight every attention kernel gives each key: the visibility census with unequal logits, held to the fp64
softmax and the rounding-error bound of tests/softmax_bound.py.

tests/test_gpu_visibility_census.py gives every probe the same logit, so every tile, warp, split-KV partial and merge
group sees the same row maximum and a wrong but consistent reference cancels.  Here the same census runs with

* K = a_p u_h, a_p = 15 j_p / 128 (j_p = 1..17): exact in bf16 and fp16, and K1 (INT4) quantises it exactly
  (scale j/64, zero -a), so every kernel reads the same keys; q = +-A_g u_h per query head, the first head of each
  GQA group positive (poison has a negative logit for the negative heads);
* every position a probe whose V is one-hot on a REGION label: the split index (or 64-key tile) of its position, the
  sinks on a dimension of their own, batch rows on disjoint dimension ranges, dimension 127 poison.  Output dimension
  r is the softmax mass of the regions labelled r, which is what the rescales and merges compute;
* logit patterns: rising and falling ramps, sawtooth with the period of the tile or split length +- 1, isolated peaks
  at split / tile / ring boundaries, a 183-log2 gap (earlier partials contribute exactly 0), mirror-image heads in
  one group, a different pattern on each batch row.

Every element is within the bound (unlit dimensions and poison exactly 0); the worst err / bound of every call is
logged through ``parity.record``.  The INT4 kernels are held to the same bound (P' = fp16(p s) rounding): they recentre
the V codes to c - 8 before the truncating tensor-core accumulation (DESIGN §4), which with a 1024 offset lost about
one ulp of 1024 sum P' per 16-key step, an absolute error on every dimension that this census exposed.  Also here:
the shared-prefix fold of duo_decode_ragged_shared and the partial merge of duo_merge_partials, and INT4 on Gaussian
data at the benchmarked lengths with the keys per accumulator chain named.
"""
import math

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import INT4_RAGGED_POLICY, DuoKVCache, ragged_partition, ring_slot
from parity import record
from softmax_bound import LOG2E, bound_terms, worst_ratio
from test_gpu_visibility_census import (DTYPES, POISON, Census, _decode_must, _graph_schedule, _schedule_must,
                                        _split_contexts, _u)
from visibility_model import TupleVisibility

pytestmark = pytest.mark.gpu
D = 128
QAMP = [0.5, -0.5, 1.5, 6.0, 0.25, -6.0]   # per head of a GQA group; the first is positive


def _qamp(Hq, Hkv):
    G = Hq // Hkv
    return torch.tensor([QAMP[i % len(QAMP)] for i in range(G)] * Hkv, dtype=torch.float32)


def _region_labels(B, npos, gran, sink):
    """[B, npos]: row b owns dimensions [b nd, (b + 1) nd); the sinks light b nd + nd - 1, position p >= sink lights
    b nd + (p // gran) % (nd - 1)."""
    nd = POISON // B
    p = torch.arange(npos)
    reg = torch.where(p < sink, nd - 1, (p // gran) % (nd - 1))
    return torch.stack([b * nd + reg for b in range(B)])


def _levels(pattern, npos, period, peaks):
    """K levels a_p = 15 j_p / 128 of one logit pattern over positions [0, npos)."""
    p = torch.arange(npos)
    if pattern == "rise":
        j = 1 + (16 * p) // npos
    elif pattern == "fall":
        j = 17 - (16 * p) // npos
    elif pattern in ("saw+1", "saw-1"):
        per = max(2, period + (1 if pattern == "saw+1" else -1))
        j = 1 + ((p % per) * 16) // per
    elif pattern == "peaks":
        j = torch.full((npos,), 3)
        for i, e in enumerate(sorted({e for e in peaks if 0 <= e < npos})):
            j[e] = (17, 11, 14, 8)[i % 4]
    elif pattern == "gap":                 # qamp 6: 16 levels = 183 log2 units above the first half
        j = torch.where(p < npos // 2, 1, 17)
    elif pattern == "gap_rev":
        j = torch.where(p < npos // 3, 17, 1)
    else:
        raise ValueError(pattern)
    return j.to(torch.float32) * (15.0 / 128.0)


class MassCensus(Census):
    """The census with levels and query amplitudes, checked against fp64 softmax weights within the bound."""

    def _check(self, out, rows, chs, l, S, first, force_mma, ctx):
        c = self.cache
        nf = c.num_full_kv_head_list[l]
        G, dev = self.G, self.dev
        image = self.int4 and not first and S >= 128 and c.W <= 2048 and not force_mma
        int4_kernel = self.int4 and not first and not image
        p_dtype = torch.float16 if int4_kernel else self.dtype
        lit = self._lit(S, first, force_mma)
        worst = 0.0
        for i, (b, ch) in enumerate(zip(rows, chs)):
            P = ch.start
            npos = P + S
            pos = torch.arange(npos, device=dev)
            own = (pos[None] >= P) & (pos[None] <= P + torch.arange(S, device=dev)[:, None])     # [S, npos]
            lev = self.level[b, :npos].double()
            v = torch.zeros(npos, D, dtype=torch.float64, device=dev)
            v[pos, self.lab[b, :npos]] = lit
            for h in range(self.Hkv):
                base = torch.zeros(npos, dtype=torch.bool, device=dev)
                for a, e in (ch.full if h < nf else ch.stream):
                    base[a:e] = True
                mask = base[None] | own
                qa = self.qamp[h * G : (h + 1) * G].to(dev, torch.float64)
                l2 = (qa[:, None] * lev[None] * (D * D ** -0.5 * LOG2E))[None].expand(S, G, npos)
                l2 = l2.masked_fill(~mask[:, None], -math.inf).reshape(S * G, npos)
                # INT4 kernels: P' = fp16(p s) with s = lit / 15, the K2 scale of the one-hot rows
                want, bound, _ = bound_terms(l2, v, p_dtype, self.dtype, p_scale=torch.full(
                    (npos,), lit / 15, dtype=torch.float64, device=dev) if int4_kernel else None)
                got = out[i, :, h * G : (h + 1) * G].reshape(S * G, D).double()
                dark = want == 0
                bad = dark & (got != 0)
                if bad.any():
                    r_, d = torch.nonzero(bad)[0].tolist()
                    raise AssertionError(f"{ctx}: kv head {h} row {r_ // G} head {r_ % G} of batch row {b} lights "
                                         f"dimension {d} ({'POISON' if d == POISON else 'unlit'}) = "
                                         f"{got[r_, d].item():.6g}")
                r = worst_ratio(got[:, ~(dark.all(0))], want[:, ~(dark.all(0))], bound[:, ~(dark.all(0))])
                if not r <= 1.0:
                    err = (got - want).abs() / bound
                    r_, d = divmod(int(torch.nan_to_num(err, nan=math.inf).argmax()), D)
                    raise AssertionError(f"{ctx}: kv head {h} row {r_ // G} head {r_ % G} (q amp "
                                         f"{qa[r_ % G].item()}) of batch row {b}, dimension {d}: got "
                                         f"{got[r_, d].item():.8g}, want {want[r_, d].item():.8g}, bound "
                                         f"{bound[r_, d].item():.3g} (err / bound {r:.3f})")
                worst = max(worst, r)
        record("softmax_mass", what=ctx, dtype=str(self.dtype), int4_kernel=int4_kernel,
               worst_err_over_bound=worst)


def _mass_run(ops, Hq, Hkv, nf, patterns, gran, sink, recent, dtype, kv_format="same", peaks=(), force_mma=False,
              fused=True, stage_cap=64, B=1, what=""):
    """ops as in the visibility census's ``_run``; ``patterns``: one per batch row."""
    total = mx = 0
    for op, n in ops:
        total = total + n if op != "evict" else total - n
        mx = max(mx, total)
    npos = mx + 8
    peaks = list(peaks) + _schedule_must(ops, sink, recent)
    lab = _region_labels(B, npos, gran, sink)
    level = torch.stack([_levels(patterns[b], npos, gran, peaks) for b in range(B)])
    cen = MassCensus(Hq, Hkv, [nf], B, npos, sink, recent, dtype, lab, kv_format=kv_format, stage_cap=stage_cap,
                     level=level, qamp=_qamp(Hq, Hkv))
    for op, n in ops:
        if op == "chunk":
            cen.chunk(0, n, force_mma=force_mma, fused=fused, what=f"{what} [{patterns}]")
        elif op == "fill":
            cen.fill(0, n)
        else:
            cen.evict(n)
    torch.cuda.synchronize()
    return cen


PATTERNS = ["rise", "fall", "saw+1", "saw-1", "peaks", "gap", "gap_rev"]


# ---- 16-bit caches ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force_mma", [False, True], ids=["wgmma", "mma"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_prefill_chunks(pattern, dtype, force_mma):
    """wgmma prefill (chunks >= 128, W <= 2048) and duo_attention_mma: a first chunk, a continuation over 4,097
    cached tokens, B = 2 with the mirror pattern on row 1."""
    pats = [pattern, {"rise": "fall", "fall": "rise", "gap": "gap_rev"}.get(pattern, "rise")]
    _mass_run([("chunk", 200), ("chunk", 129), ("chunk", 1000)], 16, 4, 2, pats, 64, 64, 256, dtype,
              force_mma=force_mma, stage_cap=1000, B=2, what="prefill")
    _mass_run([("fill", 4097), ("chunk", 300)], 8, 2, 1, [pattern], 64, 64, 256, dtype, force_mma=force_mma,
              stage_cap=300, what="continuation over 4097")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pattern", ["rise", "fall", "saw+1", "peaks", "gap"])
def test_wide_window_mma_fallback(pattern, dtype):
    """W = 2049 > TC_MAX_W: duo_attn_mma_kernel<T,1> over a ring of more than 2048 slots."""
    _mass_run([("chunk", 700), ("chunk", 1500), ("chunk", 300), ("chunk", 1), ("evict", 1), ("chunk", 128)], 8, 2,
              1, [pattern], 64, 64, 1985, dtype, stage_cap=1500, what="W 2049")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S,Hq", [(5, 8), (2, 8), (16, 2)], ids=["T1", "T4", "T4-mha"])
def test_small_chunks_unfused(S, Hq, dtype):
    for pattern in ("rise", "fall", "saw-1", "peaks"):
        _mass_run([("chunk", 300), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S)], Hq, 2, 1, [pattern],
                  16, 16, 48, dtype, fused=False, stage_cap=300, what="unfused")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("target", [20000, 131072])
def test_fused_decode_at_split_boundaries(target, dtype):
    """duo_decode_fused with the region label = the split index: a weight error in one split or merge level moves
    that split's dimension."""
    Hq, Hkv, nf, sink, recent = 16, 4, 2, 64, 256
    ctxs, kps = _split_contexts(target, nf, Hkv - nf)
    pats = ["rise", "fall", "peaks", "saw+1", "gap"] if target == 20000 else ["fall", "peaks"]
    for N in ctxs[:2]:
        for pattern in pats:
            S = 1 if N % 2 else 4
            _mass_run([("fill", N), ("chunk", S), ("chunk", S)], Hq, Hkv, nf, [pattern], kps, sink, recent, dtype,
                      peaks=_decode_must(N, kps, sink, recent), what=f"fused decode N={N} kps={kps}")


# ---- INT4 caches --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("S", [1, 3, 17, 130], ids=["dec8", "I4", "I1", "image"])
def test_int4_kernels(S, dtype):
    for pattern in ("rise", "fall", "saw+1", "peaks", "gap"):
        _mass_run([("chunk", 300), ("chunk", S), ("chunk", S), ("evict", 1), ("chunk", S)], 8, 2, 1, [pattern], 64,
                  16, 240, dtype, kv_format="int4", stage_cap=300, what="int4")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_int4_dec8_at_split_boundaries(dtype):
    Hq, Hkv, nf, sink, recent = 8, 2, 1, 64, 256
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = 20000
    kps = ragged_partition([n + 1], nf, Hkv - nf, sm, **INT4_RAGGED_POLICY)["keys_per_split"]
    N = round(n / kps) * kps - 1
    for pattern in ("rise", "fall", "peaks", "saw-1"):
        _mass_run([("fill", N), ("chunk", 1), ("chunk", 2)], Hq, Hkv, nf, [pattern], kps, sink, recent, dtype,
                  kv_format="int4", peaks=_decode_must(N, kps, sink, recent), what=f"int4 dec8 N={N} kps={kps}")


# ---- ragged batches and graph replay -------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pooled", [False, True], ids=["uniform", "pooled"])
@pytest.mark.parametrize("kv_format", ["same", "int4"])
def test_ragged_decode(kv_format, pooled, dtype):
    """Rows at different lengths, each with its own pattern and dimension range."""
    Hq, Hkv, nf, sink, recent = 8, 4, 2, 16, 48
    lengths, caps = [6000, 2500, 700], [6100, 2600, 800]
    pats = ["rise", "peaks", "fall"]
    npos = max(caps)
    lab = _region_labels(3, npos, 512, sink)
    level = torch.stack([_levels(p, npos, 512, _decode_must(N, 512, sink, recent)) for p, N in zip(pats, lengths)])
    cen = MassCensus(Hq, Hkv, [nf], 3, caps if pooled else npos, sink, recent, dtype, lab, kv_format=kv_format,
                     stage_cap=64, ragged=True, pool_size=sum(caps) + 2048 if pooled else None, level=level,
                     qamp=_qamp(Hq, Hkv))
    for b, N in enumerate(lengths):
        cen.fill(0, N, rows=[b])
    for S in (1, 2, 1):
        cen.chunk(0, S, what=f"ragged {kv_format}")
    cen.evict(1)
    cen.chunk(0, 1, what="ragged after evict_last(1)")
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_graph_replay_fused_decode(dtype):
    Hq, Hkv, nf, sink, recent = 16, 4, 2, 16, 48
    N = 9000
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    kps = ragged_partition([N], nf, Hkv - nf, sm)["keys_per_split"]
    lab = _region_labels(1, N + 16, kps, sink)
    level = _levels("saw+1", N + 16, kps, [])[None]
    cen = MassCensus(Hq, Hkv, [nf], 1, N + 16, sink, recent, dtype, lab, level=level, qamp=_qamp(Hq, Hkv))
    cen.fill(0, N)
    _graph_schedule(cen, "graph fused")


# ---- INT4 on Gaussian data at the benchmarked lengths ---------------------------------------------------------------
def _quant(x16, lib):
    n = x16.shape[0]
    p = torch.empty(n, D // 2, dtype=torch.uint8, device=x16.device)
    s = torch.empty(n, dtype=torch.float16, device=x16.device)
    z = torch.empty(n, dtype=torch.float16, device=x16.device)
    _C.check(lib.duo_quant_int4(x16.data_ptr(), D, n, p.data_ptr(), s.data_ptr(), z.data_ptr(),
                                torch.cuda.current_stream().cuda_stream))
    return p, s, z


def _deq(t, name, h, idx):
    """(s c + z, s c, s): fp64 [n, D], [n, D], [n] of rows ``idx`` of head h of ``t[name]`` (codes: high nibble =
    even dimension)."""
    pk = t[name][0, h, idx].long()
    c = torch.stack([pk >> 4, pk & 15], -1).reshape(pk.shape[0], D).double()
    s = t[name + "_scale"][0, h, idx].double()[:, None]
    z = t[name + "_zero"][0, h, idx].double()[:, None]
    return c * s + z, c * s, s[:, 0]


REAL = {  # name: (N, S, sink, recent, chain): chain = keys one warp's accumulator holds, from the launch plan
    "dec8_131072": (131072, 1, 64, 256, "dec8: keys_per_split / 4 (retrieval), at most (W + 1) / 4 (streaming)"),
    "dec8_1048576": (1048576, 1, 64, 256, "dec8: keys_per_split / 4 (retrieval), at most (W + 1) / 4 (streaming)"),
    "I4_20000": (20000, 3, 64, 256, "<4>: at most a quarter of the visible keys"),
    "I1_20000": (20000, 5, 64, 256, "<1>: at most every visible key"),
    "ring_W2112": (20000, 1, 64, 2048, "dec8 streaming CTA: (W + 1) / 4 = 528"),
    "ring_W2112_S130": (20000, 130, 64, 2048, "<1> over the ring: at most W + S = 2242"),
}


@pytest.mark.parametrize("sd", [1.0, 3.0])
@pytest.mark.parametrize("case", list(REAL))
def test_int4_gaussian_data(case, sd):
    """Gaussian K / V quantised by duo_quant_int4, q so that the logit sd is ``sd``; every head against fp64 over
    the dequantised cache, within the bound; the keys per accumulator chain of the launch plan are logged and named
    on failure.  Also logs the RMS
    error of flash_attn_func on the fp16 image of the same cache, when it is installed."""
    N, S, sink, recent, chain = REAL[case]
    dev = torch.device("cuda:0")
    dtype = torch.float16
    Hq, Hkv, nf = 8, 2, 1
    G = Hq // Hkv
    g = torch.Generator(device=dev).manual_seed(int(sd) * 7 + N)
    cache = DuoKVCache(1, Hq, Hkv, D, [nf], 1, N + S + 8, sink, recent, dtype, dev, stage_cap=max(64, S),
                       kv_format="int4")
    lib, t = cache.lib, cache.tensors[0]
    model = TupleVisibility(sink, recent)
    model.chunk(N)
    live = model.stream_live()
    slots = torch.tensor([ring_slot(p, sink, recent) for p in live], device=dev)
    for name, rows in (("full_k", None), ("full_v", None), ("ring_k", slots), ("ring_v", slots)):
        for a in range(0, N if rows is None else len(live), 1 << 16):
            n = min(1 << 16, (N if rows is None else len(live)) - a)
            p, s, z = _quant(torch.randn(n, D, generator=g, device=dev, dtype=torch.float32).half(), lib)
            idx = torch.arange(a, a + n, device=dev) if rows is None else rows[a : a + n]
            t[name][0, 0, idx], t[name + "_scale"][0, 0, idx], t[name + "_zero"][0, 0, idx] = p, s, z
    cache.kv_seq_len_list[0] = cache.total_list[0] = N
    cache.lo_list[0] = max(sink, N - recent)
    cache.sync_device_state()
    ring_before = {k: v.clone() for k, v in t.items() if k.startswith("ring")}
    qkv = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g, device=dev).to(dtype)
    qkv[..., : Hq * D] *= sd
    out = torch.empty(1, S, Hq, D, dtype=dtype, device=dev)
    cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)
    ch = model.chunk(S)
    q = qkv[0, :, : Hq * D].view(S, Hq, D).double()
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    worst, fa_rms, our_rms, chains = 0.0, None, 0.0, {}
    for h in range(Hkv):
        if h < nf:
            rows = torch.arange(N + S, device=dev)
            k = _deq(t, "full_k", 0, rows)[0]
            v, r, s_v = _deq(t, "full_v", 0, rows)
            posv = rows
        else:
            old = [p for a, e in ch.stream for p in range(a, e)]
            so = torch.tensor([ring_slot(p, sink, recent) for p in old], device=dev)
            sn = torch.tensor([ring_slot(p, sink, recent) for p in range(N, N + S)], device=dev)
            k = torch.cat([_deq(ring_before, "ring_k", 0, so)[0], _deq(t, "ring_k", 0, sn)[0]])
            v, r, s_v = (torch.cat(x) for x in zip(_deq(ring_before, "ring_v", 0, so), _deq(t, "ring_v", 0, sn)))
            posv = torch.tensor(old + list(range(N, N + S)), device=dev)
        mask = (posv[None] <= (N + torch.arange(S, device=dev))[:, None]).repeat_interleave(G, 0)   # [S G, n]
        qh = q[:, h * G : (h + 1) * G].reshape(S * G, D)
        l2 = ((qh @ k.T) * (D ** -0.5 * LOG2E)).masked_fill(~mask, -math.inf)
        want, bound, _ = bound_terms(l2, v, torch.float16, dtype, r, s_v)
        # keys one warp accumulates: dec8 retrieval CTAs give each warp 32 keys of every 128-key tile of a split;
        # the dec8 streaming CTA and <4> a quarter of what the row sees (at most); <1> everything (at most)
        n_vis = mask.sum(-1, keepdim=True)
        if S * G <= 8 and h < nf:
            n = torch.clamp(n_vis, max=ragged_partition([N + S], nf, Hkv - nf, sm, **INT4_RAGGED_POLICY)
                            ["keys_per_split"] // 4)
        elif S * G <= 16:
            n = (n_vis + 3) // 4
        else:
            n = n_vis
        chains[h] = int(n.max())
        got = out[0, :, h * G : (h + 1) * G].reshape(S * G, D).double()
        worst = max(worst, worst_ratio(got, want, bound))
        our_rms = max(our_rms, float(((got - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt()))
        try:
            from flash_attn import flash_attn_func
        except ImportError:
            flash_attn_func = None
        if flash_attn_func is not None and S == 1:
            fa = flash_attn_func(qh.half().view(1, S * G, 1, D), k.half()[None, :, None],
                                 v.half()[None, :, None], causal=False).view(S * G, D).double()
            e = float(((fa - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt())
            fa_rms = e if fa_rms is None else max(fa_rms, e)
        del k, v, r
    record("int4_gaussian", what=case, sd=sd, chain=chain, chain_keys=chains, worst_err_over_bound=worst,
           rel_rms=our_rms, fa2_image_rel_rms=fa_rms)
    assert worst <= 1.0, f"{case} sd {sd} ({chain}; keys per chain {chains}): worst err / bound {worst:.3f}"


# ---- duo_merge_partials: partials of unequal weight ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pattern", ["rise", "fall", "peaks", "gap"])
def test_merge_partials(pattern, dtype):
    """duo_merge_partials (the head-parallel / tensor-parallel partial merge) over 2-16 partials whose log-sum-exps
    follow a pattern; partial s holds o = e_s, so output dimension s is the weight the merge gives partial s.  The
    merge rounds no P: the bound is the logit and output-rounding terms."""
    dev = torch.device("cuda:0")
    tokens, heads = 3, 8
    for n in (2, 5, 16):
        s = torch.arange(n, dtype=torch.float64, device=dev)
        lse = {"rise": 3.0 * s, "fall": -3.0 * s, "peaks": torch.where(s % 3 == 1, 9.0, 0.0) - 0.5 * s,
               "gap": torch.where(s < n // 2, 0.0, 160.0)}[pattern]
        lse = lse[:, None, None] + torch.tensor([0.0, 0.5, -1.25], device=dev)[None, :, None] * (1 + s[:, None, None])
        lse = lse.expand(n, tokens, heads).clone()
        lse[:, :, 1::2] *= -1                                   # mirror-image heads
        po = torch.zeros(n, tokens, heads, D, device=dev)
        po[torch.arange(n), :, :, torch.arange(n)] = 1.0
        pl = lse.float()
        out = torch.empty(tokens, heads, D, dtype=dtype, device=dev)
        _C.check(_C.load().duo_merge_partials(po.data_ptr(), pl.data_ptr(), n, tokens, heads, heads, out.data_ptr(),
                                              0 if dtype == torch.bfloat16 else 1,
                                              torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        l2 = pl.double().permute(1, 2, 0).reshape(tokens * heads, n)
        want, _, terms = bound_terms(l2, po[:, 0, 0].double(), dtype, dtype)
        bound = terms["logit"] + terms["out_round"]
        got = out.reshape(tokens * heads, D).double()
        assert (got[want == 0] == 0).all(), f"{pattern} n={n}: a dimension no partial holds is lit"
        r = worst_ratio(got, want, bound)
        record("softmax_mass", what=f"merge_partials {pattern} n={n}", dtype=str(dtype), worst_err_over_bound=r)
        assert r <= 1.0, f"{pattern} n={n}: worst err / bound {r:.3f}"


# ---- duo_decode_ragged_shared: the shared-prefix fold ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("pattern", ["prefix_high", "own_high", "rise"])
@pytest.mark.parametrize("q_len", [1, 2])
def test_shared_prefix_fold(q_len, pattern, dtype):
    """Row 0 holds a prompt, rows 1 and 2 fork it (row 2 from row 1) and decode their own tokens: the retrieval heads
    of the forks fold the prefix partial into their own keys (Share::OwnSuffix).  Prefix keys light dimensions by split of
    512 keys, the unshared tail and the decoded keys their own; ``prefix_high``: prefix logits 183 log2 units above
    the own keys (for the q = 6 heads), ``own_high`` the reverse."""
    from duo_attention_b200.kv_cache import DuoRaggedKVCache

    dev = torch.device("cuda:0")
    Hq, Hkv, nf, sink, recent, LA, B = 8, 4, 2, 16, 48, 1300, 3
    G = Hq // Hkv
    room = 128 + 6 * q_len
    cache = DuoRaggedKVCache.from_geometry(1, Hq, Hkv, D, [nf], B, [LA + room, room, room], sink, recent, dtype, dev,
                                           stage_cap=64)
    qamp = _qamp(Hq, Hkv).to(dev)
    uu = _u(Hkv, dev)
    hi, lo = 17 * 15 / 128, 15 / 128
    plev = {"prefix_high": hi, "own_high": lo, "rise": None}[pattern]
    olev = {"prefix_high": lo, "own_high": hi, "rise": None}[pattern]

    def level(p):
        if plev is None:
            return (1 + (16 * p) // (LA + room)) * 15 / 128
        return plev if p < LA else olev

    def label(p, b):
        return (p // 512) % 60 if p < LA // 128 * 128 else 60 + b if p >= LA else 63

    def qkv_of(positions_per_row):
        S = len(positions_per_row[0])
        x = torch.zeros(len(positions_per_row), S, Hq + 2 * Hkv, D, device=dev)
        x[:, :, :Hq] = qamp[:, None] * uu.repeat_interleave(G, 0)
        for i, ps in enumerate(positions_per_row):
            for t, p in enumerate(ps):
                x[i, t, Hq : Hq + Hkv] = level(p) * uu
                x[i, t, Hq + Hkv + torch.arange(Hkv), label(p, i)] = 1.0
        return x.view(len(positions_per_row), S, -1).to(dtype).contiguous()

    hist = [[] for _ in range(B)]     # (level, label) of every position of each row
    out0 = torch.empty(1, LA, Hq, D, dtype=dtype, device=dev)
    cache.row(0).attend(0, qkv_of([list(range(LA))]), None, None, _C.ROPE_NONE, out0)
    hist[0] = [(level(p), label(p, 0)) for p in range(LA)]
    models = [TupleVisibility(sink, recent) for _ in range(B)]
    models[0].chunk(LA)
    cache.share_prefix(0, 1, room)
    cache.share_prefix(1, 2, room)
    assert cache.row_prefix[1] and cache.row_prefix[2] and cache.sharing
    for b in (1, 2):
        hist[b] = list(hist[0])
        models[b].chunk(LA)
    worst = 0.0
    for step in range(3):
        pos = [list(range(LA + step * q_len, LA + (step + 1) * q_len)) for _ in range(B)]
        qkv = qkv_of(pos)
        for b in range(B):
            hist[b] += [(level(p), label(p, b)) for p in pos[b]]
        out = torch.empty(B, q_len, Hq, D, dtype=dtype, device=dev)
        cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)
        for b in range(B):
            ch = models[b].chunk(q_len)
            npos = len(hist[b])
            lev = torch.tensor([h[0] for h in hist[b]], dtype=torch.float64, device=dev)
            v = torch.zeros(npos, D, dtype=torch.float64, device=dev)
            v[torch.arange(npos), torch.tensor([h[1] for h in hist[b]], device=dev)] = 1.0
            for h in range(Hkv):
                mask = torch.zeros(q_len, npos, dtype=torch.bool, device=dev)
                for t in range(q_len):
                    for a, e in ch.intervals(t, h < nf):
                        mask[t, a:e] = True
                qa = qamp[h * G : (h + 1) * G].double()
                l2 = (qa[:, None] * lev[None] * (D * D ** -0.5 * LOG2E))[None].expand(q_len, G, npos)
                l2 = l2.masked_fill(~mask[:, None], -math.inf).reshape(q_len * G, npos)
                want, bound, _ = bound_terms(l2, v, dtype, dtype)
                got = out[b, :, h * G : (h + 1) * G].reshape(q_len * G, D).double()
                assert (got[want == 0] == 0).all(), f"step {step} row {b} kv head {h}: an unlit dimension is lit"
                r = worst_ratio(got, want, bound)
                assert r <= 1.0, f"step {step} row {b} kv head {h} ({pattern}): worst err / bound {r:.3f}"
                worst = max(worst, r)
    record("softmax_mass", what=f"shared prefix {pattern} q_len={q_len}", dtype=str(dtype),
           worst_err_over_bound=worst)
