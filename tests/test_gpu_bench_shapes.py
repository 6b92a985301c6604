"""Parity at the shapes the headline numbers are measured on (bench.py): the wgmma prefill kernel on a
32,768-token chunk over 98,304 cached tokens (the last chunk of the 128K prefill: 4,096 CTAs, up to 1,024 K/V tiles
per CTA) and the INT4 decode kernel at 1,048,576 tokens (~290 key splits per retrieval head).

The CPU oracle cannot finish these sizes in seconds, so the checker is the reference's own GPU attention:
duo_attn/patch/llama.py:374-421 restated with the INSTALLED flash_attn_func on token-major copies of the same
caches (tests/test_gpu_oracle_pin.py pins that library against the oracle at small sizes), plus exact fp64
attention on a sample of query rows, plus the mma.sync kernel family on the same inputs.  INT4 at 1M uses the
size-independent properties of tests/test_gpu_attention.py::test_full_size_decode_properties.
"""
import ctypes as C

import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from parity import ATOL, RTOL, assert_parity, record

pytestmark = pytest.mark.gpu
D = 128


def _filled_cache(Hq, Hkv, n_full, past, chunk, sink, recent, dev, seed):
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, past + chunk + 8, sink, recent, torch.bfloat16, dev,
                       stage_cap=chunk)
    g = torch.Generator(device=dev).manual_seed(seed)
    t = cache.tensors[0]
    for n in ("full_k", "full_v", "ring_k", "ring_v"):
        if t[n].numel():
            t[n].normal_(generator=g)
    cache.kv_seq_len_list[0] = past
    cache.total_list[0] = past
    cache.lo_list[0] = max(sink, past - recent)
    return cache, g


def _fa2_reference(cache, qkv, Hq, Hkv, n_full, past, chunk, sink, recent):
    """llama.py:374-421 with the installed flash_attn_func on token-major views of the SAME cache contents
    (after duo_rope_append has appended / staged the chunk's K and V)."""
    from flash_attn import flash_attn_func

    G = Hq // Hkv
    W = sink + recent
    t = cache.tensors[0]
    q = qkv[..., : Hq * D].view(1, chunk, Hq, D)
    outs = []
    if n_full:
        fk = t["full_k"][0, :, : past + chunk].transpose(0, 1).unsqueeze(0).contiguous()
        fv = t["full_v"][0, :, : past + chunk].transpose(0, 1).unsqueeze(0).contiguous()
        outs.append(flash_attn_func(q[:, :, : n_full * G], fk, fv, causal=True))
        del fk, fv
    if n_full < Hkv:
        # live sink + ring rows in any order (softmax is permutation invariant), then the staged chunk
        rows = torch.cat([torch.arange(0, W, device=qkv.device), torch.arange(W, W + chunk, device=qkv.device)])
        sk = t["ring_k"][0][:, rows].transpose(0, 1).unsqueeze(0).contiguous()
        sv = t["ring_v"][0][:, rows].transpose(0, 1).unsqueeze(0).contiguous()
        outs.append(flash_attn_func(q[:, :, n_full * G :], sk, sv, causal=True))
    return torch.cat(outs, dim=2)


def _exact_rows(cache, qkv, rows, Hq, Hkv, n_full, past, chunk, sink, recent):
    """fp64 attention of a sample of query rows (all heads) against the same cache contents: no rounding anywhere."""
    G = Hq // Hkv
    W = sink + recent
    t = cache.tensors[0]
    q = qkv[0, rows, : Hq * D].view(len(rows), Hq, D).double()
    out = torch.empty(len(rows), Hq, D, dtype=torch.float64, device=qkv.device)
    for h in range(Hq):
        kvh = h // G
        if kvh < n_full:
            k = t["full_k"][0, kvh, : past + chunk].double()
            v = t["full_v"][0, kvh, : past + chunk].double()
            limit = past + rows  # last visible key per row
        else:
            k = t["ring_k"][0, kvh - n_full, : W + chunk].double()
            v = t["ring_v"][0, kvh - n_full, : W + chunk].double()
            limit = W + rows
        s = (q[:, h] @ k.T) / D ** 0.5
        jj = torch.arange(k.shape[0], device=qkv.device)[None, :]
        s = s.masked_fill(jj > limit[:, None], float("-inf"))
        out[:, h] = torch.softmax(s, -1) @ v
    return out


@pytest.mark.parametrize("n_full", [0, 1, 4, 8])
def test_tc_prefill_at_the_benchmarked_shape(n_full):
    pytest.importorskip("flash_attn")
    dev = torch.device("cuda:0")
    Hq, Hkv, sink, recent = 32, 8, 64, 256
    past, chunk = 98304, 32768
    cache, g = _filled_cache(Hq, Hkv, n_full, past, chunk, sink, recent, dev, seed=20 + n_full)
    qkv = torch.randn(1, chunk, (Hq + 2 * Hkv) * D, device=dev, dtype=torch.float32, generator=g).to(torch.bfloat16)
    st = cache.state(0)
    stream = torch.cuda.current_stream().cuda_stream
    lib, h = cache.lib, cache.handles[0]
    _C.check(lib.duo_rope_append(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), None, None, _C.ROPE_NONE, chunk, stream))
    out = torch.empty(1, chunk, Hq, D, dtype=torch.bfloat16, device=dev)
    _C.check(lib.duo_attention(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out.data_ptr(), chunk, D ** -0.5,
                               cache.workspace.data_ptr(), cache.workspace.numel(), stream))
    ref = _fa2_reference(cache, qkv, Hq, Hkv, n_full, past, chunk, sink, recent)
    # (a) whole output vs the reference's GPU attention
    assert_parity(out, ref, f"wgmma prefill 32768 over 98304, n_full={n_full} vs flash_attn_func")
    # (b) sampled rows vs exact math: not less accurate than FlashAttention-2 on the same inputs
    rows = torch.randint(0, chunk, (48,), device=dev, generator=g).sort().values
    rows[0], rows[-1] = 0, chunk - 1
    truth = _exact_rows(cache, qkv, rows, Hq, Hkv, n_full, past, chunk, sink, recent)
    e_ours = (out[0, rows].double() - truth).abs()
    e_fa2 = (ref[0, rows].double() - truth).abs()
    tol = ATOL + RTOL * truth.abs()
    v_ours, v_fa2 = (e_ours > tol).double().mean().item(), (e_fa2 > tol).double().mean().item()
    rms_ours, rms_fa2 = e_ours.pow(2).mean().sqrt().item(), e_fa2.pow(2).mean().sqrt().item()
    record("bench_shape_vs_fp64", n_full=n_full, viol_ours=v_ours, viol_fa2=v_fa2, rms_ours=rms_ours,
           rms_fa2=rms_fa2, max_ours=e_ours.max().item(), max_fa2=e_fa2.max().item())
    assert v_ours <= v_fa2 + 1e-3, (v_ours, v_fa2)
    assert rms_ours <= 1.3 * rms_fa2 + 1e-6, (rms_ours, rms_fa2)
    # (c) the other kernel family on the same inputs (mma.sync, 64-row blocks); one configuration: it is slow
    if n_full == 1:
        out2 = torch.empty_like(out)
        _C.check(lib.duo_attention_mma(h, C.byref(st), qkv.data_ptr(), qkv.stride(1), out2.data_ptr(), chunk,
                                       D ** -0.5, cache.workspace.data_ptr(), cache.workspace.numel(), stream))
        assert_parity(out, out2, "wgmma vs mma.sync kernel family at the benchmarked shape")
    torch.cuda.synchronize()


def test_tc_prefill_first_chunk_of_the_benchmark():
    """First 32,768-token chunk (empty cache: every head is plain causal, llama.py:225-233)."""
    fa = pytest.importorskip("flash_attn")
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent, chunk = 32, 8, 4, 64, 256, 32768
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, chunk + 8, sink, recent, torch.bfloat16, dev, stage_cap=chunk)
    g = torch.Generator(device=dev).manual_seed(3)
    qkv = torch.randn(1, chunk, (Hq + 2 * Hkv) * D, device=dev, dtype=torch.float32, generator=g).to(torch.bfloat16)
    out = torch.empty(1, chunk, Hq, D, dtype=torch.bfloat16, device=dev)
    q = qkv[..., : Hq * D].view(1, chunk, Hq, D)
    k = qkv[..., Hq * D : (Hq + Hkv) * D].view(1, chunk, Hkv, D)
    v = qkv[..., (Hq + Hkv) * D :].view(1, chunk, Hkv, D)
    ref = fa.flash_attn_func(q, k, v, causal=True)
    cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)
    assert_parity(out, ref, "wgmma prefill, first chunk of 32768 vs flash_attn_func")


# ------------------------------------------------------------------------------------------------
# INT4 decode at the benchmark's context length: size-independent properties
# ------------------------------------------------------------------------------------------------
def _dequant_rows(cache, name, head, n_rows):
    t = cache.tensors[0]
    out = torch.empty(n_rows, D, dtype=torch.float16, device=cache.device)
    _C.check(cache.lib.duo_dequant_int4(t[name][0, head].data_ptr(), t[name + "_scale"][0, head].data_ptr(),
                                        t[name + "_zero"][0, head].data_ptr(), n_rows, out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    return out


@pytest.mark.parametrize("N", [131072, 1048576])
def test_int4_full_size_decode_properties(N):
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent = 32, 8, 4, 64, 256
    W = sink + recent
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, N + 8, sink, recent, torch.float16, dev, kv_format="int4")
    t = cache.tensors[0]
    g = torch.Generator(device=dev).manual_seed(2)

    def fill(names):
        for n in names:
            t[n].random_(0, 256, generator=g)
            t[n + "_scale"].uniform_(0.05, 0.25, generator=g)
            t[n + "_zero"].uniform_(-2.0, -0.5, generator=g)

    fill(("full_k", "ring_k", "full_v", "ring_v"))
    qkv0 = (torch.randn(1, 1, (Hq + 2 * Hkv) * D, generator=g, device=dev) * 0.5).to(torch.float16)
    out = torch.empty(1, 1, Hq, D, dtype=torch.float16, device=dev)

    def decode(qkv):
        cache.kv_seq_len_list[0] = N
        cache.total_list[0] = N
        cache.lo_list[0] = N - recent
        cache.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
        return out.float().clone()

    # (1) every cached V row dequantises to the same vector c (codes d % 16, scale 0.125, zero -1)  ->  output == c
    codes = (torch.arange(D, device=dev) % 16).to(torch.uint8)
    packed = (codes[0::2] << 4) | codes[1::2]
    for n in ("full_v", "ring_v"):
        t[n][:] = packed
        t[n + "_scale"].fill_(0.125)
        t[n + "_zero"].fill_(-1.0)
    c = codes.float() * 0.125 - 1.0
    q1 = qkv0.clone()
    q1[..., (Hq + Hkv) * D :] = c.to(torch.float16).repeat(Hkv)  # the new token's V quantises to c exactly
    o = decode(q1)
    torch.testing.assert_close(o, c.expand_as(o), rtol=1e-2, atol=1e-3)

    # (2) q == 0 -> uniform attention -> output == mean of the visible (dequantised) V rows
    fill(("full_v", "ring_v"))
    q2 = qkv0.clone()
    q2[..., : Hq * D] = 0
    from oracle import int4_oracle as Q

    vnew = q2[0, 0, (Hq + Hkv) * D :].view(Hkv, D).cpu().numpy()
    p_, s_, z_ = Q.quantize_int4(vnew)
    vnew_rt = torch.from_numpy(Q.dequantize_int4(p_, s_, z_)).float().to(dev)
    means = []
    for kvh in range(Hkv):  # taken BEFORE the call: the ring commit overwrites one slot afterwards
        if kvh < n_full:
            means.append((_dequant_rows(cache, "full_v", kvh, N).float().sum(0) + vnew_rt[kvh]) / (N + 1))
        else:
            means.append((_dequant_rows(cache, "ring_v", kvh - n_full, W).float().sum(0) + vnew_rt[kvh]) / (W + 1))
    o = decode(q2)[0, 0]
    for h in range(Hq):
        torch.testing.assert_close(o[h], means[h // 4], rtol=1e-2, atol=1e-3)

    # (3) one key with an overwhelming logit -> output == that key's dequantised V row, wherever it sits
    #     (first key, tile / split boundaries, middle, last cached key)
    kvh = 1
    qrow = qkv0[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D].float()
    big = (qrow / qrow.norm() * 40.0).to(torch.float16)
    kp = torch.empty(1, 64, dtype=torch.uint8, device=dev)
    ks = torch.empty(1, dtype=torch.float16, device=dev)
    kz = torch.empty(1, dtype=torch.float16, device=dev)
    _C.check(cache.lib.duo_quant_int4(big.data_ptr(), D, 1, kp.data_ptr(), ks.data_ptr(), kz.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream))
    q3 = qkv0.clone()
    q3[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D] = big
    for pos in [0, 127, 128, 4095, N // 2 + 17, N - 1]:
        saved = (t["full_k"][0, kvh, pos].clone(), t["full_k_scale"][0, kvh, pos].clone(),
                 t["full_k_zero"][0, kvh, pos].clone())
        t["full_k"][0, kvh, pos] = kp[0]
        t["full_k_scale"][0, kvh, pos] = ks[0]
        t["full_k_zero"][0, kvh, pos] = kz[0]
        want = _dequant_rows(cache, "full_v", kvh, pos + 1)[pos].float()
        o = decode(q3)[0, 0, kvh * 4]
        torch.testing.assert_close(o, want, rtol=1e-2, atol=2e-3)
        t["full_k"][0, kvh, pos], t["full_k_scale"][0, kvh, pos], t["full_k_zero"][0, kvh, pos] = saved
