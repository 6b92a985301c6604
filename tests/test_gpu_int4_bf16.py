"""bf16 activations over the INT4 KV cache (packed nibbles + fp16 scale / zero, K1 on the fp32 value of each rotated
bf16 row): every path the fp16 INT4 tests cover — decode and small chunks, split-KV, the one-launch decode, chunks of
>= 128 tokens on the bf16 image, CUDA-graph replay, the drop-in class — against the oracle, whose bf16 INT4 core
attends the K2 (fp16) values of the cache kept in fp32."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from oracle import duo_oracle as O
from oracle import int4_oracle as Q
import int4_bf16_oracle as H
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128
BF = torch.bfloat16


def run(Hq, Hkv, n_full, sink, recent, chunks, seed=0, B=1, stage_cap=8, q_mul=1.0, scale=None):
    """Chunks of bf16 qkv through an INT4 cache, each output against the oracle.  ``q_mul`` (a power of two) scales
    q; the oracle sees q * scale / D^-0.5, i.e. the same logits as the kernel's softmax scale ``scale``."""
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(seed)
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], B, sum(chunks) + 8, sink, recent, BF, dev, stage_cap=stage_cap,
                       kv_format="int4")
    past = None
    for i, S in enumerate(chunks):
        qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(BF)
        qkv[..., : Hq * D] *= q_mul
        out = torch.empty(B, S, Hq, D, dtype=BF, device=dev)
        cache.attend(0, qkv.to(dev), None, None, _C.ROPE_NONE, out, scale=scale)
        q = qkv[..., : Hq * D].reshape(B, S, Hq, D) * (1.0 if scale is None else scale / D ** -0.5)
        k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D)
        v = qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D)
        ref, past = H.int4_attention_core(q, k, v, past, n_full, Hq // Hkv, sink, recent)
        assert torch.isfinite(out).all(), f"chunk {i} (len {S}): non-finite output"
        assert_parity(out.float().cpu(), ref.float(), f"bf16 chunk {i} (len {S})")
        assert cache.kv_seq_len == past[0].shape[2] and cache.streaming_kv_seq_len == past[1].shape[2]
    return cache


@pytest.mark.parametrize("n_full", [0, 1, 2])
def test_bf16_int4_decode_and_small_chunks(n_full):
    run(8, 2, n_full, 8, 24, [40, 1, 1, 3, 1, 30, 1, 5, 1], seed=n_full)


def test_bf16_int4_deploy_config_long():
    run(16, 4, 2, 64, 256, [700, 1, 1, 200, 1, 2, 1], seed=5, stage_cap=700)


@pytest.mark.parametrize("chunks", [[12000, 1, 1, 4, 1], [20000, 1, 2, 1]], ids=["12k", "20k_many_splits"])
def test_bf16_int4_split_kv_long_context(chunks):
    run(4, 1, 1, 64, 256, chunks, seed=6, stage_cap=chunks[0])


def test_bf16_int4_mha_rows_up_to_8_and_9_to_16():
    run(4, 4, 2, 4, 12, [50, 1, 8, 7, 5, 1, 3, 9, 16, 1], seed=18, stage_cap=50)


def test_bf16_int4_batch2_decode():
    run(8, 2, 1, 8, 24, [3000, 1, 2, 1, 1], seed=17, B=2, stage_cap=3000)


def test_bf16_int4_large_chunks():
    """Chunks of >= 128 tokens after the first call: wgmma prefill kernel on the bf16 image (duo_dequant_int4_bf16)."""
    run(8, 2, 1, 16, 48, [300, 130, 1, 256, 1, 2, 128, 1], seed=19, B=2, stage_cap=300)
    run(8, 2, 0, 16, 48, [200, 129, 1, 140], seed=20, stage_cap=200)   # no retrieval head in the layer
    run(8, 2, 2, 16, 48, [200, 129, 1, 140], seed=21, stage_cap=200)   # no streaming head in the layer


def test_bf16_int4_large_chunk_wide_window_takes_the_int4_kernel():
    """sink + recent > 2048: a >= 128-token chunk stays on the INT4 mma.sync kernel (duo_attn_int4_kernel<1>).  That
    fallback scans all ~2400 ring keys of a streaming head in one warp, and with a near-uniform softmax the fp32
    accumulator holding 1024 * sum(p') loses low bits of sum(p' c): it misses the oracle's rtol/atol on a share of the
    elements for fp16 activations as well.  What bf16 must guarantee here is the fp16 kernel's result: on inputs exact
    in both dtypes (same cache bytes, same fp16 q), the outputs agree up to their own roundings to fp16 and bf16."""
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent, chunks = 8, 2, 1, 64, 2048, [2500, 300, 1]
    caches = {dt: DuoKVCache(1, Hq, Hkv, D, [n_full], 1, sum(chunks) + 8, sink, recent, dt, dev, stage_cap=2500,
                             kv_format="int4") for dt in (BF, torch.float16)}
    g = torch.Generator().manual_seed(22)
    for i, S in enumerate(chunks):
        x = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(BF).float()
        x[x.abs() < 2.0 ** -14] = 0.0
        outs = {}
        for dt, cache in caches.items():
            outs[dt] = torch.empty(1, S, Hq, D, dtype=dt, device=dev)
            cache.attend(0, x.to(dt).to(dev), None, None, _C.ROPE_NONE, outs[dt])
        ob, of = outs[BF].float(), outs[torch.float16].float()
        assert torch.isfinite(ob).all()
        if i == 0:  # the first chunk attends the raw K / V on a 16-bit layer of the activation dtype: not INT4
            continue
        bound = of.abs() * (2.0 ** -8 + 2.0 ** -11) + 2.0 ** -24
        assert ((ob - of).abs() <= bound).all(), f"chunk of {S}: max |bf16 - fp16| {(ob - of).abs().max().item():.3g}"


def test_bf16_int4_large_q_stays_finite():
    """|q| up to ~3e4 (fp16 range, which the bf16 kernels' fp16 inner loop needs): q scaled by 2^13 with the softmax
    scale divided by the same power of two gives the same logits, so the outputs must still match the oracle."""
    run(8, 2, 1, 8, 24, [40, 1, 1, 3, 1, 20, 1, 200, 1], seed=24, stage_cap=200, q_mul=8192.0,
        scale=D ** -0.5 / 8192.0)


def test_bf16_int4_cache_content_is_k1_quantisation():
    """The cache holds bit-for-bit the oracle's K1 of the bf16 rows (fp32 values of bf16)."""
    cache = run(8, 2, 1, 4, 4, [10], seed=9)
    g = torch.Generator().manual_seed(9)
    qkv = torch.randn(1, 10, 12 * D, generator=g).to(BF)
    t = cache.tensors[0]
    for name, lo in (("full_k", 8), ("full_v", 10)):
        x = qkv[..., lo * D : (lo + 1) * D].float().numpy()
        p, s, z = H.quantize_int4(x)
        assert np.array_equal(t[name][0, 0, :10].cpu().numpy(), p[0])
        assert np.array_equal(t[name + "_scale"][0, 0, :10].cpu().numpy(), s[0, :, 0])
        assert np.array_equal(t[name + "_zero"][0, 0, :10].cpu().numpy(), z[0, :, 0])


def test_bf16_and_fp16_caches_hold_the_same_bytes_for_shared_values():
    """Inputs representable in both dtypes, no RoPE: a bf16 INT4 cache and an fp16 INT4 cache end up byte-identical
    (the format does not depend on the activation dtype), through first chunk, decode, small and large chunks."""
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent, chunks = 8, 2, 1, 4, 12, [40, 1, 1, 3, 1, 200, 1, 1]
    caches = {dt: DuoKVCache(1, Hq, Hkv, D, [n_full], 1, sum(chunks) + 8, sink, recent, dt, dev, stage_cap=200,
                             kv_format="int4") for dt in (BF, torch.float16)}
    g = torch.Generator().manual_seed(41)
    pos = 0
    for S in chunks:
        x = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(BF).float()
        x[x.abs() < 2.0 ** -14] = 0.0  # bf16 values that are fp16 normals (or zero): exact in both
        for dt, cache in caches.items():
            xd = x.to(dt)
            assert torch.equal(xd.float(), x)
            cache.attend(0, xd.to(dev), None, None, _C.ROPE_NONE, torch.empty(1, S, Hq, D, dtype=dt, device=dev))
        pos += S
        a, b = caches[BF].tensors[0], caches[torch.float16].tensors[0]
        for name in a:
            n = caches[BF].W if name.startswith("ring") else pos
            assert torch.equal(a[name][:, :, :n], b[name][:, :, :n]), f"{name} differs after {pos} tokens"


@pytest.mark.parametrize("rope", ["none", "hf", "fp32"])
@pytest.mark.parametrize("shape", ["gqa4", "mha", "b2"])
def test_bf16_int4_one_launch_decode_is_bit_identical_to_three_launches(rope, shape):
    """duo_decode_fused on a bf16 INT4 layer against duo_rope_append + duo_attention + duo_stream_commit: the same
    output and cache bits after every step."""
    from duo_attention_b200.patch.w8a8kv4 import rope_tables_fp32

    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, B, chunks = {
        "gqa4": (8, 2, 1, 1, [3, 1, 1, 2, 1, 40, 1, 2, 1, 1, 2, 5000, 1, 2, 1, 1]),
        "mha": (4, 4, 2, 1, [2, 1, 8, 7, 1, 3, 30, 5, 1, 8, 8, 8, 1]),
        "b2": (8, 2, 2, 2, [130, 1, 2, 1, 1, 1, 2, 2, 1]),
    }[shape]
    sink, recent = 4, 12
    mode = {"none": _C.ROPE_NONE, "hf": _C.ROPE_HF, "fp32": _C.ROPE_FP32}[rope]
    caches = [DuoKVCache(1, Hq, Hkv, D, [n_full], B, sum(chunks) + 8, sink, recent, BF, dev, stage_cap=max(chunks),
                         kv_format="int4") for _ in range(2)]
    g = torch.Generator().manual_seed(91)
    pos, n_fused = 0, 0
    for S in chunks:
        qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(BF).to(dev)
        cos = sin = None
        if mode != _C.ROPE_NONE:
            cos, sin = rope_tables_fp32(pos, S, D, 10000.0, 1.0, dev)
            if mode == _C.ROPE_HF:
                cos, sin = cos.to(BF), sin.to(BF)
        outs = []
        for cache, fused in zip(caches, (True, False)):
            x = qkv.clone()
            out = torch.empty(B, S, Hq, D, dtype=BF, device=dev)
            before = cache.launch_count
            cache.attend(0, x, cos, sin, mode, out, fused=fused)
            if fused and cache.launch_count - before == 1:
                n_fused += 1
                assert torch.equal(x, qkv), "the one-launch path must not modify qkv"
            outs.append(out)
        assert torch.equal(outs[0], outs[1]), f"outputs differ at chunk of {S} tokens (pos {pos})"
        for name in caches[0].tensors[0]:
            a, b = caches[0].tensors[0][name], caches[1].tensors[0][name]
            n = caches[0].W if name.startswith("ring") else pos + S
            assert torch.equal(a[:, :, :n], b[:, :, :n]), f"cache tensor {name} differs after {S} tokens (pos {pos})"
        pos += S
    G = Hq // Hkv
    assert n_fused == sum(1 for i, S in enumerate(chunks) if i > 0 and S * G <= 8), "one-launch path not taken"


def test_dequant_int4_bf16_matches_the_numpy_restatement_bit_for_bit():
    dev = torch.device("cuda:0")
    rows = 1000
    g = torch.Generator().manual_seed(3)
    packed = torch.randint(0, 256, (rows, 64), generator=g, dtype=torch.uint8)
    scale = (torch.rand(rows, generator=g) * 4.0).to(torch.float16)
    scale[:200] = (torch.rand(200, generator=g) * 1e-3).to(torch.float16)   # includes fp16 subnormals
    zero = (torch.randn(rows, generator=g) * 30.0).to(torch.float16)
    out = torch.empty(rows, D, dtype=BF, device=dev)
    pd, sd, zd = packed.to(dev), scale.to(dev), zero.to(dev)
    _C.check(_C.load().duo_dequant_int4_bf16(pd.data_ptr(), sd.data_ptr(), zd.data_ptr(), rows, out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
    want = H.dequantize_int4_bf16(packed.numpy(), scale.numpy()[:, None], zero.numpy()[:, None])
    got = out.float().cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_bf16_int4_large_chunk_kernel_families_agree():
    """The same >= 128-token chunk through the INT4 mma.sync kernel (dequantisation in the load stage) and through the
    wgmma prefill kernel on the bf16 image."""
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full = 8, 2, 1
    outs = []
    for force in (False, True):
        g = torch.Generator().manual_seed(23)
        cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, 2048, 16, 48, BF, dev, stage_cap=700, kv_format="int4")
        res = []
        for S in [700, 384, 1, 200]:
            qkv = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(BF).to(dev)
            out = torch.empty(1, S, Hq, D, dtype=BF, device=dev)
            if force and cache.kv_seq_len > 0:  # duo_attention on the INT4 layer handle itself = the mma.sync kernel
                st = cache.state(0)
                stream = torch.cuda.current_stream().cuda_stream
                cache._ensure_room(0, S)
                _C.check(cache.lib.duo_rope_append(cache.handles[0], C.byref(st), qkv.data_ptr(), qkv.stride(1), None,
                                                   None, _C.ROPE_NONE, S, stream))
                _C.check(cache.lib.duo_attention(cache.handles[0], C.byref(st), qkv.data_ptr(), qkv.stride(1),
                                                 out.data_ptr(), S, D ** -0.5, cache.workspace.data_ptr(),
                                                 cache.workspace.numel(), stream))
                _C.check(cache.lib.duo_stream_commit(cache.handles[0], C.byref(st), S, stream))
                cache.advance(0, S)
            else:
                cache.attend(0, qkv, None, None, _C.ROPE_NONE, out)
            res.append(out.float().cpu())
        outs.append(res)
    for a, b in zip(*outs):
        assert_parity(a, b, "bf16 INT4 chunk: wgmma on the bf16 image vs mma.sync fused-dequant kernel")


# ---- model level --------------------------------------------------------------------------------------------------
def _tiny_llama(seed):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=512, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                      intermediate_size=1024, vocab_size=512, max_position_embeddings=8192, rope_theta=10000.0,
                      attn_implementation="eager")
    return LlamaForCausalLM(cfg).to(BF).eval()


def test_bf16_int4_model_through_the_drop_in_cache_class():
    """Tiny bf16 Llama, static enable + DuoAttentionStaticINT4KVCache vs OracleModel(kv_format="int4") on the same bf16
    weights, over a schedule with a >= 128-token chunk."""
    from duo_attn.patch import DuoAttentionStaticINT4KVCache, enable_llama_duo_attention_static_kv_cache_eval

    model = _tiny_llama(11)
    gates = np.array([[1.0, 0.0], [1.0, 1.0]])
    sink, recent = 8, 16
    oracle = O.OracleModel(copy.deepcopy(model), gates, sink, recent, kv_format="int4")
    oracle.core = H.int4_attention_core  # the INT4 core for bf16 q/k/v
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    cache = DuoAttentionStaticINT4KVCache(model, gates, 1, 512, sink, recent, 160)
    assert cache.dtype == BF and cache.kv_format == "int4"
    g = torch.Generator().manual_seed(5)
    past_o = None
    with torch.no_grad():
        for S in [150, 1, 1, 140, 1, 33, 1, 1]:
            ids = torch.randint(0, 512, (1, S), generator=g)
            lo, past_o = oracle(ids, past_o)
            out = model(input_ids=ids.cuda(), past_key_values=cache, use_cache=True)
            torch.testing.assert_close(out.logits.float().cpu(), lo, rtol=5e-2, atol=5e-2)
            assert cache.kv_seq_len == past_o[0][0].shape[2]


def test_bf16_int4_cuda_graph_decode_matches_eager():
    """DuoDecodeGraph replay (device-resident occupancy) == eager decode, token by token, on a bf16 INT4 cache."""
    from duo_attention_b200.graph import DuoDecodeGraph
    from duo_attn.patch import DuoAttentionStaticKVCache, enable_llama_duo_attention_static_kv_cache_eval

    model = _tiny_llama(7)
    gates = np.array([[1.0, 0.0], [0.0, 1.0]])
    sink, recent = 4, 6
    enable_llama_duo_attention_static_kv_cache_eval(model, gates)
    model.cuda()
    ca = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent, kv_format="int4")
    cb = DuoAttentionStaticKVCache(model, gates, 1, 256, sink, recent, kv_format="int4")
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 512, (1, 37), generator=g).cuda()
    with torch.no_grad():
        model(input_ids=ids, past_key_values=ca, use_cache=True)
        model(input_ids=ids, past_key_values=cb, use_cache=True)
        graph = DuoDecodeGraph(model, cb)
        toks = torch.randint(0, 512, (20, 1, 1), generator=g).cuda()
        for i in range(20):
            want = model(input_ids=toks[i], past_key_values=ca, use_cache=True).logits
            got = graph.step(toks[i])
            torch.testing.assert_close(got.float(), want.float(), rtol=0, atol=0, msg=lambda m: f"step {i}: {m}")
            if i == 9:
                ca.evict_last(1)
                cb.evict_last(1)
                graph.resync()


# ---- decode at full context length: size-independent properties ----------------------------------------------------
def _dequant_rows(cache, name, head, n_rows):
    """K2 (fp16) values of cache rows: what the INT4 decode kernels attend."""
    t = cache.tensors[0]
    out = torch.empty(n_rows, D, dtype=torch.float16, device=cache.device)
    _C.check(cache.lib.duo_dequant_int4(t[name][0, head].data_ptr(), t[name + "_scale"][0, head].data_ptr(),
                                        t[name + "_zero"][0, head].data_ptr(), n_rows, out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    return out


@pytest.mark.parametrize("N", [131072, 1048576])
def test_bf16_int4_full_size_decode_properties(N):
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent = 32, 8, 4, 64, 256
    W = sink + recent
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, N + 8, sink, recent, BF, dev, kv_format="int4")
    t = cache.tensors[0]
    g = torch.Generator(device=dev).manual_seed(2)

    def fill(names):
        for n in names:
            t[n].random_(0, 256, generator=g)
            t[n + "_scale"].uniform_(0.05, 0.25, generator=g)
            t[n + "_zero"].uniform_(-2.0, -0.5, generator=g)

    fill(("full_k", "ring_k", "full_v", "ring_v"))
    qkv0 = (torch.randn(1, 1, (Hq + 2 * Hkv) * D, generator=g, device=dev) * 0.5).to(BF)
    out = torch.empty(1, 1, Hq, D, dtype=BF, device=dev)

    def decode(qkv):
        cache.kv_seq_len_list[0] = N
        cache.total_list[0] = N
        cache.lo_list[0] = N - recent
        cache.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
        return out.float().clone()

    # (1) every V row dequantises to the same vector c (codes d % 16, scale 0.125, zero -1)  ->  output == c
    codes = (torch.arange(D, device=dev) % 16).to(torch.uint8)
    packed = (codes[0::2] << 4) | codes[1::2]
    for n in ("full_v", "ring_v"):
        t[n][:] = packed
        t[n + "_scale"].fill_(0.125)
        t[n + "_zero"].fill_(-1.0)
    c = codes.float() * 0.125 - 1.0
    q1 = qkv0.clone()
    q1[..., (Hq + Hkv) * D :] = c.to(BF).repeat(Hkv)  # the new token's V quantises to c exactly
    o = decode(q1)
    torch.testing.assert_close(o, c.expand_as(o), rtol=1e-2, atol=1e-3)

    # (2) q == 0 -> uniform attention -> output == mean of the visible (dequantised) V rows
    fill(("full_v", "ring_v"))
    q2 = qkv0.clone()
    q2[..., : Hq * D] = 0
    vnew = q2[0, 0, (Hq + Hkv) * D :].view(Hkv, D).float().cpu().numpy()
    p_, s_, z_ = H.quantize_int4(vnew)
    vnew_rt = torch.from_numpy(Q.dequantize_int4(p_, s_, z_)).float().to(dev)
    means = []
    for kvh in range(Hkv):  # taken BEFORE the call: the ring commit overwrites one slot afterwards
        if kvh < n_full:
            means.append((_dequant_rows(cache, "full_v", kvh, N).float().sum(0) + vnew_rt[kvh]) / (N + 1))
        else:
            means.append((_dequant_rows(cache, "ring_v", kvh - n_full, W).float().sum(0) + vnew_rt[kvh]) / (W + 1))
    o = decode(q2)[0, 0]
    for h in range(Hq):  # the fp16 test's tolerance plus one bf16 rounding of the output (2^-8 relative)
        torch.testing.assert_close(o[h], means[h // 4], rtol=1e-2 + 2.0 ** -8, atol=1e-3)

    # (3) one key with an overwhelming logit -> output == that key's dequantised V row, wherever it sits
    kvh = 1
    qrow = qkv0[0, 0, kvh * 4 * D : (kvh * 4 + 1) * D].float()
    big = (qrow / qrow.norm() * 40.0).to(BF)
    kp = torch.empty(1, 64, dtype=torch.uint8, device=dev)
    ks = torch.empty(1, dtype=torch.float16, device=dev)
    kz = torch.empty(1, dtype=torch.float16, device=dev)
    big16 = big.to(torch.float16)
    _C.check(cache.lib.duo_quant_int4(big16.data_ptr(), D, 1, kp.data_ptr(), ks.data_ptr(), kz.data_ptr(),
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
