"""INT4-KV attention with the dequantisation folded into the K/V load vs the oracle restating
demo/w8a8kv4_llama.py:215-278 + demo/int4_kv.py (quantise on put, dequantise-everything on get)."""
import numpy as np
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from oracle import duo_oracle as O
from oracle import int4_oracle as Q
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128


def run(Hq, Hkv, n_full, sink, recent, chunks, seed=0, B=1, stage_cap=8, scale_kv=1.0):
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(seed)
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], B, sum(chunks) + 8, sink, recent, torch.float16, dev,
                       stage_cap=stage_cap, kv_format="int4")
    past = None
    for i, S in enumerate(chunks):
        qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(torch.float16)
        qkv[..., Hq * D :] *= scale_kv
        out = torch.empty(B, S, Hq, D, dtype=torch.float16, device=dev)
        cache.attend(0, qkv.to(dev), None, None, _C.ROPE_NONE, out)
        q = qkv[..., : Hq * D].reshape(B, S, Hq, D)
        k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(B, S, Hkv, D)
        v = qkv[..., (Hq + Hkv) * D :].reshape(B, S, Hkv, D)
        ref, past = O.int4_attention_core(q, k, v, past, n_full, Hq // Hkv, sink, recent)
        assert_parity(out.float().cpu(), ref.float(), f"chunk {i} (len {S})")
        assert cache.kv_seq_len == past[0].shape[2] and cache.streaming_kv_seq_len == past[1].shape[2]
    return cache


@pytest.mark.parametrize("n_full", [0, 1, 2])
def test_int4_decode_and_small_chunks(n_full):
    run(8, 2, n_full, 8, 24, [40, 1, 1, 3, 1, 30, 1, 5, 1], seed=n_full)


def test_int4_deploy_config_long():
    run(16, 4, 2, 64, 256, [700, 1, 1, 200, 1, 2, 1], seed=5, stage_cap=700)


def test_int4_split_kv_long_context():
    run(4, 1, 1, 64, 256, [12000, 1, 1, 4, 1], seed=6, stage_cap=12000)


def test_int4_odd_window_and_mha():
    run(4, 4, 2, 3, 7, [5, 1, 1, 1, 20, 1, 1, 2, 1, 1], seed=7)


def test_int4_cache_content_is_k1_quantisation():
    """What lands in the cache is bit-for-bit the oracle's K1 output (scale/zero/codes)."""
    cache = run(8, 2, 1, 4, 4, [10], seed=9)
    g = torch.Generator().manual_seed(9)
    qkv = torch.randn(1, 10, 12 * D, generator=g).to(torch.float16)
    k = qkv[..., 8 * D : 10 * D].reshape(1, 10, 2, D)
    p, s, z = Q.quantize_int4(k[:, :, 0].numpy())
    t = cache.tensors[0]
    assert np.array_equal(t["full_k"][0, 0, :10].cpu().numpy(), p[0])
    assert np.array_equal(t["full_k_scale"][0, 0, :10].cpu().numpy(), s[0, :, 0])
    assert np.array_equal(t["full_k_zero"][0, 0, :10].cpu().numpy(), z[0, :, 0])


def test_int4_many_splits():
    """> 16 splits per retrieval head: the split-KV merge loop takes more than one pass per warp."""
    run(4, 1, 1, 64, 256, [20000, 1, 2, 1], seed=16, stage_cap=20000)


def test_int4_batch2_decode():
    run(8, 2, 1, 8, 24, [3000, 1, 2, 1, 1], seed=17, B=2, stage_cap=3000)


def test_int4_mha_rows_up_to_8():
    """group 1: q_len 1..8 all fit the 8-row (keys-as-M) decode kernel; 9..16 the row-major one."""
    run(4, 4, 2, 4, 12, [50, 1, 8, 7, 5, 1, 3, 9, 16, 1], seed=18, stage_cap=50)


def test_int4_large_chunks_batch2():
    """Chunks of >= 128 tokens after the first call run on the wgmma prefill kernel over a dequantised fp16 image of the
    cache (kv_cache._dequant_scratch) and must match the oracle's dequantise-everything attention."""
    run(8, 2, 1, 16, 48, [300, 130, 1, 256, 1, 2, 128, 1], seed=19, B=2, stage_cap=300)
    run(8, 2, 0, 16, 48, [200, 129, 1, 140], seed=20, stage_cap=200)   # no retrieval head in the layer
    run(8, 2, 2, 16, 48, [200, 129, 1, 140], seed=21, stage_cap=200)   # no streaming head in the layer


def test_int4_large_chunk_kernel_families_agree():
    """The same >= 128-token chunk through the mma.sync INT4 kernel (dequant in the load stage) and through the
    wgmma prefill kernel on the fp16 image."""
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full = 8, 2, 1
    outs = []
    for force in (False, True):
        g = torch.Generator().manual_seed(23)
        cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, 2048, 16, 48, torch.float16, dev, stage_cap=700, kv_format="int4")
        res = []
        for S in [700, 384, 1, 200]:
            qkv = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(torch.float16).to(dev)
            out = torch.empty(1, S, Hq, D, dtype=torch.float16, device=dev)
            if force and cache.kv_seq_len > 0:
                # duo_attention on the INT4 layer handle itself = the mma.sync INT4 kernel
                import ctypes as C
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
        assert_parity(a, b, "INT4 chunk: wgmma-on-fp16-image vs mma.sync fused-dequant kernel")


def test_w8a8kv4_attention_core_through_the_fused_qkv_boundary():
    """duo_w8a8kv4_attention (what demo/w8a8kv4_llama.py:174-287 does between the fused int8 projection and the output
    quantisation): fp16 activation buffer [bsz*q_len, q+2kv] in, fp32 on-the-fly RoPE, INT4-KV cache, attention out —
    vs the oracle's flashinfer-style RoPE + INT4 attention core."""
    import types

    from duo_attention_b200.patch import w8a8kv4

    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent, theta = 8, 2, 1, 8, 24, 10000.0
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, 512, sink, recent, torch.float16, dev, stage_cap=200,
                       kv_format="int4")
    mod = types.SimpleNamespace(layer_idx=0, head_dim=D, num_heads=Hq, num_kv_heads=Hkv, rope_theta=theta)
    g = torch.Generator().manual_seed(31)
    past, pos = None, 0
    for S in [150, 1, 1, 20, 1, 130, 1]:
        act = torch.randn(S, (Hq + 2 * Hkv) * D, generator=g).to(torch.float16)
        out = w8a8kv4.duo_w8a8kv4_attention(mod, act.to(dev), cache, S)
        q = act[:, : Hq * D].reshape(1, S, Hq, D)
        k = act[:, Hq * D : (Hq + Hkv) * D].reshape(1, S, Hkv, D)
        v = act[:, (Hq + Hkv) * D :].reshape(1, S, Hkv, D)
        qr, kr = O.rope_flashinfer(q, k, pos, 1.0, theta)
        ref, past = O.int4_attention_core(qr, kr, v, past, n_full, Hq // Hkv, sink, recent)
        assert_parity(out.view(1, S, Hq, D).float().cpu(), ref.float(), f"chunk of {S} at {pos}")
        pos += S


@pytest.mark.parametrize("rope", ["none", "hf", "fp32"])
@pytest.mark.parametrize("shape", ["gqa4", "mha", "b2"])
def test_int4_one_launch_decode_is_bit_identical_to_three_launches(rope, shape):
    """duo_decode_fused on an INT4 cache (RoPE + K1 quantise + append + attention + ring commit in one launch) against
    duo_rope_append + duo_attention + duo_stream_commit on the same inputs: outputs and every cache tensor must hold
    the same bits after every step (the two paths share the RoPE / K1 device functions).  Schedules cross the sink
    boundary, wrap the ring and straddle split / tile boundaries of the retrieval cache."""
    from duo_attention_b200.patch.w8a8kv4 import rope_tables_fp32

    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, B, chunks = {
        "gqa4": (8, 2, 1, 1, [3, 1, 1, 2, 1, 40, 1, 2, 1, 1, 2, 5000, 1, 2, 1, 1]),
        "mha": (4, 4, 2, 1, [2, 1, 8, 7, 1, 3, 30, 5, 1, 8, 8, 8, 1]),
        "b2": (8, 2, 2, 2, [130, 1, 2, 1, 1, 1, 2, 2, 1]),
    }[shape]
    sink, recent = 4, 12
    mode = {"none": _C.ROPE_NONE, "hf": _C.ROPE_HF, "fp32": _C.ROPE_FP32}[rope]
    caches = [DuoKVCache(1, Hq, Hkv, D, [n_full], B, sum(chunks) + 8, sink, recent, torch.float16, dev,
                         stage_cap=max(chunks), kv_format="int4") for _ in range(2)]
    g = torch.Generator().manual_seed(91)
    pos, n_fused = 0, 0
    for S in chunks:
        qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(torch.float16).to(dev)
        cos = sin = None
        if mode != _C.ROPE_NONE:
            cos, sin = rope_tables_fp32(pos, S, D, 10000.0, 1.0, dev)
            if mode == _C.ROPE_HF:
                cos, sin = cos.to(torch.float16), sin.to(torch.float16)
        outs = []
        for cache, fused in zip(caches, (True, False)):
            x = qkv.clone()
            out = torch.empty(B, S, Hq, D, dtype=torch.float16, device=dev)
            before = cache.launch_count
            cache.attend(0, x, cos, sin, mode, out, fused=fused)
            if fused and cache.launch_count - before == 1:
                n_fused += 1
                assert torch.equal(x, qkv), "the one-launch path must not modify qkv"
            outs.append(out)
        assert torch.equal(outs[0], outs[1]), f"outputs differ at chunk of {S} tokens (pos {pos})"
        for name in caches[0].tensors[0]:
            a, b = caches[0].tensors[0][name], caches[1].tensors[0][name]
            if name.startswith("ring"):  # staging rows beyond the ring hold leftovers of the unfused path only
                a, b = a[:, :, : caches[0].W], b[:, :, : caches[0].W]
            else:
                a, b = a[:, :, : pos + S], b[:, :, : pos + S]
            assert torch.equal(a, b), f"cache tensor {name} differs after a chunk of {S} tokens (pos {pos})"
        pos += S
    G = Hq // Hkv
    assert n_fused == sum(1 for i, S in enumerate(chunks) if i > 0 and S * G <= 8), "one-launch path not taken"
