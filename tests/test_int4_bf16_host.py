"""bf16 activations over the INT4 KV cache, host side: layer creation (INT4 layers encode no TMA maps, so no GPU is
needed) and the bf16 K1 / dequantise / round-trip oracle paths of tests/int4_bf16_oracle.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import int4_bf16_oracle as H
from oracle import int4_oracle as Q


def _lib():
    from duo_attention_b200 import _C

    if not os.path.exists(_C.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    return _C, _C.load()


def _int4_desc(_C, dtype):
    d = _C.LayerDesc()
    d.full_k, d.full_v, d.ring_k, d.ring_v = 0x10000, 0x20000, 0x30000, 0x40000
    d.full_k_scale, d.full_k_zero, d.full_v_scale, d.full_v_zero = 0x50000, 0x60000, 0x70000, 0x80000
    d.ring_k_scale, d.ring_k_zero, d.ring_v_scale, d.ring_v_zero = 0x90000, 0xA0000, 0xB0000, 0xC0000
    d.full_cap, d.batch, d.n_full, d.n_stream, d.group, d.head_dim = 256, 1, 1, 1, 4, 128
    d.sink, d.recent, d.stage_cap = 4, 12, 64
    d.dtype, d.kv_format = dtype, _C.KV_INT4
    return d


def test_layer_create_accepts_int4_with_bf16_and_rejects_a_bad_dtype():
    _C, lib = _lib()
    for dt in (_C.DT_BF16, _C.DT_FP16):
        h = C.c_void_p()
        assert lib.duo_layer_create(C.byref(_int4_desc(_C, dt)), C.byref(h)) == _C.DUO_OK, _C.last_error()
        assert h.value
        lib.duo_layer_destroy(h)
    h = C.c_void_p()
    assert lib.duo_layer_create(C.byref(_int4_desc(_C, 7)), C.byref(h)) == _C.DUO_EINVAL
    assert "bad dtype" in _C.last_error() and not h.value


def test_dequant_int4_bf16_validates_before_touching_cuda():
    _C, lib = _lib()
    assert lib.duo_dequant_int4_bf16(None, None, None, 0, None, None) == _C.DUO_OK  # nothing to do
    assert lib.duo_dequant_int4_bf16(None, None, None, 4, None, None) == _C.DUO_EINVAL
    assert "duo_dequant_int4_bf16" in _C.last_error()
    assert lib.duo_dequant_int4_bf16(0x100, 0x100, 0x100, -1, 0x100, None) == _C.DUO_EINVAL


def _bf16_values(shape, seed, mul=3.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * mul).to(torch.bfloat16).float().numpy()


def test_k1_on_bf16_values_equals_k1_on_the_same_fp16_values():
    """K1 sees fp32 values: bf16-valued float32 input that is also exact in fp16 quantises exactly as fp16 input."""
    x = _bf16_values((64, 4, 128), 0)
    x[np.abs(x) < 2.0 ** -14] = 0.0
    assert np.array_equal(x.astype(np.float16).astype(np.float32), x)
    a = H.quantize_int4(x)
    b = Q.quantize_int4(x.astype(np.float16))
    for u, v in zip(a, b):
        assert u.dtype == v.dtype and np.array_equal(u, v)


def test_k1_rejects_float32_that_is_not_bf16_valued():
    x = _bf16_values((2, 128), 1)
    x[0, 5] = np.float32(1.0 + 2.0 ** -20)
    with pytest.raises(AssertionError):
        H.quantize_int4(x)
    with pytest.raises(AssertionError):
        H.quantize_int4(x.astype(np.float64))


def test_k1_on_bf16_values_min_max_codes():
    x = _bf16_values((32, 128), 2, mul=100.0)
    p, s, z = H.quantize_int4(x)
    codes = Q.unpack_codes(p)
    assert (np.take_along_axis(codes, x.argmin(-1)[:, None], -1) == 0).all()
    assert (np.take_along_axis(codes, x.argmax(-1)[:, None], -1) == 15).all()
    assert np.array_equal(z[:, 0], x.min(-1).astype(np.float16))


def test_round_to_bf16_matches_torch():
    rng = np.random.RandomState(3)
    f = (rng.randn(100000) * np.exp(rng.uniform(-20, 20, 100000))).astype(np.float32)
    f[:4] = [0.0, -0.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8]  # exact ties: to even
    want = torch.from_numpy(f).to(torch.bfloat16).float().numpy()
    assert np.array_equal(H.round_to_bf16(f).view(np.uint32), want.view(np.uint32))


def test_dequant_bf16_is_the_fp32_fma_rounded_to_bf16():
    rng = np.random.RandomState(4)
    p = rng.randint(0, 256, size=(500, 64)).astype(np.uint8)
    s = (rng.uniform(0, 4, size=(500, 1))).astype(np.float16)
    z = (rng.randn(500, 1) * 30).astype(np.float16)
    y = H.dequantize_int4_bf16(p, s, z)
    assert y.dtype == np.float32 and H.is_bf16_valued(y)
    codes = Q.unpack_codes(p).astype(np.float64)
    f32 = (codes * s.astype(np.float64) + z.astype(np.float64)).astype(np.float32)
    want = torch.from_numpy(f32).to(torch.bfloat16).float().numpy()
    assert np.array_equal(y, want)
    # within one bf16 rounding of K2's fp16 value; code 0 gives bf16(zero)
    k2 = Q.dequantize_int4(p, s, z).astype(np.float32)
    assert (np.abs(y - k2) <= np.abs(k2) * 2.0 ** -8 + np.abs(k2) * 2.0 ** -11 + 2.0 ** -24).all()
    zero_codes = codes == 0
    assert np.array_equal(y[zero_codes], H.round_to_bf16(np.broadcast_to(z.astype(np.float32), y.shape))[zero_codes])


def test_roundtrip_of_bf16_keeps_the_k2_values_in_fp32():
    x = torch.from_numpy(_bf16_values((2, 5, 3, 128), 5)).to(torch.bfloat16)
    y = H.int4_roundtrip(x)
    assert y.dtype == torch.float32 and y.shape == x.shape
    p, s, z = H.quantize_int4(x.float().numpy())
    assert np.array_equal(y.numpy(), Q.dequantize_int4(p, s, z).astype(np.float32))
    # fp16 input still takes the fp16 path and returns fp16
    h = x.to(torch.float16)
    assert H.int4_roundtrip(h).dtype == torch.float16
