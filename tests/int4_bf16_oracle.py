"""bf16 activations over the INT4 KV cache: the oracle paths the reference does not have (its INT4 demo runs in fp16).
TEST INFRASTRUCTURE ONLY, built on ``oracle/int4_oracle.py`` and ``oracle/duo_oracle.py``.

* ``quantize_int4``        – K1 of float32 arrays that hold bf16 values (numpy has no bf16): the arithmetic of
  ``int4_oracle.quantize_int4`` on their fp32 values (fp32 min/max, ``scale = (max-min)/15 + 1e-8``, ``zero = min``,
  IEEE division, roundf, clamp, fp16 scale / zero).  fp16 input is handed to ``int4_oracle.quantize_int4`` itself.
* ``dequantize_int4_bf16`` – the bf16 image duo_dequant_int4_bf16 writes: ``bf16_rn(fmaf(q, float(s), float(z)))``.
* ``int4_roundtrip`` / ``int4_attention_core`` – ``duo_oracle``'s INT4 core for bf16 q/k/v: the dequantised K/V are the
  K2 (fp16) values kept in fp32, not rounded again to bf16 (what the INT4 decode kernels attend); P is rounded to
  bf16.  fp16 input goes to ``duo_oracle`` unchanged.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import duo_oracle as O
from oracle import int4_oracle as Q


def is_bf16_valued(x: np.ndarray) -> bool:
    """float32 array whose every value is exactly representable in bf16 (low 16 bits of the encoding zero)."""
    return bool((np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & 0xFFFF == 0).all())


def round_to_bf16(x: np.ndarray) -> np.ndarray:
    """float32 -> nearest bf16 (ties to even), returned as float32 (finite inputs)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def quantize_int4(x: np.ndarray, group_size: int = 128):
    """float16 array, or float32 array holding bf16 values, ``[..., head_dim]`` -> (packed uint8 ``[..., head_dim//2]``,
    scale fp16 ``[..., head_dim//group_size]``, zero fp16 same shape)."""
    if x.dtype == np.float16:
        return Q.quantize_int4(x, group_size)
    assert x.dtype == np.float32 and is_bf16_valued(x), x.dtype
    hd = x.shape[-1]
    ng = hd // group_size
    xf = x.reshape(*x.shape[:-1], ng, group_size)
    gmin = xf.min(axis=-1, keepdims=True)
    gmax = xf.max(axis=-1, keepdims=True)
    scale = ((gmax - gmin) / np.float32(15.0) + np.float32(1e-8)).astype(np.float32)
    qf = (xf - gmin) / scale
    qf = np.sign(qf) * np.floor(np.abs(qf) + np.float32(0.5))
    q = np.clip(qf, 0.0, 15.0).astype(np.uint8).reshape(*x.shape[:-1], hd)
    packed = ((q[..., 0::2] << 4) | q[..., 1::2]).astype(np.uint8)
    return packed, scale[..., 0].astype(np.float16), gmin[..., 0].astype(np.float16)


def dequantize_int4_bf16(packed: np.ndarray, scale: np.ndarray, zero: np.ndarray, group_size: int = 128):
    """-> float32 ``[..., head_dim]`` holding bf16 values: the exact ``q s + z`` rounded once to fp32 (the fma), then
    to bf16."""
    codes = Q.unpack_codes(packed)
    hd = codes.shape[-1]
    ng = hd // group_size
    c = codes.reshape(*codes.shape[:-1], ng, group_size).astype(np.float64)
    s = scale.astype(np.float16).astype(np.float64)[..., None]
    z = zero.astype(np.float16).astype(np.float64)[..., None]
    f32 = (c * s + z).astype(np.float32)  # q s + z is exact in fp64 (4 + 11 significant bits, fp16 exponents)
    return round_to_bf16(f32).reshape(*codes.shape[:-1], hd)


def int4_roundtrip(x: torch.Tensor) -> torch.Tensor:
    """K1 -> K2 of a ``[..., 128]`` tensor; bf16 input: K1 of its fp32 values, K2's fp16 values returned as float32."""
    if x.dtype != torch.bfloat16:
        return O.int4_roundtrip(x)
    p, s, z = quantize_int4(x.detach().cpu().float().numpy())
    return torch.from_numpy(Q.dequantize_int4(p, s, z).astype(np.float32))


def int4_attention_core(q, k, v, past, n_full, groups, sink, recent):
    """``duo_oracle.int4_attention_core`` (demo/w8a8kv4_llama.py:215-278 after RoPE) for fp16 or bf16 q/k/v: the first
    call attends the raw k/v, later calls the round trip of everything; ``past`` holds the round-tripped values
    (float32 for bf16)."""
    kq, vq = int4_roundtrip(k), int4_roundtrip(v)
    if past is None:
        out = O.flash_attn_contract(q, k, v, causal=True)
        _, new_past = O.tuple_attention_core(q, kq, vq, None, n_full, groups, sink, recent)
        return out, new_past
    return O.tuple_attention_core(q, kq, vq, past, n_full, groups, sink, recent)
