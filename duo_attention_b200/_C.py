"""ctypes binding of csrc/libduo_b200.so (C ABI declared in include/duo_b200.h).

The library is mandatory: there is deliberately no fallback path.  ``load()`` raises
``RuntimeError`` with build instructions if the shared object is absent.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DUO_B200_LIB") or os.path.join(_HERE, "csrc", "libduo_b200.so")  # env: tuning builds

DUO_OK, DUO_EINVAL, DUO_EOVERFLOW, DUO_ECUDA, DUO_EWORKSPACE = 0, -1, -2, -3, -4
DT_BF16, DT_FP16 = 0, 1
KV_SAME, KV_INT4 = 0, 1
ROPE_NONE, ROPE_HF, ROPE_FP32 = 0, 1, 2
ROPE_SKIP_Q = 0x100
DECODE_MAX_Q = 16
DECODE_MAX_Q_INT4 = 8  # packed rows (group x q_len) of duo_decode_fused on an INT4 cache
RAGGED_MAX_BATCH = 64  # rows of one duo_decode_ragged batch
ROW_IDLE = 1  # row_state[b][3] flag: row b sits out the batched launches

# every symbol include/duo_b200.h declares (checked by tests/test_cabi_symbols.py)
SYMBOLS = [
    "duo_layer_create", "duo_layer_destroy", "duo_workspace_bytes", "duo_rope_append", "duo_attention",
    "duo_attention_mma", "duo_decode_fused", "duo_decode_ragged", "duo_ragged_workspace_bytes",
    "duo_decode_ragged_int4", "duo_ragged_int4_workspace_bytes", "duo_layer_create_pooled", "duo_decode_ragged_pooled",
    "duo_decode_ragged_shared", "duo_ragged_shared_workspace_bytes", "duo_attention_shared", "duo_prefill_ragged",
    "duo_ragged_state_advance", "duo_state_advance", "duo_state_set", "duo_stream_commit", "duo_quant_int4", "duo_dequant_int4", "duo_dequant_int4_bf16", "duo_add_rmsnorm", "duo_silu_mul",
    "duo_attention_partial", "duo_merge_partials", "duo_attention_seq", "duo_decode_fused_seq", "duo_prefill_seq",
    "duo_attention_seq_int4", "duo_decode_fused_seq_int4", "duo_decode_fused_seq_shared", "duo_seq_shared_workspace_bytes",
    "duo_prefill_seq_shared",
    "duo_seqcomm_data_bytes", "duo_seqcomm_flag_bytes", "duo_seqcomm_create", "duo_seqcomm_destroy", "duo_seq_merge",
    "duo_comm_data_bytes", "duo_comm_flag_bytes", "duo_comm_create", "duo_comm_destroy", "duo_allreduce_add_rmsnorm",
    "duo_last_error_string", "duo_version",
]


class LayerDesc(C.Structure):
    _fields_ = [
        ("full_k", C.c_void_p), ("full_v", C.c_void_p), ("ring_k", C.c_void_p), ("ring_v", C.c_void_p),
        ("full_k_scale", C.c_void_p), ("full_k_zero", C.c_void_p), ("full_v_scale", C.c_void_p),
        ("full_v_zero", C.c_void_p), ("ring_k_scale", C.c_void_p), ("ring_k_zero", C.c_void_p),
        ("ring_v_scale", C.c_void_p), ("ring_v_zero", C.c_void_p),
        ("full_cap", C.c_int64),
        ("batch", C.c_int32), ("n_full", C.c_int32), ("n_stream", C.c_int32), ("group", C.c_int32),
        ("head_dim", C.c_int32), ("sink", C.c_int32), ("recent", C.c_int32), ("stage_cap", C.c_int32),
        ("dtype", C.c_int32), ("kv_format", C.c_int32),
    ]


class CacheState(C.Structure):
    _fields_ = [("full_len", C.c_int64), ("total", C.c_int64), ("lo", C.c_int64), ("device_state", C.c_void_p),
                ("seq_rank", C.c_int32), ("seq_world", C.c_int32), ("seq_block", C.c_int32), ("seq_reserved", C.c_int32)]


class SeqCommDesc(C.Structure):
    _fields_ = [("data", C.c_void_p * 8), ("flags", C.c_void_p * 8), ("local_state", C.c_void_p),
                ("rank", C.c_int32), ("world", C.c_int32), ("max_rows", C.c_int32)]


class CommDesc(C.Structure):
    _fields_ = [("data", C.c_void_p * 8), ("flags", C.c_void_p * 8), ("local_state", C.c_void_p),
                ("rank", C.c_int32), ("world", C.c_int32), ("hidden", C.c_int32), ("max_rows", C.c_int32),
                ("dtype", C.c_int32)]


_lib = None


def load():
    """Load libduo_b200.so once and declare the prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: the CUDA extension is mandatory (no fallback). Build it with "
            "`python -c 'import __graft_entry__ as g; g.build()'` or `make -C duo_attention_b200/csrc`."
        )
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, f32, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t
    lib.duo_layer_create.argtypes = [C.POINTER(LayerDesc), C.POINTER(vp)]
    lib.duo_layer_create.restype = C.c_int
    lib.duo_layer_create_pooled.argtypes = [C.POINTER(LayerDesc), i64, C.POINTER(vp)]
    lib.duo_layer_create_pooled.restype = C.c_int
    lib.duo_layer_destroy.argtypes = [vp]
    lib.duo_layer_destroy.restype = None
    lib.duo_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.duo_workspace_bytes.restype = sz
    lib.duo_rope_append.argtypes = [vp, C.POINTER(CacheState), vp, i64, vp, vp, i32, i32, vp]
    lib.duo_rope_append.restype = C.c_int
    for name in ("duo_attention", "duo_attention_mma"):
        fn = getattr(lib, name)
        fn.argtypes = [vp, C.POINTER(CacheState), vp, i64, vp, i32, f32, vp, sz, vp]
        fn.restype = C.c_int
    lib.duo_decode_fused.argtypes = [vp, C.POINTER(CacheState), vp, i64, vp, vp, i32, vp, i32, f32, vp, sz, vp]
    lib.duo_decode_fused.restype = C.c_int
    for name in ("duo_decode_ragged", "duo_decode_ragged_int4"):
        fn = getattr(lib, name)
        fn.argtypes = [vp, vp, i64, vp, i64, vp, vp, i32, vp, i32, f32, vp, sz, vp]
        fn.restype = C.c_int
    lib.duo_decode_ragged_pooled.argtypes = [vp, vp, vp, i64, vp, i64, vp, vp, i32, vp, i32, f32, vp, sz, vp]
    lib.duo_decode_ragged_pooled.restype = C.c_int
    lib.duo_decode_ragged_shared.argtypes = [vp, vp, vp, vp, i64, vp, i64, vp, vp, i32, vp, i32, f32, vp, sz, vp]
    lib.duo_decode_ragged_shared.restype = C.c_int
    lib.duo_attention_shared.argtypes = [vp, vp, i64, C.POINTER(CacheState), vp, i64, vp, i32, f32, vp, sz, vp]
    lib.duo_attention_shared.restype = C.c_int
    lib.duo_prefill_ragged.argtypes = [vp, vp, vp, vp, C.POINTER(i32), C.POINTER(i64), vp, i64, vp, vp, i32, vp, f32,
                                       vp, sz, vp]
    lib.duo_prefill_ragged.restype = C.c_int
    for name in ("duo_ragged_workspace_bytes", "duo_ragged_int4_workspace_bytes", "duo_ragged_shared_workspace_bytes"):
        fn = getattr(lib, name)
        fn.argtypes = [i32, i32]
        fn.restype = sz
    lib.duo_ragged_state_advance.argtypes = [vp, i32, i32, i32, i32, vp]
    lib.duo_ragged_state_advance.restype = C.c_int
    lib.duo_state_advance.argtypes = [vp, i32, i32, i32, vp]
    lib.duo_state_advance.restype = C.c_int
    lib.duo_state_set.argtypes = [vp, i64, i64, i64, vp]
    lib.duo_state_set.restype = C.c_int
    lib.duo_stream_commit.argtypes = [vp, C.POINTER(CacheState), i32, vp]
    lib.duo_stream_commit.restype = C.c_int
    lib.duo_quant_int4.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    lib.duo_quant_int4.restype = C.c_int
    for name in ("duo_dequant_int4", "duo_dequant_int4_bf16"):
        fn = getattr(lib, name)
        fn.argtypes = [vp, vp, vp, i64, vp, vp]
        fn.restype = C.c_int
    lib.duo_add_rmsnorm.argtypes = [vp, vp, vp, vp, vp, i64, i32, f32, i32, vp]
    lib.duo_add_rmsnorm.restype = C.c_int
    lib.duo_silu_mul.argtypes = [vp, vp, i64, i32, i32, vp]
    lib.duo_silu_mul.restype = C.c_int
    lib.duo_attention_partial.argtypes = [vp, i64, vp, i64, vp, vp, i32, f32, vp, sz, vp]
    lib.duo_attention_partial.restype = C.c_int
    for name in ("duo_attention_seq", "duo_attention_seq_int4", "duo_prefill_seq"):
        fn = getattr(lib, name)
        fn.argtypes = [vp, C.POINTER(CacheState), vp, i64, vp, vp, vp, i32, f32, vp, sz, vp]
        fn.restype = C.c_int
    for name in ("duo_decode_fused_seq", "duo_decode_fused_seq_int4"):
        fn = getattr(lib, name)
        fn.argtypes = [vp, C.POINTER(CacheState), vp, i64, vp, vp, i32, vp, vp, vp, f32, vp, sz, vp]
        fn.restype = C.c_int
    lib.duo_decode_fused_seq_shared.argtypes = [vp, vp, i64, C.POINTER(CacheState), vp, i64, vp, vp, i32, vp, vp, vp,
                                                f32, vp, sz, vp]
    lib.duo_decode_fused_seq_shared.restype = C.c_int
    lib.duo_prefill_seq_shared.argtypes = [vp, vp, i64, C.POINTER(CacheState), vp, i64, vp, vp, vp, i32, f32, vp, sz, vp]
    lib.duo_prefill_seq_shared.restype = C.c_int
    lib.duo_seq_shared_workspace_bytes.argtypes = [i32, i32]
    lib.duo_seq_shared_workspace_bytes.restype = sz
    lib.duo_seqcomm_data_bytes.argtypes = [i32, i32]
    lib.duo_seqcomm_data_bytes.restype = sz
    lib.duo_seqcomm_flag_bytes.argtypes = [i32, i32]
    lib.duo_seqcomm_flag_bytes.restype = sz
    lib.duo_seqcomm_create.argtypes = [C.POINTER(SeqCommDesc), C.POINTER(vp)]
    lib.duo_seqcomm_create.restype = C.c_int
    lib.duo_seqcomm_destroy.argtypes = [vp]
    lib.duo_seqcomm_destroy.restype = None
    lib.duo_seq_merge.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.duo_seq_merge.restype = C.c_int
    lib.duo_merge_partials.argtypes = [vp, vp, i32, i64, i32, i32, vp, i32, vp]
    lib.duo_merge_partials.restype = C.c_int
    lib.duo_comm_data_bytes.argtypes = [i32, i32, i32, i32]
    lib.duo_comm_data_bytes.restype = sz
    lib.duo_comm_flag_bytes.argtypes = [i32, i32]
    lib.duo_comm_flag_bytes.restype = sz
    lib.duo_comm_create.argtypes = [C.POINTER(CommDesc), C.POINTER(vp)]
    lib.duo_comm_create.restype = C.c_int
    lib.duo_comm_destroy.argtypes = [vp]
    lib.duo_comm_destroy.restype = None
    lib.duo_allreduce_add_rmsnorm.argtypes = [vp, vp, vp, vp, vp, vp, i32, f32, vp]
    lib.duo_allreduce_add_rmsnorm.restype = C.c_int
    lib.duo_last_error_string.argtypes = []
    lib.duo_last_error_string.restype = C.c_char_p
    lib.duo_version.argtypes = []
    lib.duo_version.restype = C.c_int
    _lib = lib
    return lib


def last_error() -> str:
    return load().duo_last_error_string().decode("utf-8", "replace")


def check(rc: int):
    """Map a C status to the reference's Python error conventions: cache overflow ->
    ValueError (static_kv_cache.py:112-115); anything else -> RuntimeError."""
    if rc == DUO_OK:
        return
    msg = last_error()
    if rc == DUO_EOVERFLOW or rc == DUO_EINVAL:
        raise ValueError(msg)
    raise RuntimeError(f"libduo_b200 error {rc}: {msg}")
