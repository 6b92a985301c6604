"""duo_attention_b200 — H100-native (sm_90a) implementation of DuoAttention's mixed-head attention
hot path behind the reference's own Python API.

Public surface mirrors mit-han-lab/duo-attention:

    from duo_attention_b200.utils import load_attn_pattern, sparsify_attention_heads
    from duo_attention_b200.patch import enable_duo_attention_eval

(the ``duo_attn`` shim package at the repo root re-exports the same names under the reference's
import paths ``duo_attn.utils`` / ``duo_attn.patch``).  All attention math runs in hand-written CUDA
reached through the C ABI in ``include/duo_b200.h`` (``csrc/libduo_b200.so``); there is no CPU or
PyTorch fallback — ops raise if the library is missing or a tensor is not on a CUDA device.
"""
__version__ = "0.1.0"
