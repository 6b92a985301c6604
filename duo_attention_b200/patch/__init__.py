"""Drop-in for ``duo_attn.patch`` (reference: duo_attn/patch/__init__.py:58-82, llama.py:504-598,
mistral.py:504-598): same function names, argument order and error behaviour; underneath, the patched
forward calls the CUDA kernels instead of FlashAttention-2 + torch.cat + cache copies."""
from __future__ import annotations

from ..kv_cache import DuoAttentionStaticINT4KVCache, DuoAttentionStaticKVCache, DuoKVCache
from .hf_driver import install as _install
from .reorder import reorder_full_attn_heads, reorder_linear_weights

_SUPPORTED_LLAMA = ("llama",)
_SUPPORTED_MISTRAL = ("mistral", "mixtral")


def enable_llama_duo_attention_eval(model, full_attention_heads, sink_size, recent_size):
    _install(model, full_attention_heads, sink_size, recent_size, logits_float=True)


def enable_mistral_duo_attention_eval(model, full_attention_heads, sink_size, recent_size):
    _install(model, full_attention_heads, sink_size, recent_size, logits_float=True)


def enable_duo_attention_eval(model, full_attention_heads, sink_size, recent_size):
    """duo_attn/patch/__init__.py:58-82.  Must run before the model is moved to the GPU / TP-wrapped,
    like the reference (README.md:141-150); mutates the attention weights in place."""
    print(f"Enabling DuoAttention evaluation using sink size {sink_size} and recent size {recent_size}")
    mt = model.config.model_type
    if "llama" in mt:
        enable_llama_duo_attention_eval(model, full_attention_heads, sink_size, recent_size)
    elif "mistral" in mt or "mixtral" in mt:
        enable_mistral_duo_attention_eval(model, full_attention_heads, sink_size, recent_size)
    else:
        raise ValueError(f"Model type {model.config.model_type} not supported")


def enable_llama_duo_attention_static_kv_cache_eval(model, full_attention_heads, rope: str = "hf"):
    """llama.py:557-598.  The caller builds a ``DuoAttentionStaticKVCache`` (which carries sink/recent)
    and passes it as ``past_key_values`` every call (benchmark_static.py:58-103).  Llama static eval
    keeps bf16 logits (static_kv_cache.py:360-364).

    ``rope`` (extra keyword): "hf" rotates with HuggingFace's tables in the activation dtype, bit-exact with the
    tuple path (the parity target north_star names); "flashinfer" reproduces what the reference's static forward
    actually calls (llama.py:347-352 -> flashinfer_utils.py:29-59): fp32 angles on the fly, one rounding, linear
    ``rope_scaling["factor"]`` only."""
    _install(model, full_attention_heads, None, None, logits_float=False, rope=rope)


def enable_mistral_duo_attention_static_kv_cache_eval(model, full_attention_heads, rope: str = "hf"):
    """mistral.py:557-598; mistral's static driver returns fp32 logits (static_kv_cache.py:612-617)."""
    _install(model, full_attention_heads, None, None, logits_float=True, rope=rope)


__all__ = [
    "enable_duo_attention_eval",
    "enable_llama_duo_attention_eval",
    "enable_mistral_duo_attention_eval",
    "enable_llama_duo_attention_static_kv_cache_eval",
    "enable_mistral_duo_attention_static_kv_cache_eval",
    "DuoAttentionStaticKVCache",
    "DuoAttentionStaticINT4KVCache",
    "DuoKVCache",
    "reorder_linear_weights",
    "reorder_full_attn_heads",
]
