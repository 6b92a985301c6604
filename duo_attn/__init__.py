"""Import-path shim: lets code written against mit-han-lab/duo-attention
(``from duo_attn.utils import load_attn_pattern, sparsify_attention_heads``,
``from duo_attn.patch import enable_duo_attention_eval`` — reference README.md:119-150) run unchanged on
the CUDA implementation in ``duo_attention_b200``."""
