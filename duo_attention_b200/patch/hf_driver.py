"""Model / decoder-layer / attention forwards that route HuggingFace Llama & Mistral through the
CUDA kernels.

The reference swaps ``.forward`` on ForCausalLM / Model / DecoderLayer / Attention with HF-4.34-style
functions (duo_attn/patch/tuple_kv_cache.py:241-490, static_kv_cache.py:318-567) and an attention
forward that calls FlashAttention-2 twice (llama.py:146-306, :309-434).  Here the causal-LM forward is
replaced by one driver written against attributes that are stable across transformers versions (the
``nn.Linear`` projections, norms, ``embed_tokens``, ``lm_head``, ``rotary_emb``), and each layer's
attention is ONE call into ``DuoKVCache.attend`` (RoPE+append → fused mixed-head attention → ring
commit, all CUDA).  Call protocol is the reference's (SURVEY.md §8b):

    out = model(input_ids=ids, past_key_values=None | cache, use_cache=True)
    out.logits[:, -1, :]          # only the last position is produced
    out.past_key_values           # feed back verbatim (a DuoKVCache here, a tuple in the reference)
"""
from __future__ import annotations

import types
from typing import Optional

import torch
from transformers.modeling_outputs import CausalLMOutputWithPast

from .. import _C
from ..kv_cache import DuoKVCache, DuoRaggedKVCache, model_geometry, ragged_prefill_plan


class _AttnPlan:
    """Per-attention-module state created at enable time."""

    def __init__(self, n_full, n_kv, group, head_dim):
        self.n_full, self.n_kv, self.group, self.head_dim = n_full, n_kv, group, head_dim
        self.wqkv = None
        self.bqkv = None


def _fuse_qkv(attn):
    """Concatenate the (already reordered) q/k/v projections into one GEMM operand on first use and
    re-point the three nn.Linear weights at views of it (no extra memory)."""
    plan = attn._duo_plan
    w = torch.cat([attn.q_proj.weight.data, attn.k_proj.weight.data, attn.v_proj.weight.data], dim=0).contiguous()
    nq, nk = attn.q_proj.weight.shape[0], attn.k_proj.weight.shape[0]
    attn.q_proj.weight.data = w[:nq]
    attn.k_proj.weight.data = w[nq : nq + nk]
    attn.v_proj.weight.data = w[nq + nk :]
    plan.wqkv = w
    if attn.q_proj.bias is not None:
        plan.bqkv = torch.cat([attn.q_proj.bias.data, attn.k_proj.bias.data, attn.v_proj.bias.data]).contiguous()


def _fuse_gate_up(mlp):
    """gate_proj | up_proj as one GEMM operand (views re-pointed, no extra memory)."""
    w = torch.cat([mlp.gate_proj.weight.data, mlp.up_proj.weight.data], dim=0).contiguous()
    n = mlp.gate_proj.weight.shape[0]
    mlp.gate_proj.weight.data = w[:n]
    mlp.up_proj.weight.data = w[n:]
    mlp._duo_wgu = w


def _mlp_forward(mlp, x):
    """LlamaMLP / MistralMLP: down(silu(gate(x)) * up(x)) with one fused gate|up GEMM and one fused SiLU*mul."""
    from .. import ops

    w = getattr(mlp, "_duo_wgu", None)
    if w is None or w.device != x.device:
        _fuse_gate_up(mlp)
        w = mlp._duo_wgu
    return mlp.down_proj(ops.silu_mul(torch.nn.functional.linear(x, w)))


def _fusable(layer):
    m = layer.mlp
    return (all(hasattr(m, n) for n in ("gate_proj", "up_proj", "down_proj"))
            and m.gate_proj.bias is None and m.up_proj.bias is None
            and type(getattr(m, "act_fn", None)).__name__ in ("SiLU", "SiLUActivation")
            and hasattr(layer.input_layernorm, "variance_epsilon"))


def duo_attention_layer_forward(attn, hidden_states, cos, sin, kv_cache: DuoKVCache, layer_idx: int,
                                rope_mode: int = _C.ROPE_HF, project: bool = True, chunk_lengths=None, verify=False):
    """The hot path of one layer (replaces llama.py:146-306 / :309-434).  ``project=False`` returns the attention
    context ``[B, S, Hq * D]`` before ``o_proj`` (the pipelined tensor-parallel driver projects it block by block).
    ``chunk_lengths``: the rows of a DuoRaggedKVCache take packed chunks of these lengths (``attend_rows``).
    ``verify``: the chunk is a verify chunk of drafted tokens (``kv_cache.verify``), committed later by ``accept``."""
    plan = attn._duo_plan
    if plan.wqkv is None or plan.wqkv.device != hidden_states.device:
        _fuse_qkv(attn)
    B, S, _ = hidden_states.shape
    qkv = torch.nn.functional.linear(hidden_states, plan.wqkv, plan.bqkv)
    out = torch.empty(B, S, plan.n_kv * plan.group, plan.head_dim, dtype=qkv.dtype, device=qkv.device)
    if verify:
        kv_cache.verify(layer_idx, qkv, cos, sin, rope_mode, out)
    elif chunk_lengths is None:
        kv_cache.attend(layer_idx, qkv, cos, sin, rope_mode, out)
    else:
        kv_cache.attend_rows(layer_idx, qkv, cos, sin, rope_mode, out, chunk_lengths)
    return attn.o_proj(out.view(B, S, -1)) if project else out.view(B, S, -1)


def _tp_layer_pipelined(layer, ctx, h, next_norm, group, n_blocks):
    """Head-parallel TP, large chunks: the two bandwidth-bound all-reduces of a layer (attention output and MLP output,
    duo_attn/utils.py:174-179 — 256 MiB each for a 32K-token chunk) overlapped with the GEMMs by row blocks.  Block b's
    row-parallel o_proj partial is all-reduced (NCCL, asynchronously on the communicator's stream) while block b+1 is
    projected; its add+RMSNorm -> gate|up -> SiLU*mul -> down runs while later blocks are still in flight, and the MLP
    partials are reduced the same way.  Only the last block's exchange of each site is exposed.
    ctx ``[1, S, Hq_local * D]``, h ``[1, S, hidden]`` (updated in place); returns the normalised input of the next
    layer."""
    import torch.distributed as dist

    from .. import ops

    S = ctx.shape[1]
    step = (S + n_blocks - 1) // n_blocks
    spans = [(r, min(S, r + step)) for r in range(0, S, step)]
    ln2 = layer.post_attention_layernorm
    parts, works = [], []
    for r0, r1 in spans:
        a = layer.self_attn.o_proj(ctx[:, r0:r1])
        works.append(dist.all_reduce(a, op=dist.ReduceOp.SUM, group=group, async_op=True))
        parts.append(a)
    mparts, mworks = [], []
    for (r0, r1), a, w in zip(spans, parts, works):
        w.wait()  # stream-level wait: the host keeps enqueueing
        x, _ = ops.add_rmsnorm(a, h[:, r0:r1], ln2.weight, ln2.variance_epsilon)
        m = _mlp_forward(layer.mlp, x)
        mworks.append(dist.all_reduce(m, op=dist.ReduceOp.SUM, group=group, async_op=True))
        mparts.append(m)
    outs = []
    for (r0, r1), m, w in zip(spans, mparts, mworks):
        w.wait()
        x, _ = ops.add_rmsnorm(m, h[:, r0:r1], next_norm.weight, next_norm.variance_epsilon)
        outs.append(x)
    return torch.cat(outs, dim=1)


def plans_head_dim(model):
    return model.model.layers[0].self_attn._duo_plan.head_dim


def _rope_theta_and_scale(cfg):
    """(rope_theta, linear factor) the way the reference's static forward reads them (llama.py:347-350:
    ``config.rope_scaling["factor"]`` if set, whatever the scaling type), across transformers config layouts."""
    rp = getattr(cfg, "rope_parameters", None) or {}
    rs = getattr(cfg, "rope_scaling", None) or {}
    theta = getattr(cfg, "rope_theta", None) or rp.get("rope_theta") or 10000.0
    factor = rs.get("factor") or rp.get("factor") or 1.0
    return float(theta), float(factor)


def _new_dynamic_cache(model, batch_size, first_len):
    plans = [layer.self_attn._duo_plan for layer in model.model.layers]
    p = next(model.parameters())
    cfg = model.config
    return DuoKVCache(
        num_layers=len(plans),
        num_heads=cfg.num_attention_heads,
        num_kv_heads=cfg.num_key_value_heads,
        head_dim=plans[0].head_dim,
        num_full_kv_head_list=[pl.n_full for pl in plans],
        batch_size=batch_size,
        max_size=max(256, 2 * first_len),
        sink_size=model._duo_sink,
        recent_size=model._duo_recent,
        dtype=p.dtype,
        device=p.device,
        stage_cap=first_len,
        growable=True,
    )


def duo_causal_lm_forward(self, input_ids: Optional[torch.LongTensor] = None, attention_mask=None,
                          position_ids=None, past_key_values=None, inputs_embeds=None, labels=None,
                          use_cache=None, **kwargs):
    """Patched ``ForCausalLM.forward``.  ``past_key_values`` is ``None`` (first call: a growable
    DuoKVCache is created, tuple-path behaviour) or a ``DuoKVCache`` / ``DuoAttentionStaticKVCache``
    (static-path behaviour, benchmark_static.py:58-103).  Padding is not supported, exactly like the
    reference's duo forwards (llama.py:154).  With a ``DuoRaggedKVCache``, rows set idle
    (``cache.set_active(b, False)``) still go through the GEMMs but not through attention, and their cache is not
    touched: their logits are meaningless and should be ignored.

    ``chunk_lengths=[n_0, ..., n_{B-1}]`` with a ``DuoRaggedKVCache`` prefills many rows in one forward: ``input_ids``
    ``[1, T]`` holds the rows' chunks packed back to back (T = the sum; rows with 0 tokens are not touched), token t of
    row b at position ``row_lengths[b] + t``.  The GEMMs run once on the T packed tokens, and each layer's attention is
    one ``attend_rows`` call.  The logits are ``[B, 1, vocab]``: row b's are those of its last packed token (meaningless
    for a row with no tokens).  Not with tensor-parallel or sequence-sharded models.

    ``verify=True`` verifies drafted tokens (speculative decoding): ``input_ids`` ``[B, S]`` holds, per row, the last
    sampled token and S - 1 drafts; every layer takes them as a verify chunk (``cache.verify``: token t attends what a
    one-token step at its position would), and the logits are ``[B, S, vocab]``, one per position.  Nothing is committed
    and the occupancy does not move: ``cache.accept(a)`` (static caches) or ``cache.accept(counts)`` (a
    ``DuoRaggedKVCache``, one count per row) keeps the accepted tokens.  Needs a cache; not with tensor-parallel or
    sequence-sharded models, packed chunks, or an attached ``DuoDecodeGraph``."""
    if labels is not None:
        raise ValueError("the DuoAttention eval forward does not compute a loss")
    base = self.model
    if inputs_embeds is None:
        inputs_embeds = base.embed_tokens(input_ids)
    B, S, _ = inputs_embeds.shape
    cache = past_key_values
    if cache is None:
        cache = _new_dynamic_cache(self, B, S)
    elif not isinstance(cache, DuoKVCache):
        raise ValueError("past_key_values must be None or a DuoKVCache produced by this model")
    ragged = isinstance(cache, DuoRaggedKVCache)
    chunk_lengths = kwargs.get("chunk_lengths")
    packed = chunk_lengths is not None
    verify = bool(kwargs.get("verify", False))
    if verify and (past_key_values is None or packed or getattr(self, "_duo_tp", False)
                   or getattr(self, "_duo_seq", None) is not None):
        raise ValueError("verify=True needs a DuoKVCache as past_key_values, no chunk_lengths, and a model that is "
                         "neither tensor-parallel nor sequence-sharded")
    if packed:
        # the rows' chunks packed into one sequence: per-token positions, [T, D] RoPE tables as for one sequence below
        if not ragged:
            raise ValueError("chunk_lengths needs a DuoRaggedKVCache as past_key_values")
        if getattr(self, "_duo_tp", False) or getattr(self, "_duo_seq", None) is not None:
            raise ValueError("DuoRaggedKVCache is not supported with tensor-parallel or sequence-sharded models")
        if B != 1:
            raise ValueError(f"chunk_lengths takes the rows' chunks packed into input_ids [1, T] (got batch {B})")
        plan = ragged_prefill_plan(chunk_lengths, S, cache.batch_size)
        chunk_lengths = [int(n) for n in chunk_lengths]
        if position_ids is None:
            position_ids = torch.cat([torch.arange(n0, n0 + n, dtype=torch.long) for n0, n in
                                      zip(cache.row_lengths, chunk_lengths)])[None].to(inputs_embeds.device)
        else:
            position_ids = position_ids.view(1, S).long()
        # row b's next-token logits: its last packed token (a row without tokens reads token 0: meaningless)
        last = torch.tensor([max(o + n - 1, 0) for o, n in zip(plan["offsets"], chunk_lengths)],
                            device=inputs_embeds.device)
    elif ragged:
        # rows at different lengths: per-row positions and RoPE tables, one duo_decode_ragged launch per layer
        if S * cache.num_kv_groups > cache.max_rows:
            raise ValueError(f"a DuoRaggedKVCache takes decode-sized chunks (group x q_len <= {cache.max_rows}, got "
                             f"{S} tokens): prefill each row through cache.row(b)")
        if getattr(self, "_duo_tp", False) or getattr(self, "_duo_seq", None) is not None:
            raise ValueError("DuoRaggedKVCache is not supported with tensor-parallel or sequence-sharded models")
        if position_ids is None:
            first = torch.tensor(cache.row_lengths, dtype=torch.long, device=inputs_embeds.device)
            position_ids = first[:, None] + torch.arange(S, dtype=torch.long, device=inputs_embeds.device)[None]
        else:
            position_ids = position_ids.view(B, S).long()
    else:
        past_len = cache.kv_seq_len
        if position_ids is None:
            position_ids = torch.arange(past_len, past_len + S, dtype=torch.long, device=inputs_embeds.device)[None]
        else:
            position_ids = position_ids.view(-1, S).long()[:1]
    rope_mode = getattr(self, "_duo_rope_mode", _C.ROPE_HF)
    if ragged and not packed and rope_mode == _C.ROPE_FP32:  # [B, S, D] fp32 tables, the flashinfer formula below per row
        theta, factor = _rope_theta_and_scale(self.config)
        pos = position_ids.to(torch.float32) / factor
        idx = torch.arange(plans_head_dim(self) // 2, dtype=torch.float32, device=pos.device)
        ang = pos[..., None] * torch.pow(torch.tensor(theta, device=pos.device), -2.0 * idx / plans_head_dim(self))
        cos, sin = torch.cat([ang.cos(), ang.cos()], -1).contiguous(), torch.cat([ang.sin(), ang.sin()], -1).contiguous()
    elif ragged and not packed:
        cos, sin = base.rotary_emb(inputs_embeds, position_ids)  # [B, S, D] in the activation dtype
        cos, sin = cos.contiguous(), sin.contiguous()
    elif rope_mode == _C.ROPE_FP32:
        # the reference's STATIC path rotates with flashinfer: fp32 angles computed on the fly from the first position
        # of the chunk, linear `rope_scale` only (llama.py:347-352, flashinfer_utils.py:29-59)
        theta, factor = _rope_theta_and_scale(self.config)
        pos = position_ids[0].to(torch.float32) / factor
        idx = torch.arange(plans_head_dim(self) // 2, dtype=torch.float32, device=pos.device)
        ang = pos[:, None] * torch.pow(torch.tensor(theta, device=pos.device), -2.0 * idx / plans_head_dim(self))[None]
        cos, sin = torch.cat([ang.cos(), ang.cos()], -1).contiguous(), torch.cat([ang.sin(), ang.sin()], -1).contiguous()
    else:
        cos, sin = base.rotary_emb(inputs_embeds, position_ids)  # [1, S, D] in the activation dtype
        cos, sin = cos[0].contiguous(), sin[0].contiguous()
    h = inputs_embeds.contiguous() if input_ids is not None else inputs_embeds.clone()  # updated in place below
    tp_on = getattr(self, "_duo_tp", False)
    seq_on = getattr(self, "_duo_seq", None) is not None  # sequence-sharded decode: attention output needs no exchange
    if tp_on:
        from ..tp import all_reduce_sum
    layers = list(base.layers)
    if h.is_cuda and h.shape[-1] % 8 == 0 and all(_fusable(l) for l in layers):
        # fused glue: residual add + RMSNorm in one launch, gate|up in one GEMM, SiLU*up in one launch
        from .. import ops

        comm = getattr(self, "_duo_comm", None) if tp_on else None
        if comm is not None and not comm.usable(h):
            comm = None  # large chunks are bandwidth-bound: NCCL

        def reduce_add_norm(part, res, w, eps):
            """sum over ranks (if TP) + residual add + RMSNorm: one fused peer-memory kernel for small exchanges
            (tp.FusedAllReduce), otherwise NCCL all-reduce followed by duo_add_rmsnorm."""
            if comm is not None:
                return comm.add_rmsnorm(part, res, w, eps)
            if tp_on:  # row-parallel partials -> one all-reduce per site (NCCL over NVLink)
                part = all_reduce_sum(part, self._duo_tp_group)
            return ops.add_rmsnorm(part, res, w, eps)

        x, _ = ops.add_rmsnorm(h, None, layers[0].input_layernorm.weight, layers[0].input_layernorm.variance_epsilon)
        pipe_rows = getattr(self, "_duo_tp_pipeline_rows", 4096)
        pipelined = tp_on and not seq_on and comm is None and B == 1 and S >= pipe_rows
        for idx, layer in enumerate(layers):
            if pipelined and idx + 1 < len(layers):
                ctx = duo_attention_layer_forward(layer.self_attn, x, cos, sin, cache, idx, rope_mode, project=False)
                x = _tp_layer_pipelined(layer, ctx, h, layers[idx + 1].input_layernorm, self._duo_tp_group,
                                        getattr(self, "_duo_tp_pipeline_blocks", 2))
                continue
            a = duo_attention_layer_forward(layer.self_attn, x, cos, sin, cache, idx, rope_mode,
                                            chunk_lengths=chunk_lengths, verify=verify)
            ln2 = layer.post_attention_layernorm
            if seq_on:  # merged attention output is already complete (and bit-identical) on every rank
                x, h = ops.add_rmsnorm(a, h, ln2.weight, ln2.variance_epsilon)
            else:
                x, h = reduce_add_norm(a, h, ln2.weight, ln2.variance_epsilon)
            m = _mlp_forward(layer.mlp, x)
            if idx + 1 < len(layers):
                nxt = layers[idx + 1].input_layernorm
                x, h = reduce_add_norm(m, h, nxt.weight, nxt.variance_epsilon)
            else:  # only the last position feeds the head (tuple_kv_cache.py:283-288)
                if tp_on and comm is None:
                    m = all_reduce_sum(m, self._duo_tp_group)
                if verify:  # every position feeds the head
                    m_last, h_last = m, h
                elif packed:
                    m_last, h_last = m[0, last, None, :].contiguous(), h[0, last, None, :].contiguous()
                else:
                    m_last, h_last = m[:, -1:, :].contiguous(), h[:, -1:, :].contiguous()
                if comm is not None:
                    x, _ = comm.add_rmsnorm(m_last, h_last, base.norm.weight, base.norm.variance_epsilon)
                else:
                    x, _ = ops.add_rmsnorm(m_last, h_last, base.norm.weight, base.norm.variance_epsilon)
        h = x
    else:
        for idx, layer in enumerate(layers):
            res = h
            x = layer.input_layernorm(h)
            x = duo_attention_layer_forward(layer.self_attn, x, cos, sin, cache, idx, rope_mode,
                                            chunk_lengths=chunk_lengths, verify=verify)
            if tp_on and not seq_on:
                x = all_reduce_sum(x, self._duo_tp_group)
            h = res + x
            res = h
            x = layer.post_attention_layernorm(h)
            x = layer.mlp(x)
            if tp_on:
                x = all_reduce_sum(x, self._duo_tp_group)
            h = res + x
        h = base.norm(h if verify else h[0, last, None, :] if packed else h[:, -1:, :])
    if cache.dev_state is not None and not packed and not verify:  # (attend_rows leaves row_state at the rows' new occupancy)  # device-resident occupancy (graph replay): advance it on the stream
        cache.advance_device(S)
    logits = self.lm_head(h)
    if getattr(self, "_duo_logits_float", True):
        logits = logits.float()
    return CausalLMOutputWithPast(logits=logits, past_key_values=cache if use_cache is not False else None)


def install(model, full_attention_heads, sink_size, recent_size, logits_float=True, rope="hf"):
    """Shared body of enable_{llama,mistral}_duo_attention_eval (llama.py:504-554): reorder weights so
    retrieval heads come first, remember the split, swap the model forward."""
    from .reorder import reorder_linear_weights, reorder_full_attn_heads

    geo = model_geometry(model)
    n_kv, head_dim = geo["num_kv_heads"], geo["head_dim"]
    group = geo["num_heads"] // n_kv
    for idx, layer in enumerate(model.model.layers):
        module = layer.self_attn
        gate = torch.tensor(full_attention_heads[idx], device=geo["device"], dtype=geo["dtype"])
        reorder_linear_weights(module.q_proj, gate, group * head_dim, "out")
        reorder_linear_weights(module.k_proj, gate, head_dim, "out")
        reorder_linear_weights(module.v_proj, gate, head_dim, "out")
        reorder_linear_weights(module.o_proj, gate, group * head_dim, "in")
        gate = reorder_full_attn_heads(gate)
        module.sink_size = sink_size
        module.recent_size = recent_size
        module.register_buffer("full_attention_heads", gate)
        module._duo_plan = _AttnPlan(int((gate > 0.5).sum().item()), n_kv, group, head_dim)
    model._duo_sink = sink_size
    model._duo_recent = recent_size
    model._duo_logits_float = logits_float
    if rope not in ("hf", "flashinfer"):
        raise ValueError(f"rope must be 'hf' or 'flashinfer', got {rope!r}")
    model._duo_rope_mode = _C.ROPE_FP32 if rope == "flashinfer" else _C.ROPE_HF
    model.forward = types.MethodType(duo_causal_lm_forward, model)
    return model
