"""Head-parallel tensor parallelism for the DuoAttention hot path: one process per GPU, KV heads (with
their q-head groups) sharded across ranks, one all-reduce (sum) on the attention output per layer.

The reference shards the same way through the third-party ``tensor_parallel`` library inside ONE process
(duo_attn/utils.py:132-227: q/k/v split by KV-head chunks on dim 0, o_proj on dim 1, outputs "sum",
``full_attention_heads`` buffer split on dim 0).  Differences here, on purpose (SURVEY.md §8e):

* one process per GPU + ``torch.distributed`` (NCCL over NVLink on the box, gloo in the CPU tests);
* heads are dealt to ranks BEFORE the retrieval-first reorder so every rank gets a balanced mix — the
  reference reorders first and then cuts contiguous chunks, which hands rank 0 most retrieval heads.

Host-side only: planning, weight slicing and the collective.  The attention itself is the CUDA path.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch
import torch.distributed as dist


class HeadPlan:
    """Which original KV heads each rank owns in each layer (retrieval heads first inside a rank)."""

    def __init__(self, owners: List[List[List[int]]], mask: np.ndarray, world: int):
        self.owners = owners  # [layer][rank] -> list of original kv head ids, retrieval heads first
        self.mask = mask
        self.world = world

    def local_mask(self, rank: int) -> np.ndarray:
        """``[layers, kv_heads / world]`` binary mask of the rank's heads in its local order."""
        return np.array([[float(self.mask[l][h] > 0.5) for h in self.owners[l][rank]]
                         for l in range(len(self.owners))])

    def n_full(self, layer: int, rank: int) -> int:
        return int(sum(self.mask[layer][h] > 0.5 for h in self.owners[layer][rank]))


def plan_heads(mask: Sequence[Sequence[float]], world: int) -> HeadPlan:
    """Deal each layer's retrieval heads round-robin over the ranks (rotating the starting rank from layer
    to layer so the per-rank totals even out), then top every rank up to ``kv_heads / world`` with streaming
    heads."""
    mask = np.asarray(mask, dtype=np.float64)
    L, H = mask.shape
    if H % world != 0:
        raise ValueError(f"{H} KV heads cannot be split over {world} ranks")
    quota = H // world
    owners = []
    load = [0] * world  # retrieval heads handed out so far (across layers)
    for l in range(L):
        full = [h for h in range(H) if mask[l][h] > 0.5]
        stream = [h for h in range(H) if mask[l][h] <= 0.5]
        per_rank: List[List[int]] = [[] for _ in range(world)]
        for h in full:
            # least-loaded rank that still has room in this layer
            cand = [r for r in range(world) if len(per_rank[r]) < quota]
            r = min(cand, key=lambda r_: (load[r_], len(per_rank[r_]), r_))
            per_rank[r].append(h)
            load[r] += 1
        it = iter(stream)
        for r in range(world):
            while len(per_rank[r]) < quota:
                per_rank[r].append(next(it))
        owners.append(per_rank)
    return HeadPlan(owners, mask, world)


@torch.no_grad()
def shard_attention_weights(wq, wk, wv, wo, heads: Sequence[int], group: int, head_dim: int):
    """Rows of q/k/v and columns of o that belong to the given original KV heads, in that order."""
    qrows = torch.cat([torch.arange(h * group * head_dim, (h + 1) * group * head_dim) for h in heads])
    krows = torch.cat([torch.arange(h * head_dim, (h + 1) * head_dim) for h in heads])
    return wq[qrows], wk[krows], wv[krows], wo[:, qrows]


def all_reduce_sum(x: torch.Tensor, group=None) -> torch.Tensor:
    """The per-layer exchange step: sum of the row-parallel o_proj partials (duo_attn/utils.py:174-176)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(x, op=dist.ReduceOp.SUM, group=group)
    return x


def _symmetric_buffer(nbytes: int, device, group):
    """A zeroed byte buffer mapped on every rank of ``group`` (torch symmetric memory: the plumbing; the kernels
    that use it are ours).  Returns ``(tensor, [peer pointers in rank order])``."""
    import torch.distributed._symmetric_memory as symm

    try:  # older torch needs the group enabled explicitly; newer versions do it inside rendezvous
        symm.enable_symm_mem_for_group(group.group_name)
    except Exception:
        pass
    buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
    buf.zero_()
    handle = symm.rendezvous(buf, group)
    return buf, handle, list(handle.buffer_ptrs)


class FusedAllReduce:
    """Peer-memory communicator for ``duo_allreduce_add_rmsnorm`` (csrc/comm.cu): the latency-bound
    exchanges (decode, chunks of <= ``max_rows`` tokens) become one kernel that pushes the partial row to every
    rank over NVLink, sums in rank order and applies the residual add + RMSNorm that follows.

    PyTorch only provides the plumbing here: a symmetric-memory allocation whose peer mappings
    (``buffer_ptrs``) are handed to the C ABI.  Larger chunks keep using NCCL (``all_reduce_sum``)."""

    def __init__(self, group, hidden: int, dtype: torch.dtype, device, max_rows: int = 16):
        import ctypes as C

        from . import _C

        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if not 2 <= self.world <= 8:
            raise ValueError(f"FusedAllReduce supports 2..8 ranks, got {self.world}")
        self.hidden, self.max_rows, self.dtype = int(hidden), int(max_rows), dtype
        dt = _C.DT_BF16 if dtype == torch.bfloat16 else _C.DT_FP16
        lib = _C.load()
        data_bytes = lib.duo_comm_data_bytes(self.world, self.hidden, self.max_rows, dt)
        flag_bytes = lib.duo_comm_flag_bytes(self.world, self.max_rows)
        self.buf, self.handle, ptrs = _symmetric_buffer(data_bytes + flag_bytes, device, self.group)
        self.state = torch.zeros(self.max_rows + 1, dtype=torch.int32, device=device)
        desc = _C.CommDesc()
        for r in range(self.world):
            desc.data[r] = ptrs[r]
            desc.flags[r] = ptrs[r] + data_bytes
        desc.local_state = self.state.data_ptr()
        desc.rank, desc.world, desc.hidden, desc.max_rows, desc.dtype = self.rank, self.world, self.hidden, self.max_rows, dt
        out = C.c_void_p()
        _C.check(lib.duo_comm_create(C.byref(desc), C.byref(out)))
        self._h = out
        torch.cuda.synchronize(device)
        dist.barrier(self.group)  # every rank has zeroed its buffers before anyone pushes into them

    def usable(self, x: torch.Tensor) -> bool:
        return x.numel() // x.shape[-1] <= self.max_rows and x.shape[-1] == self.hidden and x.dtype == self.dtype

    def add_rmsnorm(self, partial: torch.Tensor, residual, weight: torch.Tensor, eps: float):
        """``h = residual + sum_ranks(partial)`` (in place in ``residual`` if given) -> ``(rmsnorm(h) * weight, h)``."""
        from . import _C, ops

        partial = partial if partial.is_contiguous() else partial.contiguous()
        rows = partial.numel() // self.hidden
        out = torch.empty_like(partial)
        if residual is not None:
            assert residual.is_contiguous() and residual.shape == partial.shape and residual.dtype == partial.dtype
            h = residual
        else:
            h = torch.empty_like(partial)
        _C.check(_C.load().duo_allreduce_add_rmsnorm(
            self._h, partial.data_ptr(), None if residual is None else residual.data_ptr(), weight.data_ptr(),
            out.data_ptr(), h.data_ptr(), rows, float(eps), torch.cuda.current_stream(partial.device).cuda_stream))
        ops.LAUNCHES += 1
        return out, h

    def error(self) -> bool:
        """True if some call timed out waiting for a peer (synchronises)."""
        return bool(self.state[self.max_rows].item())

    def __del__(self):
        try:
            from . import _C

            if getattr(self, "_h", None):
                _C.load().duo_comm_destroy(self._h)
                self._h = None
        except Exception:
            pass


def install_allreduce(model, group=None, fused: bool = True):
    """Mark a patched (enable_duo_attention_eval) per-rank model shard as tensor-parallel: the driver then sums the
    row-parallel attention and MLP outputs of every layer over the ranks (duo_attn/utils.py:174-176).  Exchanges of
    <= 16 rows (decode, small chunks) go through the fused peer-memory kernel (``FusedAllReduce``: all-reduce +
    residual add + RMSNorm in one launch), larger ones through NCCL.  ``fused=False`` keeps everything on NCCL.
    Call after the model is on its GPU."""
    model._duo_tp_group = group
    model._duo_tp = True
    model._duo_comm = None
    if fused and dist.is_initialized() and dist.get_world_size(group) > 1:
        p = next(model.parameters())
        if p.is_cuda:
            model._duo_comm = FusedAllReduce(group, model.config.hidden_size, p.dtype, p.device)
    return model


# ----------------------------------------------------------------------------------------------------------------------
# Sequence-sharded decode (scope row f1): every rank holds 1/world of EVERY retrieval head's cache (block-cyclic by
# position), the attention weights and the streaming heads are replicated, the MLP stays tensor-parallel.  Per layer and
# decode step each rank streams its slice of all retrieval heads (perfectly balanced, whatever the head pattern), then
# ONE small exchange merges the (O, log-sum-exp) partials; there is no all-reduce on the attention output at all.
# The reference shards by head only (duo_attn/utils.py:151-179), which leaves up to world-1 ranks idle while one rank
# streams a whole retrieval head.
# ----------------------------------------------------------------------------------------------------------------------
class SeqComm:
    """Peer-memory communicator of ``duo_seq_merge`` (csrc/comm.cu)."""

    def __init__(self, group, device, max_rows: int = 128):
        import ctypes as C

        from . import _C

        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if not 2 <= self.world <= 8:
            raise ValueError(f"SeqComm supports 2..8 ranks, got {self.world}")
        self.max_rows = int(max_rows)
        lib = _C.load()
        data_bytes = lib.duo_seqcomm_data_bytes(self.world, self.max_rows)
        flag_bytes = lib.duo_seqcomm_flag_bytes(self.world, self.max_rows)
        self.buf, self.handle, ptrs = _symmetric_buffer(data_bytes + flag_bytes, device, self.group)
        self.state = torch.zeros(self.max_rows + 1, dtype=torch.int32, device=device)
        desc = _C.SeqCommDesc()
        for r in range(self.world):
            desc.data[r] = ptrs[r]
            desc.flags[r] = ptrs[r] + data_bytes
        desc.local_state = self.state.data_ptr()
        desc.rank, desc.world, desc.max_rows = self.rank, self.world, self.max_rows
        out = C.c_void_p()
        _C.check(lib.duo_seqcomm_create(C.byref(desc), C.byref(out)))
        self._h = out
        torch.cuda.synchronize(device)
        dist.barrier(self.group)

    def merge(self, part_o, part_lse, out, tokens, heads_total, heads_used):
        from . import _C

        dt = _C.DT_BF16 if out.dtype == torch.bfloat16 else _C.DT_FP16
        _C.check(_C.load().duo_seq_merge(self._h, part_o.data_ptr(), part_lse.data_ptr(), out.data_ptr(), tokens,
                                         heads_total, heads_used, dt, torch.cuda.current_stream(out.device).cuda_stream))

    def merge_scattered(self, part_o, part_lse, out, tokens, heads_total, heads_used):
        """``merge`` for prefill-sized chunks, whose rows far exceed ``max_rows``: see :func:`merge_scattered`."""
        merge_scattered(part_o, part_lse, out, tokens, heads_total, heads_used, self.group)

    def error(self) -> bool:
        return bool(self.state[self.max_rows].item())

    def __del__(self):
        try:
            from . import _C

            if getattr(self, "_h", None):
                _C.load().duo_seqcomm_destroy(self._h)
                self._h = None
        except Exception:
            pass


def scatter_counts(n_rows: int, world: int) -> List[int]:
    """Rows each rank merges in :func:`merge_scattered`: consecutive shares, the first ``n_rows % world`` ranks one more."""
    base, extra = divmod(int(n_rows), world)
    return [base + (k < extra) for k in range(world)]


def merge_partials_cuda(o_parts, lse_parts, out):
    """``out[r] = merge over p of (o_parts[p, r], lse_parts[p, r])`` in order p = 0, 1, .. (``duo_merge_partials``).
    ``o_parts`` fp32 ``[n_parts, rows, D]``, ``lse_parts`` fp32 ``[n_parts, rows]``, ``out`` ``[rows, D]``, all contiguous."""
    from . import _C

    dt = _C.DT_BF16 if out.dtype == torch.bfloat16 else _C.DT_FP16
    _C.check(_C.load().duo_merge_partials(o_parts.data_ptr(), lse_parts.data_ptr(), o_parts.shape[0], out.shape[0], 1, 1,
                                          out.data_ptr(), dt, torch.cuda.current_stream(out.device).cuda_stream))


def merge_scattered(part_o, part_lse, out, tokens, heads_total, heads_used, group=None, merge_fn=None):
    """The cross-rank merge of a prefill-sized chunk of the sequence-sharded layout, scattered by rows so that no rank
    holds every rank's partials: of the ``tokens * heads_used`` (token, retrieval head) rows, rank k merges the share
    ``scatter_counts`` gives it.

    1. ``all_to_all_single`` hands each rank its share of the rows from every rank (O and lse together: 516 B a row);
    2. the rank merges its share with ``merge_fn`` (default :func:`merge_partials_cuda`), partials in rank order;
    3. ``all_gather_into_tensor`` collects the merged rows (activation dtype), which are written to
       ``out[..., :heads_used, :]``.

    Every row is merged once, by one rank, in rank order, so every rank ends with the same bits, equal to stacking all
    partials and merging them in rank order.  ``part_o`` fp32 ``[tokens][heads_total][D]``, ``part_lse`` fp32
    ``[tokens][heads_total]`` (any leading shape with these strides), ``out`` ``[tokens][heads_total][D]`` contiguous."""
    merge_fn = merge_fn or merge_partials_cuda
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    D = part_o.shape[-1]
    n = tokens * heads_used
    rows = torch.cat([part_o.reshape(tokens, heads_total, D)[:, :heads_used].reshape(n, D),
                      part_lse.reshape(tokens, heads_total)[:, :heads_used].reshape(n, 1)], 1)
    counts = scatter_counts(n, world)
    mine, most = counts[rank], counts[0]
    got = rows.new_empty(world * mine, D + 1)
    dist.all_to_all_single(got, rows, output_split_sizes=[mine] * world, input_split_sizes=counts, group=group)
    got = got.view(world, mine, D + 1)
    merged = out.new_zeros(most, D)  # every rank contributes `most` rows to the gather; a smaller share is padded
    if mine:
        merge_fn(got[..., :D].contiguous(), got[..., D].contiguous(), merged[:mine])
    gathered = out.new_empty(world * most, D)
    dist.all_gather_into_tensor(gathered, merged, group=group)
    res = torch.cat([gathered[k * most : k * most + counts[k]] for k in range(world)])
    out.view(tokens, heads_total, D)[:, :heads_used] = res.view(tokens, heads_used, D)
    return out


class SeqShardContext:
    def __init__(self, rank, world, block, comm):
        self.rank, self.world, self.block, self.comm = rank, world, block, comm


def install_seq_shard(model, group=None, block: int = 1024, max_rows: int = 128):
    """Decode-phase tensor parallelism with sequence-sharded retrieval heads: ``model`` is a shard built by
    ``shard_model_seq`` (attention replicated, MLP split) and patched with the FULL head mask.  The driver then
    skips the attention-output exchange (the merged attention output is identical on every rank) and keeps the fused
    all-reduce for the MLP; caches are ``DuoSeqShardKVCache`` objects."""
    install_allreduce(model, group, fused=True)
    g = group if group is not None else dist.group.WORLD
    p = next(model.parameters())
    model._duo_seq = SeqShardContext(dist.get_rank(g), dist.get_world_size(g), int(block),
                                     SeqComm(g, p.device, max_rows=max_rows))
    return model


@torch.no_grad()
def shard_model_seq(model, rank: int, world: int):
    """This rank's shard for the sequence-sharded decode: attention projections, embeddings, norms and lm_head
    replicated; MLP gate/up rows and down columns split evenly (outputs "sum", duo_attn/utils.py:163-179)."""
    import copy

    cfg = copy.deepcopy(model.config)
    inter = cfg.intermediate_size
    if inter % world:
        raise ValueError(f"intermediate_size {inter} not divisible by {world}")
    cfg.intermediate_size = inter // world
    shard = type(model)(cfg).to(next(model.parameters()).dtype)
    src_rot, dst_rot = getattr(model.model, "rotary_emb", None), getattr(shard.model, "rotary_emb", None)
    if src_rot is not None and dst_rot is not None:
        for name, buf in src_rot.named_buffers(recurse=False):
            dst_rot.register_buffer(name, buf.detach().clone(), persistent=False)
    lo, hi = rank * (inter // world), (rank + 1) * (inter // world)
    sd = model.state_dict()
    own = shard.state_dict()
    for name, t in own.items():
        src = sd[name]
        if name.endswith("mlp.gate_proj.weight") or name.endswith("mlp.up_proj.weight"):
            t.copy_(src[lo:hi])
        elif name.endswith("mlp.down_proj.weight"):
            t.copy_(src[:, lo:hi])
        else:
            t.copy_(src)
    return shard.eval()


def reshard_heads_to_seq(src_full, owners, mask_row, rank, world, n_tokens, block, dst_full, group=None):
    """Move ONE layer's retrieval cache tensor from the head-parallel layout of the prefill phase to the
    sequence-sharded layout of the decode phase.

    ``src_full``  ``[B, n_f_local, >= n_tokens, ...]``: this rank's retrieval heads (order of ``owners[rank]``, which
                  lists ORIGINAL kv head ids, retrieval heads first — ``HeadPlan.owners[layer]``)
    ``dst_full``  ``[B, n_f_total, >= local_len, ...]``: all retrieval heads in the reference's reordered order
                  (original id ascending), this rank's block-cyclic position slice
    Point-to-point (``batch_isend_irecv``: NCCL on the box, gloo in the CPU test); each rank sends 1/world of its
    heads' rows to every peer.  Device-agnostic: works on any tensors with the layout above."""
    from .seqshard import SeqShardPlan

    plan = SeqShardPlan(world, block)
    full_ids = [h for h in range(len(mask_row)) if mask_row[h] > 0.5]
    gidx = {h: i for i, h in enumerate(full_ids)}                      # original id -> row of dst_full
    mine = [h for h in owners[rank] if mask_row[h] > 0.5]
    ops, keep = [], []
    my_len = plan.local_len(rank, n_tokens)
    for peer in range(world):
        pos = plan.positions(peer, n_tokens).to(src_full.device)
        theirs = [h for h in owners[peer] if mask_row[h] > 0.5]
        if peer == rank:
            for i, h in enumerate(mine):
                dst_full[:, gidx[h], :my_len] = src_full[:, i].index_select(1, pos)
            continue
        if mine and len(pos):
            send = src_full[:, : len(mine)].index_select(2, pos).contiguous()
            keep.append(send)
            ops.append(dist.P2POp(dist.isend, send, peer, group))
        if theirs and my_len:
            recv = torch.empty((src_full.shape[0], len(theirs), my_len) + tuple(src_full.shape[3:]),
                               dtype=src_full.dtype, device=src_full.device)
            keep.append((recv, theirs))
            ops.append(dist.P2POp(dist.irecv, recv, peer, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for item in keep:
        if isinstance(item, tuple):
            recv, theirs = item
            for i, h in enumerate(theirs):
                dst_full[:, gidx[h], :my_len] = recv[:, i]
    return dst_full


def all_gather_rings(src_ring, owners, mask_row, rank, world, W, dst_ring, group=None):
    """Replicate ONE layer's streaming-head ring tensor on every rank (the sequence-sharded layout keeps all streaming
    heads on all ranks).

    ``src_ring``  ``[B, n_s_local, >= W, ...]``: this rank's streaming heads (order of ``owners[rank]``)
    ``dst_ring``  ``[B, n_s_total, >= W, ...]``: all streaming heads, original id ascending; slots ``[0, W)`` are set
    One ``all_gather`` of ``[B, max_r n_s(r), W, ...]``; any trailing shape and dtype (16-bit K/V, INT4 codes, fp16
    scale / zero rows)."""
    stream_ids = [h for h in range(len(mask_row)) if mask_row[h] <= 0.5]
    sidx = {h: i for i, h in enumerate(stream_ids)}
    per_rank = [[h for h in owners[r] if mask_row[h] <= 0.5] for r in range(world)]
    n_loc = max(len(hs) for hs in per_rank)
    send = torch.zeros((dst_ring.shape[0], n_loc, W) + tuple(dst_ring.shape[3:]), dtype=dst_ring.dtype,
                       device=dst_ring.device)
    if per_rank[rank]:
        send[:, : len(per_rank[rank])] = src_ring[:, :, :W]
    got = [torch.empty_like(send) for _ in range(world)]
    dist.all_gather(got, send, group=group)
    for r in range(world):
        for i, h in enumerate(per_rank[r]):
            dst_ring[:, sidx[h], :W] = got[r][:, i]
    return dst_ring


@torch.no_grad()
def shard_model(model, full_attention_heads, rank: int, world: int):
    """Build this rank's head-parallel shard of an UNPATCHED HF Llama/Mistral model (real weights):
    q/k/v rows and o_proj columns of the KV heads `plan_heads` assigns to `rank`, MLP gate/up rows and down columns
    split evenly, embeddings / norms / lm_head replicated.  Returns ``(shard_model, local_mask)``; call
    ``enable_duo_attention_eval(shard, local_mask, sink, recent)`` and ``install_allreduce(shard)`` on it.
    The reference gets the same split from tensor_parallel's config (duo_attn/utils.py:132-195)."""
    import copy

    from .kv_cache import model_geometry

    cfg = copy.deepcopy(model.config)
    plan = plan_heads(full_attention_heads, world)
    n_heads, n_kv = cfg.num_attention_heads, cfg.num_key_value_heads
    head_dim = model_geometry(model)["head_dim"]
    group = n_heads // n_kv
    inter = cfg.intermediate_size
    if inter % world:
        raise ValueError(f"intermediate_size {inter} not divisible by {world}")
    cfg.head_dim = head_dim
    cfg.num_attention_heads = n_heads // world
    cfg.num_key_value_heads = n_kv // world
    cfg.intermediate_size = inter // world
    shard = type(model)(cfg).to(next(model.parameters()).dtype)
    # `.to(dtype)` also casts the rotary inverse frequencies; a checkpoint loaded with torch_dtype=bf16 keeps them in
    # fp32 (non-persistent buffer computed at construction).  Take the source model's buffers so every shard rotates
    # with exactly the angles of the single-GPU model (the error of bf16 frequencies grows with position).
    src_rot, dst_rot = getattr(model.model, "rotary_emb", None), getattr(shard.model, "rotary_emb", None)
    if src_rot is not None and dst_rot is not None:
        for name, buf in src_rot.named_buffers(recurse=False):
            dst_rot.register_buffer(name, buf.detach().clone(), persistent=False)
    shard.model.embed_tokens.weight.copy_(model.model.embed_tokens.weight)
    shard.model.norm.weight.copy_(model.model.norm.weight)
    shard.lm_head.weight.copy_(model.lm_head.weight)
    lo, hi = rank * (inter // world), (rank + 1) * (inter // world)
    for l, (src, dst) in enumerate(zip(model.model.layers, shard.model.layers)):
        a, b = src.self_attn, dst.self_attn
        wq, wk, wv, wo = shard_attention_weights(a.q_proj.weight, a.k_proj.weight, a.v_proj.weight, a.o_proj.weight,
                                                 plan.owners[l][rank], group, head_dim)
        b.q_proj.weight.copy_(wq)
        b.k_proj.weight.copy_(wk)
        b.v_proj.weight.copy_(wv)
        b.o_proj.weight.copy_(wo)
        dst.mlp.gate_proj.weight.copy_(src.mlp.gate_proj.weight[lo:hi])
        dst.mlp.up_proj.weight.copy_(src.mlp.up_proj.weight[lo:hi])
        dst.mlp.down_proj.weight.copy_(src.mlp.down_proj.weight[:, lo:hi])
        dst.input_layernorm.weight.copy_(src.input_layernorm.weight)
        dst.post_attention_layernorm.weight.copy_(src.post_attention_layernorm.weight)
    return shard.eval(), plan.local_mask(rank)
