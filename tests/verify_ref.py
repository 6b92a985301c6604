"""Reference of a verify chunk (DESIGN §2): token t of the chunk gets the keys a one-token decode step at its position
sees.  The keys are read from a twin cache that takes the chunk one token per step: its sink / ring slots before step
t (with the twin's total / lo then) plus the new token's streaming row after it, and its retrieval rows after it.
Attention is evaluated in fp64."""
import torch

from duo_attention_b200 import _C

D = 128


def slot_valid(j, sink, recent, total, lo):
    """stream_slot_valid (duo_common.cuh): does sink / ring slot j hold a live position?"""
    if j < sink:
        return j < total
    if total <= sink:
        return False
    last = total - 1
    diff = (last - sink - (j - sink)) % recent
    return last - diff >= lo


def rope_tables(positions, mode, dtype, device, theta=10000.0):
    """[len(positions), D] cos / sin tables: the activation dtype for ROPE_HF, fp32 for ROPE_FP32, None for ROPE_NONE.
    ``positions`` may also be a [B, S] list of lists (per-row tables of a ragged batch)."""
    if mode == _C.ROPE_NONE:
        return None, None
    inv = theta ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
    ang = torch.tensor(positions, dtype=torch.float64)[..., None] * inv
    dt = dtype if mode == _C.ROPE_HF else torch.float32
    cos, sin = (torch.cat([f(ang), f(ang)], -1).to(dt).to(device).contiguous() for f in (torch.cos, torch.sin))
    return cos, sin


def rotate(x, cos, sin):
    """RoPE of x [..., D] (fp64) with table rows cos / sin broadcast over the heads."""
    if cos is None:
        return x
    rh = torch.cat([-x[..., 64:], x[..., :64]], -1)
    return x * cos.double() + rh * sin.double()


class SequentialTwin:
    """Wraps a batch-B DuoKVCache that takes the chunk one token per step (``attend``) and records, per step, the keys each
    head of each row saw, as fp64 [n, D] K and V."""

    def __init__(self, cache):
        self.c = cache
        self.keys = []  # per step: [b][kv head] -> (K, V)

    def step(self, qkv_t, cos_t, sin_t, rope, out_t):
        c = self.c
        t0 = c.tensors[0]
        n_full = c.num_full_kv_head_list[0]
        ring_k, ring_v = t0["ring_k"][:, :, : c.W].clone(), t0["ring_v"][:, :, : c.W].clone()
        n, total, lo = c.kv_seq_len_list[0], c.total_list[0], c.lo_list[0]
        c.attend(0, qkv_t, cos_t, sin_t, rope, out_t)
        if c.dev_state is not None:  # as the model driver does after a step
            c.advance_device(1)
        live = [j for j in range(c.W) if slot_valid(j, c.sink_size, c.recent_size, total, lo)]
        new = total if total < c.sink_size else c.sink_size + (total - c.sink_size) % c.recent_size
        step = []
        for b in range(c.batch_size):
            heads = []
            for h in range(c.num_kv_heads):
                if h < n_full:
                    heads.append((t0["full_k"][b, h, : n + 1].double(), t0["full_v"][b, h, : n + 1].double()))
                    continue
                hs = h - n_full
                heads.append((torch.cat([ring_k[b, hs, live], t0["ring_k"][b, hs, new : new + 1]]).double(),
                              torch.cat([ring_v[b, hs, live], t0["ring_v"][b, hs, new : new + 1]]).double()))
            step.append(heads)
        self.keys.append(step)


def reference(twin, q_rot, group, scale):
    """fp64 attention of q_rot [B, S, Hq, D] (rotated, fp64) over the keys the twin's steps saw."""
    B, S, Hq, _ = q_rot.shape
    out = torch.zeros(B, S, Hq, D, dtype=torch.float64, device=q_rot.device)
    for t in range(S):
        for b in range(B):
            for h in range(Hq):
                k, v = twin.keys[t][b][h // group]
                p = torch.softmax((k @ q_rot[b, t, h]) * scale, 0)
                out[b, t, h] = p @ v
    return out
