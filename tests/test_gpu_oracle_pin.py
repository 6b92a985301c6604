"""Pin the oracle's restatement of flash_attn_func's contract against the installed flash_attn library —
the very kernels the reference calls (llama.py:227,239,252,...) — on the GPU box, and cross-check the
CUDA product against that library too (second, independent GPU oracle; SURVEY.md §8c)."""
import pytest
import torch

from duo_attention_b200 import _C
from duo_attention_b200.kv_cache import DuoKVCache
from oracle import duo_oracle as O
from parity import assert_parity

pytestmark = pytest.mark.gpu
D = 128


@pytest.mark.parametrize("Sq,Sk,Hq,Hkv", [(1, 700, 8, 2), (37, 37, 8, 8), (16, 300, 4, 1), (128, 500, 8, 2)])
def test_contract_restatement_vs_flash_attn(Sq, Sk, Hq, Hkv):
    fa = pytest.importorskip("flash_attn")
    g = torch.Generator().manual_seed(Sq * 1000 + Sk)
    q = torch.randn(2, Sq, Hq, D, generator=g).to(torch.bfloat16)
    k = torch.randn(2, Sk, Hkv, D, generator=g).to(torch.bfloat16)
    v = torch.randn(2, Sk, Hkv, D, generator=g).to(torch.bfloat16)
    ref = O.flash_attn_contract(q, k, v, causal=True)
    got = fa.flash_attn_func(q.cuda(), k.cuda(), v.cuda(), causal=True, dropout_p=0.0).cpu()
    assert_parity(got, ref, "flash_attn_func vs contract restatement")


def test_product_vs_reference_forward_restated_with_flash_attn():
    """llama.py:374-421 restated verbatim on the GPU with the installed flash_attn_func, token-major caches,
    torch.cat and compaction — vs the fused CUDA path."""
    fa = pytest.importorskip("flash_attn")
    dev = torch.device("cuda:0")
    Hq, Hkv, n_full, sink, recent = 32, 8, 3, 64, 256
    G = Hq // Hkv
    g = torch.Generator().manual_seed(0)
    cache = DuoKVCache(1, Hq, Hkv, D, [n_full], 1, 4096, sink, recent, torch.bfloat16, dev, stage_cap=1024)
    fk = fv = sk = sv = None
    for S in [1000, 1, 1, 600, 1, 64, 1]:
        qkv = torch.randn(1, S, (Hq + 2 * Hkv) * D, generator=g).to(torch.bfloat16).to(dev)
        q = qkv[..., : Hq * D].reshape(1, S, Hq, D)
        k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(1, S, Hkv, D)
        v = qkv[..., (Hq + Hkv) * D :].reshape(1, S, Hkv, D)
        if fk is None:
            ref = fa.flash_attn_func(q, k, v, causal=True)
            fk, fv, sk, sv = k[:, :, :n_full], v[:, :, :n_full], k[:, :, n_full:], v[:, :, n_full:]
        else:
            fk = torch.cat([fk, k[:, :, :n_full]], 1)
            fv = torch.cat([fv, v[:, :, :n_full]], 1)
            sk = torch.cat([sk, k[:, :, n_full:]], 1)
            sv = torch.cat([sv, v[:, :, n_full:]], 1)
            a = fa.flash_attn_func(q[:, :, : n_full * G], fk, fv, causal=True)
            b = fa.flash_attn_func(q[:, :, n_full * G :], sk, sv, causal=True)
            ref = torch.cat([a, b], dim=2)
        if sk.shape[1] > sink + recent:
            sk = torch.cat([sk[:, :sink], sk[:, -recent:]], 1)
            sv = torch.cat([sv[:, :sink], sv[:, -recent:]], 1)
        out = torch.empty(1, S, Hq, D, dtype=torch.bfloat16, device=dev)
        cache.attend(0, qkv.clone(), None, None, _C.ROPE_NONE, out)
        assert_parity(out.float().cpu(), ref.float().cpu(), f"chunk of {S}")


def _truth(q, k, v):
    """fp64 causal (bottom-right) GQA attention, no rounding anywhere."""
    B, Sq, Hq, _ = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    G = Hq // Hkv
    qd, kd, vd = q.double(), k.double(), v.double()
    out = torch.empty(B, Sq, Hq, D, dtype=torch.float64)
    ii = torch.arange(Sq)[:, None] + (Sk - Sq)
    jj = torch.arange(Sk)[None, :]
    for h in range(Hq):
        s = torch.einsum("bqd,bkd->bqk", qd[:, :, h], kd[:, :, h // G]) / D ** 0.5
        s = s.masked_fill((jj > ii)[None], float("-inf"))
        out[:, :, h] = torch.einsum("bqk,bkd->bqd", torch.softmax(s, -1), vd[:, :, h // G])
    return out


@pytest.mark.parametrize("Sq,Sk,qscale", [(1, 40, 1.0), (1, 3000, 1.0), (4, 500, 1.0), (256, 256, 1.0),
                                          (384, 900, 1.0), (512, 512, 6.0)])
def test_accuracy_vs_fp64_truth_not_worse_than_flash_attn(Sq, Sk, qscale):
    """Against exact math our kernels (split-KV decode, small-chunk and wgmma prefill) must be as accurate as
    the FlashAttention-2 kernel the reference calls: RMS error within 1.3x of FA2's, max error within 2x."""
    fa = pytest.importorskip("flash_attn")
    dev = torch.device("cuda:0")
    Hq, Hkv = 8, 2
    g = torch.Generator().manual_seed(Sq * 7 + Sk)
    qkv = torch.randn(1, Sk, (Hq + 2 * Hkv) * D, generator=g).to(torch.bfloat16)
    qkv[..., : Hq * D] *= qscale
    q = qkv[:, Sk - Sq :, : Hq * D].reshape(1, Sq, Hq, D)
    k = qkv[..., Hq * D : (Hq + Hkv) * D].reshape(1, Sk, Hkv, D)
    v = qkv[..., (Hq + Hkv) * D :].reshape(1, Sk, Hkv, D)
    truth = _truth(q, k, v)
    ref = fa.flash_attn_func(q.cuda(), k.cuda(), v.cuda(), causal=True).double().cpu()
    cache = DuoKVCache(1, Hq, Hkv, D, [Hkv], 1, Sk + 8, 4, 4, torch.bfloat16, dev, stage_cap=max(Sq, Sk - Sq, 1))
    if Sk > Sq:
        o0 = torch.empty(1, Sk - Sq, Hq, D, dtype=torch.bfloat16, device=dev)
        cache.attend(0, qkv[:, : Sk - Sq].to(dev).contiguous(), None, None, _C.ROPE_NONE, o0)
    o1 = torch.empty(1, Sq, Hq, D, dtype=torch.bfloat16, device=dev)
    cache.attend(0, qkv[:, Sk - Sq :].to(dev).contiguous(), None, None, _C.ROPE_NONE, o1)
    mine = o1.double().cpu()
    e_ref, e_mine = (ref - truth).abs(), (mine - truth).abs()
    rms_ref, rms_mine = e_ref.pow(2).mean().sqrt().item(), e_mine.pow(2).mean().sqrt().item()
    assert rms_mine <= 1.3 * rms_ref + 1e-6, (rms_mine, rms_ref)
    assert e_mine.max().item() <= 2.0 * e_ref.max().item() + 1e-4, (e_mine.max().item(), e_ref.max().item())
