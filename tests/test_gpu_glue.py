"""Caller-side glue kernels (duo_add_rmsnorm, duo_silu_mul) vs plain PyTorch (HF arithmetic)."""
import pytest
import torch

from duo_attention_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
# hidden 12288 (48 KB of dynamic shared memory plus the kernel's static array), 12296 and 16384 take the opt-in
# launch path
@pytest.mark.parametrize("rows,hidden", [(1, 4096), (37, 512), (300, 4096), (3, 8), (5, 520), (3, 12288), (2, 12296),
                                         (4, 16384)])
def test_add_rmsnorm_matches_hf_formula(dtype, rows, hidden):
    g = torch.Generator(device="cuda").manual_seed(rows + hidden)
    x = torch.randn(1, rows, hidden, device="cuda", generator=g).to(dtype)
    res = torch.randn(1, rows, hidden, device="cuda", generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(hidden, device="cuda", generator=g)).to(dtype)
    eps = 1e-5

    def hf_norm(h):
        hf = h.float()
        var = hf.pow(2).mean(-1, keepdim=True)
        return w * (hf * torch.rsqrt(var + eps)).to(dtype)

    out, h = ops.add_rmsnorm(x, None, w, eps)
    assert h is x
    torch.testing.assert_close(out.float(), hf_norm(x).float(), rtol=2e-2, atol=2e-2)
    assert (out.float() - hf_norm(x).float()).abs().max() <= 2 * torch.finfo(dtype).eps * hf_norm(x).float().abs().max()
    r2 = res.clone()
    out2, h2 = ops.add_rmsnorm(x, r2, w, eps)
    want_h = res + x
    assert h2 is r2 and torch.equal(h2, want_h)  # residual add is bit-exact and written in place
    assert (out2.float() - hf_norm(want_h).float()).abs().max() <= 2 * torch.finfo(dtype).eps * hf_norm(want_h).float().abs().max()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_add_rmsnorm_with_residual_and_no_out_res(dtype):
    """duo_add_rmsnorm(x, residual, ..., out_res = NULL): the norm of residual + x, and nothing else written."""
    from duo_attention_b200 import _C

    rows, hidden, eps = 7, 4096, 1e-5
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(rows, hidden, device="cuda", generator=g).to(dtype)
    res = torch.randn(rows, hidden, device="cuda", generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(hidden, device="cuda", generator=g)).to(dtype)
    x0, res0 = x.clone(), res.clone()
    out = torch.full_like(x, float("nan"))
    dt = _C.DT_BF16 if dtype == torch.bfloat16 else _C.DT_FP16
    _C.check(_C.load().duo_add_rmsnorm(x.data_ptr(), res.data_ptr(), w.data_ptr(), out.data_ptr(), None, rows, hidden,
                                       eps, dt, torch.cuda.current_stream().cuda_stream))
    want_out, want_h = ops.add_rmsnorm(x.clone(), res.clone(), w, eps)
    assert torch.equal(x, x0) and torch.equal(res, res0)
    assert torch.equal(want_h, res0 + x0)
    assert torch.equal(out, want_out)  # the same kernel with out_res given: the same bits


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_silu_mul_matches_torch(dtype):
    g = torch.Generator(device="cuda").manual_seed(0)
    gu = (2 * torch.randn(3, 5, 2 * 1024, device="cuda", generator=g)).to(dtype)
    want = torch.nn.functional.silu(gu[..., :1024]) * gu[..., 1024:]
    got = ops.silu_mul(gu)
    torch.testing.assert_close(got.float(), want.float(), rtol=2 ** -7, atol=1e-6)
