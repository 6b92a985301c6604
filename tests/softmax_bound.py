"""fp64 expectation of one attention call and a per-element forward-error bound for it.

The attention kernels compute ``o = sum_p w_p v_p / sum_p w_p`` with ``w_p = exp2(l_p - m)``: tiled online softmax,
split-KV partials and merges in fp32, P rounded once to the MMA type.  A consistent reference ``m`` cancels, so the
bound below holds whatever tiles, splits and merges the launch plan uses; what it does not allow is a weight that one
partial, one merge level or one rescale gets wrong (a partial's ``m`` with another partial's ``l``, a rescale applied
to ``o`` but not to ``l``, a factor 1 % off).  tests/test_softmax_bound_host.py pins the bound on an emulated tiled
kernel before any GPU runs; tests/test_gpu_softmax_mass.py holds every attention entry point to it.

Notation, per query row and output dimension d (keys p the row may see, log2-domain logits ``l_p``, weights
``w_p = 2^(l_p - max l)`` so the largest is 1, ``Z = sum_p w_p``):

* ``want_d = sum_p w_p v_pd / Z`` in fp64.
* P rounding to the MMA type, relative ``eps_P`` = 2^-8 (bf16) or 2^-10 (fp16): twice the unit roundoff, which also
  covers the mismatch between the rounded numerator and the fp32 denominator.  It multiplies
  ``E_d = sum_p w_p |r_pd| / Z`` where ``r`` is the value the rounded P multiplies: ``v`` on 16-bit caches; on INT4
  caches ``s_p c_pd`` (scale times code), because the INT4 kernels round ``P' = fp16(p s_p)`` and add ``p z_p`` in
  fp32.
* fp16 P underflow, absolute: a rounded P below the fp16 normal range is off by at most half the subnormal spacing,
  2^-25, against the running maximum, which is never above the final one: ``2^-25 sum_p |r_pd| / (s_p Z)``, where
  ``s_p`` is the factor folded into the rounded P (INT4: P' = p s_p, so the term multiplies the codes; 1 on 16-bit
  caches).  bf16 P has no such term (its subnormals start at 2^-126).
* logit and exp2 error: the fp32 logit and its scaling to log2 units are good to ~2^-23 of ``|l_p|``, ``ex2.approx``
  to ~2^-22; a relative weight error ``delta_p`` moves the output by ``sum_p w_p delta_p (v_pd - want_d) / Z``, so the
  term is ``(2^-20 max_p |l_p| + 2^-21) (E_d + |want_d|)``.
* output rounding: 1 ulp of the output dtype at ``|want_d|``, never below the fp16 subnormal spacing 2^-24.

There is no term for the fp32 accumulations (tens to hundreds of adds: ~1e-5 relative), and none for an offset the
kernel adds and subtracts around an accumulation: amplified cancellation is not something the format requires (the
INT4 kernels recentre their V codes to ``c - 8`` before the tensor-core accumulation for that reason, DESIGN §4).
"""
from __future__ import annotations

import math

import torch

LOG2E = 1.0 / math.log(2.0)


def eps_p(p_dtype: torch.dtype) -> float:
    """Relative rounding of P to the MMA type (twice the unit roundoff)."""
    return 2.0 ** -8 if p_dtype == torch.bfloat16 else 2.0 ** -10


def ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """1 ulp of ``dtype`` at |x| (fp64), floored at 2^-24."""
    bits = 7 if dtype == torch.bfloat16 else 10
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -24)))
    return torch.pow(2.0, e - bits).clamp_min(2.0 ** -24)


def bound_terms(l2: torch.Tensor, v: torch.Tensor, p_dtype: torch.dtype, out_dtype: torch.dtype,
                r: torch.Tensor = None, p_scale: torch.Tensor = None):
    """``l2`` [R, n] log2-domain logits (-inf: not visible), ``v`` [n, D] the values as the kernel reads them, ``r``
    [n, D] what the rounded P multiplies (default ``v``), ``p_scale`` [n] the factor folded into the rounded P (INT4:
    the V scales; default 1).  Returns ``(want, bound, terms)``: ``want`` and ``bound``
    [R, D] fp64, ``terms`` a dict of the four [R, D] contributions."""
    l2 = l2.double()
    v = v.double()
    r = v if r is None else r.double()
    m = l2.amax(-1, keepdim=True)
    assert torch.isfinite(m).all(), "every row must see at least one key"
    w = torch.exp2(l2 - m)                                   # exactly 0 where l2 = -inf
    z = w.sum(-1, keepdim=True)
    want = (w @ v) / z
    e = (w @ r.abs()) / z
    u = r.abs() if p_scale is None else r.abs() / p_scale.double()[:, None]
    lmax = torch.where(torch.isfinite(l2), l2.abs(), torch.zeros_like(l2)).amax(-1, keepdim=True)
    terms = {
        "p_round": eps_p(p_dtype) * e,
        "p_underflow": ((l2 > -math.inf).double() @ u) * 2.0 ** -25 / z if p_dtype == torch.float16
        else torch.zeros_like(want),
        "logit": (2.0 ** -20 * lmax + 2.0 ** -21) * (e + want.abs()),
        "out_round": ulp(want, out_dtype),
    }
    return want, sum(terms.values()), terms


def expect(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, p_dtype: torch.dtype,
           out_dtype: torch.dtype, mask: torch.Tensor = None, r: torch.Tensor = None, p_scale: torch.Tensor = None):
    """``q`` [R, D] query rows, ``k`` / ``v`` [n, D] the keys and values exactly as the kernel reads them (on INT4
    caches ``s c + z`` from the stored codes, or the 16-bit image where the wgmma path runs), ``mask`` [R, n] the keys
    each row may see (tests/visibility_model.py decides which), ``r`` [n, D] what the rounded P multiplies (INT4:
    ``s c``), ``p_scale`` [n] the factor folded into the rounded P (INT4: ``s``).  Returns ``(want, bound)`` [R, D]
    fp64."""
    l2 = (q.double() @ k.double().T) * (scale * LOG2E)
    if mask is not None:
        l2 = l2.masked_fill(~mask, -math.inf)
    want, bound, _ = bound_terms(l2, v, p_dtype, out_dtype, r, p_scale)
    return want, bound


def worst_ratio(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - want| / bound over all elements (NaN counts as infinitely wrong)."""
    err = (got.double() - want).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return float((err / bound).max())
