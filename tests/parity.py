"""The parity bar used by every GPU test.

north_star: outputs match the reference forward "within bf16 rtol=1e-2 / atol=1e-3".  The reference's attention
IS FlashAttention-2, and FA2 itself does not meet that bar element-for-element against an fp32-softmax
restatement: P is rounded to bf16 block by block against the *running* max, so a few elements land up to a couple
of bf16 ulps away (the installed flash_attn 2.8.3 vs oracle.flash_attn_contract: 0 violations for ordinary logits,
2.7e-4 of the elements — max |err| 0.0156 — when the softmax is sharp; see DESIGN.md §Parity).  The gate therefore has two parts:

  * absolute, against the oracle: a violation rate of at most 0.5 % of the elements outside rtol=1e-2 / atol=1e-3, tested
    at 4 sigma of the binomial count (`violation_allowance`: 0.53 % of a 1M-element output, 9 elements of a 512-element
    decode output), and none outside rtol=2e-2 / atol=8e-3 (two bf16 ulps of an O(1) output);
  * relative to the reference's own kernel, wherever it can run on the test's inputs (`fa2=` + `truth=`): against
    EXACT fp64 attention on the same inputs, the number of our elements outside rtol=1e-2 / atol=1e-3 may exceed
    FlashAttention-2's own count by at most max(0.2 % of the elements, 2) (`REL_EPS`), and we may have no hard-bound violation
    that FA2 does not have.  (Measured against the oracle instead, FA2 looks better than it is: the oracle rounds P
    against the same running max FA2 uses, so their rounding errors are correlated; a kernel with a different — equally
    valid — reference for P is only comparable against exact math.
    The log keeps both counts.)

With DUO_PARITY_LOG=<file> set, every call appends the achieved counts to that file.  That the kernels are not
LESS accurate than the reference's kernel is also asserted against an fp64 ground truth
(tests/test_gpu_oracle_pin.py::test_accuracy_vs_fp64_truth_not_worse_than_flash_attn, tests/test_gpu_bench_shapes.py).
"""
import json
import math
import os

import torch

RTOL, ATOL = 1e-2, 1e-3
MAX_VIOLATION_FRACTION = 5e-3
HARD_RTOL, HARD_ATOL = 2e-2, 8e-3
# Allowed excess of OUR violation count over FlashAttention-2's, both against exact fp64 attention, as a fraction of the
# elements.  For ordinary logits the two counts agree to within a few elements; a kernel that rounds P against a reference
# other than the running max (e.g. a lazily rescaled one) shows its excess on the sharp-softmax stress cases (logit std 6-8).
REL_EPS = 2e-3
LOG_PATH = os.environ.get("DUO_PARITY_LOG")


def record(kind: str, **fields):
    """Append one JSON line per parity measurement (achieved violation fractions, errors) to $DUO_PARITY_LOG, if set."""
    if not LOG_PATH:
        return
    try:
        os.makedirs(os.path.dirname(LOG_PATH), exist_ok=True)
        with open(LOG_PATH, "a") as f:
            f.write(json.dumps({"test": os.environ.get("PYTEST_CURRENT_TEST", ""), "kind": kind, **fields}) + "\n")
    except OSError:
        pass


def violation_allowance(n: int) -> int:
    """Elements allowed outside rtol/atol: a violation RATE of 0.5 %, tested at 4 sigma of the binomial count — for a
    1M-element output that is 0.53 %, for a 512-element decode output (where 0.5 % is 2.6 elements and one unlucky
    element is 0.2 %) it is 9 elements.  Measured rate of BOTH kernels (ours and FlashAttention-2) against exact math with
    only a handful of visible keys: ~0.3 % (bf16 rounding of P against atol = 1e-3 near zero outputs)."""
    mean = MAX_VIOLATION_FRACTION * n
    return int(math.ceil(mean + 4.0 * math.sqrt(mean)))


def _counts(x, ref):
    err = (x - ref).abs()
    viol = err > (ATOL + RTOL * ref.abs())
    hard = err > (HARD_ATOL + HARD_RTOL * ref.abs())
    return err, int(viol.sum().item()), int(hard.sum().item())


def assert_parity(got: torch.Tensor, ref: torch.Tensor, what: str = "", fa2: torch.Tensor = None,
                  truth: torch.Tensor = None):
    """``got`` (the CUDA product) against ``ref`` (oracle / reference output) at the north_star tolerance.

    Absolute gate (always): at least 99.5 % of the elements of ``got`` within rtol/atol of ``ref`` and none outside the
    hard bound.  Relative gate (when the test supplies ``fa2`` = the installed flash_attn_func's output and ``truth`` =
    exact fp64 attention on the SAME inputs): measured against exact math, our count of elements outside rtol/atol may
    exceed FlashAttention-2's own count by at most max(REL_EPS = 0.2 % of the elements, 2 elements), and we may have no
    hard-bound violation FA2 does not have.  Every call logs what was achieved (``record``)."""
    got, ref = got.float(), ref.float()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    n = got.numel()
    err, n_viol, n_hard = _counts(got, ref)
    frac = n_viol / n
    allowed = violation_allowance(n)
    log = dict(what=what, n=n, viol=n_viol, hard=n_hard, max_err=err.max().item())
    rel_fail = ""
    if fa2 is not None:
        fa2 = fa2.float().to(ref.device)
        e2, fa2_viol, fa2_hard = _counts(fa2, ref)
        log.update(fa2_viol=fa2_viol, fa2_hard=fa2_hard, fa2_max_err=e2.max().item())
        if truth is not None:
            truth = truth.float().to(ref.device)
            _, t_ours, th_ours = _counts(got, truth)
            _, t_fa2, th_fa2 = _counts(fa2, truth)
            log.update(truth_viol=t_ours, truth_hard=th_ours, fa2_truth_viol=t_fa2, fa2_truth_hard=th_fa2)
            eps = max(math.ceil(REL_EPS * n), 2)
            if t_ours > t_fa2 + eps or th_ours > th_fa2:
                rel_fail = (f"; against exact math {t_ours} elements outside the tolerance vs FlashAttention-2's "
                            f"{t_fa2} (+{eps} allowed), hard bound {th_ours} vs {th_fa2}")
    record("parity", **log)
    if n_viol > allowed or n_hard > 0 or rel_fail:
        idx = tuple(int(i) for i in torch.nonzero(err == err.max())[0])
        raise AssertionError(
            f"{what}: {n_viol} of {n} elements ({frac:.2e}) outside rtol={RTOL}/atol={ATOL} (allowed {allowed}), "
            f"{n_hard} outside the hard bound; max |err| {err.max().item():.5f} at {idx} "
            f"(got {got[idx].item():.5f}, ref {ref[idx].item():.5f}){rel_fail}")
    return err.max().item(), frac
