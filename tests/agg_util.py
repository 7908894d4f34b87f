"""Comparison rule for Float64 SUM / AVG results against the oracle's correctly rounded sums (DESIGN.md §7).

Any summation order of n_g finite addends stays within
    |got − exact| ≤ 2·(n_g − 1)·2⁻⁵³ · Σ|x_i|          (SUM)
    |got − exact| ≤ that / n_g + 2⁻⁵²·|exact|          (AVG: one more rounding in the division)
A group with a NaN or with both infinities sums to NaN, a group with infinities of one sign to that infinity, whatever
the order: those are compared exactly (NaN ↔ NaN, ±inf ↔ the same ±inf).
"""
import numpy as np


def float_sum_bound(n_g, abs_sum, want, avg=False):
    """The tolerance of a finite SUM (avg=False) or AVG over n_g addends of absolute sum abs_sum; numpy-vectorised."""
    n_g = np.asarray(n_g, dtype=np.float64)
    bound = 2 * np.maximum(n_g - 1, 1) * 2.0 ** -53 * np.asarray(abs_sum, dtype=np.float64) + 1e-300
    if avg:
        bound = bound / np.maximum(n_g, 1) + np.abs(np.asarray(want, dtype=np.float64)) * 2.0 ** -52
    return bound


def float_sum_mismatches(got, want, n_g, abs_sum, avg=False):
    """Indices where `got` breaks the rule above.  got / want: float64 arrays (NULLs removed or equal on both sides)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    nan_w, nan_g = np.isnan(want), np.isnan(got)
    inf_w = np.isinf(want)
    with np.errstate(invalid="ignore", over="ignore"):
        err = np.abs(got - want)  # NaN or inf when got is: both fail the bound
        ok = np.where(nan_w, nan_g, np.where(inf_w, got == want, err <= float_sum_bound(n_g, abs_sum, want, avg)))
    return np.flatnonzero(~ok)
