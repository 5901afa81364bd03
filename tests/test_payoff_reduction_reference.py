"""CPU: the dyadic construction of tests/payoff_reduction_reference.py is exact -- the integer reference, math.fsum and two plain fp64
summation orders of the per-path payoffs agree bit for bit -- and its std-error reference and bound behave as stated."""
import math

import numpy as np
import pytest

import payoff_reduction_reference as R


@pytest.mark.parametrize("n,J", [(1, 1), (257, 9), (20_011, 17), (70_001, 64)])
def test_dyadic_sums_exact_in_any_order(n, J):
    m, x, q = R.dyadic_states(n, seed=n)
    k, types = R.dyadic_strikes(J, seed=J)
    for tys in (types, np.where(np.arange(J) % 2 == 1, types + 2, types).astype(np.int8)):
        ref = R.dyadic_sums(m, x, k, tys, 2.0)
        pay = R.dyadic_pay_floats(m, x, k, tys, 2.0)
        for j in range(J):
            p = pay[:, j][~np.isnan(pay[:, j])]
            fs = (math.fsum(p), math.fsum(p * p), float(p.size))
            fwd = (np.cumsum(p)[-1] if p.size else 0.0, np.cumsum(p * p)[-1] if p.size else 0.0)
            rev = (np.cumsum(p[::-1])[-1] if p.size else 0.0, np.cumsum((p * p)[::-1])[-1] if p.size else 0.0)
            assert fs == tuple(ref[3 * j: 3 * j + 3]), (j, fs, ref[3 * j: 3 * j + 3])
            assert fwd == rev == fs[:2]


def test_dyadic_states_cover_edges_and_are_float_exact():
    m, x, q = R.dyadic_states(1000, seed=1)
    assert m[0] == 0 and m[1] == R.M_MAX - 1 and not np.isnan(x[0]) and np.isnan(x).sum() > 0
    assert np.array_equal(q.astype(np.float32).astype(np.float64), q)
    assert np.array_equal(q / R.TTM, q * (1.0 / R.TTM))
    k, _ = R.dyadic_strikes(201, seed=3)
    assert k.min() == 0 and k.max() == R.K_MAX and np.any(np.isin(k, 4 * m))


def test_finalize_reference_matches_plain_formula_and_bound_holds():
    """on exact sums the one-pass formula evaluated in fp64 (as the kernel does) lies within the stated bound of the exact value"""
    m, x, q = R.dyadic_states(5003, seed=5)
    k, types = R.dyadic_strikes(17, seed=5)
    sums = R.dyadic_sums(m, x, k, types, 2.0)
    prices, se, tol = R.finalize_reference(sums, 0.5, 5003)
    s1, s2, cnt = sums[0::3], sums[1::3], sums[2::3]
    mean = s1 / cnt
    var = s2 / cnt - mean * mean
    se_fp = 0.5 * np.sqrt(np.where(var < 0, 0.0, var)) / np.sqrt(5003.0)
    assert np.array_equal(prices, 0.5 * mean)
    assert np.all(np.abs(se_fp - se) <= tol) and np.all(tol < 1e-12 + 1e-10 * se)


def test_negative_one_pass_constant():
    p = R.negative_one_pass_constant()
    mean, A = (3.0 * p) / 3.0, (3.0 * (p * p)) / 3.0
    assert A - mean * mean < 0.0


def test_exact_two_pass():
    pay = np.array([0.1, 0.2, 0.7, 1e-3])
    mean, var = R.exact_two_pass(pay)
    assert float(mean) == pytest.approx(np.mean(pay), rel=1e-15) and float(var) == pytest.approx(np.var(pay), rel=1e-14)
