"""CPU: the references and bars of tests/fourier_edges_reference.py, validated before they judge a kernel.

  - the numpy restatements (oracle/mgf.py, oracle/hawkes.py) lie inside every bar at every case: the closed form at every parameter
    extreme, maturity and transform point, every strike sum at every grid length, strike count and constructed non-finite entry, with
    numpy's NaN / +-inf pattern reproduced by the reference's summand-by-summand semantics;
  - the bars reject deliberately wrong variants: psi+ and psi- swapped, b not carried between maturities, the legacy Simpson quirk
    dropped, np.nansum skipping +-inf as well, one summand scaled by (1 + 1e-6);
  - the numpy forward modes of the Heston sensitivities (first order, hyper-dual second order) lie inside the bars of mp.diff, and those
    bars reject the b' v0 term dropped from the parameter tangents and the Hessian rows in the wrong triangle order;
  - no closed-form point is singular in mpmath while numpy is finite (such a point would go unchecked on the device).
"""
import numpy as np
import pytest

pytest.importorskip("mpmath")

import fourier_edges_reference as R  # noqa: E402


def _report(name, worst):
    print(f"{name}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


def test_numpy_closed_form_inside_every_bar():
    worst = {}
    for c in R.heston_cases():
        got = R.heston_numpy(c["par"], c["taus"], c["phi"], c["psi"])
        r = R.heston_ratio(got, c)
        key = "psi" if "psi" in c["name"] else f"M={len(c['taus'])}"
        worst[key] = max(worst.get(key, 0.0), float(r.max()))
        assert r.max() <= 1.0, (c["name"], np.unravel_index(np.argmax(r), r.shape), r.max())
    _report("numpy closed form, max err / bar", worst)


def test_numpy_sums_inside_every_bar():
    worst = {}
    for c in R.sum_cases():
        assert R.nonfinite_mismatch(c["numpy"], c["exact"]).size == 0, (R.case_name(c), c["numpy"], c["exact"])
        assert np.all(np.isfinite(c["bar"][np.isfinite(c["exact"])])), R.case_name(c)
        r = R.bar_ratio(c["numpy"], c["exact"], c["bar"])
        worst[c["kind"]] = max(worst.get(c["kind"], 0.0), float(r.max()))
        assert r.max() <= 1.0, (R.case_name(c), r.max())
    _report("numpy sums, max err / bar", worst)
    # the constructed entries do reach every non-finite outcome: -inf / +inf prices (an overflowing or +inf term kept) and finite ones
    out = np.concatenate([c["exact"] for c in R.sum_cases() if c["tag"].startswith("lm[")])
    assert np.isneginf(out).any() and np.isposinf(out).any() and np.isfinite(out).any()


def test_bars_reject_swapped_psi():
    for c in R.heston_cases():
        r = R.heston_ratio(R.heston_numpy(c["par"], c["taus"], c["phi"], c["psi"], swap_psi=True), c)
        assert r.max() > 1.0, c["name"]


def test_bars_reject_b_not_carried():
    chains = [c for c in R.heston_cases() if len(c["taus"]) > 1]
    assert chains
    for c in chains:
        r = R.heston_ratio(R.heston_numpy(c["par"], c["taus"], c["phi"], c["psi"], carry_b=False), c)
        assert r.max() > 1.0, c["name"]


def _sum_defect(P, kind="vanilla_half", lm=None, **defect):
    g = R.grid(-0.5, R.STOP, P)
    lm = R.heston_lm(g) if lm is None else lm
    cs = -np.log(R.F0 / R.strikes_for())
    S, sbar, _ = R.exact_sums(kind, lm, g, cs)
    with np.errstate(all="ignore"):
        bad = R.numpy_sums(kind, lm, g, cs, **defect)
        good = R.numpy_sums(kind, lm, g, cs)
    return S, sbar, good, bad


@pytest.mark.parametrize("P", [4, 256, 1000])
def test_bars_reject_dropped_simpson_quirk(P):
    """on an even grid the legacy weights end ..., 2, 4 (every odd index 4 after first / last = 1): a last weight of 1 must fail"""
    wq = R.legacy_weights(R.grid(-0.5, R.STOP, P))
    assert wq[-1] == 4.0
    wq[-1] = 1.0
    S, sbar, good, bad = _sum_defect(P, wq=wq)
    assert np.all(np.abs(good - S) <= sbar)
    assert np.any(np.abs(bad - S) > sbar)


def test_bars_reject_nansum_skipping_inf():
    P = R.CONSTRUCTED_P
    lm = R.constructed(R.heston_lm(R.grid(-0.5, R.STOP, P)), "+inf", 0)
    S, sbar, good, bad = _sum_defect(P, lm=lm, nansum_inf=True)
    assert np.all(np.isposinf(S)) and np.all(np.isposinf(good))
    assert np.all(np.isfinite(bad))
    assert R.nonfinite_mismatch(bad, S).size == S.size


@pytest.mark.parametrize("P", [5, 257, 1001])
def test_bars_reject_one_summand_scaled(P):
    g = R.grid(-0.5, R.STOP, P)
    t = R.numpy_terms("vanilla_half", R.heston_lm(g), g, -np.log(R.F0 / R.strikes_for()))
    j = int(np.argmax(np.abs(t[0])))
    S, sbar, good, bad = _sum_defect(P, scale=(j, 1.0 + 1e-6))
    assert np.all(np.abs(good - S) <= sbar)
    assert np.any(np.abs(bad - S) > sbar)


def test_closed_form_singular_only_where_numpy_is_not_finite():
    """a point where the exact formula is singular but numpy finite would go unchecked on the device: there is none in the case set"""
    for c in R.heston_cases():
        sing = ~np.isfinite(c["exact"]) | ~np.isfinite(c["bar"])
        got = R.heston_numpy(c["par"], c["taus"], c["phi"], c["psi"])
        assert np.all(~np.isfinite(got[sing])), c["name"]


def test_numpy_forward_modes_inside_the_derivative_bars():
    worst = {"d1": 0.0, "d2": 0.0}
    for c in R.heston_deriv_cases():
        for k in ("d1", "d2"):
            assert np.all(np.isfinite(c[k])) and np.all(np.isfinite(c["bar" + k[1]])), c["name"]
            r = R.bar_ratio(c["numpy_" + k], c[k], c["bar" + k[1]])
            worst[k] = max(worst[k], float(r.max()))
            assert r.max() <= 1.0, (c["name"], k, r.max())
    _report("numpy forward modes, max err / bar", worst)


def test_derivative_bars_reject_a_dropped_b_tangent():
    """the parameter rows without the b' v0 term of d(a + b v0)"""
    for c in R.heston_deriv_cases():
        bad = R.heston_dlog_mgf_numpy(c["par"], R.DERIV_TTMS, c["phi"], with_b_tangent=False)
        assert R.bar_ratio(bad, c["d1"], c["bar1"]).max() > 1.0, c["name"]


def test_derivative_bars_reject_hessian_rows_out_of_order():
    """the 15 second derivatives in column-major order of the upper triangle instead of the row-major order of the outputs"""
    col_major = sorted(R.PAIRS5, key=lambda pq: (pq[1], pq[0]))
    assert col_major != R.PAIRS5
    for c in R.heston_deriv_cases():
        bad = R.heston_d2log_mgf_numpy(c["par"], R.DERIV_TTMS, c["phi"], col_major)
        assert R.bar_ratio(bad, c["d2"], c["bar2"]).max() > 1.0, c["name"]
