"""CPU: the host Black-76 inversions of oracle/bsm.py -- the bisection checker and the numpy restatement of the kernel's Newton
iteration (black.cuh) -- against the exact implied vol of each fp64 quote (mpmath, 50 digits), at the bar of tests/ivol_cases.py.

The same quotes and bar run on the device in tests/test_gpu_ivol_edges.py.  Here they fix A of the bar: the restatement and the
bisection are printed with the largest |iv - iv*| / bar they reach (4.6 and 8.4 on the 3200-quote grid, 2.4 on the constructed
edges; A = 32).  The restatement must also need fewer than 64 iterations everywhere, and cutting its cap to 8 must break the bar.
"""
import numpy as np
import pytest

import ivol_cases as ic
from oracle import bsm

pytest.importorskip("mpmath")


@pytest.fixture(scope="module")
def grid():
    g = ic.random_grid()
    g["iv_star"], g["bar"] = ic.reference(g)
    return g


@pytest.fixture(scope="module")
def edges():
    e = ic.edge_cases()
    e["iv_star"], e["bar"] = ic.reference(e, "guess")
    return e


def _newton(c, **kw):
    return bsm.black_implied_vol_newton(c["F"], c["K"], c["T"], c["D"], c["price"], c["type"], **kw)


def _bisect(c):
    return np.array([bsm.infer_bsm_implied_vol(c["F"][i], c["T"][i], [c["K"][i]], [c["price"][i]], [c["type"][i]], c["D"][i])[0]
                     for i in range(c["F"].size)])


def _assert_bar(name, iv, c):
    ratio, nan_mismatch, bad = ic.check(iv, c["iv_star"], c["bar"])
    print(f"{name}: {c['F'].size} quotes, {np.isnan(c['iv_star']).sum()} outside the bounds, max |iv - iv*| / bar = {ratio:.2f} (A = {ic.A_BAR:g})")
    assert nan_mismatch.size == 0, [(c["type"][i], c["F"][i], c["K"][i], c["T"][i], c["D"][i], c["price"][i], iv[i]) for i in nan_mismatch[:5]]
    assert bad.size == 0, [(c["type"][i], c["F"][i], c["K"][i], c["T"][i], c["price"][i], iv[i], c["iv_star"][i]) for i in bad[:5]]
    return ratio


def test_grid_covers_what_it_claims(grid):
    z = np.log(grid["F"] / grid["K"]) / (grid["vol"] * np.sqrt(grid["T"]))
    assert grid["F"].size >= 3000 and set(grid["type"]) == set(ic.TYPES) and set(grid["F"]) == {1.0, ic.F_BTC}
    assert z.min() < -8.9 and z.max() > 8.9 and grid["D"].min() < 0.51 and grid["D"].max() > 0.99
    otm_put = (grid["K"] < grid["F"]) & np.isin(grid["type"], ("P", "IP"))
    assert np.sum(otm_put & (grid["price"] / grid["D"] < 2e-17 * grid["F"])) >= 50          # where the call-side parity gave NaN
    nan = np.isnan(grid["iv_star"])
    assert 0 < nan.sum() < grid["F"].size // 10                                            # in-the-money quotes rounded onto intrinsic


def test_newton_restatement_meets_the_bar_on_the_grid(grid):
    iv, it = _newton(grid)
    _assert_bar("newton restatement, grid", iv, grid)
    print(f"iterations: max {it.max()}, mean {it[np.isfinite(iv)].mean():.1f}")
    assert it.max() < bsm.MAX_ITER


def test_bisection_meets_the_bar_on_the_grid(grid):
    _assert_bar("bisection, grid", _bisect(grid), grid)


def test_edges(edges):
    """K = F, 1 ulp inside either no-arbitrage bound, vols on both sides of the bracket ends, T = 1e-6 and 30, quotes down to 1e-300 F,
    and invalid inputs (NaN whatever the price)"""
    iv, it = _newton(edges)
    _assert_bar("newton restatement, edges", iv, edges)
    _assert_bar("bisection, edges", _bisect(edges), edges)
    assert it.max() < bsm.MAX_ITER
    for tag in ("lower+1ulp", "upper-1ulp", "tiny", "atm", "ttm"):
        assert np.all(np.isfinite(edges["iv_star"][edges["tag"] == tag])), tag
    for tag in ("at-lower", "at-upper", "invalid"):           # with D != 1 the rounded D x bound may land inside: iv* decides
        assert np.all(np.isnan(edges["iv_star"][(edges["tag"] == tag) & ((edges["D"] == 1.0) | (tag == "invalid"))])), tag
    # outside the bracket: the nearer end (pinned), reached from quotes made at vols 0.9999e-8, 10.01 and 20
    out = np.isfinite(edges["iv_star"]) & ((edges["iv_star"] < bsm.VOL_LO) | (edges["iv_star"] > bsm.VOL_HI))
    assert out.sum() >= 20
    np.testing.assert_allclose(iv[out], np.where(edges["iv_star"][out] < 1.0, bsm.VOL_LO, bsm.VOL_HI), rtol=1e-15, atol=0)


def test_put_and_call_at_the_same_strike_and_vol_agree():
    pp = ic.parity_pairs()
    ty = np.array(["P", "C"])
    for k in range(pp["F"].size):
        args = [np.full(2, pp[key][k]) for key in ("F", "K", "T", "D")]
        price = np.array([pp["put"][k], pp["call"][k]])
        iv, _ = bsm.black_implied_vol_newton(*args, price, ty)
        iv_star, bar = ic.exact(pp["F"][k], pp["K"][k], pp["T"][k], 1.0, pp["put"][k], "P")
        assert iv_star == ic.exact(pp["F"][k], pp["K"][k], pp["T"][k], 1.0, pp["call"][k], "C")[0]
        tol = ic.A_BAR * bar + 4.0 * np.spacing(iv_star)
        assert np.all(np.abs(iv - iv_star) <= tol), (k, iv, iv_star, tol)
        assert abs(iv[0] - iv[1]) <= tol


def test_the_bar_catches_a_short_iteration_cap(grid):
    """the check is sharp enough to see an inversion stopped early: at 8 iterations most quotes are far over the bar"""
    iv, _ = _newton(grid, max_iter=8)
    _, _, bad = ic.check(iv, grid["iv_star"], grid["bar"])
    assert bad.size > 100
