"""CPU checks of the theta of the Fourier chain pricers (DESIGN.md §4.8): the numpy restatement in tests/fourier_theta_oracle.py against
central differences of the mesh-replay pricers (only slice m's last step moved), of the adaptive oracle pricer with the grid pinned and
of the Heston closed form; the Black-76 theta transform; and the public methods' routing and rejections without the library."""
import numpy as np
import pytest

import fourier_theta_oracle as O
from conftest import load_golden
from oracle import bsm, mgf
from oracle import hawkes_greeks as H
from oracle import mgf_greeks as G

MESH_EPS = 2e-6          # truncation-dominated below: 1e-5 gives 5.9e-9 on btc slice 0, 3e-6 gives 5.6e-10
MESH_RTOL = 1e-8
# Central differences of the ADAPTIVE oracle pricer in ttms[m] alone (vol_scaler pinned, step 1e-5 ttm) against the mesh-held theta,
# relative to max(1, max |cd|): measured 6.0e-11 (quickstart), 5.4e-9 (btc), 9.3e-9 (c3_5x21) on both measures -- a small bump of T
# keeps the accepted mesh but for its last step, so the scheme's theta is what a re-pricing sees.
ADAPTIVE_THETA_GAP = 3e-8


def logsv_golden(tag):
    g = load_golden(f"logsv_fourier_{tag}.npz")
    M = int(g["nslices"])
    return (tuple(float(v) for v in g["params"]), g["ttms"], g["forwards"], g["discfactors"], [g[f"strikes_{m}"] for m in range(M)],
            [g[f"types_{m}"] for m in range(M)])


def hawkes_golden(which):
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    return p, g["ttms"], g["forwards"], g["discfactors"], [g["strikes"]] * 3, [g["types"]] * 3


def _mesh_cd(price_on_meshes, meshes, m):
    up, dn = list(meshes), list(meshes)
    up[m] = O.bump_last_step(meshes[m], MESH_EPS)
    dn[m] = O.bump_last_step(meshes[m], -MESH_EPS)
    return -(price_on_meshes(up)[m] - price_on_meshes(dn)[m]) / (2 * MESH_EPS)


def _close(got, ref, rtol, floor, what):
    err = float(np.max(np.abs(got - ref)))
    assert err <= rtol * max(float(np.max(np.abs(ref))), floor), (what, err)


@pytest.mark.parametrize("tag", ["g1_quickstart", "btc", "c3_5x21"])
@pytest.mark.parametrize("spot", [True, False])
@pytest.mark.parametrize("order", [1, 2])
def test_logsv_theta_vs_central_differences_of_the_last_step(tag, spot, order):
    q, ttms, fwd, df, K, T = logsv_golden(tag)
    theta, gr = O.logsv_chain_theta(q, ttms, fwd, df, K, T, spot, order)
    price = lambda meshes: G.logsv_chain_prices_on_meshes(q, ttms, fwd, df, K, T, meshes, gr["vol_scaler"], spot, order)[0]
    # the replayed meshes are the adaptive pricer's: same prices bit for bit
    ref = mgf.logsv_chain_prices(q, ttms, fwd, df, K, T, spot, order)
    for m in range(len(ttms)):
        np.testing.assert_array_equal(price(gr["meshes"])[m], ref[m])
        _close(theta[m], _mesh_cd(price, gr["meshes"], m), MESH_RTOL, 1e-3, (tag, m))


@pytest.mark.parametrize("which", ["dflt", "alt"])
@pytest.mark.parametrize("spot", [True, False])
def test_hawkes_theta_vs_central_differences_of_the_last_step(which, spot):
    p, ttms, fwd, df, K, T = hawkes_golden(which)
    theta, gr = O.hawkes_chain_theta(p, ttms, fwd, df, K, T, spot)
    price = lambda meshes: H.hawkes_chain_prices_on_meshes(p, ttms, fwd, df, K, T, meshes, gr["vol_scaler"], spot)[0]
    for m in range(3):
        _close(theta[m], _mesh_cd(price, gr["meshes"], m), MESH_RTOL, 1e-3, (which, m))


@pytest.mark.parametrize("tag", ["g1_quickstart", "btc", "c3_5x21"])
@pytest.mark.parametrize("spot", [True, False])
def test_logsv_theta_vs_central_differences_of_the_adaptive_pricer(tag, spot):
    q, ttms, fwd, df, K, T = logsv_golden(tag)
    theta, gr = O.logsv_chain_theta(q, ttms, fwd, df, K, T, spot, 2)
    for m in range(len(ttms)):
        h = 1e-5 * ttms[m]
        tu, td = ttms.copy(), ttms.copy()
        tu[m] += h
        td[m] -= h
        pu = mgf.logsv_chain_prices(q, tu, fwd, df, K, T, spot, 2, vol_scaler=gr["vol_scaler"])[m]
        pd = mgf.logsv_chain_prices(q, td, fwd, df, K, T, spot, 2, vol_scaler=gr["vol_scaler"])[m]
        _close(theta[m], -(pu - pd) / (2 * h), ADAPTIVE_THETA_GAP, 1.0, (tag, m))


@pytest.mark.parametrize("params", [(0.04, 0.05, 3.0, -0.6, 0.5), (0.8, 1.0, 2.0, 0.0, 2.0)])
def test_heston_theta_vs_central_differences_of_the_closed_form(params):
    """unit forwards (on the 7e4 btc forwards the differences are rounding-limited at ~1e-9); step 1e-5 ttm: measured <= 3.2e-10 of
    max(1, |cd|)"""
    ttms, fwd = np.array([0.0429, 0.1012, 0.1984, 0.5, 1.0]), np.array([1.0, 1.01, 1.02, 1.03, 1.05])
    df = np.array([1.0, 0.999, 0.995, 0.99, 0.98])
    K = [np.array([0.8, 0.9, 1.0, 1.1, 1.2]) * f for f in fwd]
    T = [np.array(["P", "P", "C", "C", "C"])] * len(ttms)
    vs = mgf.heston_vol_scaler(params[0], ttms)
    theta, _ = O.heston_chain_theta(params, ttms, fwd, df, K, T, vs)
    for m in range(len(ttms)):
        h = 1e-5 * ttms[m]
        tu, td = ttms.copy(), ttms.copy()
        tu[m] += h
        td[m] -= h
        cd = -(mgf.heston_chain_prices(params, tu, fwd, df, K, T, vs)[m] - mgf.heston_chain_prices(params, td, fwd, df, K, T, vs)[m]) / (2 * h)
        _close(theta[m], cd, 1e-9, 1.0, m)


# ---- the Black-76 theta transform ------------------------------------------------------------------------------------------------------
QUOTES = [(1.0, 0.8, 0.25, 0.99, "P"), (1.0, 1.0, 0.25, 0.99, "C"), (1.0, 1.3, 1.5, 0.95, "C"), (100.0, 90.0, 0.05, 1.0, "C"),
          (100.0, 120.0, 2.0, 0.9, "IP")]


@pytest.mark.parametrize("quote", QUOTES)
def test_black_theta_transform_vs_central_differences_of_the_inversion(quote):
    F, K, T0, D, ty = quote
    call = ty in ("C", "IC")
    p0 = O.black_price(F, K, T0, 0.35, call, D)
    theta = 0.07 * p0                              # any model theta: the price moves as p0 - theta (T - T0)
    inv = lambda T: bsm.infer_bsm_implied_vol(F, T, np.array([K]), np.array([p0 - theta * (T - T0)]), np.array([ty]), D)[0]
    vol = inv(T0)
    h = 1e-4 * T0
    cd = -(inv(T0 + h) - inv(T0 - h)) / (2 * h)
    assert abs(O.black_ivol_theta(F, K, T0, D, vol, theta) - cd) <= 1e-6 * max(1.0, abs(cd)), (cd,)


def test_black_in_black_out_returns_the_slope_of_the_vol():
    """Black prices with sigma(T) = a + b T: P(T) = B(sigma(T), T), theta = -(B_sigma b + B_T); the transform returns -b"""
    a, b = 0.2, 0.1
    for F, K, T, D, ty in QUOTES:
        vol = a + b * T
        vega = O.black_vega(F, K, T, vol, D)
        theta = -(vega * b + vega * vol / (2 * T))
        assert abs(O.black_ivol_theta(F, K, T, D, vol, theta) + b) <= 1e-12
    assert np.isnan(O.black_ivol_theta(1.0, 1.0, 1.0, 1.0, np.nan, 0.1))
    assert O.black_ivol_theta(1.0, 1.0, 1.0, 1.0, 10.0, 0.1) == 0.0


# ---- routing and rejections: nothing reaches the library ------------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


def _pricers():
    from stochvolmodels_b200 import (HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer,
                                     OptionChain)
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[np.array([0.9, 1.1])],
                        optiontypes_ttms=[np.array(["P", "C"])])
    return chain, [(LogSVPricer(), LogSvParams()), (HestonPricer(), HestonParams()), (HawkesJDPricer(), HawkesJDParams())]


def test_theta_rejections_before_any_library_call(no_library):
    chain, pricers = _pricers()
    for pricer, params in pricers:
        with pytest.raises(NotImplementedError):
            pricer.price_chain_hessian(chain, params, with_theta=True)
        with pytest.raises(NotImplementedError):
            pricer.compute_chain_ivol_hessian(chain, params, with_theta=True)
        with pytest.raises(NotImplementedError):
            pricer.price_chain_greeks(chain, params, with_theta=True, variable_type=2)
    with pytest.raises(NotImplementedError):
        pricers[0][0].price_chain_greeks(chain, pricers[0][1], with_theta=True, is_analytic=True)
    with pytest.raises(NotImplementedError):
        pricers[0][0].compute_chain_ivol_greeks(chain, pricers[0][1], with_theta=True, is_stiff_solver=True)


def test_with_theta_routes_to_the_theta_entry_points(monkeypatch):
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.fourier_greeks import ChainIvolGreeks, FourierChainGreeks, FourierChainHessian
    chain, pricers = _pricers()
    seen = []

    def fake(name, n):
        def f(*args, with_theta=False, **kw):
            seen.append((name, with_theta))
            out = ([np.zeros(2)], np.arange((2 + n) * 2, dtype=float).reshape(2 + n, 2), np.array([0, 2], dtype=np.int32))
            return out + ((np.array([0.5, -0.25]),) if with_theta else ())
        return f
    for name, n in (("logsv", 6), ("heston", 5), ("hawkesjd", 15)):
        monkeypatch.setattr(engine, f"{name}_price_chain_greeks", fake(name, n))
    for (pricer, params), name in zip(pricers, ("logsv", "heston", "hawkesjd")):
        plain, with_theta = pricer.price_chain_greeks(chain, params), pricer.price_chain_greeks(chain, params, with_theta=True)
        assert plain.theta is None
        np.testing.assert_array_equal(with_theta.theta[0], [0.5, -0.25])
        np.testing.assert_array_equal(with_theta.params[list(with_theta.params)[0]][0], plain.params[list(plain.params)[0]][0])
        assert seen[-2:] == [(name, False), (name, True)]
    # the *Hessian result types still construct positionally; theta is keyword-only and defaults to None
    h = FourierChainHessian([np.zeros(1)], [np.zeros(1)], [np.zeros(1)], {}, {}, {})
    assert h.theta is None and ChainIvolGreeks([np.zeros(1)], [np.zeros(1)], None, {}).theta is None
    assert FourierChainGreeks([], [], [], {}, theta=[np.ones(1)]).theta[0][0] == 1.0


def test_ivol_theta_argument_checks_before_any_library_call(no_library):
    from stochvolmodels_b200 import engine
    args = (np.array([0.25]), np.ones(1), np.ones(1), [np.array([0.9, 1.1])], [np.array(["P", "C"])], [np.array([0.01, 0.02])])
    with pytest.raises(ValueError):
        engine.bsm_implied_vol_theta(*args, np.zeros(3))
