"""GPU checks of theta (``price_chain_greeks(with_theta=True)``, ``compute_chain_ivol_greeks(with_theta=True)``; DESIGN.md §4.8): every
other output bit for bit as without it, the numpy restatement of tests/fourier_theta_oracle.py, the theta kernel's mesh, central
differences of the GPU pricer in ttms[m] alone, and the implied-vol transform."""
import numpy as np
import pytest

import fourier_theta_oracle as O
from test_fourier_theta_oracle import ADAPTIVE_THETA_GAP, hawkes_golden, logsv_golden

pytestmark = pytest.mark.gpu


def _chain(ttms, fwd, df, K, T):
    from stochvolmodels_b200 import OptionChain
    return OptionChain(ttms=np.asarray(ttms, dtype=float), forwards=np.asarray(fwd, dtype=float), discfactors=np.asarray(df, dtype=float),
                       strikes_ttms=list(K), optiontypes_ttms=list(T))


def _rel_close(got, ref, rtol, floor, what):
    err = float(np.max(np.abs(got - ref)))
    assert err <= rtol * max(float(np.max(np.abs(ref))), floor), (what, err)


def _same_outputs(plain, theta):
    """the outputs of the _greeks twin, bit for bit"""
    for a, b in zip(plain, theta):
        if isinstance(a, list):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y)
        else:
            np.testing.assert_array_equal(a, b)


LOGSV_CASES = [("g1_quickstart", True, 2), ("btc", True, 2), ("btc", False, 2), ("c3_5x21", True, 1), ("c3_5x21", False, 2)]


@pytest.mark.parametrize("tag,spot,order", LOGSV_CASES)
def test_logsv_theta_bitwise_twin_and_oracle(cuda_lib, tag, spot, order):
    from stochvolmodels_b200 import engine
    q, ttms, fwd, df, K, T = logsv_golden(tag)
    args = (engine.logsv_params_c(*q), ttms, fwd, df, None, K, T)
    kw = dict(is_spot_measure=spot, expansion_order=order, return_grids=True)
    plain = engine.logsv_price_chain_greeks(*args, **kw)
    out = engine.logsv_price_chain_greeks(*args, **kw, with_theta=True)
    again = engine.logsv_price_chain_greeks(*args, **kw, with_theta=True)
    _same_outputs(plain, out[:5])
    _same_outputs(out, again)
    theta, dlm_t, nfev_t = out[5:]
    offsets = out[2]
    np.testing.assert_array_equal(nfev_t, plain[4])                 # the theta kernel stepped the pricing route's mesh
    ref, gr = O.logsv_chain_theta(q, ttms, fwd, df, K, T, spot, order)
    for m in range(len(ttms)):
        _rel_close(dlm_t[m], gr["dlog_mgf_theta"][m], 1e-10, 1e-300, (tag, "dlog_mgf_theta", m))
        _rel_close(theta[offsets[m]:offsets[m + 1]], ref[m], 1e-10, 1e-6, (tag, "theta", m))


@pytest.mark.parametrize("which", ["dflt", "alt"])
@pytest.mark.parametrize("spot", [True, False])
def test_hawkes_theta_bitwise_twin_and_oracle(cuda_lib, which, spot):
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    p, ttms, fwd, df, K, T = hawkes_golden(which)
    args = (_params_c(**p), ttms, fwd, df, K, T)
    plain = engine.hawkesjd_price_chain_greeks(*args, is_spot_measure=spot, return_grids=True)
    out = engine.hawkesjd_price_chain_greeks(*args, is_spot_measure=spot, return_grids=True, with_theta=True)
    again = engine.hawkesjd_price_chain_greeks(*args, is_spot_measure=spot, return_grids=True, with_theta=True)
    _same_outputs(plain, out[:5])
    _same_outputs(out, again)
    theta, dlm_t, nfev_t = out[5:]
    offsets = out[2]
    np.testing.assert_array_equal(nfev_t, plain[4])
    ref, gr = O.hawkes_chain_theta(p, ttms, fwd, df, K, T, spot)
    for m in range(3):
        _rel_close(dlm_t[m], gr["dlog_mgf_theta"][m], 1e-10, 1e-300, (which, "dlog_mgf_theta", m))
        _rel_close(theta[offsets[m]:offsets[m + 1]], ref[m], 1e-10, 1e-6, (which, "theta", m))


HESTON_SETS = [(0.04, 0.05, 3.0, -0.6, 0.5), (0.8, 1.0, 2.0, 0.0, 2.0)]


def _heston_chain():
    ttms, fwd = np.array([0.0429, 0.1012, 0.1984, 0.5, 1.0]), np.array([1.0, 1.01, 1.02, 1.03, 1.05])
    df = np.array([1.0, 0.999, 0.995, 0.99, 0.98])
    return ttms, fwd, df, [np.array([0.8, 0.9, 1.0, 1.1, 1.2]) * f for f in fwd], [np.array(["P", "P", "C", "C", "C"])] * 5


@pytest.mark.parametrize("params", HESTON_SETS)
def test_heston_theta_bitwise_twin_oracle_and_central_differences(cuda_lib, params):
    from stochvolmodels_b200 import HestonParams, HestonPricer, engine
    from oracle import mgf
    ttms, fwd, df, K, T = _heston_chain()
    from stochvolmodels_b200.pricers.heston_pricer import _params_c
    pc = _params_c(*params)
    vs = mgf.heston_vol_scaler(params[0], ttms)
    args = (pc, ttms, fwd, df, K, T)
    plain = engine.heston_price_chain_greeks(*args, vol_scaler=vs, return_grids=True)
    out = engine.heston_price_chain_greeks(*args, vol_scaler=vs, return_grids=True, with_theta=True)
    _same_outputs(plain, out[:4])
    _same_outputs(out, engine.heston_price_chain_greeks(*args, vol_scaler=vs, return_grids=True, with_theta=True))
    theta, dlm_t = out[4:]
    offsets = out[2]
    ref, dlm_ref = O.heston_chain_theta(params, ttms, fwd, df, K, T, vs)
    v0, th, ka, rho, vv = params
    pricer, hp = HestonPricer(), HestonParams(v0=v0, theta=th, kappa=ka, rho=rho, volvol=vv)
    for m in range(5):
        _rel_close(dlm_t[m], dlm_ref[m], 1e-10, 1e-300, ("dlog_mgf_theta", m))
        _rel_close(theta[offsets[m]:offsets[m + 1]], ref[m], 1e-10, 1e-6, ("theta", m))
        h = 1e-5 * ttms[m]
        tu, td = ttms.copy(), ttms.copy()
        tu[m] += h
        td[m] -= h
        cd = -(pricer.price_chain(_chain(tu, fwd, df, K, T), hp, vol_scaler=vs)[m]
               - pricer.price_chain(_chain(td, fwd, df, K, T), hp, vol_scaler=vs)[m]) / (2 * h)
        _rel_close(theta[offsets[m]:offsets[m + 1]], cd, 1e-9, 1.0, ("cd", m))


@pytest.mark.parametrize("tag", ["g1_quickstart", "btc"])
def test_logsv_theta_vs_central_differences_of_the_gpu_pricer(cuda_lib, tag):
    """re-pricing with ttms[m] alone moved, the grid pinned at the unmoved chain's default and no backbone: within the CPU-measured gap"""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer
    from oracle import mgf
    q, ttms, fwd, df, K, T = logsv_golden(tag)
    params = LogSvParams(*q)
    pricer = LogSVPricer()
    vs = mgf.logsv_vol_scaler(q[0], ttms)
    g = pricer.price_chain_greeks(_chain(ttms, fwd, df, K, T), params, with_theta=True, vol_scaler=vs)
    for m in range(len(ttms)):
        h = 1e-5 * ttms[m]
        tu, td = ttms.copy(), ttms.copy()
        tu[m] += h
        td[m] -= h
        cd = -(pricer.price_chain(_chain(tu, fwd, df, K, T), params, vol_scaler=vs)[m]
               - pricer.price_chain(_chain(td, fwd, df, K, T), params, vol_scaler=vs)[m]) / (2 * h)
        _rel_close(g.theta[m], cd, ADAPTIVE_THETA_GAP, 1.0, (tag, m))


def test_public_theta_and_ivol_theta(cuda_lib):
    """price_chain_greeks / compute_chain_ivol_greeks with theta: the rest bit for bit, the ivols those of compute_chain_prices_with_vols,
    and the ivol theta against central differences of compute_chain_prices_with_vols in ttms[m] (grid pinned)"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, LogSvParams, LogSVPricer
    from oracle import mgf
    q, ttms, fwd, df, K, T = logsv_golden("g1_quickstart")
    chain = _chain(ttms, fwd, df, K, T)
    vs = mgf.logsv_vol_scaler(q[0], ttms)
    p, hw_ttms, hw_fwd, hw_df, hw_K, hw_T = hawkes_golden("alt")
    cases = [(LogSVPricer(), LogSvParams(*q), chain, vs),
             (HawkesJDPricer(), HawkesJDParams(**p), _chain(hw_ttms, hw_fwd, hw_df, hw_K, hw_T), 0.1)]
    for pricer, params, ch, scaler in cases:
        plain = pricer.price_chain_greeks(ch, params, vol_scaler=scaler)
        g = pricer.price_chain_greeks(ch, params, vol_scaler=scaler, with_theta=True)
        for name in ("prices", "delta", "gamma"):
            _same_outputs(getattr(plain, name), getattr(g, name))
        for name in plain.params:
            _same_outputs(plain.params[name], g.params[name])
        iv_plain = pricer.compute_chain_ivol_greeks(ch, params, vol_scaler=scaler)
        iv = pricer.compute_chain_ivol_greeks(ch, params, vol_scaler=scaler, with_theta=True)
        assert iv_plain.theta is None
        ref_ivols = pricer.compute_chain_prices_with_vols(ch, params, vol_scaler=scaler)[1]
        _same_outputs(iv.ivols, ref_ivols)
        _same_outputs(iv.delta, iv_plain.delta)
        for name in iv_plain.params:
            _same_outputs(iv.params[name], iv_plain.params[name])
        for m in range(len(ch.ttms)):
            h = 1e-5 * ch.ttms[m]
            tu, td = ch.ttms.copy(), ch.ttms.copy()
            tu[m] += h
            td[m] -= h
            up = pricer.compute_chain_prices_with_vols(_chain(tu, ch.forwards, ch.discfactors, ch.strikes_ttms, ch.optiontypes_ttms), params,
                                                       vol_scaler=scaler)[1][m]
            dn = pricer.compute_chain_prices_with_vols(_chain(td, ch.forwards, ch.discfactors, ch.strikes_ttms, ch.optiontypes_ttms), params,
                                                       vol_scaler=scaler)[1][m]
            _rel_close(iv.theta[m], -(up - dn) / (2 * h), 1e-6, 1.0, (type(pricer).__name__, m))


def test_bsm_implied_vol_theta_black_in_black_out(cuda_lib):
    """Black prices with a known sigma(T) = a + b T and theta = -(B_sigma b + B_T): the ivols equal b200sv_bsm_implied_vols bit for bit
    and the ivol theta is -b; a NaN quote gives NaN"""
    from stochvolmodels_b200 import engine
    a, b = 0.2, 0.1
    ttms, fwd, df = np.array([0.05, 0.25, 1.0, 2.0]), np.array([1.0, 100.0, 1.0, 1.0]), np.array([1.0, 0.99, 0.95, 0.9])
    K = [np.array([0.8, 1.0, 1.2]) * f for f in fwd]
    T = [np.array(["P", "C", "C"]), np.array(["P", "IC", "C"]), np.array(["IP", "C", "C"]), np.array(["P", "P", "C"])]
    prices, theta = [], []
    for m in range(4):
        vol = a + b * ttms[m]
        calls = np.array([t in ("C", "IC") for t in T[m]])
        prices.append(np.array([O.black_price(fwd[m], k, ttms[m], vol, c, df[m]) for k, c in zip(K[m], calls)]))
        vega = O.black_vega(fwd[m], K[m], ttms[m], vol, df[m])
        theta.append(-(vega * b + vega * vol / (2 * ttms[m])))
    prices[0][0] = -1.0
    ivols, ivol_theta = engine.bsm_implied_vol_theta(ttms, fwd, df, K, T, prices, np.concatenate(theta))
    ref = engine.bsm_implied_vols(ttms, fwd, df, K, T, prices)
    _same_outputs(ivols, ref)
    assert np.isnan(ivol_theta[0])
    np.testing.assert_allclose(ivol_theta[1:], -b, rtol=0, atol=1e-9)
