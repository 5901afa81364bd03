"""GPU checks of ``price_chain_greeks`` (forward-mode Fourier sensitivities, DESIGN.md §4.2) against ``price_chain``, the numpy forward
mode of oracle/mgf_greeks.py, central differences of the public pricer, and the Monte Carlo pathwise route."""
import dataclasses

import numpy as np
import pytest

from oracle import mgf_greeks as G

pytestmark = pytest.mark.gpu

Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
HESTON_SETS = [(0.04, 0.05, 3.0, -0.6, 0.5), (0.8, 1.0, 2.0, 0.0, 2.0)]


def _chain(name):
    from stochvolmodels_b200 import OptionChain, get_btc_test_chain_data
    if name == "btc":
        return get_btc_test_chain_data()
    if name == "quickstart":
        return OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[T5])
    return OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.array([1.0, 1.02]), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5],
                       discfactors=np.array([0.99, 0.98]))


def _rel_close(got, ref, rtol, what):
    scale = max(float(np.max(np.abs(ref))), 1e-300)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err <= rtol, (what, err)
    return err


# (chain, params, is_spot_measure, order, etas)
LOGSV_CASES = {
    "quickstart": ("quickstart", Q, True, 2, None),
    "btc_spot": ("btc", "btc", True, 2, None),
    "btc_inverse": ("btc", "btc", False, 2, None),
    "eta": ("two", Q, True, 2, np.array([1.3, 0.8])),
    "first_order": ("two", Q, True, 1, None),
}


def _logsv_params(p):
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS
    if p == "btc":
        b = LOGSV_BTC_PARAMS
        return (b.sigma0, b.theta, b.kappa1, b.kappa2, b.beta, b.volvol)
    return p


@pytest.mark.parametrize("case", list(LOGSV_CASES))
def test_logsv_greeks_vs_price_chain_and_oracle(cuda_lib, case):
    from stochvolmodels_b200 import engine
    chain_name, p, spot, order, etas = LOGSV_CASES[case]
    chain, q = _chain(chain_name), _logsv_params(p)
    pc = engine.logsv_params_c(*q)
    M = len(chain.ttms)
    args = (pc, chain.ttms, chain.forwards, chain.discfactors, etas, chain.strikes_ttms, chain.optiontypes_ttms)
    prices, greeks, offsets, dlm, nfev = engine.logsv_price_chain_greeks(*args, is_spot_measure=spot, expansion_order=order, return_grids=True)
    ref = engine.logsv_price_chain(*args, is_spot_measure=spot, expansion_order=order)
    again = engine.logsv_price_chain_greeks(*args, is_spot_measure=spot, expansion_order=order, return_grids=True)
    for m in range(M):
        np.testing.assert_array_equal(prices[m], ref[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
    np.testing.assert_array_equal(again[1], greeks)
    np.testing.assert_array_equal(again[3], dlm)
    # the oracle runs the same mesh: right-hand-side evaluations per grid point agree everywhere
    out, grids = G.logsv_chain_greeks(q, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                      is_spot_measure=spot, order=order, etas=etas)
    np.testing.assert_array_equal(nfev, grids["nfev"])
    for d in range(6):
        for m in range(M):
            _rel_close(dlm[d, m], grids["dlog_mgf"][d, m], 1e-10, (case, "dlog_mgf", d, m))
    for m in range(M):
        sl = slice(offsets[m], offsets[m + 1])
        for r in range(8):
            _rel_close(greeks[r, sl], out[m][1 + r], 1e-10, (case, "row", r, m))


def _cd_forward(price, chain, m, h=1e-4):
    from stochvolmodels_b200 import OptionChain
    def bumped(f):
        fw = chain.forwards.copy()
        fw[m] *= f
        return price(OptionChain(ttms=chain.ttms, forwards=fw, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                                 discfactors=chain.discfactors))[m]
    hh = h * chain.forwards[m]
    p0, pp, pm = price(chain)[m], bumped(1 + h), bumped(1 - h)
    return (pp - pm) / (2 * hh), (pp - 2 * p0 + pm) / (hh * hh)


@pytest.mark.parametrize("chain_name,spot", [("quickstart", True), ("btc", True), ("btc", False)])
def test_logsv_public_greeks_vs_central_differences(cuda_lib, chain_name, spot):
    """delta / gamma against central differences of price_chain in the forwards; parameters against central differences with the
    transform grid pinned, within the gap the CPU oracle measures per chain (the derivative of the adaptive mesh choice)"""
    from test_fourier_greeks_oracle import ADAPTIVE_GAP
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSvParams, LogSVPricer
    chain = _chain(chain_name)
    params = LOGSV_BTC_PARAMS if chain_name == "btc" else LogSvParams(*Q)
    pricer = LogSVPricer()
    vs = float(params.sigma0 * np.sqrt(min(np.min(chain.ttms), 0.5 / 12.0)))
    g = pricer.price_chain_greeks(chain, params, is_spot_measure=spot)
    price = lambda c, p=params: pricer.price_chain(c, p, is_spot_measure=spot, vol_scaler=vs)
    for m in range(len(chain.ttms)):
        d_cd, g_cd = _cd_forward(price, chain, m)
        np.testing.assert_allclose(g.delta[m], d_cd, rtol=0, atol=1e-7)
        np.testing.assert_allclose(g.gamma[m], g_cd, rtol=0, atol=2e-4 * max(1.0, np.max(np.abs(g_cd))))
    for name in g.params:
        value, h = getattr(params, name), 1e-5
        up = price(chain, dataclasses.replace(params, **{name: value + h}))
        dn = price(chain, dataclasses.replace(params, **{name: value - h}))
        for m in range(len(chain.ttms)):
            cd = (up[m] - dn[m]) / (2 * h)
            assert np.max(np.abs(g.params[name][m] - cd)) <= ADAPTIVE_GAP[chain_name] * max(1.0, np.max(np.abs(cd))), (name, m)


@pytest.mark.parametrize("hp", HESTON_SETS)
def test_heston_greeks(cuda_lib, hp):
    from stochvolmodels_b200 import HestonParams, HestonPricer, engine
    chain = _chain("two")
    pricer, params = HestonPricer(), HestonParams(*hp)
    pc = engine.heston_params_c(*hp)
    args = (pc, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    prices, greeks, offsets, dlm = engine.heston_price_chain_greeks(*args, return_grids=True)
    ref = engine.heston_price_chain(*args)
    again = engine.heston_price_chain_greeks(*args, return_grids=True)
    for m in range(2):
        np.testing.assert_array_equal(prices[m], ref[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
    np.testing.assert_array_equal(again[1], greeks)
    out, odlm = G.heston_chain_greeks(hp, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    for d in range(5):
        for m in range(2):
            _rel_close(dlm[d, m], odlm[d, m], 1e-10, ("dlog_mgf", d, m))
    for m in range(2):
        for r in range(7):
            _rel_close(greeks[r, offsets[m]:offsets[m + 1]], out[m][1 + r], 1e-10, ("row", r, m))
    vs = float(min(0.3, np.sqrt(hp[0] * chain.ttms[0])))
    g = pricer.price_chain_greeks(chain, params)
    price = lambda c, p=params: pricer.price_chain(c, p, vol_scaler=vs)
    for m in range(2):
        d_cd, g_cd = _cd_forward(price, chain, m)
        np.testing.assert_allclose(g.delta[m], d_cd, rtol=0, atol=1e-7)
        np.testing.assert_allclose(g.gamma[m], g_cd, rtol=0, atol=2e-4 * max(1.0, np.max(np.abs(g_cd))))
    for name in g.params:
        value, h = getattr(params, name), 1e-6
        up = price(chain, dataclasses.replace(params, **{name: value + h}))
        dn = price(chain, dataclasses.replace(params, **{name: value - h}))
        for m in range(2):
            cd = (up[m] - dn[m]) / (2 * h)
            assert np.max(np.abs(g.params[name][m] - cd)) <= 1e-6 * max(1.0, np.max(np.abs(cd))), (name, m)


def _gate(mc_val, mc_se, ref, what):
    """the cross-route gate of the Monte Carlo greeks: 4 standard errors plus the 1e-3 Euler-bias allowance (DESIGN.md §6)"""
    assert np.all(np.abs(mc_val - ref) <= 4.0 * mc_se + 1e-3), (what, mc_val, ref, mc_se)


def test_cross_route_vs_monte_carlo_greeks(cuda_lib):
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    for pricer, params, kw in ((LogSVPricer(), LogSvParams(*Q), dict(nb_steps=252, seed=2024)),
                               (HestonPricer(), HestonParams(), dict(seed=5))):
        mc = pricer.model_mc_chain_greeks(chain, params, nb_path=4_000_000, **kw)
        fg = pricer.price_chain_greeks(chain, params)
        for m in range(2):
            _gate(mc.delta[m], mc.delta_se[m], fg.delta[m], (type(pricer).__name__, "delta", m))
            for name in fg.params:
                _gate(mc.params[name][m], mc.params_se[name][m], fg.params[name][m], (type(pricer).__name__, name, m))


def test_library_rejects_qvar_and_bad_order(cuda_lib):
    from stochvolmodels_b200 import _capi as C, engine
    chain = _chain("quickstart")
    M, ttms, fw, df, offsets, strikes, types = engine._chain_arrays(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                                    chain.optiontypes_ttms)
    prices, greeks = np.empty(5), np.empty((8, 5))
    pc = engine.logsv_params_c(*Q)
    for vt, order in ((C.Q_VAR, C.ORDER_SECOND), (C.LOG_RETURN, 7)):
        with pytest.raises(C.B200svError, match="not implemented"):
            C.call("b200sv_logsv_price_chain_greeks", engine.byref(pc), M, C.dptr(ttms), C.dptr(fw), C.dptr(df), None, C.iptr(offsets),
                   C.dptr(strikes), C.i8ptr(types), 1, vt, order, -1.0, 0, C.dptr(prices), C.dptr(greeks), None, None)
    with pytest.raises(C.B200svError, match="not implemented"):
        C.call("b200sv_heston_price_chain_greeks", engine.byref(engine.heston_params_c(*HESTON_SETS[0])), M, C.dptr(ttms), C.dptr(fw),
               C.dptr(df), C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), C.Q_VAR, -1.0, 0, C.dptr(prices), C.dptr(greeks), None)
