"""GPU checks of ``price_chain_hessian`` (second-order forward-mode Fourier sensitivities, DESIGN.md §4.4) against
``price_chain_greeks``, the numpy forward-over-forward restatement of mgf_hessian_oracle.py, and central differences of the public
first-order rows."""
import dataclasses

import numpy as np
import pytest

import mgf_hessian_oracle as H
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


def _logsv_params(p):
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS
    if p == "btc":
        b = LOGSV_BTC_PARAMS
        return (b.sigma0, b.theta, b.kappa1, b.kappa2, b.beta, b.volvol)
    return p


# (chain, params, is_spot_measure, order, etas): the first-order route's fixtures
LOGSV_CASES = {
    "quickstart": ("quickstart", Q, True, 2, None),
    "btc_spot": ("btc", "btc", True, 2, None),
    "btc_inverse": ("btc", "btc", False, 2, None),
    "eta": ("two", Q, True, 2, np.array([1.3, 0.8])),
    "first_order": ("two", Q, True, 1, None),
}


@pytest.mark.parametrize("case", list(LOGSV_CASES))
def test_logsv_hessian_vs_price_chain_greeks_and_oracle(cuda_lib, case):
    from stochvolmodels_b200 import engine
    chain_name, p, spot, order, etas = LOGSV_CASES[case]
    chain, q = _chain(chain_name), _logsv_params(p)
    pc = engine.logsv_params_c(*q)
    M = len(chain.ttms)
    args = (pc, chain.ttms, chain.forwards, chain.discfactors, etas, chain.strikes_ttms, chain.optiontypes_ttms)
    kw = dict(is_spot_measure=spot, expansion_order=order)
    prices, greeks, vanna, hess, offsets, dlm, d2lm = engine.logsv_price_chain_hessian(*args, **kw, return_grids=True)
    ref_p, ref_g, _, ref_dlm, _ = engine.logsv_price_chain_greeks(*args, **kw, return_grids=True)
    again = engine.logsv_price_chain_hessian(*args, **kw, return_grids=True)
    for m in range(M):
        np.testing.assert_array_equal(prices[m], ref_p[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
    np.testing.assert_array_equal(greeks, ref_g)
    np.testing.assert_array_equal(dlm, ref_dlm)
    for i in (1, 2, 3, 6):
        np.testing.assert_array_equal(again[i], (prices, greeks, vanna, hess, offsets, dlm, d2lm)[i])
    out, grids = H.logsv_chain_hessian(q, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                       is_spot_measure=spot, order=order, etas=etas)
    # d2lm_pq enters the Fourier sums as d2lm_pq + dlm_p dlm_q: relative to that integrand's scale (a row can be small against the primal
    # it is built from, e.g. (sigma0, sigma0) = 2 A_2 at y = 0 under FIRST order, where rounding of A is 3e-10 of the row itself)
    for r, (a, b) in enumerate(H.pairs(6)):
        for m in range(M):
            ref = grids["d2log_mgf"][r, m]
            scale = max(float(np.max(np.abs(ref))), float(np.max(np.abs(ref + ref_dlm[a, m] * ref_dlm[b, m]))))
            assert float(np.max(np.abs(d2lm[r, m] - ref))) <= 1e-10 * scale, (case, "d2log_mgf", r, m)
    for m in range(M):
        sl = slice(offsets[m], offsets[m + 1])
        for k in range(6):
            _rel_close(vanna[k, sl], out[m][1][k], 1e-10, (case, "vanna", k, m))
        for r in range(21):
            _rel_close(hess[r, sl], out[m][2][r], 1e-10, (case, "hessian", r, m))


def _cd_rows(greeks_of, chain, params, names, h):
    """central differences of the public first-order rows: in each parameter (hessian), and in each slice forward (vanna)"""
    hess = {}
    for q in names:
        v = getattr(params, q)
        up, dn = greeks_of(chain, dataclasses.replace(params, **{q: v + h})), greeks_of(chain, dataclasses.replace(params, **{q: v - h}))
        hess[q] = {p: [(up.params[p][m] - dn.params[p][m]) / (2 * h) for m in range(len(chain.ttms))] for p in names}
    from stochvolmodels_b200 import OptionChain
    vanna = {p: [] for p in names}
    for m in range(len(chain.ttms)):
        hf = 1e-5 * chain.forwards[m]
        bumped = []
        for s in (1, -1):
            fw = chain.forwards.copy()
            fw[m] += s * hf
            bumped.append(greeks_of(OptionChain(ttms=chain.ttms, forwards=fw, strikes_ttms=chain.strikes_ttms,
                                                optiontypes_ttms=chain.optiontypes_ttms, discfactors=chain.discfactors), params))
        for p in names:
            vanna[p].append((bumped[0].params[p][m] - bumped[1].params[p][m]) / (2 * hf))
    return vanna, hess


@pytest.mark.parametrize("chain_name,spot", [("quickstart", True), ("btc", True), ("btc", False)])
def test_logsv_public_hessian_vs_central_differences(cuda_lib, chain_name, spot):
    """vanna against central differences of price_chain_greeks in the forwards; the Hessian against central differences in the
    parameters with vol_scaler pinned, within the gap the CPU oracle measures per chain (the derivative of the adaptive mesh choice)"""
    from test_fourier_hessian_oracle import HESSIAN_ADAPTIVE_GAP
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSvParams, LogSVPricer, engine
    chain = _chain(chain_name)
    params = LOGSV_BTC_PARAMS if chain_name == "btc" else LogSvParams(*Q)
    pricer = LogSVPricer()
    vs = float(params.sigma0 * np.sqrt(min(np.min(chain.ttms), 0.5 / 12.0)))
    res = pricer.price_chain_hessian(chain, params, is_spot_measure=spot, vol_scaler=vs)
    greeks_of = lambda c, p: pricer.price_chain_greeks(c, p, is_spot_measure=spot, vol_scaler=vs)
    vanna, hess = _cd_rows(greeks_of, chain, params, engine.LOGSV_GREEK_PARAMS, 1e-5)
    for p in engine.LOGSV_GREEK_PARAMS:
        for m in range(len(chain.ttms)):
            cd = vanna[p][m]
            assert np.max(np.abs(res.vanna[p][m] - cd)) <= 1e-6 * max(1.0, np.max(np.abs(cd))), ("vanna", p, m)
            for q in engine.LOGSV_GREEK_PARAMS:
                cd = hess[q][p][m]
                gap = HESSIAN_ADAPTIVE_GAP[chain_name] * max(1.0, np.max(np.abs(cd)))
                assert np.max(np.abs(res.hessian[p][q][m] - cd)) <= gap, ("hessian", p, q, m)


@pytest.mark.parametrize("hp", HESTON_SETS)
def test_heston_hessian(cuda_lib, hp):
    from stochvolmodels_b200 import HestonParams, HestonPricer, engine
    chain = _chain("two")
    pc = engine.heston_params_c(*hp)
    args = (pc, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    prices, greeks, vanna, hess, offsets, dlm, d2lm = engine.heston_price_chain_hessian(*args, return_grids=True)
    ref_p, ref_g, _, ref_dlm = engine.heston_price_chain_greeks(*args, return_grids=True)
    again = engine.heston_price_chain_hessian(*args, return_grids=True)
    for m in range(2):
        np.testing.assert_array_equal(prices[m], ref_p[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
    np.testing.assert_array_equal(greeks, ref_g)
    np.testing.assert_array_equal(dlm, ref_dlm)
    for i in (1, 2, 3, 6):
        np.testing.assert_array_equal(again[i], (prices, greeks, vanna, hess, offsets, dlm, d2lm)[i])
    out, _, od2lm = H.heston_chain_hessian(hp, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    for r in range(15):
        for m in range(2):
            if np.any(od2lm[r, m]):
                _rel_close(d2lm[r, m], od2lm[r, m], 1e-10, ("d2log_mgf", r, m))
            else:
                assert not np.any(d2lm[r, m])
    for m in range(2):
        sl = slice(offsets[m], offsets[m + 1])
        for k in range(5):
            _rel_close(vanna[k, sl], out[m][1][k], 1e-10, ("vanna", k, m))
        for r in range(15):
            if np.any(out[m][2][r]):
                _rel_close(hess[r, sl], out[m][2][r], 1e-10, ("hessian", r, m))
    pricer, params = HestonPricer(), HestonParams(*hp)
    vs = float(min(0.3, np.sqrt(hp[0] * chain.ttms[0])))
    res = pricer.price_chain_hessian(chain, params, vol_scaler=vs)
    vanna_cd, hess_cd = _cd_rows(lambda c, p: pricer.price_chain_greeks(c, p, vol_scaler=vs), chain, params, engine.HESTON_GREEK_PARAMS, 1e-6)
    for p in engine.HESTON_GREEK_PARAMS:
        for m in range(2):
            cd = vanna_cd[p][m]
            assert np.max(np.abs(res.vanna[p][m] - cd)) <= 1e-6 * max(1.0, np.max(np.abs(cd))), ("vanna", p, m)
            for q in engine.HESTON_GREEK_PARAMS:
                cd = hess_cd[q][p][m]
                assert np.max(np.abs(res.hessian[p][q][m] - cd)) <= 1e-6 * max(1.0, np.max(np.abs(cd))), ("hessian", p, q, m)


def test_library_rejects_qvar(cuda_lib):
    from stochvolmodels_b200 import _capi as C, engine
    chain = _chain("quickstart")
    M, ttms, fw, df, offsets, strikes, types = engine._chain_arrays(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                                    chain.optiontypes_ttms)
    prices, greeks, vanna, hess = np.empty(5), np.empty((8, 5)), np.empty((6, 5)), np.empty((21, 5))
    with pytest.raises(C.B200svError, match="not implemented"):
        C.call("b200sv_logsv_price_chain_hessian", engine.byref(engine.logsv_params_c(*Q)), M, C.dptr(ttms), C.dptr(fw), C.dptr(df), None,
               C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), 1, C.Q_VAR, C.ORDER_SECOND, -1.0, 0, C.dptr(prices), C.dptr(greeks), None,
               None, C.dptr(vanna), C.dptr(hess), None)
    with pytest.raises(C.B200svError, match="not implemented"):
        C.call("b200sv_heston_price_chain_hessian", engine.byref(engine.heston_params_c(*HESTON_SETS[0])), M, C.dptr(ttms), C.dptr(fw),
               C.dptr(df), C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), C.Q_VAR, -1.0, 0, C.dptr(prices), C.dptr(greeks), None,
               C.dptr(vanna[:5]), C.dptr(hess[:15]), None)
