"""GPU checks of ``HawkesJDPricer.price_chain_hessian`` (second-order forward-mode Fourier sensitivities, DESIGN.md §4.5) against
``price_chain_greeks`` and ``price_chain``, the numpy forward-over-forward restatement of hawkes_hessian_oracle.py, and central differences
of the public first-order rows."""
import dataclasses

import numpy as np
import pytest

import hawkes_hessian_oracle as O
from conftest import load_golden
from oracle import hawkes, mgf

pytestmark = pytest.mark.gpu


def _case(which):
    from stochvolmodels_b200 import HawkesJDParams, OptionChain
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    chain = OptionChain(ttms=g["ttms"], forwards=g["forwards"], strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["types"]] * 3,
                        discfactors=g["discfactors"])
    return p, HawkesJDParams(**p), chain


def _rel_close(got, ref, rtol, what):
    scale = max(float(np.max(np.abs(ref))), 1e-300)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err <= rtol, (what, err)


def _call_hessian(pc, chain, spot):
    """b200sv_hawkesjd_price_chain_hessian with every optional output, nfev included"""
    from stochvolmodels_b200 import _capi as C, engine
    ch = engine._chain_arrays(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    J, P = ch.strikes.shape[0], 500
    out = dict(prices=np.empty(J), greeks=np.empty((17, J)), dlm=np.empty((15, ch.M, P), dtype=np.complex128),
               nfev=np.empty(P, dtype=np.int32), vanna=np.empty((15, J)), hess=np.empty((120, J)),
               d2lm=np.empty((120, ch.M, P), dtype=np.complex128))
    C.call("b200sv_hawkesjd_price_chain_hessian", engine.byref(pc), *C.chain_ptrs(ch), int(spot), -1.0, P, C.dptr(out["prices"]),
           C.dptr(out["greeks"]), C.dptr(out["dlm"]), C.iptr(out["nfev"]), C.dptr(out["vanna"]), C.dptr(out["hess"]), C.dptr(out["d2lm"]))
    return out, ch.offsets


@pytest.fixture(scope="module")
def oracle_d2lm():
    """hawkes_hessian_oracle's grids per parameter set (d2 log_mgf does not depend on the measure: the grid sits on Re phi = -1/2 under both)"""
    cache = {}

    def get(which):
        if which not in cache:
            p, _, chain = _case(which)
            cache[which] = O.hawkes_chain_hessian(p, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                  chain.optiontypes_ttms)[1]
        return cache[which]
    return get


@pytest.mark.parametrize("which,spot", [("dflt", True), ("dflt", False), ("alt", True), ("alt", False)])
def test_hawkes_hessian_vs_greeks_and_oracle(cuda_lib, oracle_d2lm, which, spot):
    from stochvolmodels_b200 import HawkesJDPricer, engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    p, params, chain = _case(which)
    pc = _params_c(**p)
    out, offsets = _call_hessian(pc, chain, spot)
    again = _call_hessian(pc, chain, spot)[0]
    for key in out:
        np.testing.assert_array_equal(again[key], out[key], err_msg=key)
    ref_p, ref_g, _, ref_dlm, ref_nfev = engine.hawkesjd_price_chain_greeks(pc, chain.ttms, chain.forwards, chain.discfactors,
                                                                            chain.strikes_ttms, chain.optiontypes_ttms, is_spot_measure=spot,
                                                                            return_grids=True)
    np.testing.assert_array_equal(out["prices"], np.concatenate(ref_p))
    np.testing.assert_array_equal(out["prices"], np.concatenate(HawkesJDPricer().price_chain(chain, params, is_spot_measure=spot)))
    np.testing.assert_array_equal(out["greeks"], ref_g)
    np.testing.assert_array_equal(out["dlm"], ref_dlm)
    np.testing.assert_array_equal(out["nfev"], ref_nfev)
    grids = oracle_d2lm(which)
    d2lm, dlm = out["d2lm"], out["dlm"]
    # d2lm_pq enters the Fourier sums as d2lm_pq + dlm_p dlm_q: relative to that integrand's scale
    for r, (a, b) in enumerate(O.PAIRS):
        for m in range(3):
            ref = grids["d2log_mgf"][r, m]
            scale = max(float(np.max(np.abs(ref))), float(np.max(np.abs(ref + dlm[a, m] * dlm[b, m]))))
            assert float(np.max(np.abs(d2lm[r, m] - ref))) <= 1e-10 * scale, (which, spot, "d2log_mgf", O.NAMES[a], O.NAMES[b], m)
    for a, b in (("lambda_p", "lambda_p"), ("lambda_p", "lambda_m"), ("lambda_m", "lambda_m")):
        assert not np.any(d2lm[O.PAIRS.index((O.NAMES.index(a), O.NAMES.index(b)))])
    vs = float(np.clip(p["sigma"], 0.2, 0.5) * np.sqrt(min(np.min(chain.ttms), 1.0 / 12.0)))
    phi = mgf.phi_grid(vs, True, hawkes.MAX_PHI)
    rows = O.chain_rows(p, phi, grids["log_mgf"], grids["dlog_mgf"], grids["d2log_mgf"], chain.forwards, chain.discfactors,
                        chain.strikes_ttms, chain.optiontypes_ttms, spot)
    for m in range(3):
        sl = slice(offsets[m], offsets[m + 1])
        for k in range(15):
            _rel_close(out["vanna"][k, sl], rows[m][0][k], 1e-10, (which, spot, "vanna", O.NAMES[k], m))
        for r in range(120):
            _rel_close(out["hess"][r, sl], rows[m][1][r], 1e-10, (which, spot, "hessian", r, m))


def _btc():
    from stochvolmodels_b200 import HawkesJDParams, get_btc_test_chain_data
    return HawkesJDParams(), get_btc_test_chain_data()


@pytest.mark.parametrize("chain_name,which,spot", [("hawkes", "dflt", True), ("hawkes", "alt", True), ("hawkes", "alt", False),
                                                   ("btc", None, True)])
def test_hawkes_public_hessian_vs_central_differences(cuda_lib, chain_name, which, spot):
    """vanna against central differences of price_chain_greeks in the forwards; the Hessian against central differences in the
    parameters with vol_scaler pinned, within the gap the CPU oracle measures per chain (the derivative of the adaptive mesh choice)"""
    from test_hawkes_hessian_oracle import HAWKES_HESSIAN_ADAPTIVE_GAP
    from stochvolmodels_b200 import HawkesJDPricer, OptionChain, engine
    params, chain = _btc() if chain_name == "btc" else _case(which)[1:]
    pricer = HawkesJDPricer()
    vs = float(np.clip(params.sigma, 0.2, 0.5) * np.sqrt(min(np.min(chain.ttms), 1.0 / 12.0)))
    res = pricer.price_chain_hessian(chain, params, is_spot_measure=spot, vol_scaler=vs)
    greeks_of = lambda c, q: pricer.price_chain_greeks(c, q, is_spot_measure=spot, vol_scaler=vs)
    names, M = engine.HAWKES_GREEK_PARAMS, len(chain.ttms)
    for m in range(M):
        hf = 1e-5 * chain.forwards[m]
        bumped = []
        for s in (1, -1):
            fw = chain.forwards.copy()
            fw[m] += s * hf
            bumped.append(greeks_of(OptionChain(ttms=chain.ttms, forwards=fw, strikes_ttms=chain.strikes_ttms,
                                                optiontypes_ttms=chain.optiontypes_ttms, discfactors=chain.discfactors), params))
        for p in names:
            cd = (bumped[0].params[p][m] - bumped[1].params[p][m]) / (2 * hf)
            assert np.max(np.abs(res.vanna[p][m] - cd)) <= 1e-6 * max(1.0, np.max(np.abs(cd))), ("vanna", p, m)
    for q in names:
        v = getattr(params, q)
        h = 1e-6 * max(1.0, abs(v))
        up, dn = greeks_of(chain, dataclasses.replace(params, **{q: v + h})), greeks_of(chain, dataclasses.replace(params, **{q: v - h}))
        for p in names:
            for m in range(M):
                cd = (up.params[p][m] - dn.params[p][m]) / (2 * h)
                gap = HAWKES_HESSIAN_ADAPTIVE_GAP[chain_name] * max(1.0, np.max(np.abs(cd)))
                assert np.max(np.abs(res.hessian[p][q][m] - cd)) <= gap, ("hessian", p, q, m)


def test_hawkes_hessian_empty_chain(cuda_lib):
    """a chain without strikes: no sums, the grids still come back and match a chain with strikes"""
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    p, _, chain = _case("dflt")
    pc = _params_c(**p)
    empty = [np.array([])] * 3
    res = engine.hawkesjd_price_chain_hessian(pc, chain.ttms, chain.forwards, chain.discfactors, empty, empty, return_grids=True)
    full = engine.hawkesjd_price_chain_hessian(pc, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                               return_grids=True)
    assert res[1].shape == (17, 0) and res[2].shape == (15, 0) and res[3].shape == (120, 0)
    np.testing.assert_array_equal(res[5], full[5])
    np.testing.assert_array_equal(res[6], full[6])
