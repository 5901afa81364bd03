"""GPU checks of ``HawkesJDPricer.price_chain_risk_premia_greeks`` and ``compute_chain_risk_premia_ivol_greeks`` (forward-mode Fourier
sensitivities under the risk kernel, DESIGN.md §4.12) against ``price_chain``, the numpy forward mode of oracle/hawkes_rp_greeks.py,
``price_chain_greeks`` at gamma = 0 and central differences of the public pricer, on both parameter sets of hawkes_fourier.npz at five
gammas and on the BTC chain."""
import numpy as np
import pytest

from oracle import hawkes_rp_greeks as R
from test_hawkes_risk_premia_greeks_oracle import ADAPTIVE_GAP, GAMMAS, _golden_case

pytestmark = pytest.mark.gpu


def _case(name):
    """(params dict, HawkesJDParams with the gamma, OptionChain, gamma) of 'dflt-<gamma>', 'alt-<gamma>' or 'btc'"""
    from stochvolmodels_b200 import HawkesJDParams, OptionChain, get_btc_test_chain_data
    which, gamma = ("dflt", 0.4) if name == "btc" else (name.split("|")[0], float(name.split("|")[1]))
    p, ttms, fw, df, K, T = _golden_case(which)
    chain = get_btc_test_chain_data() if name == "btc" else OptionChain(ttms=ttms, forwards=fw, strikes_ttms=K, optiontypes_ttms=T,
                                                                         discfactors=df)
    return p, HawkesJDParams(**p, risk_premia_gamma=gamma), chain, gamma


CASES = [f"{w}|{g}" for w in ("dflt", "alt") for g in GAMMAS] + ["btc"]


def _rel_close(got, ref, rtol, what, floor=1e-300):
    scale = max(float(np.max(np.abs(ref))), floor)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err <= rtol, (what, err)


def _args(p, chain):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    return (_params_c(**p), chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)


@pytest.mark.parametrize("case", CASES)
def test_risk_premia_greeks_vs_price_chain_and_oracle(cuda_lib, case):
    from stochvolmodels_b200 import HawkesJDPricer, engine
    p, params, chain, gamma = _case(case)
    pc, *chain_args = _args(p, chain)
    prices, greeks, offsets, dlm, dnorm, nfev = engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *chain_args, return_grids=True)
    again = engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *chain_args, return_grids=True)
    ref = HawkesJDPricer().price_chain(chain, params)
    public = HawkesJDPricer().price_chain_risk_premia_greeks(chain, params)
    M = len(chain.ttms)
    for m in range(M):
        np.testing.assert_array_equal(prices[m], ref[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
        np.testing.assert_array_equal(public.prices[m], prices[m])
    for a, b in zip(again[1:], (greeks, offsets, dlm, dnorm, nfev)):
        np.testing.assert_array_equal(a, b)
    out, grids = R.hawkes_rp_chain_greeks(p, gamma, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    np.testing.assert_array_equal(nfev, grids["nfev"])           # the same mesh at every grid point
    # At phi = -1 (a normaliser point when gamma = 0 or 1) the log-MGF vanishes (the martingale condition), A is rounding noise and the step
    # control acts on it, so the GPU's mesh there may differ from numpy's: those rows agree to the solver's truncation error (measured
    # 8.1e-8 relative to max(1, |ref|), alt at gamma = 0 and 1); every other case to <= 7.4e-13.
    tol = 1e-6 if gamma in (0.0, 1.0) else 1e-10
    for d, name in enumerate(R.RP_NAMES):
        for m in range(M):
            _rel_close(dlm[d, m], grids["dlog_mgf"][d, m], 1e-10, (case, "dlog_mgf", name, m))
            _rel_close(dnorm[d, m], grids["dlog_norm"][d, m], tol, (case, "dlog_norm", name, m), floor=1.0)
    for m in range(M):
        sl = slice(offsets[m], offsets[m + 1])
        for r in range(18):
            _rel_close(greeks[r, sl], out[m][1 + r], tol, (case, "row", r, m), floor=1.0)
            np.testing.assert_array_equal(public.params[R.RP_NAMES[r - 2]][m] if r >= 2 else (public.delta, public.gamma)[r][m], greeks[r, sl])


@pytest.mark.parametrize("case", ["dflt|0.4", "alt|-1.0", "btc"])
def test_gamma_and_sigma_rows_vs_central_differences_of_the_public_pricer(cuda_lib, case):
    """with vol_scaler pinned, the gamma and sigma rows against central differences of price_chain: within the mesh-choice gap of the
    adaptive solver (ADAPTIVE_GAP, measured on the oracle)"""
    import dataclasses
    from stochvolmodels_b200 import HawkesJDPricer
    p, params, chain, gamma = _case(case)
    vs = 0.1
    pricer = HawkesJDPricer()
    g = pricer.price_chain_risk_premia_greeks(chain, params, vol_scaler=vs)
    for name in ("risk_premia_gamma", "sigma"):
        h = 1e-6 * max(1.0, abs(getattr(params, name)))
        up = pricer.price_chain(chain, dataclasses.replace(params, **{name: getattr(params, name) + h}), vol_scaler=vs)
        dn = pricer.price_chain(chain, dataclasses.replace(params, **{name: getattr(params, name) - h}), vol_scaler=vs)
        for m in range(len(chain.ttms)):
            cd = (up[m] - dn[m]) / (2 * h)
            assert np.max(np.abs(g.params[name][m] - cd)) <= ADAPTIVE_GAP * max(1.0, np.max(np.abs(cd))), (case, name, m)


@pytest.mark.parametrize("which", ["dflt", "alt"])
def test_gamma_zero_parameter_rows_match_price_chain_greeks(cuda_lib, which):
    """at gamma = 0 with discount factors 1 the risk-kernel pricer is the plain one up to the normalisers, which vanish to solver accuracy
    (L(0) = 0 exactly, L(-1) = 0 to rounding): the 15 parameter rows, delta and gamma agree (measured on the oracle: <= 4e-15 relative)"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain
    p, ttms, fw, df, K, T = _golden_case(which)
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=K, optiontypes_ttms=T, discfactors=np.ones(3))
    rp = HawkesJDPricer().price_chain_risk_premia_greeks(chain, HawkesJDParams(**p, risk_premia_gamma=0.0))
    plain = HawkesJDPricer().price_chain_greeks(chain, HawkesJDParams(**p))
    for m in range(3):
        _rel_close(rp.prices[m], plain.prices[m], 1e-12, ("price", m))
        _rel_close(rp.delta[m], plain.delta[m], 1e-12, ("delta", m))
        _rel_close(rp.gamma[m], plain.gamma[m], 1e-10, ("gamma", m))
        for name in plain.params:
            _rel_close(rp.params[name][m], plain.params[name][m], 1e-10, (name, m))


def test_empty_chain_and_launch_count(cuda_lib):
    """pricing launches as b200sv_hawkesjd_price_chain with a gamma (normalisers, Riccati, sums), then the normaliser and grid tangent
    launches and one sum launch; an empty chain skips both sum launches"""
    from stochvolmodels_b200 import engine
    lib = cuda_lib
    p, _, chain, gamma = _case("dflt|0.4")
    pc, *chain_args = _args(p, chain)
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chain(pc, *chain_args, True, None, 500, gamma)
    assert lib.b200sv_launch_count() == 3
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *chain_args)
    assert lib.b200sv_launch_count() == 3 + 3
    empty = (chain.ttms, chain.forwards, chain.discfactors, [np.array([])] * 3, [np.array([])] * 3)
    lib.b200sv_reset_launch_count()
    prices, greeks, offsets, dlm, dnorm, nfev = engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *empty, return_grids=True)
    assert lib.b200sv_launch_count() == 2 + 2
    assert greeks.shape == (18, 0) and all(x.size == 0 for x in prices) and list(offsets) == [0, 0, 0, 0]
    assert np.all(np.isfinite(dlm)) and np.all(np.isfinite(dnorm)) and np.all(nfev > 0)


@pytest.mark.parametrize("case", ["dflt|0.4", "alt|-1.0", "btc"])
def test_risk_premia_ivol_greeks(cuda_lib, case):
    """ivols bit-identical to compute_chain_prices_with_vols, the first 15 rows bit-identical to one 15-row transform of the same prices,
    and d ivol / d gamma against central differences of the ivols (vol_scaler pinned; within the mesh-choice gap, scaled by the ivol)"""
    import dataclasses
    from stochvolmodels_b200 import HawkesJDPricer, engine
    p, params, chain, gamma = _case(case)
    vs = 0.1
    pricer = HawkesJDPricer()
    iv = pricer.compute_chain_risk_premia_ivol_greeks(chain, params, vol_scaler=vs)
    ivols = pricer.compute_chain_prices_with_vols(chain, params, vol_scaler=vs)[1]
    g = pricer.price_chain_risk_premia_greeks(chain, params, vol_scaler=vs)
    flat = lambda rows: np.concatenate([np.asarray(r, dtype=np.float64).ravel() for r in rows])
    rows = np.vstack([flat(g.delta), flat(g.gamma), *(flat(g.params[n]) for n in engine.HAWKES_GREEK_PARAMS)])
    _, ref, _, _ = engine.bsm_implied_vol_sensitivities(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                        chain.optiontypes_ttms, g.prices, rows)
    assert tuple(iv.params) == R.RP_NAMES
    for m in range(len(chain.ttms)):
        np.testing.assert_array_equal(iv.ivols[m], ivols[m])
    np.testing.assert_array_equal(flat(iv.delta), ref[0])
    np.testing.assert_array_equal(flat(iv.gamma), ref[1])
    for k, name in enumerate(engine.HAWKES_GREEK_PARAMS):
        np.testing.assert_array_equal(flat(iv.params[name]), ref[2 + k])
    h = 1e-6 * max(1.0, abs(gamma))
    up = pricer.compute_chain_prices_with_vols(chain, dataclasses.replace(params, risk_premia_gamma=gamma + h), vol_scaler=vs)[1]
    dn = pricer.compute_chain_prices_with_vols(chain, dataclasses.replace(params, risk_premia_gamma=gamma - h), vol_scaler=vs)[1]
    for m in range(len(chain.ttms)):
        cd = (up[m] - dn[m]) / (2 * h)
        ok = np.isfinite(cd) & np.isfinite(iv.params["risk_premia_gamma"][m])
        if ok.any():
            assert np.max(np.abs(iv.params["risk_premia_gamma"][m][ok] - cd[ok])) <= 1e-3 * max(1.0, np.max(np.abs(cd[ok]))), (case, m)
