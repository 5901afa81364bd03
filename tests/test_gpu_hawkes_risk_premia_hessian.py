"""GPU checks of ``HawkesJDPricer.price_chain_risk_premia_hessian`` and ``compute_chain_risk_premia_ivol_hessian`` (second-order Fourier
sensitivities under the risk kernel, DESIGN.md §4.13) against ``price_chain_risk_premia_greeks``, the numpy forward-over-forward mode of
tests/hawkes_rp_hessian_oracle.py, ``price_chain_hessian`` at gamma = 0 and central differences of the public first-order rows, on both
parameter sets of hawkes_fourier.npz at five gammas and on the BTC chain."""
import numpy as np
import pytest

import hawkes_rp_hessian_oracle as RH
from test_gpu_hawkes_risk_premia_greeks import CASES, _args, _case, _rel_close
from test_hawkes_risk_premia_hessian_oracle import ADAPTIVE_GAP

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES)
def test_risk_premia_hessian_vs_greeks_and_oracle(cuda_lib, case):
    from stochvolmodels_b200 import HawkesJDPricer, engine
    p, params, chain, gamma = _case(case)
    pc, *chain_args = _args(p, chain)
    out = engine.hawkesjd_price_chain_risk_premia_hessian(pc, gamma, *chain_args, return_grids=True)
    prices, greeks, vanna, hessian, offsets, dlm, dnorm, nfev, d2lm, d2norm = out
    again = engine.hawkesjd_price_chain_risk_premia_hessian(pc, gamma, *chain_args, return_grids=True)
    first = engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *chain_args, return_grids=True)
    M = len(chain.ttms)
    for m in range(M):                                   # the first-order outputs bit for bit, and a repeated call equals itself
        np.testing.assert_array_equal(prices[m], first[0][m])
        np.testing.assert_array_equal(again[0][m], prices[m])
    for a, b in zip((greeks, offsets, dlm, dnorm, nfev), first[1:]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(again[1:], out[1:]):
        np.testing.assert_array_equal(a, b)
    public = HawkesJDPricer().price_chain_risk_premia_hessian(chain, params)
    names = RH.NAMES
    for m in range(M):
        sl = slice(offsets[m], offsets[m + 1])
        np.testing.assert_array_equal(public.prices[m], prices[m])
        for k, n in enumerate(names):
            np.testing.assert_array_equal(public.vanna[n][m], vanna[k, sl])
        for r, (i, j) in enumerate(RH.PAIRS):
            np.testing.assert_array_equal(public.hessian[names[i]][names[j]][m], hessian[r, sl])
    rows, grids = RH.hawkes_rp_chain_hessian(p, gamma, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                             chain.optiontypes_ttms)
    # as for the first-order rows: where a normaliser point sits at phi = -1 (gamma = 0 or 1) the log-MGF there is rounding noise and the
    # step control acts on it, so the rows that read the normaliser agree to the solver's truncation error (measured 1.9e-6, alt at
    # gamma = 0); every other case to <= 1.2e-11 (the BTC chain's Hessian rows), d2log_mgf to <= 4.5e-12
    tol = 1e-5 if gamma in (0.0, 1.0) else 1e-9
    for r in range(len(RH.PAIRS)):
        for m in range(M):
            _rel_close(d2lm[r, m], grids["d2log_mgf"][r, m], 1e-9, (case, "d2log_mgf", RH.PAIRS[r], m))
            _rel_close(d2norm[r, m], grids["d2log_norm"][r, m], tol, (case, "d2log_norm", RH.PAIRS[r], m), floor=1.0)
    for m in range(M):
        sl = slice(offsets[m], offsets[m + 1])
        for k in range(len(names)):
            _rel_close(vanna[k, sl], rows[m][1][k], tol, (case, "vanna", names[k], m), floor=1.0)
        for r in range(len(RH.PAIRS)):
            _rel_close(hessian[r, sl], rows[m][2][r], tol, (case, "hessian", RH.PAIRS[r], m), floor=1.0)


# the mesh-choice gap of these rows on the BTC chain (vol_scaler = 0.1), measured on the CPU oracle: 2.1e-3, the (sigma, kappa_m) entry of
# the second maturity; on the hawkes_fourier.npz cases here <= 5.9e-5, within ADAPTIVE_GAP
BTC_ADAPTIVE_GAP = 5e-3


@pytest.mark.parametrize("case", ["dflt|0.4", "alt|-1.0", "btc"])
def test_gamma_row_and_sigma_column_vs_central_differences_of_the_public_rows(cuda_lib, case):
    """with vol_scaler pinned, the gamma row and the sigma column of the Hessian against central differences of the public first-order
    rows (price_chain_risk_premia_greeks): within the mesh-choice gap of the adaptive solver, measured on the oracle"""
    import dataclasses
    from stochvolmodels_b200 import HawkesJDPricer
    p, params, chain, gamma = _case(case)
    vs = 0.1
    pricer = HawkesJDPricer()
    hs = pricer.price_chain_risk_premia_hessian(chain, params, vol_scaler=vs)
    for name in ("risk_premia_gamma", "sigma"):
        h = 1e-6 * max(1.0, abs(getattr(params, name)))
        up = pricer.price_chain_risk_premia_greeks(chain, dataclasses.replace(params, **{name: getattr(params, name) + h}), vol_scaler=vs)
        dn = pricer.price_chain_risk_premia_greeks(chain, dataclasses.replace(params, **{name: getattr(params, name) - h}), vol_scaler=vs)
        for other in RH.NAMES:
            for m in range(len(chain.ttms)):
                cd = (up.params[other][m] - dn.params[other][m]) / (2 * h)
                err = np.max(np.abs(hs.hessian[name][other][m] - cd)) / max(1.0, np.max(np.abs(cd)))
                assert err <= (BTC_ADAPTIVE_GAP if case == "btc" else ADAPTIVE_GAP), (case, name, other, m, err)


@pytest.mark.parametrize("which", ["dflt", "alt"])
def test_gamma_zero_matches_price_chain_hessian(cuda_lib, which):
    """at gamma = 0 with discount factors 1 the 15 x 15 block and the 15 vanna rows equal price_chain_hessian (measured: <= 2e-15
    relative to max(1, |plain|))"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain
    from test_hawkes_risk_premia_greeks_oracle import _golden_case
    p, ttms, fw, df, K, T = _golden_case(which)
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=K, optiontypes_ttms=T, discfactors=np.ones(3))
    rp = HawkesJDPricer().price_chain_risk_premia_hessian(chain, HawkesJDParams(**p, risk_premia_gamma=0.0))
    plain = HawkesJDPricer().price_chain_hessian(chain, HawkesJDParams(**p))
    for m in range(3):
        for a in plain.params:
            _rel_close(rp.vanna[a][m], plain.vanna[a][m], 1e-10, ("vanna", a, m), floor=1.0)
            for b in plain.params:
                _rel_close(rp.hessian[a][b][m], plain.hessian[a][b][m], 1e-10, ("hessian", a, b, m), floor=1.0)


def test_empty_chain_and_launch_count(cuda_lib):
    """the greeks call's launches, then the restarted and the carried Hessian launches and one sum launch; an empty chain skips both sum
    launches"""
    from stochvolmodels_b200 import engine
    lib = cuda_lib
    p, _, chain, gamma = _case("dflt|0.4")
    pc, *chain_args = _args(p, chain)
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *chain_args)
    greeks_launches = lib.b200sv_launch_count()
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chain_risk_premia_hessian(pc, gamma, *chain_args)
    assert lib.b200sv_launch_count() == greeks_launches + 3 == 9
    empty = (chain.ttms, chain.forwards, chain.discfactors, [np.array([])] * 3, [np.array([])] * 3)
    lib.b200sv_reset_launch_count()
    prices, greeks, vanna, hessian, offsets, dlm, dnorm, nfev, d2lm, d2norm = engine.hawkesjd_price_chain_risk_premia_hessian(
        pc, gamma, *empty, return_grids=True)
    assert lib.b200sv_launch_count() == 4 + 2
    assert greeks.shape == (18, 0) and vanna.shape == (16, 0) and hessian.shape == (136, 0) and list(offsets) == [0, 0, 0, 0]
    assert all(np.all(np.isfinite(x)) for x in (dlm, dnorm, d2lm, d2norm)) and np.all(nfev > 0)


@pytest.mark.parametrize("case", ["dflt|0.4", "alt|-1.0", "btc"])
def test_risk_premia_ivol_hessian(cuda_lib, case):
    """ivols bit-identical to compute_chain_prices_with_vols; the first 15 x 15 block, its vanna and first-order rows bit-identical to one
    15-row transform of the same prices; every entry finite where the ivol is"""
    from stochvolmodels_b200 import HawkesJDPricer, engine
    p, params, chain, gamma = _case(case)
    vs = 0.1
    pricer = HawkesJDPricer()
    iv = pricer.compute_chain_risk_premia_ivol_hessian(chain, params, vol_scaler=vs)
    ivols = pricer.compute_chain_prices_with_vols(chain, params, vol_scaler=vs)[1]
    h = pricer.price_chain_risk_premia_hessian(chain, params, vol_scaler=vs)
    flat = lambda rows: np.concatenate([np.asarray(r, dtype=np.float64).ravel() for r in rows])
    head = engine.HAWKES_GREEK_PARAMS
    rows = np.vstack([flat(h.delta), flat(h.gamma), *(flat(h.params[n]) for n in head)])
    _, g, v, hh = engine.bsm_implied_vol_sensitivities(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                       chain.optiontypes_ttms, h.prices, rows, np.vstack([flat(h.vanna[n]) for n in head]),
                                                       np.vstack([flat(h.hessian[a][b]) for i, a in enumerate(head) for b in head[i:]]))
    assert tuple(iv.params) == tuple(iv.vanna) == RH.NAMES
    for m in range(len(chain.ttms)):
        np.testing.assert_array_equal(iv.ivols[m], ivols[m])
    np.testing.assert_array_equal(flat(iv.delta), g[0])
    np.testing.assert_array_equal(flat(iv.gamma), g[1])
    r = 0
    for i, a in enumerate(head):
        np.testing.assert_array_equal(flat(iv.params[a]), g[2 + i])
        np.testing.assert_array_equal(flat(iv.vanna[a]), v[i])
        for b in head[i:]:
            np.testing.assert_array_equal(flat(iv.hessian[a][b]), hh[r])
            r += 1
    ok = np.isfinite(flat(iv.ivols))
    for a in RH.NAMES:
        assert np.all(np.isfinite(flat(iv.vanna[a])[ok])) and np.all(np.isfinite(flat(iv.hessian[a]["risk_premia_gamma"])[ok])), a
