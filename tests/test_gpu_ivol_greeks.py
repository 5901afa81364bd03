"""GPU checks of the implied-vol sensitivities (b200sv_bsm_implied_vol_sensitivities, ModelPricer.compute_chain_ivol_greeks /
compute_chain_ivol_hessian; DESIGN.md §4.6) and of the exact-gradient calibration mode built on them."""
import dataclasses

import numpy as np
import pytest

import ivol_greeks_oracle as og
from conftest import load_golden

pytestmark = pytest.mark.gpu

Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)


def _flat(rows):
    return np.concatenate([np.asarray(r, dtype=float).ravel() for r in rows])


def _quickstart():
    from stochvolmodels_b200 import OptionChain
    g = load_golden("logsv_fourier_g1_quickstart.npz")
    M = int(g["nslices"])
    return OptionChain(ttms=g["ttms"], forwards=g["forwards"], discfactors=g["discfactors"], strikes_ttms=[g[f"strikes_{m}"] for m in range(M)],
                       optiontypes_ttms=[g[f"types_{m}"] for m in range(M)]), tuple(g["params"])


def _hawkes(which="alt"):
    from stochvolmodels_b200 import HawkesJDParams, OptionChain
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    chain = OptionChain(ttms=g["ttms"], forwards=g["forwards"], strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["types"]] * 3,
                        discfactors=g["discfactors"])
    return chain, HawkesJDParams(**p)


def _cases():
    """(name, pricer, chain, params, kwargs, central-difference gap of the price rows measured on the CPU oracle)"""
    from test_fourier_greeks_oracle import ADAPTIVE_GAP
    from test_hawkes_greeks_oracle import ADAPTIVE_GAP as HAWKES_GAP
    from stochvolmodels_b200 import (LOGSV_BTC_PARAMS, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer,
                                     get_btc_test_chain_data)
    qs_chain, qs = _quickstart()
    btc = get_btc_test_chain_data()
    hk_chain, hk = _hawkes()
    return {"logsv_quickstart": (LogSVPricer(), qs_chain, LogSvParams(*qs), {}, ADAPTIVE_GAP["quickstart"]),
            "logsv_btc_spot": (LogSVPricer(), btc, LOGSV_BTC_PARAMS, {"is_spot_measure": True}, ADAPTIVE_GAP["btc"]),
            "logsv_btc_inverse": (LogSVPricer(), btc, LOGSV_BTC_PARAMS, {"is_spot_measure": False}, ADAPTIVE_GAP["btc"]),
            "heston": (HestonPricer(), qs_chain, HestonParams(v0=0.8, theta=1.0, kappa=2.0, rho=-0.3, volvol=1.5), {}, 1e-7),
            "hawkes": (HawkesJDPricer(), hk_chain, hk, {}, HAWKES_GAP)}


CASES = list(_cases())


@pytest.mark.parametrize("case", CASES)
def test_ivols_bitwise_and_rows_vs_oracle(cuda_lib, case):
    """ivols equal compute_chain_prices_with_vols bit for bit (two calls too); every first- and second-order row equals the numpy
    transform of the GPU's own price rows and ivols to 1e-12 of the size of its terms"""
    pricer, chain, params, kw, _ = _cases()[case]
    _, ref = pricer.compute_chain_prices_with_vols(chain, params, **kw)
    first = pricer.compute_chain_ivol_greeks(chain, params, **kw)
    again = pricer.compute_chain_ivol_greeks(chain, params, **kw)
    second = pricer.compute_chain_ivol_hessian(chain, params, **kw)
    for m in range(len(chain.ttms)):
        np.testing.assert_array_equal(first.ivols[m], ref[m])
        np.testing.assert_array_equal(again.ivols[m], ref[m])
        np.testing.assert_array_equal(second.ivols[m], ref[m])
    for name in first.params:
        np.testing.assert_array_equal(_flat(again.params[name]), _flat(first.params[name]))
    # the oracle on the GPU's own inputs
    ph = pricer.price_chain_hessian(chain, params, **kw)
    names = list(ph.params)
    F = np.concatenate([np.full(len(k), f) for k, f in zip(chain.strikes_ttms, chain.forwards)])
    T = np.concatenate([np.full(len(k), t) for k, t in zip(chain.strikes_ttms, chain.ttms)])
    D = np.concatenate([np.full(len(k), d) for k, d in zip(chain.strikes_ttms, chain.discfactors)])
    K, is_call = _flat(chain.strikes_ttms), og.is_call_type(np.concatenate(chain.optiontypes_ttms))
    greeks = np.vstack([_flat(ph.delta), _flat(ph.gamma), *(_flat(ph.params[n]) for n in names)])
    vanna = np.vstack([_flat(ph.vanna[n]) for n in names])
    hessian = np.vstack([_flat(ph.hessian[p][q]) for i, p in enumerate(names) for q in names[i:]])
    vol = _flat(second.ivols)
    g, v, h = og.ivol_sensitivities(F, K, T, D, vol, is_call, greeks, vanna, hessian)
    vega, dF, dFF, dFv, dvv = og.black_partials(F, K, T, D, vol, is_call)
    sF = g[0]
    # size of the terms each row is formed from, over vega: the relative rounding of any two restatements of the same arithmetic
    terms_g = np.vstack([np.abs(greeks[0]) + np.abs(dF), np.abs(greeks[1]) + np.abs(dFF) + 2 * np.abs(dFv * sF) + np.abs(dvv) * sF ** 2,
                         np.abs(greeks[2:])]) / vega
    terms_v = (np.abs(vanna) + (np.abs(dFv) + np.abs(dvv * sF)) * np.abs(g[2:])) / vega
    idx = [(a, c) for a in range(len(names)) for c in range(a, len(names))]
    terms_h = (np.abs(hessian) + np.abs(dvv) * np.vstack([np.abs(g[2 + a] * g[2 + c]) for a, c in idx])) / vega
    got_g = np.vstack([_flat(second.delta), _flat(second.gamma), *(_flat(second.params[n]) for n in names)])
    got_v = np.vstack([_flat(second.vanna[n]) for n in names])
    got_h = np.vstack([_flat(second.hessian[p][q]) for p, q in ((names[a], names[c]) for a, c in idx)])
    for got, want, terms, what in ((got_g, g, terms_g, "greeks"), (got_v, v, terms_v, "vanna"), (got_h, h, terms_h, "hessian")):
        ok = np.isfinite(want)
        np.testing.assert_array_equal(np.isfinite(got), ok, err_msg=what)
        assert np.all(np.abs(got[ok] - want[ok]) <= 1e-12 * (np.abs(want[ok]) + terms[ok])), what
    for name in names:                                  # first order of the Hessian call = first order of the greeks call
        np.testing.assert_allclose(_flat(second.params[name]), _flat(first.params[name]), rtol=1e-14, atol=0)


@pytest.mark.parametrize("case", ["logsv_quickstart", "logsv_btc_spot", "heston", "hawkes"])
def test_rows_vs_central_differences_of_the_public_vols(cuda_lib, case):
    """d ivol / d parameter against central differences of compute_chain_prices_with_vols with the grid pinned, and d ivol / d forward
    against differences in the forwards.  The bound is the CPU-measured gap of the price rows to the adaptive pricer
    (ADAPTIVE_GAP of the oracle tests, relative to max(1, |cd price|)) divided by each quote's vega, plus the inversion's own rounding
    over the step."""
    from stochvolmodels_b200 import OptionChain
    pricer, chain, params, kw, gap = _cases()[case]
    vs = {"logsv": lambda: float(params.sigma0 * np.sqrt(min(np.min(chain.ttms), 0.5 / 12.0))),
          "heston": lambda: float(min(0.3, np.sqrt(params.v0 * chain.ttms[0]))),
          "hawkes": lambda: float(np.clip(params.sigma, 0.2, 0.5) * np.sqrt(min(np.min(chain.ttms), 1.0 / 12.0)))}[case.split("_")[0]]()
    sens = pricer.compute_chain_ivol_greeks(chain, params, vol_scaler=vs, **kw)
    vols = lambda c, p=params: pricer.compute_chain_prices_with_vols(c, p, vol_scaler=vs, **kw)
    F = np.concatenate([np.full(len(k), f) for k, f in zip(chain.strikes_ttms, chain.forwards)])
    T = np.concatenate([np.full(len(k), t) for k, t in zip(chain.strikes_ttms, chain.ttms)])
    D = np.concatenate([np.full(len(k), d) for k, d in zip(chain.strikes_ttms, chain.discfactors)])
    K, is_call = _flat(chain.strikes_ttms), og.is_call_type(np.concatenate(chain.optiontypes_ttms))
    vega = og.black_partials(F, K, T, D, _flat(sens.ivols), is_call)[0]
    for name in sens.params:
        value = getattr(params, name)
        h = 1e-6 * max(1.0, abs(value)) if case == "hawkes" else 1e-5        # the steps the price rows' gap was measured with
        up_p, up_v = vols(chain, dataclasses.replace(params, **{name: value + h}))
        dn_p, dn_v = vols(chain, dataclasses.replace(params, **{name: value - h}))
        cd_p = (_flat(up_p) - _flat(dn_p)) / (2 * h)
        cd_v = (_flat(up_v) - _flat(dn_v)) / (2 * h)
        bound = (gap * max(1.0, np.max(np.abs(cd_p))) + 8e-16 * (F + K) / h) / vega
        err = np.abs(_flat(sens.params[name]) - cd_v)
        assert np.all(err <= bound), (name, float(np.max(err / bound)))
    hr = 1e-4
    for m in range(len(chain.ttms)):
        def bumped(f):
            fw = chain.forwards.copy()
            fw[m] *= f
            c = OptionChain(ttms=chain.ttms, forwards=fw, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                            discfactors=chain.discfactors)
            return [np.asarray(a[m]) for a in vols(c)]
        p_all, v_all = vols(chain)
        (p0, v0), (pp, vp), (pm, vm) = (p_all[m], v_all[m]), bumped(1 + hr), bumped(1 - hr)
        hh = hr * chain.forwards[m]
        sl = slice(sum(len(k) for k in chain.strikes_ttms[:m]), sum(len(k) for k in chain.strikes_ttms[:m + 1]))
        # the price route's own check: delta to 1e-7, gamma to 2e-4 max(1, |gamma cd|); here over vega, plus the inversion's rounding
        d_bound = (1e-7 + 8e-16 * (F[sl] + K[sl]) / hh) / vega[sl] + 1e-9 * np.abs(sens.delta[m])
        np.testing.assert_array_less(np.abs(sens.delta[m] - (vp - vm) / (2 * hh)), d_bound)
        g_cd_p = (pp - 2 * p0 + pm) / (hh * hh)
        g_bound = (2e-4 * max(1.0, np.max(np.abs(g_cd_p))) + 8e-16 * (F[sl] + K[sl]) / hh ** 2) / vega[sl]
        np.testing.assert_array_less(np.abs(sens.gamma[m] - (vp - 2 * v0 + vm) / (hh * hh)), g_bound)


# ---- the C entry point on constructed inputs ---------------------------------------------------------------------------------------
def _black_in_chain(n):
    """one slice of the Black-in model (tests/ivol_greeks_oracle.py): every type near the money, out-of-the-money types to |d1| = 8"""
    from test_ivol_greeks_oracle import _case
    c = _case(n)
    price, greeks, vanna, hessian, want = og.black_in_model(c["F"], c["K"], c["T"], c["D"], c["types"], c["p"], c["F0"], *c["model"])
    return c, price, greeks, vanna, hessian, want


@pytest.mark.parametrize("n", [5, 6, 15])
@pytest.mark.parametrize("second", [False, True])
def test_black_in_black_out_through_the_entry_point(cuda_lib, n, second):
    from stochvolmodels_b200 import engine
    c, price, greeks, vanna, hessian, want = _black_in_chain(n)
    chain = (np.array([c["T"]]), np.array([c["F"]]), np.array([c["D"]]), [c["K"]], [c["types"]])
    ivols, g, v, h = engine.bsm_implied_vol_sensitivities(*chain, [price], greeks, vanna if second else None, hessian if second else None)
    np.testing.assert_array_equal(ivols[0], np.concatenate(engine.bsm_implied_vols(*chain, [price])))
    np.testing.assert_allclose(ivols[0], want["ivol"], rtol=1e-10)
    pairs = [(g, want["greeks"], "greeks")] + ([(v, want["vanna"], "vanna"), (h, want["hessian"], "hessian")] if second else [])
    if not second:
        assert v is None and h is None
    for got, exp, what in pairs:
        scale = np.max(np.abs(exp), axis=1, keepdims=True)
        np.testing.assert_array_less(np.abs(got - exp), 1e-10 * np.maximum(np.abs(exp), 1e-3 * scale) + 1e-300, err_msg=what)


def test_entry_point_conventions_nan_and_bracket_ends(cuda_lib):
    """a NaN price gives NaN rows; a price above Black(vol = 10) or below Black(vol = 1e-8) gives zero rows (T = 0.01, F = 1: Black(10) of
    the at-the-money call is 0.383 D, Black(1e-8) about 4e-10 D)"""
    from oracle import bsm as obsm
    from stochvolmodels_b200 import engine
    T, F, D = 0.01, 1.0, 0.98
    K = np.array([1.0, 1.0, 1.0, 1.1, 0.9])
    types = np.array(["C", "IC", "C", "C", "P"])
    prices = np.array([np.nan, 0.5 * D, 1e-13 * D, *obsm.compute_bsm_vanilla_price(F, K[3:], T, 0.3, types[3:], D)])
    n = 6
    rng = np.random.RandomState(2)
    greeks, vanna, hessian = rng.rand(2 + n, 5), rng.rand(n, 5), rng.rand(n * (n + 1) // 2, 5)
    ivols, g, v, h = engine.bsm_implied_vol_sensitivities(np.array([T]), np.array([F]), np.array([D]), [K], [types], [prices], greeks, vanna,
                                                          hessian)
    iv = ivols[0]
    assert np.isnan(iv[0]) and np.isnan(g[:, 0]).all() and np.isnan(v[:, 0]).all() and np.isnan(h[:, 0]).all()
    assert iv[1] == pytest.approx(10.0, rel=1e-12) and iv[2] == pytest.approx(1e-8, rel=1e-12)
    for rows in (g, v, h):
        assert (rows[:, 1:3] == 0.0).all() and np.isfinite(rows[:, 3:]).all() and (rows[:, 3:] != 0.0).all()
    np.testing.assert_allclose(iv[3:], 0.3, rtol=1e-6)


# ---- exact-gradient calibration ----------------------------------------------------------------------------------------------------------
def _exact_and_difference_at_start(pricer, chain, fields, codec_jacobian, x0, batch_ivols, names, vol_scaler, kw, weights, market, gap):
    """fun of both modes at the start point (bit for bit) and the exact jac against a central difference of the exact objective, within
    the CPU-derived bound sum_j 2 w_j |r_j| sum_f |D_fi| gap max(1, |P_f|) / vega_j + truncation"""
    from stochvolmodels_b200.pricers.calibration import ExactGradientObjective, flat_ivol_rows
    obj = ExactGradientObjective(lambda x: flat_ivol_rows(pricer.compute_chain_ivol_greeks(chain, fields(x), vol_scaler=vol_scaler, **kw), names),
                                 codec_jacobian, market, weights)
    diff_vols = batch_ivols(x0[None, :])[0]
    assert obj.fun(x0) == float(np.nansum(weights * np.square(diff_vols - market)))
    jac = obj.jac(x0)
    pg = pricer.price_chain_greeks(chain, fields(x0), vol_scaler=vol_scaler, **kw)
    F = np.concatenate([np.full(len(k), f) for k, f in zip(chain.strikes_ttms, chain.forwards)])
    T = np.concatenate([np.full(len(k), t) for k, t in zip(chain.strikes_ttms, chain.ttms)])
    Dd = np.concatenate([np.full(len(k), d) for k, d in zip(chain.strikes_ttms, chain.discfactors)])
    vols = flat_ivol_rows(pricer.compute_chain_ivol_greeks(chain, fields(x0), vol_scaler=vol_scaler, **kw), names)[0]
    ok = np.isfinite(vols)
    vega = og.black_partials(F, _flat(chain.strikes_ttms), T, Dd, vols, og.is_call_type(np.concatenate(chain.optiontypes_ttms)))[0]
    per_field = np.array([gap * max(1.0, np.max(np.abs(_flat(pg.params[n])))) for n in names])
    weight = np.sum(2 * weights[ok] * np.abs(vols[ok] - market[ok]) / vega[ok])
    Dm = np.abs(codec_jacobian(x0))
    for i in range(x0.size):
        hstep = 1e-5 * max(1.0, abs(x0[i]))
        e = np.eye(x0.size)[i] * hstep
        fresh = lambda y: ExactGradientObjective(obj.ivol_greeks, codec_jacobian, market, weights).fun(y)
        cd = (fresh(x0 + e) - fresh(x0 - e)) / (2 * hstep)
        bound = weight * (Dm[:, i] @ per_field) + 1e-6 * abs(cd) + 1e-12
        assert abs(jac[i] - cd) <= bound, (i, jac[i], cd, bound)


def test_logsv_params4_exact_calibration_vs_reference_driver(cuda_lib):
    from test_gpu_calibration import _chain, _objective
    from test_fourier_greeks_oracle import ADAPTIVE_GAP
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, LogsvModelCalibrationType, engine
    from stochvolmodels_b200.pricers.calibration import LogSvParameterCodec, calibration_weights
    from stochvolmodels_b200.pricers.logsv_pricer import _params_c
    g = load_golden("calib_logsv_params4.npz")
    chain, pricer = _chain(g), LogSVPricer()
    market = g["market_vols"].ravel()
    f_ref = _objective(chain, g["fit_vols"].ravel(), market)
    start = LogSvParams(*g["start"])
    lo, hi = LogSvParams(sigma0=0.1, theta=0.1, kappa1=0.25, kappa2=0.25, beta=-3.0, volvol=0.2), LogSvParams(1.5, 1.5, 10.0, 10.0, 3.0, 3.0)
    codec = LogSvParameterCodec(start, lo, hi, LogsvModelCalibrationType.PARAMS4)
    x0 = codec.initial_and_bounds()[0]
    vs = pricer.set_vol_scaler(chain)
    weights = calibration_weights(chain, market, True, False)
    batch = lambda pts: engine.logsv_price_chain_batch([_params_c(codec.parse(p)) for p in pts], chain.ttms, chain.forwards, chain.discfactors,
                                                       None, chain.strikes_ttms, chain.optiontypes_ttms, vol_scaler=vs)[1]
    _exact_and_difference_at_start(pricer, chain, codec.parse, codec.field_jacobian, x0, batch, engine.LOGSV_GREEK_PARAMS, vs, {}, weights,
                                   market, ADAPTIVE_GAP["btc"])
    fit, info = pricer.calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS4,
                                                       return_info=True, gradient="exact")
    assert set(info) == {"fun", "nit", "nb_batches", "x", "nan_quotes"}
    assert info["fun"] == pytest.approx(f_ref, rel=1e-3)
    np.testing.assert_allclose([fit.sigma0, fit.theta, fit.kappa1, fit.kappa2, fit.beta, fit.volvol], g["fit"], atol=2e-2)


def test_heston_exact_calibration_vs_reference_driver(cuda_lib):
    from test_gpu_calibration import _chain, _objective
    from stochvolmodels_b200 import HestonParams, HestonPricer, engine
    from stochvolmodels_b200.pricers.calibration import calibration_weights, heston_default_vol_scaler
    g = load_golden("calib_heston.npz")
    chain, pricer = _chain(g), HestonPricer()
    market = g["market_vols"].ravel()
    f_ref = _objective(chain, g["fit_vols"].ravel(), market)
    x0 = np.asarray(g["start"], dtype=float)
    vs = heston_default_vol_scaler(x0[0], float(chain.ttms[0]))
    weights = calibration_weights(chain, market, True, False)
    batch = lambda pts: engine.heston_price_chain_batch([engine.heston_params_c(*p) for p in pts], chain.ttms, chain.forwards, chain.discfactors,
                                                        chain.strikes_ttms, chain.optiontypes_ttms)[1]
    _exact_and_difference_at_start(pricer, chain, lambda x: HestonParams(*x), lambda x: np.eye(5), x0, batch, engine.HESTON_GREEK_PARAMS, vs,
                                   {}, weights, market, 1e-7)
    fit, info = pricer.calibrate_model_params_to_chain(chain, HestonParams(*g["start"]), return_info=True, gradient="exact")
    assert info["fun"] <= 1.5 * f_ref + 1e-9
    assert 2.0 * fit.kappa * fit.theta - fit.volvol ** 2 >= -1e-8


def test_hawkes_exact_calibration_no_worse_than_the_difference_route(cuda_lib):
    """a chain generated from known parameters plus fixed vol noise; both modes from the same start.  sigma stays above 0.5, where the
    default grid clip(sigma, 0.2, 0.5) sqrt(min(T0, 1/12)) no longer moves, so the difference route's per-set grids and the exact route's
    pinned one are the same grid and both minimise the same objective.  SLSQP stops once a step changes the objective by less than
    ftol = 1e-8, so two converged runs can differ by that much."""
    from test_hawkes_greeks_oracle import ADAPTIVE_GAP
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c, hawkes_fit_jacobian, set_vol_scaler
    base, _ = _hawkes("dflt")
    unpack = lambda x: HawkesJDParams(mu=0.0, sigma=x[0], shift_p=0.06, mean_p=x[1], shift_m=-0.06, mean_m=x[2], lambda_p=6.55, theta_p=x[3],
                                      kappa_p=x[5], beta1_p=x[6], beta2_p=-x[6], lambda_m=8.5, theta_m=x[4], kappa_m=x[5], beta1_m=x[7],
                                      beta2_m=-x[7])
    truth = unpack(np.array([0.7, 0.03, -0.03, 6.55, 8.5, 25.0, 70.0, 100.0]))
    pricer = HawkesJDPricer()
    strikes = [np.linspace(0.8, 1.2, 9) * f for f in base.forwards]
    types = [np.where(k >= f, "C", "P") for k, f in zip(strikes, base.forwards)]
    grid = OptionChain(ttms=base.ttms, forwards=base.forwards, discfactors=base.discfactors, strikes_ttms=strikes, optiontypes_ttms=types)
    vols = pricer.compute_model_ivols_for_chain(grid, truth)
    rng = np.random.RandomState(4)
    noisy = [v + rng.uniform(-2e-3, 2e-3, v.size) for v in vols]
    chain = OptionChain(ttms=base.ttms, forwards=base.forwards, discfactors=base.discfactors, strikes_ttms=strikes, optiontypes_ttms=types,
                        ids=np.array(["a", "b", "c"]), bid_ivs=noisy, ask_ivs=[v.copy() for v in noisy])
    start = unpack(np.array([0.8, 0.05, -0.05, 8.0, 7.0, 30.0, 60.0, 90.0]))
    x0 = np.array([start.sigma, start.mean_p, start.mean_m, start.theta_p, start.theta_m, 0.5 * (start.kappa_p + start.kappa_m),
                   0.5 * (start.beta1_p - start.beta2_p), 0.5 * (start.beta2_p - start.beta2_m)])
    market = _flat(noisy)
    weights = np.concatenate([v / np.sum(v) for v in chain.get_chain_vegas()])
    vs = set_vol_scaler(start.sigma, float(chain.ttms[0]))
    batch = lambda pts: engine.hawkesjd_price_chain_batch([_params_c(**{k: v for k, v in unpack(p).to_dict().items()}) for p in pts],
                                                          chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                          chain.optiontypes_ttms)[1]
    D = hawkes_fit_jacobian()
    _exact_and_difference_at_start(pricer, chain, unpack, lambda x: D, x0, batch, engine.HAWKES_GREEK_PARAMS, vs, {}, weights, market,
                                   ADAPTIVE_GAP)
    _, diff = pricer.calibrate_model_params_to_chain(chain, start, return_info=True)
    fit, exact = pricer.calibrate_model_params_to_chain(chain, start, return_info=True, gradient="exact")
    assert exact["fun"] <= diff["fun"] + 1e-8, (exact["fun"], diff["fun"])
    assert min(fit.sigma, exact["x"][0], diff["x"][0]) > 0.5
    assert exact["nb_batches"] == 2 * (exact["nb_batches"] // 2)


def test_btc_params5_exact_calibration_vs_difference_route(cuda_lib):
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS as ref, LogSvParams, LogSVPricer, LogsvModelCalibrationType, get_btc_test_chain_data
    chain, pricer = get_btc_test_chain_data(), LogSVPricer()
    start = LogSvParams(sigma0=0.7, theta=0.9, kappa1=ref.kappa1, kappa2=None, beta=0.0, volvol=1.4)
    _, diff = pricer.calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS5, return_info=True)
    _, exact = pricer.calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS5, return_info=True,
                                                      gradient="exact")
    assert exact["fun"] <= diff["fun"] * (1 + 1e-3), (exact["fun"], diff["fun"])
