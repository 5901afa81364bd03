"""CPU: the implied-vol sensitivity transform (tests/ivol_greeks_oracle.py, the numpy restatement of black_ivol_sensitivities_kernel),
the exact-gradient calibration objective on a numpy stand-in for the ivol-greeks call, and every rejection before a library call."""
import numpy as np
import pytest

import ivol_greeks_oracle as og
from oracle import bsm as obsm

TYPES = ("C", "P", "IC", "IP")
D1S = np.array([-8.0, -5.0, -2.0, -0.5, 0.0, 0.5, 2.0, 5.0, 8.0])


def _case(n, T=0.7, D=0.93, F0=100.0, F=103.0, seed=7):
    """every type for |d1| <= 2; beyond, the out-of-the-money types only (an in-the-money quote there is its intrinsic value to more
    digits than its vol carries)"""
    p, sigma0, a, b, Q, e = og.default_black_in(n, seed)
    g = og.black_in_vol(F, p, F0, sigma0, a, b, Q, e)[0]
    quotes = [(k, t) for d1, k in zip(D1S, og.strikes_for_d1(F, T, g, D1S))
              for t in (TYPES if abs(d1) <= 2 else ("C", "IC") if d1 < 0 else ("P", "IP"))]
    K, types = np.array([q[0] for q in quotes]), np.array([q[1] for q in quotes])
    return dict(F=F, K=K, T=T, D=D, types=types, p=p, F0=F0, model=(sigma0, a, b, Q, e))


def test_black_partials_vs_differences_of_the_black_price():
    """the closed-form partials against 4-point central differences of oracle/bsm.py's Black price (independent of the partials)"""
    F, T, D = 1.3, 0.4, 0.97
    for vol in (0.05, 0.3, 1.5):
        K = og.strikes_for_d1(F, T, vol, np.linspace(-4, 4, 9))
        for t in TYPES:
            is_call = og.is_call_type(np.full(K.shape, t))
            B = lambda f, v: obsm.compute_bsm_vanilla_price(f, K, T, v, t, D)
            hv, hF = 1e-3 * vol, 1e-2 * F * vol * np.sqrt(T)          # steps small against the scale of d1
            d = lambda fn, h: (8 * (fn(h) - fn(-h)) - (fn(2 * h) - fn(-2 * h))) / (12 * h)
            vega, dF, dFF, dFv, dvv = og.black_partials(F, K, T, D, vol, is_call)
            scale = D * F
            np.testing.assert_allclose(vega, d(lambda h: B(F, vol + h), hv), rtol=1e-8, atol=1e-10 * scale)
            np.testing.assert_allclose(dF, d(lambda h: B(F + h, vol), hF), rtol=1e-7, atol=1e-10)
            np.testing.assert_allclose(dFF, d(lambda h: og.black_partials(F + h, K, T, D, vol, is_call)[1], hF), rtol=1e-6, atol=1e-10 / F)
            np.testing.assert_allclose(dFv, d(lambda h: og.black_partials(F + h, K, T, D, vol, is_call)[0], hF), rtol=1e-6, atol=1e-10)
            np.testing.assert_allclose(dvv, d(lambda h: og.black_partials(F, K, T, D, vol + h, is_call)[0], hv), rtol=1e-6,
                                       atol=1e-9 * scale)


@pytest.mark.parametrize("n", [1, 5, 15])
def test_transform_recovers_the_black_in_model(n):
    """P = B(F, g(F, p)) with its rows written analytically: the transform gives back g's derivatives to 1e-10 relative, every type,
    |d1| up to 8, D != 1"""
    c = _case(n)
    price, greeks, vanna, hessian, want = og.black_in_model(c["F"], c["K"], c["T"], c["D"], c["types"], c["p"], c["F0"], *c["model"])
    vol = obsm.infer_bsm_implied_vol(c["F"], c["T"], c["K"], price, c["types"], c["D"])
    np.testing.assert_allclose(vol, want["ivol"], rtol=1e-10)
    g, v, h = og.ivol_sensitivities(c["F"], c["K"], c["T"], c["D"], want["ivol"], og.is_call_type(c["types"]), greeks, vanna, hessian)
    for got, exp, name in ((g, want["greeks"], "greeks"), (v, want["vanna"], "vanna"), (h, want["hessian"], "hessian")):
        scale = np.max(np.abs(exp), axis=1, keepdims=True)           # rows whose value crosses zero are judged against the row's size
        np.testing.assert_array_less(np.abs(got - exp), 1e-10 * np.maximum(np.abs(exp), 1e-3 * scale) + 1e-300, err_msg=name)


def _inverted(c, F, p):
    """the Black-in model's price at (F, p), inverted by oracle/bsm.py's independent bisection"""
    price = og.black_in_model(F, c["K"], c["T"], c["D"], c["types"], p, c["F0"], *c["model"])[0]
    return obsm.infer_bsm_implied_vol(F, c["T"], c["K"], price, c["types"], c["D"])


def test_transform_vs_central_differences_of_the_inversion():
    """the transform's first-order rows and vanna against 4-point central differences of the inverted prices, to 1e-6"""
    n = 3
    c = _case(n)
    F, p = c["F"], c["p"]
    price, greeks, vanna, hessian, want = og.black_in_model(F, c["K"], c["T"], c["D"], c["types"], p, c["F0"], *c["model"])
    vol = obsm.infer_bsm_implied_vol(F, c["T"], c["K"], price, c["types"], c["D"])
    g, v, h = og.ivol_sensitivities(F, c["K"], c["T"], c["D"], vol, og.is_call_type(c["types"]), greeks, vanna, hessian)
    d = lambda fn, hh: (8 * (fn(hh) - fn(-hh)) - (fn(2 * hh) - fn(-2 * hh))) / (12 * hh)
    hF, hp = 1e-3 * F, 1e-3
    np.testing.assert_allclose(g[0], d(lambda s: _inverted(c, F + s, p), hF), rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(g[1], d(lambda s: (_inverted(c, F + s + 1e-3, p) - _inverted(c, F + s - 1e-3, p)) / 2e-3, hF), rtol=1e-4,
                               atol=1e-7)
    for k in range(n):
        ek = np.eye(n)[k]
        np.testing.assert_allclose(g[2 + k], d(lambda s: _inverted(c, F, p + s * ek), hp), rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(v[k], d(lambda s: og.ivol_sensitivities(F + s, c["K"], c["T"], c["D"], _inverted(c, F + s, p),
                                                                           og.is_call_type(c["types"]),
                                                                           og.black_in_model(F + s, c["K"], c["T"], c["D"], c["types"], p,
                                                                                             c["F0"], *c["model"])[1])[0][2 + k], hF),
                                   rtol=1e-6, atol=1e-8)


def test_nan_and_bracket_end_conventions():
    c = _case(2)
    price, greeks, vanna, hessian, want = og.black_in_model(c["F"], c["K"], c["T"], c["D"], c["types"], c["p"], c["F0"], *c["model"])
    vol = want["ivol"].copy()
    vol[0], vol[1], vol[2] = np.nan, obsm.VOL_LO, obsm.VOL_HI * (1 - 1e-15)
    g, v, h = og.ivol_sensitivities(c["F"], c["K"], c["T"], c["D"], vol, og.is_call_type(c["types"]), greeks, vanna, hessian)
    for rows in (g, v, h):
        assert np.isnan(rows[:, 0]).all() and (rows[:, 1:3] == 0.0).all() and np.isfinite(rows[:, 3:]).all()


# ---- the exact-gradient objective ------------------------------------------------------------------------------------------------------
def _stand_in(nfields: int, J: int = 23, seed: int = 3, nan_at=()):
    """a smooth numpy model of the ivol-greeks call: vols(fields) = v0 + A tanh(fields - c), exact d vols / d fields, a call counter"""
    rng = np.random.RandomState(seed)
    v0, A, c = rng.uniform(0.2, 0.6, J), rng.uniform(-0.3, 0.3, (J, nfields)), rng.uniform(-0.5, 0.5, nfields)
    calls = []

    def vols_and_rows(fields):
        calls.append(1)
        t = np.tanh(fields - c)
        vols = v0 + A @ t
        rows = (A * (1.0 - t * t)).T
        vols[list(nan_at)] = np.nan
        return vols, rows
    return vols_and_rows, calls


def _codecs():
    from stochvolmodels_b200 import LogSvParams
    from stochvolmodels_b200.pricers.calibration import LogsvModelCalibrationType as T, LogSvParameterCodec
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import hawkes_fit_jacobian
    lo, hi = LogSvParams(0.1, 0.1, 0.25, 0.25, -3.0, 0.2), LogSvParams(1.5, 1.5, 10.0, 10.0, 3.0, 3.0)
    start = LogSvParams(0.8, 0.9, 2.0, 3.0, 0.2, 1.3)
    out = []
    for kind, names in ((T.PARAMS4, ("sigma0", "theta", "beta", "volvol")), (T.PARAMS5, ("sigma0", "theta", "kappa1", "beta", "volvol"))):
        codec = LogSvParameterCodec(start, lo, hi, kind)

        def fields(x, codec=codec):
            q = codec.parse(x)
            return np.array([q.sigma0, q.theta, q.kappa1, q.kappa2, q.beta, q.volvol])
        out.append((kind.name, codec.initial_and_bounds()[0], fields, codec.field_jacobian))
    out.append(("heston", np.array([0.6, 0.8, 3.0, -0.3, 1.1]), lambda x: x.copy(), lambda x: np.eye(5)))
    D = hawkes_fit_jacobian()

    def hawkes_fields(x):
        from stochvolmodels_b200 import HawkesJDParams
        from stochvolmodels_b200.engine import HAWKES_GREEK_PARAMS
        q = HawkesJDParams(sigma=x[0], mean_p=x[1], mean_m=x[2], theta_p=x[3], theta_m=x[4], kappa_p=x[5], kappa_m=x[5], beta1_p=x[6],
                           beta2_p=-x[6], beta1_m=x[7], beta2_m=-x[7])
        return np.array([getattr(q, n) for n in HAWKES_GREEK_PARAMS])
    out.append(("hawkes", np.array([0.4, 0.2, -0.3, 6.0, 8.0, 25.0, 70.0, 100.0]), hawkes_fields, lambda x: D))
    return out


@pytest.mark.parametrize("codec", _codecs(), ids=lambda c: c[0])
@pytest.mark.parametrize("nan_at", [(), (2, 7)])
def test_exact_objective_gradient_vs_central_differences(codec, nan_at):
    from stochvolmodels_b200.pricers.calibration import ExactGradientObjective
    name, x0, fields, jacobian = codec
    nf = jacobian(x0).shape[0]
    model, calls = _stand_in(nf, nan_at=nan_at)
    rng = np.random.RandomState(1)
    market = model(fields(x0) * 1.01)[0] + rng.uniform(-0.01, 0.01, 23)
    weights = rng.uniform(0.5, 1.5, 23)
    calls.clear()
    obj = ExactGradientObjective(ivol_greeks=lambda x: model(fields(x)), field_jacobian=jacobian, market_vols=market, weights=weights)
    f, g = obj.fun(x0), obj.jac(x0)
    assert len(calls) == 1 and obj.nb_batches == 2 and obj.nan_quotes == len(nan_at)       # fun then jac at x: one call
    assert np.isfinite(f) and np.isfinite(g).all()
    vols = model(fields(x0))[0]
    assert f == float(np.nansum(weights * np.square(vols - market)))
    fd = np.empty_like(x0)
    for i in range(x0.size):
        h = 1e-5 * max(1.0, abs(x0[i]))
        e = np.eye(x0.size)[i] * h
        fun = lambda y: ExactGradientObjective(lambda z: model(fields(z)), jacobian, market, weights).fun(y)
        fd[i] = (8 * (fun(x0 + e) - fun(x0 - e)) - (fun(x0 + 2 * e) - fun(x0 - 2 * e))) / (12 * h)
    np.testing.assert_allclose(g, fd, rtol=1e-7, atol=1e-7 * np.max(np.abs(fd)))


def test_to_chain_ivol_sensitivities_layout(monkeypatch):
    """FourierChainHessian -> ChainIvolHessian: rows split per maturity, hessian symmetric with shared arrays, rows sent in the entry
    point's layout"""
    from stochvolmodels_b200 import OptionChain, engine
    from stochvolmodels_b200.pricers import fourier_greeks as fg
    chain = OptionChain(ttms=np.array([0.1, 0.5]), forwards=np.array([1.0, 1.1]), strikes_ttms=[np.array([0.9, 1.0]), np.array([1.0, 1.1, 1.2])],
                        optiontypes_ttms=[np.array(["P", "C"]), np.array(["P", "C", "C"])])
    names = ("a", "b", "c")
    J, split = 5, (lambda r: [r[:2].copy(), r[2:].copy()])
    rng = np.random.RandomState(0)
    greeks, vanna, hessian = rng.rand(5, J), rng.rand(3, J), rng.rand(6, J)
    src = fg.to_fourier_chain_hessian(split(rng.rand(J)), greeks, vanna, hessian, np.array([0, 2, 5]), names)
    seen = {}

    def fake(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms, g, v, h):
        seen.update(g=g, v=v, h=h)
        return split(np.arange(J, dtype=float)), 2 * g, None if v is None else 3 * v, None if h is None else 4 * h
    monkeypatch.setattr(engine, "bsm_implied_vol_sensitivities", fake)
    out = fg.to_chain_ivol_sensitivities(chain, src)
    np.testing.assert_array_equal(seen["g"], greeks)
    np.testing.assert_array_equal(seen["v"], vanna)
    np.testing.assert_array_equal(seen["h"], hessian)
    assert isinstance(out, fg.ChainIvolHessian) and list(out.params) == list(names)
    np.testing.assert_array_equal(np.concatenate(out.gamma), 2 * greeks[1])
    np.testing.assert_array_equal(np.concatenate(out.params["c"]), 2 * greeks[4])
    np.testing.assert_array_equal(np.concatenate(out.vanna["b"]), 3 * vanna[1])
    np.testing.assert_array_equal(np.concatenate(out.hessian["b"]["c"]), 4 * hessian[4])
    assert out.hessian["c"]["b"] is out.hessian["b"]["c"]
    first = fg.to_chain_ivol_sensitivities(chain, fg.to_fourier_chain_greeks(src.prices, greeks, np.array([0, 2, 5]), names))
    assert type(first) is fg.ChainIvolGreeks and seen["v"] is None


# ---- rejections: nothing reaches the library -------------------------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def refuse(*args, **kwargs):
        raise AssertionError("library call")
    monkeypatch.setattr(_capi, "call", refuse)
    monkeypatch.setattr(_capi, "load_library", refuse)


def _market_chain():
    from stochvolmodels_b200 import get_btc_test_chain_data
    return get_btc_test_chain_data()


def test_calibration_rejections_before_any_library_call(no_library):
    from stochvolmodels_b200 import (CalibrationEngine, HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer,
                                     LogsvModelCalibrationType)
    chain, start = _market_chain(), LogSvParams(0.8, 1.0, 3.0, 3.0, 0.1, 1.8)
    for engine_kind in (CalibrationEngine.MC, CalibrationEngine.ROUGH_MC):
        with pytest.raises(NotImplementedError, match="exact"):
            LogSVPricer().calibrate_model_params_to_chain(chain, start, calibration_engine=engine_kind, gradient="exact")
    with pytest.raises(NotImplementedError, match="VARSWAP"):
        LogSVPricer().calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT,
                                                      gradient="exact")
    with pytest.raises(NotImplementedError, match="risk"):
        HawkesJDPricer().calibrate_risk_premia_gamma_to_chain(chain, HawkesJDParams(risk_premia_gamma=0.1), gradient="exact", print_iter=False)
    for call in (lambda: LogSVPricer().calibrate_model_params_to_chain(chain, start, gradient="adjoint"),
                 lambda: HestonPricer().calibrate_model_params_to_chain(chain, HestonParams(), gradient="central"),
                 lambda: HawkesJDPricer().calibrate_model_params_to_chain(chain, HawkesJDParams(), gradient=None),
                 lambda: HawkesJDPricer().calibrate_risk_premia_gamma_to_chain(chain, HawkesJDParams(), gradient="exactly", print_iter=False)):
        with pytest.raises(ValueError, match="gradient must be"):
            call()


def test_ivol_sensitivity_rejections_before_any_library_call(no_library):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer
    from stochvolmodels_b200.utils.config import VariableType
    chain = _market_chain()
    for pricer, params in ((LogSVPricer(), LogSvParams()), (HestonPricer(), HestonParams())):
        for method in (pricer.compute_chain_ivol_greeks, pricer.compute_chain_ivol_hessian):
            for kw in ({"variable_type": VariableType.Q_VAR}, {"is_analytic": True}, {"is_stiff_solver": True}):
                with pytest.raises(NotImplementedError):
                    method(chain, params, **kw)
    hawkes = HawkesJDPricer()
    for method in (hawkes.compute_chain_ivol_greeks, hawkes.compute_chain_ivol_hessian):
        with pytest.raises(NotImplementedError, match="risk"):
            method(chain, HawkesJDParams(risk_premia_gamma=0.2))
        with pytest.raises(NotImplementedError):
            method(chain, HawkesJDParams(), is_stiff_solver=True)


def test_engine_argument_checks_before_any_library_call(no_library):
    from stochvolmodels_b200 import engine
    chain = _market_chain()
    J = sum(len(k) for k in chain.strikes_ttms)
    args = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms, [np.ones(len(k)) for k in chain.strikes_ttms])
    for bad in (np.zeros((2, J)), np.zeros((18, J)), np.zeros((7, J - 1))):
        with pytest.raises(ValueError, match="greeks"):
            engine.bsm_implied_vol_sensitivities(*args, bad)
    with pytest.raises(ValueError, match="together"):
        engine.bsm_implied_vol_sensitivities(*args, np.zeros((7, J)), vanna=np.zeros((5, J)))
    with pytest.raises(ValueError, match="shape"):
        engine.bsm_implied_vol_sensitivities(*args, np.zeros((7, J)), vanna=np.zeros((5, J)), hessian=np.zeros((14, J)))


def test_c_entry_point_rejects_before_touching_the_device():
    """the entry point's argument checks return before any CUDA call: -1 for NP outside 1..15 and NULL mismatches, -3 for unknown
    type codes"""
    import os
    from stochvolmodels_b200 import _capi as C
    if not os.path.exists(C.LIB_PATH):
        from stochvolmodels_b200._build import build_library
        build_library()
    lib = C.load_library()
    M, J = 1, 3
    ttms, fw, df = np.array([0.5]), np.ones(1), np.ones(1)
    offsets = np.array([0, J], dtype=np.int32)
    strikes, prices = np.array([0.9, 1.0, 1.1]), np.full(J, 0.05)
    types = np.zeros(J, dtype=np.int8)
    out = lambda rows: np.zeros((rows, J))

    def rc(NP, vanna, hessian, ov, oh, t=types):
        return lib.b200sv_bsm_implied_vol_sensitivities(M, C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(offsets), C.dptr(strikes), C.i8ptr(t),
                                                       C.dptr(prices), NP, C.dptr(out(2 + max(NP, 1))), C.dptr(vanna), C.dptr(hessian),
                                                       C.dptr(np.zeros(J)), C.dptr(out(2 + max(NP, 1))), C.dptr(ov), C.dptr(oh))
    assert rc(0, None, None, None, None) == -1
    assert rc(16, None, None, None, None) == -1
    assert rc(2, out(2), None, out(2), None) == -1                  # vanna without hessian
    assert rc(2, out(2), out(3), None, out(3)) == -1                # an input without its output
    assert rc(2, None, None, out(2), out(3)) == -1                  # outputs without inputs
    assert rc(2, None, None, None, None, np.array([0, 4, 1], dtype=np.int8)) == -3
