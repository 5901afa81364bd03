"""GPU: ``gradient='pathwise'`` of the LogSV calibration on the Monte Carlo engines (DESIGN.md §4.7).

  objective -- the pathwise objective's value equals the difference route's at the same point (bit for bit for CalibrationEngine.MC with
               either source of normals, to 1e-12 for ROUGH_MC) and its gradient equals central differences of that value on the same normals
  fits      -- the own-market fits of tests/test_gpu_calibration.py and tests/test_gpu_rough.py converge as well with the pathwise gradient
               and land within 1e-3 of the difference-route fit's objective from the same start
"""
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
KR = np.array([0.85, 0.95, 1.0, 1.05, 1.15])
W2, X2 = np.array([0.80082171, 0.34941995]), np.array([0.0015625, 1.31611315])     # the two-node H = 0.45 kernel of test_gpu_rough.py


def _own_market_chain(engine_kind, mc_randoms):
    """(chain, flat chain, truth, start, kwargs): the market is the model's own vols on the calibration's fixed normals, as in the existing
    own-market tests"""
    from stochvolmodels_b200 import CalibrationEngine, LogSvParams, LogSVPricer, OptionChain, engine
    from stochvolmodels_b200.multi_gpu import _fixed_randoms_chain_device
    from stochvolmodels_b200.pricers.logsv_pricer import _params_c, get_randoms_for_chain_valuation
    if engine_kind == CalibrationEngine.ROUGH_MC:
        ttms, K = np.array([0.1, 0.25]), KR
        truth = LogSvParams(sigma0=0.9, theta=1.0, kappa1=4.0, kappa2=4.0, beta=0.3, volvol=1.5, H=0.45, weights=W2, nodes=X2)
        start = LogSvParams(sigma0=0.8, theta=1.1, kappa1=4.0, kappa2=4.0, beta=0.2, volvol=1.3, H=0.45, weights=W2, nodes=X2)
        kw = dict(nb_path=50_000, nb_steps=120, seed=10)
    else:
        ttms, K = np.array([1.0 / 12.0, 0.25]), K5
        truth = LogSvParams(sigma0=0.9, theta=1.0, kappa1=4.0, kappa2=4.0, beta=0.3, volvol=1.5)
        start = LogSvParams(sigma0=0.8, theta=0.9, kappa1=4.0, kappa2=4.0, beta=0.1, volvol=1.2)
        kw = dict(nb_path=50_000 if mc_randoms == "numpy" else 200_000, nb_steps=360, seed=10)
    fw, types = np.ones(2), [T5, T5]
    flat = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K, K], optiontypes_ttms=types, ids=np.array(["a", "b"]))
    if engine_kind == CalibrationEngine.ROUGH_MC:
        prices = LogSVPricer().model_mc_price_chain(flat, truth, use_rough_mc=True, **kw)[0]
    elif mc_randoms == "numpy":
        rnd = get_randoms_for_chain_valuation(ttms=ttms, nb_path=kw["nb_path"], nb_steps_per_year=360, seed=10, device=True)
        prices = _fixed_randoms_chain_device(rnd, ttms, fw, np.ones(2), [K, K], types, _params_c(truth), np.ones(2), True, 1, True)[0]
    else:
        prices = engine.logsv_mc_chain(_params_c(truth), ttms, fw, np.ones(2), None, [K, K], types, kw["nb_path"], 360, True, 1, 10,
                                       engine.mc_flags("fp64", "fp32"))[0]
    vols = flat.compute_model_ivols_from_chain_data(prices)
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K, K], optiontypes_ttms=types, ids=np.array(["a", "b"]),
                        bid_ivs=[v.copy() for v in vols], ask_ivs=[v.copy() for v in vols])
    return chain, flat, vols, start, dict(kw, calibration_engine=engine_kind, mc_randoms=mc_randoms)


def _objective(monkeypatch, chain, start, calibration_type, gradient, kw):
    """the objective calibrate_logsv builds, taken from its call to run_slsqp (which returns the start without optimizing)"""
    from stochvolmodels_b200 import LogSVPricer
    from stochvolmodels_b200.pricers import calibration
    seen = {}

    def capture(objective, p0, bounds, constraints=None, disp=False):
        seen.update(objective=objective, p0=np.asarray(p0, dtype=float), bounds=bounds)
        return np.asarray(p0, dtype=float), SimpleNamespace(fun=np.nan, nit=0)

    monkeypatch.setattr(calibration, "run_slsqp", capture)
    LogSVPricer().calibrate_model_params_to_chain(chain, start, model_calibration_type=calibration_type, gradient=gradient, **kw)
    return seen["objective"], seen["p0"], seen["bounds"]


ROUTES = [("MC", "numpy"), ("MC", "philox"), ("ROUGH_MC", "numpy"), ("ROUGH_MC", "philox")]


@pytest.mark.parametrize("engine_name,mc_randoms", ROUTES)
@pytest.mark.parametrize("calibration_type", ["PARAMS4", "PARAMS5"])
def test_pathwise_objective_and_gradient(cuda_lib, monkeypatch, engine_name, mc_randoms, calibration_type):
    """value: the difference route's at the same x (bit for bit on MC; ROUGH_MC sensitivity prices match its batch route to ~1e-13, so
    1e-12 relative).  Gradient: central differences of the pathwise value on the same normals, relative step 1e-5 per coordinate.  The
    sample objective is piecewise smooth (a path changes payoff branch, or a rough path its reset branch, inside the bump): that and the
    O(h^2) truncation are well inside 1e-3 of the gradient's largest component; PARAMS5 exercises the kappa2 = kappa1 / theta chain rule."""
    from stochvolmodels_b200 import CalibrationEngine, LogsvModelCalibrationType
    engine_kind, ctype = CalibrationEngine[engine_name], LogsvModelCalibrationType[calibration_type]
    chain, _, _, start, kw = _own_market_chain(engine_kind, mc_randoms)
    pathwise, p0, _ = _objective(monkeypatch, chain, start, ctype, "pathwise", kw)
    difference, _, _ = _objective(monkeypatch, chain, start, ctype, "difference", kw)
    x = p0 * np.linspace(0.97, 1.03, p0.size)            # off the start, where every component of the gradient is alive
    if engine_kind == CalibrationEngine.MC:
        assert pathwise.fun(x) == difference.fun(x)
    else:
        assert pathwise.fun(x) == pytest.approx(difference.fun(x), rel=1e-12, abs=0)
    g = pathwise.jac(x)
    fd = np.empty_like(g)
    for i in range(x.size):
        h = 1e-5 * abs(x[i])
        up, dn = x.copy(), x.copy()
        up[i] += h
        dn[i] -= h
        fd[i] = (pathwise.fun(up) - pathwise.fun(dn)) / (2 * h)
    assert np.all(np.abs(g - fd) <= 1e-3 * np.max(np.abs(g)) + 1e-12), (g, fd)


@pytest.mark.parametrize("engine_name,mc_randoms", [("MC", "numpy"), ("MC", "philox"), ("ROUGH_MC", "numpy")])
def test_own_market_fit_with_the_pathwise_gradient(cuda_lib, engine_name, mc_randoms):
    """the own-market fits of tests/test_gpu_calibration.py (MC, both sources of normals) and tests/test_gpu_rough.py (ROUGH_MC, H = 0.45)
    with gradient='pathwise': the same objective and vol tolerances, and an objective within 1e-3 of the difference-route fit's"""
    from stochvolmodels_b200 import CalibrationEngine, LogSVPricer, LogsvModelCalibrationType
    from stochvolmodels_b200.pricers.logsv_pricer import _params_c
    engine_kind = CalibrationEngine[engine_name]
    chain, flat, vols, start, kw = _own_market_chain(engine_kind, mc_randoms)
    fit_kw = dict(kw, model_calibration_type=LogsvModelCalibrationType.PARAMS4, return_info=True)
    pricer = LogSVPricer()
    fit, info = pricer.calibrate_model_params_to_chain(chain, start, gradient="pathwise", **fit_kw)
    _, ref = pricer.calibrate_model_params_to_chain(chain, start, **fit_kw)
    assert info["fun"] <= ref["fun"] * (1 + 1e-3) + 1e-9, (info, ref)
    if engine_kind == CalibrationEngine.ROUGH_MC:
        assert info["fun"] < 2e-6 and info["nit"] >= 3, info
        assert info["reset_paths"].shape == (2,) and "reset_paths" not in ref
        fit_prices = pricer.model_mc_price_chain(flat, fit, nb_path=kw["nb_path"], nb_steps=kw["nb_steps"], use_rough_mc=True, seed=kw["seed"])[0]
        fit_vols = flat.compute_model_ivols_from_chain_data(model_prices=fit_prices)
        assert max(np.max(np.abs(a - b)) for a, b in zip(fit_vols, vols)) < 3e-3
        return
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.multi_gpu import _fixed_randoms_chain_device
    from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_chain_valuation
    assert info["fun"] < 1e-5
    if mc_randoms == "numpy":
        rnd = get_randoms_for_chain_valuation(ttms=chain.ttms, nb_path=kw["nb_path"], nb_steps_per_year=360, seed=10, device=True)
        fit_prices = _fixed_randoms_chain_device(rnd, chain.ttms, chain.forwards, np.ones(2), chain.strikes_ttms, chain.optiontypes_ttms,
                                                 _params_c(fit), np.ones(2), True, 1, True)[0]
    else:
        fit_prices = engine.logsv_mc_chain(_params_c(fit), chain.ttms, chain.forwards, np.ones(2), None, chain.strikes_ttms, chain.optiontypes_ttms,
                                           kw["nb_path"], 360, True, 1, 10, engine.mc_flags("fp64", "fp32"))[0]
    fit_vols = flat.compute_model_ivols_from_chain_data(fit_prices)
    np.testing.assert_allclose(np.concatenate(fit_vols), np.concatenate(vols), atol=5e-3)
