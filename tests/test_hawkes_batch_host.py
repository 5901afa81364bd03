"""CPU tests of the batched Hawkes chain pricer's host side: the argument checks of b200sv_hawkesjd_price_chain_batch (each case has exactly
one defect and must return before the first stream operation, so the library is needed but no GPU), the objective / gradient of the
calibration drivers against scipy's own differencing of the one-set objective, and both drivers against the sequential oracle -- the last two
with a numpy stand-in for the GPU pricer."""
import ctypes
import math

import numpy as np
import pytest
from scipy.optimize._numdiff import approx_derivative

import hawkes_sequential as seq
from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine
from stochvolmodels_b200 import _capi as C
from stochvolmodels_b200.pricers import calibration as cal

NULL = (-1, "invalid argument: null pointer")
TTMS = (-1, "invalid argument: ttms must be positive and strictly increasing")
BMP = (-1, "invalid argument: 1 <= B <= 65535, M >= 1, P >= 3")
STRIKE = (-1, "invalid argument: strikes must be positive")
EMPTY = (-1, "invalid argument: the chain has no strikes")
GAMMAS = (-1, "invalid argument: gammas must be finite (NULL: no risk kernel)")
NOT_IMPL = (-5, "not implemented")

KP = C.HawkesParamsC(0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5)


def _valid():
    return dict(B=2, M=2, ttms=[0.25, 0.5], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2, spot=1,
                P=0, gammas=None, params=True, fw=True, df=True, prices=True)


def _call(c):
    lib = C.load_library()
    ttms = None if c["ttms"] is None else C.f64(c["ttms"])
    off = None if c["offsets"] is None else np.asarray(c["offsets"], dtype=np.int32)
    strikes = None if c["strikes"] is None else C.f64(c["strikes"])
    types = None if c["types"] is None else np.asarray(c["types"], dtype=np.int8)
    gammas = None if c["gammas"] is None else C.f64(c["gammas"])
    fw, df, out, iv = np.ones(2), np.ones(2), np.zeros(64), np.zeros(64)
    params = (C.HawkesParamsC * 2)(KP, KP) if c["params"] else None
    return lib.b200sv_hawkesjd_price_chain_batch(params, c["B"], c["M"], C.dptr(ttms), C.dptr(fw) if c["fw"] else None,
                                                 C.dptr(df) if c["df"] else None, C.iptr(off), C.dptr(strikes),
                                                 None if types is None else C.i8ptr(types), c["spot"], -1.0, c["P"], C.dptr(gammas),
                                                 C.dptr(out) if c["prices"] else None, C.dptr(iv))


CASES = [
    (dict(params=False), NULL), (dict(ttms=None), NULL), (dict(fw=False), NULL), (dict(df=False), NULL), (dict(offsets=None), NULL),
    (dict(strikes=None), NULL), (dict(types=None), NULL), (dict(prices=False), NULL),
    (dict(B=0), BMP), (dict(B=65536), BMP), (dict(M=0), BMP), (dict(P=2), BMP),
    (dict(offsets=[0, 0, 0]), EMPTY),
    (dict(ttms=[0.5, 0.25]), TTMS),
    (dict(strikes=[0.9, 1.0, 1.1, 0.9, 0.0, 1.1]), STRIKE),
    (dict(types=[C.PUT, 4, C.CALL] * 2), NOT_IMPL),
    (dict(types=[C.PUT, C.INV_CALL, C.CALL] * 2), NOT_IMPL),                        # inverse payoffs under the spot measure
    (dict(gammas=[0.2, math.nan]), GAMMAS),                                          # NaN and finite mixed
    (dict(gammas=[math.nan, math.nan]), GAMMAS),
    (dict(gammas=[0.2, math.inf]), GAMMAS),
    (dict(gammas=[0.2, 0.3], spot=0), NOT_IMPL),                                     # the risk kernel: spot measure only
    (dict(gammas=[0.2, 0.3], spot=0, types=[C.PUT, C.INV_CALL, C.CALL] * 2), NOT_IMPL),
    (dict(gammas=[0.2, 0.3], types=[C.PUT, C.INV_CALL, C.CALL] * 2), NOT_IMPL),      # ... and 'C' / 'P' only
]


@pytest.mark.parametrize("change,expected", [pytest.param(ch, e, id="-".join(f"{k}={v}" for k, v in ch.items())) for ch, e in CASES])
def test_batch_entry_point_rejects(change, expected):
    c = _valid()
    c.update(change)
    rc = _call(c)
    assert (rc, C.load_library().b200sv_last_error().decode()) == expected


def test_engine_wrapper_rejects_what_the_risk_kernel_does_not_price():
    chain = (np.array([0.25]), np.ones(1), np.ones(1), [np.array([1.0])], [np.array(["IC"])])
    with pytest.raises(ValueError, match="not implemented"):
        engine.hawkesjd_price_chain_batch([KP], *chain, gammas=[0.2])
    with pytest.raises(ValueError, match="not implemented"):
        engine.hawkesjd_price_chain_batch([KP], *chain, is_spot_measure=False, gammas=[0.2])
    with pytest.raises(ValueError, match="gammas must have shape"):
        engine.hawkesjd_price_chain_batch([KP, KP], *chain[:4], [np.array(["C"])], gammas=[0.2])


# ---- a numpy stand-in for the GPU chain pricer: a smooth map from a parameter set to the chain's implied vols --------------------------
_FIELDS = ("sigma", "mean_p", "mean_m", "theta_p", "theta_m", "kappa_p", "beta1_p", "beta1_m")


def _features(values, gamma):
    v = dict(values)
    return np.array([v["sigma"], 4 * v["mean_p"], 4 * v["mean_m"], v["theta_p"] / 20, v["theta_m"] / 20, v["kappa_p"] / 50, v["beta1_p"] / 60,
                     v["beta1_m"] / 60, 0.0 if gamma is None else gamma])


class StandIn:
    """vols = 0.2 + 0.6 sigmoid(A f) per quote; a quote has no vol (NaN) where its score leaves a band, as a quote whose model price leaves
    the no-arbitrage bounds has none"""

    def __init__(self, J, seed=3):
        rng = np.random.default_rng(seed)
        self.A = rng.normal(size=(J, 9)) * np.linspace(0.5, 1.5, 9)
        self.calls = 0

    def vols(self, values, gamma):
        s = self.A @ _features(values, gamma)
        v = 0.2 + 0.6 / (1.0 + np.exp(-s))
        return np.where(np.abs(s) > 6.0, np.nan, v)

    def batch(self, params_list, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_spot_measure=True, vol_scaler=None,
              max_phi=500, gammas=None, with_ivols=True):
        self.calls += 1
        rows = [self.vols({k: getattr(p, k) for k in _FIELDS}, None if gammas is None else gammas[b]) for b, p in enumerate(params_list)]
        return np.full((len(rows), rows[0].size), np.nan), np.vstack(rows)

    def per_set(self, option_chain, params):
        flat = self.vols({k: getattr(params, k) for k in _FIELDS}, params.risk_premia_gamma)
        return np.split(flat, np.cumsum([len(k) for k in option_chain.strikes_ttms])[:-1])


def _chain(vols=None):
    K = np.linspace(0.75, 1.3, 12)
    ttms = np.array([0.08, 0.25, 0.5])
    vols = vols or [0.5 * np.ones_like(K)] * 3
    return OptionChain(ttms=ttms, forwards=np.ones(3), strikes_ttms=[K] * 3, optiontypes_ttms=[np.where(K >= 1.0, "C", "P")] * 3,
                       ids=np.array(["1m", "3m", "6m"]), bid_ivs=vols, ask_ivs=[v.copy() for v in vols])


@pytest.fixture
def stand_in(monkeypatch):
    s = StandIn(36)
    monkeypatch.setattr(engine, "hawkesjd_price_chain_batch", s.batch)
    monkeypatch.setattr(HawkesJDPricer, "compute_model_ivols_for_chain", lambda self, option_chain, params, **kw: s.per_set(option_chain, params))
    return s


def _market(stand_in, true):
    return _chain([np.where(np.isnan(v), 0.5, v) for v in stand_in.per_set(_chain(), true)])      # quotes are finite


GAMMA_CASES = [
    ("interior", np.array([0.45, 0.05]), 0.025),
    ("negative", np.array([0.30, -0.40]), 0.025),
    ("near_upper", np.array([1.5 - 0.01, 1.0 - 0.004]), 0.025),            # within eps of both upper bounds: backward steps
    ("at_upper", np.array([1.5, 1.0]), 0.025),
    ("at_lower", np.array([0.01, -1.0]), 0.025),
]
MODEL_CASES = [
    ("interior", np.array([0.45, 0.03, -0.04, 7.0, 7.0, 25.0, 33.0, 36.0]), cal.SLSQP_EPS),
    ("negative", np.array([0.2, 0.5, -0.6, 3.0, 80.0, 2.0, 90.0, 1.5]), cal.SLSQP_EPS),
    ("near_upper", np.array([2.0 - 1e-8, 0.99 - 5e-9, -0.01, 100.0, 100.0 - 1e-9, 100.0, 50.0, 100.0]), cal.SLSQP_EPS),
]


def _both(stand_in, which, x, eps):
    """(batched objective, sequential objective) of the driver ``which`` at step ``eps``"""
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _batched_vol_objective
    pricer = HawkesJDPricer()
    if which == "gamma":
        chain = _market(stand_in, HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5))
        fixed = {k: v for k, v in HawkesJDParams().to_dict().items() if k != "risk_premia_gamma"}
        to_params = lambda p: HawkesJDParams(**{**fixed, "sigma": float(p[0])}, risk_premia_gamma=float(8.0 * p[1]))
        bounds, scale = seq.GAMMA_BOUNDS, 10000.0
    else:
        chain = _market(stand_in, HawkesJDParams(sigma=0.4, mean_p=0.04, mean_m=-0.05, theta_p=6.0, theta_m=8.0, kappa_p=25.0, kappa_m=25.0,
                                                 beta1_p=30.0, beta2_p=-30.0, beta1_m=40.0, beta2_m=-40.0))
        to_params = seq.model_unpack(HawkesJDParams())
        bounds, scale = seq.MODEL_BOUNDS, 1.0
    batched = _batched_vol_objective(chain, to_params, True, False, bounds, eps, scale=scale)
    return batched, seq.vol_objective(pricer, chain, to_params, scale=scale), bounds


@pytest.mark.parametrize("which,name,x,eps", [pytest.param("gamma", n, x, e, id=f"gamma-{n}") for n, x, e in GAMMA_CASES]
                         + [pytest.param("model", n, x, e, id=f"model-{n}") for n, x, e in MODEL_CASES]
                         + [pytest.param("model", "gamma_step", MODEL_CASES[0][1], 0.025, id="model-eps0.025"),
                            pytest.param("gamma", "slsqp_step", GAMMA_CASES[1][1], cal.SLSQP_EPS, id="gamma-slsqp_eps")])
def test_objective_and_gradient_are_scipys_own_difference(stand_in, which, name, x, eps):
    batched, sequential, bounds = _both(stand_in, which, x, eps)
    lb, ub = np.array([b[0] for b in bounds]), np.array([b[1] for b in bounds])
    f0 = sequential(x)
    g = approx_derivative(sequential, x, method="2-point", abs_step=eps, bounds=(lb, ub), f0=f0)
    assert batched.fun(x) == f0
    np.testing.assert_array_equal(batched.jac(x), g)
    assert batched.nb_batches == 2 and stand_in.calls == 2              # x alone, then its n neighbours in one batch
    assert batched.fun(x) == f0 and batched.nb_batches == 2             # memoised on the last point


def test_value_only_points_price_one_set(stand_in):
    """a point SLSQP asks only the value of (a line-search trial) prices x alone; the neighbours wait for jac"""
    batched, _, _ = _both(stand_in, "gamma", GAMMA_CASES[0][1], 0.025)
    sizes = []
    inner = batched.batch_vols
    batched.batch_vols = lambda pts: (sizes.append(len(pts)), inner(pts))[1]
    batched.fun(GAMMA_CASES[0][1])
    batched.fun(GAMMA_CASES[1][1])
    batched.jac(GAMMA_CASES[1][1])
    assert sizes == [1, 1, 2]


def test_neighbours_are_the_points_scipy_evaluates_signed_zeros_included():
    """the difference points handed to the pricer and to on_point are scipy's own, bit for bit (a -0.0 coordinate stays -0.0 where it
    is not the one being moved, as in scipy's copy-and-move construction)"""
    x = np.array([-0.0, 0.5, -0.0])
    bounds = [(-1.0, 1.0)] * 3
    seen_scipy, seen_ours = [], []

    def f(p):
        seen_scipy.append(np.array(p, copy=True))
        return float(np.sum(p * p))
    approx_derivative(f, x, method="2-point", abs_step=0.025, bounds=([-1.0] * 3, [1.0] * 3), f0=f(x))
    obj = cal.ScipyDifferenceObjective(batch_vols=lambda pts: np.array([[float(np.sqrt(np.sum(p * p)))] for p in pts]), market_vols=np.zeros(1),
                                       weights=np.ones(1), bounds=bounds, eps=0.025, on_point=lambda p: seen_ours.append(np.array(p, copy=True)))
    obj.fun(x)
    obj.jac(x)
    assert len(seen_ours) == len(seen_scipy) == 4
    for a, b in zip(seen_ours, seen_scipy):
        np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(np.signbit(a), np.signbit(b))


def test_difference_steps_fall_back_where_the_step_vanishes():
    """x + eps == x: scipy's relative step sqrt(machine eps) sign(x) max(1, |x|); no bounds: nothing else changes"""
    x = np.array([3e9, -3e9, 0.5, -0.5])
    f = lambda p: float(np.sum(np.sin(p * 1e-9) + p * p))
    obj = cal.ScipyDifferenceObjective(batch_vols=lambda pts: np.array([[f(p)] for p in pts]), market_vols=np.zeros(1), weights=np.ones(1),
                                       bounds=[(None, None)] * 4, eps=1e-8)
    h = cal.scipy_difference_steps(x, 1e-8, [(None, None)] * 4)
    assert h[0] == cal.SLSQP_EPS * 3e9 and h[1] == -cal.SLSQP_EPS * 3e9 and h[2] == 1e-8
    seq_f = lambda p: float(np.nansum(np.ones(1) * np.square(np.array([f(p)]) - np.zeros(1))))
    np.testing.assert_array_equal(obj.jac(x), approx_derivative(seq_f, x, method="2-point", abs_step=1e-8, f0=seq_f(x)))


def test_model_params_driver_equals_the_sequential_fit(stand_in):
    true = HawkesJDParams(sigma=0.4, mean_p=0.04, mean_m=-0.05, theta_p=6.0, theta_m=8.0, kappa_p=25.0, kappa_m=25.0, beta1_p=30.0, beta2_p=-30.0,
                          beta1_m=40.0, beta2_m=-40.0)
    chain = _market(stand_in, true)
    start = HawkesJDParams(sigma=0.45, mean_p=0.03, mean_m=-0.04, theta_p=7.0, theta_m=7.0, kappa_p=22.0, kappa_m=28.0, beta1_p=33.0,
                           beta2_p=-33.0, beta1_m=36.0, beta2_m=-36.0)
    ref, res = seq.calibrate_model_params(HawkesJDPricer(), chain, start, maxiter=60)
    stand_in.calls = 0
    fit, info = HawkesJDPricer().calibrate_model_params_to_chain(chain, start, maxiter=60, return_info=True)
    np.testing.assert_array_equal(info["x"], res.x)
    assert fit == ref and info["fun"] == res.fun and info["nit"] == res.nit and res.nit > 3
    assert info["nb_batches"] == stand_in.calls == seq.batches(res, 8)
    assert HawkesJDPricer().calibrate_model_params_to_chain(chain, start, maxiter=60) == ref       # default return: the fitted parameters


@pytest.mark.parametrize("print_iter", [True, False])
def test_risk_premia_driver_equals_the_sequential_fit_and_prints_the_same_lines(stand_in, capsys, print_iter):
    chain = _market(stand_in, HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5))
    start = HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2)
    ref, res = seq.calibrate_risk_premia_gamma(HawkesJDPricer(), chain, start, print_iter=print_iter)
    expected = capsys.readouterr().out
    stand_in.calls = 0
    fit, info = HawkesJDPricer().calibrate_risk_premia_gamma_to_chain(chain, start, print_iter=print_iter, return_info=True)
    out = capsys.readouterr().out
    np.testing.assert_array_equal(info["x"], res.x)
    assert fit == ref and info["fun"] == res.fun and res.nit > 2
    assert info["nb_batches"] == stand_in.calls == seq.batches(res, 2)
    assert out == expected and (out.count("\n") > 3) == print_iter
