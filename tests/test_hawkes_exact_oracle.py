"""The exact event-driven route of the Hawkes jump-diffusion Monte Carlo (DESIGN.md §3.13) without a GPU: its numpy restatement
(oracle/hawkes_exact.py) against the closed forms of the linear mean equations, the martingale condition and the reference's own Fourier
prices, the degenerate no-event case, the expected-event bound, and what the public API and the C entry points reject before any device
work."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes, hawkes_exact

KEYS = hawkes.KEYS


def _param_sets():
    from stochvolmodels_b200 import HawkesJDParams
    g = load_golden("hawkes_mc.npz")
    d = HawkesJDParams().to_dict()
    d.pop("risk_premia_gamma")
    return {"defaults": d, "mc_dflt": dict(zip(KEYS, g["dflt_params"])), "mc_drift": dict(zip(KEYS, g["drift_params"]))}


@pytest.mark.parametrize("name", ["defaults", "mc_dflt", "mc_drift"])
def test_oracle_agrees_with_the_mean_equations_and_the_martingale_condition(name):
    """1e5 paths over two carried intervals (0.12, then 0.18): E[lambda(T)], the expected event counts of each clock and E[e^x_T] = e^(mu T)
    within 4 SE of the closed forms at T = 0.3"""
    p = _param_sets()[name]
    n, seed = 100_000, 11
    ids = np.arange(n, dtype=np.uint64)
    x, lp, lm, ev0 = hawkes_exact.interval(np.zeros(n), np.full(n, p["lambda_p"]), np.full(n, p["lambda_m"]), 0.12, p, seed, 0, ids)
    x, lp, lm, ev1 = hawkes_exact.interval(x, lp, lm, 0.3 - 0.12, p, seed, 1, ids)
    ref = hawkes_exact.mean_equations(p, 0.3)
    for est, want in ((lp, ref[0]), (lm, ref[1]), (ev0[0] + ev1[0], ref[2]), (ev0[1] + ev1[1], ref[3]), (np.exp(x), np.exp(p["mu"] * 0.3))):
        assert abs(est.mean() - want) < 4.0 * est.std() / np.sqrt(n), (name, est.mean(), want)
    assert np.all(ev0[2] >= ev0[0] + ev0[1]) and ev0[0].sum() > 0 and ev0[1].sum() > 0


def _negative_kappa_sets():
    """kappa < 0: the intensities grow away from theta between events, so the thinning bound must look ahead to the interval end"""
    d = _param_sets()["defaults"]
    free = {**d, "beta1_p": 0.0, "beta2_p": 0.0, "beta1_m": 0.0, "beta2_m": 0.0, "lambda_p": 20.0, "lambda_m": 20.0, "theta_p": 5.0,
            "theta_m": 5.0, "kappa_p": -4.0, "kappa_m": -4.0}
    return {"no_excitation": free, "excited_kappa_p": {**d, "kappa_p": -4.0}}


@pytest.mark.parametrize("name", ["no_excitation", "excited_kappa_p"])
def test_oracle_at_negative_kappa_agrees_with_the_mean_equations(name):
    """kappa < 0 (lambda0 >= theta, so the intensities stay non-negative and the mean equations are exact): E[lambda(T)], the expected
    event counts and E[e^x_T] = e^(mu T) within 4 SE at 1e5 paths.  A bound that ignored the growth away from theta would lose events
    while charging their compensator in full: -110 SE on the '-' count and +36 SE on E[e^x] in the no-excitation case."""
    p = _negative_kappa_sets()[name]
    n, T = 100_000, 0.5
    x, lp, lm, ev = hawkes_exact.terminal(p, T, n, seed=7)
    ref = hawkes_exact.mean_equations(p, T)
    for est, want in ((lp, ref[0]), (lm, ref[1]), (ev[0], ref[2]), (ev[1], ref[3]), (np.exp(x), np.exp(p["mu"] * T))):
        assert abs(est.mean() - want) < 4.0 * est.std() / np.sqrt(n) + 1e-12 * abs(want), (name, est.mean(), want)
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import hawkes_expected_events_bound
    bound = hawkes_expected_events_bound(T, **p)
    assert ref[2] + ref[3] <= bound, (ref[2] + ref[3], bound)


@pytest.mark.parametrize("name", ["dflt", "alt"])
def test_oracle_prices_the_reference_fourier_chain_without_an_allowance(name):
    """the reference's own Fourier prices (hawkes_fourier.npz, three carried maturities) within 4 SE of the exact route at 1e5 paths, with no
    additive allowance.  The Fourier route does not read mu; the Monte Carlo payoffs re-centre the spots on the forward additively
    (utils/mc_payoffs.py), which a drift e^(mu T) != 1 then shifts, so the comparison runs at mu = 0 (the 'alt' set has mu = 0.05)."""
    g = load_golden("hawkes_fourier.npz")
    p = {**dict(zip(KEYS, g[f"{name}_params"])), "mu": 0.0}
    K, T, ttms, fw, df = g["strikes"], g["types"], g["ttms"], g["forwards"], g["discfactors"]
    prices, stds, _, _ = hawkes_exact.chain(p, ttms, fw, df, [K * f for f in fw], [T] * 3, 100_000, seed=3)
    for m in range(3):
        z = (prices[m] - g[f"{name}_prices"][m]) / stds[m]
        assert np.all(np.abs(z) < 4.0), (name, m, z)


def test_no_events_when_both_intensities_vanish():
    """lambda0 = theta = 0 on both clocks: no candidate is ever drawn, the intensities stay 0 and x_T = (mu - sigma^2/2) T + sigma sqrt(T) z
    on every path, z the interval's normal"""
    p = {**_param_sets()["mc_drift"], "lambda_p": 0.0, "theta_p": 0.0, "lambda_m": 0.0, "theta_m": 0.0}
    n, T, seed = 5000, 0.37, 5
    x, lp, lm, ev = hawkes_exact.terminal(p, T, n, seed, slice_idx=2, path0=123)
    z = hawkes_exact.normals(seed, np.arange(123, 123 + n, dtype=np.uint64), 2)
    np.testing.assert_allclose(x, (p["mu"] - 0.5 * p["sigma"] ** 2) * T + p["sigma"] * np.sqrt(T) * z, rtol=1e-15, atol=1e-16)
    assert not ev.any() and not lp.any() and not lm.any()
    assert abs(z.mean()) < 4 / np.sqrt(n) and abs(z.var() - 1) < 4 * np.sqrt(2 / n)


def test_oracle_budget_and_candidate_counts():
    """a budget below the candidates a path needs raises; the budget the paths need does not"""
    p = _param_sets()["defaults"]
    x, lp, lm, ev = hawkes_exact.terminal(p, 0.2, 500, seed=9)
    need = int(ev[2].max())
    hawkes_exact.terminal(p, 0.2, 500, seed=9, budget=need)
    with pytest.raises(hawkes_exact.BudgetExhausted):
        hawkes_exact.terminal(p, 0.2, 500, seed=9, budget=need - 1)


@pytest.mark.parametrize("name", ["defaults", "mc_drift"])
def test_expected_event_bound_dominates_the_mean_equations(name):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import HAWKES_EXACT_MAX_EXPECTED_EVENTS, hawkes_expected_events_bound
    p = _param_sets()[name]
    for T in (0.05, 0.5, 2.0):
        exact = sum(hawkes_exact.mean_equations(p, T)[2:])
        bound = hawkes_expected_events_bound(T, **p)
        assert exact <= bound * (1 + 1e-12) < HAWKES_EXACT_MAX_EXPECTED_EVENTS, (T, exact, bound)
    # kappa = 0: the bound stays finite and is the linear growth lambda0 T without excitation
    assert hawkes_expected_events_bound(1.5, **{**p, "kappa_p": 0.0, "kappa_m": 0.0, "beta1_p": 0.0, "beta2_p": 0.0, "beta1_m": 0.0,
                                                  "beta2_m": 0.0}) == pytest.approx(1.5 * (abs(p["lambda_p"]) + abs(p["lambda_m"])), rel=1e-13)


# ---- rejections before any library call ---------------------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


def _chain():
    from stochvolmodels_b200 import OptionChain
    return OptionChain(ttms=np.array([0.1, 0.25]), forwards=np.ones(2), strikes_ttms=[np.array([0.9, 1.1])] * 2,
                       optiontypes_ttms=[np.array(["P", "C"])] * 2)


RUNAWAY = dict(kappa_p=1.0, beta1_p=400.0, kappa_m=1.0, beta1_m=400.0)      # branching far above 1: the event bound explodes


def test_public_api_rejections_before_any_library_call(no_library):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import hawkesjd_mc_chain_pricer, simulate_hawkesjd_terminal
    pricer, params, chain = HawkesJDPricer(), HawkesJDParams(), _chain()
    for scheme in ("Exact", "qe", None):
        with pytest.raises(ValueError, match="scheme must be"):
            pricer.model_mc_price_chain(chain, params, nb_path=1000, seed=1, scheme=scheme)
        with pytest.raises(ValueError, match="scheme must be"):
            pricer.simulate_terminal_values(params, ttm=0.1, nb_path=1000, seed=1, scheme=scheme)
        with pytest.raises(ValueError, match="scheme must be"):
            pricer.model_mc_chain_greeks(chain, params, nb_path=1000, seed=1, scheme=scheme)
    with pytest.raises(NotImplementedError, match="exact route has no sensitivities"):
        pricer.model_mc_chain_greeks(chain, params, nb_path=1000, seed=1, scheme="exact")
    d = params.to_dict()
    d.pop("risk_premia_gamma")
    kw = {k: v for k, v in d.items() if k not in ("lambda_p", "lambda_m")}
    S = 181          # 0.1 years at 1800 steps per year
    inputs = [np.zeros((S, 4))] * 5
    with pytest.raises(ValueError, match="cannot be combined with scheme='exact'"):
        simulate_hawkesjd_terminal(0.1, np.zeros(1), np.full(1, params.lambda_p), np.full(1, params.lambda_m), nb_path=4, inputs=inputs,
                                   scheme="exact", **kw)
    with pytest.raises(ValueError, match="scheme must be"):
        hawkesjd_mc_chain_pricer(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms, nb_path=100,
                                 seed=1, scheme="EULER", **d)
    runaway = HawkesJDParams(**{**d, **RUNAWAY})
    with pytest.raises(ValueError, match="expected events per path"):
        pricer.model_mc_price_chain(chain, runaway, nb_path=1000, seed=1, scheme="exact")
    with pytest.raises(ValueError, match="expected events per path"):
        pricer.simulate_terminal_values(runaway, ttm=0.25, nb_path=1000, seed=1, scheme="exact")


# ---- C entry points: argument defects before any device work --------------------------------------------------------------------
def _c_chain_args(**over):
    import ctypes
    from stochvolmodels_b200 import _capi as C
    a = dict(params=ctypes.byref(C.HawkesParamsC(0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, -0.5, 1.0, 1.0, 2.0, 0.5, -0.5)), M=1,
             ttms=np.array([0.1]), forwards=np.ones(1), discfactors=np.ones(1), offsets=np.array([0, 1], dtype=np.int32), strikes=np.ones(1),
             types=np.zeros(1, dtype=np.int8), nb_path=100, vt=C.LOG_RETURN, seed=1, flags=0, prices=np.zeros(1), stds=np.zeros(1), budget=0,
             n_out=0, states=None, events=None)
    a.update(over)
    ptr = lambda v: None if v is None else (C.iptr(v) if v.dtype == np.int32 else C.i8ptr(v) if v.dtype == np.int8 else C.dptr(v))
    return [a["params"], a["M"], *(ptr(a[k]) for k in ("ttms", "forwards", "discfactors", "offsets", "strikes", "types")), a["nb_path"], a["vt"],
            a["seed"], a["flags"], ptr(a["prices"]), ptr(a["stds"]), a["budget"], a["n_out"], ptr(a["states"]), ptr(a["events"])]


@pytest.mark.parametrize("over, want", [
    (dict(prices=None), "null pointer"),
    (dict(ttms=None), "null pointer"),
    (dict(nb_path=0), "nb_path must be >= 1"),
    (dict(n_out=101), "n_paths_out must be in [0, nb_path]"),
    (dict(n_out=-1), "n_paths_out must be in [0, nb_path]"),
    (dict(flags=1), "the Hawkes route is float64 only"),
    (dict(ttms=np.array([-0.1])), "ttms must be positive"),
])
def test_chain_exact_argument_defects(over, want):
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    rc = lib.b200sv_hawkesjd_mc_chain_exact(*_c_chain_args(**over))
    assert rc == -1 and want in lib.b200sv_last_error().decode()


def test_terminal_and_device_slice_exact_argument_defects():
    import ctypes
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    kp = ctypes.byref(C.HawkesParamsC(*([0.1] * 16)))
    x = np.zeros(4)
    cases = [
        (lambda: lib.b200sv_hawkesjd_terminal_exact(kp, 0.1, 4, 1, 0, 0, 0, 0, None, C.dptr(x), C.dptr(x)), "null pointer"),
        (lambda: lib.b200sv_hawkesjd_terminal_exact(kp, 0.0, 4, 1, 0, 0, 0, 0, C.dptr(x), C.dptr(x), C.dptr(x)), "nb_path, ttm must be positive"),
        (lambda: lib.b200sv_hawkesjd_terminal_exact(kp, 0.1, 0, 1, 0, 0, 0, 0, C.dptr(x), C.dptr(x), C.dptr(x)), "nb_path, ttm must be positive"),
        (lambda: lib.b200sv_hawkesjd_terminal_exact(kp, 0.1, 4, 1, C.STATE_F32, 0, 0, 0, C.dptr(x), C.dptr(x), C.dptr(x)), "float64 only"),
        (lambda: lib.b200sv_dev_hawkesjd_exact_slice(1, 1, 1, 4, 0, 1, kp, 0.1, 0, 1.0, 1, 0, None, 1, None, None), "null pointer"),
        (lambda: lib.b200sv_dev_hawkesjd_exact_slice(1, 1, 1, 4, 0, 1, kp, -0.1, 0, 1.0, 1, 0, 1, 1, None, None), "n_local and tau must be positive"),
        (lambda: lib.b200sv_dev_hawkesjd_exact_slice(1, 1, 1, 0, 0, 1, kp, 0.1, 0, 1.0, 1, 0, 1, 1, None, None), "n_local and tau must be positive"),
    ]
    for call, want in cases:
        rc = call()
        assert rc == -1 and want in lib.b200sv_last_error().decode(), (rc, want)
