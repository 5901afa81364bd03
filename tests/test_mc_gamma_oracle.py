"""CPU: the Monte Carlo gamma by conditional smoothing of the last step (oracle/mc_gamma.py, DESIGN.md §3.9).

  estimator  -- the oracle's gamma against common-random-number second differences of the oracle's own price in the forward, LogSV in
                both measures and Heston, C / P / IC / IP; a one-step slice against the closed-form Black-76 gamma; the Q_VAR rows
  interface  -- the routes without a Monte Carlo gamma reject with_gamma=True before any library call; the gamma outputs of the engine
                reach McChainGreeks
"""
import numpy as np
import pytest
from scipy.stats import norm

from oracle import mc, mc_gamma as og

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T_ALL = np.array(["P", "IP", "C", "IC", "C", "IC", "P", "IP"])
K_ALL = np.array([0.85, 0.9, 0.95, 1.0, 1.05, 1.1, 1.0, 1.15])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                    # quickstart LogSV parameters
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)


def _pays(x, forward, strikes, types):
    """per-path payoffs of oracle.mc.mc_payoffs (LOG_RETURN) at forward F: [J, N]"""
    fe = forward * np.exp(x)
    spots = fe - (np.nanmean(fe) - forward)
    out = []
    for k, ty in zip(strikes, types):
        put = ty in ("P", "IP")
        h = np.where(spots < k, k - spots, 0.0) if put else np.where(spots > k, spots - k, 0.0)
        out.append(h / spots if ty in ("IC", "IP") else h)
    return np.array(out)


def _logsv_draws(n, ttm, npy, seed):
    S, dt = mc.set_time_grid(ttm, npy)
    rng = np.random.default_rng(seed)
    return rng.standard_normal((S, n)), rng.standard_normal((S, n)), dt


def _crn_gate(x, g, g_se, forward, discfactor, h, what, strikes=K_ALL):
    """|gamma - CRN second difference| <= 4 combined SE; the second difference over +-h relative bumps of the forward with the same paths"""
    F = forward
    pays = [_pays(x, F * f, strikes, T_ALL) for f in (1 + h, 1.0, 1 - h)]
    d2 = (pays[0] - 2 * pays[1] + pays[2]) / (F * h) ** 2
    crn = discfactor * d2.mean(axis=1)
    crn_se = discfactor * d2.std(axis=1) / np.sqrt(x.shape[0])
    np.testing.assert_allclose(discfactor * pays[1].mean(axis=1), mc.mc_payoffs(x, x, 1.0, F, strikes, T_ALL, discfactor)[0], rtol=1e-12)
    z = np.abs(g - crn) / np.sqrt(g_se ** 2 + crn_se ** 2)
    assert np.all(z <= 4.0), (what, g, crn, z)
    # the smoothing pays: the gamma's own SE is below the bump's at the same paths
    assert np.all(g_se < crn_se), (what, g_se, crn_se)


@pytest.mark.parametrize("is_spot,eta", [(True, 1.0), (False, 0.9)])
def test_logsv_gamma_matches_crn_second_differences(is_spot, eta):
    n, ttm, npy, F, df = 200_000, 0.25, 256, 1.0, 0.97
    Z0, Z1, dt = _logsv_draws(n, ttm, npy, 11 + int(is_spot))
    p, e, g, ge, st = og.logsv_mc_chain_gamma_fixed(Q, [ttm], [F], [df], [K_ALL], [T_ALL], [eta], [Z0], [Z1], [dt], is_spot,
                                                   return_states=True)
    x = st[0][0]
    pr, er = mc.logsv_mc_chain_fixed(Q, [ttm], [F], [df], [K_ALL], [T_ALL], [eta], [Z0], [Z1], [dt], is_spot)
    np.testing.assert_array_equal(p[0], pr[0])                     # the gamma chain prices what the price chain prices
    np.testing.assert_allclose(st[0][4] + st[0][3] * Z0[-1], x, rtol=0, atol=1e-14)
    _crn_gate(x, g[0], ge[0], F, df, 0.01, ("logsv", is_spot))


def test_heston_gamma_matches_crn_second_differences():
    n, ttm, npy, F, df = 200_000, 0.5, 360, 1.3, 1.0
    Z0, Z1, dt = _logsv_draws(n, ttm, npy, 5)
    p, e, g, ge, st = og.heston_mc_chain_gamma_fixed(HESTON, [ttm], [F], [df], [K_ALL * F], [T_ALL], [Z0], [Z1], [dt], return_states=True)
    _crn_gate(st[0][0], g[0], ge[0], F, df, 0.01, "heston", K_ALL * F)


def test_heston_gamma_crn_multi_slice():
    """second maturity of a two-slice chain: the last step and the re-centring are those of the slice being priced"""
    n, npy, F = 200_000, 360, 1.0
    ttms = [0.1, 0.3]
    steps = mc.chain_steps(ttms, npy)
    rng = np.random.default_rng(8)
    Z0s = [rng.standard_normal((S, n)) for S, _ in steps]
    Z1s = [rng.standard_normal((S, n)) for S, _ in steps]
    p, e, g, ge, st = og.heston_mc_chain_gamma_fixed(HESTON, ttms, [F, F], [1.0, 1.0], [K_ALL, K_ALL], [T_ALL, T_ALL], Z0s, Z1s,
                                                     [dt for _, dt in steps], return_states=True)
    _crn_gate(st[1][0], g[1], ge[1], F, 1.0, 0.01, "heston slice 2")


def _black_gamma(F, K, vol_t):
    d1 = (np.log(F / K) + 0.5 * vol_t ** 2) / vol_t
    return norm.pdf(d1) / (F * vol_t)


def test_one_step_slice_gives_black76_gamma():
    """one LogSV step under the spot measure is lognormal with vol sigma0 sqrt(T): the smoothed gamma of C and P is Black-76's gamma at
    the strike shifted by the re-centring correction; the tolerance is that shift's first-order effect (O(F sigma sqrt(T) / sqrt(n)))"""
    n, ttm, sigma0, F = 400_000, 0.25, 0.3, 1.0
    params = (sigma0, 0.3, 2.0, 0.0, 0.0, 0.0)           # no vol-of-vol: the vol path does not matter for one step anyway
    S, dt = mc.set_time_grid(ttm, 1)
    assert S == 1
    rng = np.random.default_rng(3)
    Z0, Z1 = rng.standard_normal((1, n)), rng.standard_normal((1, n))
    types = np.array(["C", "P"] * 3)
    strikes = np.repeat([0.85, 1.0, 1.2], 2)
    p, e, g, ge, st = og.logsv_mc_chain_gamma_fixed(params, [ttm], [F], [1.0], [strikes], [types], [1.0], [Z0], [Z1], [dt], True,
                                                   return_states=True)
    x = st[0][0]
    corr = np.mean(F * np.exp(x)) - F
    vol_t = sigma0 * np.sqrt(ttm)
    ref = _black_gamma(F, strikes, vol_t)
    dref_dk = (_black_gamma(F, strikes + 1e-5, vol_t) - _black_gamma(F, strikes - 1e-5, vol_t)) / 2e-5
    tol = 3.0 * abs(corr) * np.abs(dref_dk) + 1e-4 * ref
    assert np.all(np.abs(g[0] - ref) <= tol), (g[0], ref, tol)
    np.testing.assert_array_equal(g[0][0::2], g[0][1::2])           # C and P: the same per-path term
    assert np.all(ge[0] < 1e-2 * ref)                                # one step: the smoothed term is nearly deterministic


def test_q_var_rows():
    n, ttm, npy, F, df = 20_000, 0.25, 128, 1.1, 0.95
    Z0, Z1, dt = _logsv_draws(n, ttm, npy, 4)
    K = np.array([0.8, 0.8, 0.8, 0.8, 1.2, 1.2])
    T = np.array(["C", "P", "IC", "IP", "IC", "IP"])
    p, e, g, ge = og.logsv_mc_chain_gamma_fixed(Q, [ttm], [F], [df], [K], [T], [1.0], [Z0], [Z1], [dt], True, variable_type=mc.Q_VAR)
    assert np.all(g[0][:2] == 0.0) and np.all(ge[0][:2] == 0.0)
    np.testing.assert_allclose(g[0][2:], 2.0 * p[0][2:] / F ** 2, rtol=1e-13)
    np.testing.assert_allclose(ge[0][2:], 2.0 * e[0][2:] / F ** 2, rtol=1e-12)
    assert np.all(g[0][2:] > 0.0)


@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


def test_with_gamma_rejected_before_the_library_on_hawkes_and_rough(no_library):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[np.array(["C"] * 5)])
    with pytest.raises(NotImplementedError, match="with_gamma"):
        HawkesJDPricer().model_mc_chain_greeks(chain, HawkesJDParams(), nb_path=1000, seed=1, with_gamma=True)
    with pytest.raises(NotImplementedError, match="with_gamma"):
        LogSVPricer().rough_mc_chain_greeks(chain, LogSvParams(*Q), nb_path=1000, nb_steps=100, seed=1, gauss="fp64", with_gamma=True)


def test_gamma_outputs_reach_mc_chain_greeks(monkeypatch):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, engine
    chain = OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5[:3]],
                        optiontypes_ttms=[np.array(["C"] * 5), np.array(["P"] * 3)])
    J, P = 8, len(engine.LOGSV_GREEK_PARAMS)
    offsets = np.array([0, 5, 8], dtype=np.int32)
    calls = []

    def fake(*args):
        calls.append(args)
        flat = lambda: np.arange(J, dtype=float)
        return ([flat()[:5], flat()[5:]], [flat()[:5], flat()[5:]], np.zeros((1 + P, J)), np.zeros((1 + P, J)), offsets,
                10.0 + np.arange(J), 20.0 + np.arange(J), None)
    monkeypatch.setattr(engine, "logsv_mc_chain_greeks_gamma", fake)
    monkeypatch.setattr(engine, "logsv_mc_chain_greeks", lambda *a: pytest.fail("the greeks route without gamma was called"))
    res = LogSVPricer().model_mc_chain_greeks(chain, LogSvParams(*Q), nb_path=1000, seed=1, with_gamma=True)
    assert len(calls) == 1
    np.testing.assert_array_equal(res.gamma[0], 10.0 + np.arange(5))
    np.testing.assert_array_equal(res.gamma_se[1], 25.0 + np.arange(3))
