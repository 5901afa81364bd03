"""CPU tests of the Monte Carlo theta (DESIGN.md §3.12) on the numpy oracle ``oracle/mc_theta.py``: its d/d dt tangents against central
differences of its own scheme in dt on fixed normals, its theta rows against common-random-number (CRN) central differences of its own
expected price with ttm_m moved alone and the step count held, and the Python plumbing (rejections before any library call, result layout)."""
import numpy as np
import pytest

from oracle import mc, mc_theta as ot

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
TYPES4 = np.array(["P", "IP", "C", "IC", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)


def _normals(S, n, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((S, n)), rng.standard_normal((S, n))


def _close(a, b, rtol):
    scale = np.max(np.abs(b))
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * scale)


# ---- 1. the d/d dt tangents against central differences of the oracle's own scheme, per path -------------------------------------------
@pytest.mark.parametrize("is_spot", [True, False])
def test_logsv_tangent_matches_dt_central_differences(is_spot):
    S, n, dt = 24, 400, 0.25 / 24
    Z0, Z1 = _normals(S, n, 1)
    x0, s0, q0 = 0.1 * np.ones(n), np.linspace(0.5, 1.5, n), 0.05 * np.ones(n)
    xk, sk, qk, dx, dq = ot.logsv_theta_step_fixed(x0, s0, q0, Z0, Z1, dt, *Q[1:], eta=1.3, is_spot_measure=is_spot)
    # the primal is oracle.mc's scheme
    xr, sr, qr = mc.logsv_step_fixed(x0, s0, q0, Z0, Z1, dt, *Q[1:], eta=1.3, is_spot_measure=is_spot)
    _close(xk, xr, 1e-12)
    _close(sk, sr, 1e-12)
    _close(qk, qr, 1e-12)
    h = 1e-6 * dt
    xp, _, qp, _, _ = ot.logsv_theta_step_fixed(x0, s0, q0, Z0, Z1, dt + h, *Q[1:], eta=1.3, is_spot_measure=is_spot)
    xm, _, qm, _, _ = ot.logsv_theta_step_fixed(x0, s0, q0, Z0, Z1, dt - h, *Q[1:], eta=1.3, is_spot_measure=is_spot)
    assert np.all(np.abs(np.log(sk)) < 50.0)          # no path near the clamp
    _close(dx, (xp - xm) / (2 * h), 1e-7)
    _close(dq, (qp - qm) / (2 * h), 1e-7)


def test_heston_tangent_matches_dt_central_differences():
    S, n, dt = 30, 400, 0.25 / 30
    Z0, Z1 = _normals(S, n, 2)
    x0, v0, q0 = np.zeros(n), np.linspace(0.02, 0.08, n), np.zeros(n)
    h = 1e-6 * dt
    base = ot.heston_theta_step_fixed(x0, v0, q0, Z0, Z1, dt, *HESTON[1:])
    xr, vr, qr = mc.heston_step_fixed(x0, v0, q0, Z0, Z1, dt, *HESTON[1:])
    _close(base[0], xr, 1e-12)
    _close(base[2], qr, 1e-12)
    # leave out the paths on which the floor binds (or nearly does) at some step
    v, vmin = v0.copy(), v0.copy()
    for k in range(S):
        _, v, _ = mc.heston_step_fixed(np.zeros(n), v, np.zeros(n), Z0[k:k + 1], Z1[k:k + 1], dt, *HESTON[1:])
        vmin = np.minimum(vmin, v)
    ok = vmin > 2e-4
    assert ok.sum() > n // 2
    xp, _, qp, _, _ = ot.heston_theta_step_fixed(x0, v0, q0, Z0, Z1, dt + h, *HESTON[1:])
    xm, _, qm, _, _ = ot.heston_theta_step_fixed(x0, v0, q0, Z0, Z1, dt - h, *HESTON[1:])
    _close(base[3][ok], ((xp - xm) / (2 * h))[ok], 1e-7)
    _close(base[4][ok], ((qp - qm) / (2 * h))[ok], 1e-7)


# ---- 2. the theta rows against CRN central differences of the oracle's expected price ----------------------------------------------------
NPY = 100
TTMS = np.array([0.255, 0.51])          # slices of 0.255 years: 25.5 steps -> S = 26, and S stays 26 under a +-1e-3 bump


def _chain_case(model, variable_type, is_spot=True, n=20000, seed=5):
    steps = mc.chain_steps(TTMS, NPY)
    h = 1e-3
    for m in range(len(TTMS)):
        t0 = TTMS[m - 1] if m else 0.0
        assert mc.set_time_grid(TTMS[m] + h - t0, NPY)[0] == mc.set_time_grid(TTMS[m] - h - t0, NPY)[0] == steps[m][0]
    Ss = [S for S, _ in steps]
    rng = np.random.default_rng(seed)
    Z0s = [rng.standard_normal((S, n)) for S in Ss]
    Z1s = [rng.standard_normal((S, n)) for S in Ss]
    fw, df = np.array([1.0, 1.02]), np.array([0.99, 0.97])
    ks = K5 * (HESTON[1] if model == "heston" and variable_type == mc.Q_VAR else 1.0)    # strikes around q/ttm under Q_VAR
    Ks, Ts = [ks, ks], [TYPES4, TYPES4]

    def run(ttms, dts):
        if model == "logsv":
            return ot.logsv_mc_chain_theta_fixed(Q, ttms, fw, df, Ks, Ts, np.array([1.0, 1.2]), Z0s, Z1s, dts, is_spot, variable_type,
                                                 return_states=True)
        return ot.heston_mc_chain_theta_fixed(HESTON, ttms, fw, df, Ks, Ts, Z0s, Z1s, dts, variable_type, return_states=True)

    base = run(TTMS, [dt for _, dt in steps])
    for m in range(len(TTMS)):
        pays = []
        for sgn in (1.0, -1.0):
            ttms = TTMS.copy()
            ttms[m] += sgn * h
            dts = [dt for _, dt in steps]
            dts[m] = (ttms[m] - (ttms[m - 1] if m else 0.0)) / Ss[m]
            pays.append(_path_payoffs(run(ttms, dts)[4][m], ttms[m], fw[m], df[m], variable_type, ks))
        g = -(pays[0] - pays[1]) / (2 * h)
        cd, cd_se = np.nanmean(g, axis=1), np.nanstd(g, axis=1) / np.sqrt(n)
        th, se = base[2][m], base[3][m]
        assert np.all(np.isfinite(th)) and np.all(se > 0)
        np.testing.assert_array_less(np.abs(th - cd), 4.0 * np.sqrt(se ** 2 + cd_se ** 2))


def _path_payoffs(state, ttm, forward, discfactor, variable_type, strikes):
    """discounted per-path payoffs [J, n] of oracle.mc.mc_payoffs, NaN where it skips a path"""
    x, q = state[0], state[2]
    spots = forward * np.exp(x)
    spots = spots - (np.nanmean(spots) - forward)
    under = spots if variable_type == mc.LOG_RETURN else q / ttm
    rows = []
    for k, ty in zip(strikes, TYPES4):
        put = ty in ("P", "IP")
        h = np.where(under < k, k - under, 0.0) if put else np.where(under > k, under - k, 0.0)
        rows.append(discfactor * (h / spots if ty in ("IC", "IP") else h))
    return np.array(rows)


@pytest.mark.parametrize("variable_type", [mc.LOG_RETURN, mc.Q_VAR])
@pytest.mark.parametrize("is_spot", [True, False])
def test_logsv_theta_matches_crn_central_differences(variable_type, is_spot):
    _chain_case("logsv", variable_type, is_spot)


@pytest.mark.parametrize("variable_type", [mc.LOG_RETURN, mc.Q_VAR])
def test_heston_theta_matches_crn_central_differences(variable_type):
    _chain_case("heston", variable_type)


def test_one_step_black_theta():
    """Heston with volvol = 0, kappa = 0 and one step is Black-76 with variance v0 over dt, up to the forward re-centring: its theta row
    is the Black-76 theta of that slice"""
    from scipy.stats import norm
    n, v0 = 400000, 0.04
    rng = np.random.default_rng(11)
    Z0, Z1 = rng.standard_normal((1, n)), rng.standard_normal((1, n))
    ttm = 0.5
    th, se = ot.heston_mc_chain_theta_fixed((v0, v0, 0.0, 0.0, 0.0), np.array([ttm]), np.ones(1), np.ones(1), [K5], [np.array(["C"] * 5)],
                                            [Z0], [Z1], [ttm])[2:4]
    d1 = (-np.log(K5) + 0.5 * v0 * ttm) / np.sqrt(v0 * ttm)
    black_theta = -norm.pdf(d1) * np.sqrt(v0) / (2.0 * np.sqrt(ttm))
    np.testing.assert_array_less(np.abs(th[0] - black_theta), 4.0 * se[0] + 1e-4)


# ---- 3. Python plumbing --------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


def test_with_theta_rejected_before_the_library_on_hawkes(no_library):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[np.array(["C"] * 5)])
    with pytest.raises(NotImplementedError, match="firing clock"):
        HawkesJDPricer().model_mc_chain_greeks(chain, HawkesJDParams(), nb_path=1000, seed=1, with_theta=True)


@pytest.mark.parametrize("model", ["logsv", "heston"])
@pytest.mark.parametrize("with_gamma", [False, True])
def test_theta_outputs_reach_mc_chain_greeks(monkeypatch, model, with_gamma):
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, OptionChain, engine
    chain = OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5[:3]],
                        optiontypes_ttms=[np.array(["C"] * 5), np.array(["P"] * 3)])
    J = 8
    P = len(engine.LOGSV_GREEK_PARAMS if model == "logsv" else engine.HESTON_GREEK_PARAMS)
    offsets = np.array([0, 5, 8], dtype=np.int32)
    calls = []

    def fake(*args, with_gamma=False):
        calls.append(with_gamma)
        flat = lambda: np.arange(J, dtype=float)
        gamma = (10.0 + np.arange(J), 20.0 + np.arange(J)) if with_gamma else (None, None)
        return ([flat()[:5], flat()[5:]], [flat()[:5], flat()[5:]], np.zeros((1 + P, J)), np.zeros((1 + P, J)), offsets, *gamma,
                30.0 + np.arange(J), 40.0 + np.arange(J), None)
    fail = lambda *a, **k: pytest.fail("a route without theta was called")
    if model == "logsv":
        monkeypatch.setattr(engine, "logsv_mc_chain_greeks_theta", fake)
        monkeypatch.setattr(engine, "logsv_mc_chain_greeks_gamma", fail)
        monkeypatch.setattr(engine, "logsv_mc_chain_greeks", fail)
        res = LogSVPricer().model_mc_chain_greeks(chain, LogSvParams(*Q), nb_path=1000, seed=1, with_gamma=with_gamma, with_theta=True)
    else:
        monkeypatch.setattr(engine, "heston_mc_chain_greeks_theta", fake)
        monkeypatch.setattr(engine, "heston_mc_chain_greeks_gamma", fail)
        monkeypatch.setattr(engine, "heston_mc_chain_greeks", fail)
        res = HestonPricer().model_mc_chain_greeks(chain, HestonParams(*HESTON), nb_path=1000, seed=1, with_gamma=with_gamma, with_theta=True)
    assert calls == [with_gamma]
    np.testing.assert_array_equal(res.theta[0], 30.0 + np.arange(5))
    np.testing.assert_array_equal(res.theta_se[1], 45.0 + np.arange(3))
    if with_gamma:
        np.testing.assert_array_equal(res.gamma[1], 15.0 + np.arange(3))
    else:
        assert res.gamma is None and res.gamma_se is None
    assert "theta" in res.params and res.params["theta"][0].shape == (5,)     # d/d theta, not the time row


def test_mc_chain_greeks_theta_defaults_to_none():
    from stochvolmodels_b200.pricers.mc_greeks import McChainGreeks, to_mc_chain_greeks
    import dataclasses
    names = [f.name for f in dataclasses.fields(McChainGreeks)]
    assert names[-2:] == ["theta", "theta_se"]
    offsets = np.array([0, 2], dtype=np.int32)
    out = to_mc_chain_greeks(([np.zeros(2)], [np.zeros(2)], np.zeros((2, 2)), np.zeros((2, 2)), offsets), ["a"])
    assert out.theta is None and out.theta_se is None and out.gamma is None


# ---- 4. rough-LogSV: the h-tangent against central differences of the oracle's own path in h, per path --------------------------------
ROUGH_FACTORS = {1: (np.array([1.0]), np.array([1e-3])),
                 3: (np.array([0.8, 0.45, 0.2]), np.array([0.05, 2.0, 40.0]))}
ROUGH_PARAMS = (0.6, 0.5, 2.0, 2.5, -0.4, 1.2)                 # sigma0, theta, kappa1, kappa2, beta, orthog_vol


@pytest.mark.parametrize("n", [1, 3])
def test_rough_h_tangent_matches_h_central_differences(n):
    from oracle import rough
    w, x = ROUGH_FACTORS[n]
    S, P, h = 40, 300, 0.25 / 40
    Z0, Z1 = _normals(S, P, 7 + n)
    ls, v, y, dls, dy, reset = ot.rough_theta_path(x, w, *ROUGH_PARAMS, S, h, Z0, Z1)
    # the primal is oracle.rough's path
    grid = np.linspace(0.0, S * h, S + 1)
    vt = np.sqrt(ROUGH_PARAMS[4] ** 2 + ROUGH_PARAMS[5] ** 2)
    v0 = np.full((n, P), ROUGH_PARAMS[0] / np.sum(w))
    ls_r, _, y_r = rough.log_spot_full_combined(np.repeat(x[:, None], P, axis=1), np.repeat(w[:, None], P, axis=1), v0, *ROUGH_PARAMS[1:4], 0.0,
                                                v0.copy(), ROUGH_PARAMS[4] / vt, vt, grid, Z0, Z1)
    np.testing.assert_array_equal(ls, ls_r[0])
    np.testing.assert_array_equal(y, y_r[0])
    eps = 1e-6 * h
    up = ot.rough_theta_path(x, w, *ROUGH_PARAMS, S, h + eps, Z0, Z1)
    dn = ot.rough_theta_path(x, w, *ROUGH_PARAMS, S, h - eps, Z0, Z1)
    ok = ~(reset | up[5] | dn[5])
    assert ok.sum() > P // 2
    _close(dls[ok], ((up[0] - dn[0]) / (2 * eps))[ok], 1e-7)
    _close(dy[ok], ((up[2] - dn[2]) / (2 * eps))[ok], 1e-7)


def test_rough_theta_rows_match_crn_central_differences():
    """all ttms moved at once (every maturity restarts at t = 0 on its own grid, so the rows do not interact), step counts held"""
    from oracle import rough
    w, x = ROUGH_FACTORS[3]
    ttms, npy, dT, n = np.array([0.255, 0.505]), 100, 1e-3, 20000
    nsteps = [mc.set_time_grid(t, npy)[0] for t in ttms]
    for t, S in zip(ttms, nsteps):
        assert mc.set_time_grid(t + dT, npy)[0] == mc.set_time_grid(t - dT, npy)[0] == S
    rng = np.random.default_rng(21)
    Z0, Z1 = rng.standard_normal((max(nsteps), n)), rng.standard_normal((max(nsteps), n))
    fw, df = np.array([1.0, 1.02]), np.array([0.99, 0.97])
    Ks, Ts = [K5, K5], [TYPES4, TYPES4]
    th, se, _ = ot.rough_chain_theta_fixed(ttms, fw, df, Ks, Ts, Z0, Z1, *ROUGH_PARAMS, w, x, nsteps, ttms / nsteps)
    pays = []
    for sgn in (1.0, -1.0):
        t = ttms + sgn * dT
        grids = [np.linspace(0.0, tm, S + 1) for tm, S in zip(t, nsteps)]
        states = rough.rough_chain_fixed(t, fw, df, Ks, Ts, Z0, Z1, *ROUGH_PARAMS, w, x, grids, return_states=True)[2]
        pays.append([_path_payoffs((st[0][0], None, st[2][0]), tm, fw[m], df[m], mc.LOG_RETURN, K5) for m, (st, tm) in enumerate(zip(states, t))])
    for m in range(2):
        g = -(pays[0][m] - pays[1][m]) / (2 * dT)
        cd, cd_se = np.nanmean(g, axis=1), np.nanstd(g, axis=1) / np.sqrt(n)
        np.testing.assert_array_less(np.abs(th[m] - cd), 4.0 * np.sqrt(se[m] ** 2 + cd_se[m] ** 2))
