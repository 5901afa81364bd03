"""Monte Carlo sensitivities of the Hawkes jump-diffusion chain (HawkesJDPricer.model_mc_chain_greeks, DESIGN.md §3.11) on the GPU:
prices bit for bit against the pricing route, the per-path state, tangents and scores against the numpy oracle (oracle/hawkes_mc_greeks.py)
fed with the draws the kernel exports, every row against CRN central differences of the GPU route itself, and every row against the exact
Fourier sensitivities of the same model (HawkesJDPricer.price_chain_greeks)."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes
from oracle import hawkes_mc_greeks as hg

pytestmark = pytest.mark.gpu


def _golden_chain():
    from stochvolmodels_b200 import HawkesJDParams, OptionChain
    g = load_golden("hawkes_mc.npz")
    params = HawkesJDParams(**dict(zip(hawkes.KEYS, g["chain_params"])))
    M = g["chain_ttms"].shape[0]
    types = np.array(["P", "IP", "C", "IC", "C"])
    chain = OptionChain(ttms=g["chain_ttms"], forwards=g["chain_forwards"], discfactors=g["chain_discfactors"],
                        strikes_ttms=[g["chain_strikes"] * f for f in g["chain_forwards"]], optiontypes_ttms=[types] * M)
    return params, chain


@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
def test_prices_bit_identical_to_the_pricing_route_and_runs_reproducible(cuda_lib, gauss):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, get_btc_test_chain_data
    chain, params, pricer = get_btc_test_chain_data(), HawkesJDParams(), HawkesJDPricer()
    kw = dict(nb_path=200_003, seed=29, gauss=gauss)
    res = pricer.model_mc_chain_greeks(chain, params, **kw)
    p, e = pricer.model_mc_price_chain(chain, params, **kw)
    again = pricer.model_mc_chain_greeks(chain, params, **kw)
    assert len(res.prices) == len(chain.ttms) == 4
    for m in range(len(p)):
        np.testing.assert_array_equal(res.prices[m], p[m])
        np.testing.assert_array_equal(res.std_errors[m], e[m])
        np.testing.assert_array_equal(again.delta[m], res.delta[m])
        np.testing.assert_array_equal(again.delta_se[m], res.delta_se[m])
        for name in hg.PARAMS:
            np.testing.assert_array_equal(again.params[name][m], res.params[name][m])
            np.testing.assert_array_equal(again.params_se[name][m], res.params_se[name][m])
            assert np.all(np.isfinite(res.params[name][m])) and np.all(res.params_se[name][m] > 0.0)
    assert set(res.params) == set(hg.PARAMS)


@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
def test_per_path_tangents_and_scores_match_the_oracle_on_the_kernel_draws(cuda_lib, gauss):
    """the first paths of a two-maturity chain: state, dx, dlambda_p, dlambda_m and score after each maturity == the oracle on the draws
    b200sv_hawkesjd_device_draws exports (same paths, Philox sub-stream m per maturity), up to FMA contraction"""
    from stochvolmodels_b200 import HawkesJDParams, engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c, hawkesjd_device_draws
    p = HawkesJDParams(mu=0.02, sigma=0.4, lambda_p=20.0, lambda_m=25.0, theta_p=15.0, theta_m=18.0)
    d = {k: v for k, v in p.to_dict().items() if k in hawkes.KEYS}
    N, n_out, seed = 5000, 3000, 77
    ttms, fw, df = np.array([0.04, 0.1]), np.array([1.0, 1.01]), np.array([0.999, 0.99])
    K = np.array([0.9, 1.0, 1.1])
    T = np.array(["P", "C", "IC"])
    res = engine.hawkesjd_mc_chain_greeks(_params_c(**d), ttms, fw, df, [K, K], [T, T], N, 1, seed, engine.mc_flags("fp64", gauss), n_out)
    states, tangents = res[5], res[6]
    inputs, t0 = [], 0.0
    for m, ttm in enumerate(ttms):
        inputs.append(hawkesjd_device_draws(seed, 0, n_out, m, ttm - t0, gauss=gauss, **d))
        t0 = ttm
    x, lp, lm = np.zeros(n_out), p.lambda_p * np.ones(n_out), p.lambda_m * np.ones(n_out)
    dx, dlp, dlm, sc = hg.initial_tangents(n_out)
    kw = {k: v for k, v in d.items() if k not in ("lambda_p", "lambda_m")}
    fired = np.zeros((2, n_out), dtype=int)
    together = 0
    for m in range(2):
        x, lp, lm, dx, dlp, dlm, sc, fires = hg.tangent_step_fixed(x, lp, lm, dx, dlp, dlm, sc, *inputs[m], return_fires=True, **kw)
        fired += fires.sum(axis=0)
        together += int(np.sum(fires[:, 0] & fires[:, 1]))
        for a, b, what in zip(states[m], (x, lp, lm), ("x", "lambda_p", "lambda_m")):
            np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-10 * np.max(np.abs(b)), err_msg=what)
        for c, ref, what in zip(tangents[m], (dx, dlp, dlm, sc), ("dx", "dlambda_p", "dlambda_m", "score")):
            for q, name in enumerate(hg.PARAMS):
                scale = max(float(np.max(np.abs(ref[q]))), 1e-300)
                assert np.max(np.abs(c[q] - ref[q])) <= 1e-10 * scale, (what, name, m, np.max(np.abs(c[q] - ref[q])) / scale)
    both = fired.sum(axis=0)
    assert np.any(fired.min(axis=0) >= 1) and np.sum(both == 1) > 100 and np.sum(both >= 2) > 100, "single and repeated firings covered"
    assert together >= 5, ("steps where both clocks fire (hawkes_two_sizes, all four jump loads at once)", together)


def _terminal_x(params, chain, N, seed, gauss):
    """per-path terminal log-returns of every maturity on the pricing route's stream (slice m continues slice m - 1)"""
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import simulate_hawkesjd_terminal
    d = {k: v for k, v in params.items() if k in hawkes.KEYS and k not in ("lambda_p", "lambda_m")}
    x, lp, lm, t0, out = np.zeros(1), np.array([params["lambda_p"]]), np.array([params["lambda_m"]]), 0.0, []
    for m, ttm in enumerate(chain.ttms):
        x, lp, lm = simulate_hawkesjd_terminal(ttm=ttm - t0, x0=x, lambda_p0=lp, lambda_m0=lm, nb_path=N, seed=seed, gauss=gauss, slice_index=m, **d)
        x, lp, lm = x.copy(), lp.copy(), lm.copy()
        out.append(x)
        t0 = ttm
    return out


def _per_path_payoffs(x, fwd, df, strikes, types):
    fe = fwd * np.exp(x)
    s = fe - (np.mean(fe) - fwd)
    cols = []
    for k, ty in zip(strikes, types):
        h = np.maximum(k - s, 0.0) if ty in ("P", "IP") else np.maximum(s - k, 0.0)
        cols.append(df * (h / s if ty in ("IC", "IP") else h))
    return np.array(cols)


def test_every_row_matches_crn_central_differences_of_the_gpu_route(cuda_lib):
    """hawkes_mc.npz chain parameters, 1e6 paths: delta and all 15 rows against central differences of the GPU route's own per-path payoffs
    at bumped parameters on the same seed (the terminal states come from the pricing kernel); within 4 combined standard errors, the
    difference's SE from its per-path values"""
    from stochvolmodels_b200 import HawkesJDPricer
    params, chain = _golden_chain()
    N, seed, gauss = 1_000_000, 41, "fp32"
    res = HawkesJDPricer().model_mc_chain_greeks(chain, params, nb_path=N, seed=seed, gauss=gauss)
    base = params.to_dict()
    xs = _terminal_x(base, chain, N, seed, gauss)
    M = len(chain.ttms)

    def check(row, se, fd_paths, what):
        fd, fd_se = fd_paths.mean(axis=1), fd_paths.std(axis=1) / np.sqrt(N)
        z = np.abs(row - fd) / np.sqrt(se ** 2 + fd_se ** 2)
        assert np.all(z < 4.0), (what, row, fd, se, fd_se)

    hf = 1e-4
    for m in range(M):
        f, df, K, T = chain.forwards[m], chain.discfactors[m], chain.strikes_ttms[m], chain.optiontypes_ttms[m]
        pay = _per_path_payoffs(xs[m], f, df, K, T)
        np.testing.assert_allclose(pay.mean(axis=1), res.prices[m], rtol=1e-10)
        up, dn = _per_path_payoffs(xs[m], f * (1 + hf), df, K, T), _per_path_payoffs(xs[m], f * (1 - hf), df, K, T)
        check(res.delta[m], res.delta_se[m], (up - dn) / (2 * hf * f), ("delta", m))
    for name in hg.PARAMS:
        h = 0.01 * max(abs(base[name]), 0.05)
        xu = _terminal_x({**base, name: base[name] + h}, chain, N, seed, gauss)
        xd = _terminal_x({**base, name: base[name] - h}, chain, N, seed, gauss)
        for m in range(M):
            f, df, K, T = chain.forwards[m], chain.discfactors[m], chain.strikes_ttms[m], chain.optiontypes_ttms[m]
            fd_paths = (_per_path_payoffs(xu[m], f, df, K, T) - _per_path_payoffs(xd[m], f, df, K, T)) / (2 * h)
            check(res.params[name][m], res.params_se[name][m], fd_paths, (name, m))


def test_library_refuses_q_var_and_f32_state(cuda_lib):
    from stochvolmodels_b200 import HawkesJDParams, engine
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    d = {k: v for k, v in HawkesJDParams().to_dict().items() if k in hawkes.KEYS}
    K, T = np.array([0.9, 1.1]), np.array(["P", "C"])
    with pytest.raises(Exception, match="LOG_RETURN"):
        engine.hawkesjd_mc_chain_greeks(_params_c(**d), [0.1], [1.0], [1.0], [K], [T], 1000, C.Q_VAR, 1, engine.mc_flags("fp64", "fp32"))
    with pytest.raises(Exception, match="fp64 state"):
        engine.hawkesjd_mc_chain_greeks(_params_c(**d), [0.1], [1.0], [1.0], [K], [T], 1000, C.LOG_RETURN, 1, engine.mc_flags("fp32", "fp32"))


# |MC row - Fourier row| the Euler scheme (1800 steps per year) may leave, fixed from the CPU oracles before any GPU run and re-derived by
# tools/hawkes_mc_greeks_allowance.py: on the hawkes_mc.npz chain (its parameters, maturities 0.05 / 0.12, P P C C C), the rows of
# oracle/hawkes_mc_greeks.py on 4 x 1e5 RandomState paths against oracle/hawkes_greeks.py, max over the 10 options of |MC - Fourier| + 4 SE:
# delta 5.33e-3, sigma 2.26e-3, shift_p 2.47e-2, mean_p 2.64e-2, shift_m 1.36e-2, mean_m 1.48e-2, lambda_p 1.80e-4, theta_p 1.87e-4,
# kappa_p 3.53e-5, beta1_p 1.58e-5, beta2_p 9.27e-6, lambda_m 8.13e-5, theta_m 1.60e-4, kappa_m 2.38e-5, beta1_m 7.11e-6, beta2_m 6.77e-6,
# each rounded up.  An upper bound on the scheme's bias in each row at ~4 sigma of the CPU sample.
HAWKES_MC_ALLOWANCE = {"delta": 6e-3, "sigma": 3e-3, "shift_p": 3e-2, "mean_p": 3e-2, "shift_m": 1.5e-2, "mean_m": 1.5e-2, "lambda_p": 2e-4,
                       "theta_p": 2e-4, "kappa_p": 4e-5, "beta1_p": 2e-5, "beta2_p": 1e-5, "lambda_m": 1e-4, "theta_m": 2e-4, "kappa_m": 3e-5,
                       "beta1_m": 8e-6, "beta2_m": 8e-6}


def test_every_row_matches_the_fourier_sensitivities(cuda_lib):
    """hawkes_mc.npz chain with its own option types, 4e6 paths: delta and the 15 rows against price_chain_greeks of the same model within
    4.5 SE plus the allowance above"""
    from stochvolmodels_b200 import HawkesJDPricer, OptionChain
    params, chain = _golden_chain()
    g = load_golden("hawkes_mc.npz")
    chain = OptionChain(ttms=chain.ttms, forwards=chain.forwards, discfactors=chain.discfactors, strikes_ttms=chain.strikes_ttms,
                        optiontypes_ttms=[g["chain_types"]] * len(chain.ttms))
    pricer = HawkesJDPricer()
    mc = pricer.model_mc_chain_greeks(chain, params, nb_path=4_000_000, seed=3)
    four = pricer.price_chain_greeks(chain, params)
    for m in range(len(chain.ttms)):
        rows = [("delta", mc.delta[m], mc.delta_se[m], four.delta[m])]
        rows += [(n, mc.params[n][m], mc.params_se[n][m], four.params[n][m]) for n in hg.PARAMS]
        for name, gm, se, f in rows:
            assert np.all(np.abs(gm - f) <= 4.5 * se + HAWKES_MC_ALLOWANCE[name]), (name, m, gm, f, se)
