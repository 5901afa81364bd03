"""GPU: the Monte Carlo gamma of the LogSV / Heston chain pricers by conditional smoothing of the last step (DESIGN.md §3.9).

  unchanged   -- with_gamma=True returns the prices, standard errors, delta and parameter rows of with_gamma=False bit for bit, and two
                 runs are bit-identical
  path level  -- the recorded last step (s, mu) equals the oracle (oracle/mc_gamma.py) on the kernel's own normals; the gamma rows equal
                 the oracle's estimator on the kernel's own per-path states
  statistics  -- every gamma row against the Fourier gamma of price_chain_greeks within 4.5 SE plus the Euler scheme's allowance of
                 tools/mc_gamma_allowance.py, and against common-random-number second differences of the public price route
"""
import numpy as np
import pytest

from oracle import mc, mc_gamma as og

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                   # quickstart LogSV parameters
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)                # HestonParams() defaults
# max over the chain's options of |MC gamma - Fourier gamma| + 4 SE of the CPU oracles (tools/mc_gamma_allowance.py): an upper bound on the
# Euler scheme's bias in the gamma row at the route's step grid, allowed on top of 4.5 SE of the GPU's own noise
# (1e5 paths x 8 batches: 1.24e-2, 3.83e-7, 5.85e-2, rounded up; the oracle rows sit at most 1.25, 3.85 and 1.34 SE from the Fourier rows)
GAMMA_ALLOWANCE = {"quickstart": 1.3e-2, "btc": 4.0e-7, "g4": 6.0e-2}


def _chain(name):
    from stochvolmodels_b200 import OptionChain, get_btc_test_chain_data
    if name == "btc":
        return get_btc_test_chain_data()
    ttms = np.array([0.25, 0.5]) if name == "quickstart" else np.array([0.25, 1.0])
    return OptionChain(ttms=ttms, forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])


def _case(model, chain_name):
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, LOGSV_BTC_PARAMS
    chain = _chain(chain_name)
    if model == "heston":
        return HestonPricer(), chain, HestonParams(*HESTON)
    return LogSVPricer(), chain, (LOGSV_BTC_PARAMS if chain_name == "btc" else LogSvParams(*Q))


CASES = [("logsv", "quickstart", True, "fp32"), ("logsv", "quickstart", False, "fp64"), ("logsv", "btc", True, "fp32"),
         ("heston", "g4", True, "fp32"), ("heston", "g4", True, "fp64")]


def _kw(model, is_spot, gauss, nb_path, seed):
    kw = dict(nb_path=nb_path, seed=seed, gauss=gauss)
    if model == "logsv":
        kw.update(nb_steps=252, is_spot_measure=is_spot)
    return kw


@pytest.mark.parametrize("model,chain_name,is_spot,gauss", CASES)
def test_with_gamma_leaves_every_other_output_unchanged(cuda_lib, model, chain_name, is_spot, gauss):
    pricer, chain, params = _case(model, chain_name)
    kw = _kw(model, is_spot, gauss, 300_000, 2024)
    plain = pricer.model_mc_chain_greeks(chain, params, **kw)
    res = pricer.model_mc_chain_greeks(chain, params, with_gamma=True, **kw)
    again = pricer.model_mc_chain_greeks(chain, params, with_gamma=True, **kw)
    assert plain.gamma is None and plain.gamma_se is None
    for m in range(len(chain.ttms)):
        for a, b in ((res.prices, plain.prices), (res.std_errors, plain.std_errors), (res.delta, plain.delta), (res.delta_se, plain.delta_se),
                     (again.gamma, res.gamma), (again.gamma_se, res.gamma_se)):
            np.testing.assert_array_equal(a[m], b[m])
        for name in plain.params:
            np.testing.assert_array_equal(res.params[name][m], plain.params[name][m])
            np.testing.assert_array_equal(res.params_se[name][m], plain.params_se[name][m])
        assert res.gamma[m].shape == plain.prices[m].shape and np.all(np.isfinite(res.gamma[m])) and np.all(res.gamma_se[m] > 0)


K8 = np.array([0.85, 0.9, 0.95, 1.0, 1.0, 1.05, 1.1, 1.2])
T8 = np.array(["P", "IP", "C", "IC", "P", "IC", "C", "IP"])


@pytest.mark.parametrize("model,is_spot,gauss,vt", [("logsv", True, "fp32", mc.LOG_RETURN), ("logsv", False, "fp64", mc.LOG_RETURN),
                                                    ("logsv", True, "fp64", mc.Q_VAR), ("heston", True, "fp32", mc.LOG_RETURN),
                                                    ("heston", True, "fp64", mc.Q_VAR)])
def test_laststep_and_gamma_rows_vs_oracle_on_device_normals(cuda_lib, model, is_spot, gauss, vt):
    from stochvolmodels_b200 import engine
    N, npy, seed = 4096, 300, 31
    ttms, fw, df = np.array([0.1, 0.35]), np.array([1.0, 1.05]), np.array([0.99, 0.97])
    strikes, types = [K8, K8 * 1.05], [T8, T8]
    flags = engine.mc_flags("fp64", gauss)
    steps = mc.chain_steps(ttms, npy)
    Z = [engine.device_normals(seed, 0, N, m, S, flags) for m, (S, _) in enumerate(steps)]
    dts = [dt for _, dt in steps]
    if model == "logsv":
        etas = np.array([1.0, 1.0]) if is_spot else np.array([0.9, 1.1])
        res = engine.logsv_mc_chain_greeks_gamma(engine.logsv_params_c(*Q), ttms, fw, df, etas, strikes, types, N, npy, is_spot, vt, seed, flags,
                                                 n_paths_out=N)
        ref = og.logsv_mc_chain_gamma_fixed(Q, ttms, fw, df, strikes, types, etas, [z[0] for z in Z], [z[1] for z in Z], dts, is_spot, vt,
                                            return_states=True)
    else:
        res = engine.heston_mc_chain_greeks_gamma(engine.heston_params_c(*HESTON), ttms, fw, df, strikes, types, N, npy, vt, seed, flags,
                                                  n_paths_out=N)
        ref = og.heston_mc_chain_gamma_fixed(HESTON, ttms, fw, df, strikes, types, [z[0] for z in Z], [z[1] for z in Z], dts, vt,
                                             return_states=True)
    gamma, gamma_se, laststep, offsets = res[5], res[6], res[7], res[4]
    for m in range(2):
        x_o, v_o, q_o, s_o, mu_o = ref[4][m]
        s, mu = laststep[m]
        np.testing.assert_allclose(s, s_o, rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(mu, mu_o, rtol=1e-11, atol=1e-12)
        x = mu + s * Z[m][0][-1]                                    # the kernel's own terminal log-spot
        g, ge = og.mc_payoff_gamma(x, q_o, s, mu, ttms[m], fw[m], strikes[m], types[m], df[m], vt)
        sl = slice(offsets[m], offsets[m + 1])
        scale = max(float(np.max(np.abs(g))), 1e-300)
        assert float(np.max(np.abs(gamma[sl] - g))) <= 1e-10 * scale, (m, gamma[sl], g)
        assert float(np.max(np.abs(gamma_se[sl] - ge))) <= 1e-10 * max(float(np.max(ge)), 1e-300), (m, gamma_se[sl], ge)


@pytest.mark.parametrize("model,chain_name,is_spot", [("logsv", "quickstart", True), ("logsv", "btc", True), ("heston", "g4", True)])
def test_gamma_vs_fourier(cuda_lib, model, chain_name, is_spot):
    pricer, chain, params = _case(model, chain_name)
    res = pricer.model_mc_chain_greeks(chain, params, with_gamma=True, **_kw(model, is_spot, "fp32", 4_000_000, 5))
    four = pricer.price_chain_greeks(chain, params)
    A = GAMMA_ALLOWANCE[chain_name]
    for m in range(len(chain.ttms)):
        gap = np.abs(res.gamma[m] - four.gamma[m])
        assert np.all(gap <= 4.5 * res.gamma_se[m] + A), (chain_name, m, res.gamma[m], four.gamma[m], res.gamma_se[m])


def _bump(chain, f):
    from stochvolmodels_b200 import OptionChain
    return OptionChain(ttms=chain.ttms, forwards=chain.forwards * f, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                       discfactors=chain.discfactors)


@pytest.mark.parametrize("model,chain_name,is_spot", [("logsv", "quickstart", True), ("logsv", "quickstart", False), ("logsv", "btc", True),
                                                      ("heston", "g4", True)])
def test_gamma_vs_crn_second_differences_of_the_price_route(cuda_lib, model, chain_name, is_spot):
    """over 8 seeds: the mean gamma row against the mean CRN second difference (+-1 % of the forward) of model_mc_price_chain, within 4
    combined SE (the second difference's SE from its spread over the seeds)"""
    pricer, chain, params = _case(model, chain_name)
    h, seeds, M = 0.01, range(100, 108), len(chain.ttms)
    g, g_var, d2 = [[] for _ in range(M)], [[] for _ in range(M)], [[] for _ in range(M)]
    for seed in seeds:
        kw = _kw(model, is_spot, "fp32", 500_000, seed)
        res = pricer.model_mc_chain_greeks(chain, params, with_gamma=True, **kw)
        up, mid, dn = (pricer.model_mc_price_chain(_bump(chain, f), params, **kw)[0] for f in (1 + h, 1.0, 1 - h))
        for m in range(M):
            np.testing.assert_allclose(mid[m], res.prices[m], rtol=1e-13, atol=0)      # the price route's own reduction order
            g[m].append(res.gamma[m])
            g_var[m].append(res.gamma_se[m] ** 2)
            d2[m].append((up[m] - 2 * mid[m] + dn[m]) / (h * chain.forwards[m]) ** 2)
    B = len(seeds)
    for m in range(M):
        gm, gse = np.mean(g[m], axis=0), np.sqrt(np.mean(g_var[m], axis=0) / B)
        cm, cse = np.mean(d2[m], axis=0), np.std(d2[m], axis=0, ddof=1) / np.sqrt(B)
        z = np.abs(gm - cm) / np.sqrt(gse ** 2 + cse ** 2)
        assert np.all(z <= 4.0), (chain_name, m, gm, cm, z)


def test_gamma_rejects_what_the_greeks_route_rejects(cuda_lib):
    from stochvolmodels_b200 import _capi as C, engine
    chain = _chain("quickstart")
    args = (chain.ttms, chain.forwards, chain.discfactors)
    for flags in (C.STATE_F32, C.GAUSS_F64_PAIRED):
        with pytest.raises(C.B200svError, match="invalid argument"):
            engine.logsv_mc_chain_greeks_gamma(engine.logsv_params_c(*Q), *args, None, chain.strikes_ttms, chain.optiontypes_ttms, 1000, 100, True,
                                               1, 1, flags)
    with pytest.raises(C.B200svError, match="EULER_FLOOR"):
        engine.heston_mc_chain_greeks_gamma(engine.heston_params_c(*HESTON), *args, chain.strikes_ttms, chain.optiontypes_ttms, 1000, 100, 1, 1, 0,
                                            C.HESTON_QE)
    with pytest.raises(C.B200svError, match="n_paths_out"):
        engine.logsv_mc_chain_greeks_gamma(engine.logsv_params_c(*Q), *args, None, chain.strikes_ttms, chain.optiontypes_ttms, 1000, 100, True,
                                           1, 1, 0, n_paths_out=1001)
