"""GPU: the Monte Carlo theta of the LogSV / Heston chain pricers, pathwise in each slice's step length with its step count held
(DESIGN.md §3.12).

  unchanged   -- with_theta=True returns the prices, standard errors, delta, parameter rows and gamma of with_theta=False bit for bit, and
                 two runs are bit-identical
  path level  -- the theta pass's (dx, dq) / d dt equal the oracle (oracle/mc_theta.py) on the kernel's own normals, and so do the rows
  statistics  -- every theta row against common-random-number central differences of the GPU price route with ttm_m moved alone, and
                 against the Fourier theta of price_chain_greeks within 4.5 SE plus the Euler allowance of tools/mc_theta_allowance.py
"""
import numpy as np
import pytest

from oracle import mc, mc_theta as ot

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                   # quickstart LogSV parameters
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)                # HestonParams() defaults
# max over the chain's options of |MC theta - Fourier theta| + 4 SE of the CPU oracles (tools/mc_theta_allowance.py): an upper bound on the
# Euler scheme's bias in the theta row at the route's step grid, allowed on top of 4.5 SE of the GPU's own noise
# (1e5 paths x 8 batches: 1.128e-2, 7.16e-4, rounded up; the oracle rows sit at most 7.87 and 1.47 SE from the Fourier rows)
THETA_ALLOWANCE = {"quickstart": 1.2e-2, "g4": 8.0e-4}


def _chain(name):
    from stochvolmodels_b200 import OptionChain
    ttms = np.array([0.25, 0.5]) if name == "quickstart" else np.array([0.25, 1.0])
    return OptionChain(ttms=ttms, forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])


def _case(model):
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer
    if model == "heston":
        return HestonPricer(), _chain("g4"), HestonParams(*HESTON)
    return LogSVPricer(), _chain("quickstart"), LogSvParams(*Q)


def _kw(model, is_spot, gauss, nb_path, seed):
    kw = dict(nb_path=nb_path, seed=seed, gauss=gauss)
    if model == "logsv":
        kw.update(nb_steps=252, is_spot_measure=is_spot)
    return kw


@pytest.mark.parametrize("model,is_spot,gauss", [("logsv", True, "fp32"), ("logsv", False, "fp64"), ("logsv", True, "fp64"),
                                                 ("heston", True, "fp32"), ("heston", True, "fp64")])
@pytest.mark.parametrize("with_gamma", [False, True])
def test_with_theta_leaves_every_other_output_unchanged(cuda_lib, model, is_spot, gauss, with_gamma):
    pricer, chain, params = _case(model)
    kw = _kw(model, is_spot, gauss, 300_000, 2024)
    plain = pricer.model_mc_chain_greeks(chain, params, with_gamma=with_gamma, **kw)
    res = pricer.model_mc_chain_greeks(chain, params, with_gamma=with_gamma, with_theta=True, **kw)
    again = pricer.model_mc_chain_greeks(chain, params, with_gamma=with_gamma, with_theta=True, **kw)
    assert plain.theta is None and plain.theta_se is None
    for m in range(len(chain.ttms)):
        pairs = [(res.prices, plain.prices), (res.std_errors, plain.std_errors), (res.delta, plain.delta), (res.delta_se, plain.delta_se),
                 (again.theta, res.theta), (again.theta_se, res.theta_se)]
        if with_gamma:
            pairs += [(res.gamma, plain.gamma), (res.gamma_se, plain.gamma_se)]
        else:
            assert res.gamma is None
        for a, b in pairs:
            np.testing.assert_array_equal(a[m], b[m])
        for name in plain.params:
            np.testing.assert_array_equal(res.params[name][m], plain.params[name][m])
            np.testing.assert_array_equal(res.params_se[name][m], plain.params_se[name][m])
        assert np.all(np.isfinite(res.theta[m])) and np.all(res.theta_se[m] > 0)


K8 = np.array([0.85, 0.9, 0.95, 1.0, 1.0, 1.05, 1.1, 1.2])
T8 = np.array(["P", "IP", "C", "IC", "P", "IC", "C", "IP"])


@pytest.mark.parametrize("model,is_spot,gauss,vt", [("logsv", True, "fp32", mc.LOG_RETURN), ("logsv", False, "fp64", mc.LOG_RETURN),
                                                    ("logsv", True, "fp64", mc.Q_VAR), ("heston", True, "fp32", mc.LOG_RETURN),
                                                    ("heston", True, "fp64", mc.Q_VAR)])
def test_dtheta_and_rows_vs_oracle_on_device_normals(cuda_lib, model, is_spot, gauss, vt):
    from stochvolmodels_b200 import engine
    N, npy, seed = 4096, 300, 31
    ttms, fw, df = np.array([0.1, 0.35]), np.array([1.0, 1.05]), np.array([0.99, 0.97])
    kq = 1.0 if model == "logsv" or vt == mc.LOG_RETURN else HESTON[1]
    strikes, types = [K8 * kq, K8 * 1.05 * kq], [T8, T8]
    flags = engine.mc_flags("fp64", gauss)
    steps = mc.chain_steps(ttms, npy)
    Z = [engine.device_normals(seed, 0, N, m, S, flags) for m, (S, _) in enumerate(steps)]
    dts = [dt for _, dt in steps]
    if model == "logsv":
        etas = np.array([1.0, 1.0]) if is_spot else np.array([0.9, 1.1])
        res = engine.logsv_mc_chain_greeks_theta(engine.logsv_params_c(*Q), ttms, fw, df, etas, strikes, types, N, npy, is_spot, vt, seed, flags,
                                                 n_paths_out=N)
        ref = ot.logsv_mc_chain_theta_fixed(Q, ttms, fw, df, strikes, types, etas, [z[0] for z in Z], [z[1] for z in Z], dts, is_spot, vt,
                                            return_states=True)
    else:
        res = engine.heston_mc_chain_greeks_theta(engine.heston_params_c(*HESTON), ttms, fw, df, strikes, types, N, npy, vt, seed, flags,
                                                  n_paths_out=N)
        ref = ot.heston_mc_chain_theta_fixed(HESTON, ttms, fw, df, strikes, types, [z[0] for z in Z], [z[1] for z in Z], dts, vt,
                                             return_states=True)
    offsets, theta, theta_se, dtheta = res[4], res[7], res[8], res[9]
    for m in range(2):
        dx_o, dq_o = ref[4][m][3], ref[4][m][4]
        for got, want in ((dtheta[m][0], dx_o), (dtheta[m][1], dq_o)):
            scale = float(np.max(np.abs(want)))
            assert float(np.max(np.abs(got - want))) <= 1e-10 * scale, (m, got[:4], want[:4])
        sl = slice(offsets[m], offsets[m + 1])
        for got, want in ((theta[sl], ref[2][m]), (theta_se[sl], ref[3][m])):
            assert float(np.max(np.abs(got - want))) <= 1e-9 * max(float(np.max(np.abs(want))), 1e-300), (m, got, want)


# ttms whose slices keep their step count under a +-1e-3 move at 252 steps per year: 0.252 * 252 = 63.5 -> S = 64 from 63.25 to 63.76
TTMS_CRN = np.array([0.252, 0.504])
NPY_CRN, H_CRN = 252, 1e-3


@pytest.mark.parametrize("model,is_spot,vt", [("logsv", True, mc.LOG_RETURN), ("logsv", False, mc.Q_VAR), ("heston", True, mc.LOG_RETURN)])
def test_theta_vs_crn_central_differences_of_the_price_route(cuda_lib, model, is_spot, vt):
    from stochvolmodels_b200 import engine
    N, seeds = 1_000_000, range(100, 108)
    fw, df = np.array([1.0, 1.02]), np.array([0.99, 0.97])
    kq = HESTON[1] if model == "heston" and vt == mc.Q_VAR else 1.0
    strikes, types = [K8 * kq, K8 * kq], [T8, T8]
    etas = np.array([1.0, 1.1])
    flags = engine.mc_flags("fp64", "fp32")
    steps = mc.chain_steps(TTMS_CRN, NPY_CRN)
    for m in range(2):
        t0 = TTMS_CRN[m - 1] if m else 0.0
        for s in (1.0, -1.0):
            assert mc.set_time_grid(TTMS_CRN[m] + s * H_CRN - t0, NPY_CRN)[0] == steps[m][0]

    def price(ttms, seed):
        if model == "logsv":
            return engine.logsv_mc_chain(engine.logsv_params_c(*Q), ttms, fw, df, etas, strikes, types, N, NPY_CRN, is_spot, vt, seed, flags)[0]
        return engine.heston_mc_chain(engine.heston_params_c(*HESTON), ttms, fw, df, strikes, types, N, NPY_CRN, vt, seed, flags)[0]

    th, cd = [[], []], [[], []]
    for seed in seeds:
        if model == "logsv":
            res = engine.logsv_mc_chain_greeks_theta(engine.logsv_params_c(*Q), TTMS_CRN, fw, df, etas, strikes, types, N, NPY_CRN, is_spot, vt,
                                                     seed, flags)
        else:
            res = engine.heston_mc_chain_greeks_theta(engine.heston_params_c(*HESTON), TTMS_CRN, fw, df, strikes, types, N, NPY_CRN, vt, seed,
                                                      flags)
        for m in range(2):
            up, dn = TTMS_CRN.copy(), TTMS_CRN.copy()
            up[m] += H_CRN
            dn[m] -= H_CRN
            th[m].append(res[7][res[4][m]:res[4][m + 1]])
            cd[m].append(-(price(up, seed)[m] - price(dn, seed)[m]) / (2 * H_CRN))
    k = len(seeds)
    for m in range(2):
        a, b = np.array(th[m]), np.array(cd[m])
        se = np.sqrt(a.var(axis=0, ddof=1) / k + b.var(axis=0, ddof=1) / k)
        gap = np.abs(a.mean(axis=0) - b.mean(axis=0))
        assert np.all(gap <= 4.0 * se), (m, a.mean(axis=0), b.mean(axis=0), se)


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_theta_vs_fourier(cuda_lib, model):
    pricer, chain, params = _case(model)
    res = pricer.model_mc_chain_greeks(chain, params, with_theta=True, **_kw(model, True, "fp32", 4_000_000, 5))
    four = pricer.price_chain_greeks(chain, params, with_theta=True)
    A = THETA_ALLOWANCE["quickstart" if model == "logsv" else "g4"]
    for m in range(len(chain.ttms)):
        gap = np.abs(res.theta[m] - four.theta[m])
        assert np.all(gap <= 4.5 * res.theta_se[m] + A), (model, m, res.theta[m], four.theta[m], res.theta_se[m])


# ---- rough-LogSV route ------------------------------------------------------------------------------------------------------------------
R_FACTORS = {1: (np.array([1.0]), np.array([1e-3])), 3: (np.linspace(0.5, 1.5, 3), np.geomspace(3e-2, 300.0, 3))}
R_P6 = (0.8, 1.0, 3.0, 3.0, 0.15, 1.8)               # sigma0, theta, kappa1, kappa2, beta, orthog_vol


def _rough_params(n, H=0.3):
    from stochvolmodels_b200 import LogSvParams
    w, x = R_FACTORS[n]
    return LogSvParams(sigma0=R_P6[0], theta=R_P6[1], kappa1=R_P6[2], kappa2=R_P6[3], beta=R_P6[4], volvol=R_P6[5], H=H, weights=w, nodes=x)


@pytest.mark.parametrize("gauss", [None, "fp32", "fp64"])
@pytest.mark.parametrize("vt", [mc.LOG_RETURN, mc.Q_VAR])
def test_rough_with_theta_leaves_every_other_output_unchanged(cuda_lib, gauss, vt):
    from stochvolmodels_b200 import LogSVPricer, OptionChain, VariableType
    K = K5 if vt == mc.LOG_RETURN else 0.5 * K5
    chain = OptionChain(ttms=np.array([0.1, 0.25]), forwards=np.array([1.0, 1.05]), strikes_ttms=[K, K * 1.05], optiontypes_ttms=[T5, T5],
                        discfactors=np.array([0.999, 0.99]))
    pricer, p = LogSVPricer(), _rough_params(3)
    kw = dict(nb_path=20000, nb_steps=360, seed=5, gauss=gauss, variable_type=VariableType(vt))
    plain = pricer.rough_mc_chain_greeks(chain, p, **kw)
    res = pricer.rough_mc_chain_greeks(chain, p, with_theta=True, **kw)
    again = pricer.rough_mc_chain_greeks(chain, p, with_theta=True, **kw)
    assert plain.theta is None
    np.testing.assert_array_equal(res.reset_paths, plain.reset_paths)
    for m in range(2):
        for a, b in ((res.prices, plain.prices), (res.std_errors, plain.std_errors), (res.delta, plain.delta), (res.delta_se, plain.delta_se),
                     (again.theta, res.theta), (again.theta_se, res.theta_se)):
            np.testing.assert_array_equal(a[m], b[m])
        for name in plain.params:
            np.testing.assert_array_equal(res.params[name][m], plain.params[name][m])
            np.testing.assert_array_equal(res.params_se[name][m], plain.params_se[name][m])
        assert np.all(np.isfinite(res.theta[m])) and np.all(res.theta_se[m] > 0)


@pytest.mark.parametrize("n", [1, 3])
def test_rough_dtheta_and_rows_vs_oracle_on_uploaded_normals(cuda_lib, n):
    from oracle import rough
    from stochvolmodels_b200 import engine
    P, ttms, npy = 4096, np.array([0.1, 0.25]), 360
    Z0, Z1, grids = rough.rough_randoms(ttms, P, npy, 13)
    nsteps, hs = [g.size - 1 for g in grids], [g[1] - g[0] for g in grids]
    w, x = R_FACTORS[n]
    fw, df = np.array([1.0, 1.05]), np.array([0.999, 0.99])
    strikes, types = [K8, K8 * 1.05], [T8, T8]
    out = engine.rough_logsv_mc_chain_greeks(engine.logsv_params_c(*R_P6), w, x, ttms, fw, df, strikes, types, P, nsteps, hs, Z0, Z1, 1, 0, 0,
                                             with_theta=True, n_paths_out=P)
    offsets, theta, theta_se, dtheta = out[4], out[8], out[9], out[10]
    th, se, states = ot.rough_chain_theta_fixed(ttms, fw, df, strikes, types, Z0, Z1, *R_P6, w, x, nsteps, hs)
    for m in range(2):
        ls, _, y, dls, dy, reset = states[m]
        assert out[7][m] == reset.sum()
        for got, want in ((dtheta[m][0], dls), (dtheta[m][1], dy)):
            scale = float(np.max(np.abs(want)))
            assert float(np.max(np.abs(got - want))) <= 1e-10 * scale, (m, got[:4], want[:4])
        sl = slice(offsets[m], offsets[m + 1])
        for got, want in ((theta[sl], th[m]), (theta_se[sl], se[m])):
            assert float(np.max(np.abs(got - want))) <= 1e-9 * max(float(np.max(np.abs(want))), 1e-300), (m, got, want)


def test_rough_theta_vs_crn_central_differences_of_the_price_route(cuda_lib):
    """BTC chain, H = 0.1 (three factors, the reference's regression fixture), 1e6 Philox paths on a 5760-step grid where no path resets:
    every ttm moved at once by +-1e-6 (each maturity restarts at t = 0 on its own grid, so the rows do not interact) with the step counts
    asserted unchanged, against the theta rows on the same normals within 0.1 SE"""
    from conftest import load_golden
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, get_btc_test_chain_data
    g = load_golden("rough_mc_reference_regression.npz")
    sigma0, theta, kappa1, kappa2, beta, volvol, H = g["params"]
    p = LogSvParams(sigma0=sigma0, theta=theta, kappa1=kappa1, kappa2=kappa2, beta=beta, volvol=volvol, H=H, weights=g["weights"], nodes=g["nodes"])
    chain, pricer = get_btc_test_chain_data(), LogSVPricer()
    npy, hT = 5760, 1e-6
    for t in chain.ttms:
        assert mc.set_time_grid(t + hT, npy)[0] == mc.set_time_grid(t - hT, npy)[0] == mc.set_time_grid(t, npy)[0]
    kw = dict(nb_path=1_000_000, nb_steps=npy, seed=17, gauss="fp32")
    res = pricer.rough_mc_chain_greeks(chain, p, with_theta=True, **kw)
    assert np.all(res.reset_paths == 0), res.reset_paths
    moved = lambda s: OptionChain(ttms=chain.ttms + s * hT, forwards=chain.forwards, strikes_ttms=chain.strikes_ttms,
                                  optiontypes_ttms=chain.optiontypes_ttms, discfactors=chain.discfactors)
    pu = pricer.model_mc_price_chain(moved(1.0), p, use_rough_mc=True, distributed=False, **kw)[0]
    pd = pricer.model_mc_price_chain(moved(-1.0), p, use_rough_mc=True, distributed=False, **kw)[0]
    for m in range(chain.ttms.size):
        fd = -(pu[m] - pd[m]) / (2 * hT)
        assert np.all(np.abs(res.theta[m] - fd) <= 0.1 * res.theta_se[m] + 1e-7 * (1 + np.abs(fd))), (m, res.theta[m], fd, res.theta_se[m])
