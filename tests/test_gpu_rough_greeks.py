"""Pathwise sensitivities of the rough-LogSV chain MC on the GPU (b200sv_rough_logsv_mc_chain_greeks, LogSVPricer.rough_mc_chain_greeks)
against the production pricing kernel (terminal states bit for bit), the numpy forward-mode oracle (oracle/rough_greeks.py) on the same
normals, CRN central differences of the public price route, and the Fourier sensitivities at H = 1/2."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import rough, rough_greeks as rg

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = [np.array(["P", "IP", "C", "IC", "C"]), np.array(["P", "P", "IC", "C", "IP"])]
P6 = (0.8, 1.0, 3.0, 3.0, 0.15, 1.8)               # sigma0, theta, kappa1, kappa2, beta, orthog_vol


def _factors(n):
    if n == 1:
        return np.array([1.0]), np.array([1e-3])
    return np.linspace(0.5, 1.5, n), np.geomspace(3e-2, 300.0, n)


def _close(a, b, rtol, what):
    """relative to the reference array's scale (rows that vanish on most paths are compared at the scale they have elsewhere)"""
    scale = max(float(np.max(np.abs(b))), 1e-300)
    err = float(np.max(np.abs(np.asarray(a) - np.asarray(b))))
    assert err <= rtol * scale, (what, err / scale)


def _grid(ttm, npy):
    from stochvolmodels_b200.utils.funcs import set_time_grid
    return set_time_grid(ttm, npy)[2]


@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("gauss", [None, "fp32", "fp64"])
def test_states_bit_identical_to_the_pricing_kernel_and_tangents_match_the_oracle(cuda_lib, n, gauss):
    from stochvolmodels_b200 import _capi as C, engine
    from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_rough_vol_chain_valuation
    ttms, fw, df = np.array([0.1, 0.25]), np.array([1.0, 1.05]), np.array([0.999, 0.99])
    N, npy, seed = 3000, 200, 21
    w, x = _factors(n)
    Z0, Z1, grids = get_randoms_for_rough_vol_chain_valuation(ttms, N, npy, seed)
    nsteps, hs = [g.size - 1 for g in grids], [g[1] - g[0] for g in grids]
    flags = engine.mc_flags("fp64", gauss or "fp32")
    if gauss is not None:
        Z0, Z1 = engine.device_normals(seed, 0, N, 0, nsteps[-1], C.GAUSS_F64 if gauss == "fp64" else C.GAUSS_F32)
    zin = (Z0, Z1) if gauss is None else (None, None)
    pc = engine.logsv_params_c(*P6)
    strikes = [K5, K5 * 1.05]
    _, _, _, s_ref, _ = engine.rough_logsv_mc_chain([pc], w, x, ttms, fw, df, strikes, T5, N, nsteps, hs, *zin, 1, seed, flags, return_states=True)
    p, e, g, gse, offs, states, tangents, resets = engine.rough_logsv_mc_chain_greeks(pc, w, x, ttms, fw, df, strikes, T5, N, nsteps, hs, *zin, 1, seed,
                                                                              flags, return_states=True, return_tangents=True)
    np.testing.assert_array_equal(states, s_ref)
    for m in range(2):
        ls, vol, qv, dls, dvol, dqv, reset = rg.path_tangents(x, w, *P6, grids[m], Z0[: nsteps[m]], Z1[: nsteps[m]])
        assert resets[m] == reset.sum()
        np.testing.assert_allclose(states[m, 0], ls, rtol=0, atol=1e-10)
        for q, name in enumerate(rg.PARAMS):
            _close(tangents[m, q, 0], dls[q], 1e-10, (name, "log_spot", m))
            _close(tangents[m, q, 1:1 + n], dvol[q], 1e-10, (name, "vol", m))
            _close(tangents[m, q, 1 + n], dqv[q], 1e-10, (name, "qv", m))


def test_prices_equal_the_price_route_and_calls_are_deterministic(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, VariableType
    chain = OptionChain(ttms=np.array([0.1, 0.25]), forwards=np.array([1.0, 1.05]), strikes_ttms=[K5, K5 * 1.05], optiontypes_ttms=T5,
                        discfactors=np.array([0.999, 0.99]))
    w, x = _factors(3)
    p = LogSvParams(sigma0=P6[0], theta=P6[1], kappa1=P6[2], kappa2=P6[3], beta=P6[4], volvol=P6[5], H=0.3, weights=w, nodes=x)
    pricer = LogSVPricer()
    for gauss in (None, "fp32", "fp64"):
        for vt, chain_vt in ((VariableType.LOG_RETURN, chain), (VariableType.Q_VAR, OptionChain(
                ttms=chain.ttms, forwards=chain.forwards, strikes_ttms=[0.5 * K5, 0.6 * K5], optiontypes_ttms=T5, discfactors=chain.discfactors))):
            kw = dict(nb_path=20000, nb_steps=360, variable_type=vt, seed=5, gauss=gauss)
            pr, er = pricer.model_mc_price_chain(chain_vt, p, use_rough_mc=True, distributed=False, **kw)
            a = pricer.rough_mc_chain_greeks(chain_vt, p, **kw)
            b = pricer.rough_mc_chain_greeks(chain_vt, p, **kw)
            for m in range(2):
                np.testing.assert_allclose(a.prices[m], pr[m], rtol=1e-13, atol=1e-16)
                np.testing.assert_allclose(a.std_errors[m], er[m], rtol=1e-13, atol=1e-16)
                for f in ("prices", "std_errors", "delta", "delta_se"):
                    np.testing.assert_array_equal(getattr(a, f)[m], getattr(b, f)[m])
                for name in a.params:
                    np.testing.assert_array_equal(a.params[name][m], b.params[name][m])
                    np.testing.assert_array_equal(a.params_se[name][m], b.params_se[name][m])


def test_reset_count_and_tangents_on_paths_that_reset(cuda_lib):
    """a coarse grid with doubled vol shocks (the reset case of test_gpu_rough.py): the kernel's count of paths that reset at any step ==
    the oracle's per-path flag, states bit-identical to the pricing kernel, tangents (zero through a reset) == the oracle"""
    from stochvolmodels_b200 import engine
    P, ttms = 4000, np.array([0.25, 0.5])
    Z0, Z1, grids = rough.rough_randoms(ttms, P, 12, 77)
    Z0 = 2.0 * Z0
    w, x = np.array([0.8, 0.35]), np.array([0.0015625, 1.316])
    prm = (0.5, 0.6, 1.0, 10.0, -0.3, 2.0)
    K = [np.array([0.02, 0.05, 0.1]), np.array([0.05, 0.1, 0.2])]
    T = [np.array(["C", "P", "C"])] * 2
    nsteps, hs = [g.size - 1 for g in grids], [g[1] - g[0] for g in grids]
    pc = engine.logsv_params_c(*prm)
    _, _, _, s_ref, _ = engine.rough_logsv_mc_chain([pc], w, x, ttms, np.ones(2), np.ones(2), K, T, P, nsteps, hs, Z0, Z1, 2, 0, 0,
                                                    return_states=True)
    out = engine.rough_logsv_mc_chain_greeks(pc, w, x, ttms, np.ones(2), np.ones(2), K, T, P, nsteps, hs, Z0, Z1, 2, 0, 0, return_states=True,
                                             return_tangents=True)
    np.testing.assert_array_equal(out[5], s_ref)
    for m in range(2):
        ls, vol, qv, dls, dvol, dqv, reset = rg.path_tangents(x, w, *prm, grids[m], Z0[: nsteps[m]], Z1[: nsteps[m]])
        terminal = np.all(out[5][m, 1:3] == 1e-6, axis=0)
        assert out[7][m] == reset.sum() > terminal.sum()
        for q, name in enumerate(rg.PARAMS):
            _close(out[6][m, q, 0], dls[q], 1e-10, (name, "log_spot", m))
            _close(out[6][m, q, 1:3], dvol[q], 1e-10, (name, "vol", m))
            _close(out[6][m, q, 3], dqv[q], 1e-10, (name, "qv", m))


@pytest.mark.parametrize("name", ["h030_n3", "h045_n2", "h050_n1"])
def test_every_row_matches_the_oracle_on_the_golden_normals(cuda_lib, name):
    from stochvolmodels_b200 import engine
    g = load_golden(f"rough_mc_{name}.npz")
    M = int(g["nslices"])
    strikes, types = [g[f"strikes_{m}"] for m in range(M)], [g[f"types_{m}"] for m in range(M)]
    P, npy, seed = int(g["nb_path"]), int(g["npy"]), int(g["seed"])
    prm = tuple(g["params"][:6])
    Z0, Z1, grids = rough.rough_randoms(g["ttms"], P, npy, seed)
    nsteps, hs = [gr.size - 1 for gr in grids], [gr[1] - gr[0] for gr in grids]
    for vt in (1, 2):
        K = strikes if vt == 1 else [0.5 * k for k in strikes]
        po, eo, go, gseo = rg.rough_chain_greeks_fixed(g["ttms"], g["forwards"], g["discfactors"], K, types, Z0, Z1, *prm, g["weights"],
                                                       g["nodes"], grids, vt)
        p, e, gg, gse, offs, _, _, _ = engine.rough_logsv_mc_chain_greeks(engine.logsv_params_c(*prm), g["weights"], g["nodes"], g["ttms"],
                                                                       g["forwards"], g["discfactors"], K, types, P, nsteps, hs, Z0, Z1, vt, seed,
                                                                       engine.mc_flags("fp64", "fp32"))
        for m in range(M):
            sl = slice(offs[m], offs[m + 1])
            _close(p[m], po[m], 1e-10, ("price", m))
            _close(e[m], eo[m], 1e-10, ("std", m))
            for r in range(7):
                _close(gg[r, sl], go[m][r], 1e-10, ("greek", r, m, vt))
                _close(gse[r, sl], gseo[m][r], 1e-10, ("greek se", r, m, vt))


def _regression_case():
    from stochvolmodels_b200 import LogSvParams, get_btc_test_chain_data
    g = load_golden("rough_mc_reference_regression.npz")
    sigma0, theta, kappa1, kappa2, beta, volvol, H = g["params"]
    p = LogSvParams(sigma0=sigma0, theta=theta, kappa1=kappa1, kappa2=kappa2, beta=beta, volvol=volvol, H=H, weights=g["weights"], nodes=g["nodes"])
    return get_btc_test_chain_data(), p


def test_every_row_matches_crn_central_differences_of_the_price_route(cuda_lib):
    """BTC chain, H = 0.1 (three factors, the reference's regression fixture), 1e6 paths on one Philox seed: the pathwise rows against
    central differences of the public model_mc_price_chain(use_rough_mc=True) with common random numbers, within 0.1 standard error.
    At the fixture's 360 steps per year ~1 % of the paths take the reset branch at some step (the RK4 drift overshoots through zero), and
    the rows omit the mass they move across it; on a 5760-step grid no path resets at any step, which the kernel's per-path count asserts."""
    import dataclasses
    from stochvolmodels_b200 import LogSVPricer, OptionChain, engine
    chain, p = _regression_case()
    pricer = LogSVPricer()
    N, seed = 1_000_000, 17
    coarse = pricer.rough_mc_chain_greeks(chain, p, nb_path=N, nb_steps=360, seed=seed, gauss="fp32")
    assert coarse.reset_paths[-1] > 1000, coarse.reset_paths          # the counter sees resets that do not last to maturity
    kw = dict(nb_path=N, nb_steps=5760, seed=seed, gauss="fp32")
    res = pricer.rough_mc_chain_greeks(chain, p, **kw)
    assert np.all(res.reset_paths == 0), res.reset_paths
    price = lambda q, c=chain: pricer.model_mc_price_chain(c, q, use_rough_mc=True, distributed=False, **kw)[0]
    hf = 1e-6
    bump = lambda f: OptionChain(ttms=chain.ttms, forwards=chain.forwards * f, strikes_ttms=chain.strikes_ttms,
                                 optiontypes_ttms=chain.optiontypes_ttms, discfactors=chain.discfactors)
    pu, pd = price(p, bump(1 + hf)), price(p, bump(1 - hf))
    for m in range(chain.ttms.size):
        fd = (pu[m] - pd[m]) / (2 * hf * chain.forwards[m])
        assert np.all(np.abs(res.delta[m] - fd) <= 0.1 * res.delta_se[m] + 1e-9 * (1 + np.abs(fd))), ("delta", m)
    for name in engine.LOGSV_GREEK_PARAMS:
        x = getattr(p, name)
        h = 1e-6 * max(abs(x), 1e-2)
        pu, pd = price(dataclasses.replace(p, **{name: x + h})), price(dataclasses.replace(p, **{name: x - h}))
        for m in range(chain.ttms.size):
            fd = (pu[m] - pd[m]) / (2 * h)
            g, se = res.params[name][m], res.params_se[name][m]
            assert np.all(np.abs(g - fd) <= 0.1 * se + 1e-9 * (1 + np.abs(fd))), (name, m, g, fd, se)


# Discretisation allowance of the H = 1/2 gate, per row: max over the 10 strikes of |rough MC - Fourier| + SE in a CPU run of the numpy
# oracles, re-derived by tools/rough_greeks_h05_allowance.py (oracle/rough_greeks.py at 360 steps/yr, 4 x 1e5 RandomState paths, against
# oracle/mgf_greeks.py): delta 2.23e-3, sigma0 1.32e-3, theta 9.8e-4, kappa1 8.9e-5, kappa2 9.5e-5, beta 1.01e-3, volvol 7.2e-4, each
# rounded up (kappa2 to 2e-4).  The gap is the Strang / RK4 time-step bias plus the Fourier route's second-order expansion error.
H05_ALLOWANCE = {"delta": 3e-3, "sigma0": 2e-3, "theta": 1e-3, "kappa1": 1e-4, "kappa2": 2e-4, "beta": 2e-3, "volvol": 8e-4}


def test_single_node_rows_match_the_fourier_sensitivities(cuda_lib):
    """H = 1/2 (one node at 1e-3): the rough scheme is the article's LogSV dynamics, so its pathwise rows estimate the Fourier route's
    sensitivities: within 4.5 SE plus the discretisation allowance above"""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    K = np.array([0.8, 0.9, 1.0, 1.1, 1.2]); T = np.array(["P", "P", "C", "C", "C"])
    chain = OptionChain(ttms=np.array([0.1, 0.25]), forwards=np.ones(2), strikes_ttms=[K, K], optiontypes_ttms=[T, T])
    q = LogSvParams(sigma0=1.0, theta=1.0, kappa1=5.0, kappa2=5.0, beta=0.2, volvol=2.0)
    q.approximate_kernel(T=0.25)
    pricer = LogSVPricer()
    mc = pricer.rough_mc_chain_greeks(chain, q, nb_path=4_000_000, nb_steps=360, seed=11, gauss="fp32")
    four = pricer.price_chain_greeks(chain, q)
    for m in range(2):
        rows = [("delta", mc.delta[m], mc.delta_se[m], four.delta[m])]
        rows += [(n, mc.params[n][m], mc.params_se[n][m], four.params[n][m]) for n in mc.params]
        for name, g, se, f in rows:
            assert np.all(np.abs(g - f) <= 4.5 * se + H05_ALLOWANCE[name]), (name, m, g, f, se)
