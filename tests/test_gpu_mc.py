"""GPU parity tests of the Monte Carlo path, through the C ABI (ctypes) and the Pricer API.

Tiers (SURVEY.md §8c):
  arithmetic  -- fixed-random steppers vs golden states from the reference: <= 1e-12 abs
                 fused Philox kernel vs the oracle fed with the same normals: <= 1e-10
  statistical -- Philox prices within 3 standard errors of the Fourier price (reference tests use 4 SE)
"""
import numpy as np
import pytest

from conftest import chain_from_golden, load_golden
from oracle import cport, mc, mgf

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)


def _fixed_randoms(g):
    rng = np.random.RandomState(int(g["seed"]))
    N = int(g["nb_path"])
    out0, out1 = [], []
    for S in g["nsteps"]:
        out0.append(rng.normal(0, 1, size=(int(S), N)))
        out1.append(rng.normal(0, 1, size=(int(S), N)))
    return out0, out1


def test_exp_pair_accuracy(cuda_lib):
    from stochvolmodels_b200 import engine
    L = np.concatenate([np.linspace(-30, 30, 200001), np.random.RandomState(0).normal(0, 2, 100000), [0.0, -700.0, 700.0, 1e-300, -1e-17]])
    ep, em = engine.debug_exp_pair(L)
    rel_p = np.abs(ep / np.exp(L) - 1)
    rel_m = np.abs(em / np.exp(-L) - 1)
    assert rel_p.max() < 4.5e-16 and rel_m.max() < 4.5e-16, (rel_p.max(), rel_m.max())


def test_exp_pair_scaled_accuracy(cuda_lib):
    """the stepper's exp pair on table units Ls = L*256/ln2, against exp in extended precision of the SAME argument Ls*ln2/256"""
    from stochvolmodels_b200 import engine
    rs = np.random.RandomState(1)
    Ls = np.concatenate([np.linspace(-11000, 11000, 200001), rs.normal(0, 700, 100000), rs.uniform(-258530, 258530, 50000),
                         [0.0, 0.5, -0.5, 1.5, 255.5, 256.0, -256.5, 258530.0, -258530.0, 1e-300, 3e5, -1e9]])
    ep, em = engine.debug_exp_pair_scaled(Ls)
    ld = np.longdouble
    arg = np.clip(Ls, -258530.0, 258530.0).astype(ld) * (np.log(ld(2)) / ld(256))
    rel_p = np.abs((ep.astype(ld) / np.exp(arg) - 1).astype(float))
    rel_m = np.abs((em.astype(ld) / np.exp(-arg) - 1).astype(float))
    assert rel_p.max() < 4.5e-16 and rel_m.max() < 4.5e-16, (rel_p.max(), rel_m.max())


@pytest.mark.parametrize("tag", ["g5_c1", "inverse_eta", "btc_small", "qvar"])
def test_logsv_fixed_randoms_vs_reference_golden(cuda_lib, tag):
    """b200sv_logsv_step_fixed + b200sv_mc_payoffs == logsv_mc_chain_pricer_fixed_randoms of the reference."""
    from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_chain_valuation, logsv_mc_chain_pricer_fixed_randoms
    from stochvolmodels_b200.utils.config import VariableType
    g = load_golden(f"logsv_mc_fixed_{tag}.npz")
    strikes, types = chain_from_golden(g)
    W0s, W1s, dts = get_randoms_for_chain_valuation(g["ttms"], int(g["nb_path"]), int(g["n_per_year"]), int(g["seed"]))
    np.testing.assert_array_equal(np.array(dts), g["dts"])
    np.testing.assert_array_equal(W0s[0][0, :3], g["W0_head"])
    s0, th, k1, k2, b, vv = g["params"]
    p, e, st = logsv_mc_chain_pricer_fixed_randoms(g["ttms"], g["forwards"], g["discfactors"], strikes, types, W0s, W1s, dts, s0, th, k1,
                                                   k2, b, vv, g["etas"], bool(g["is_spot"]), VariableType(int(g["variable_type"])), True)
    for m in range(int(g["nslices"])):
        for a, name in zip(st[m], ("x", "sigma", "qvar")):
            np.testing.assert_allclose(a, g[f"{name}_{m}"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(p[m], g[f"prices_{m}"], rtol=1e-9, atol=1e-13)      # 1/S payoffs amplify 1e-16 to ~1e-11
        np.testing.assert_allclose(e[m], g[f"stderr_{m}"], rtol=1e-8, atol=1e-13)


@pytest.mark.parametrize("tag", ["dflt", "floor"])
def test_heston_fixed_randoms_vs_reference_golden(cuda_lib, tag):
    from stochvolmodels_b200.pricers.heston_pricer import simulate_heston_x_vol_terminal
    from stochvolmodels_b200.utils.mc_payoffs import compute_mc_vars_payoff
    g = load_golden(f"heston_mc_fixed_{tag}.npz")
    N, S = int(g["nb_path"]), int(g["nsteps"])
    rng = np.random.RandomState(int(g["seed"]))
    W0, W1 = rng.normal(0, 1, size=(S, N)), rng.normal(0, 1, size=(S, N))
    v0, theta, kappa, rho, volvol = g["params"]
    x, v, q = simulate_heston_x_vol_terminal(float(g["ttm"]), np.zeros(1), v0 * np.ones(1), np.zeros(1), theta, kappa, rho, volvol,
                                             nb_path=N, W0=W0, W1=W1, dt=float(g["dt"]))
    np.testing.assert_allclose(x, g["x"], rtol=0, atol=1e-13)
    np.testing.assert_allclose(v, g["var"], rtol=0, atol=1e-13)
    np.testing.assert_allclose(q, g["qvar"], rtol=0, atol=1e-13)
    p, e = compute_mc_vars_payoff(x, np.sqrt(v), q, float(g["ttm"]), float(g["forward"]), g["strikes"], g["types"], float(g["discfactor"]))
    np.testing.assert_allclose(p, g["prices"], rtol=1e-11)
    np.testing.assert_allclose(e, g["stderr"], rtol=1e-9)


def test_payoffs_vs_reference_golden_incl_nan_paths(cuda_lib):
    from stochvolmodels_b200.utils.config import VariableType
    from stochvolmodels_b200.utils.mc_payoffs import compute_mc_vars_payoff
    g = load_golden("payoffs.npz")
    kw = dict(sigma0=np.ones(1), ttm=float(g["ttm"]), forward=float(g["forward"]), discfactor=float(g["discfactor"]))
    for xs, suf in (("x", ""), ("x_nan", "_nan")):
        p, e = compute_mc_vars_payoff(x0=g[xs], qvar0=g["qvar"], strikes_ttm=g["strikes"], optiontypes_ttm=g["types"], **kw)
        np.testing.assert_allclose(p, g["prices" + suf], rtol=1e-12)
        np.testing.assert_allclose(e, g["stderr" + suf], rtol=1e-10)
        p, e = compute_mc_vars_payoff(x0=g[xs], qvar0=g["qvar"], strikes_ttm=g["qstrikes"], optiontypes_ttm=g["qtypes"],
                                      variable_type=VariableType.Q_VAR, **kw)
        np.testing.assert_allclose(p, g["qprices" + suf], rtol=1e-12)
        np.testing.assert_allclose(e, g["qstderr" + suf], rtol=1e-10)
    with pytest.raises(ValueError, match="payoff"):                       # utils/mc_payoffs.py:83-84
        compute_mc_vars_payoff(x0=g["x"], qvar0=g["qvar"], strikes_ttm=np.ones(1), optiontypes_ttm=np.array(["BAD"]), **kw)
    with pytest.raises(NotImplementedError):                              # utils/mc_payoffs.py:69-70
        compute_mc_vars_payoff(x0=g["x"], qvar0=g["qvar"], strikes_ttm=np.ones(1), optiontypes_ttm=np.array(["C"]),
                               variable_type=VariableType.SIGMA, **kw)


def test_device_normals_match_oracle_restatement(cuda_lib):
    from stochvolmodels_b200 import _capi as C, engine
    ids = 123456789012 + np.arange(4096)            # exercises the high counter word
    for slice_idx, nsteps in ((0, 5), (3, 8)):
        z0, z1 = engine.device_normals(10, int(ids[0]), ids.shape[0], slice_idx, nsteps, C.GAUSS_F64)
        o0, o1 = mc.device_normals(10, ids, slice_idx, nsteps, "f64")
        np.testing.assert_allclose(z0, o0, rtol=0, atol=5e-15)
        np.testing.assert_allclose(z1, o1, rtol=0, atol=5e-15)
        z0, z1 = engine.device_normals(10, int(ids[0]), ids.shape[0], slice_idx, nsteps, C.GAUSS_F32)
        o0, o1 = mc.device_normals(10, ids, slice_idx, nsteps, "f32")
        np.testing.assert_allclose(z0, o0, rtol=0, atol=2e-5)          # SFU lg2/sin/cos vs libm float
        np.testing.assert_allclose(z1, o1, rtol=0, atol=2e-5)
        p0, p1 = engine.device_normals(10, int(ids[0]), ids.shape[0], slice_idx, nsteps, C.GAUSS_F64_PAIRED)
        o0, o1 = mc.device_normals(10, ids, slice_idx, nsteps, "f64_paired")
        np.testing.assert_allclose(p0, o0, rtol=0, atol=5e-15)         # same 32-bit uniforms, fp64 arithmetic
        np.testing.assert_allclose(p1, o1, rtol=0, atol=5e-15)
        np.testing.assert_allclose(z0, p0, rtol=0, atol=2e-5)          # ... which the SFU float draws approximate
        np.testing.assert_allclose(z1, p1, rtol=0, atol=2e-5)
    z = np.concatenate([a.ravel() for a in engine.device_normals(99, 0, 1 << 20, 0, 4, C.GAUSS_F32)])
    n = z.size
    assert abs(z.mean()) < 4 / np.sqrt(n) and abs(z.var() - 1) < 4 * np.sqrt(2 / n) and abs(np.mean(z ** 4) - 3) < 4 * np.sqrt(96 / n)


@pytest.mark.parametrize("gauss", ["fp64", "fp32"])
@pytest.mark.parametrize("is_spot", [True, False])
def test_fused_logsv_kernel_vs_oracle_same_normals(cuda_lib, gauss, is_spot):
    """terminal states and chain prices of the fused Philox kernel == numpy oracle stepper fed with the kernel's own normals."""
    from stochvolmodels_b200 import _capi as C, engine
    N, npy, seed = 20000, 252, 4242
    params = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)
    ttms, fw, df, etas = np.array([0.1, 0.3, 0.35]), np.array([1.0, 1.02, 1.03]), np.array([0.999, 0.99, 0.98]), np.array([0.9, 1.1, 1.0])
    types = [T5, T5, T5] if is_spot else [np.array(["IP", "IP", "IC", "IC", "IC"])] * 3
    flags = engine.mc_flags("fp64", gauss)
    steps = mc.chain_steps(ttms, npy)
    Z = [engine.device_normals(seed, 0, N, m, steps[m][0], flags) for m in range(3)]
    po, eo, st = mc.logsv_mc_chain_fixed(params, ttms, fw, df, [K5] * 3, types, etas, [z[0] for z in Z], [z[1] for z in Z],
                                         [d for _, d in steps], is_spot, 1, True)
    pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*params), ttms, fw, df, etas, [K5] * 3, types, N, npy, is_spot, 1, seed, flags)
    for m in range(3):
        np.testing.assert_allclose(pg[m], po[m], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(eg[m], eo[m], rtol=1e-8, atol=1e-12)
    # single slice terminal values: paths themselves
    x, s, q = engine.logsv_terminal(engine.logsv_params_c(*params), 0.1, N, npy, is_spot, 0.9, seed, flags)
    np.testing.assert_allclose(x, st[0][0], rtol=0, atol=1e-11)
    np.testing.assert_allclose(s, st[0][1], rtol=1e-11, atol=0)
    np.testing.assert_allclose(q, st[0][2], rtol=0, atol=1e-11)


@pytest.mark.parametrize("gauss", ["fp64", "fp32"])
def test_fused_heston_kernel_vs_oracle_same_normals(cuda_lib, gauss):
    from stochvolmodels_b200 import engine
    N, npy, seed = 20000, 360, 777
    params = (0.01, 0.02, 1.0, -0.7, 1.0)           # Feller violated -> floor binds
    ttms, fw, df = np.array([0.2, 0.5]), np.array([1.0, 1.01]), np.array([0.995, 0.98])
    flags = engine.mc_flags("fp64", gauss)
    steps = mc.chain_steps(ttms, npy)
    Z = [engine.device_normals(seed, 0, N, m, steps[m][0], flags) for m in range(2)]
    po, eo, st = mc.heston_mc_chain_fixed(params, ttms, fw, df, [K5] * 2, [T5] * 2, [z[0] for z in Z], [z[1] for z in Z],
                                          [d for _, d in steps], 1, True)
    pg, eg = engine.heston_mc_chain(engine.heston_params_c(*params), ttms, fw, df, [K5] * 2, [T5] * 2, N, npy, 1, seed, flags)
    for m in range(2):
        np.testing.assert_allclose(pg[m], po[m], rtol=1e-9, atol=1e-13)
        np.testing.assert_allclose(eg[m], eo[m], rtol=1e-8, atol=1e-13)
    x, v, q = engine.heston_terminal(engine.heston_params_c(*params), 0.2, N, npy, seed, flags)
    np.testing.assert_allclose(x, st[0][0], rtol=0, atol=1e-11)
    np.testing.assert_allclose(v, st[0][1], rtol=0, atol=1e-12)
    assert v.min() >= 1e-4 and np.isclose(v.min(), 1e-4)


def test_large_n_fp64_chain_vs_c_port(cuda_lib):
    """1e6 paths x BTC chain: GPU (all-fp64 mode) vs the C port of the reference algorithm on the same Philox stream."""
    from stochvolmodels_b200 import engine, get_btc_test_chain_data
    chain = get_btc_test_chain_data()
    params = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)
    N, npy, seed = 1_000_000, 252, 31337
    pc, ec = cport.mc_chain("logsv", params, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms,
                            chain.optiontypes_ttms, N, npy, True, 1, seed, "f64")
    pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*params), chain.ttms, chain.forwards, chain.discfactors, None,
                                   chain.strikes_ttms, chain.optiontypes_ttms, N, npy, True, 1, seed, engine.mc_flags("fp64", "fp64"))
    for m in range(4):
        np.testing.assert_allclose(pg[m], pc[m], rtol=1e-9)
        np.testing.assert_allclose(eg[m], ec[m], rtol=1e-8)


@pytest.mark.parametrize("model,N", [("logsv", 4_000_003), ("heston", 500_001)])
def test_large_n_fp64_chain_vs_c_port_multi_launch_driver(cuda_lib, model, N):
    """BTC chain, as test_large_n_fp64_chain_vs_c_port, at path counts just above the cooperative driver's limits (4e6 LogSV, 5e5 Heston):
    the multi-launch driver (slice kernel, stand-alone payoff kernels, reductions) against the C port on the same Philox stream.  The LogSV
    case gives slice 2 mixed C / P / IC / IP codes, so the general payoff kernel runs next to the vanilla one."""
    from stochvolmodels_b200 import engine, get_btc_test_chain_data
    chain = get_btc_test_chain_data()
    seed, flags = 31337, engine.mc_flags("fp64", "fp64")
    types = list(chain.optiontypes_ttms)
    if model == "logsv":
        types[2] = np.array(["C", "P", "IC", "IP"] * 4)[:len(chain.strikes_ttms[2])]
        params, npy = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458), 252
        pc, ec = cport.mc_chain("logsv", params, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms, types, N, npy, True, 1,
                                seed, "f64")
        pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*params), chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms,
                                       types, N, npy, True, 1, seed, flags)
    else:
        params, npy = (0.04, 0.04, 4.0, -0.5, 0.4), 360
        pc, ec = cport.mc_chain("heston", params, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms, types, N, npy, True, 1,
                                seed, "f64")
        pg, eg = engine.heston_mc_chain(engine.heston_params_c(*params), chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, types,
                                        N, npy, 1, seed, flags)
    for m in range(4):
        np.testing.assert_allclose(pg[m], pc[m], rtol=1e-9)
        np.testing.assert_allclose(eg[m], ec[m], rtol=1e-8)


def test_small_n_same_normals_tests_on_the_multi_launch_driver(cuda_lib):
    """The same-normals chain tests run at path counts the cooperative driver serves.  Re-run them in a process that forces the
    multi-launch driver (B200SV_CHAIN_COOP=0; the choice is cached per process): at 1 to 20000 paths most of its CTAs are empty, which
    is where the vanilla payoff kernel's per-CTA path count and the grid / strike-chunk split matter."""
    import os
    import subprocess
    import sys
    from conftest import ROOT
    tests = ["fused_logsv_kernel_vs_oracle_same_normals", "fused_heston_kernel_vs_oracle_same_normals",
             "edge_cases_ragged_chain_many_strikes_single_step_tiny_path_counts", "qvar_payoffs_in_fused_chain"]
    env = dict(os.environ, B200SV_CHAIN_COOP="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.join("tests", "test_gpu_mc.py"),
                        "-k", " or ".join(tests)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "8 passed" in r.stdout, r.stdout[-2000:]


def _assert_within_3se(p_gpu, se_gpu, p_ref, se_ref, what):
    """MC-vs-MC gate.  z uses the combined standard error of the two independent samples.  Every strike must be within 4 SE
    (the reference's own bar: tests/test_logsv_characterization.py:407, test_heston_characterization.py:292) and at least 90% of
    the strikes of a slice within the 3 SE the north_star / docs/analytic_vs_monte_carlo.md:19-20 quote -- strikes of one slice
    share the same paths, so a single ~3-sigma fluctuation of the reference sample moves several of them together (DESIGN.md §6)."""
    z = np.abs(p_gpu - p_ref) / np.sqrt(se_gpu ** 2 + se_ref ** 2)
    assert np.all(z < 4.0), (what, z)
    assert np.mean(z < 3.0) >= 0.9 or z.size < 10 and np.sum(z >= 3.0) <= 1, (what, z)


@pytest.mark.parametrize("precision,gauss", [("fp64", "fp32"), ("fp64", "fp64"), ("fp32", "fp32")])
def test_logsv_mc_within_3se_of_reference_mc_quickstart(cuda_lib, precision, gauss):
    """north_star gate: Philox MC within 3 MC standard errors of the reference Numba CPU path (golden refmc: the reference's
    own stepper + payoffs at 4e6 paths), and <= 1e-3 abs from the reference Fourier price.  MC-vs-Fourier is NOT a 3-SE test at
    these path counts: the Euler scheme's discretisation bias is ~2-4 SE with any generator (see make_golden.reference_mc)."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    ref = load_golden("refmc_logsv_quickstart.npz")
    fourier = load_golden("logsv_fourier_g1_quickstart.npz")
    chain = OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    prices, ses = LogSVPricer().model_mc_price_chain(chain, LogSvParams(*Q), nb_path=4_000_000, nb_steps=252, seed=2024,
                                                     precision=precision, gauss=gauss)
    for m in range(2):
        _assert_within_3se(prices[m], ses[m], ref[f"prices_{m}"], ref[f"stderr_{m}"], (precision, gauss, m))
        # SE * sqrt(N) is a property of the payoff distribution: same scale as the reference's (fat tails make it noisy)
        np.testing.assert_allclose(ses[m] * np.sqrt(4_000_000), ref[f"stderr_{m}"] * np.sqrt(float(ref["nb_path"])), rtol=0.25)
        assert np.all(np.abs(prices[m] - fourier[f"prices_{m}"]) < 1e-3)


def test_logsv_mc_btc_chain_within_3se_of_reference_mc(cuda_lib):
    """BASELINE config 4 shape: 1e7 paths, full BTC chain, every one of the 49 strikes."""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, get_btc_test_chain_data
    ref = load_golden("refmc_logsv_btc.npz")
    fourier = load_golden("logsv_fourier_btc.npz")
    chain = get_btc_test_chain_data()
    prices, ses = LogSVPricer().model_mc_price_chain(chain, LOGSV_BTC_PARAMS, nb_path=10_000_000, nb_steps=252, seed=7)
    for m in range(4):
        _assert_within_3se(prices[m], ses[m], ref[f"prices_{m}"], ref[f"stderr_{m}"], m)
        assert np.all(np.abs(prices[m] - fourier[f"prices_{m}"]) / chain.forwards[m] < 1e-3)


def test_logsv_mc_btc_chain_strict_3se_at_1e8_paths(cuda_lib):
    """the north_star's bar without softening: every one of the 49 strikes of the BTC chain within 3 (combined) MC standard errors of the
    reference's own Numba MC (golden: 16e6 reference paths), with the GPU estimate at 1e8 paths (its own error is 2.5x smaller than the
    reference sample's), default arithmetic (fp64 state, float draws) and the all-fp64 mode; abs error vs the reference Fourier prices <= 1e-3 F"""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, get_btc_test_chain_data
    ref = load_golden("refmc_logsv_btc.npz")
    fourier = load_golden("logsv_fourier_btc.npz")
    chain = get_btc_test_chain_data()
    for gauss, seed in (("fp32", 10), ("fp64", 11)):
        prices, ses = LogSVPricer().model_mc_price_chain(chain, LOGSV_BTC_PARAMS, nb_path=100_000_000, nb_steps=252, seed=seed, gauss=gauss)
        zmax = 0.0
        for m in range(4):
            z = np.abs(prices[m] - ref[f"prices_{m}"]) / np.sqrt(ses[m] ** 2 + ref[f"stderr_{m}"] ** 2)
            zmax = max(zmax, float(z.max()))
            assert np.all(z < 3.0), (gauss, m, z)
            assert np.all(np.abs(prices[m] - fourier[f"prices_{m}"]) / chain.forwards[m] < 1e-3)
        print(f"BTC chain, 1e8 GPU paths ({gauss} draws) vs 16e6-path reference Numba MC: max z over 49 strikes = {zmax:.2f}")


def test_heston_mc_within_3se_of_reference_mc(cuda_lib):
    from stochvolmodels_b200 import HestonParams, HestonPricer, OptionChain
    ref = load_golden("refmc_heston_g4.npz")
    fourier = load_golden("heston_fourier_g4.npz")
    chain = OptionChain(ttms=np.array([0.25, 1.0]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    prices, ses = HestonPricer().model_mc_price_chain(chain, HestonParams(), nb_path=4_000_000, seed=5)
    for m in range(2):
        _assert_within_3se(prices[m], ses[m], ref[f"prices_{m}"], ref[f"stderr_{m}"], m)
        assert np.all(np.abs(prices[m] - fourier[f"prices_{m}"]) < 1e-3)


def test_terminal_moments_and_api(cuda_lib):
    """E[e^x] = 1 under the MMA measure, finite positive vols (reference tests/test_logsv_characterization.py:442-458)."""
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer
    x, s, q = LogSVPricer().simulate_terminal_values(LogSvParams(*Q), ttm=0.25, nb_path=2_000_000, seed=11)
    assert x.shape == s.shape == q.shape == (2_000_000,) and x.dtype == np.float64
    ex = np.exp(x)
    assert abs(ex.mean() - 1.0) < 4 * ex.std() / np.sqrt(x.size)
    assert np.all(s > 0) and np.all(q > 0) and np.all(np.isfinite(x))
    x2, s2, q2 = LogSVPricer().simulate_terminal_values(LogSvParams(*Q), ttm=0.25, nb_path=2_000_000, seed=11)
    np.testing.assert_array_equal(x, x2)                       # same seed replays bit-for-bit
    x3, _, _ = LogSVPricer().simulate_terminal_values(LogSvParams(*Q), ttm=0.25, nb_path=1000, seed=12)
    assert not np.array_equal(x3, x[:1000])
    xh, vh, qh = HestonPricer().simulate_terminal_values(HestonParams(), ttm=1.0, nb_path=1_000_000, seed=3)
    assert vh.min() >= 1e-4 and abs(np.exp(xh).mean() - 1.0) < 4 * np.exp(xh).std() / 1000.0
    assert abs(qh.mean() - 0.04) < 1e-3                         # E[int v dt] = theta*T when v0 = theta


def test_path_offset_makes_shards_consistent(cuda_lib):
    """device-level API: two half-ranges with path offsets reproduce the unsharded terminal states bit-for-bit."""
    import torch
    from ctypes import byref, c_void_p
    from stochvolmodels_b200 import _capi as C, engine
    N = 100_000
    pc = engine.logsv_params_c(*Q)
    def run(n, off):
        st = torch.empty((3, n), dtype=torch.float64, device="cuda")
        mom = torch.zeros(2, dtype=torch.float64, device="cuda")
        C.call("b200sv_dev_logsv_slice", c_void_p(st[0].data_ptr()), c_void_p(st[1].data_ptr()), c_void_p(st[2].data_ptr()), n, off, 1,
               byref(pc), 1.0, 1, 64, 0.25 / 64, 0, 1.0, 10, 0, c_void_p(mom.data_ptr()), None, c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return st.cpu().numpy(), mom.cpu().numpy()
    full, mfull = run(N, 0)
    a, ma = run(N // 2, 0)
    b, mb = run(N - N // 2, N // 2)
    np.testing.assert_array_equal(np.concatenate([a, b], axis=1), full)
    np.testing.assert_allclose(ma + mb, mfull, rtol=1e-13)
    assert mfull[1] == N


def test_logsv_vol_paths_vs_reference_golden(cuda_lib):
    """simulate_vol_paths (SURVEY.md §8f #4a): fixed increments == reference; Philox draws == oracle fed with the device normals."""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, engine, _capi as C
    from stochvolmodels_b200.pricers.logsv_pricer import simulate_vol_paths
    g = load_golden("logsv_vol_paths.npz")
    S, dt = mc.set_time_grid(0.1, 360)
    W = np.sqrt(dt) * np.random.RandomState(5).normal(0, 1, size=(S, 500))
    for tag, spot in (("mma", True), ("inv", False)):
        sig, grid_t = simulate_vol_paths(0.1, *g["params"], is_spot_measure=spot, nb_path=500, nb_steps_per_year=360, brownians=W)
        np.testing.assert_allclose(sig, g[f"sigma_t_{tag}"], rtol=0, atol=1e-12)
        np.testing.assert_array_equal(grid_t, g[f"grid_t_{tag}"])
    sig, grid_t = LogSVPricer().simulate_vol_paths(params=LOGSV_BTC_PARAMS, ttm=0.02, nb_path=4, seed=1)
    assert sig.shape == tuple(g["method_shape"]) and np.all(sig > 0) and np.all(sig[0] == LOGSV_BTC_PARAMS.sigma0)
    np.testing.assert_array_equal(grid_t, g["method_grid"])
    # Philox route: Z0 of the fp64 stream, slice 0
    N, seed = 3000, 9
    z0, _ = engine.device_normals(seed, 0, N, 0, S, C.GAUSS_F64)
    sig, _ = simulate_vol_paths(0.1, *g["params"], nb_path=N, nb_steps_per_year=360, seed=seed)
    np.testing.assert_allclose(sig, mc.logsv_vol_paths(*g["params"], np.sqrt(dt) * z0, dt, True), rtol=0, atol=1e-11)


def test_device_resident_fixed_randoms_chain(cuda_lib):
    """calibration inner loop shape (reference :1100-1162): W0s/W1s resident in HBM, same prices as the host-array path and as the
    reference golden; re-pricing with other parameters reuses the resident normals."""
    from stochvolmodels_b200.pricers.logsv_pricer import DeviceRandoms, get_randoms_for_chain_valuation, logsv_mc_chain_pricer_fixed_randoms
    g = load_golden("logsv_mc_fixed_btc_small.npz")
    strikes, types = chain_from_golden(g)
    rnd = get_randoms_for_chain_valuation(g["ttms"], int(g["nb_path"]), int(g["n_per_year"]), int(g["seed"]), device="cuda")
    assert isinstance(rnd, DeviceRandoms) and rnd.nbytes() == 2 * 8 * int(g["nb_path"]) * int(np.sum(g["nsteps"]))
    s0, th, k1, k2, b, vv = g["params"]
    p, e = logsv_mc_chain_pricer_fixed_randoms(g["ttms"], g["forwards"], g["discfactors"], strikes, types, rnd, v0=s0, theta=th, kappa1=k1,
                                               kappa2=k2, beta=b, volvol=vv, vol_backbone_etas=g["etas"], is_spot_measure=bool(g["is_spot"]))
    for m in range(int(g["nslices"])):
        np.testing.assert_allclose(p[m], g[f"prices_{m}"], rtol=1e-9, atol=1e-13)
        np.testing.assert_allclose(e[m], g[f"stderr_{m}"], rtol=1e-8, atol=1e-13)
    ps, es = logsv_mc_chain_pricer_fixed_randoms(g["ttms"], g["forwards"], g["discfactors"], strikes, types, rnd, v0=s0, theta=th, kappa1=k1,
                                                 kappa2=k2, beta=b, volvol=vv, vol_backbone_etas=g["etas"], fast=False)
    for m in range(int(g["nslices"])):
        np.testing.assert_allclose(ps[m], p[m], rtol=1e-11, atol=1e-13)          # throughput vs strict stepper
        np.testing.assert_allclose(ps[m], g[f"prices_{m}"], rtol=1e-10, atol=1e-13)
    p2, _ = logsv_mc_chain_pricer_fixed_randoms(g["ttms"], g["forwards"], g["discfactors"], strikes, types, rnd, v0=s0 * 1.01, theta=th,
                                                kappa1=k1, kappa2=k2, beta=b, volvol=vv, vol_backbone_etas=g["etas"])
    assert np.all(np.abs(p2[0] / p[0] - 1) < 0.1) and not np.allclose(p2[0], p[0], rtol=1e-6)


def test_heston_qe_scheme(cuda_lib):
    """opt-in Andersen QE (BASELINE.json config 2; not in the reference): (i) terminal states == oracle restatement fed with the kernel's
    normals, incl. a Feller-violating case that exercises the exponential branch; (ii) 1e6 paths x 252 steps (config 2 shape) within
    3 SE of the reference's Heston Fourier price (golden G4) -- QE's discretisation bias is far below the MC error."""
    from stochvolmodels_b200 import HestonParams, HestonPricer, OptionChain, _capi as C, engine
    N, seed = 20000, 4321
    for params, ttm, npy in (((0.04, 0.04, 4.0, -0.5, 0.4), 0.5, 100), ((0.01, 0.02, 1.0, -0.7, 1.0), 0.5, 50)):
        S, dt = mc.set_time_grid(ttm, npy)
        flags = engine.mc_flags("fp64", "fp64")
        Z0, Z1 = engine.device_normals(seed, 0, N, 0, S, flags)
        xo, vo, qo = mc.heston_qe_step_fixed(np.zeros(N), params[0] * np.ones(N), np.zeros(N), Z0, Z1, dt, params[1], params[2], params[3], params[4])
        x, v, q = engine.heston_terminal(engine.heston_params_c(*params), ttm, N, npy, seed, flags, C.HESTON_QE)
        np.testing.assert_allclose(x, xo, rtol=0, atol=1e-10)
        np.testing.assert_allclose(v, vo, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(q, qo, rtol=0, atol=1e-11)
        assert v.min() >= 0.0
    assert (vo == 0.0).any()                                   # the exponential branch produced exact zeros in the second case
    g = load_golden("heston_fourier_g4.npz")
    chain = OptionChain(ttms=np.array([1.0]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[T5])
    prices, ses = HestonPricer().model_mc_price_chain(chain, HestonParams(), nb_path=1_000_000, nb_steps_per_year=251, seed=17, scheme="qe")
    z = (prices[0] - g["prices_1"]) / ses[0]
    assert np.all(np.abs(z) < 3.0), z
    with pytest.raises(ValueError):
        HestonPricer().model_mc_price_chain(chain, HestonParams(), nb_path=1000, scheme="milstein")


def test_edge_cases_ragged_chain_many_strikes_single_step_tiny_path_counts(cuda_lib):
    """ragged chain: a 21-strike slice (3 register chunks) with mixed inverse codes, an EMPTY slice (J = 0 through the C ABI), a
    single-step slice (ttm gap * n < 1), path counts 1 / 33 / 257 (not multiples of the warp or CTA size), odd step counts."""
    from stochvolmodels_b200 import engine
    params = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)
    K21 = np.linspace(0.5, 1.5, 21)
    T21 = np.array(["IP", "P", "IC", "C"] * 5 + ["IC"])
    ttms = np.array([0.002, 0.05, 0.051, 0.2])           # 360/yr: steps 1, 18, 1, 54
    fw, df = np.array([1.0, 1.01, 1.01, 1.02]), np.array([1.0, 0.999, 0.999, 0.99])
    strikes = [K21, np.zeros(0), K5, K21[:9]]
    types = [T21, np.zeros(0, dtype="<U2"), T5, T21[:9]]
    steps = mc.chain_steps(ttms, 360)
    assert [s for s, _ in steps] == [1, 18, 1, 54]
    for N in (1, 33, 257, 5000):
        for gauss in ("fp64", "fp32"):
            flags = engine.mc_flags("fp64", gauss)
            Z = [engine.device_normals(5, 0, N, m, steps[m][0], flags) for m in range(4)]
            po, eo = mc.logsv_mc_chain_fixed(params, ttms, fw, df, [K21, K5[:0], K5, K21[:9]], [T21, T5[:0], T5, T21[:9]], np.ones(4),
                                             [z[0] for z in Z], [z[1] for z in Z], [d for _, d in steps], False, 1)
            pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*params), ttms, fw, df, None, strikes, types, N, 360, False, 1, 5, flags)
            assert [len(p) for p in pg] == [21, 0, 5, 9]
            for m in (0, 2, 3):
                np.testing.assert_allclose(pg[m], po[m], rtol=1e-8, atol=1e-11)
                # one-pass population variance (sum p^2 / n - mean^2): absolute floor sqrt(eps)*|mean|/sqrt(N), visible only when the
                # sample variance is ~0 (N = 1); numpy's two-pass nanstd returns exactly 0 there (DESIGN.md §3.5)
                np.testing.assert_allclose(eg[m], eo[m], rtol=1e-7, atol=1e-11 + 3e-8 * np.max(np.abs(po[m])) / np.sqrt(N))


def test_qvar_payoffs_in_fused_chain(cuda_lib):
    """MC options on quadratic variance through the fused chain (variable_type = Q_VAR): vanilla and general payoff kernels."""
    from stochvolmodels_b200 import engine
    params = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
    ttms, N = np.array([0.25, 0.5]), 20000
    Kq = np.array([0.5, 0.8, 1.0, 1.2, 1.6])
    steps = mc.chain_steps(ttms, 252)
    flags = engine.mc_flags("fp64", "fp32")
    Z = [engine.device_normals(3, 0, N, m, steps[m][0], flags) for m in range(2)]
    for types in ([np.array(["C", "P", "C", "P", "C"])] * 2, [np.array(["C", "IC", "P", "IP", "C"])] * 2):
        po, eo = mc.logsv_mc_chain_fixed(params, ttms, np.ones(2), np.ones(2), [Kq, Kq], types, np.ones(2), [z[0] for z in Z],
                                         [z[1] for z in Z], [d for _, d in steps], True, mc.Q_VAR)
        pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*params), ttms, np.ones(2), np.ones(2), None, [Kq, Kq], types, N, 252, True, 2, 3, flags)
        for m in range(2):
            np.testing.assert_allclose(pg[m], po[m], rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(eg[m], eo[m], rtol=1e-8, atol=1e-12)


def test_full_size_properties_1e8_paths(cuda_lib):
    """BASELINE.json full size (1e8 paths x 252 steps, BTC chain) through size-independent properties: put-call parity is EXACT under the
    forward re-centring (C - P = df (F - K) for every strike), prices are bitwise reproducible for a seed, monotone in strike, standard errors
    scale as 1/sqrt(N), and every strike is within the north_star's 1e-3 (forward-normalised) of the reference Fourier price."""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, OptionChain, get_btc_test_chain_data
    btc = get_btc_test_chain_data()
    fourier = load_golden("logsv_fourier_btc.npz")
    calls = OptionChain(ttms=btc.ttms, forwards=btc.forwards, strikes_ttms=btc.strikes_ttms, optiontypes_ttms=[np.array(["C"] * len(k)) for k in btc.strikes_ttms])
    puts = OptionChain(ttms=btc.ttms, forwards=btc.forwards, strikes_ttms=btc.strikes_ttms, optiontypes_ttms=[np.array(["P"] * len(k)) for k in btc.strikes_ttms])
    N = 100_000_000
    pricer = LogSVPricer()
    pc, ec = pricer.model_mc_price_chain(calls, LOGSV_BTC_PARAMS, nb_path=N, nb_steps=582, seed=42)
    pp, ep = pricer.model_mc_price_chain(puts, LOGSV_BTC_PARAMS, nb_path=N, nb_steps=582, seed=42)
    pm, em = pricer.model_mc_price_chain(btc, LOGSV_BTC_PARAMS, nb_path=N, nb_steps=582, seed=42)
    pm2, _ = pricer.model_mc_price_chain(btc, LOGSV_BTC_PARAMS, nb_path=N, nb_steps=582, seed=42)
    ps, es = pricer.model_mc_price_chain(btc, LOGSV_BTC_PARAMS, nb_path=N // 100, nb_steps=582, seed=42)
    for m in range(4):
        F, K = btc.forwards[m], btc.strikes_ttms[m]
        np.testing.assert_allclose(pc[m] - pp[m], F - K, rtol=0, atol=2e-9 * F)            # exact parity (fp64 summation of 1e8 terms)
        np.testing.assert_array_equal(pm[m], pm2[m])                                          # same seed => same bits
        is_call = btc.optiontypes_ttms[m] == "C"
        np.testing.assert_allclose(pm[m], np.where(is_call, pc[m], pp[m]), rtol=1e-12)         # mixed chain == per-type chains
        assert np.all(np.diff(pc[m]) < 0) and np.all(np.diff(pp[m]) > 0)                       # monotone in strike
        np.testing.assert_allclose(es[m] / em[m], 10.0, rtol=0.05)                             # SE ~ 1/sqrt(N)
        assert np.all(np.abs(pm[m] - fourier[f"prices_{m}"]) / F < 1e-3)


def test_terminal_values_from_per_path_initial_arrays(cuda_lib):
    """simulate_logsv_x_vol_terminal with length-N x0 / sigma0 / qvar0 and in-kernel draws (reference :1007-1020): equals the oracle stepper
    fed with the kernel's own normals; a two-leg continuation (slice 0 then slice 1 from the first leg's state) equals the chain pricer's
    own slice sequence."""
    from stochvolmodels_b200 import _capi as C, engine
    from stochvolmodels_b200.pricers.logsv_pricer import simulate_logsv_x_vol_terminal
    N, npy, seed = 6000, 252, 77
    theta, kappa1, kappa2, beta, volvol = 1.0413, 3.1844, 3.058, 0.1514, 1.8458
    rs = np.random.RandomState(3)
    x0, s0, q0 = rs.normal(0, 0.1, N), np.exp(rs.normal(-0.2, 0.3, N)), rs.uniform(0, 0.05, N)
    ttm = 0.2
    S, dt = mc.set_time_grid(ttm, npy)
    for gauss, flag in (("fp64", C.GAUSS_F64), ("fp32", C.GAUSS_F32)):
        x, s, q = simulate_logsv_x_vol_terminal(ttm=ttm, x0=x0, sigma0=s0, qvar0=q0, theta=theta, kappa1=kappa1, kappa2=kappa2, beta=beta, volvol=volvol,
                                                vol_backbone_eta=0.9, is_spot_measure=False, nb_path=N, nb_steps_per_year=npy, seed=seed, gauss=gauss)
        Z0, Z1 = engine.device_normals(seed, 0, N, 0, S, flag)
        xo, so, qo = mc.logsv_step_fixed(x0.copy(), s0.copy(), q0.copy(), Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, 0.9, False)
        np.testing.assert_allclose(x, xo, rtol=0, atol=2e-11)
        np.testing.assert_allclose(s, so, rtol=2e-11, atol=0)
        np.testing.assert_allclose(q, qo, rtol=2e-11, atol=1e-14)
    assert x0[0] != x[0] and np.all(x0 == np.asarray(x0))                      # inputs untouched
    # continuation: leg 2 on sub-stream 1 from the state of leg 1 == oracle on the slice-1 normals
    x2, s2, q2 = simulate_logsv_x_vol_terminal(ttm=ttm, x0=x, sigma0=s, qvar0=q, theta=theta, kappa1=kappa1, kappa2=kappa2, beta=beta, volvol=volvol,
                                               vol_backbone_eta=0.9, is_spot_measure=False, nb_path=N, nb_steps_per_year=npy, seed=seed, gauss="fp32",
                                               slice_index=1)
    Z0, Z1 = engine.device_normals(seed, 0, N, 1, S, C.GAUSS_F32)
    xo, so, qo = mc.logsv_step_fixed(x.copy(), s.copy(), q.copy(), Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, 0.9, False)
    np.testing.assert_allclose(x2, xo, rtol=0, atol=2e-11)
    np.testing.assert_allclose(s2, so, rtol=2e-11, atol=0)


def test_host_level_calls_follow_set_stream(cuda_lib):
    """b200sv_set_stream: host-level calls run on the caller's stream (same results; the call synchronises that stream before returning)."""
    import torch
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, engine
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[T5])
    p = LogSvParams(1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
    base = LogSVPricer().model_mc_price_chain(chain, p, nb_path=50_000, nb_steps=252, seed=9)
    fourier = LogSVPricer().price_chain(chain, p)
    st = torch.cuda.Stream()
    engine.set_stream(st)
    try:
        assert cuda_lib.b200sv_get_stream() == st.cuda_stream
        on_stream = LogSVPricer().model_mc_price_chain(chain, p, nb_path=50_000, nb_steps=252, seed=9)
        fourier2 = LogSVPricer().price_chain(chain, p)
    finally:
        engine.set_stream(None)
    assert not cuda_lib.b200sv_get_stream()
    np.testing.assert_array_equal(on_stream[0][0], base[0][0])
    np.testing.assert_array_equal(on_stream[1][0], base[1][0])
    np.testing.assert_array_equal(fourier2[0], fourier[0])


def test_terminal_values_shards_concatenate_to_the_single_gpu_arrays(cuda_lib):
    """SURVEY.md 8e: simulate_terminal_values beyond one GPU returns per-GPU shards of the global path ids; three uneven shards == one run"""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer
    from stochvolmodels_b200.multi_gpu import shard_paths
    p, N = LogSvParams(*Q), 100_003
    full = LogSVPricer().simulate_terminal_values(p, ttm=0.3, nb_path=N, seed=21, distributed=False)
    parts = [LogSVPricer().simulate_terminal_values(p, ttm=0.3, nb_path=N, seed=21, path_range=shard_paths(N, 3, r)[::-1]) for r in range(3)]
    for k in range(3):
        np.testing.assert_array_equal(np.concatenate([part[k] for part in parts]), full[k])
    with pytest.raises(ValueError):
        LogSVPricer().simulate_terminal_values(p, ttm=0.3, nb_path=N, path_range=(0, 10))


def test_set_seed_reproduces_seedless_monte_carlo(cuda_lib):
    """reference usage `set_seed(123)` before MC (its tests/test_heston_characterization.py:282): seedless calls after the same set_seed
    return the same prices, consecutive seedless calls differ"""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, get_btc_test_chain_data, set_seed
    chain, pricer = get_btc_test_chain_data(), LogSVPricer()
    runs = []
    for _ in range(2):
        set_seed(123)
        runs.append([pricer.model_mc_price_chain(chain, LOGSV_BTC_PARAMS, nb_path=20000, nb_steps=100)[0] for _ in range(2)])
    set_seed(None)
    for a, b in zip(runs[0], runs[1]):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    assert not np.array_equal(runs[0][0][0], runs[0][1][0])
