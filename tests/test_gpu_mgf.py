"""GPU parity tests of the Fourier / MGF path (north_star: <= 1e-10 relative vs the reference CPU path)."""
import numpy as np
import pytest

from conftest import chain_from_golden, load_golden
from oracle import mgf

pytestmark = pytest.mark.gpu
K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])


@pytest.mark.parametrize("tag", ["g1_quickstart", "g2_inverse", "c3_5x21", "btc", "first_order", "backbone_inverse"])
def test_logsv_fourier_chain_vs_reference_golden(cuda_lib, tag):
    from stochvolmodels_b200 import engine
    g = load_golden(f"logsv_fourier_{tag}.npz")
    strikes, types = chain_from_golden(g)
    prices, a, lm = engine.logsv_price_chain(engine.logsv_params_c(*g["params"]), g["ttms"], g["forwards"], g["discfactors"], g["etas"],
                                             strikes, types, bool(g["is_spot"]), int(g["order"]), None, 1000, True)
    for m in range(int(g["nslices"])):
        np.testing.assert_allclose(a[m], g[f"a_t1_{m}"], rtol=0, atol=1e-11)
        np.testing.assert_allclose(lm[m], g[f"log_mgf_{m}"], rtol=0, atol=1e-11)
        np.testing.assert_allclose(prices[m], g[f"prices_{m}"], rtol=1e-10, atol=1e-13 * g["forwards"][m])


@pytest.mark.parametrize("tag", ["g4", "c3_5x21", "btc"])
def test_heston_fourier_chain_vs_reference_golden(cuda_lib, tag):
    from stochvolmodels_b200 import engine
    g = load_golden(f"heston_fourier_{tag}.npz")
    strikes, types = chain_from_golden(g)
    prices, lm = engine.heston_price_chain(engine.heston_params_c(*g["params"]), g["ttms"], g["forwards"], g["discfactors"], strikes, types,
                                           None, 1000, True)
    for m in range(int(g["nslices"])):
        np.testing.assert_allclose(lm[m], g[f"log_mgf_{m}"], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(prices[m], g[f"prices_{m}"], rtol=1e-10, atol=1e-13 * g["forwards"][m])


def test_single_maturity_grid_entry_points(cuda_lib):
    """compute_logsv_a_mgf_grid / compute_heston_mgf_grid with carried state == golden second slice."""
    from stochvolmodels_b200.pricers.heston_pricer import compute_heston_mgf_grid
    from stochvolmodels_b200.pricers.logsv.affine_expansion import ExpansionOrder, compute_logsv_a_mgf_grid
    g = load_golden("logsv_fourier_g1_quickstart.npz")
    s0, th, k1, k2, b, vv = g["params"]
    phi = g["phi"]
    z = np.zeros_like(phi)
    a1, lm1 = compute_logsv_a_mgf_grid(0.25, phi, z, z, s0, th, k1, k2, b, vv, expansion_order=ExpansionOrder.SECOND)
    a2, lm2 = compute_logsv_a_mgf_grid(0.25, phi, z, z, s0, th, k1, k2, b, vv, a_t0=a1)
    np.testing.assert_allclose(a1, g["a_t1_0"], atol=1e-11, rtol=0)
    np.testing.assert_allclose(lm2, g["log_mgf_1"], atol=1e-11, rtol=0)
    # MGF roots: log-MGF == 0 at Phi in {0, -1} under the MMA measure (reference tests/test_logsv_characterization.py:141-163)
    roots = np.array([0.0 + 0j, -1.0 + 0j])
    _, lm0 = compute_logsv_a_mgf_grid(0.25, roots, np.zeros(2, complex), np.zeros(2, complex), s0, th, k1, k2, b, vv)
    np.testing.assert_allclose(lm0, 0.0, atol=1e-14)
    with pytest.raises(NotImplementedError):
        compute_logsv_a_mgf_grid(0.25, phi, z, z, s0, th, k1, k2, b, vv, expansion_order=ExpansionOrder.ZERO)
    # solve_a_ode_grid / get_init_conditions_a: the two steps compute_logsv_a_mgf_grid is made of in the reference (:492-567)
    from stochvolmodels_b200 import VariableType
    from stochvolmodels_b200.pricers.logsv.affine_expansion import get_init_conditions_a, solve_a_ode_grid
    a0 = get_init_conditions_a(phi, z, z, 5, VariableType.LOG_RETURN)
    assert a0.shape == (phi.shape[0], 5) and not a0.any()
    np.testing.assert_array_equal(get_init_conditions_a(phi, z, phi, 3, VariableType.SIGMA)[:, 1], -phi)
    np.testing.assert_array_equal(solve_a_ode_grid(phi, z, 0.25, th, k1, k2, b, vv, a_t0=a0, expansion_order=ExpansionOrder.SECOND), a1)
    h = load_golden("heston_fourier_g4.npz")
    v0, theta, kappa, rho, volvol = h["params"]
    lm, a, bb = compute_heston_mgf_grid(v0, theta, kappa, volvol, rho, 0.25, h["phi"], np.zeros_like(h["phi"]))
    np.testing.assert_allclose(lm, h["log_mgf_0"], rtol=1e-12, atol=1e-12)
    lm, a, bb = compute_heston_mgf_grid(v0, theta, kappa, volvol, rho, 0.75, h["phi"], np.zeros_like(h["phi"]), a, bb)
    np.testing.assert_allclose(lm, h["log_mgf_1"], rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(a, h["a_t1_1"], rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(bb, h["b_t1_1"], rtol=1e-11, atol=1e-11)


@pytest.mark.parametrize("tag", ["mma", "inv"])
def test_fourier_sum_vs_reference_golden(cuda_lib, tag):
    from stochvolmodels_b200.utils.mgf_pricer import vanilla_slice_pricer_with_mgf_grid
    g = load_golden(f"fourier_sum_{tag}.npz")
    p = vanilla_slice_pricer_with_mgf_grid(g["log_mgf"], g["phi"], float(g["forward"]), g["strikes"], g["types"], float(g["discfactor"]), bool(g["is_spot"]))
    np.testing.assert_allclose(p, g["prices"], rtol=1e-12)
    # general branch (|Re phi| != 1/2) against the oracle
    phi = g["phi"] + (0.2 if tag == "mma" else -0.2)
    sgn = 1.0 if tag == "mma" else -1.0
    lm = 0.5 * 0.09 * 0.4 * (phi * phi + sgn * phi)
    p = vanilla_slice_pricer_with_mgf_grid(lm, phi, 1.5, g["strikes"], g["types"], 0.9, bool(g["is_spot"]))
    o = mgf.vanilla_slice_prices(lm, phi, 1.5, g["strikes"], g["types"], 0.9, bool(g["is_spot"]))
    np.testing.assert_allclose(p, o, rtol=1e-12)
    # nansum semantics: a NaN grid entry is skipped
    lm2 = g["log_mgf"].copy()
    lm2[17] = np.nan
    p = vanilla_slice_pricer_with_mgf_grid(lm2, g["phi"], float(g["forward"]), g["strikes"], g["types"], float(g["discfactor"]), bool(g["is_spot"]))
    o = mgf.vanilla_slice_prices(lm2, g["phi"], float(g["forward"]), g["strikes"], g["types"], float(g["discfactor"]), bool(g["is_spot"]))
    np.testing.assert_allclose(p, o, rtol=1e-12)


def test_error_conventions(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, VariableType
    from stochvolmodels_b200.utils.mgf_pricer import vanilla_slice_pricer_with_mgf_grid
    g = load_golden("fourier_sum_mma.npz")
    with pytest.raises(ValueError, match="not implemented"):          # MMA measure rejects inverse payoffs (utils/mgf_pricer.py:206-212)
        vanilla_slice_pricer_with_mgf_grid(g["log_mgf"], g["phi"], 1.5, g["strikes"][:1], np.array(["IC"]), 1.0, True)
    chain = OptionChain.slice_to_chain(0.25, 1.0, K5, T5)
    with pytest.raises(NotImplementedError):                          # pricers/logsv_pricer.py:733-734
        LogSVPricer().price_chain(chain, LogSvParams(1, 1, 5, 5, 0.2, 2), variable_type=VariableType.SIGMA)


def test_quickstart_through_pricer_api(cuda_lib):
    """examples/getting_started/quickstart.py:23-46 with the reference's asserted values (rtol 5e-6)."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    params = LogSvParams(sigma0=1.0, theta=1.0, kappa1=5.0, kappa2=5.0, beta=0.2, volvol=2.0)
    pricer = LogSVPricer()
    price, ivol = pricer.price_vanilla(params=params, ttm=0.25, forward=1.0, strike=1.0, optiontype="C")
    chain = OptionChain.get_uniform_chain(ttms=np.array([0.25, 0.5]), ids=np.array(["3m", "6m"]), forwards=np.array([1.0, 1.0]), strikes=K5)
    prices, ivols = pricer.compute_chain_prices_with_vols(option_chain=chain, params=params)
    np.testing.assert_allclose(price, 0.197331, rtol=5e-6, atol=1e-8)
    np.testing.assert_allclose(ivol, 0.999577, rtol=5e-6, atol=1e-8)
    np.testing.assert_allclose(prices[1][2], 0.275202, rtol=5e-6, atol=1e-8)
    np.testing.assert_allclose(ivols[1][2], 0.995757, rtol=5e-6, atol=1e-8)
    # price_chain == price_slice == price_vanilla (reference tests/test_logsv_characterization.py:101-138)
    sl, _ = pricer.price_slice(params=params, ttm=0.25, forward=1.0, strikes=K5, optiontypes=T5)
    np.testing.assert_allclose(sl, prices[0], rtol=0, atol=1e-14)
    assert abs(sl[2] - price) < 1e-14
    assert [p.shape for p in prices] == [(5,), (5,)] and all(p.dtype == np.float64 for p in prices)


def test_heston_pricer_api(cuda_lib):
    from stochvolmodels_b200 import HestonParams, HestonPricer, OptionChain, VariableType
    g = load_golden("heston_fourier_g4.npz")
    chain = OptionChain(ttms=np.array([0.25, 1.0]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    prices = HestonPricer().price_chain(chain, HestonParams(), variable_type=VariableType.LOG_RETURN, some_unknown_kwarg=1)
    for m in range(2):
        np.testing.assert_allclose(prices[m], g[f"prices_{m}"], rtol=1e-10, atol=1e-13)


# ---- SURVEY.md §8f rows #1 and #3 -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["mma", "inv"])
def test_logsv_qvar_fourier_chain_vs_reference_golden(cuda_lib, tag):
    """40,000 RK45 solves per maturity on the psi grid (the reference needs ~80 s per maturity)."""
    from stochvolmodels_b200 import LogSvParams, VariableType
    from stochvolmodels_b200.pricers.logsv_pricer import logsv_chain_pricer
    g = load_golden(f"logsv_fourier_qvar_{tag}.npz")
    K, T = g["strikes"], np.array(["C"] * len(g["strikes"]))
    prices, a, lm = logsv_chain_pricer(LogSvParams(*g["params"]), g["ttms"], np.ones(2), g["discfactors"], [K, K], [T, T],
                                       is_spot_measure=bool(g["is_spot"]), variable_type=VariableType.Q_VAR, return_grids=True)
    assert a.shape == (2, 40000, 5)
    for m in range(2):
        np.testing.assert_allclose(a[m][::40], g[f"a_sub_{m}"], rtol=0, atol=1e-10)
        np.testing.assert_allclose(lm[m][::40], g[f"log_mgf_sub_{m}"], rtol=0, atol=1e-10)
        np.testing.assert_allclose(prices[m], g[f"prices_{m}"], rtol=1e-10)
    with pytest.raises(ValueError, match="not implemented"):
        logsv_chain_pricer(LogSvParams(*g["params"]), g["ttms"][:1], np.ones(1), np.ones(1), [K], [np.array(["P"] * 5)],
                           variable_type=VariableType.Q_VAR)


def test_logsv_pdfs_vs_reference_golden(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, VariableType
    g = load_golden("logsv_pdfs.npz")
    for vt in (VariableType.LOG_RETURN, VariableType.Q_VAR, VariableType.SIGMA):
        pdf = LogSVPricer().logsv_pdfs(LogSvParams(*g["params"]), ttm=float(g["ttm"]), space_grid=g[f"grid_{vt.name}"], variable_type=vt)
        np.testing.assert_allclose(pdf, g[f"pdf_{vt.name}"], rtol=1e-9, atol=1e-12)


def test_heston_qvar_and_digitals_vs_reference_golden(cuda_lib):
    from stochvolmodels_b200 import VariableType
    from stochvolmodels_b200.pricers.heston_pricer import heston_chain_pricer
    from stochvolmodels_b200.utils.mgf_pricer import digital_slice_pricer_with_mgf_grid, slice_qvar_pricer_with_a_grid
    g = load_golden("heston_fourier_qvar.npz")
    K, T = g["strikes"], np.array(["C"] * len(g["strikes"]))
    v0, theta, kappa, rho, volvol = g["params"]
    prices = heston_chain_pricer(v0, theta, kappa, volvol, rho, g["ttms"], np.ones(2), [K, K], [T, T], g["discfactors"], variable_type=VariableType.Q_VAR)
    for m in range(2):
        np.testing.assert_allclose(prices[m], g[f"prices_{m}"], rtol=1e-10, atol=1e-14)
    for tag in ("neg", "pos"):
        d = load_golden(f"fourier_digital_{tag}.npz")
        p = digital_slice_pricer_with_mgf_grid(d["log_mgf"], d["phi"], float(d["forward"]), d["strikes"], d["types"], float(d["discfactor"]))
        np.testing.assert_allclose(p, d["prices"], rtol=1e-12)
    with pytest.raises(ValueError, match="not implemented"):
        digital_slice_pricer_with_mgf_grid(d["log_mgf"], d["phi"], 1.5, d["strikes"][:1], np.array(["IC"]))
    with pytest.raises(ValueError, match="not implemented"):
        slice_qvar_pricer_with_a_grid(d["log_mgf"], d["phi"], 0.25, d["strikes"][:1], np.array(["P"]), 1.0)


def test_gpu_black_implied_vols(cuda_lib):
    """the chain inversion kernel and the host bisection both within the exact-reference bar, and the reference's pinned quickstart vols; round trips."""
    from oracle import bsm
    from stochvolmodels_b200 import OptionChain, engine
    K = np.array([0.6, 0.9, 1.0, 1.1, 1.6])
    types = np.array(["P", "P", "C", "IC", "C"])
    ttms, fw, df = np.array([0.1, 0.5, 2.0]), np.array([1.0, 1.03, 0.97]), np.array([0.999, 0.97, 0.9])
    vols = [0.05, 0.2, 1.5]
    prices = [bsm.compute_bsm_vanilla_price(fw[m], K, ttms[m], vols[m], types, df[m]) for m in range(3)]
    iv = engine.bsm_implied_vols(ttms, fw, df, [K] * 3, [types] * 3, prices)
    host = bsm.infer_bsm_ivols_from_model_chain_prices(ttms, fw, df, [K] * 3, [types] * 3, prices)
    import ivol_cases as ic
    pytest.importorskip("mpmath")
    for m in range(3):
        # every quote against the exact implied vol of the fp64 quote as given (tests/ivol_cases.py), the far-OTM ones (~1e-12) included;
        # the host bisection meets the same bar
        c = dict(F=np.full(5, fw[m]), K=K, T=np.full(5, ttms[m]), D=np.full(5, df[m]), type=types, price=prices[m], vol=np.full(5, vols[m]))
        iv_star, bar = ic.reference(c)
        for got in (iv[m], host[m]):
            ratio, nan_mismatch, bad = ic.check(got, iv_star, bar)
            assert nan_mismatch.size == 0 and bad.size == 0, (m, ratio, got, iv_star)
        good = prices[m] > 1e-8
        np.testing.assert_allclose(iv[m][good], vols[m], rtol=1e-8)
    chain = OptionChain.slice_to_chain(0.25, 1.0, np.array([1.0, 1.0]), np.array(["C", "C"]))
    out = chain.compute_model_ivols_from_chain_data([np.array([0.197330882838064, 1.5])])[0]
    np.testing.assert_allclose(out[0], 0.999577, rtol=5e-6)            # examples/getting_started/quickstart.py:44
    assert np.isnan(out[1])                                              # above the no-arbitrage bound
    # the third-party entry points the reference re-exports, keyword for keyword (slice and chain form)
    import stochvolmodels_b200 as sv
    one = sv.infer_bsm_ivols_from_slice_prices(ttm=ttms[1], forward=fw[1], strikes=K, optiontypes=types, model_prices=prices[1], discfactor=df[1])
    np.testing.assert_array_equal(one, iv[1])
    whole = sv.infer_bsm_ivols_from_model_chain_prices(ttms=ttms, forwards=fw, discfactors=df, strikes_ttms=[K] * 3, optiontypes_ttms=[types] * 3,
                                                       model_prices_ttms=prices)
    np.testing.assert_array_equal(whole[2], iv[2])


def test_mc_chain_implied_vols_api(cuda_lib):
    """ModelPricer.compute_mc_chain_implied_vols (reference model_pricer.py:216-241): 7 lists, bands ordered."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    out = LogSVPricer().compute_mc_chain_implied_vols(chain, LogSvParams(1.0, 1.0, 5.0, 5.0, 0.2, 2.0), nb_path=200_000, nb_steps=252, seed=3)
    assert len(out) == 7
    prices, ups, downs, mid, up, down, ses = out
    for m in range(2):
        assert np.all(downs[m] <= prices[m]) and np.all(prices[m] <= ups[m])
        assert np.all(down[m] <= mid[m] + 1e-12) and np.all(mid[m] <= up[m] + 1e-12) and np.all(np.abs(mid[m] - 1.0) < 0.1)


def test_ode_terms_and_rhs_vs_reference_golden(cuda_lib):
    """func_a_ode_quadratic_terms / func_rhs (affine_expansion.py:67-205) on the GPU against the reference's own outputs (mlh.npz: FIRST and
    SECOND order, both measures, eta != 1, psi != 0): dense M / L / H from the kernels' row tables, the dense rhs, and the production
    sparse rhs<>() -- all three must tell the same story."""
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.logsv.affine_expansion import ExpansionOrder, func_a_ode_quadratic_terms, func_rhs
    g = load_golden("mlh.npz")
    theta, kappa1, kappa2, beta, volvol = g["params"]
    for k in range(int(g["ncases"])):
        order, spot, eta, pr, pi, sr, si = g[f"case{k}_in"]
        phi, psi = complex(pr, pi), complex(sr, si)
        M, L, H = func_a_ode_quadratic_terms(theta, kappa1, kappa2, beta, volvol, phi, psi, is_spot_measure=bool(spot),
                                             expansion_order=ExpansionOrder(int(order)), vol_backbone_eta=eta)
        np.testing.assert_allclose(M, g[f"case{k}_M"], rtol=0, atol=5e-15)
        np.testing.assert_allclose(L, g[f"case{k}_L"], rtol=1e-15, atol=5e-15)
        np.testing.assert_allclose(H, g[f"case{k}_H"], rtol=1e-15, atol=5e-15)
        n = M.shape[0]
        A = (np.arange(1, n + 1) * (0.1 - 0.05j)).astype(np.complex128)
        np.testing.assert_allclose(func_rhs(0.0, A, g[f"case{k}_M"], g[f"case{k}_L"], g[f"case{k}_H"]), g[f"case{k}_rhs"], rtol=1e-14, atol=1e-14)
        fast = engine.logsv_ode_rhs(np.array([phi]), np.array([psi]), A[None, :], engine.logsv_params_c(theta, theta, kappa1, kappa2, beta, volvol),
                                    eta, bool(spot), int(order))
        np.testing.assert_allclose(fast[0], g[f"case{k}_rhs"], rtol=1e-14, atol=1e-14)


@pytest.mark.parametrize("name", ["quick_first", "mild_second", "mild2_second_inverse"])
def test_semi_analytic_branch_vs_reference_golden(cuda_lib, name):
    """is_analytic=True (solve_analytic_ode_for_a, affine_expansion.py:306-384): a_t1 / log_mgf carried over three maturities and the chain
    prices against the reference's own outputs.  The reference forms exp(L dt) through LAPACK eig + inv, the kernel through a scaled Taylor
    series -- they agree to the conditioning of the reference's eigenvector matrix (measured <= 1e-9 on these sets)."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    from stochvolmodels_b200.pricers.logsv.affine_expansion import ExpansionOrder
    g = load_golden("logsv_analytic_branch.npz")
    sigma0, theta, k1, k2, beta, vv, order, spot = g[f"{name}_params"]
    p = LogSvParams(sigma0, theta, k1, k2, beta, vv)
    K, types, ttms = g["strikes"], g[f"{name}_types"], g["ttms"]
    chain = OptionChain(ttms=ttms, forwards=np.ones(3), strikes_ttms=[K] * 3, optiontypes_ttms=[types] * 3, discfactors=g["discfactors"])
    prices, grids = LogSVPricer().price_chain(chain, p, is_analytic=True, expansion_order=ExpansionOrder(int(order)), is_spot_measure=bool(spot),
                                              return_grids=True)
    for m in range(3):
        a, lm = grids[m]
        np.testing.assert_allclose(a[::8], g[f"{name}_a_{m}"], rtol=1e-8, atol=1e-10)
        np.testing.assert_allclose(lm[::8], g[f"{name}_lm_{m}"], rtol=1e-8, atol=1e-10)
        np.testing.assert_allclose(prices[m], g[f"{name}_prices"][m], rtol=1e-8, atol=1e-12)


def test_semi_analytic_branch_diverges_where_the_reference_does(cuda_lib):
    """quickstart parameters at SECOND order: the reference's unchecked fixed-point sweeps blow up beyond |phi| ~ 16 and it returns NaN for
    every strike.  The drop-in agrees with it on the convergent part of the grid, is non-finite in the divergent tail as well (which grid
    points of a chaotic iteration end up inf vs NaN is not comparable), and returns NaN prices -- it does not silently fall back to RK45."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    g = load_golden("logsv_analytic_branch.npz")
    assert np.all(np.isnan(g["quick_second_nan_prices"]))
    chain = OptionChain(ttms=g["ttms"], forwards=np.ones(3), strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["quick_second_nan_types"]] * 3)
    prices, grids = LogSVPricer().price_chain(chain, LogSvParams(1.0, 1.0, 5.0, 5.0, 0.2, 2.0), is_analytic=True, return_grids=True)
    assert np.all(np.isnan(np.concatenate(prices)))
    for m in range(3):
        ref, lm = g[f"quick_second_nan_lm_{m}"], grids[m][1][::8]
        first_bad = int(np.argmin(np.isfinite(ref)))
        assert first_bad > 40
        np.testing.assert_allclose(lm[: first_bad - 8], ref[: first_bad - 8], rtol=1e-6, atol=1e-8)      # converged region
        assert not np.all(np.isfinite(lm[first_bad:]))                                                     # diverged tail


@pytest.mark.parametrize("name", ["quick_second", "btc_second_inverse_eta", "mild_first"])
def test_bdf_branch_vs_reference_golden(cuda_lib, name):
    """is_stiff_solver=True: the CUDA clone of SciPy's BDF control law against the reference's own outputs (solve_ivp(method='BDF',
    jac=func_rhs_jac) per grid point, affine_expansion.py:229-303): a_t1 and log_mgf on 125 grid points carried over two maturities.
    Reproducing the reference here means reproducing its accepted steps, order changes and Newton iteration counts."""
    from stochvolmodels_b200.pricers.logsv.affine_expansion import ExpansionOrder, compute_logsv_a_mgf_grid
    g = load_golden("logsv_bdf_branch.npz")
    sigma0, theta, k1, k2, beta, vv, order, spot, eta = g[f"{name}_params"]
    phi = g[f"{name}_phi"]
    a = np.zeros((phi.shape[0], 3 if int(order) == 1 else 5), dtype=np.complex128)
    t0 = 0.0
    for m, ttm in enumerate(g["ttms"]):
        a, lm = compute_logsv_a_mgf_grid(ttm - t0, phi, np.zeros_like(phi), np.zeros_like(phi), sigma0, theta, k1, k2, beta, vv, a_t0=a,
                                         is_stiff_solver=True, expansion_order=ExpansionOrder(int(order)), is_spot_measure=bool(spot),
                                         vol_backbone_eta=eta)
        np.testing.assert_allclose(a, g[f"{name}_a_{m}"], rtol=1e-10, atol=1e-11)
        np.testing.assert_allclose(lm, g[f"{name}_lm_{m}"], rtol=1e-10, atol=1e-11)
        t0 = ttm


def test_bdf_branch_chain_prices_and_oracle(cuda_lib):
    """full-grid chain prices on the stiff branch vs the reference (quickstart parameters), and the kernel vs SciPy's BDF itself on a grid
    the goldens do not cover (Q_VAR transform variable psi != 0, inverse measure)"""
    from oracle import mgf as omgf
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    from stochvolmodels_b200.pricers.logsv.affine_expansion import ExpansionOrder, solve_a_ode_grid
    g = load_golden("logsv_bdf_branch.npz")
    chain = OptionChain(ttms=g["ttms"], forwards=np.ones(2), strikes_ttms=[g["strikes"]] * 2, optiontypes_ttms=[g["types"]] * 2, discfactors=g["discfactors"])
    prices = LogSVPricer().price_chain(chain, LogSvParams(1.0, 1.0, 5.0, 5.0, 0.2, 2.0), is_stiff_solver=True)
    for m in range(2):
        np.testing.assert_allclose(prices[m], g["quick_second_prices"][m], rtol=1e-10, atol=0)
    psi = -0.5 + 1j * np.linspace(0, 400, 60)
    phi = np.ones_like(psi)
    a_gpu = solve_a_ode_grid(phi, psi, 0.3, 1.0413, 3.1844, 3.058, 0.1514, 1.8458, is_spot_measure=False, is_stiff_solver=True,
                             expansion_order=ExpansionOrder.SECOND, vol_backbone_eta=1.1)
    a_ref = omgf.logsv_bdf_a_grid(0.3, phi, psi, np.zeros((60, 5), complex), 1.0413, 3.1844, 3.058, 0.1514, 1.8458, False, 2, 1.1)
    np.testing.assert_allclose(a_gpu, a_ref, rtol=1e-10, atol=1e-11)


def test_single_point_solver_entry_points(cuda_lib):
    """solve_ode_for_a (RK45 and BDF), solve_analytic_ode_for_a and func_rhs_jac of the reference's interface (affine_expansion.py:209-384):
    one transform point at a time == the corresponding rows of the grid goldens; the Jacobian == a central difference of func_rhs"""
    from stochvolmodels_b200.pricers.logsv.affine_expansion import (ExpansionOrder, func_a_ode_quadratic_terms, func_rhs, func_rhs_jac,
                                                                    solve_analytic_ode_for_a, solve_ode_for_a)
    g = load_golden("logsv_bdf_branch.npz")
    name = "quick_second"
    sigma0, theta, k1, k2, beta, vv, order, spot, eta = g[f"{name}_params"]
    phi, ttm = g[f"{name}_phi"], float(g["ttms"][0])
    kw = dict(ttm=ttm, theta=theta, kappa1=k1, kappa2=k2, beta=beta, volvol=vv, psi=0j, is_spot_measure=bool(spot),
              expansion_order=ExpansionOrder(int(order)), vol_backbone_eta=eta)
    for j in (0, 17, 124):
        sol = solve_ode_for_a(phi=phi[j], is_stiff_solver=True, **kw)
        assert sol.success and sol.t[-1] == ttm and sol.y.shape == (5, 2)
        np.testing.assert_allclose(sol.y[:, -1], g[f"{name}_a_0"][j], rtol=1e-10, atol=1e-11)
        nxt = solve_ode_for_a(phi=phi[j], is_stiff_solver=True, a_t0=sol.y[:, -1], **{**kw, "ttm": float(g["ttms"][1]) - ttm})
        np.testing.assert_allclose(nxt.y[:, -1], g[f"{name}_a_1"][j], rtol=1e-10, atol=1e-11)
    with pytest.raises(NotImplementedError):
        solve_ode_for_a(phi=phi[0], dense_output=True, **kw)
    # RK45 branch: rows of the quickstart Fourier golden (first maturity)
    q = load_golden("logsv_fourier_g1_quickstart.npz")
    s0, th, a1, a2, be, vo = q["params"][:6]
    for j in (1, 400):
        sol = solve_ode_for_a(ttm=float(q["ttms"][0]), theta=th, kappa1=a1, kappa2=a2, beta=be, volvol=vo, phi=q["phi"][j], psi=0j,
                              is_spot_measure=bool(q["is_spot"]), expansion_order=ExpansionOrder(int(q["order"])),
                              vol_backbone_eta=float(q["etas"][0]))
        np.testing.assert_allclose(sol.y[:, -1], q["a_t1_0"][j], rtol=1e-10, atol=1e-12)
    # semi-analytic branch
    ga = load_golden("logsv_analytic_branch.npz")
    sigma0, theta, k1, k2, beta, vv, order, spot = ga["mild_second_params"]
    phi_a = ga["mild_second_phi"][::8]
    for j in (0, 60):
        a = solve_analytic_ode_for_a(float(ga["ttms"][0]), theta, k1, k2, beta, vv, phi_a[j], 0j, bool(spot), expansion_order=ExpansionOrder(int(order)))
        np.testing.assert_allclose(a, ga["mild_second_a_0"][j], rtol=1e-8, atol=1e-10)
    # Jacobian
    M, L, H = func_a_ode_quadratic_terms(theta, k1, k2, beta, vv, phi_a[5], 0.1 + 0j, is_spot_measure=True, expansion_order=ExpansionOrder.SECOND)
    A = np.array([0.1 + 0.2j, -0.3 + 0.1j, 0.05j, 0.02, -0.01 + 0.03j])
    J = func_rhs_jac(0.0, A, M, L, H)
    h = 1e-6
    for k in range(5):
        e = np.zeros(5, dtype=np.complex128)
        e[k] = h
        np.testing.assert_allclose(J[:, k], (func_rhs(0.0, A + e, M, L, H) - func_rhs(0.0, A - e, M, L, H)) / (2 * h), rtol=1e-6, atol=1e-8)
