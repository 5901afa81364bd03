"""The exact event-driven route of the Hawkes jump-diffusion Monte Carlo on the GPU (DESIGN.md §3.13): the kernel path by path against
oracle/hawkes_exact.py, reproducibility across runs and shards, agreement with the Fourier route without an allowance, the terminal
moments, the candidate budget's error return, and the unchanged Euler default."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes, hawkes_exact

pytestmark = pytest.mark.gpu


def _pc(d):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    return _params_c(**{k: d[k] for k in hawkes.KEYS})


def _mc_chain():
    from stochvolmodels_b200 import OptionChain
    g = load_golden("hawkes_mc.npz")
    M = g["chain_ttms"].shape[0]
    return OptionChain(ttms=g["chain_ttms"], forwards=g["chain_forwards"], discfactors=g["chain_discfactors"],
                       strikes_ttms=[g["chain_strikes"] * f for f in g["chain_forwards"]], optiontypes_ttms=[g["chain_types"]] * M)


@pytest.mark.parametrize("name", ["dflt", "drift", "dflt_kappa_p_negative"])
def test_kernel_equals_the_oracle_path_by_path(name):
    """first 1000 of 5000 paths of a two-maturity chain: event counts equal, states to 1e-12, with multi-event paths and bursts that
    straddle the maturity boundary among them; also with kappa_p < 0, where the thinning bound looks ahead to the interval end"""
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200 import engine
    g = load_golden("hawkes_mc.npz")
    sets = {"dflt": {}, "drift": {}, "dflt_kappa_p_negative": {"kappa_p": -4.0}}
    p = {**dict(zip(hawkes.KEYS, g[f"{name.split('_')[0]}_params"])), **sets[name]}
    chain, n_out, seed = _mc_chain(), 1000, 29
    _, _, states, events = engine.hawkesjd_mc_chain_exact(_pc(p), chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                          chain.optiontypes_ttms, 5000, C.LOG_RETURN, seed, n_paths_out=n_out)
    _, _, o_states, o_events = hawkes_exact.chain(p, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                                  n_out, seed)
    np.testing.assert_array_equal(events, o_events)
    np.testing.assert_allclose(states, o_states, rtol=1e-12, atol=1e-12)
    accepted = events[:, 0] + events[:, 1]
    assert accepted.max() >= 5 and np.all(events[:, 2] >= accepted)
    # a burst over the boundary: intensity well above its mean level at the first maturity and events right after it
    burst = (states[0, 1] > 2 * p["theta_p"]) & (accepted[1] > 0) & (accepted[0] > 0)
    assert burst.sum() >= 5, burst.sum()


def test_reproducible_across_runs_and_shards():
    """two runs bitwise equal; two half-shards through CudaMcEngine('hawkes_exact') hold the unsharded terminal states bitwise; the sharded
    driver equals the host-level chain to 1e-12; the exact route does not consult gauss"""
    import torch
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, get_btc_test_chain_data
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.multi_gpu import CudaMcEngine, mc_chain_distributed
    chain, params = get_btc_test_chain_data(), HawkesJDParams()
    d = params.to_dict()
    d.pop("risk_premia_gamma")
    pc = _pc(d)
    N, seed = 200_003, 17
    pricer = HawkesJDPricer()
    p1, e1 = pricer.model_mc_price_chain(chain, params, nb_path=N, seed=seed, scheme="exact")
    p2, e2 = pricer.model_mc_price_chain(chain, params, nb_path=N, seed=seed, scheme="exact")
    for m in range(len(p1)):
        assert np.array_equal(p1[m], p2[m]) and np.array_equal(e1[m], e2[m]), "two runs of the same call differ"
    p3, e3 = pricer.model_mc_price_chain(chain, params, nb_path=N, seed=seed, scheme="exact", gauss="fp64")
    for m in range(len(p1)):
        assert np.array_equal(p1[m], p3[m]) and np.array_equal(e1[m], e3[m]), "the exact route consulted gauss"
    t = chain.ttms
    grid = [(1, float(t[m] - (t[m - 1] if m > 0 else 0.0))) for m in range(t.shape[0])]
    p_d, e_d = mc_chain_distributed("hawkes_exact", pc, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms,
                                    chain.optiontypes_ttms, N, 1800, True, C.LOG_RETURN, seed, 0, grid=grid)
    for m in range(len(p1)):
        np.testing.assert_allclose(p_d[m], p1[m], rtol=1e-12)
        np.testing.assert_allclose(e_d[m], e1[m], rtol=1e-10)
    T0 = float(chain.ttms[0])
    whole = CudaMcEngine("hawkes_exact", pc, N, 0, 0, 4)
    whole.simulate_slice(0, True, 1, T0, 1.0, True, float(chain.forwards[0]), seed)
    n0 = N // 2
    parts = [CudaMcEngine("hawkes_exact", pc, n0, 0, 0, 4), CudaMcEngine("hawkes_exact", pc, N - n0, n0, 0, 4)]
    moments = 0.0
    for e in parts:
        moments = moments + e.simulate_slice(0, True, 1, T0, 1.0, True, float(chain.forwards[0]), seed).cpu().numpy()
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([e.state for e in parts], dim=1), whole.state)
    np.testing.assert_allclose(moments, whole.moments.cpu().numpy(), rtol=1e-12)
    assert not any(int(e.overflow.item()) for e in (whole, *parts))
    x, lp, lm = (np.zeros(N) for _ in range(3))
    engine.hawkesjd_terminal_exact(pc, T0, x, lp, lm, seed, 0, False)
    assert np.array_equal(x, whole.state[0].cpu().numpy()) and np.array_equal(lm, whole.state[2].cpu().numpy())


def test_mc_equals_fourier_without_an_allowance(record_property):
    """4e6 paths, BTC chain at the default parameters and the hawkes_mc.npz chain: |MC - Fourier| < 4.5 SE on every strike with no additive
    term.  The Euler route's distance from Fourier at the same paths is recorded, not asserted."""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, get_btc_test_chain_data
    pricer, params = HawkesJDPricer(), HawkesJDParams()
    for label, chain in (("btc", get_btc_test_chain_data()), ("hawkes_mc", _mc_chain())):
        four = pricer.price_chain(chain, params)
        zs = {}
        for scheme in ("exact", "euler"):
            p, e = pricer.model_mc_price_chain(chain, params, nb_path=4_000_000, seed=41, scheme=scheme)
            zs[scheme] = [(p[m] - four[m]) / e[m] for m in range(len(p))]
            record_property(f"{label}_{scheme}_max_abs_z", float(max(np.abs(z).max() for z in zs[scheme])))
            print(f"{label} {scheme}: max |MC - Fourier| / SE = {max(np.abs(z).max() for z in zs[scheme]):.2f}; per maturity",
                  [float(np.round(np.abs(z).max(), 2)) for z in zs[scheme]])
        for m, z in enumerate(zs["exact"]):
            assert np.all(np.abs(z) < 4.5), (label, m, z)


def test_terminal_moments_match_the_mean_equations():
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    g = load_golden("hawkes_mc.npz")
    free = dict(beta1_p=0.0, beta2_p=0.0, beta1_m=0.0, beta2_m=0.0, lambda_p=20.0, lambda_m=20.0, theta_p=5.0, theta_m=5.0, kappa_p=-4.0,
                kappa_m=-4.0)      # kappa < 0: the intensities grow away from theta
    for params in (HawkesJDParams(), HawkesJDParams(**dict(zip(hawkes.KEYS, g["drift_params"]))), HawkesJDParams(**free)):
        d = params.to_dict()
        T, n = 0.3, 2_000_000
        x, lp, lm = HawkesJDPricer().simulate_terminal_values(params, ttm=T, nb_path=n, seed=8, scheme="exact")
        ref = hawkes_exact.mean_equations(d, T)
        for est, want in ((lp, ref[0]), (lm, ref[1]), (np.exp(x), np.exp(d["mu"] * T))):
            assert abs(est.mean() - want) < 4.0 * est.std() / np.sqrt(n) + 1e-12 * abs(want), (est.mean(), want)


def test_candidate_budget_returns_an_error_and_no_prices():
    """a budget of 3 candidates on a high-intensity set: the C entry point returns -6 promptly and leaves prices_out unwritten, the pricer
    and the sharded driver raise"""
    import ctypes
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.multi_gpu import CudaMcEngine, mc_chain_distributed
    chain = _mc_chain()
    params = HawkesJDParams(lambda_p=200.0, theta_p=200.0, lambda_m=200.0, theta_m=200.0)
    d = params.to_dict()
    d.pop("risk_premia_gamma")
    ch = engine._chain_arrays(chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    J = ch.strikes.shape[0]
    prices, stds = np.full(J, -7.0), np.full(J, -7.0)
    lib = C.load_library()
    rc = lib.b200sv_hawkesjd_mc_chain_exact(ctypes.byref(_pc(d)), *C.chain_ptrs(ch), 256, C.LOG_RETURN, 3, 0, C.dptr(prices), C.dptr(stds), 3, 0, None, None)
    assert rc == -6 and "candidate budget exhausted" in lib.b200sv_last_error().decode()
    assert np.all(prices == -7.0) and np.all(stds == -7.0)
    with pytest.raises(C.B200svError) as err:
        HawkesJDPricer().model_mc_price_chain(chain, params, nb_path=256, seed=3, scheme="exact", max_candidates=3)
    assert err.value.code == -6
    t = chain.ttms
    with pytest.raises(C.B200svError) as err:
        mc_chain_distributed("hawkes_exact", _pc(d), t, chain.forwards, chain.discfactors, None, chain.strikes_ttms, chain.optiontypes_ttms, 256,
                             1800, True, C.LOG_RETURN, 3, 0, grid=[(1, float(t[0])), (1, float(t[1] - t[0]))], max_candidates=3,
                             engine_factory=lambda *a, **k: CudaMcEngine(*a, **k))
    assert err.value.code == -6


def test_euler_default_unchanged():
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    chain, params, pricer = _mc_chain(), HawkesJDParams(), HawkesJDPricer()
    p0, e0 = pricer.model_mc_price_chain(chain, params, nb_path=300_000, seed=12)
    p1, e1 = pricer.model_mc_price_chain(chain, params, nb_path=300_000, seed=12, scheme="euler")
    for m in range(len(p0)):
        assert np.array_equal(p0[m], p1[m]) and np.array_equal(e0[m], e1[m])
    x0 = pricer.simulate_terminal_values(params, ttm=0.1, nb_path=10_000, seed=6)
    x1 = pricer.simulate_terminal_values(params, ttm=0.1, nb_path=10_000, seed=6, scheme="euler")
    assert all(np.array_equal(a, b) for a, b in zip(x0, x1))
