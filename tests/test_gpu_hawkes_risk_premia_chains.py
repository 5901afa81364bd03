"""GPU tests of the Hawkes multi-chain pricer under the risk kernel (b200sv_hawkesjd_price_chains_batch_gamma) and of
HawkesJDPricer.calibrate_risk_premia_gamma_to_chains on it: every (set, maturity) normaliser pair of a call is solved by one restarted
hawkes_mgf_sets_kernel launch, each chain's Riccati grids by one more, and every row is bit for bit the single-chain batch's row with
gammas (one hawkes_mgf_kernel launch per set for each) on its own chain, whatever shares the call; so every lock-step fit is the
single-chain driver's."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes

pytestmark = pytest.mark.gpu

SPECIAL_GAMMAS = (8.0, -8.0, 0.0, -0.5, -1.0)      # the fit's bounds, no tilt, the gamma slice pricer's fast branch, and -1


def _chains():
    """chains of 1 maturity, the 3-maturity hawkes_fourier.npz chain, the 4-maturity BTC chain, and a 2-maturity chain"""
    from stochvolmodels_b200 import get_btc_test_chain_data
    g = load_golden("hawkes_fourier.npz")
    btc = get_btc_test_chain_data()
    k1 = np.array([0.8, 0.9, 1.0, 1.1, 1.2]) * 1.01
    k2 = np.array([0.7, 0.95, 1.05, 1.4])
    return [
        (np.array([0.1]), np.array([1.01]), np.array([0.995]), [k1], [np.array(["P", "P", "C", "C", "C"])]),
        (g["ttms"], g["forwards"], g["discfactors"], [g["strikes"] * f for f in g["forwards"]], [g["types"]] * 3),
        (btc.ttms, btc.forwards, btc.discfactors, btc.strikes_ttms, btc.optiontypes_ttms),
        (np.array([0.05, 0.3]), np.ones(2), np.array([0.999, 0.99]), [k2, k2], [np.array(["P", "P", "C", "C"])] * 2),
    ]


def _sets(n, seed):
    """(parameter sets, gammas) as the risk-premia fit builds them: sigma and gamma move, the rest stays at HawkesJDParams' defaults;
    the gammas cycle through SPECIAL_GAMMAS and draws from the fit's bounds"""
    from stochvolmodels_b200 import HawkesJDParams
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    rng = np.random.RandomState(seed)
    d = {k: v for k, v in HawkesJDParams().to_dict().items() if k != "risk_premia_gamma"}
    params = [_params_c(**{**d, "sigma": float(s)}) for s in rng.uniform(0.05, 1.5, n)]
    gammas = [SPECIAL_GAMMAS[i // 2] if i % 2 == 0 and i // 2 < len(SPECIAL_GAMMAS) else float(rng.uniform(-8, 8)) for i in range(n)]
    return params, gammas


def _check_rows(params, gammas, chain_of_set, chains, scalers, max_phi=500):
    from stochvolmodels_b200 import engine
    got = engine.hawkesjd_price_chains_batch(params, chain_of_set, chains, scalers, max_phi=max_phi, gammas=gammas)
    for k, chain in enumerate(chains):
        idx = [b for b, c in enumerate(chain_of_set) if c == k]
        if not idx:
            continue
        prices, ivols = engine.hawkesjd_price_chain_batch([params[b] for b in idx], *chain, vol_scaler=scalers[k], max_phi=max_phi,
                                                          gammas=[gammas[b] for b in idx])
        for i, b in enumerate(idx):
            np.testing.assert_array_equal(got[0][b], prices[i], err_msg=f"prices of set {b}")
            np.testing.assert_array_equal(got[1][b], ivols[i], err_msg=f"ivols of set {b}")
    return got


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("max_phi", [500, 333, 1201])      # 1201 points: 16 threads per block on 132 SMs
def test_rows_equal_the_single_chain_batch_bitwise(cuda_lib, pinned, max_phi):
    chains = _chains()
    sizes = (1, 17, 2, 0)                                   # the 2-maturity chain has no sets
    params, gammas = _sets(sum(sizes), 7)
    cos = np.random.RandomState(11).permutation(np.concatenate([np.full(n, k) for k, n in enumerate(sizes)]))
    scalers = [0.12, 0.05, 0.3, 0.2] if pinned else [None] * 4
    prices, _ = _check_rows(params, gammas, cos, chains, scalers, max_phi)
    assert all(np.isfinite(p).any() for p in prices)


def test_rows_with_shuffled_and_reordered_chains(cuda_lib):
    chains = _chains()
    params, gammas = _sets(13, 3)
    cos = np.array([2, 0, 1, 2, 2, 1, 0, 3, 3, 2, 1, 1, 3])    # groups of 2, 4, 4 and 3 sets
    _check_rows(params, gammas, cos, chains, [None, None, None, None])
    rev = chains[::-1]                                          # the same sets in the chains given in reverse, one chain pinned
    _check_rows(params, gammas, 3 - cos, rev, [None, 0.05, None, 0.3])
    _check_rows(params[:3], gammas[:3], [2, 2, 2], chains, [None] * 4)       # one group of 3, three chains without sets


def test_two_launches_besides_one_riccati_launch_per_chain(cuda_lib):
    from stochvolmodels_b200 import _capi, engine
    lib = _capi.load_library()
    chains = _chains()
    params, gammas = _sets(12, 5)
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chains_batch(params, np.repeat([0, 1, 2], 4), chains, gammas=gammas)
    assert lib.b200sv_launch_count() == 3 + 2
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chains_batch(params[:4], np.full(4, 3), chains, gammas=gammas[:4])     # chains without sets cost nothing
    assert lib.b200sv_launch_count() == 1 + 2


def _markets():
    """the BTC chain and three risk-kernel markets on the 3 x 12 strikes of test_gpu_hawkes.py priced from known (sigma, gamma)"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, get_btc_test_chain_data
    K = np.linspace(0.75, 1.3, 12)
    ttms, fw = np.array([0.08, 0.25, 0.5]), np.ones(3)
    mk = lambda vols: OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K] * 3, optiontypes_ttms=[np.where(K >= 1.0, "C", "P")] * 3,
                                  bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    flat = mk([0.5 * np.ones_like(K)] * 3)
    pricer = HawkesJDPricer()
    out = [get_btc_test_chain_data()]
    for s, g in ((0.42, 0.5), (0.38, 0.3), (0.47, 0.6)):
        vols = pricer.compute_model_ivols_for_chain(flat, HawkesJDParams(sigma=s, risk_premia_gamma=g))
        assert all(np.isfinite(v).all() for v in vols)
        out.append(mk(vols))
    return out


@pytest.mark.parametrize("max_sets_per_call", [None, 2])
def test_lockstep_fits_equal_single_chain_fits_bitwise(cuda_lib, capsys, max_sets_per_call):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    pricer = HawkesJDPricer()
    markets = _markets()
    starts = [HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2), HawkesJDParams(sigma=0.4), HawkesJDParams(sigma=0.5, risk_premia_gamma=0.1),
              HawkesJDParams(sigma=0.45, risk_premia_gamma=0.4, lambda_p=7.0)]
    seq, printed = [], []
    for c, s in zip(markets, starts):
        seq.append(pricer.calibrate_risk_premia_gamma_to_chain(c, s, maxiter=15, print_iter=True, return_info=True))
        printed.append(capsys.readouterr().out)
    fits, infos = pricer.calibrate_risk_premia_gamma_to_chains(markets, starts, maxiter=15, print_iter=True, return_info=True,
                                                               max_sets_per_call=max_sets_per_call)
    assert capsys.readouterr().out == "".join(printed)
    for (fit, info), lock, linfo in zip(seq, fits, infos):
        for key in hawkes.KEYS + ("risk_premia_gamma",):
            assert getattr(lock, key) == getattr(fit, key), key
        for key in ("fun", "nit", "nb_batches", "nan_quotes", "x"):
            np.testing.assert_array_equal(linfo[key], info[key], err_msg=key)
    rounds = infos[0]["rounds"]
    assert all(i["rounds"] == rounds for i in infos)
    if max_sets_per_call is None:
        assert rounds == max(i["nb_batches"] for _, i in seq)
    else:                              # a gradient round of 4 x 2 sets needs four calls of at most 2 sets
        assert rounds > max(i["nb_batches"] for _, i in seq)


def test_a_rejected_round_reaches_every_fit(cuda_lib, monkeypatch):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, _capi, engine
    markets = _markets()
    real = engine.hawkesjd_price_chains_batch
    calls = []

    def reject_second(params, chain_of_set, chains, **kw):
        calls.append(len(params))
        if len(calls) == 2:
            return real(params, chain_of_set, chains, max_phi=2, **{k: v for k, v in kw.items() if k != "max_phi"})   # P < 3: rejected
        return real(params, chain_of_set, chains, **kw)
    monkeypatch.setattr(engine, "hawkesjd_price_chains_batch", reject_second)
    fits = HawkesJDPricer().calibrate_risk_premia_gamma_to_chains(markets, HawkesJDParams(sigma=0.45), return_exceptions=True, maxiter=5)
    assert len(calls) == 2
    assert all(isinstance(f, _capi.B200svError) for f in fits), fits
