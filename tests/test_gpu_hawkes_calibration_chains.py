"""GPU tests of the Hawkes multi-chain batched pricer (b200sv_hawkesjd_price_chains_batch) and of HawkesJDPricer.calibrate_model_params_to_chains
on it: each chain's sets are integrated by one hawkes_mgf_sets_kernel launch, and every row is bit for bit the single-chain batch's row
(hawkes_mgf_kernel, one launch per set) on its own chain, whatever shares the call; so every lock-step fit is the single-chain driver's."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes

pytestmark = pytest.mark.gpu


def _chains():
    """chains of 1 maturity, the 3-maturity hawkes_fourier.npz chain and the 4-maturity BTC chain"""
    from stochvolmodels_b200 import get_btc_test_chain_data
    g = load_golden("hawkes_fourier.npz")
    btc = get_btc_test_chain_data()
    k1 = np.array([0.8, 0.9, 1.0, 1.1, 1.2]) * 1.01
    return [
        (np.array([0.1]), np.array([1.01]), np.array([0.995]), [k1], [np.array(["P", "P", "C", "C", "C"])]),
        (g["ttms"], g["forwards"], g["discfactors"], [g["strikes"] * f for f in g["forwards"]], [g["types"]] * 3),
        (btc.ttms, btc.forwards, btc.discfactors, btc.strikes_ttms, btc.optiontypes_ttms),
    ]


def _sets(n, seed):
    """parameter sets around the default HawkesJDParams, as the model-parameter fit builds them"""
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        u = 1.0 + 0.2 * rng.uniform(-1, 1, 8)
        kappa, bp, bm = 25.0 * u[5], 70.0 * u[6], 105.0 * u[7]
        out.append(_params_c(mu=0.0, sigma=0.45 * u[0], shift_p=0.06, mean_p=0.03 * u[1], shift_m=-0.06, mean_m=-0.03 * u[2], lambda_p=6.55,
                             theta_p=6.55 * u[3], kappa_p=kappa, beta1_p=bp, beta2_p=-bp, lambda_m=8.5, theta_m=8.5 * u[4], kappa_m=kappa,
                             beta1_m=bm, beta2_m=-bm))
    return out


def _extreme_sets():
    """the corners of the model-parameter fit's bounds: mean near +-0.99, kappa and beta at 100, sigma at 0.1 and 2.0"""
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    out = []
    for sigma, mp, mm, th, k, b in ((0.1, 0.99, -0.99, 100.0, 100.0, 100.0), (2.0, 0.01, -0.01, 0.01, 1.0, 1.0),
                                    (2.0, 0.99, -0.01, 50.0, 100.0, 1.0), (0.1, 0.01, -0.99, 0.01, 100.0, 100.0)):
        out.append(_params_c(mu=0.0, sigma=sigma, shift_p=0.06, mean_p=mp, shift_m=-0.06, mean_m=mm, lambda_p=6.55, theta_p=th, kappa_p=k,
                             beta1_p=b, beta2_p=-b, lambda_m=8.5, theta_m=th, kappa_m=k, beta1_m=b, beta2_m=-b))
    return out


def _check_rows(params, chain_of_set, chains, scalers, is_spot_measure=True, max_phi=500):
    from stochvolmodels_b200 import engine
    got = engine.hawkesjd_price_chains_batch(params, chain_of_set, chains, scalers, is_spot_measure=is_spot_measure, max_phi=max_phi)
    for k, chain in enumerate(chains):
        idx = [b for b, c in enumerate(chain_of_set) if c == k]
        if not idx:
            continue
        prices, ivols = engine.hawkesjd_price_chain_batch([params[b] for b in idx], *chain, is_spot_measure=is_spot_measure,
                                                          vol_scaler=scalers[k], max_phi=max_phi)
        for i, b in enumerate(idx):
            np.testing.assert_array_equal(got[0][b], prices[i], err_msg=f"prices of set {b}")
            np.testing.assert_array_equal(got[1][b], ivols[i], err_msg=f"ivols of set {b}")


@pytest.mark.parametrize("is_spot_measure", [True, False])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("max_phi", [500, 333, 1201])      # 1201 points: hawkes_mgf_kernel at 16 threads per block on 132 SMs
def test_rows_equal_the_single_chain_batch_bitwise(cuda_lib, is_spot_measure, pinned, max_phi):
    chains = _chains()
    if not is_spot_measure:            # calls and puts under the inverse measure
        chains = [c[:4] + ([np.where(np.asarray(t) == "C", "IC", "IP") for t in c[4]],) for c in chains]
    sizes = (1, 9, 17)
    params = _sets(sum(sizes), 7)
    cos = np.random.RandomState(11).permutation(np.concatenate([np.full(n, k) for k, n in enumerate(sizes)]))
    scalers = [0.12, 0.05, 0.3] if pinned else None
    _check_rows(params, cos, chains, scalers or [None] * 3, is_spot_measure, max_phi)


def test_rows_with_shuffled_chains_and_parameter_extremes(cuda_lib):
    chains = _chains()
    params = _sets(12, 3) + _extreme_sets()
    cos = np.array([2, 0, 1, 2, 2, 1, 0, 0, 1, 2, 1, 0] + [1, 1, 1, 1])
    _check_rows(params, cos, chains, [None, None, None])
    # the same sets in another call order, the chains given in reverse
    rev = chains[::-1]
    _check_rows(params, 2 - cos, rev, [None, 0.05, None])


def test_one_riccati_launch_per_chain(cuda_lib):
    from stochvolmodels_b200 import _capi, engine
    lib = _capi.load_library()
    chains = _chains()
    params = _sets(27, 5)
    cos = np.repeat([0, 1, 2], 9)
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chains_batch(params, cos, chains)
    assert lib.b200sv_launch_count() == 3 + 1
    lib.b200sv_reset_launch_count()
    engine.hawkesjd_price_chains_batch(params[:9], np.full(9, 2), chains)      # chains without sets cost nothing
    assert lib.b200sv_launch_count() == 1 + 1


def _markets():
    """the BTC chain and two model markets on its strikes priced from known parameters"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, get_btc_test_chain_data
    btc = get_btc_test_chain_data()
    pricer = HawkesJDPricer()
    out = [btc]
    for s, kappa in ((0.4, 24.0), (0.55, 30.0)):
        truth = HawkesJDParams(sigma=s, kappa_p=kappa, kappa_m=kappa)
        c = OptionChain(ttms=btc.ttms, forwards=btc.forwards, discfactors=btc.discfactors, strikes_ttms=btc.strikes_ttms,
                        optiontypes_ttms=btc.optiontypes_ttms)
        vols = pricer.compute_model_ivols_for_chain(c, truth)
        out.append(OptionChain(ttms=btc.ttms, forwards=btc.forwards, discfactors=btc.discfactors, strikes_ttms=btc.strikes_ttms,
                               optiontypes_ttms=btc.optiontypes_ttms, bid_ivs=[v - 0.005 for v in vols], ask_ivs=[v + 0.005 for v in vols]))
    return out


def _assert_same_fits(out, seq):
    fits, infos = out
    for (fit, info), lock, linfo in zip(seq, fits, infos):
        for key in hawkes.KEYS:
            assert getattr(lock, key) == getattr(fit, key), key
        for key in ("fun", "nit", "nb_batches", "nan_quotes", "x"):
            np.testing.assert_array_equal(linfo[key], info[key], err_msg=key)


@pytest.mark.parametrize("max_sets_per_call", [None, 10])
def test_lockstep_fits_equal_single_chain_fits_bitwise(cuda_lib, max_sets_per_call):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    pricer = HawkesJDPricer()
    markets = _markets()
    starts = [HawkesJDParams(), HawkesJDParams(sigma=0.5, kappa_p=25.0, kappa_m=25.0), HawkesJDParams(sigma=0.4, risk_premia_gamma=0.3)]
    seq = [pricer.calibrate_model_params_to_chain(c, s, return_info=True, maxiter=15) for c, s in zip(markets, starts)]
    out = pricer.calibrate_model_params_to_chains(markets, starts, return_info=True, maxiter=15, max_sets_per_call=max_sets_per_call)
    _assert_same_fits(out, seq)
    rounds = out[1][0]["rounds"]
    assert all(i["rounds"] == rounds for i in out[1])
    if max_sets_per_call is None:
        assert rounds == max(i["nb_batches"] for _, i in seq)
    else:                              # a gradient round of 3 x 8 sets needs three calls of at most 10 sets
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
    fits = HawkesJDPricer().calibrate_model_params_to_chains(markets, HawkesJDParams(), return_exceptions=True, maxiter=5)
    assert len(calls) == 2
    assert all(isinstance(f, _capi.B200svError) for f in fits), fits
