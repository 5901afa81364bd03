"""The batched Hawkes Fourier chain pricer (b200sv_hawkesjd_price_chain_batch) on the GPU: row b bit for bit the single-set pricer of set b
(prices) and the chain inversion of those prices (implied vols), on both routes, both measures, per-set and pinned grids; and the two
calibration drivers on it bit for bit the sequential fits."""
import numpy as np
import pytest

import hawkes_sequential as seq
from conftest import load_golden
from oracle import hawkes

pytestmark = pytest.mark.gpu


def _sets(B, base, seed=0):
    """B parameter sets around ``base``: the first is ``base``, the others move every field by up to +-3 % (as a difference batch would)"""
    from stochvolmodels_b200 import HawkesJDParams
    rng = np.random.default_rng(seed)
    d = {k: v for k, v in base.to_dict().items() if k != "risk_premia_gamma"}
    out = [HawkesJDParams(**d)]
    for _ in range(B - 1):
        out.append(HawkesJDParams(**{k: v * (1.0 + 0.03 * rng.uniform(-1, 1)) for k, v in d.items()}))
    return out


def _golden_chain():
    from stochvolmodels_b200 import OptionChain
    g = load_golden("hawkes_fourier.npz")
    return g, OptionChain(ttms=g["ttms"], forwards=g["forwards"], discfactors=g["discfactors"], strikes_ttms=[g["strikes"] * f for f in g["forwards"]],
                          optiontypes_ttms=[g["types"]] * 3)


def _check_rows(chain, sets, gammas=None, is_spot_measure=True, vol_scaler=None, types=None):
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    types = chain.optiontypes_ttms if types is None else types
    args = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, types)
    pcs = [_params_c(**s.to_dict()) for s in sets]
    prices, ivols = engine.hawkesjd_price_chain_batch(pcs, *args, is_spot_measure=is_spot_measure, vol_scaler=vol_scaler, gammas=gammas)
    assert prices.shape == ivols.shape == (len(sets), sum(len(k) for k in chain.strikes_ttms))
    for b, pc in enumerate(pcs):
        one = engine.hawkesjd_price_chain(pc, *args, is_spot_measure, vol_scaler, 500, None if gammas is None else gammas[b])
        np.testing.assert_array_equal(prices[b], np.concatenate(one))
        iv = engine.bsm_implied_vols(*args, one)
        np.testing.assert_array_equal(ivols[b], np.concatenate(iv))
    return prices, ivols


@pytest.mark.parametrize("B", [1, 3, 9, 40])          # 40: well beyond a difference batch
@pytest.mark.parametrize("name", ["dflt", "alt"])
def test_rows_equal_the_single_set_pricer_on_the_golden_chain(cuda_lib, B, name):
    from stochvolmodels_b200 import HawkesJDParams
    g, chain = _golden_chain()
    sets = _sets(B, HawkesJDParams(**dict(zip(hawkes.KEYS, g[f"{name}_params"]))), seed=B)
    for vol_scaler in (None, 0.2):
        _check_rows(chain, sets, vol_scaler=vol_scaler)
        inverse = [np.array(["IP", "P", "C", "IC", "IC"])] * 3
        _check_rows(chain, sets, is_spot_measure=False, vol_scaler=vol_scaler, types=inverse)


@pytest.mark.parametrize("B", [1, 3, 9, 40])
def test_rows_equal_the_single_set_pricer_on_the_btc_chain(cuda_lib, B):
    from stochvolmodels_b200 import HawkesJDParams, get_btc_test_chain_data
    chain = get_btc_test_chain_data()
    sets = _sets(B, HawkesJDParams(), seed=10 + B)
    prices, ivols = _check_rows(chain, sets)
    assert np.isfinite(ivols[0]).mean() > 0.9
    _check_rows(chain, sets, vol_scaler=0.3)


@pytest.mark.parametrize("B", [4, 9, 40])
def test_risk_kernel_rows_equal_price_chain_with_risk_premia_gamma(cuda_lib, B):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, get_btc_test_chain_data
    g, golden = _golden_chain()
    btc = get_btc_test_chain_data()
    gammas = np.resize([-0.3, 0.0, 0.2, 0.5], B)
    for chain, base in ((golden, HawkesJDParams(**dict(zip(hawkes.KEYS, g["dflt_params"])))), (btc, HawkesJDParams())):
        sets = _sets(B, base, seed=20 + B)
        _check_rows(chain, sets, gammas=gammas, vol_scaler=0.25)
        prices, _ = _check_rows(chain, sets, gammas=gammas)
        # the pricer API with risk_premia_gamma set is the route the rows reproduce
        for b in range(4):
            p = HawkesJDParams(**{**sets[b].to_dict(), "risk_premia_gamma": float(gammas[b])})
            np.testing.assert_array_equal(np.concatenate(HawkesJDPricer().price_chain(chain, p)), prices[b])


def test_permuting_the_sets_permutes_the_rows_and_calls_repeat(cuda_lib):
    from stochvolmodels_b200 import HawkesJDParams, engine, get_btc_test_chain_data
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    chain = get_btc_test_chain_data()
    sets = [_params_c(**s.to_dict()) for s in _sets(33, HawkesJDParams(), seed=5)]
    args = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    perm = np.random.default_rng(1).permutation(33)
    gammas = np.linspace(-0.3, 0.5, 33)
    for gm in (None, gammas):
        p, v = engine.hawkesjd_price_chain_batch(sets, *args, gammas=gm)
        p2, v2 = engine.hawkesjd_price_chain_batch(sets, *args, gammas=gm)
        pp, vp = engine.hawkesjd_price_chain_batch([sets[i] for i in perm], *args, gammas=None if gm is None else gm[perm])
        np.testing.assert_array_equal(p, p2)
        np.testing.assert_array_equal(v, v2)
        np.testing.assert_array_equal(pp, p[perm])
        np.testing.assert_array_equal(vp, v[perm])
    for gm in (None, gammas[:3]):                        # ivols_out = NULL on both routes: prices only, the same bits
        prices, none = engine.hawkesjd_price_chain_batch(sets[:3], *args, gammas=gm, with_ivols=False)
        assert none is None
        np.testing.assert_array_equal(prices, engine.hawkesjd_price_chain_batch(sets[:3], *args, gammas=gm)[0])


def _synthetic_market(pricer, true):
    from stochvolmodels_b200 import OptionChain
    K = np.linspace(0.75, 1.3, 12)
    ttms, fw = np.array([0.08, 0.25, 0.5]), np.array([1.0, 1.0, 1.0])
    mk = lambda vols: OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K] * 3, optiontypes_ttms=[np.where(K >= 1.0, "C", "P")] * 3,
                                  ids=np.array(["1m", "3m", "6m"]), bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    return mk(pricer.compute_model_ivols_for_chain(mk([0.5 * np.ones_like(K)] * 3), true))


def test_drivers_return_the_sequential_fits_bit_for_bit(cuda_lib, capsys):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer
    pricer = HawkesJDPricer()
    true = HawkesJDParams(sigma=0.4, mean_p=0.04, mean_m=-0.05, theta_p=6.0, theta_m=8.0, kappa_p=25.0, kappa_m=25.0, beta1_p=30.0, beta2_p=-30.0,
                          beta1_m=40.0, beta2_m=-40.0)
    chain = _synthetic_market(pricer, true)
    start = HawkesJDParams(sigma=0.45, mean_p=0.03, mean_m=-0.04, theta_p=7.0, theta_m=7.0, kappa_p=22.0, kappa_m=28.0, beta1_p=33.0, beta2_p=-33.0,
                           beta1_m=36.0, beta2_m=-36.0)
    ref, res = seq.calibrate_model_params(pricer, chain, start, maxiter=60)
    fit, info = pricer.calibrate_model_params_to_chain(chain, start, maxiter=60, return_info=True)
    np.testing.assert_array_equal(info["x"], res.x)
    assert fit == ref and info["fun"] == res.fun and info["nb_batches"] == seq.batches(res, 8)
    chain_g = _synthetic_market(pricer, HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5))
    start_g = HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2)
    capsys.readouterr()
    ref_g, res_g = seq.calibrate_risk_premia_gamma(pricer, chain_g, start_g)
    expected = capsys.readouterr().out
    fit_g, info_g = pricer.calibrate_risk_premia_gamma_to_chain(chain_g, start_g, return_info=True)
    assert capsys.readouterr().out == expected
    np.testing.assert_array_equal(info_g["x"], res_g.x)
    assert fit_g == ref_g and info_g["fun"] == res_g.fun and info_g["nb_batches"] == seq.batches(res_g, 2)
