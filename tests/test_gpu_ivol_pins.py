"""The reference's own pins of the Black-76 implied-vol step, ported to the GPU inversion (SURVEY.md §8f #1; VERDICT r1 next #8).

The inversion itself is third-party in the reference (vanilla_option_pricers 2.1.0, absent from /root/reference and from the image), so its
bits cannot be pinned; what the reference's OWN test suite asserts about it can, at the reference's own tolerances:
  * flat-vol recovery                 tests/test_model_calibration_contracts.py:95-116     atol 1e-10 (ivols), 1e-14 (two routes agree)
  * chain price -> ivol round trip    tests/test_option_chain_characterization.py:193-222  atol 2e-10
  * price_slice == price_vanilla      tests/test_logsv_characterization.py:110-138         prices atol 1e-14, ivols atol 1e-12, ivols finite
  * single-option round trip          tests/test_analytic_bsm.py:75-101                    atol 2e-12
  * quickstart vols                   examples/getting_started/quickstart.py:44,46         0.999577 / 0.995757
Prices are made with the exact Black-76 formula in float64 (oracle/bsm.py, scipy ndtr): the checker only produces the inputs.
"""
import numpy as np
import pytest

from oracle import bsm

pytestmark = pytest.mark.gpu


class _FlatVolParams:
    vol = 0.2


def _flat_pricer():
    from stochvolmodels_b200 import ModelPricer

    class FlatVolPricer(ModelPricer):                 # the reference test's `_FlatVolPricer`: Black prices at one vol, MC = prices + 1e-4 SE
        def price_chain(self, option_chain, params, **kwargs):
            return [bsm.compute_bsm_vanilla_price(f, k, t, params.vol, ty, d) for t, f, k, ty, d in
                    zip(option_chain.ttms, option_chain.forwards, option_chain.strikes_ttms, option_chain.optiontypes_ttms, option_chain.discfactors)]

        def model_mc_price_chain(self, option_chain, params, variable_type=None, **kwargs):
            prices = self.price_chain(option_chain, params)
            return prices, [1.0e-4 * np.ones_like(p) for p in prices]
    return FlatVolPricer()


def test_flat_vol_recovery_through_the_common_interfaces(cuda_lib):
    from stochvolmodels_b200 import OptionChain, VariableType
    chain = OptionChain(ttms=np.array([0.5]), forwards=np.array([1.0]), strikes_ttms=[np.array([0.9, 1.0, 1.1])],
                        optiontypes_ttms=[np.array(["P", "C", "C"])], ids=np.array(["6m"]), discfactors=np.array([0.98]))
    params, pricer = _FlatVolParams(), _flat_pricer()
    prices, ivols = pricer.compute_chain_prices_with_vols(chain, params)
    model_ivols = pricer.compute_model_ivols_for_chain(chain, params)
    mc = pricer.compute_mc_chain_implied_vols(chain, params, variable_type=VariableType.LOG_RETURN, nb_path=100)
    np.testing.assert_allclose(ivols[0], params.vol, rtol=0.0, atol=1.0e-10)
    np.testing.assert_allclose(model_ivols[0], ivols[0], rtol=0.0, atol=1.0e-14)
    np.testing.assert_allclose(mc[0][0], prices[0], rtol=0.0, atol=0.0)
    assert np.all(mc[1][0] > mc[0][0]) and np.all(mc[2][0] < mc[0][0])
    assert np.all(mc[4][0] > mc[3][0]) and np.all(mc[5][0] < mc[3][0])
    np.testing.assert_allclose(mc[6][0], 1.0e-4, rtol=0.0, atol=0.0)


def test_chain_price_ivol_round_trip(cuda_lib):
    from stochvolmodels_b200 import OptionChain
    ttms, fw, df = np.array([0.5, 1.0]), np.array([1.0, 1.02]), np.array([0.99, 0.97])
    strikes = [np.array([0.9, 1.0, 1.1]), np.array([0.85, 1.0, 1.15, 1.3])]
    types = [np.array(["P", "C", "C"]), np.array(["P", "P", "C", "C"])]
    target = [np.array([0.30, 0.25, 0.27]), np.array([0.34, 0.26, 0.24, 0.29])]
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=strikes, optiontypes_ttms=types, ids=np.array(["6m", "1y"]), discfactors=df,
                        bid_ivs=[t - 0.01 for t in target], ask_ivs=[t + 0.01 for t in target])
    prices = [bsm.compute_bsm_vanilla_price(f, k, t, v, ty, d) for t, f, k, v, ty, d in zip(ttms, fw, strikes, target, types, df)]
    recovered = chain.compute_model_ivols_from_chain_data(prices)
    for actual, expected in zip(recovered, target):
        np.testing.assert_allclose(actual, expected, rtol=0.0, atol=2.0e-10)


def test_price_slice_and_price_vanilla_self_consistency(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.array([1.0]), strikes_ttms=[np.array([0.9, 1.0, 1.1])],
                        optiontypes_ttms=[np.array(["P", "C", "C"])], ids=np.array(["3m"]), discfactors=np.array([0.99]))
    params = LogSvParams(sigma0=0.4, theta=0.45, kappa1=2.0, kappa2=2.5, beta=-0.4, volvol=0.8)
    pricer = LogSVPricer()
    chain_prices = np.asarray(pricer.price_chain(chain, params)[0])
    slice_prices, slice_ivols = pricer.price_slice(params=params, ttm=chain.ttms[0], forward=chain.forwards[0], strikes=np.asarray(chain.strikes_ttms[0]),
                                                   optiontypes=np.asarray(chain.optiontypes_ttms[0]), discfactor=chain.discfactors[0])
    np.testing.assert_allclose(slice_prices, chain_prices, rtol=0.0, atol=1.0e-14)
    assert np.all(np.isfinite(slice_ivols))
    for i, (strike, optiontype) in enumerate(zip(chain.strikes_ttms[0], chain.optiontypes_ttms[0])):
        price, ivol = pricer.price_vanilla(params=params, ttm=chain.ttms[0], forward=chain.forwards[0], strike=strike, optiontype=optiontype,
                                           discfactor=chain.discfactors[0])
        np.testing.assert_allclose(price, chain_prices[i], rtol=0.0, atol=1.0e-14)
        np.testing.assert_allclose(ivol, slice_ivols[i], rtol=0.0, atol=1.0e-12)


def test_single_option_round_trip_2e12(cuda_lib):
    from stochvolmodels_b200 import engine
    forward, strike, ttm, discfactor, vol = 0.98, 1.04, 1.4, 0.94, 0.37
    price = bsm.compute_bsm_vanilla_price(forward, np.array([strike]), ttm, vol, np.array(["P"]), discfactor)
    iv = engine.bsm_implied_vols(np.array([ttm]), np.array([forward]), np.array([discfactor]), [np.array([strike])], [np.array(["P"])], [price])
    np.testing.assert_allclose(iv[0][0], vol, rtol=0.0, atol=2.0e-12)
    # a grid of moneyness / maturity / vol, both payoff types and the inverse codes: same bar wherever vega is not negligible
    rs = np.random.RandomState(4)
    n = 4000
    F = rs.uniform(0.5, 2.0, n); K = F * np.exp(rs.uniform(-0.5, 0.5, n)); T = rs.uniform(0.02, 3.0, n); V = rs.uniform(0.05, 2.0, n)
    ty = rs.choice(["C", "P", "IC", "IP"], n)
    D = rs.uniform(0.8, 1.0, n)
    prices = [bsm.compute_bsm_vanilla_price(F[i], K[i:i + 1], T[i], V[i], ty[i:i + 1], D[i]) for i in range(n)]
    iv = engine.bsm_implied_vols(T, F, D, [K[i:i + 1] for i in range(n)], [ty[i:i + 1] for i in range(n)], prices)
    iv = np.array([v[0] for v in iv])
    tv = V * np.sqrt(T)
    d1 = np.log(F / K) / tv + 0.5 * tv
    # conditioning: the input price carries an ABSOLUTE rounding error ~1e-16 F (it is F N(d1) - K N(d2)), so d vol = 1e-16 F / vega
    vega = F * np.exp(-0.5 * d1 * d1) / np.sqrt(2.0 * np.pi) * np.sqrt(T)
    well = vega / F > 2e-3
    assert well.mean() > 0.5
    np.testing.assert_allclose(iv[well], V[well], rtol=0.0, atol=2.0e-12)
    # every quote, however far out: the exact implied vol of the fp64 quote as given, at the bar of tests/ivol_cases.py; NaN exactly where
    # the quote is outside the no-arbitrage bounds
    import ivol_cases as ic
    pytest.importorskip("mpmath")
    iv_star, bar = ic.reference(dict(F=F, K=K, T=T, D=D, type=ty, price=np.array([p[0] for p in prices]), vol=V))
    ratio, nan_mismatch, bad = ic.check(iv, iv_star, bar)
    assert nan_mismatch.size == 0 and bad.size == 0, (ratio, nan_mismatch[:5], bad[:5])


def test_quickstart_vanilla_vol(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer
    pricer, params = LogSVPricer(), LogSvParams(sigma0=1.0, theta=1.0, kappa1=5.0, kappa2=5.0, beta=0.2, volvol=2.0)
    p, v = pricer.price_vanilla(params=params, ttm=0.25, forward=1.0, strike=1.0, optiontype="C")
    np.testing.assert_allclose([p, v], [0.197331, 0.999577], rtol=5e-6, atol=1e-8)        # quickstart.py:43-44 (the 6m ATM vol: test_gpu_mgf.py)
