"""GPU tests of the batched chain pricers and the calibration drivers built on them (SURVEY.md §8f #2)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, chain_from_golden, load_golden
from oracle import bsm as obsm

pytestmark = pytest.mark.gpu
K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])


def _sets():
    base = np.array([1.0, 1.0, 5.0, 5.0, 0.2, 2.0])
    rng = np.random.RandomState(3)
    return [base * (1.0 + 0.2 * rng.uniform(-1, 1, 6)) for _ in range(7)]


@pytest.mark.parametrize("vol_scaler", [None, 0.21])
@pytest.mark.parametrize("spot", [True, False])
def test_logsv_batch_rows_equal_single_calls_bitwise(cuda_lib, vol_scaler, spot):
    from stochvolmodels_b200 import engine
    ttms, fw, df = np.array([0.1, 0.3, 0.7]), np.array([1.0, 1.01, 1.02]), np.array([1.0, 0.99, 0.98])
    strikes = [K5, K5[:3], np.linspace(0.7, 1.4, 9)]
    types = [T5, T5[:3], np.where(strikes[2] >= 1.02, "C", "P")]
    sets = _sets()
    etas = np.tile(np.array([1.0, 0.95, 1.1]), (len(sets), 1)) * np.linspace(0.9, 1.1, len(sets))[:, None]
    prices, ivols = engine.logsv_price_chain_batch([engine.logsv_params_c(*s) for s in sets], ttms, fw, df, etas, strikes, types,
                                                   is_spot_measure=spot, vol_scaler=vol_scaler)
    assert prices.shape == ivols.shape == (len(sets), 17)
    for b, s in enumerate(sets):
        single = engine.logsv_price_chain(engine.logsv_params_c(*s), ttms, fw, df, etas[b], strikes, types, spot, 2, vol_scaler, 1000, False)
        np.testing.assert_array_equal(prices[b], np.concatenate(single))
        iv = engine.bsm_implied_vols(ttms, fw, df, strikes, types, single)
        np.testing.assert_array_equal(ivols[b], np.concatenate(iv))
    # no etas == etas of ones; prices only
    p1, none = engine.logsv_price_chain_batch([engine.logsv_params_c(*sets[0])], ttms, fw, df, None, strikes, types, is_spot_measure=spot,
                                              vol_scaler=vol_scaler, with_ivols=False)
    assert none is None
    single = engine.logsv_price_chain(engine.logsv_params_c(*sets[0]), ttms, fw, df, np.ones(3), strikes, types, spot, 2, vol_scaler, 1000, False)
    np.testing.assert_array_equal(p1[0], np.concatenate(single))


def test_lane_parallel_and_thread_per_point_ode_kernels_agree(cuda_lib):
    """a 12-set batch (12000 grid points: thread-per-point kernel) against single calls (1000 points: lane-parallel kernel): the two
    kernels take the same accepted steps and differ only in the last bits of the right-hand side's sums."""
    from stochvolmodels_b200 import engine
    ttms, fw, df = np.array([0.1, 0.3, 0.7]), np.array([1.0, 1.01, 1.02]), np.array([1.0, 0.99, 0.98])
    strikes, types = [K5, K5, K5], [T5, T5, T5]
    rng = np.random.RandomState(11)
    base = np.array([1.0, 1.0, 5.0, 5.0, 0.2, 2.0])
    sets = [base * (1.0 + 0.2 * rng.uniform(-1, 1, 6)) for _ in range(12)]
    for order in (2, 1):
        prices, _ = engine.logsv_price_chain_batch([engine.logsv_params_c(*s) for s in sets], ttms, fw, df, None, strikes, types,
                                                   expansion_order=order, vol_scaler=0.2)
        for b in (0, 5, 11):
            single = engine.logsv_price_chain(engine.logsv_params_c(*sets[b]), ttms, fw, df, np.ones(3), strikes, types, True, order, 0.2, 1000, False)
            np.testing.assert_allclose(prices[b], np.concatenate(single), rtol=1e-12, atol=1e-15)


def test_heston_batch_rows_equal_single_calls_bitwise(cuda_lib):
    from stochvolmodels_b200 import engine
    ttms, fw, df = np.array([0.1, 0.3]), np.array([1.0, 1.01]), np.array([1.0, 0.99])
    strikes, types = [K5, K5], [T5, T5]
    rng = np.random.RandomState(5)
    sets = [np.array([0.6, 0.8, 3.0, -0.3, 1.1]) * (1.0 + 0.2 * rng.uniform(-1, 1, 5)) for _ in range(6)]
    for vs in (None, 0.25):
        prices, ivols = engine.heston_price_chain_batch([engine.heston_params_c(*s) for s in sets], ttms, fw, df, strikes, types, vol_scaler=vs)
        for b, s in enumerate(sets):
            single = engine.heston_price_chain(engine.heston_params_c(*s), ttms, fw, df, strikes, types, vs)
            np.testing.assert_array_equal(prices[b], np.concatenate(single))
            np.testing.assert_array_equal(ivols[b], np.concatenate(engine.bsm_implied_vols(ttms, fw, df, strikes, types, single)))


def test_batch_matches_reference_golden_and_checker_inversion(cuda_lib):
    """row 0 of a batch == the reference's golden prices of the quickstart chain; fused ivols == oracle/bsm.py bisection."""
    from stochvolmodels_b200 import engine
    g = load_golden("logsv_fourier_g1_quickstart.npz")
    strikes, types = chain_from_golden(g)
    pc = engine.logsv_params_c(*g["params"])
    prices, ivols = engine.logsv_price_chain_batch([pc, pc], g["ttms"], g["forwards"], g["discfactors"], np.tile(g["etas"], (2, 1)), strikes, types,
                                                   is_spot_measure=bool(g["is_spot"]))
    ref = np.concatenate([g[f"prices_{m}"] for m in range(int(g["nslices"]))])
    np.testing.assert_allclose(prices[0], ref, rtol=1e-10)
    np.testing.assert_array_equal(prices[0], prices[1])
    split = np.split(prices[0], np.cumsum([len(s) for s in strikes])[:-1])
    want = obsm.infer_bsm_ivols_from_model_chain_prices(g["ttms"], g["forwards"], g["discfactors"], strikes, types, split)
    np.testing.assert_allclose(ivols[0], np.concatenate(want), rtol=0, atol=1e-13)


def test_batch_argument_errors(cuda_lib):
    from stochvolmodels_b200 import engine
    pc = engine.logsv_params_c(1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
    with pytest.raises(ValueError):
        engine.logsv_price_chain_batch([pc], np.array([0.1]), np.ones(1), np.ones(1), np.ones((2, 1)), [K5], [T5])
    with pytest.raises(ValueError, match="not implemented"):
        engine.logsv_price_chain_batch([pc], np.array([0.1]), np.ones(1), np.ones(1), None, [K5], [np.array(["IC"] * 5)], is_spot_measure=True)


def _chain(g):
    from stochvolmodels_b200 import OptionChain
    vols = [np.asarray(v) for v in g["market_vols"]]
    M = len(g["ttms"])
    return OptionChain(ttms=g["ttms"], ids=np.array([f"{t:0.2f}" for t in g["ttms"]]), forwards=g["forwards"],
                       strikes_ttms=[g["strikes"]] * M, optiontypes_ttms=[g["types"]] * M, bid_ivs=vols, ask_ivs=[v.copy() for v in vols])


def _objective(chain, vols_flat, market_flat):
    from stochvolmodels_b200.pricers.calibration import calibration_weights
    w = calibration_weights(chain, market_flat, True, False)
    return float(np.nansum(w * np.square(vols_flat - market_flat)))


def test_logsv_calibration_vs_reference_driver(cuda_lib):
    """same market, start, bounds and optimizer as the reference's own calibrate_model_params_to_chain run (tests/golden/make_golden.py
    --only-calib, 116 s on the CPU).  The objective is pinned exactly at the reference's optimum (its fitted vols reproduce to 1e-9).
    The optimizer path is not bit-reproducible (scipy differences the objective with h = 1.5e-8 on top of an adaptive ODE solver, so
    1e-13 price differences move the gradient's last digits), but both drivers must stop at the same optimum: the objective
    must agree with the reference's 2.69514e-6."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, LogsvModelCalibrationType
    g = load_golden("calib_logsv_params4.npz")
    chain = _chain(g)
    pricer = LogSVPricer()
    assert pricer.set_vol_scaler(chain) == pytest.approx(float(g["vol_scaler"]), rel=1e-14)
    market = g["market_vols"].ravel()
    ref_vols = pricer.compute_model_ivols_for_chain(chain, LogSvParams(*g["fit"]), vol_scaler=pricer.set_vol_scaler(chain))
    np.testing.assert_allclose(np.array(ref_vols), g["fit_vols"], rtol=0, atol=1e-9)
    f_ref = _objective(chain, g["fit_vols"].ravel(), market)
    assert _objective(chain, np.array(ref_vols).ravel(), market) == pytest.approx(f_ref, rel=1e-5)
    fit, info = pricer.calibrate_model_params_to_chain(chain, LogSvParams(*g["start"]), model_calibration_type=LogsvModelCalibrationType.PARAMS4,
                                                       return_info=True)
    assert fit.kappa1 == g["start"][2] and fit.kappa2 == g["start"][3]            # PARAMS4 keeps kappa1, kappa2
    vols = np.array(pricer.compute_model_ivols_for_chain(chain, fit, vol_scaler=pricer.set_vol_scaler(chain)))
    assert info["fun"] == pytest.approx(_objective(chain, vols.ravel(), market), rel=1e-9)
    assert info["fun"] == pytest.approx(f_ref, rel=1e-3)
    got = np.array([fit.sigma0, fit.theta, fit.kappa1, fit.kappa2, fit.beta, fit.volvol])
    np.testing.assert_allclose(got, g["fit"], atol=2e-2)
    np.testing.assert_allclose(vols, g["fit_vols"], atol=2e-4)
    assert info["nb_batches"] < 200
    # a coarser difference step (opt-in kwarg) reaches the same optimum
    fit2, info2 = pricer.calibrate_model_params_to_chain(chain, LogSvParams(*g["start"]), model_calibration_type=LogsvModelCalibrationType.PARAMS4,
                                                         return_info=True, fd_step=1e-4)
    assert info2["fun"] == pytest.approx(info["fun"], rel=1e-2)


def test_logsv_varswap_fit_calibration_vs_reference_driver(cuda_lib):
    """PARAMS_WITH_VARSWAP_FIT: (beta, volvol) with the eta backbone re-fitted at every optimizer point, against the reference's run."""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, LogsvModelCalibrationType
    g = load_golden("calib_logsv_varswap.npz")
    M = len(g["ttms"])
    from stochvolmodels_b200 import OptionChain
    vols = [np.asarray(v) for v in g["market_vols"]]
    chain = OptionChain(ttms=g["ttms"], ids=np.array([f"{t:0.2f}" for t in g["ttms"]]), forwards=g["forwards"], strikes_ttms=[g["strikes"]] * M,
                        optiontypes_ttms=[g["types"]] * M, bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    pricer = LogSVPricer()
    market = g["market_vols"].ravel()
    ref_fit = LogSvParams(*g["fit"])
    ref_fit.set_vol_backbone(__import__("pandas").Series(g["fit_eta"], index=g["ttms"]))
    ref_vols = np.array(pricer.compute_model_ivols_for_chain(chain, ref_fit, vol_scaler=pricer.set_vol_scaler(chain)))
    np.testing.assert_allclose(ref_vols, g["fit_vols"], rtol=0, atol=1e-9)          # same objective at the reference's optimum
    f_ref = _objective(chain, g["fit_vols"].ravel(), market)
    fit, info = pricer.calibrate_model_params_to_chain(chain, LogSvParams(*g["start"]),
                                                       model_calibration_type=LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT, return_info=True)
    assert (fit.sigma0, fit.theta, fit.kappa1, fit.kappa2) == tuple(g["start"][:4])
    assert info["fun"] <= 1.05 * f_ref + 1e-9
    np.testing.assert_allclose([fit.beta, fit.volvol], g["fit"][4:], atol=3e-2)
    np.testing.assert_allclose(fit.get_vol_backbone_etas(g["ttms"]), g["fit_eta"], rtol=2e-2)


def test_heston_calibration_vs_reference_driver(cuda_lib):
    from stochvolmodels_b200 import HestonParams, HestonPricer
    g = load_golden("calib_heston.npz")
    chain = _chain(g)
    pricer = HestonPricer()
    market = g["market_vols"].ravel()
    ref_vols = pricer.compute_model_ivols_for_chain(chain, HestonParams(*g["fit"]))
    np.testing.assert_allclose(np.array(ref_vols), g["fit_vols"], rtol=0, atol=1e-9)
    f_ref = _objective(chain, g["fit_vols"].ravel(), market)
    fit, info = pricer.calibrate_model_params_to_chain(chain, HestonParams(*g["start"]), return_info=True)
    vols = np.array(pricer.compute_model_ivols_for_chain(chain, fit))
    assert info["fun"] == pytest.approx(_objective(chain, vols.ravel(), market), rel=1e-9)
    assert info["fun"] <= 1.5 * f_ref + 1e-9
    np.testing.assert_allclose(vols, g["market_vols"], atol=3e-3)
    assert 2.0 * fit.kappa * fit.theta - fit.volvol ** 2 >= -1e-8                  # Feller constraint honoured


def test_logsv_calibration_mc_engine_recovers_own_market(cuda_lib):
    """MC engine with fixed device-resident normals (reference :251-266): calibrating to vols produced by the same normals recovers
    the generating beta / volvol."""
    from stochvolmodels_b200 import CalibrationEngine, LogSvParams, LogSVPricer, LogsvModelCalibrationType, OptionChain
    from stochvolmodels_b200.multi_gpu import _fixed_randoms_chain_device
    from stochvolmodels_b200.pricers.logsv_pricer import _params_c, get_randoms_for_chain_valuation
    ttms, fw = np.array([1.0 / 12.0, 0.25]), np.ones(2)
    truth = LogSvParams(sigma0=0.9, theta=1.0, kappa1=4.0, kappa2=4.0, beta=0.3, volvol=1.5)
    flat = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5], ids=np.array(["a", "b"]))
    rnd = get_randoms_for_chain_valuation(ttms=ttms, nb_path=50000, nb_steps_per_year=360, seed=10, device=True)
    prices, _ = _fixed_randoms_chain_device(rnd, ttms, fw, np.ones(2), [K5, K5], [T5, T5], _params_c(truth), np.ones(2), True, 1, True)
    vols = flat.compute_model_ivols_from_chain_data(prices)
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5], ids=np.array(["a", "b"]),
                        bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    start = LogSvParams(sigma0=0.8, theta=0.9, kappa1=4.0, kappa2=4.0, beta=0.1, volvol=1.2)
    fit, info = LogSVPricer().calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS4,
                                                              calibration_engine=CalibrationEngine.MC, nb_path=50000, nb_steps=360, seed=10,
                                                              return_info=True)
    assert info["fun"] < 1e-5
    fit_prices, _ = _fixed_randoms_chain_device(rnd, ttms, fw, np.ones(2), [K5, K5], [T5, T5], _params_c(fit), np.ones(2), True, 1, True)
    fit_vols = flat.compute_model_ivols_from_chain_data(fit_prices)
    np.testing.assert_allclose(np.array(fit_vols), np.array(vols), atol=5e-3)


def test_mc_chain_batch_rows_equal_single_calls_bitwise(cuda_lib):
    """b200sv_*_mc_chain_batch: row b == the single-set fused chain on the same seed; fused ivols == separate Black inversion."""
    from stochvolmodels_b200 import _capi as C, engine
    ttms, fw, df = np.array([0.1, 0.3]), np.array([1.0, 1.01]), np.array([1.0, 0.99])
    strikes, types = [K5, K5[:3]], [T5, T5[:3]]
    sets = _sets()[:4]
    etas = np.array([[1.0, 0.9]] * 4) * np.linspace(0.9, 1.1, 4)[:, None]
    flags = engine.mc_flags("fp64", "fp32")
    for spot in (True, False):
        p, e, iv = engine.logsv_mc_chain_batch([engine.logsv_params_c(*s) for s in sets], ttms, fw, df, etas, strikes, types, 100_000, 360, spot, 42, flags)
        for b, s in enumerate(sets):
            ps, es = engine.logsv_mc_chain(engine.logsv_params_c(*s), ttms, fw, df, etas[b], strikes, types, 100_000, 360, spot, 1, 42, flags)
            np.testing.assert_array_equal(p[b], np.concatenate(ps))
            np.testing.assert_array_equal(e[b], np.concatenate(es))
            np.testing.assert_array_equal(iv[b], np.concatenate(engine.bsm_implied_vols(ttms, fw, df, strikes, types, ps)))
    hsets = [np.array([0.6, 0.8, 3.0, -0.3, 1.1]) * f for f in (1.0, 1.1, 0.9)]
    for scheme in (C.HESTON_EULER_FLOOR, C.HESTON_QE):
        p, e, iv = engine.heston_mc_chain_batch([engine.heston_params_c(*s) for s in hsets], ttms, fw, df, strikes, types, 100_000, 360, 7, flags, scheme)
        for b, s in enumerate(hsets):
            ps, es = engine.heston_mc_chain(engine.heston_params_c(*s), ttms, fw, df, strikes, types, 100_000, 360, 1, 7, flags, scheme)
            np.testing.assert_array_equal(p[b], np.concatenate(ps))
            np.testing.assert_array_equal(iv[b], np.concatenate(engine.bsm_implied_vols(ttms, fw, df, strikes, types, ps)))


def test_logsv_calibration_mc_engine_philox_common_random_numbers(cuda_lib):
    """MC engine on the counter-based generator: the market is produced by the same seed, so the objective has an exact zero at the
    generating parameters and SLSQP must find (near) it; one batched call per evaluation."""
    from stochvolmodels_b200 import CalibrationEngine, LogSvParams, LogSVPricer, LogsvModelCalibrationType, OptionChain, engine
    from stochvolmodels_b200.pricers.logsv_pricer import _params_c
    ttms, fw = np.array([1.0 / 12.0, 0.25]), np.ones(2)
    truth = LogSvParams(sigma0=0.9, theta=1.0, kappa1=4.0, kappa2=4.0, beta=0.3, volvol=1.5)
    _, _, iv = engine.logsv_mc_chain_batch([_params_c(truth)], ttms, fw, np.ones(2), None, [K5, K5], [T5, T5], 200_000, 360, True, 10,
                                           engine.mc_flags("fp64", "fp32"))
    vols = [iv[0, :5].copy(), iv[0, 5:].copy()]
    chain = OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5], ids=np.array(["a", "b"]),
                        bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    start = LogSvParams(sigma0=0.8, theta=0.9, kappa1=4.0, kappa2=4.0, beta=0.1, volvol=1.2)
    fit, info = LogSVPricer().calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS4,
                                                              calibration_engine=CalibrationEngine.MC, nb_path=200_000, nb_steps=360, seed=10,
                                                              mc_randoms="philox", return_info=True)
    assert info["fun"] < 1e-5
    _, _, fit_iv = engine.logsv_mc_chain_batch([_params_c(fit)], ttms, fw, np.ones(2), None, [K5, K5], [T5, T5], 200_000, 360, True, 10,
                                               engine.mc_flags("fp64", "fp32"))
    np.testing.assert_allclose(fit_iv[0], iv[0], atol=5e-3)


def test_calibration_to_the_btc_market_quotes_recovers_the_references_published_fit(cuda_lib):
    """the reference ships LOGSV_BTC_PARAMS as its fit of the BTC sample chain (logsv_pricer.py:102).  Calibrating to the chain's bid/ask
    vols on the GPU, from a perturbed start, lands on those values to the precision they are quoted at, with an objective no worse than
    at the published point."""
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS as ref, LogSvParams, LogSVPricer, LogsvModelCalibrationType, get_btc_test_chain_data
    chain, pricer = get_btc_test_chain_data(), LogSVPricer()
    start = LogSvParams(sigma0=0.7, theta=0.9, kappa1=ref.kappa1, kappa2=ref.kappa2, beta=0.0, volvol=1.4)
    fit, info = pricer.calibrate_model_params_to_chain(chain, start, model_calibration_type=LogsvModelCalibrationType.PARAMS4, return_info=True)
    at_ref = pricer.calibrate_model_params_to_chain(chain, ref, model_calibration_type=LogsvModelCalibrationType.PARAMS4, return_info=True)[1]
    assert info["fun"] <= at_ref["fun"] * (1 + 1e-3)
    for name, tol in (("sigma0", 0.03), ("theta", 0.03), ("beta", 0.03), ("volvol", 0.08)):
        assert abs(getattr(fit, name) - getattr(ref, name)) < tol, (name, getattr(fit, name), getattr(ref, name))
    model = pricer.compute_model_ivols_for_chain(chain, fit)
    rms = np.sqrt(np.mean(np.concatenate([a - b for a, b in zip(model, chain.get_mid_vols())]) ** 2))
    assert rms < 0.02          # 1.5 vol points on a 49-quote BTC surface with vols of 0.85 .. 1.15
