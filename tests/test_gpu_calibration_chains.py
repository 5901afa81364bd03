"""GPU tests of the multi-chain batched pricers (b200sv_{logsv,heston}_price_chains_batch) and of the lock-step calibration drivers on
them: every row is bit for bit the single-chain batch's row on its own chain, whatever shares the call, and so every lock-step fit is
bit for bit the single-chain driver's."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _chains():
    """four chains of different shapes: M = 1, 3, the BTC sample chain, M = 4; forwards and discount factors away from 1"""
    from stochvolmodels_b200 import get_btc_test_chain_data
    k5, t5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2]), np.array(["P", "P", "C", "C", "C"])
    btc = get_btc_test_chain_data()
    k3 = [np.linspace(0.7, 1.3, n) * f for n, f in ((5, 1.01), (3, 1.02), (9, 1.04))]
    k4 = [np.linspace(0.6, 1.5, n) * 100.0 for n in (4, 7, 11, 2)]
    return [
        (np.array([0.15]), np.array([1.0]), np.array([1.0]), [k5], [t5]),
        (np.array([0.05, 0.3, 0.7]), np.array([1.01, 1.02, 1.04]), np.array([0.999, 0.99, 0.97]), k3,
         [np.where(k >= f, "C", "P") for k, f in zip(k3, (1.01, 1.02, 1.04))]),
        (btc.ttms, btc.forwards, btc.discfactors, btc.strikes_ttms, btc.optiontypes_ttms),
        (np.array([0.02, 0.25, 0.5, 1.5]), np.full(4, 100.0), np.array([1.0, 0.99, 0.98, 0.95]), k4,
         [np.where(k >= 100.0, "C", "P") for k in k4]),
    ]


GROUP_SIZES = (6, 9, 5, 3)        # 9 x 1000 grid points: the thread-per-point ODE kernel; the other groups run on the lane-parallel one


def _logsv_sets(n, seed):
    from stochvolmodels_b200 import engine
    rng = np.random.RandomState(seed)
    base = np.array([0.9, 1.0, 4.0, 4.0, 0.2, 1.5])
    return [engine.logsv_params_c(*(base * (1.0 + 0.2 * rng.uniform(-1, 1, 6)))) for _ in range(n)]


def _heston_sets(n, seed):
    from stochvolmodels_b200 import engine
    rng = np.random.RandomState(seed)
    return [engine.heston_params_c(*(np.array([0.6, 0.8, 3.0, -0.3, 1.1]) * (1.0 + 0.2 * rng.uniform(-1, 1, 5)))) for _ in range(n)]


def _interleaved(sizes, seed):
    """chain_of_set with sizes[k] sets on chain k, in a shuffled interleaving"""
    cos = np.concatenate([np.full(n, k) for k, n in enumerate(sizes)])
    return np.random.RandomState(seed).permutation(cos)


def _reinterleaved(cos, perm):
    """the set indices of chain_of_set ``cos`` in another call order: round-robin over the chains taken in the order ``perm``, each chain's
    sets in their original relative order"""
    queues = {k: [b for b in range(len(cos)) if cos[b] == k] for k in perm}
    seq = []
    while any(queues.values()):
        for k in perm:
            if queues[k]:
                seq.append(queues[k].pop(0))
    return np.array(seq)


def _per_chain_reference(single, chains, chain_of_set, params, etas, scalers):
    """row b of the single-chain batch call on chain k(b) with the sets of k(b), in call order"""
    want = [None] * len(params)
    for k, chain in enumerate(chains):
        idx = [b for b, c in enumerate(chain_of_set) if c == k]
        if not idx:
            continue
        e = None if etas is None else np.array([etas[b] for b in idx])
        prices, ivols = single([params[b] for b in idx], chain, e, scalers[k])
        for i, b in enumerate(idx):
            want[b] = (prices[i], ivols[i])
    return want


def _assert_rows(got, want):
    prices, ivols = got
    for b, (p, v) in enumerate(want):
        np.testing.assert_array_equal(prices[b], p, err_msg=f"prices of set {b}")
        np.testing.assert_array_equal(ivols[b], v, err_msg=f"ivols of set {b}")


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("spot", [True, False])
def test_logsv_chains_rows_equal_single_chain_batches_bitwise(cuda_lib, order, spot):
    from stochvolmodels_b200 import LogSVPricer, engine, get_btc_test_chain_data
    chains = _chains()
    cos = _interleaved(GROUP_SIZES, 1)
    params = _logsv_sets(len(cos), 2)
    rng = np.random.RandomState(3)
    etas = [rng.uniform(0.85, 1.15, len(chains[k][0])) for k in cos]
    btc_scaler = LogSVPricer().set_vol_scaler(get_btc_test_chain_data())
    for scalers in ([None, 0.2, btc_scaler, None], [None] * 4, [0.15, 0.25, 0.3, 0.1]):
        def single(ps, chain, e, vs):
            return engine.logsv_price_chain_batch(ps, *chain[:3], e, *chain[3:], is_spot_measure=spot, expansion_order=order, vol_scaler=vs)

        want = _per_chain_reference(single, chains, cos, params, etas, scalers)
        got = engine.logsv_price_chains_batch(params, cos, chains, etas, scalers, is_spot_measure=spot, expansion_order=order)
        _assert_rows(got, want)
        # the chains in another order and the sets interleaved otherwise (each chain's sets still in the same relative order)
        perm = [2, 0, 3, 1]
        new_of_old = np.argsort(perm)
        seq = _reinterleaved(cos, perm)
        got2 = engine.logsv_price_chains_batch([params[b] for b in seq], new_of_old[cos[seq]], [chains[i] for i in perm],
                                               [etas[b] for b in seq], [scalers[i] for i in perm], is_spot_measure=spot, expansion_order=order)
        _assert_rows(got2, [want[b] for b in seq])
    # no etas == etas of ones
    none = engine.logsv_price_chains_batch(params, cos, chains, None, None, is_spot_measure=spot, expansion_order=order)
    ones = engine.logsv_price_chains_batch(params, cos, chains, [np.ones(len(chains[k][0])) for k in cos], None, is_spot_measure=spot,
                                           expansion_order=order)
    for a, b in zip(none[0] + none[1], ones[0] + ones[1]):
        np.testing.assert_array_equal(a, b)


def test_heston_chains_rows_equal_single_chain_batches_bitwise(cuda_lib):
    from stochvolmodels_b200 import engine
    chains = _chains()
    cos = _interleaved(GROUP_SIZES, 4)
    params = _heston_sets(len(cos), 5)
    for scalers in ([None, 0.2, 0.3, None], [None] * 4):
        def single(ps, chain, e, vs):
            return engine.heston_price_chain_batch(ps, *chain, vol_scaler=vs)

        want = _per_chain_reference(single, chains, cos, params, None, scalers)
        _assert_rows(engine.heston_price_chains_batch(params, cos, chains, scalers), want)
        perm = [3, 1, 0, 2]
        new_of_old = np.argsort(perm)
        seq = _reinterleaved(cos, perm)
        got = engine.heston_price_chains_batch([params[b] for b in seq], new_of_old[cos[seq]], [chains[i] for i in perm],
                                               [scalers[i] for i in perm])
        _assert_rows(got, [want[b] for b in seq])


def test_chains_batch_argument_errors(cuda_lib):
    from stochvolmodels_b200 import engine
    chains = _chains()[:2]
    lp, hp = _logsv_sets(2, 0), _heston_sets(2, 0)
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch(lp, [0, 2], chains)                                # chain index out of range
    with pytest.raises(ValueError):
        engine.heston_price_chains_batch(hp, [0, -1], chains)
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch(lp, [0], chains)                                   # one chain index per set
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch(lp, [0, 1], chains, [np.ones(1), np.ones(1)])      # set 1's chain has 3 maturities
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch(lp, [0, 1], chains, [np.ones(1)])                  # one backbone per set
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch(lp, [0, 1], chains, None, [0.2])                   # one scaler per chain
    with pytest.raises(ValueError):
        engine.heston_price_chains_batch(hp, [0, 1], chains, [0.2, 0.2, 0.2])
    with pytest.raises(ValueError):
        engine.logsv_price_chains_batch([], [], chains)
    inverse = (chains[0][0], chains[0][1], chains[0][2], chains[0][3], [np.array(["IC"] * 5)])
    with pytest.raises(ValueError, match="not implemented"):
        engine.logsv_price_chains_batch(lp, [0, 0], [inverse], is_spot_measure=True)


# ---- lock-step calibration ----------------------------------------------------------------------------------------------------
def _option_chain(chain, vols):
    from stochvolmodels_b200 import OptionChain
    ttms, forwards, discfactors, strikes, types = chain
    split = np.split(vols, np.cumsum([len(k) for k in strikes])[:-1])
    return OptionChain(ttms=ttms, forwards=forwards, discfactors=discfactors, strikes_ttms=strikes, optiontypes_ttms=types,
                       ids=np.array([f"{t:0.4f}" for t in ttms]), bid_ivs=[v - 0.002 for v in split], ask_ivs=[v + 0.002 for v in split])


def _logsv_markets():
    """synthetic model markets at drifting parameters on three chains, plus the BTC sample chain's own quotes"""
    from stochvolmodels_b200 import engine, get_btc_test_chain_data
    chains = _chains()
    out = []
    for i, k in enumerate((0, 1, 3)):
        truth = engine.logsv_params_c(0.8 + 0.05 * i, 0.9 + 0.05 * i, 3.0, 3.0, 0.3 - 0.1 * i, 1.3 + 0.1 * i)
        _, iv = engine.logsv_price_chain_batch([truth], *chains[k][:3], None, *chains[k][3:], vol_scaler=0.2)
        out.append(_option_chain(chains[k], iv[0]))
    out.append(get_btc_test_chain_data())
    return out


def _heston_markets():
    from stochvolmodels_b200 import engine, get_btc_test_chain_data
    chains = _chains()
    out = []
    for i, k in enumerate((0, 1, 3)):
        truth = engine.heston_params_c(0.5 + 0.05 * i, 0.6, 2.5 + i, -0.4 + 0.1 * i, 0.9)
        _, iv = engine.heston_price_chain_batch([truth], *chains[k])
        out.append(_option_chain(chains[k], iv[0]))
    out.append(get_btc_test_chain_data())
    return out


def _assert_same_fits(lockstep, sequential):
    (fits, infos), seq = lockstep, sequential
    for k, (fit, info) in enumerate(seq):
        for key in ("fun", "nit", "nb_batches"):
            assert infos[k][key] == info[key], (k, key)
        np.testing.assert_array_equal(infos[k]["x"], info["x"])
        assert infos[k].get("nan_quotes") == info.get("nan_quotes")
        assert infos[k]["rounds"] == max(i["nb_batches"] for i in infos)
        for name in ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol", "v0", "kappa", "rho"):
            if hasattr(fit, name):
                assert getattr(fits[k], name) == getattr(fit, name), (k, name)


@pytest.mark.parametrize("calibration_type, constraints", [("PARAMS4", "UNCONSTRAINT"), ("PARAMS5", "MMA_MARTINGALE"),
                                                           ("PARAMS_WITH_VARSWAP_FIT", "UNCONSTRAINT")])
def test_logsv_lockstep_fits_equal_single_chain_fits_bitwise(cuda_lib, calibration_type, constraints):
    from stochvolmodels_b200 import ConstraintsType, LogSvParams, LogSVPricer, LogsvModelCalibrationType, _capi
    pricer = LogSVPricer()
    markets = _logsv_markets()
    start = LogSvParams(sigma0=0.85, theta=0.95, kappa1=3.0, kappa2=3.0, beta=0.1, volvol=1.2)
    kw = dict(model_calibration_type=LogsvModelCalibrationType[calibration_type], constraints_type=ConstraintsType[constraints])
    seq = [pricer.calibrate_model_params_to_chain(c, start, return_info=True, **kw) for c in markets]
    lib = _capi.load_library()
    lib.b200sv_reset_launch_count()
    out = pricer.calibrate_model_params_to_chains(markets, start, return_info=True, **kw)
    _assert_same_fits(out, seq)
    # one multi-chain call per round: one log-MGF launch per chain still fitting and one Fourier-sum launch
    assert lib.b200sv_launch_count() == sum(i["nb_batches"] for i in out[1]) + out[1][0]["rounds"]
    if calibration_type == "PARAMS_WITH_VARSWAP_FIT":
        for (fit, _), lock, market in zip(seq, out[0], markets):
            np.testing.assert_array_equal(lock.get_vol_backbone_etas(market.ttms), fit.get_vol_backbone_etas(market.ttms))


def test_small_max_sets_per_call_gives_the_same_fits(cuda_lib):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer
    pricer = LogSVPricer()
    markets = _logsv_markets()
    start = LogSvParams(sigma0=0.85, theta=0.95, kappa1=3.0, kappa2=3.0, beta=0.1, volvol=1.2)
    fits, infos = pricer.calibrate_model_params_to_chains(markets, start, return_info=True)
    fits2, infos2 = pricer.calibrate_model_params_to_chains(markets, start, return_info=True, max_sets_per_call=7)
    assert infos2[0]["rounds"] > infos[0]["rounds"] == max(i["nb_batches"] for i in infos)
    for a, b, ia, ib in zip(fits, fits2, infos, infos2):
        np.testing.assert_array_equal(ia["x"], ib["x"])
        assert ia["fun"] == ib["fun"] and ia["nit"] == ib["nit"]


def test_heston_lockstep_fits_equal_single_chain_fits_bitwise(cuda_lib):
    from stochvolmodels_b200 import HestonParams, HestonPricer
    pricer = HestonPricer()
    markets = _heston_markets()
    start = HestonParams(v0=0.5, theta=0.5, kappa=3.0, rho=-0.2, volvol=1.0)
    seq = [pricer.calibrate_model_params_to_chain(c, start, return_info=True) for c in markets]
    _assert_same_fits(pricer.calibrate_model_params_to_chains(markets, start, return_info=True), seq)


def test_a_rejected_round_reaches_every_fit_as_value_error(cuda_lib):
    """one chain quotes inverse payoffs, which the spot measure does not price: the round's multi-chain call is rejected with ValueError
    before any launch, and that error is the answer of every fit of the round (they share the call)"""
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain, _capi
    k, v = np.array([0.9, 1.0, 1.1]), np.full(3, 0.5)
    inverse = OptionChain(ttms=np.array([0.1]), forwards=np.ones(1), strikes_ttms=[k], optiontypes_ttms=[np.array(["IP", "IC", "IC"])],
                          ids=np.array(["a"]), bid_ivs=[v - 0.01], ask_ivs=[v + 0.01])
    markets = _logsv_markets()
    markets.insert(2, inverse)
    start = LogSvParams(sigma0=0.85, theta=0.95, kappa1=3.0, kappa2=3.0, beta=0.1, volvol=1.2)
    lib = _capi.load_library()
    lib.b200sv_reset_launch_count()
    fits = LogSVPricer().calibrate_model_params_to_chains(markets, start, return_exceptions=True)
    assert all(isinstance(f, ValueError) and str(f) == "not implemented" for f in fits)
    with pytest.raises(ValueError, match="not implemented"):
        LogSVPricer().calibrate_model_params_to_chains(markets, start)
    assert lib.b200sv_launch_count() == 0
    # the same chains without the inverse one fit as usual
    del markets[2]
    assert all(isinstance(f, LogSvParams) for f in LogSVPricer().calibrate_model_params_to_chains(markets, start, return_exceptions=True))
