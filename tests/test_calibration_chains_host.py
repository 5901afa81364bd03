"""CPU tests of the lock-step multi-chain calibration drivers (LogSVPricer / HestonPricer.calibrate_model_params_to_chains): the
coordinator, the argument checks and the error handling, on a numpy stand-in for the batched chain pricers.  The stand-in prices every
row from its own set and chain only, as the library does, so lock-step fits must equal the sequential ones bit for bit."""
import threading

import numpy as np
import pytest

from stochvolmodels_b200 import (CalibrationEngine, ConstraintsType, HestonParams, HestonPricer, LogSvParams, LogSVPricer,
                                 LogsvModelCalibrationType, OptionChain, engine)
from stochvolmodels_b200.pricers.calibration import CalibrationError

FAIL_FORWARD = 13.0        # a chain whose first forward is this gets infinite model vols from the stand-in, and its fit fails


def _logsv_vols(p, ttms, forwards, eta, strikes_ttms, fail=True):
    rows = []
    for m, (t, f, ks) in enumerate(zip(ttms, forwards, strikes_ttms)):
        x = np.log(np.asarray(ks, dtype=float) / f)
        v = (p.sigma0 * eta[m] * (1.0 + 0.2 * p.beta * x + 0.1 * p.volvol * x * x) + 0.05 * (p.theta - p.sigma0) * np.sqrt(t)
             + 0.01 * p.kappa1 * t)
        rows.append(np.full_like(x, np.inf) if fail and f == FAIL_FORWARD else v)
    return np.concatenate(rows)


def _heston_vols(p, ttms, forwards, strikes_ttms, fail=True):
    rows = []
    for t, f, ks in zip(ttms, forwards, strikes_ttms):
        x = np.log(np.asarray(ks, dtype=float) / f)
        v = np.sqrt(p.v0) + 0.3 * p.rho * x + 0.1 * p.volvol * x * x + 0.02 * p.kappa * (p.theta - p.v0) * t
        rows.append(np.full_like(x, np.inf) if fail and f == FAIL_FORWARD else v)
    return np.concatenate(rows)


class StandIn:
    """numpy stand-ins for engine.{logsv,heston}_price_chain{,s}_batch that count their calls"""

    def __init__(self, monkeypatch, fail_on_call=None, fail_with=RuntimeError):
        self.calls, self.sets, self.fail_on_call, self.fail_with = 0, [], fail_on_call, fail_with
        for name in ("logsv_price_chain_batch", "heston_price_chain_batch", "logsv_price_chains_batch", "heston_price_chains_batch"):
            monkeypatch.setattr(engine, name, getattr(self, name))

    def _count(self, n):
        self.calls += 1
        self.sets.append(n)
        if self.fail_on_call == self.calls:
            raise self.fail_with("library failure")

    def logsv_price_chain_batch(self, params_list, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, is_spot_measure=True,
                                vol_scaler=None, **kw):
        self._count(len(params_list))
        etas = np.ones((len(params_list), len(ttms))) if etas is None else etas
        return None, np.vstack([_logsv_vols(p, ttms, forwards, e, strikes_ttms) for p, e in zip(params_list, etas)])

    def heston_price_chain_batch(self, params_list, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, vol_scaler=None, **kw):
        self._count(len(params_list))
        return None, np.vstack([_heston_vols(p, ttms, forwards, strikes_ttms) for p in params_list])

    def logsv_price_chains_batch(self, params_list, chain_of_set, chains, etas=None, vol_scalers=None, is_spot_measure=True, **kw):
        self._count(len(params_list))
        assert len(vol_scalers) == len(chains)
        rows = [_logsv_vols(p, chains[k][0], chains[k][1], np.ones(len(chains[k][0])) if etas is None else etas[b], chains[k][3])
                for b, (p, k) in enumerate(zip(params_list, chain_of_set))]
        return None, rows

    def heston_price_chains_batch(self, params_list, chain_of_set, chains, vol_scalers=None, **kw):
        self._count(len(params_list))
        return None, [_heston_vols(p, chains[k][0], chains[k][1], chains[k][3]) for p, k in zip(params_list, chain_of_set)]


def _chain(ttms, forward, truth_vols, n_strikes):
    strikes = [forward * np.linspace(0.8, 1.2, n_strikes) for _ in ttms]
    types = [np.where(k >= forward, "C", "P") for k in strikes]
    vols = truth_vols(np.asarray(ttms), np.full(len(ttms), forward), strikes)
    split = np.split(vols, np.cumsum([len(k) for k in strikes])[:-1])
    return OptionChain(ttms=np.asarray(ttms), forwards=np.full(len(ttms), forward), strikes_ttms=strikes, optiontypes_ttms=types,
                       ids=np.array([f"{t:0.3f}" for t in ttms]), bid_ivs=[v - 0.001 for v in split], ask_ivs=[v + 0.001 for v in split])


def _logsv_chains(fail_index=None):
    shapes = [([0.1], 1.0, 5), ([0.05, 0.2, 0.5], 100.0, 7), ([0.1, 0.25, 0.5, 1.0], 2.0, 9), ([0.02, 0.3], 0.5, 11)]
    out = []
    for i, (ttms, fw, n) in enumerate(shapes):
        truth = LogSvParams(sigma0=0.8 + 0.05 * i, theta=1.0, kappa1=3.0, kappa2=3.0, beta=0.2 - 0.1 * i, volvol=1.2 + 0.1 * i)
        out.append(_chain(ttms, FAIL_FORWARD if i == fail_index else fw,
                          lambda t, f, k, p=truth: _logsv_vols(p, t, f, np.ones(len(t)), k, False), n))
    return out


def _heston_chains(fail_index=None):
    shapes = [([0.1], 1.0, 5), ([0.05, 0.2, 0.5], 100.0, 7), ([0.1, 0.25, 0.5, 1.0], 2.0, 9), ([0.02, 0.3], 0.5, 11)]
    out = []
    for i, (ttms, fw, n) in enumerate(shapes):
        truth = HestonParams(v0=0.3 + 0.05 * i, theta=0.4, kappa=2.0 + i, rho=-0.3 + 0.1 * i, volvol=0.8)
        out.append(_chain(ttms, FAIL_FORWARD if i == fail_index else fw, lambda t, f, k, p=truth: _heston_vols(p, t, f, k, False), n))
    return out


START = LogSvParams(sigma0=0.9, theta=0.9, kappa1=3.0, kappa2=3.0, beta=0.0, volvol=1.0)


def _sequential_logsv(chains, starts, **kw):
    pricer = LogSVPricer()
    return [pricer.calibrate_model_params_to_chain(c, s, return_info=True, **kw) for c, s in zip(chains, starts)]


def _same_fit(a, b):
    (fa, ia), (fb, ib) = a, b
    for k in ("fun", "nit", "nb_batches", "nan_quotes"):
        assert ia.get(k) == ib.get(k), (k, ia.get(k), ib.get(k))
    np.testing.assert_array_equal(ia["x"], ib["x"])
    _same_params(fa, fb)


def _same_params(a, b):
    assert type(a) is type(b) and vars(a).keys() == vars(b).keys()
    for name, v in vars(a).items():
        w = vars(b)[name]
        if hasattr(v, "equals"):                  # the vol backbone of PARAMS_WITH_VARSWAP_FIT (a pandas Series)
            assert v.equals(w), name
        elif v is None or w is None:
            assert v is w, name
        else:
            np.testing.assert_array_equal(v, w, err_msg=name)


@pytest.mark.parametrize("calibration_type, constraints", [
    (LogsvModelCalibrationType.PARAMS4, ConstraintsType.UNCONSTRAINT),
    (LogsvModelCalibrationType.PARAMS5, ConstraintsType.MMA_MARTINGALE),
    (LogsvModelCalibrationType.PARAMS5, ConstraintsType.INVERSE_MARTINGALE_MOMENT4),
])
def test_logsv_lockstep_fits_equal_sequential_fits(monkeypatch, calibration_type, constraints):
    chains = _logsv_chains()
    stand_in = StandIn(monkeypatch)
    kw = dict(model_calibration_type=calibration_type, constraints_type=constraints)
    seq = _sequential_logsv(chains, [START] * 4, **kw)
    stand_in.calls, stand_in.sets = 0, []
    fits, infos = LogSVPricer().calibrate_model_params_to_chains(chains, START, return_info=True, **kw)
    for k in range(4):
        _same_fit((fits[k], infos[k]), seq[k])
        assert infos[k]["rounds"] == stand_in.calls
    assert stand_in.calls == max(i["nb_batches"] for i in infos)
    assert max(stand_in.sets) <= 4 * (1 + len(infos[0]["x"]))
    # without return_info: the fits alone
    for a, b in zip(LogSVPricer().calibrate_model_params_to_chains(chains, START, **kw), fits):
        _same_params(a, b)


def test_max_sets_per_call_splits_rounds_and_keeps_the_fits(monkeypatch):
    chains = _logsv_chains()
    stand_in = StandIn(monkeypatch)
    fits, infos = LogSVPricer().calibrate_model_params_to_chains(chains, START, return_info=True)
    calls = stand_in.calls
    stand_in.calls, stand_in.sets = 0, []
    fits2, infos2 = LogSVPricer().calibrate_model_params_to_chains(chains, START, return_info=True, max_sets_per_call=7)
    for a, b in zip(fits2, fits):
        _same_params(a, b)
    assert all(n <= 7 for n in stand_in.sets)          # a fit's 6 sets never split, two fits never share a call
    assert stand_in.calls == infos2[0]["rounds"] > calls
    assert [i["x"].tolist() for i in infos2] == [i["x"].tolist() for i in infos]


def test_per_chain_and_scalar_start_points_and_bounds(monkeypatch):
    chains = _logsv_chains()
    StandIn(monkeypatch)
    starts = [LogSvParams(sigma0=0.7 + 0.1 * i, theta=0.9, kappa1=3.0, kappa2=3.0, beta=0.1, volvol=1.1) for i in range(4)]
    lo = LogSvParams(sigma0=0.2, theta=0.2, kappa1=0.5, kappa2=0.5, beta=-2.0, volvol=0.3)
    his = [LogSvParams(sigma0=1.2 + 0.1 * i, theta=1.5, kappa1=8.0, kappa2=8.0, beta=2.0, volvol=2.5) for i in range(4)]
    fits, infos = LogSVPricer().calibrate_model_params_to_chains(chains, starts, params_min=lo, params_max=his, return_info=True)
    pricer = LogSVPricer()
    for k in range(4):
        _same_fit((fits[k], infos[k]), pricer.calibrate_model_params_to_chain(chains[k], starts[k], params_min=lo, params_max=his[k],
                                                                               return_info=True))


def test_varswap_fit_lockstep_equals_sequential(monkeypatch):
    chains = _logsv_chains()[1:3]
    StandIn(monkeypatch)
    kw = dict(model_calibration_type=LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT)
    seq = _sequential_logsv(chains, [START] * 2, **kw)
    fits, infos = LogSVPricer().calibrate_model_params_to_chains(chains, START, return_info=True, **kw)
    for k in range(2):
        _same_fit((fits[k], infos[k]), seq[k])
        np.testing.assert_array_equal(fits[k].get_vol_backbone_etas(chains[k].ttms), seq[k][0].get_vol_backbone_etas(chains[k].ttms))


def test_heston_lockstep_fits_equal_sequential_fits(monkeypatch):
    chains = _heston_chains()
    stand_in = StandIn(monkeypatch)
    pricer = HestonPricer()
    start = HestonParams(v0=0.35, theta=0.35, kappa=2.5, rho=-0.1, volvol=0.7)
    seq = [pricer.calibrate_model_params_to_chain(c, start, return_info=True) for c in chains]
    stand_in.calls = 0
    fits, infos = pricer.calibrate_model_params_to_chains(chains, start, return_info=True)
    for k in range(4):
        _same_fit((fits[k], infos[k]), seq[k])
    assert stand_in.calls == max(i["nb_batches"] for i in infos) == infos[0]["rounds"]
    # params0=None: the driver's default start point on every chain
    for a, c in zip(pricer.calibrate_model_params_to_chains(chains), chains):
        _same_params(a, pricer.calibrate_model_params_to_chain(c))


def test_rejections_come_before_any_library_call(monkeypatch):
    stand_in = StandIn(monkeypatch)
    chains = _logsv_chains()
    pricer = LogSVPricer()
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains([], START)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, [START] * 3)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, params_min=[None] * 5)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, params_max=(None,))
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, max_sets_per_call=0)
    for eng in (CalibrationEngine.MC, CalibrationEngine.ROUGH_MC):
        with pytest.raises(NotImplementedError):
            pricer.calibrate_model_params_to_chains(chains, START, calibration_engine=eng)
    for gradient in ("exact", "pathwise"):
        with pytest.raises(NotImplementedError):
            pricer.calibrate_model_params_to_chains(chains, START, gradient=gradient)
        with pytest.raises(NotImplementedError):
            HestonPricer().calibrate_model_params_to_chains(_heston_chains(), gradient=gradient)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, gradient="central")
    with pytest.raises(NotImplementedError):
        pricer.calibrate_model_params_to_chains(chains, START, model_calibration_type=LogsvModelCalibrationType.PARAMS6)
    with pytest.raises(ValueError):
        HestonPricer().calibrate_model_params_to_chains([])
    with pytest.raises(ValueError):
        HestonPricer().calibrate_model_params_to_chains(_heston_chains(), [None] * 2)
    assert stand_in.calls == 0


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_a_failing_fit_leaves_the_others_intact(monkeypatch, model):
    StandIn(monkeypatch)
    if model == "logsv":
        pricer, start, chains = LogSVPricer(), START, _logsv_chains(fail_index=1)
    else:
        pricer, start, chains = HestonPricer(), HestonParams(v0=0.35, theta=0.35, kappa=2.5, rho=-0.1, volvol=0.7), _heston_chains(fail_index=1)
    with pytest.raises(CalibrationError):
        pricer.calibrate_model_params_to_chain(chains[1], start)
    before = threading.active_count()
    fits, infos = pricer.calibrate_model_params_to_chains(chains, start, return_info=True, return_exceptions=True)
    assert isinstance(fits[1], CalibrationError) and infos[1] is None
    for k in (0, 2, 3):
        _same_fit((fits[k], infos[k]), pricer.calibrate_model_params_to_chain(chains[k], start, return_info=True))
    with pytest.raises(CalibrationError):
        pricer.calibrate_model_params_to_chains(chains, start)
    assert threading.active_count() == before


def test_lowest_index_error_is_raised(monkeypatch):
    StandIn(monkeypatch)
    chains = _logsv_chains(fail_index=2)
    chains[0] = _logsv_chains(fail_index=0)[0]
    out = LogSVPricer().calibrate_model_params_to_chains(chains, START, return_exceptions=True)
    assert isinstance(out[0], CalibrationError) and isinstance(out[2], CalibrationError)
    with pytest.raises(CalibrationError) as err:
        LogSVPricer().calibrate_model_params_to_chains(chains, START)
    assert err.value is out[0] or str(err.value) == str(out[0])


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_a_failing_library_call_reaches_every_fit_of_its_round(monkeypatch, model):
    stand_in = StandIn(monkeypatch, fail_on_call=3)
    pricer, start, chains = ((LogSVPricer(), START, _logsv_chains()) if model == "logsv" else
                             (HestonPricer(), HestonParams(v0=0.35, theta=0.35, kappa=2.5, rho=-0.1, volvol=0.7), _heston_chains()))
    before = threading.active_count()
    fits = pricer.calibrate_model_params_to_chains(chains, start, return_exceptions=True)
    assert all(isinstance(f, RuntimeError) and str(f) == "library failure" for f in fits)
    assert stand_in.calls == 3
    with pytest.raises(RuntimeError, match="library failure"):
        stand_in.calls = 0
        pricer.calibrate_model_params_to_chains(chains, start)
    deadline = threading.Event()
    for _ in range(100):
        if threading.active_count() == before:
            break
        deadline.wait(0.05)
    assert threading.active_count() == before


class Interrupt(BaseException):
    """not an Exception, as KeyboardInterrupt or SystemExit"""


@pytest.mark.parametrize("model", ["logsv", "heston"])
@pytest.mark.parametrize("interrupt", [Interrupt, KeyboardInterrupt])
def test_an_interrupt_inside_the_batched_call_ends_every_fit(monkeypatch, model, interrupt):
    """a BaseException raised by the multi-chain call of a round (Ctrl-C while the GPU prices it) reaches the caller, and every fit
    thread -- those of the round in flight included -- ends instead of waiting for a round that never comes"""
    stand_in = StandIn(monkeypatch, fail_on_call=3, fail_with=interrupt)
    pricer, start, chains = ((LogSVPricer(), START, _logsv_chains()) if model == "logsv" else
                             (HestonPricer(), HestonParams(v0=0.35, theta=0.35, kappa=2.5, rho=-0.1, volvol=0.7), _heston_chains()))
    before = threading.active_count()
    caught = []

    def call():
        try:
            pricer.calibrate_model_params_to_chains(chains, start)
        except BaseException as exc:                  # noqa: BLE001
            caught.append(exc)

    caller = threading.Thread(target=call, daemon=True)      # a daemon: a regression fails this test instead of hanging the run
    caller.start()
    caller.join(timeout=60)
    assert not caller.is_alive(), "the lock-step call did not return"
    assert len(caught) == 1 and type(caught[0]) is interrupt and str(caught[0]) == "library failure"
    assert stand_in.calls == 3
    assert threading.active_count() == before


def _chains_call(model, chain_of_set, Ms, order=2, null_scalers=False):
    """b200sv_{logsv,heston}_price_chains_batch on two chains of 3 strikes per maturity, with only the given ``Ms`` and ``chain_of_set``
    varied: every case below is rejected before any CUDA call"""
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    B, K = len(chain_of_set), len(Ms)
    n = sum(max(m, 0) for m in Ms)
    ttms, fw, df = C.f64(np.tile([0.25, 0.5, 0.75], 4)[:max(n, 1)]), np.ones(max(n, 1)), np.ones(max(n, 1))
    offs = np.concatenate([np.arange(max(m, 0) + 1) * 3 for m in Ms]).astype(np.int32)
    strikes, types = C.f64(np.tile([0.9, 1.0, 1.1], 12)), np.tile(np.array([C.PUT, C.CALL, C.CALL], dtype=np.int8), 12)
    cos, ms, scalers = np.asarray(chain_of_set, dtype=np.int32), np.asarray(Ms, dtype=np.int32), np.full(K, -1.0)
    out = np.zeros(256)
    sc = None if null_scalers else C.dptr(scalers)
    if model == "logsv":
        ps = (C.LogsvParamsC * B)(*[C.LogsvParamsC(1.0, 1.0, 5.0, 5.0, 0.2, 2.0)] * B)
        rc = lib.b200sv_logsv_price_chains_batch(ps, B, C.iptr(cos), K, C.iptr(ms), C.dptr(ttms), C.dptr(fw), C.dptr(df), None, C.iptr(offs),
                                                 C.dptr(strikes), C.i8ptr(types), 1, order, sc, 0, C.dptr(out), None)
    else:
        ps = (C.HestonParamsC * B)(*[C.HestonParamsC(0.04, 0.04, 4.0, -0.5, 0.5)] * B)
        rc = lib.b200sv_heston_price_chains_batch(ps, B, C.iptr(cos), K, C.iptr(ms), C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(offs),
                                                  C.dptr(strikes), C.i8ptr(types), sc, 0, C.dptr(out), None)
    return rc, lib.b200sv_last_error().decode()


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_library_rejects_bad_chains_arguments_before_any_cuda_call(model):
    assert _chains_call(model, [0, 2], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _chains_call(model, [0, -1], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _chains_call(model, [0, 0], [2, 0]) == (-1, "invalid argument: every chain needs M >= 1")      # chain 1 has no set, yet
    assert _chains_call(model, [], [2, 1]) == (-1, "invalid argument: B >= 1, K >= 1")
    assert _chains_call(model, [0, 1], [2, 1], null_scalers=True) == (-1, "invalid argument: null pointer")
    if model == "logsv":
        assert _chains_call(model, [0, 1], [2, 1], order=3) == (-4, "expansion_order not implemented")
