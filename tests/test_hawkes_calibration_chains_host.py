"""CPU tests of HawkesJDPricer.calibrate_model_params_to_chains: its rejections, the coordinator on a numpy stand-in for the batched chain
pricers (which prices every row from its own set and chain only, as the library does, so lock-step fits must equal the single-chain fits
bit for bit), the single-chain driver's library calls, and the argument checks of b200sv_hawkesjd_price_chains_batch."""
import threading

import numpy as np
import pytest

from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine


def _vols(p, ttms, forwards, strikes_ttms):
    rows = []
    for t, f, ks in zip(ttms, forwards, strikes_ttms):
        x = np.log(np.asarray(ks, dtype=float) / f)
        v = (p.sigma + 0.5 * (p.mean_p + p.mean_m) * x + 0.01 * (p.theta_p - p.theta_m) * x * x + 0.001 * p.kappa_p * t
             + 1e-4 * (p.beta1_p - p.beta2_m) * np.sqrt(t))
        rows.append(v)
    return np.concatenate(rows)


class StandIn:
    """numpy stand-ins for engine.hawkesjd_price_chain{,s}_batch that record their calls"""

    def __init__(self, monkeypatch, fail_on_call=None):
        self.calls, self.fail_on_call = [], fail_on_call
        for name in ("hawkesjd_price_chain_batch", "hawkesjd_price_chains_batch"):
            monkeypatch.setattr(engine, name, getattr(self, name))

    def _count(self, args, kw):
        self.calls.append((args, kw))
        if self.fail_on_call == len(self.calls):
            raise RuntimeError("library failure")

    def hawkesjd_price_chain_batch(self, *args, **kw):
        self._count(args, kw)
        params_list, ttms, forwards, _, strikes_ttms, _ = args
        return None, np.vstack([_vols(p, ttms, forwards, strikes_ttms) for p in params_list])

    def hawkesjd_price_chains_batch(self, params_list, chain_of_set, chains, vol_scalers=None, **kw):
        self._count((params_list, chain_of_set, chains), dict(kw, vol_scalers=vol_scalers))
        return None, [_vols(p, chains[k][0], chains[k][1], chains[k][3]) for p, k in zip(params_list, chain_of_set)]


def _chain(ttms, forward, truth, n_strikes, quoted=True):
    """a chain quoted at the stand-in's vols of ``truth``; without quotes (``quoted=False``) its fit fails before it prices anything"""
    strikes = [forward * np.linspace(0.8, 1.2, n_strikes) for _ in ttms]
    types = [np.where(k >= forward, "C", "P") for k in strikes]
    fw = np.full(len(ttms), forward)
    vols = np.split(_vols(truth, ttms, fw, strikes), len(ttms))
    return OptionChain(ttms=np.asarray(ttms), forwards=fw, discfactors=np.ones(len(ttms)), strikes_ttms=strikes, optiontypes_ttms=types,
                       bid_ivs=[v - 0.01 for v in vols] if quoted else None, ask_ivs=[v + 0.01 for v in vols] if quoted else None)


def _chains(fail_index=None):
    out = []
    for i, (s, mp) in enumerate(((0.4, 0.05), (0.6, 0.1), (0.5, 0.2), (0.45, 0.15))):
        truth = HawkesJDParams(sigma=s, mean_p=mp, theta_p=7.0 + i)
        out.append(_chain([0.1, 0.4, 1.0][: 1 + i % 3], 1.0 + 0.1 * i, truth, 5 + i, quoted=i != fail_index))
    return out


START = HawkesJDParams()


def _same_fit(a, b):
    (fa, ia), (fb, ib) = a, b
    for key in ("sigma", "mean_p", "mean_m", "theta_p", "theta_m", "kappa_p", "kappa_m", "beta1_p", "beta2_p", "beta1_m", "beta2_m"):
        assert getattr(fa, key) == getattr(fb, key), key
    for key in ("fun", "nit", "nb_batches", "nan_quotes", "x"):
        np.testing.assert_array_equal(ia[key], ib[key], err_msg=key)


def test_lockstep_fits_equal_single_chain_fits(monkeypatch):
    stand_in = StandIn(monkeypatch)
    chains = _chains()
    starts = [START, HawkesJDParams(sigma=0.5), HawkesJDParams(risk_premia_gamma=0.2), HawkesJDParams(kappa_p=25.0, kappa_m=25.0)]
    pricer = HawkesJDPricer()
    seq = [pricer.calibrate_model_params_to_chain(c, s, return_info=True, maxiter=20) for c, s in zip(chains, starts)]
    n_seq = len(stand_in.calls)
    before = threading.active_count()
    fits, infos = pricer.calibrate_model_params_to_chains(chains, starts, return_info=True, maxiter=20)
    assert threading.active_count() == before
    for a, f, i in zip(seq, fits, infos):
        _same_fit(a, (f, i))
    rounds = len(stand_in.calls) - n_seq
    assert all(i["rounds"] == rounds for i in infos) and rounds == max(i["nb_batches"] for _, i in seq)
    for args, kw in stand_in.calls[n_seq:]:
        assert kw == {"max_phi": 500, "vol_scalers": None}
    # max_sets_per_call splits the rounds, never a fit's sets, and the fits do not change
    stand_in.calls.clear()
    fits2, infos2 = pricer.calibrate_model_params_to_chains(chains, starts, return_info=True, maxiter=20, max_sets_per_call=9)
    for a, f, i in zip(seq, fits2, infos2):
        _same_fit(a, (f, i))
    assert infos2[0]["rounds"] == len(stand_in.calls) > rounds
    assert max(len(args[0]) for args, _ in stand_in.calls) <= 9


def test_single_chain_driver_calls_the_batch_as_before(monkeypatch):
    """one engine.hawkesjd_price_chain_batch call per batch of the fit, with the chain's own arrays, max_phi = 500 and no risk kernel"""
    stand_in = StandIn(monkeypatch)
    chain = _chains()[1]
    fit, info = HawkesJDPricer().calibrate_model_params_to_chain(chain, HawkesJDParams(risk_premia_gamma=0.3), return_info=True, maxiter=10)
    assert len(stand_in.calls) == info["nb_batches"] > 1
    for args, kw in stand_in.calls:
        assert kw == {"max_phi": 500, "gammas": None}
        assert len(args) == 6 and len(args[0]) in (1, 8)
        for got, want in zip(args[1:], (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)):
            assert got is want
    assert fit.risk_premia_gamma is None


def test_rejections_come_before_any_library_call(monkeypatch):
    stand_in = StandIn(monkeypatch)
    pricer, chains = HawkesJDPricer(), _chains()
    for gradient in ("exact", "pathwise"):
        with pytest.raises(NotImplementedError):
            pricer.calibrate_model_params_to_chains(chains, START, gradient=gradient)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, gradient="central")
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains([], START)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, [START] * 3)
    with pytest.raises(ValueError):
        pricer.calibrate_model_params_to_chains(chains, START, max_sets_per_call=0)
    assert stand_in.calls == []


def test_a_failing_fit_keeps_its_place_and_every_thread_ends(monkeypatch):
    StandIn(monkeypatch)
    pricer = HawkesJDPricer()
    ok = [pricer.calibrate_model_params_to_chain(c, START, return_info=True, maxiter=10) for c in _chains()]
    before = threading.active_count()
    fits, infos = pricer.calibrate_model_params_to_chains(_chains(fail_index=2), START, return_info=True, return_exceptions=True,
                                                          maxiter=10)
    assert threading.active_count() == before
    assert isinstance(fits[2], Exception) and infos[2] is None
    for k in (0, 1, 3):
        _same_fit(ok[k], (fits[k], infos[k]))
    with pytest.raises(Exception):
        pricer.calibrate_model_params_to_chains(_chains(fail_index=2), START, maxiter=10)
    assert threading.active_count() == before


def test_a_failing_library_call_reaches_every_fit_of_its_round(monkeypatch):
    StandIn(monkeypatch, fail_on_call=2)
    fits = HawkesJDPricer().calibrate_model_params_to_chains(_chains(), START, return_exceptions=True, maxiter=10)
    assert all(isinstance(f, RuntimeError) and str(f) == "library failure" for f in fits)


def _chains_call(chain_of_set, Ms, null=None):
    """b200sv_hawkesjd_price_chains_batch on chains of 3 strikes per maturity: every case below is rejected before any CUDA call"""
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    lib = C.load_library()
    B, K = len(chain_of_set), len(Ms)
    n = sum(max(m, 0) for m in Ms)
    ttms, fw, df = C.f64(np.tile([0.25, 0.5, 0.75], 4)[:max(n, 1)]), np.ones(max(n, 1)), np.ones(max(n, 1))
    offs = np.concatenate([np.arange(max(m, 0) + 1) * 3 for m in Ms]).astype(np.int32)
    strikes, types = C.f64(np.tile([0.9, 1.0, 1.1], 12)), np.tile(np.array([C.PUT, C.CALL, C.CALL], dtype=np.int8), 12)
    cos, ms, scalers = np.asarray(chain_of_set, dtype=np.int32), np.asarray(Ms, dtype=np.int32), np.full(K, -1.0)
    out = np.zeros(256)
    ps = (C.HawkesParamsC * max(B, 1))(*[_params_c(**HawkesJDParams().to_dict())] * max(B, 1))
    args = [ps, B, C.iptr(cos), K, C.iptr(ms), C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(offs), C.dptr(strikes), C.i8ptr(types), 1,
            C.dptr(scalers), 0, C.dptr(out), None]
    if null is not None:
        args[null] = None
    rc = lib.b200sv_hawkesjd_price_chains_batch(*args)
    return rc, lib.b200sv_last_error().decode()


def test_library_rejects_bad_chains_arguments_before_any_cuda_call():
    null = (-1, "invalid argument: null pointer")
    for i in (0, 2, 4, 5, 6, 7, 8, 9, 10, 12, 14):   # params, chain_of_set, Ms, ttms, forwards, discfactors, offsets, strikes, types,
        assert _chains_call([0, 1], [2, 1], null=i) == null, i      # vol_scalers, prices_out
    assert _chains_call([], [2, 1]) == (-1, "invalid argument: B >= 1, K >= 1")
    assert _chains_call([0, 2], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _chains_call([0, -1], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _chains_call([0, 0], [2, 0]) == (-1, "invalid argument: every chain needs M >= 1")
