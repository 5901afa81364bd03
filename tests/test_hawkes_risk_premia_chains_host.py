"""CPU tests of HawkesJDPricer.calibrate_risk_premia_gamma_to_chains: its rejections, the lock-step coordinator on the numpy stand-in of
test_hawkes_batch_host (which prices every row from its own set and gamma only, as the library does, so lock-step fits must equal the
single-chain fits bit for bit), the printed lines, and the argument checks of b200sv_hawkesjd_price_chains_batch_gamma and its engine
wrapper."""
import math
import threading

import numpy as np
import pytest

import test_hawkes_batch_host as hb
from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine
from stochvolmodels_b200 import _capi as C


class Recorder:
    """test_hawkes_batch_host.StandIn behind both batched pricers, recording the multi-chain calls"""

    def __init__(self, monkeypatch, fail_on_call=None):
        self.stand_in = hb.StandIn(36)
        self.calls, self.fail_on_call = [], fail_on_call
        monkeypatch.setattr(engine, "hawkesjd_price_chain_batch", self.stand_in.batch)
        monkeypatch.setattr(engine, "hawkesjd_price_chains_batch", self.chains)

    def chains(self, params_list, chain_of_set, chains, vol_scalers=None, **kw):
        self.calls.append((list(params_list), list(chain_of_set), chains, dict(kw, vol_scalers=vol_scalers)))
        if self.fail_on_call == len(self.calls):
            raise RuntimeError("library failure")
        gammas = kw["gammas"]
        return None, [self.stand_in.vols({k: getattr(p, k) for k in hb._FIELDS}, gammas[b]) for b, p in enumerate(params_list)]


TRUTHS = [HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5), HawkesJDParams(sigma=0.35, risk_premia_gamma=-0.8),
          HawkesJDParams(sigma=0.5, risk_premia_gamma=1.5), HawkesJDParams(sigma=0.3, risk_premia_gamma=-2.0),
          HawkesJDParams(sigma=0.6, risk_premia_gamma=0.1)]
STARTS = [HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2), HawkesJDParams(sigma=0.4), HawkesJDParams(sigma=0.5, risk_premia_gamma=-0.3),
          HawkesJDParams(sigma=0.3, risk_premia_gamma=1.0, kappa_p=25.0), HawkesJDParams(sigma=0.55, risk_premia_gamma=-1.0, lambda_m=9.0)]


def _markets(recorder, K, fail_index=None):
    out = [hb._market(recorder.stand_in, t) for t in TRUTHS[:K]]
    if fail_index is not None:               # no quotes: its fit fails before it prices anything
        c = out[fail_index]
        out[fail_index] = OptionChain(ttms=c.ttms, forwards=c.forwards, strikes_ttms=c.strikes_ttms, optiontypes_ttms=c.optiontypes_ttms)
    return out


def _same_fit(a, b):
    (fa, ia), (fb, ib) = a, b
    assert fa == fb
    for key in ("fun", "nit", "nb_batches", "nan_quotes", "x"):
        np.testing.assert_array_equal(ia[key], ib[key], err_msg=key)


@pytest.mark.parametrize("K", [1, 3, 5])
@pytest.mark.parametrize("max_sets_per_call", [None, 1, 2])
def test_lockstep_fits_equal_single_chain_fits(monkeypatch, K, max_sets_per_call):
    rec = Recorder(monkeypatch)
    pricer = HawkesJDPricer()
    chains, starts = _markets(rec, K), STARTS[:K]
    seq = [pricer.calibrate_risk_premia_gamma_to_chain(c, s, print_iter=False, return_info=True) for c, s in zip(chains, starts)]
    assert all(i["nit"] > 2 for _, i in seq)
    before = threading.active_count()
    fits, infos = pricer.calibrate_risk_premia_gamma_to_chains(chains, starts, return_info=True, max_sets_per_call=max_sets_per_call)
    assert threading.active_count() == before
    for a, f, i in zip(seq, fits, infos):
        _same_fit(a, (f, i))
    assert all(i["rounds"] == len(rec.calls) for i in infos)
    if max_sets_per_call is None:
        assert len(rec.calls) == max(i["nb_batches"] for _, i in seq)
    else:
        assert max(len(params) for params, _, _, _ in rec.calls) <= max(max_sets_per_call, 2)     # a fit's sets are never split
    for params, cos, chs, kw in rec.calls:
        assert kw["max_phi"] == 500 and kw["vol_scalers"] is None and len(kw["gammas"]) == len(params)
        assert list(cos) == sorted(cos) and len(chs) == len(set(cos))


def test_a_none_gamma_starts_at_zero(monkeypatch):
    rec = Recorder(monkeypatch)
    chains = _markets(rec, 2)
    starts = [HawkesJDParams(sigma=0.4), HawkesJDParams(sigma=0.4, risk_premia_gamma=0.0)]
    fits, infos = HawkesJDPricer().calibrate_risk_premia_gamma_to_chains(chains, starts, return_info=True)
    first = rec.calls[0]
    assert first[3]["gammas"] == [0.0, 0.0]
    ones = HawkesJDPricer().calibrate_risk_premia_gamma_to_chains(chains, starts[1], return_info=True)    # one start for every chain
    for a, b, c in zip(zip(fits, infos), *ones):
        _same_fit(a, (b, c))


def test_print_iter_prints_each_chains_lines_as_one_block_in_chain_order(monkeypatch, capsys):
    rec = Recorder(monkeypatch)
    pricer = HawkesJDPricer()
    chains = _markets(rec, 3)
    expected = []
    for c, s in zip(chains, STARTS):
        pricer.calibrate_risk_premia_gamma_to_chain(c, s, print_iter=True)
        expected.append(capsys.readouterr().out)
    assert all(e.count("\n") > 3 for e in expected)
    pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[:3], print_iter=True)
    assert capsys.readouterr().out == "".join(expected)
    pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[:3])
    assert capsys.readouterr().out == ""


def test_a_failing_fit_keeps_its_place(monkeypatch, capsys):
    rec = Recorder(monkeypatch)
    pricer = HawkesJDPricer()
    ok, printed = [], []
    for c, s in zip(_markets(rec, 4), STARTS):
        ok.append(pricer.calibrate_risk_premia_gamma_to_chain(c, s, print_iter=True, return_info=True))
        printed.append(capsys.readouterr().out)
    before = threading.active_count()
    fits, infos = pricer.calibrate_risk_premia_gamma_to_chains(_markets(rec, 4, fail_index=1), STARTS[:4], print_iter=True, return_info=True,
                                                               return_exceptions=True)
    assert threading.active_count() == before
    assert isinstance(fits[1], Exception) and infos[1] is None
    for k in (0, 2, 3):
        _same_fit(ok[k], (fits[k], infos[k]))
    assert capsys.readouterr().out == printed[0] + printed[2] + printed[3]      # the failed fit ends before its first point
    with pytest.raises(Exception):
        pricer.calibrate_risk_premia_gamma_to_chains(_markets(rec, 4, fail_index=1), STARTS[:4])
    assert threading.active_count() == before


def test_a_failing_library_call_reaches_every_fit_of_its_round(monkeypatch):
    rec = Recorder(monkeypatch, fail_on_call=2)
    fits = HawkesJDPricer().calibrate_risk_premia_gamma_to_chains(_markets(rec, 3), STARTS[:3], return_exceptions=True)
    assert all(isinstance(f, RuntimeError) and str(f) == "library failure" for f in fits)


def test_rejections_come_before_any_library_call(monkeypatch):
    rec = Recorder(monkeypatch)
    pricer, chains = HawkesJDPricer(), _markets(rec, 3)
    rec.stand_in.calls = 0
    for gradient in ("exact", "pathwise"):
        with pytest.raises(NotImplementedError, match="calibrate_risk_premia_gamma_to_chains"):
            pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[0], gradient=gradient)
    with pytest.raises(ValueError):
        pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[0], gradient="central")
    with pytest.raises(ValueError):
        pricer.calibrate_risk_premia_gamma_to_chains([], STARTS[0])
    with pytest.raises(ValueError):
        pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[:2])
    with pytest.raises(ValueError):
        pricer.calibrate_risk_premia_gamma_to_chains(chains, STARTS[0], max_sets_per_call=0)
    assert rec.calls == [] and rec.stand_in.calls == 0
    with pytest.raises(NotImplementedError, match="calibrate_model_params_to_chains has gradient"):    # the model-parameter text stays
        pricer.calibrate_model_params_to_chains(chains, STARTS[0], gradient="exact")


# ---- b200sv_hawkesjd_price_chains_batch_gamma: every case below is rejected before any CUDA call ----------------------------------------
NULL = (-1, "invalid argument: null pointer")
GAMMAS = (-1, "invalid argument: gammas must be finite (NULL: no risk kernel)")
NOT_IMPL = (-5, "not implemented")


def _gamma_call(chain_of_set, Ms, gammas=None, null=None, spot=1, types=None):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    lib = C.load_library()
    B, K = len(chain_of_set), len(Ms)
    n = sum(max(m, 0) for m in Ms)
    ttms, fw, df = C.f64(np.tile([0.25, 0.5, 0.75], 4)[:max(n, 1)]), np.ones(max(n, 1)), np.ones(max(n, 1))
    offs = np.concatenate([np.arange(max(m, 0) + 1) * 3 for m in Ms] or [np.zeros(1)]).astype(np.int32)
    strikes = C.f64(np.tile([0.9, 1.0, 1.1], 12))
    types = np.tile(np.array(types or [C.PUT, C.CALL, C.CALL], dtype=np.int8), 12)
    cos, ms, scalers = np.asarray(chain_of_set, dtype=np.int32), np.asarray(Ms, dtype=np.int32), np.full(K, -1.0)
    g = C.f64(gammas if gammas is not None else [0.1] * max(B, 1))
    out = np.zeros(256)
    ps = (C.HawkesParamsC * max(B, 1))(*[_params_c(**HawkesJDParams().to_dict())] * max(B, 1))
    args = [ps, C.dptr(g), B, C.iptr(cos), K, C.iptr(ms), C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(offs), C.dptr(strikes), C.i8ptr(types),
            spot, C.dptr(scalers), 0, C.dptr(out), None]
    if null is not None:
        args[null] = None
    rc = lib.b200sv_hawkesjd_price_chains_batch_gamma(*args)
    return rc, lib.b200sv_last_error().decode()


def test_library_rejects_bad_gamma_chains_arguments_before_any_cuda_call():
    # params, gammas, chain_of_set, Ms, ttms, forwards, discfactors, offsets, strikes, types, vol_scalers, prices_out
    for i in (0, 1, 3, 5, 6, 7, 8, 9, 10, 11, 13, 15):
        assert _gamma_call([0, 1], [2, 1], null=i) == NULL, i
    assert _gamma_call([], [2, 1]) == (-1, "invalid argument: B >= 1, K >= 1")
    assert _gamma_call([0, 1], []) == (-1, "invalid argument: B >= 1, K >= 1")
    assert _gamma_call([0, 2], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _gamma_call([0, -1], [2, 1]) == (-1, "invalid argument: chain_of_set out of range")
    assert _gamma_call([0, 0], [2, 0]) == (-1, "invalid argument: every chain needs M >= 1")
    for bad in (math.nan, math.inf, -math.inf):
        assert _gamma_call([0, 1, 1], [2, 1], gammas=[0.1, 0.2, bad]) == GAMMAS, bad
    assert _gamma_call([0, 1], [2, 1], spot=0) == NOT_IMPL                                   # the risk kernel: spot measure only
    assert _gamma_call([0, 1], [2, 1], types=[C.PUT, C.INV_CALL, C.CALL]) == NOT_IMPL       # ... and 'C' / 'P' only


def test_engine_wrapper_checks_gammas_first():
    kp = hb.KP
    chain = (np.array([0.25]), np.ones(1), np.ones(1), [np.array([1.0])], [np.array(["C"])])
    inverse = chain[:4] + ([np.array(["IC"])],)
    with pytest.raises(ValueError, match="not implemented"):
        engine.hawkesjd_price_chains_batch([kp], [1], [chain, inverse], gammas=[0.2])
    with pytest.raises(ValueError, match="not implemented"):
        engine.hawkesjd_price_chains_batch([kp], [0], [chain], is_spot_measure=False, gammas=[0.2])
    with pytest.raises(ValueError, match="gammas must have shape"):
        engine.hawkesjd_price_chains_batch([kp, kp], [0, 0], [chain], gammas=[0.2])
