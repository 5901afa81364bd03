"""CPU pins of the calibration drivers, bit for bit: every route that needs no GPU (LogSV ANALYTIC, Heston, the two Hawkes fits and the
lock-step drivers of all three models) run on numpy stand-ins for the library, with vega weights on slices of 9 to 36 quotes (where the
builtin ``sum`` of the LogSV / Heston weights and the ``np.sum`` of the Hawkes weights round differently).  Per case the golden file holds
the fitted fields, ``x``, ``fun``, ``nit``, ``nb_batches``, ``nan_quotes``, ``rounds``, a sha256 over every point handed to the stand-ins
(in call order, with the call's other arguments), one over the lines ``print_iter`` prints, and the type and message of any exception.

Run as a script to rewrite tests/golden/calibration_drivers.npz."""
import contextlib
import ctypes
import hashlib
import io
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

if __name__ == "__main__":                   # run as a script: the package and the stand-ins from this tree
    sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__))]

import test_calibration_chains_host as lsv                # noqa: E402  (LogSV / Heston stand-in and chains)
import test_hawkes_batch_host as hb                       # noqa: E402  (Hawkes stand-in and chain)
from stochvolmodels_b200 import (CalibrationEngine, ConstraintsType, HawkesJDParams, HawkesJDPricer, HestonParams,  # noqa: E402
                                 HestonPricer, LogSvParams, LogSVPricer, LogsvModelCalibrationType, engine)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "calibration_drivers.npz")
T = LogsvModelCalibrationType


def _feed(h, obj) -> None:
    """every byte of ``obj`` into the hash: ctypes parameter sets, arrays, numbers, strings, and containers of them"""
    if isinstance(obj, ctypes.Structure):
        h.update(type(obj).__name__.encode() + bytes(obj))
    elif isinstance(obj, np.ndarray):
        h.update(str(obj.dtype).encode() + str(obj.shape).encode() + np.ascontiguousarray(obj).tobytes())
    elif isinstance(obj, dict):
        for k in sorted(obj):
            _feed(h, k)
            _feed(h, obj[k])
    elif isinstance(obj, (list, tuple)):
        h.update(f"[{len(obj)}".encode())
        for v in obj:
            _feed(h, v)
    else:
        h.update(repr(obj).encode())


class Recorder:
    """the library stand-ins of every driver, each call hashed with all its arguments before it is answered"""

    def __init__(self, monkeypatch):
        self.sha = hashlib.sha256()
        chains = lsv.StandIn(monkeypatch)              # engine.{logsv,heston}_price_chain{,s}_batch
        self.hawkes = hb.StandIn(36)
        for name in ("logsv_price_chain_batch", "heston_price_chain_batch", "logsv_price_chains_batch", "heston_price_chains_batch"):
            monkeypatch.setattr(engine, name, self._hashed(name, getattr(chains, name)))
        monkeypatch.setattr(engine, "hawkesjd_price_chain_batch", self._hashed("hawkesjd_price_chain_batch", self.hawkes.batch))
        monkeypatch.setattr(engine, "hawkesjd_price_chains_batch", self._hashed("hawkesjd_price_chains_batch", self._hawkes_chains))
        for cls, names in ((LogSVPricer, engine.LOGSV_GREEK_PARAMS), (HestonPricer, engine.HESTON_GREEK_PARAMS),
                           (HawkesJDPricer, engine.HAWKES_GREEK_PARAMS)):
            monkeypatch.setattr(cls, "compute_chain_ivol_greeks", self._ivol_greeks(cls.__name__, names))

    def _hashed(self, name, fn):
        def call(*args, **kw):
            _feed(self.sha, (name, args, kw))
            return fn(*args, **kw)
        return call

    def _hawkes_chains(self, params_list, chain_of_set, chains, vol_scalers=None, max_phi=500):
        return None, [self.hawkes.vols({k: getattr(p, k) for k in hb._FIELDS}, None) for p in params_list]

    def _ivol_greeks(self, name, names):
        """compute_chain_ivol_greeks: vols = 0.4 + A tanh(s * fields - 1) per quote, with their exact derivatives in the fields"""
        def call(pricer, option_chain, params, **kw):
            fields = np.array([float(getattr(params, n)) for n in names])
            _feed(self.sha, (name, fields, kw))
            J = sum(len(k) for k in option_chain.strikes_ttms)
            rng = np.random.RandomState(len(names) * 100 + J)
            A, s = rng.uniform(-0.1, 0.1, (J, len(names))), 1.0 / rng.uniform(1.0, 60.0, len(names))
            t = np.tanh(s * fields - 1.0)
            vols, rows = 0.4 + A @ t, (A * ((1.0 - t * t) * s)).T
            split = lambda v: np.split(v, np.cumsum([len(k) for k in option_chain.strikes_ttms])[:-1])
            return SimpleNamespace(ivols=split(vols), params={n: split(r) for n, r in zip(names, rows)})
        return call


def _quoted(shape_chain, vols):
    """``shape_chain``'s strikes quoted at ``vols`` +- 0.001"""
    parts = np.split(vols, np.cumsum([len(k) for k in shape_chain.strikes_ttms])[:-1])
    return lsv.OptionChain(ttms=shape_chain.ttms, forwards=shape_chain.forwards, strikes_ttms=shape_chain.strikes_ttms,
                           optiontypes_ttms=shape_chain.optiontypes_ttms, ids=shape_chain.ids, bid_ivs=[v - 0.001 for v in parts],
                           ask_ivs=[v + 0.001 for v in parts])


# ---- the chains ------------------------------------------------------------------------------------------------------------------
LSV_SHAPES = [([0.05, 0.2, 0.5], 100.0, 9), ([0.1, 0.25, 0.5, 1.0], 2.0, 12), ([0.02, 0.3], 0.5, 21)]
HESTON_SHAPES = [([0.1, 0.5], 1.0, 8), ([0.05, 0.2, 0.5], 100.0, 13), ([0.1, 0.25, 0.5, 1.0], 2.0, 40)]
LSV_START = LogSvParams(sigma0=0.9, theta=0.9, kappa1=3.0, kappa2=3.0, beta=0.0, volvol=1.0)
HESTON_START = HestonParams(v0=0.35, theta=0.35, kappa=2.5, rho=-0.1, volvol=0.7)
HAWKES_START = HawkesJDParams(sigma=0.45, mean_p=0.03, mean_m=-0.04, theta_p=7.0, theta_m=7.0, kappa_p=22.0, kappa_m=28.0, beta1_p=33.0,
                              beta2_p=-33.0, beta1_m=36.0, beta2_m=-36.0)


def _logsv_chains(fail_index=None):
    out = []
    for i, (ttms, fw, n) in enumerate(LSV_SHAPES):
        truth = LogSvParams(sigma0=0.8 + 0.05 * i, theta=1.0, kappa1=3.0, kappa2=3.0, beta=0.2 - 0.1 * i, volvol=1.2 + 0.1 * i)
        out.append(lsv._chain(ttms, lsv.FAIL_FORWARD if i == fail_index else fw,
                              lambda t, f, k, p=truth: lsv._logsv_vols(p, t, f, np.ones(len(t)), k, False), n))
    return out


def _heston_chains(fail_index=None):
    out = []
    for i, (ttms, fw, n) in enumerate(HESTON_SHAPES):
        truth = HestonParams(v0=0.3 + 0.05 * i, theta=0.4, kappa=2.0 + i, rho=-0.3 + 0.1 * i, volvol=0.8)
        out.append(lsv._chain(ttms, lsv.FAIL_FORWARD if i == fail_index else fw, lambda t, f, k, p=truth: lsv._heston_vols(p, t, f, k, False), n))
    return out


def _hawkes_chains(recorder, fail_index=None):
    out = []
    for i in range(3):
        truth = HawkesJDParams(sigma=0.4 + 0.02 * i, mean_p=0.04, mean_m=-0.05, theta_p=6.0 + i, theta_m=8.0, kappa_p=25.0, kappa_m=25.0,
                               beta1_p=30.0, beta2_p=-30.0, beta1_m=40.0 - i, beta2_m=-40.0 + i)
        chain = hb._market(recorder.hawkes, truth)
        if i == fail_index:
            chain.bid_ivs = chain.ask_ivs = None          # no quotes: the fit fails before it prices anything
        out.append(chain)
    return out


def _exact_chain(pricer, params, chain):
    """``chain`` quoted at the ivol-greeks stand-in's vols of ``params``"""
    return _quoted(chain, np.concatenate(pricer.compute_chain_ivol_greeks(chain, params).ivols))


# ---- the cases -------------------------------------------------------------------------------------------------------------------
def _fields(fit) -> np.ndarray:
    if isinstance(fit, LogSvParams):
        return np.array([fit.sigma0, fit.theta, fit.kappa1, fit.kappa2, fit.beta, fit.volvol])
    if isinstance(fit, HestonParams):
        return np.array([fit.v0, fit.theta, fit.kappa, fit.rho, fit.volvol])
    d = fit.to_dict()
    return np.array([np.nan if d[k] is None else d[k] for k in sorted(d)], dtype=float)


def _record(out: dict, case: str, run) -> None:
    """run ``case`` and file what it returned (one fit, or the fits of a lock-step run) or raised"""
    rec = out["recorder"]
    rec.sha = hashlib.sha256()
    printed = io.StringIO()
    try:
        with contextlib.redirect_stdout(printed):
            res = run()
    except Exception as exc:                      # noqa: BLE001 (pinned with its message)
        res = exc
    row = {"points_sha256": rec.sha.hexdigest(), "printed_sha256": hashlib.sha256(printed.getvalue().encode()).hexdigest()}
    fits, infos = (res if isinstance(res, tuple) and isinstance(res[0], list) else
                   ([res[0]], [res[1]]) if isinstance(res, tuple) else ([res], [None]))
    for k, (fit, info) in enumerate(zip(fits, infos)):
        if isinstance(fit, BaseException):
            row[f"{k}/error"] = f"{type(fit).__name__}: {fit}"
            continue
        row[f"{k}/fields"] = _fields(fit)
        if isinstance(fit, LogSvParams) and fit.vol_backbone is not None:
            row[f"{k}/backbone"] = np.stack([np.asarray(fit.vol_backbone.index, dtype=float), np.asarray(fit.vol_backbone, dtype=float)])
        for key in ("x", "fun", "nit", "nb_batches", "nan_quotes", "rounds"):
            if info is not None and key in info:
                row[f"{k}/{key}"] = np.asarray(info[key])
        row[f"{k}/info_keys"] = np.array(",".join(info) if info is not None else "")
    for key, v in row.items():
        out[f"{case}/{key}"] = np.asarray(v)


def _cases(recorder):
    logsv, heston, hawkes = LogSVPricer(), HestonPricer(), HawkesJDPricer()
    lchains, hchains, kchains = _logsv_chains(), _heston_chains(), _hawkes_chains(recorder)
    lsv_exact = _exact_chain(logsv, LogSvParams(sigma0=0.8, theta=1.0, kappa1=3.0, kappa2=3.0, beta=0.2, volvol=1.2), lchains[1])
    heston_exact = _exact_chain(heston, HestonParams(v0=0.3, theta=0.4, kappa=2.0, rho=-0.3, volvol=0.8), hchains[1])
    hawkes_exact = _exact_chain(hawkes, HawkesJDParams(sigma=0.4, mean_p=0.04, mean_m=-0.05, theta_p=6.0, theta_m=8.0, kappa_p=25.0,
                                                       kappa_m=25.0, beta1_p=30.0, beta2_p=-30.0, beta1_m=40.0, beta2_m=-40.0), kchains[0])
    cases = {}
    for ctype in (T.PARAMS4, T.PARAMS5, T.PARAMS_WITH_VARSWAP_FIT):
        for cons in (ConstraintsType.UNCONSTRAINT, ConstraintsType.MMA_MARTINGALE):
            kw = dict(model_calibration_type=ctype, constraints_type=cons, return_info=True)
            cases[f"logsv/{ctype.name}/{cons.name}/difference"] = lambda kw=kw: logsv.calibrate_model_params_to_chain(lchains[1], LSV_START, **kw)
            cases[f"logsv/{ctype.name}/{cons.name}/exact"] = lambda kw=kw: logsv.calibrate_model_params_to_chain(lsv_exact, LSV_START,
                                                                                                                gradient="exact", **kw)
    cases["logsv/PARAMS5/unit_ttm_vega"] = lambda: logsv.calibrate_model_params_to_chain(lchains[2], LSV_START, is_unit_ttm_vega=True,
                                                                                        return_info=True)
    cases["logsv/PARAMS4/unweighted"] = lambda: logsv.calibrate_model_params_to_chain(lchains[0], LSV_START, is_vega_weighted=False,
                                                                                     model_calibration_type=T.PARAMS4, return_info=True)
    for gradient, chain in (("difference", hchains[2]), ("exact", heston_exact)):
        cases[f"heston/{gradient}"] = lambda g=gradient, c=chain: heston.calibrate_model_params_to_chain(c, HESTON_START, gradient=g,
                                                                                                        return_info=True)
    cases["heston/default_start"] = lambda: heston.calibrate_model_params_to_chain(hchains[0], return_info=True)
    for gradient, chain in (("difference", kchains[1]), ("exact", hawkes_exact)):
        cases[f"hawkes/model/{gradient}"] = lambda g=gradient, c=chain: hawkes.calibrate_model_params_to_chain(c, HAWKES_START, gradient=g,
                                                                                                              maxiter=30, return_info=True)
    gamma_chain = hb._market(recorder.hawkes, HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5))
    for print_iter in (True, False):
        cases[f"hawkes/risk_premia/print_iter={print_iter}"] = lambda p=print_iter: hawkes.calibrate_risk_premia_gamma_to_chain(
            gamma_chain, HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2), print_iter=p, return_info=True)
    cases["hawkes/risk_premia/exact"] = lambda: hawkes.calibrate_risk_premia_gamma_to_chain(gamma_chain, HawkesJDParams(), gradient="exact",
                                                                                           print_iter=False)
    for cap in (None, 7):
        kw = dict(return_info=True, max_sets_per_call=cap)
        cases[f"lockstep/logsv/cap={cap}"] = lambda kw=kw: logsv.calibrate_model_params_to_chains(
            lchains, LSV_START, constraints_type=ConstraintsType.MMA_MARTINGALE, **kw)
        cases[f"lockstep/heston/cap={cap}"] = lambda kw=kw: heston.calibrate_model_params_to_chains(hchains, HESTON_START, **kw)
        cases[f"lockstep/hawkes/cap={cap}"] = lambda kw=kw: hawkes.calibrate_model_params_to_chains(kchains, HAWKES_START, maxiter=20, **kw)
    cases["lockstep/logsv/varswap"] = lambda: logsv.calibrate_model_params_to_chains(
        lchains[:2], [LSV_START, LSV_START], params_max=[None, LogSvParams(sigma0=1.2, theta=1.5, kappa1=8.0, kappa2=8.0, beta=2.0, volvol=2.5)],
        model_calibration_type=T.PARAMS_WITH_VARSWAP_FIT, return_info=True)
    kw = dict(return_info=True, return_exceptions=True)
    cases["lockstep/logsv/failing"] = lambda: logsv.calibrate_model_params_to_chains(_logsv_chains(fail_index=1), LSV_START, **kw)
    cases["lockstep/heston/failing"] = lambda: heston.calibrate_model_params_to_chains(_heston_chains(fail_index=0), HESTON_START, **kw)
    cases["lockstep/hawkes/failing"] = lambda: hawkes.calibrate_model_params_to_chains(_hawkes_chains(recorder, fail_index=2), HAWKES_START,
                                                                                        maxiter=10, **kw)
    cases["lockstep/logsv/raises"] = lambda: logsv.calibrate_model_params_to_chains(_logsv_chains(fail_index=0), LSV_START)
    return cases


def fingerprint(monkeypatch) -> dict:
    out = {"recorder": Recorder(monkeypatch)}
    for case, run in _cases(out["recorder"]).items():
        _record(out, case, run)
    del out["recorder"]
    return out


def test_calibration_drivers_match_the_golden_file(monkeypatch):
    got = fingerprint(monkeypatch)
    with np.load(GOLDEN) as g:
        want = {k: g[k] for k in g.files}
    assert sorted(got) == sorted(want)
    for key in want:
        np.testing.assert_array_equal(got[key], want[key], err_msg=key)
        assert got[key].dtype == want[key].dtype, key


def test_the_golden_file_pins_the_weight_reductions_apart():
    """slices of 8 or more quotes, on which ``v / sum(v)`` and ``v / np.sum(v)`` differ in some last bit: both reductions are exercised"""
    chains = _logsv_chains() + _heston_chains()
    differ = [np.any(v / sum(v) != v / np.sum(v)) for c in chains for v in c.get_chain_vegas()]
    assert min(len(k) for c in chains for k in c.strikes_ttms) >= 8 and any(differ)
    vegas = hb._chain().get_chain_vegas()
    assert min(len(v) for v in vegas) >= 8


if __name__ == "__main__":
    with pytest.MonkeyPatch.context() as mp:
        np.savez_compressed(GOLDEN, **fingerprint(mp))
    print(f"wrote {GOLDEN}")
