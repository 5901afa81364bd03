"""CPU: what ``gradient='pathwise'`` of the calibration drivers rejects before any library call, and the implied-vol transform of Monte
Carlo sensitivities (DESIGN.md §4.7)."""
import numpy as np
import pytest


@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def refuse(*args, **kwargs):
        raise AssertionError("library call")
    monkeypatch.setattr(_capi, "call", refuse)
    monkeypatch.setattr(_capi, "load_library", refuse)


def _chain():
    from stochvolmodels_b200 import get_btc_test_chain_data
    return get_btc_test_chain_data()


def test_pathwise_rejections_before_any_library_call(no_library):
    from stochvolmodels_b200 import (CalibrationEngine, HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer,
                                     LogsvModelCalibrationType)
    chain, start = _chain(), LogSvParams(0.8, 1.0, 3.0, 3.0, 0.1, 1.8)
    logsv = LogSVPricer().calibrate_model_params_to_chain
    with pytest.raises(NotImplementedError, match="MC and ROUGH_MC.*gradient='exact'"):
        logsv(chain, start, calibration_engine=CalibrationEngine.ANALYTIC, gradient="pathwise")
    for engine_kind in (CalibrationEngine.MC, CalibrationEngine.ROUGH_MC):
        for ctype in (LogsvModelCalibrationType.PARAMS6, LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT):
            with pytest.raises(NotImplementedError, match="pathwise.*PARAMS4 and PARAMS5"):
                logsv(chain, start, calibration_engine=engine_kind, model_calibration_type=ctype, gradient="pathwise")
    for call in (lambda: HestonPricer().calibrate_model_params_to_chain(chain, HestonParams(), gradient="pathwise"),
                 lambda: HawkesJDPricer().calibrate_model_params_to_chain(chain, HawkesJDParams(), gradient="pathwise"),
                 lambda: HawkesJDPricer().calibrate_risk_premia_gamma_to_chain(chain, HawkesJDParams(risk_premia_gamma=0.1), gradient="pathwise",
                                                                                print_iter=False)):
        with pytest.raises(NotImplementedError, match="pathwise.*CalibrationEngine.MC or ROUGH_MC"):
            call()
    with pytest.raises(ValueError, match="gradient must be 'difference', 'exact' or 'pathwise'"):
        logsv(chain, start, calibration_engine=CalibrationEngine.MC, gradient="path-wise")


def test_mc_sensitivities_map_to_ivol_rows_through_a_zero_gamma_row(monkeypatch):
    """to_chain_ivol_sensitivities(McChainGreeks without gamma): the transform receives delta, a zero gamma row, then the parameter rows in
    LOGSV_GREEK_PARAMS order, and the result carries gamma=None"""
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.fourier_greeks import ChainIvolGreeks, to_chain_ivol_sensitivities
    from stochvolmodels_b200.pricers.mc_greeks import McChainGreeks
    chain = _chain()
    sizes = [len(k) for k in chain.strikes_ttms]
    J = sum(sizes)
    split = lambda row: np.split(row, np.cumsum(sizes)[:-1])
    names = engine.LOGSV_GREEK_PARAMS
    rows = {n: 10.0 * (1 + k) + np.arange(J) / J for k, n in enumerate(("delta",) + names)}
    greeks = McChainGreeks(prices=split(np.linspace(0.01, 0.2, J)), std_errors=split(np.ones(J)), delta=split(rows["delta"]),
                           delta_se=split(np.ones(J)), params={n: split(rows[n]) for n in names}, params_se={n: split(np.ones(J)) for n in names})
    seen = {}

    def recorder(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms, g, vanna=None, hessian=None):
        seen.update(prices=np.concatenate(prices_ttms), rows=np.array(g), vanna=vanna, hessian=hessian)
        return split(np.full(J, 0.5)), -np.array(g), None, None

    monkeypatch.setattr(engine, "bsm_implied_vol_sensitivities", recorder)
    out = to_chain_ivol_sensitivities(chain, greeks)
    want = np.vstack([rows["delta"], np.zeros(J)] + [rows[n] for n in names])
    np.testing.assert_array_equal(seen["rows"], want)
    np.testing.assert_array_equal(seen["prices"], np.concatenate(greeks.prices))
    assert seen["vanna"] is None and seen["hessian"] is None
    assert isinstance(out, ChainIvolGreeks) and out.gamma is None
    np.testing.assert_array_equal(np.concatenate(out.delta), -rows["delta"])
    for n in names:
        np.testing.assert_array_equal(np.concatenate(out.params[n]), -rows[n])
    assert list(out.params) == list(names)
