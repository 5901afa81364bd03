"""CPU: the forward-mode oracle of the pathwise Monte Carlo sensitivities (oracle/mc_greeks.py) against central finite differences of the
oracle steppers and chain pricers on fixed normals, and the argument checks of model_mc_chain_greeks (they raise before any library call)."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import mc, mc_greeks as mg

LOGSV_P = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)           # BTC parameters
HESTON_FLOOR_P = tuple(load_golden("heston_mc_fixed_floor.npz")["params"])
BUMP = 1e-6


def _normals(seed, S, N):
    rs = np.random.RandomState(seed)
    return rs.normal(size=(S, N)), rs.normal(size=(S, N))


def _bumped(params, k, h):
    p = list(params)
    p[k] += h
    return tuple(p)


def _step(h):
    return BUMP * max(abs(h), 1e-2)


def _assert_close(a, b, what, rtol=1e-6):
    """relative to the tangent array's scale (a tangent that vanishes on most paths is compared at the scale it has elsewhere)"""
    scale = max(float(np.max(np.abs(b))), 1e-300)
    assert np.max(np.abs(a - b)) <= rtol * scale, (what, np.max(np.abs(a - b)) / scale)


@pytest.mark.parametrize("is_spot,eta", [(True, 1.0), (False, 0.8), (True, 1.3)])
def test_logsv_tangents_match_central_differences(is_spot, eta):
    N = 400
    x = np.zeros(N)
    for S, dt, seed in ((12, 0.1 / 12, 1), (30, 0.5 / 30, 2)):            # several steps, two maturities
        Z0, Z1 = _normals(seed, S, N)
        s0 = LOGSV_P[0] * np.ones(N)
        d0 = np.zeros((6, N))
        d0[0] = 1.0
        xs, ss, qs, dx, ds, dq = mg.logsv_tangent_step_fixed(x, s0, x, 0 * d0, d0, 0 * d0, Z0, Z1, dt, *LOGSV_P[1:], eta, is_spot)
        ref = mc.logsv_step_fixed(x, s0, x, Z0, Z1, dt, *LOGSV_P[1:], eta, is_spot)
        for a, b in zip((xs, ss, qs), ref):
            np.testing.assert_array_equal(a, b)                            # the tangent restatement does not touch the state
        for k, name in enumerate(mg.LOGSV_PARAMS):
            h = _step(LOGSV_P[k])
            up, dn = _bumped(LOGSV_P, k, h), _bumped(LOGSV_P, k, -h)
            ru = mc.logsv_step_fixed(x, up[0] * np.ones(N), x, Z0, Z1, dt, *up[1:], eta, is_spot)
            rd = mc.logsv_step_fixed(x, dn[0] * np.ones(N), x, Z0, Z1, dt, *dn[1:], eta, is_spot)
            for t, a, b, var in zip((dx, ds, dq), ru, rd, ("x", "sigma", "q")):
                _assert_close(t[k], (a - b) / (2 * h), (name, var, S))


def test_heston_tangents_match_central_differences_floor_binds():
    N = 400
    x = np.zeros(N)
    for S, dt, seed in ((20, 0.1 / 20, 3), (60, 0.5 / 60, 4)):
        Z0, Z1 = _normals(seed, S, N)
        v0 = HESTON_FLOOR_P[0] * np.ones(N)
        d0 = np.zeros((5, N))
        d0[0] = 1.0
        xs, vs, qs, dx, dv, dq = mg.heston_tangent_step_fixed(x, v0, x, 0 * d0, d0, 0 * d0, Z0, Z1, dt, *HESTON_FLOOR_P[1:])
        assert np.any(vs == 1e-4), "the floor must bind on some paths"
        for k, name in enumerate(mg.HESTON_PARAMS):
            h = _step(HESTON_FLOOR_P[k])
            up, dn = _bumped(HESTON_FLOOR_P, k, h), _bumped(HESTON_FLOOR_P, k, -h)
            ru = mc.heston_step_fixed(x, up[0] * np.ones(N), x, Z0, Z1, dt, *up[1:])
            rd = mc.heston_step_fixed(x, dn[0] * np.ones(N), x, Z0, Z1, dt, *dn[1:])
            for t, a, b, var in zip((dx, dv, dq), ru, rd, ("x", "v", "q")):
                _assert_close(t[k], (a - b) / (2 * h), (name, var, S))


K4 = np.array([0.85, 0.95, 1.05, 1.15])
TYPES = [np.array(["C", "P", "IC", "IP"]), np.array(["IP", "C", "P", "IC"])]
QK = np.array([0.3, 0.5, 0.7, 0.9])


def _chain_case(variable_type):
    ttms, fw, df = np.array([0.1, 0.3]), np.array([1.0, 1.02]), np.array([0.999, 0.99])
    strikes = [QK, QK] if variable_type == mc.Q_VAR else [K4, K4 * 1.02]
    return ttms, fw, df, strikes


def _fd_gate(g, se, fd, what):
    """pathwise vs CRN central difference within 0.1 of the sensitivity's standard error (plus fp64 round-off of the difference)"""
    assert np.all(np.abs(g - fd) <= 0.1 * se + 1e-9 * (1.0 + np.abs(g))), (what, g, fd, se)


@pytest.mark.parametrize("variable_type", [mc.LOG_RETURN, mc.Q_VAR])
@pytest.mark.parametrize("is_spot", [True, False])
def test_logsv_chain_sensitivities_match_crn_differences(variable_type, is_spot):
    N, npy = 2000, 100
    ttms, fw, df, strikes = _chain_case(variable_type)
    params = (0.6, 0.5, 2.0, 2.5, -0.4, 1.2)
    etas = np.array([0.9, 1.1])
    steps = mc.chain_steps(ttms, npy)
    Z = [_normals(10 + m, steps[m][0], N) for m in range(2)]
    Z0s, Z1s, dts = [z[0] for z in Z], [z[1] for z in Z], [d for _, d in steps]
    p, e, g, gse = mg.logsv_mc_chain_greeks_fixed(params, ttms, fw, df, strikes, TYPES, etas, Z0s, Z1s, dts, is_spot, variable_type)
    po, eo = mc.logsv_mc_chain_fixed(params, ttms, fw, df, strikes, TYPES, etas, Z0s, Z1s, dts, is_spot, variable_type)
    price = lambda prm, f=fw: mc.logsv_mc_chain_fixed(prm, ttms, f, df, strikes, TYPES, etas, Z0s, Z1s, dts, is_spot, variable_type)[0]
    for m in range(2):
        np.testing.assert_allclose(p[m], po[m], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(e[m], eo[m], rtol=1e-12, atol=1e-15)
    h = 1e-6
    pu, pd = price(params, fw * (1 + h)), price(params, fw * (1 - h))
    for m in range(2):
        _fd_gate(g[m][0], gse[m][0], (pu[m] - pd[m]) / (2 * h * fw[m]), ("delta", m))
    for k, name in enumerate(mg.LOGSV_PARAMS):
        h = _step(params[k])
        pu, pd = price(_bumped(params, k, h)), price(_bumped(params, k, -h))
        for m in range(2):
            _fd_gate(g[m][1 + k], gse[m][1 + k], (pu[m] - pd[m]) / (2 * h), (name, m))


@pytest.mark.parametrize("variable_type", [mc.LOG_RETURN, mc.Q_VAR])
def test_heston_chain_sensitivities_match_crn_differences(variable_type):
    N, npy = 2000, 200
    ttms, fw, df, strikes = _chain_case(variable_type)
    if variable_type == mc.Q_VAR:
        strikes = [0.05 * QK, 0.05 * QK]
    steps = mc.chain_steps(ttms, npy)
    Z = [_normals(20 + m, steps[m][0], N) for m in range(2)]
    Z0s, Z1s, dts = [z[0] for z in Z], [z[1] for z in Z], [d for _, d in steps]
    params = HESTON_FLOOR_P
    p, e, g, gse = mg.heston_mc_chain_greeks_fixed(params, ttms, fw, df, strikes, TYPES, Z0s, Z1s, dts, variable_type)
    po, eo = mc.heston_mc_chain_fixed(params, ttms, fw, df, strikes, TYPES, Z0s, Z1s, dts, variable_type)
    price = lambda prm, f=fw: mc.heston_mc_chain_fixed(prm, ttms, f, df, strikes, TYPES, Z0s, Z1s, dts, variable_type)[0]
    for m in range(2):
        np.testing.assert_allclose(p[m], po[m], rtol=1e-13, atol=1e-15)
    h = 1e-6
    pu, pd = price(params, fw * (1 + h)), price(params, fw * (1 - h))
    for m in range(2):
        _fd_gate(g[m][0], gse[m][0], (pu[m] - pd[m]) / (2 * h * fw[m]), ("delta", m))
        if variable_type == mc.Q_VAR:
            vanilla = np.isin(TYPES[m], ["C", "P"])
            assert np.all(g[m][0][vanilla] == 0.0)         # C / P on the quadratic variance do not move with the forward
    for k, name in enumerate(mg.HESTON_PARAMS):
        h = _step(params[k])
        pu, pd = price(_bumped(params, k, h)), price(_bumped(params, k, -h))
        for m in range(2):
            _fd_gate(g[m][1 + k], gse[m][1 + k], (pu[m] - pd[m]) / (2 * h), (name, m))


# ---- argument checks: nothing reaches the library ------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


@pytest.mark.parametrize("kwargs", [dict(precision="fp32"), dict(use_rough_mc=True, seed=1), dict(exchange="p2p"), dict(exchange="nccl")])
def test_logsv_greeks_rejections_raise_before_the_library(no_library, kwargs):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K4], optiontypes_ttms=[TYPES[0]])
    with pytest.raises(NotImplementedError):
        LogSVPricer().model_mc_chain_greeks(chain, LogSvParams(), nb_path=1000, **kwargs)


@pytest.mark.parametrize("kwargs", [dict(precision="fp32"), dict(scheme="qe"), dict(exchange="p2p")])
def test_heston_greeks_rejections_raise_before_the_library(no_library, kwargs):
    from stochvolmodels_b200 import HestonParams, HestonPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K4], optiontypes_ttms=[TYPES[0]])
    with pytest.raises(NotImplementedError):
        HestonPricer().model_mc_chain_greeks(chain, HestonParams(), nb_path=1000, **kwargs)


def test_greeks_result_layout():
    """engine output [1+P, J] -> McChainGreeks: per-maturity arrays, parameters in dataclass field order"""
    from stochvolmodels_b200 import McChainGreeks, engine
    from stochvolmodels_b200.pricers.mc_greeks import to_mc_chain_greeks
    offsets = np.array([0, 2, 5], dtype=np.int32)
    g = np.arange(7 * 5, dtype=float).reshape(7, 5)
    res = to_mc_chain_greeks(([np.zeros(2), np.zeros(3)], [np.zeros(2), np.zeros(3)], g, -g, offsets), engine.LOGSV_GREEK_PARAMS)
    assert isinstance(res, McChainGreeks)
    assert list(res.params) == ["sigma0", "theta", "kappa1", "kappa2", "beta", "volvol"]
    np.testing.assert_array_equal(res.delta[1], g[0, 2:])
    np.testing.assert_array_equal(res.params["kappa2"][0], g[4, :2])
    np.testing.assert_array_equal(res.params_se["volvol"][1], -g[6, 2:])
    assert engine.HESTON_GREEK_PARAMS == ("v0", "theta", "kappa", "rho", "volvol")
