"""GPU: pathwise Monte Carlo sensitivities of the LogSV / Heston chain pricers (DESIGN.md §3.9).

  path level  -- the tangent stepper's state is bit-identical to the production stepper's; its tangents equal the forward-mode oracle
                 (oracle/mc_greeks.py) fed with the kernel's own normals
  prices      -- model_mc_chain_greeks returns model_mc_price_chain's prices and standard errors
  sensitivity -- every sensitivity within 0.1 of its standard error of a common-random-number central difference of the public
                 model_mc_price_chain; forward delta and Heston parameter sensitivities against the Fourier route
"""
import numpy as np
import pytest

from conftest import load_golden
from oracle import mc, mc_greeks as mg

pytestmark = pytest.mark.gpu

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                   # quickstart LogSV parameters
LOGSV_BTC = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)


def _scaled_close(a, b, rtol, what):
    scale = max(float(np.max(np.abs(b))), 1e-300)
    err = float(np.max(np.abs(a - b))) / scale
    assert err <= rtol, (what, err)


# ---- path level ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
@pytest.mark.parametrize("is_spot,eta", [(True, 1.0), (False, 0.9)])
def test_logsv_tangent_terminal_vs_production_stepper_and_oracle(cuda_lib, gauss, is_spot, eta):
    from stochvolmodels_b200 import engine
    N, npy, ttm, seed = 4096, 252, 0.2, 99
    pc = engine.logsv_params_c(*LOGSV_BTC)
    flags = engine.mc_flags("fp64", gauss)
    S, dt = mc.set_time_grid(ttm, npy)
    for slice_idx, offset in ((0, 0), (1, 0), (1, 5000)):
        x, s, q, dx, ds, dq = engine.logsv_tangent_terminal(pc, ttm, N, npy, is_spot, eta, seed, flags, slice_idx, offset)
        if offset == 0:          # same state as the production kernel, bit for bit
            if slice_idx == 0:
                xr, sr, qr = engine.logsv_terminal(pc, ttm, N, npy, is_spot, eta, seed, flags)
            else:
                xr, sr, qr = engine.logsv_terminal_from_state(pc, np.zeros(N), LOGSV_BTC[0] * np.ones(N), np.zeros(N), ttm, npy, is_spot, eta,
                                                              seed, flags, slice_idx)
            for a, b in ((x, xr), (s, sr), (q, qr)):
                np.testing.assert_array_equal(a, b)
        z0, z1 = engine.device_normals(seed, offset, N, slice_idx, S, flags)
        d0 = np.zeros((6, N))
        d0[0] = 1.0
        xo, so, qo, dxo, dso, dqo = mg.logsv_tangent_step_fixed(np.zeros(N), LOGSV_BTC[0] * np.ones(N), np.zeros(N), 0 * d0, d0, 0 * d0,
                                                                z0, z1, dt, *LOGSV_BTC[1:], eta, is_spot)
        np.testing.assert_allclose(s, so, rtol=1e-11)
        for k, name in enumerate(mg.LOGSV_PARAMS):
            for a, b, var in ((dx, dxo, "x"), (ds, dso, "sigma"), (dq, dqo, "q")):
                _scaled_close(a[k], b[k], 1e-10, (name, var, slice_idx, offset))


@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
def test_heston_tangent_terminal_vs_production_stepper_and_oracle(cuda_lib, gauss):
    from stochvolmodels_b200 import engine
    N, npy, ttm, seed = 4096, 360, 0.3, 7
    params = tuple(load_golden("heston_mc_fixed_floor.npz")["params"])      # Feller violated: the floor binds
    pc = engine.heston_params_c(*params)
    flags = engine.mc_flags("fp64", gauss)
    S, dt = mc.set_time_grid(ttm, npy)
    for slice_idx, offset in ((0, 0), (1, 12345)):
        x, v, q, dx, dv, dq = engine.heston_tangent_terminal(pc, ttm, N, npy, seed, flags, slice_idx, offset)
        if slice_idx == 0:
            xr, vr, qr = engine.heston_terminal(pc, ttm, N, npy, seed, flags)
            for a, b in ((x, xr), (v, vr), (q, qr)):
                np.testing.assert_array_equal(a, b)
        assert np.any(v == 1e-4)
        z0, z1 = engine.device_normals(seed, offset, N, slice_idx, S, flags)
        d0 = np.zeros((5, N))
        d0[0] = 1.0
        xo, vo, qo, dxo, dvo, dqo = mg.heston_tangent_step_fixed(np.zeros(N), params[0] * np.ones(N), np.zeros(N), 0 * d0, d0, 0 * d0, z0, z1,
                                                                 dt, *params[1:])
        for k, name in enumerate(mg.HESTON_PARAMS):
            for a, b, var in ((dx, dxo, "x"), (dv, dvo, "v"), (dq, dqo, "q")):
                _scaled_close(a[k], b[k], 1e-10, (name, var, slice_idx))


# ---- chains --------------------------------------------------------------------------------------------------------------
def _quickstart():
    from stochvolmodels_b200 import OptionChain
    return OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])


def _btc():
    from stochvolmodels_b200 import get_btc_test_chain_data
    return get_btc_test_chain_data()


def _bump_forwards(chain, f):
    from stochvolmodels_b200 import OptionChain
    return OptionChain(ttms=chain.ttms, forwards=chain.forwards * f, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                       discfactors=chain.discfactors)


CASES = [("logsv", "quickstart", True), ("logsv", "quickstart", False), ("logsv", "btc", True), ("logsv", "btc", False), ("heston", "g4", True)]


def _case(model, chain_name):
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, LOGSV_BTC_PARAMS
    chain = {"quickstart": _quickstart, "btc": _btc, "g4": _quickstart}[chain_name]()
    if chain_name == "g4":
        from stochvolmodels_b200 import OptionChain
        chain = OptionChain(ttms=np.array([0.25, 1.0]), forwards=np.ones(2), strikes_ttms=[K5, K5], optiontypes_ttms=[T5, T5])
    if model == "heston":
        return HestonPricer(), chain, HestonParams()
    return LogSVPricer(), chain, (LOGSV_BTC_PARAMS if chain_name == "btc" else LogSvParams(*Q))


@pytest.mark.parametrize("model,chain_name,is_spot", CASES)
def test_greeks_prices_equal_price_chain(cuda_lib, model, chain_name, is_spot):
    pricer, chain, params = _case(model, chain_name)
    kw = dict(nb_path=200_000, seed=2024)
    if model == "logsv":
        kw.update(nb_steps=252, is_spot_measure=is_spot)
    res = pricer.model_mc_chain_greeks(chain, params, **kw)
    p, e = pricer.model_mc_price_chain(chain, params, **kw)
    for m in range(len(chain.ttms)):
        np.testing.assert_allclose(res.prices[m], p[m], rtol=1e-13, atol=0)
        np.testing.assert_allclose(res.std_errors[m], e[m], rtol=1e-13, atol=0)
        assert res.delta[m].shape == p[m].shape and all(v[m].shape == p[m].shape for v in res.params.values())
    again = pricer.model_mc_chain_greeks(chain, params, **kw)       # fixed-order reductions: bitwise reproducible
    for m in range(len(chain.ttms)):
        np.testing.assert_array_equal(again.delta[m], res.delta[m])
        for name in res.params:
            np.testing.assert_array_equal(again.params[name][m], res.params[name][m])


def _crn_gate(g, se, up, dn, h, what):
    """|pathwise - CRN central difference| <= 0.1 SE; the second term is the fp64 round-off of the difference quotient (prices agree to
    ~1e-13 relative between the two bumped runs), not a statistical allowance"""
    fd = (up - dn) / (2 * h)
    roundoff = 1e-12 * np.maximum(np.abs(up), np.abs(dn)) / h
    bad = np.abs(g - fd) > 0.1 * se + roundoff
    assert not np.any(bad), (what, g[bad], fd[bad], se[bad])


@pytest.mark.parametrize("model,chain_name,is_spot", [c for c in CASES if c[2]] + [("logsv", "btc", False)])
def test_greeks_match_crn_central_differences(cuda_lib, model, chain_name, is_spot):
    import dataclasses
    pricer, chain, params = _case(model, chain_name)
    kw = dict(nb_path=1_000_000, seed=77)
    if model == "logsv":
        kw.update(nb_steps=252, is_spot_measure=is_spot)
    res = pricer.model_mc_chain_greeks(chain, params, **kw)
    M = len(chain.ttms)
    h = 1e-5
    up = pricer.model_mc_price_chain(_bump_forwards(chain, 1 + h), params, **kw)[0]
    dn = pricer.model_mc_price_chain(_bump_forwards(chain, 1 - h), params, **kw)[0]
    for m in range(M):
        _crn_gate(res.delta[m], res.delta_se[m], up[m], dn[m], h * chain.forwards[m], ("delta", m))
    for name in res.params:
        value = getattr(params, name)
        hp = 1e-5 if name in ("beta", "rho") else 1e-5 * abs(value)           # absolute bump where the parameter may sit near 0
        up = pricer.model_mc_price_chain(chain, dataclasses.replace(params, **{name: value + hp}), **kw)[0]
        dn = pricer.model_mc_price_chain(chain, dataclasses.replace(params, **{name: value - hp}), **kw)[0]
        for m in range(M):
            _crn_gate(res.params[name][m], res.params_se[name][m], up[m], dn[m], hp, (name, m))


def _fourier_delta(prices, digital_calls, strikes, types, forward, discfactor):
    """Delta = (C + K df P(S_T > K)) / F for calls; puts by parity (P = C - df (F - K))"""
    call_delta = (np.where(types == "C", prices, prices + discfactor * (forward - strikes)) + strikes * digital_calls) / forward
    return np.where(types == "C", call_delta, call_delta - discfactor)


def _fourier_gate(mc_val, mc_se, ref, what):
    """within 4 standard errors plus the 1e-3 absolute allowance of the MC-vs-Fourier price gate (Euler discretisation bias, DESIGN.md §6)"""
    assert np.all(np.abs(mc_val - ref) <= 4.0 * mc_se + 1e-3), (what, mc_val, ref, mc_se)


def test_forward_delta_and_heston_sensitivities_vs_fourier(cuda_lib):
    import dataclasses
    from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, engine
    from stochvolmodels_b200.utils.mgf_pricer import get_phi_grid
    vs = 0.3
    phi = get_phi_grid(True, 1000, vs)
    # LogSV quickstart: forward delta
    chain = _quickstart()
    res = LogSVPricer().model_mc_chain_greeks(chain, LogSvParams(*Q), nb_path=4_000_000, nb_steps=252, seed=2024)
    prices, _, lm = engine.logsv_price_chain(engine.logsv_params_c(*Q), chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms,
                                             chain.optiontypes_ttms, vol_scaler=vs, return_grids=True)
    for m in range(2):
        dig = engine.fourier_digital(lm[m], phi, chain.forwards[m], K5, np.array(["C"] * 5), chain.discfactors[m])
        ref = _fourier_delta(prices[m], dig, K5, T5, chain.forwards[m], chain.discfactors[m])
        _fourier_gate(res.delta[m], res.delta_se[m], ref, ("logsv delta", m))
    # Heston: forward delta and the five parameter sensitivities (central differences of the closed-form Fourier price)
    chain = _case("heston", "g4")[1]
    params = HestonParams()
    vs = min(0.3, np.sqrt(params.v0 * chain.ttms[0]))     # the Heston pricer's own default grid: the digital needs its longer phi range
    phi = get_phi_grid(True, 1000, vs)
    res = HestonPricer().model_mc_chain_greeks(chain, params, nb_path=4_000_000, seed=5)
    fourier = lambda p: engine.heston_price_chain(engine.heston_params_c(p.v0, p.theta, p.kappa, p.rho, p.volvol), chain.ttms, chain.forwards,
                                                  chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms, vol_scaler=vs, return_grids=True)
    prices, lm = fourier(params)
    for m in range(2):
        dig = engine.fourier_digital(lm[m], phi, chain.forwards[m], K5, np.array(["C"] * 5), chain.discfactors[m])
        ref = _fourier_delta(prices[m], dig, K5, T5, chain.forwards[m], chain.discfactors[m])
        _fourier_gate(res.delta[m], res.delta_se[m], ref, ("heston delta", m))
    for name in res.params:
        value = getattr(params, name)
        h = 1e-5 * max(abs(value), 1.0)
        up, _ = fourier(dataclasses.replace(params, **{name: value + h}))
        dn, _ = fourier(dataclasses.replace(params, **{name: value - h}))
        for m in range(2):
            _fourier_gate(res.params[name][m], res.params_se[name][m], (up[m] - dn[m]) / (2 * h), (name, m))


def test_greeks_reject_unsupported_flags_in_the_library(cuda_lib):
    from stochvolmodels_b200 import _capi as C, engine
    chain = _quickstart()
    pc = engine.logsv_params_c(*Q)
    for flags in (C.STATE_F32, C.GAUSS_F64_PAIRED):
        with pytest.raises(C.B200svError, match="invalid argument"):
            engine.logsv_mc_chain_greeks(pc, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms, chain.optiontypes_ttms,
                                         1000, 100, True, 1, 1, flags)
    with pytest.raises(C.B200svError, match="EULER_FLOOR"):
        engine.heston_mc_chain_greeks(engine.heston_params_c(0.04, 0.04, 4.0, -0.5, 0.4), chain.ttms, chain.forwards, chain.discfactors,
                                      chain.strikes_ttms, chain.optiontypes_ttms, 1000, 100, 1, 1, 0, C.HESTON_QE)
