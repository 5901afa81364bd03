"""CPU checks of the Hawkes forward-mode Fourier sensitivities (DESIGN.md §4.3): the numpy restatement in oracle/hawkes_greeks.py against
central differences, the public method's argument checks and result layout, and the argument checks of the C entry point (which run
before any device work, so they need the library but no GPU).  Measured figures (hawkes_fourier.npz chain, 500-point grid) are quoted
next to each bound."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes, mgf
from oracle import hawkes_greeks as H


def _golden_case(which):
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    return p, g["ttms"], g["forwards"], g["discfactors"], [g["strikes"]] * 3, [g["types"]] * 3


def _bump(p, name, h):
    up, dn = dict(p), dict(p)
    up[name] += h
    dn[name] -= h
    return up, dn


def _step(p, name):
    return 1e-6 * max(1.0, abs(p[name]))


@pytest.fixture(scope="module", params=["dflt", "alt"])
def case(request):
    p, ttms, fw, df, K, T = _golden_case(request.param)
    return request.param, (p, ttms, fw, df, K, T), H.hawkes_chain_greeks(p, ttms, fw, df, K, T)


@pytest.mark.parametrize("which", ["dflt", "alt"])
@pytest.mark.parametrize("spot", [True, False])
def test_tangent_rhs_vs_central_differences_of_the_rhs(which, spot):
    """J(A) dA + d_p f(A) against [f_{p+h}(A + h dA) - f_{p-h}(A - h dA)] / 2h for each ODE direction (measured <= 1.8e-8 relative to max(1, |cd|): the O(h^2) term of the differences)"""
    p = _golden_case(which)[0]
    phi = mgf.phi_grid(0.13, spot, hawkes.MAX_PHI)[::37]
    psi = np.zeros_like(phi)
    rng = np.random.default_rng(7)
    A = 0.05 * (rng.standard_normal((phi.shape[0], 3)) + 1j * rng.standard_normal((phi.shape[0], 3)))
    dA = rng.standard_normal((phi.shape[0], 3)) + 1j * rng.standard_normal((phi.shape[0], 3))
    for name in H.ODE_NAMES:
        h = _step(p, name)
        up, dn = _bump(p, name, h)
        for da in (np.zeros_like(dA), dA):
            cd = (hawkes.HawkesRhs(up, phi, psi)(A + h * da) - hawkes.HawkesRhs(dn, phi, psi)(A - h * da)) / (2 * h)
            got = H.HawkesTangentRhs(p, name, phi, psi)(A, da)
            assert np.max(np.abs(got - cd)) <= 1e-7 * max(1.0, np.max(np.abs(cd))), (name, spot)


def test_primal_and_mesh_reproduce_the_oracle_pricer(case):
    _, (p, ttms, fw, df, K, T), (out, grids) = case
    ref, ref_grids, _ = hawkes.fourier_chain_prices(p, ttms, fw, df, K, T, return_grids=True)
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    replayed, lms = H.hawkes_chain_prices_on_meshes(p, ttms, fw, df, K, T, grids["meshes"], vs)
    for m in range(3):
        assert np.array_equal(out[m][0], ref[m])
        assert np.array_equal(grids["a"][m], ref_grids[m][0])
        assert np.array_equal(replayed[m], ref[m]) and np.array_equal(lms[m], ref_grids[m][1])


def test_tangents_vs_central_differences_on_the_fixed_mesh(case):
    """the exact derivative of the scheme: d price and dlog_mgf against central differences of the replay (measured: prices <= 5.4e-10
    relative to max(1, |cd|), mean_p)"""
    _, (p, ttms, fw, df, K, T), (out, grids) = case
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    for i, name in enumerate(H.HAWKES_NAMES):
        h = _step(p, name)
        up, dn = _bump(p, name, h)
        pu, lu = H.hawkes_chain_prices_on_meshes(up, ttms, fw, df, K, T, grids["meshes"], vs)
        pd, ld = H.hawkes_chain_prices_on_meshes(dn, ttms, fw, df, K, T, grids["meshes"], vs)
        for m in range(3):
            cd = (pu[m] - pd[m]) / (2 * h)
            assert np.max(np.abs(cd - out[m][3 + i])) <= 1e-7 * max(1.0, np.max(np.abs(cd))), (name, m)
            dcd = (lu[m] - ld[m]) / (2 * h)
            assert np.max(np.abs(grids["dlog_mgf"][i, m] - dcd)) <= 1e-7 * max(1.0, np.max(np.abs(dcd))), (name, m)


# gap between the forward-mode sensitivities and central differences of the ADAPTIVE pricer (grid pinned): the derivative of the step-size
# control's mesh choice, which the scheme-exact tangents leave out.  Relative to max(1, max |cd|), over both parameter sets and the three
# maturities of hawkes_fourier.npz, both measures.  Measured under the spot measure: 4.9e-5 (mean_p), 3.6e-5 (shift_p), 2.2e-5 (mean_m), 6.0e-6 (shift_m),
# 1.1e-6 (sigma), 4.9e-7 (kappa_m), <= 4e-8 for the intensity parameters, 2e-11 for lambda_p / lambda_m (no ODE direction).
ADAPTIVE_GAP = 1e-4


@pytest.mark.parametrize("spot", [True, False])
def test_tangents_vs_central_differences_of_the_adaptive_pricer(case, spot):
    which, (p, ttms, fw, df, K, T), (out, _) = case
    if not spot:
        out = H.hawkes_chain_greeks(p, ttms, fw, df, K, T, is_spot_measure=False)[0]
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    for i, name in enumerate(H.HAWKES_NAMES):
        h = _step(p, name)
        up, dn = _bump(p, name, h)
        pu = hawkes.fourier_chain_prices(up, ttms, fw, df, K, T, is_spot_measure=spot, vol_scaler=vs)
        pd = hawkes.fourier_chain_prices(dn, ttms, fw, df, K, T, is_spot_measure=spot, vol_scaler=vs)
        for m in range(3):
            cd = (pu[m] - pd[m]) / (2 * h)
            assert np.max(np.abs(cd - out[m][3 + i])) <= ADAPTIVE_GAP * max(1.0, np.max(np.abs(cd))), (which, name, m)


@pytest.mark.parametrize("spot", [True, False])
def test_delta_gamma_vs_central_differences_in_the_forward(spot):
    """delta and gamma against central differences of the oracle pricer in the forward (grid pinned; measured: delta 2.4e-12, gamma 6.2e-8
    relative to max(1, |cd|))"""
    p, ttms, fw, df, K, T = _golden_case("alt")
    types = [T[0], np.array(["IP", "P", "C", "IC", "C"]), T[2]] if not spot else T
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    out, _ = H.hawkes_chain_greeks(p, ttms, fw, df, K, types, is_spot_measure=spot, vol_scaler=vs)
    for m in range(3):
        h = 1e-4 * fw[m]

        def price(f):
            fwd = fw.copy()
            fwd[m] = f
            return hawkes.fourier_chain_prices(p, ttms, fwd, df, K, types, is_spot_measure=spot, vol_scaler=vs)[m]

        def cd(s):          # central differences with step s h
            pu, pd = price(fw[m] + s * h), price(fw[m] - s * h)
            return (pu - pd) / (2 * s * h), (pu - 2 * p0 + pd) / (s * h) ** 2
        p0 = price(fw[m])
        assert np.max(np.abs(out[m][0] - p0)) == 0.0
        (d1, g1), (d2, g2) = cd(1.0), cd(2.0)
        d_cd, g_cd = (4.0 * d1 - d2) / 3.0, (4.0 * g1 - g2) / 3.0            # Richardson: the O(h^2) term cancels
        assert np.max(np.abs(out[m][1] - d_cd)) <= 1e-7 * max(1.0, np.max(np.abs(d_cd))), m
        assert np.max(np.abs(out[m][2] - g_cd)) <= 1e-7 * max(1.0, np.max(np.abs(g_cd))), m


# ---- the public method ----
def _chain():
    import stochvolmodels_b200 as sv
    p, ttms, fw, df, K, T = _golden_case("dflt")
    return sv.OptionChain(ttms=ttms, forwards=fw, strikes_ttms=K, optiontypes_ttms=T, discfactors=df)


@pytest.mark.parametrize("kwargs", [dict(risk_premia_gamma=0.4), dict(is_stiff_solver=True), dict(variable_type="Q_VAR")])
def test_unsupported_options_raise_before_the_engine(monkeypatch, kwargs):
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine

    def boom(*a, **k):
        raise AssertionError("engine called")

    monkeypatch.setattr(engine, "hawkesjd_price_chain_greeks", boom)
    params = sv.HawkesJDParams(risk_premia_gamma=kwargs.pop("risk_premia_gamma", None))
    if "variable_type" in kwargs:
        kwargs = dict(variable_type=sv.VariableType.Q_VAR)
    with pytest.raises(NotImplementedError):
        sv.HawkesJDPricer().price_chain_greeks(_chain(), params, **kwargs)


def test_result_layout_follows_hawkes_greek_params(monkeypatch):
    import dataclasses
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    names = tuple(f.name for f in dataclasses.fields(sv.HawkesJDParams) if f.name not in ("mu", "risk_premia_gamma"))
    assert sv.HAWKES_GREEK_PARAMS == engine.HAWKES_GREEK_PARAMS == names == H.HAWKES_NAMES
    seen = {}

    def fake(params, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, vol_scaler=None, max_phi=None):
        seen.update(vol_scaler=vol_scaler, spot=is_spot_measure, max_phi=max_phi)
        offsets = np.array([0, 5, 10, 15])
        greeks = np.arange(17 * 15, dtype=float).reshape(17, 15)
        return [np.zeros(5)] * 3, greeks, offsets

    monkeypatch.setattr(engine, "hawkesjd_price_chain_greeks", fake)
    g = sv.HawkesJDPricer().price_chain_greeks(_chain(), sv.HawkesJDParams(), is_spot_measure=False, vol_scaler=0.11)
    assert isinstance(g, sv.FourierChainGreeks)
    assert tuple(g.params) == names
    assert seen == dict(vol_scaler=0.11, spot=False, max_phi=500)
    assert np.array_equal(g.delta[1], np.arange(5, 10)) and np.array_equal(g.gamma[2], 15 + np.arange(10, 15))
    for k, name in enumerate(names):
        assert np.array_equal(g.params[name][0], (2 + k) * 15 + np.arange(5)), name


# ---- the C entry point's argument checks: one defect per call, code and message, no device work ----
NULL = (-1, "invalid argument: null pointer")
TTMS = (-1, "invalid argument: ttms must be positive and strictly increasing")
MP = (-1, "invalid argument: M >= 1, P >= 3")
STRIKE = (-1, "invalid argument: strikes must be positive")
NOT_IMPL = (-5, "not implemented")

DEFECTS = {
    "params=null": (dict(params=None), NULL),
    "ttms=null": (dict(ttms=None), NULL),
    "forwards=null": (dict(forwards=None), NULL),
    "discfactors=null": (dict(discfactors=None), NULL),
    "offsets=null": (dict(offsets=None), NULL),
    "strikes=null": (dict(strikes=None), NULL),
    "types=null": (dict(types=None), NULL),
    "prices=null": (dict(prices=None), NULL),
    "greeks=null": (dict(greeks=None), NULL),
    "M=0": (dict(M=0), MP),
    "P=2": (dict(P=2), MP),
    "ttms-decreasing": (dict(ttms=[0.5, 0.25]), TTMS),
    "strike-zero": (dict(strikes=[0.9, 1.0, 1.1, 0.9, 0.0, 1.1]), STRIKE),
    "type-4": (dict(types=[1, 4, 0] * 2), NOT_IMPL),
    "inverse-under-spot": (dict(types=[1, 2, 0] * 2), NOT_IMPL),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_c_entry_point_rejects(defect):
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    change, expected = DEFECTS[defect]
    a = dict(params=C.HawkesParamsC(*[0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5]), M=2, ttms=[0.25, 0.5],
             forwards=[1.0, 1.0], discfactors=[1.0, 1.0], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2,
             P=0, prices=np.zeros(6), greeks=np.zeros(17 * 6))
    a.update(change)
    f64 = lambda v: None if v is None else C.dptr(C.f64(v))          # the pointer keeps its array alive
    off = None if a["offsets"] is None else np.asarray(a["offsets"], dtype=np.int32)
    ty = None if a["types"] is None else np.asarray(a["types"], dtype=np.int8)
    rc = lib.b200sv_hawkesjd_price_chain_greeks(
        None if a["params"] is None else ctypes.byref(a["params"]), a["M"], f64(a["ttms"]), f64(a["forwards"]), f64(a["discfactors"]),
        None if off is None else C.iptr(off), f64(a["strikes"]), None if ty is None else C.i8ptr(ty), 1, -1.0, a["P"],
        None if a["prices"] is None else C.dptr(a["prices"]), None if a["greeks"] is None else C.dptr(a["greeks"]), None, None)
    assert (rc, lib.b200sv_last_error().decode()) == expected
