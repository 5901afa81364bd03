"""CPU checks of the Hawkes forward-mode Fourier sensitivities under the risk kernel (DESIGN.md §4.12): the numpy restatement in
oracle/hawkes_rp_greeks.py against central differences, the public methods' rejections and result layout, the implied-vol mapping of
more than 15 parameter rows, and the argument checks of the C entry point (which run before any device work, so they need the library
but no GPU).  Measured figures (hawkes_fourier.npz chain, 500-point grid) are quoted next to each bound."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes, mgf
from oracle import hawkes_rp_greeks as R

# the fixture's gamma, the fast weight branch, no risk premium, and a negative and a larger positive value with every price finite
GAMMAS = (0.4, -0.5, 0.0, -1.0, 1.0)


def _golden_case(which):
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    return p, g["ttms"], g["forwards"], g["discfactors"], [g["strikes"]] * 3, [g["types"]] * 3


def _step(p, gamma, name):
    return 1e-6 * max(1.0, abs(gamma if name == "risk_premia_gamma" else p[name]))


def _bumped(p, gamma, name, s):
    """(params, gamma) moved by s in the direction of ``name``"""
    if name == "risk_premia_gamma":
        return p, gamma + s
    q = dict(p)
    q[name] += s
    return q, gamma


@pytest.fixture(scope="module", params=[(w, g) for w in ("dflt", "alt") for g in GAMMAS], ids=lambda c: f"{c[0]}-g{c[1]}")
def case(request):
    which, gamma = request.param
    p, ttms, fw, df, K, T = _golden_case(which)
    return which, gamma, (p, ttms, fw, df, K, T), R.hawkes_rp_chain_greeks(p, gamma, ttms, fw, df, K, T)


@pytest.mark.parametrize("which", ["dflt", "alt"])
def test_phi_tangent_rhs_vs_central_differences_of_the_rhs(which):
    """J(A) dA + d f(A) / d phi against [f(phi + h, A + h dA) - f(phi - h, A - h dA)] / 2h (measured <= 3e-9 relative to max(1, |cd|))"""
    p = _golden_case(which)[0]
    phi = (-0.5 - 0.4) + 1j * np.imag(mgf.phi_grid(0.13, True, hawkes.MAX_PHI)[::37])
    psi = np.zeros_like(phi)
    rng = np.random.default_rng(11)
    A = 0.05 * (rng.standard_normal((phi.shape[0], 3)) + 1j * rng.standard_normal((phi.shape[0], 3)))
    dA = rng.standard_normal((phi.shape[0], 3)) + 1j * rng.standard_normal((phi.shape[0], 3))
    h = 1e-6
    for da in (np.zeros_like(dA), dA):
        cd = (hawkes.HawkesRhs(p, phi + h, psi)(A + h * da) - hawkes.HawkesRhs(p, phi - h, psi)(A - h * da)) / (2 * h)
        got = R.HawkesPhiTangentRhs(p, phi, psi)(A, da)
        assert np.max(np.abs(got - cd)) <= 1e-7 * max(1.0, np.max(np.abs(cd)))
    # the gamma direction: every point moves by -1
    zero = np.zeros_like(dA)
    assert np.allclose(R.HawkesPhiTangentRhs(p, phi, psi, -1.0)(A, zero), -R.HawkesPhiTangentRhs(p, phi, psi)(A, zero), rtol=1e-15, atol=0)


def test_primal_reproduces_the_oracle_pricer(case):
    _, gamma, (p, ttms, fw, df, K, T), (out, grids) = case
    ref = hawkes.fourier_chain_prices(p, ttms, fw, df, K, T, gamma=gamma)
    norm, gfw = hawkes.forwards_under_risk_kernel(p, gamma, ttms, fw)
    assert np.array_equal(np.array(grids["normalizers"]), norm) and np.array_equal(np.array(grids["gamma_forwards"]), gfw)
    for m in range(3):
        assert np.array_equal(out[m][0], ref[m])
        assert np.all(np.isfinite(out[m]))


def test_tangents_vs_central_differences_on_the_fixed_meshes(case):
    """the exact derivative of the scheme: the 16 price rows, dlog_mgf and dlog_norm against central differences of the replay on the
    recorded grid and normaliser meshes (measured over the ten cases: <= 7.3e-9 relative to max(1, |cd|), the gamma row)"""
    which, gamma, (p, ttms, fw, df, K, T), (out, grids) = case
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    for i, name in enumerate(R.RP_NAMES):
        h = _step(p, gamma, name)
        pu, lu, nu = R.hawkes_rp_chain_prices_on_meshes(*_bumped(p, gamma, name, h), ttms, fw, K, T, grids["meshes"], grids["norm_meshes"], vs)
        pd, ld, nd = R.hawkes_rp_chain_prices_on_meshes(*_bumped(p, gamma, name, -h), ttms, fw, K, T, grids["meshes"], grids["norm_meshes"], vs)
        for m in range(3):
            for got, cd in ((out[m][3 + i], (pu[m] - pd[m]) / (2 * h)), (grids["dlog_mgf"][i, m], (lu[m] - ld[m]) / (2 * h)),
                            (grids["dlog_norm"][i, m], (nu[m] - nd[m]) / (2 * h))):
                assert np.max(np.abs(got - cd)) <= 1e-7 * max(1.0, np.max(np.abs(cd))), (which, gamma, name, m)


# gap between the forward-mode rows and central differences of the ADAPTIVE pricer (grid scale pinned): the derivative of the step-size
# control's mesh choice, which the scheme-exact tangents leave out.  Relative to max(1, max |cd|), over both parameter sets, the five
# gammas and the three maturities.  Measured: 8.8e-5 (mean_p), 5.9e-5 (shift_p), 4.9e-5 (mean_m), 2.6e-5 (shift_m), 3.6e-6 (sigma),
# 3.4e-6 (risk_premia_gamma), <= 1e-6 for the intensity parameters, 4e-11 for lambda_p / lambda_m (no ODE direction).
ADAPTIVE_GAP = 2e-4


def test_tangents_vs_central_differences_of_the_adaptive_pricer(case):
    which, gamma, (p, ttms, fw, df, K, T), (out, _) = case
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    for i, name in enumerate(R.RP_NAMES):
        h = _step(p, gamma, name)
        (pu_p, gu), (pd_p, gd) = _bumped(p, gamma, name, h), _bumped(p, gamma, name, -h)
        pu = hawkes.fourier_chain_prices(pu_p, ttms, fw, df, K, T, vol_scaler=vs, gamma=gu)
        pd = hawkes.fourier_chain_prices(pd_p, ttms, fw, df, K, T, vol_scaler=vs, gamma=gd)
        for m in range(3):
            cd = (pu[m] - pd[m]) / (2 * h)
            assert np.max(np.abs(cd - out[m][3 + i])) <= ADAPTIVE_GAP * max(1.0, np.max(np.abs(cd))), (which, gamma, name, m)


@pytest.mark.parametrize("gamma", GAMMAS)
def test_delta_gamma_vs_central_differences_in_the_forward(gamma):
    """delta and gamma against Richardson central differences of the oracle pricer in the forward, which also moves the gamma forward
    (measured: delta <= 1e-11, gamma <= 1e-7 relative to max(1, |cd|))"""
    p, ttms, fw, df, K, T = _golden_case("alt")
    out, _ = R.hawkes_rp_chain_greeks(p, gamma, ttms, fw, df, K, T)
    for m in range(3):
        h = 1e-4 * fw[m]

        def price(f):
            fwd = fw.copy()
            fwd[m] = f
            return hawkes.fourier_chain_prices(p, ttms, fwd, df, K, T, gamma=gamma)[m]

        def cd(s):
            pu, pd = price(fw[m] + s * h), price(fw[m] - s * h)
            return (pu - pd) / (2 * s * h), (pu - 2 * p0 + pd) / (s * h) ** 2
        p0 = price(fw[m])
        (d1, g1), (d2, g2) = cd(1.0), cd(2.0)
        d_cd, g_cd = (4.0 * d1 - d2) / 3.0, (4.0 * g1 - g2) / 3.0
        assert np.max(np.abs(out[m][1] - d_cd)) <= 1e-7 * max(1.0, np.max(np.abs(d_cd))), (gamma, m)
        assert np.max(np.abs(out[m][2] - g_cd)) <= 1e-6 * max(1.0, np.max(np.abs(g_cd))), (gamma, m)


# ---- the public methods ----
def _chain(types=None):
    import stochvolmodels_b200 as sv
    p, ttms, fw, df, K, T = _golden_case("dflt")
    return sv.OptionChain(ttms=ttms, forwards=fw, strikes_ttms=K, optiontypes_ttms=T if types is None else types, discfactors=df)


def _no_engine(monkeypatch):
    from stochvolmodels_b200 import engine

    def boom(*a, **k):
        raise AssertionError("engine called")

    for name in ("hawkesjd_price_chain_risk_premia_greeks", "hawkesjd_price_chain", "bsm_implied_vol_sensitivities"):
        monkeypatch.setattr(engine, name, boom)


REJECTIONS = {
    "no-gamma": (dict(risk_premia_gamma=None), {}, ValueError, "price_chain_greeks"),
    "gamma-nan": (dict(risk_premia_gamma=float("nan")), {}, ValueError, "finite"),
    "gamma-inf": (dict(risk_premia_gamma=float("inf")), {}, ValueError, "finite"),
    "stiff": (dict(risk_premia_gamma=0.4), dict(is_stiff_solver=True), NotImplementedError, "is_stiff_solver"),
    "qvar": (dict(risk_premia_gamma=0.4), dict(variable_type="Q_VAR"), NotImplementedError, "LOG_RETURN"),
    "theta": (dict(risk_premia_gamma=0.4), dict(with_theta=True), NotImplementedError, "theta"),
    "inverse-measure": (dict(risk_premia_gamma=0.4), dict(is_spot_measure=False), ValueError, "not implemented"),
    "inverse-types": (dict(risk_premia_gamma=0.4), dict(types="IC"), ValueError, "not implemented"),
}


@pytest.mark.parametrize("method", ["price_chain_risk_premia_greeks", "compute_chain_risk_premia_ivol_greeks"])
@pytest.mark.parametrize("defect", list(REJECTIONS))
def test_rejections_before_any_library_call(monkeypatch, method, defect):
    import stochvolmodels_b200 as sv
    fields, kwargs, exc, text = REJECTIONS[defect]
    _no_engine(monkeypatch)
    kwargs = dict(kwargs)
    chain = _chain()
    if kwargs.pop("types", None):
        chain = _chain([np.array(["IC", "P", "C", "C", "C"])] * 3)
    if kwargs.get("variable_type"):
        kwargs["variable_type"] = sv.VariableType.Q_VAR
    with pytest.raises(exc, match=text):
        getattr(sv.HawkesJDPricer(), method)(chain, sv.HawkesJDParams(**fields), **kwargs)


def test_result_layout_follows_hawkes_risk_premia_greek_params(monkeypatch):
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    assert sv.HAWKES_RISK_PREMIA_GREEK_PARAMS == engine.HAWKES_RISK_PREMIA_GREEK_PARAMS == sv.HAWKES_GREEK_PARAMS + ("risk_premia_gamma",)
    assert sv.HAWKES_RISK_PREMIA_GREEK_PARAMS == R.RP_NAMES
    seen = {}

    def fake(params, gamma, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None, max_phi=None):
        seen.update(gamma=gamma, vol_scaler=vol_scaler, max_phi=max_phi, sigma=params.sigma)
        greeks = np.arange(18 * 15, dtype=float).reshape(18, 15)
        return [np.zeros(5)] * 3, greeks, np.array([0, 5, 10, 15])

    monkeypatch.setattr(engine, "hawkesjd_price_chain_risk_premia_greeks", fake)
    g = sv.HawkesJDPricer().price_chain_risk_premia_greeks(_chain(), sv.HawkesJDParams(sigma=0.3, risk_premia_gamma=0.25), vol_scaler=0.11)
    assert isinstance(g, sv.FourierChainGreeks) and g.theta is None
    assert tuple(g.params) == sv.HAWKES_RISK_PREMIA_GREEK_PARAMS
    assert seen == dict(gamma=0.25, vol_scaler=0.11, max_phi=500, sigma=0.3)
    assert np.array_equal(g.delta[1], np.arange(5, 10)) and np.array_equal(g.gamma[2], 15 + np.arange(10, 15))
    for k, name in enumerate(sv.HAWKES_RISK_PREMIA_GREEK_PARAMS):
        assert np.array_equal(g.params[name][0], (2 + k) * 15 + np.arange(5)), name


def test_ivol_mapping_of_more_than_15_rows_is_two_calls_on_the_same_prices(monkeypatch):
    """the transform takes at most 15 parameter rows: the 16th goes through a further call with delta and gamma in front; every row keeps
    its place"""
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.fourier_greeks import to_chain_ivol_sensitivities
    calls = []

    def fake(ttms, forwards, discfactors, strikes_ttms, types_ttms, prices, rows, vanna=None, hessian=None):
        assert 3 <= rows.shape[0] <= 17 and vanna is None and hessian is None
        calls.append(rows.copy())
        return [np.full(5, 0.5)] * 3, 10.0 * rows, None, None

    monkeypatch.setattr(engine, "bsm_implied_vol_sensitivities", fake)
    names = sv.HAWKES_RISK_PREMIA_GREEK_PARAMS
    split = lambda r: [r[0:5], r[5:10], r[10:15]]
    rows = np.arange(18 * 15, dtype=float).reshape(18, 15)
    greeks = sv.FourierChainGreeks(prices=[np.ones(5)] * 3, delta=split(rows[0]), gamma=split(rows[1]),
                                   params={n: split(rows[2 + k]) for k, n in enumerate(names)})
    iv = to_chain_ivol_sensitivities(_chain(), greeks)
    assert len(calls) == 2 and np.array_equal(calls[0], rows[:17]) and np.array_equal(calls[1], rows[[0, 1, 17]])
    assert tuple(iv.params) == names
    for k, name in enumerate(names):
        assert np.array_equal(np.concatenate(iv.params[name]), 10.0 * rows[2 + k]), name
    assert np.array_equal(np.concatenate(iv.delta), 10.0 * rows[0])


# ---- the C entry point's argument checks: one defect per call, code and message, no device work ----
NULL = (-1, "invalid argument: null pointer")
GAMMA = (-1, "invalid argument: risk_premia_gamma must be finite")
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
    "gamma=nan": (dict(gamma=float("nan")), GAMMA),
    "gamma=-inf": (dict(gamma=float("-inf")), GAMMA),
    "M=0": (dict(M=0), MP),
    "P=2": (dict(P=2), MP),
    "ttms-decreasing": (dict(ttms=[0.5, 0.25]), TTMS),
    "strike-zero": (dict(strikes=[0.9, 1.0, 1.1, 0.9, 0.0, 1.1]), STRIKE),
    "inverse-measure": (dict(spot=0), NOT_IMPL),
    "inverse-call": (dict(types=[1, 2, 0] * 2), NOT_IMPL),
    "type-4": (dict(types=[1, 4, 0] * 2), NOT_IMPL),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_c_entry_point_rejects(defect):
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    change, expected = DEFECTS[defect]
    a = dict(params=C.HawkesParamsC(*[0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5]), M=2, ttms=[0.25, 0.5],
             forwards=[1.0, 1.0], discfactors=[1.0, 1.0], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2,
             P=0, spot=1, gamma=0.4, prices=np.zeros(6), greeks=np.zeros(18 * 6))
    a.update(change)
    f64 = lambda v: None if v is None else C.dptr(C.f64(v))          # the pointer keeps its array alive
    off = None if a["offsets"] is None else np.asarray(a["offsets"], dtype=np.int32)
    ty = None if a["types"] is None else np.asarray(a["types"], dtype=np.int8)
    rc = lib.b200sv_hawkesjd_price_chain_risk_premia_greeks(
        None if a["params"] is None else ctypes.byref(a["params"]), a["M"], f64(a["ttms"]), f64(a["forwards"]), f64(a["discfactors"]),
        None if off is None else C.iptr(off), f64(a["strikes"]), None if ty is None else C.i8ptr(ty), a["spot"], -1.0, a["P"], a["gamma"],
        None if a["prices"] is None else C.dptr(a["prices"]), None if a["greeks"] is None else C.dptr(a["greeks"]), None, None, None)
    assert (rc, lib.b200sv_last_error().decode()) == expected
