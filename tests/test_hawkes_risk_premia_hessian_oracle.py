"""CPU checks of the Hawkes second-order Fourier sensitivities under the risk kernel (DESIGN.md §4.13): the numpy restatement in
tests/hawkes_rp_hessian_oracle.py against central differences of the first-order scheme, against the plain Hawkes Hessian at gamma = 0, the
public methods' rejections and result layout, the implied-vol mapping of the 16 x 16 second order past the transform's 15-row limit, and
the argument checks of the C entry point (which run before any device work, so they need the library but no GPU).  Measured figures
(hawkes_fourier.npz chain, 500-point grid) are quoted next to each bound."""
import ctypes

import numpy as np
import pytest

import hawkes_hessian_oracle as HH
import hawkes_rp_hessian_oracle as RH
import ivol_greeks_oracle as og
from oracle import bsm as obsm
from oracle import hawkes, mgf
from oracle import hawkes_rp_greeks as R
from test_hawkes_risk_premia_greeks_oracle import GAMMAS, REJECTIONS, _bumped, _chain, _golden_case, _step


@pytest.fixture(scope="module", params=[(w, g) for w in ("dflt", "alt") for g in GAMMAS], ids=lambda c: f"{c[0]}-g{c[1]}")
def case(request):
    which, gamma = request.param
    p, ttms, fw, df, K, T = _golden_case(which)
    return which, gamma, (p, ttms, fw, df, K, T), RH.hawkes_rp_chain_hessian(p, gamma, ttms, fw, df, K, T)


def _rel(got, cd):
    return float(np.max(np.abs(got - cd))) / max(1.0, float(np.max(np.abs(cd))))


@pytest.mark.parametrize("which", ["dflt", "alt"])
def test_phi_seeded_second_order_rhs_vs_central_differences(which):
    """the mixed part of the phi-seeded hyper-dual right-hand side of the pair (a, gamma) against central differences along gamma (phi
    moves by -h, A by h dA_gamma, the tangent by h d2A) of the first-order right-hand side of a: HawkesTangentRhs for an ODE direction,
    HawkesPhiTangentRhs for gamma (measured <= 1.7e-10 relative to max(1, |cd|))"""
    import oracle.hawkes_greeks as HG
    p = _golden_case(which)[0]
    phi = (-0.5 - 0.4) + 1j * np.imag(mgf.phi_grid(0.13, True, hawkes.MAX_PHI)[::37])
    psi = np.zeros_like(phi)
    rng = np.random.default_rng(12)
    c = lambda s: 0.05 * s * (rng.standard_normal((phi.shape[0], 3)) + 1j * rng.standard_normal((phi.shape[0], 3)))
    A, dAa, dAg, d2A = c(1.0), c(20.0), c(20.0), c(20.0)
    h = 1e-6
    for a, name in enumerate(RH.NAMES):
        if name in ("lambda_p", "lambda_m"):
            continue                                   # no ODE direction: the lambda rows come from the tangents, not the rhs
        first = (lambda ph: R.HawkesPhiTangentRhs(p, ph, psi, -1.0)) if a == RH.G else (lambda ph: HG.HawkesTangentRhs(p, name, ph, psi))
        dA1 = dAg if a == RH.G else dAa
        cd = (first(phi - h)(A + h * dAg, dA1 + h * d2A) - first(phi + h)(A - h * dAg, dA1 - h * d2A)) / (2 * h)
        _, dg, d12 = RH.tan2_rhs(p, a, RH.G, phi, A, dA1, dAg, d2A)
        assert _rel(d12, cd) <= 1e-7, (which, name, _rel(d12, cd))
        assert np.allclose(dg, R.HawkesPhiTangentRhs(p, phi, psi, -1.0)(A, dAg), rtol=1e-13, atol=1e-13)


def test_first_order_rows_are_the_risk_premia_greeks(case):
    _, gamma, (p, ttms, fw, df, K, T), (rows, grids) = case
    out, _ = R.hawkes_rp_chain_greeks(p, gamma, ttms, fw, df, K, T)
    for m in range(3):
        assert np.array_equal(rows[m][0], out[m])
        assert all(np.all(np.isfinite(x)) for x in rows[m])


def test_second_order_vs_central_differences_on_the_fixed_meshes(case):
    """the exact second derivative of the scheme: d2log_mgf, d2log_norm and the 136 Hessian rows against central differences in p of the
    first-order rows replayed on the recorded grid and normaliser meshes (measured over the ten cases: <= 1.4e-8 relative to
    max(1, |cd|)), and vanna against Richardson differences in the forward of the first-order parameter rows (<= 2.2e-12)"""
    which, gamma, (p, ttms, fw, df, K, T), (rows, grids) = case
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    on_meshes = lambda q, g, f=fw: RH.rp_tangents_on_meshes(q, g, ttms, f, K, T, grids["meshes"], grids["norm_meshes"], vs)
    for b, name in enumerate(RH.NAMES):
        h = _step(p, gamma, name)
        (uo, ul, un), (do, dl, dn) = on_meshes(*_bumped(p, gamma, name, h)), on_meshes(*_bumped(p, gamma, name, -h))
        for a in range(len(RH.NAMES)):
            r = RH.PAIRS.index((min(a, b), max(a, b)))
            for m in range(3):
                for got, cd in ((rows[m][2][r], (uo[m][3 + a] - do[m][3 + a]) / (2 * h)),
                                (grids["d2log_mgf"][r, m], (ul[a, m] - dl[a, m]) / (2 * h)),
                                (grids["d2log_norm"][r, m], (un[a, m] - dn[a, m]) / (2 * h))):
                    assert _rel(got, cd) <= 1e-7, (which, gamma, RH.NAMES[a], name, m, _rel(got, cd))
    for m in range(3):
        s = 1e-4 * fw[m]

        def rows_at(f):
            fwd = fw.copy()
            fwd[m] = f
            return on_meshes(p, gamma, fwd)[0][m][3:]

        d1, d2 = ((rows_at(fw[m] + k * s) - rows_at(fw[m] - k * s)) / (2 * k * s) for k in (1.0, 2.0))
        cd = (4.0 * d1 - d2) / 3.0
        assert _rel(rows[m][1], cd) <= 1e-7, (which, gamma, "vanna", m, _rel(rows[m][1], cd))


# gap between the exact Hessian rows and central differences of the first-order rows of the ADAPTIVE pricer (grid scale pinned): the
# derivative of the step-size control's mesh choice, which the scheme-exact rows leave out.  Relative to max(1, max |cd|) per row, over both
# parameter sets, the five gammas and the three maturities.  Measured: 7.9e-4 at most (the (mean_m, mean_p) row, alt at gamma = 0); the
# gamma row at most 9.3e-5 ...
ADAPTIVE_GAP = 2e-3
# ... except where a normaliser point sits at phi = -1 (gamma = 0 or 1).  There the log-MGF vanishes and the adaptive solver chooses its
# mesh on rounding noise, so each bumped first-order gamma row sits on another mesh and its difference quotient carries the tangent's
# truncation error over 2h: measured 7.5e-2 (dflt, gamma = 0) and 2.9e-2 (dflt, gamma = 1) in the (gamma, shift_p) entry.  The
# fixed-mesh test above checks those rows exactly.
PHI_MINUS_ONE_GAP = 0.15


def test_hessian_vs_central_differences_of_the_adaptive_first_order_rows(case):
    which, gamma, (p, ttms, fw, df, K, T), (rows, _) = case
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    for b, name in enumerate(RH.NAMES):
        h = _step(p, gamma, name)
        (pu, gu), (pd, gd) = _bumped(p, gamma, name, h), _bumped(p, gamma, name, -h)
        up = R.hawkes_rp_chain_greeks(pu, gu, ttms, fw, df, K, T, vol_scaler=vs)[0]
        dn = R.hawkes_rp_chain_greeks(pd, gd, ttms, fw, df, K, T, vol_scaler=vs)[0]
        for a in range(len(RH.NAMES)):
            r = RH.PAIRS.index((min(a, b), max(a, b)))
            bound = PHI_MINUS_ONE_GAP if gamma in (0.0, 1.0) and RH.G in (a, b) else ADAPTIVE_GAP
            for m in range(3):
                cd = (up[m][3 + a] - dn[m][3 + a]) / (2 * h)
                assert _rel(rows[m][2][r], cd) <= bound, (which, gamma, RH.NAMES[a], name, m, _rel(rows[m][2][r], cd))


@pytest.mark.parametrize("which", ["dflt", "alt"])
def test_gamma_zero_matches_the_plain_hawkes_hessian(which):
    """at gamma = 0 with discount factors 1 the risk-kernel pricer is the plain one up to normalisers that vanish to solver accuracy: the
    15 x 15 block and the 15 vanna rows equal hawkes_chain_hessian (measured <= 2e-15 relative to max(1, |plain|))"""
    p, ttms, fw, df, K, T = _golden_case(which)
    ones = np.ones(3)
    rows, _ = RH.hawkes_rp_chain_hessian(p, 0.0, ttms, fw, ones, K, T)
    plain, _ = HH.hawkes_chain_hessian(p, ttms, fw, ones, K, T)
    n = len(HH.NAMES)
    sub = [RH.PAIRS.index(pq) for pq in HH.PAIRS]
    for m in range(3):
        assert _rel(rows[m][1][:n], plain[m][1]) <= 1e-10, (which, "vanna", m)
        assert _rel(rows[m][2][sub], plain[m][2]) <= 1e-10, (which, "hessian", m)


# ---- the implied-vol mapping past the transform's 15 rows ----
def test_ivol_split_of_the_16_by_16_second_order_matches_one_transform(monkeypatch):
    """a 16-parameter Black-in model (tests/ivol_greeks_oracle.py) through to_chain_ivol_sensitivities with the library's transform
    replaced by the numpy one, limited to 15 rows a call as the library is: every vanna and Hessian entry equals the numpy transform of all
    16 x 16 at once (1e-10); the calls are [p0..p14], [gamma, p0..p13], [gamma, p14]"""
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.fourier_greeks import to_chain_ivol_sensitivities
    n = 16
    names = sv.HAWKES_RISK_PREMIA_GREEK_PARAMS
    pv, sigma0, a, b, Q, e = og.default_black_in(n)
    F, T, D = 1.05, 0.5, 0.97
    K = og.strikes_for_d1(F, T, sigma0, np.linspace(-2.0, 2.0, 9))
    types = np.array(["P"] * 4 + ["C"] * 5)
    price, greeks, vanna, hessian, want = og.black_in_model(F, K, T, D, types, pv, 1.0, sigma0, a, b, Q, e)
    chain = sv.OptionChain(ttms=np.array([T]), forwards=np.array([F]), strikes_ttms=[K], optiontypes_ttms=[types], discfactors=np.array([D]))
    calls = []

    def transform(ttms, forwards, discfactors, strikes_ttms, types_ttms, prices, rows, vanna=None, hessian=None):
        assert rows.shape[0] - 2 <= 15
        calls.append(rows.shape[0] - 2)
        vol = obsm.infer_bsm_implied_vol(F, T, K, np.asarray(prices[0]), types, D)
        g, v, h = og.ivol_sensitivities(F, K, T, D, vol, og.is_call_type(types), rows, vanna, hessian)
        return [vol], g, v, h

    monkeypatch.setattr(engine, "bsm_implied_vol_sensitivities", transform)
    src = sv.FourierChainHessian(prices=[price], delta=[greeks[0]], gamma=[greeks[1]], params={k: [greeks[2 + i]] for i, k in enumerate(names)},
                                 vanna={k: [vanna[i]] for i, k in enumerate(names)},
                                 hessian={k: {} for k in names})
    for r, (i, j) in enumerate(RH.PAIRS):
        src.hessian[names[i]][names[j]] = src.hessian[names[j]][names[i]] = [hessian[r]]
    iv = to_chain_ivol_sensitivities(chain, src)
    assert calls == [15, 15, 2]
    vol = obsm.infer_bsm_implied_vol(F, T, K, price, types, D)
    g, v, h = og.ivol_sensitivities(F, K, T, D, vol, og.is_call_type(types), greeks, vanna, hessian)
    close = lambda got, ref: np.max(np.abs(got - ref)) <= 1e-10 * max(1e-3, np.max(np.abs(ref)))
    assert close(iv.delta[0], g[0]) and close(iv.gamma[0], g[1])
    for i, k in enumerate(names):
        assert close(iv.params[k][0], g[2 + i]), k
        assert close(iv.vanna[k][0], v[i]), k
    for r, (i, j) in enumerate(RH.PAIRS):
        assert close(iv.hessian[names[i]][names[j]][0], h[r]), (names[i], names[j])
        assert iv.hessian[names[j]][names[i]] is iv.hessian[names[i]][names[j]]
    for i in range(n):                  # and the model's own derivatives, through the inversion
        assert np.max(np.abs(iv.vanna[names[i]][0] - want["vanna"][i])) <= 1e-8 * max(1e-3, np.max(np.abs(want["vanna"][i])))


# ---- the public methods ----
def _no_engine(monkeypatch):
    from stochvolmodels_b200 import engine

    def boom(*a, **k):
        raise AssertionError("engine called")

    for name in ("hawkesjd_price_chain_risk_premia_hessian", "hawkesjd_price_chain_risk_premia_greeks", "hawkesjd_price_chain",
                 "bsm_implied_vol_sensitivities"):
        monkeypatch.setattr(engine, name, boom)


@pytest.mark.parametrize("method", ["price_chain_risk_premia_hessian", "compute_chain_risk_premia_ivol_hessian"])
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
    seen = {}
    J = 15

    def fake(params, gamma, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None, max_phi=None):
        seen.update(gamma=gamma, vol_scaler=vol_scaler, max_phi=max_phi, sigma=params.sigma)
        rows = lambda n, base: base + np.arange(n * J, dtype=float).reshape(n, J)
        return [np.zeros(5)] * 3, rows(18, 0.0), rows(16, 1e4), rows(136, 1e6), np.array([0, 5, 10, 15])

    monkeypatch.setattr(engine, "hawkesjd_price_chain_risk_premia_hessian", fake)
    g = sv.HawkesJDPricer().price_chain_risk_premia_hessian(_chain(), sv.HawkesJDParams(sigma=0.3, risk_premia_gamma=0.25), vol_scaler=0.11)
    assert isinstance(g, sv.FourierChainHessian) and g.theta is None
    assert seen == dict(gamma=0.25, vol_scaler=0.11, max_phi=500, sigma=0.3)
    names = sv.HAWKES_RISK_PREMIA_GREEK_PARAMS
    assert tuple(g.params) == tuple(g.vanna) == tuple(g.hessian) == names
    assert np.array_equal(g.delta[1], np.arange(5, 10)) and np.array_equal(g.gamma[2], J + np.arange(10, 15))
    for k, name in enumerate(names):
        assert np.array_equal(g.params[name][0], (2 + k) * J + np.arange(5)), name
        assert np.array_equal(g.vanna[name][1], 1e4 + k * J + np.arange(5, 10)), name
    for r, (i, j) in enumerate(RH.PAIRS):
        assert np.array_equal(g.hessian[names[i]][names[j]][2], 1e6 + r * J + np.arange(10, 15)), (i, j)
        assert g.hessian[names[j]][names[i]] is g.hessian[names[i]][names[j]]


# ---- the C entry point's argument checks: one defect per call, code and message, no device work ----
from test_hawkes_risk_premia_greeks_oracle import DEFECTS, NULL  # noqa: E402

HESSIAN_DEFECTS = dict(DEFECTS, **{"vanna=null": (dict(vanna=None), NULL), "hessian=null": (dict(hessian=None), NULL)})


@pytest.mark.parametrize("defect", list(HESSIAN_DEFECTS))
def test_c_entry_point_rejects(defect):
    from stochvolmodels_b200 import _capi as C
    lib = C.load_library()
    change, expected = HESSIAN_DEFECTS[defect]
    a = dict(params=C.HawkesParamsC(*[0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5]), M=2, ttms=[0.25, 0.5],
             forwards=[1.0, 1.0], discfactors=[1.0, 1.0], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2,
             P=0, spot=1, gamma=0.4, prices=np.zeros(6), greeks=np.zeros(18 * 6), vanna=np.zeros(16 * 6), hessian=np.zeros(136 * 6))
    a.update(change)
    f64 = lambda v: None if v is None else C.dptr(C.f64(v))          # the pointer keeps its array alive
    off = None if a["offsets"] is None else np.asarray(a["offsets"], dtype=np.int32)
    ty = None if a["types"] is None else np.asarray(a["types"], dtype=np.int8)
    out = lambda k: None if a[k] is None else C.dptr(a[k])
    rc = lib.b200sv_hawkesjd_price_chain_risk_premia_hessian(
        None if a["params"] is None else ctypes.byref(a["params"]), a["M"], f64(a["ttms"]), f64(a["forwards"]), f64(a["discfactors"]),
        None if off is None else C.iptr(off), f64(a["strikes"]), None if ty is None else C.i8ptr(ty), a["spot"], -1.0, a["P"], a["gamma"],
        out("prices"), out("greeks"), None, None, None, out("vanna"), out("hessian"), None, None)
    assert (rc, lib.b200sv_last_error().decode()) == expected
