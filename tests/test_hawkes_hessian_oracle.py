"""CPU checks of the Hawkes second-order Fourier sensitivities (DESIGN.md §4.5): the numpy forward-over-forward restatement in
hawkes_hessian_oracle.py against central differences of the first-order forward mode of oracle/hawkes_greeks.py, the gap to differences of
the adaptive pricer, and the public method's argument checks and result layout.  Measured figures are quoted next to their bounds.

The 1e-7 bound on central differences with relative step r of a first-order quantity g (relative to max(1, |cd|)): the truncation
term is r^2 / 6 times g's third logarithmic derivative, the rounding term about eps / r -- with r = 1e-6, 2e-10 from rounding and, for third
derivatives up to 1e3 relative, 2e-10 from truncation.  The measured worst cases (5.2e-9 on the mesh, 4.3e-9 in the forward) leave a factor
of 20; the right-hand-side check needs the smaller step given there."""
import numpy as np
import pytest

import hawkes_hessian_oracle as O
import mgf_hessian_oracle as MH
from conftest import load_golden
from oracle import hawkes, mgf
from oracle import hawkes_greeks as HG
from oracle import mgf_greeks as G


def _golden_case(which):
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    return p, g["ttms"], g["forwards"], g["discfactors"], [g["strikes"]] * 3, [g["types"]] * 3


def _btc_case():
    from stochvolmodels_b200 import HawkesJDParams, get_btc_test_chain_data
    c = get_btc_test_chain_data()
    p = {k: v for k, v in HawkesJDParams().to_dict().items() if k != "risk_premia_gamma"}
    return p, c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms


def _bump(p, name, h):
    up, dn = dict(p), dict(p)
    up[name] += h
    dn[name] -= h
    return up, dn


def _step(p, name, rel=1e-6):
    return rel * max(1.0, abs(p[name]))


def _rel(got, ref):
    return float(np.max(np.abs(got - ref))) / max(float(np.max(np.abs(ref))), 1.0)


@pytest.mark.parametrize("which", ["dflt", "alt"])
@pytest.mark.parametrize("spot", [True, False])
def test_second_order_rhs_vs_central_differences_of_the_tangent_rhs(which, spot):
    """d_ab f = J d2A + f_AA(dA_a, dA_b) + d_a J dA_b + d_b J dA_a + d_ab f against
    [T_a(p + h e_b; A + h dA_b, dA_a + h d2A) - T_a(p - h e_b; A - h dA_b, dA_a - h d2A)] / 2h, T_a = oracle.hawkes_greeks.HawkesTangentRhs,
    for every ODE pair at random A, dA_a, dA_b, d2A; the first-order parts reproduce T_a and T_b.  Step 1e-7 max(1, |x|): the bump moves z by
    beta h dA with beta ~ 100 and |dA| ~ 1, and at 1e-6 the O(h^2) term of the jump MGF's third derivative reaches 5.5e-7 (measured at
    1e-7: 2.8e-8)"""
    p = _golden_case(which)[0]
    phi = mgf.phi_grid(0.13, spot, hawkes.MAX_PHI)[::37]
    psi = np.zeros_like(phi)
    rng = np.random.default_rng(11)
    cn = lambda *s: rng.standard_normal(s) + 1j * rng.standard_normal(s)
    A, dAa, dAb, d2A = 0.05 * cn(phi.shape[0], 3), cn(phi.shape[0], 3), cn(phi.shape[0], 3), cn(phi.shape[0], 3)
    for a, b in MH.pairs(len(O.NAMES)):
        na, nb = O.NAMES[a], O.NAMES[b]
        if na not in HG.ODE_NAMES or nb not in HG.ODE_NAMES:
            continue
        fa, fb, fab = O.tan2_rhs(p, a, b, phi, A, dAa, dAb, d2A)
        assert _rel(fa, HG.HawkesTangentRhs(p, na, phi, psi)(A, dAa)) < 1e-12, (na, nb)
        assert _rel(fb, HG.HawkesTangentRhs(p, nb, phi, psi)(A, dAb)) < 1e-12, (na, nb)
        h = _step(p, nb, 1e-7)
        up, dn = _bump(p, nb, h)
        cd = (HG.HawkesTangentRhs(up, na, phi, psi)(A + h * dAb, dAa + h * d2A)
              - HG.HawkesTangentRhs(dn, na, phi, psi)(A - h * dAb, dAa - h * d2A)) / (2 * h)
        assert _rel(fab, cd) <= 1e-7, (na, nb, _rel(fab, cd))


@pytest.fixture(scope="module", params=["dflt", "alt"])
def case(request):
    p, ttms, fw, df, K, T = _golden_case(request.param)
    return request.param, (p, ttms, fw, df, K, T), O.hawkes_chain_hessian(p, ttms, fw, df, K, T)


def _pinned(p, ttms):
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    return vs, mgf.phi_grid(vs, True, hawkes.MAX_PHI)


def test_hyper_dual_first_parts_are_the_first_order_tangents(case):
    """the d1 parts of the hyper-dual replay reproduce oracle.hawkes_greeks' tangents on the recorded mesh, every row"""
    _, (p, ttms, *_), (_, grids) = case
    _, phi = _pinned(p, ttms)
    d1 = O.hawkes_d2_log_mgf(p, grids["meshes"], phi)[1]
    for r, (a, _) in enumerate(O.PAIRS):
        assert _rel(d1[r], grids["dlog_mgf"][a]) < 1e-12, O.NAMES[a]


@pytest.mark.parametrize("spot", [True, False])
def test_hyper_dual_replay_vs_central_differences_on_the_same_mesh(case, spot):
    """d2 log_mgf of all 120 pairs and the chain's Hessian rows against central differences in b of the first-order tangents and
    rows stepped on the same recorded meshes (measured <= 5.2e-9 over both); the lambda-lambda rows are zero"""
    which, (p, ttms, fw, df, K, T), (out, grids) = case
    vs, phi = _pinned(p, ttms)
    d2lm, meshes = grids["d2log_mgf"], grids["meshes"]
    types = T if spot else [np.array(["IP", "P", "C", "IC", "C"])] * 3
    rows = O.chain_rows(p, phi, grids["log_mgf"], grids["dlog_mgf"], d2lm, fw, df, K, types, spot)
    for b, nb in enumerate(O.NAMES):
        h = _step(p, nb)
        up, dn = _bump(p, nb, h)
        (au, lu), (ad, ld) = O.hawkes_tangents_on_meshes(up, meshes, phi), O.hawkes_tangents_on_meshes(dn, meshes, phi)
        lm = lambda q, a: a[:, :, 0] + a[:, :, 1] * q["lambda_p"] + a[:, :, 2] * q["lambda_m"]
        fu = [G.vanilla_slice_greeks(lm(up, au)[m], lu[:, m], phi, fw[m], K[m], types[m], df[m], spot) for m in range(3)]
        fd = [G.vanilla_slice_greeks(lm(dn, ad)[m], ld[:, m], phi, fw[m], K[m], types[m], df[m], spot) for m in range(3)]
        for a in range(len(O.NAMES)):
            r = O.PAIRS.index((min(a, b), max(a, b)))
            cd = (lu[a] - ld[a]) / (2 * h)
            assert _rel(d2lm[r], cd) <= 1e-7, (which, O.NAMES[a], nb, _rel(d2lm[r], cd))
            for m in range(3):
                cdr = (fu[m][3 + a] - fd[m][3 + a]) / (2 * h)
                assert _rel(rows[m][1][r], cdr) <= 1e-7, (which, spot, O.NAMES[a], nb, m)
    for a, b in (("lambda_p", "lambda_p"), ("lambda_p", "lambda_m"), ("lambda_m", "lambda_m")):
        assert not np.any(d2lm[O.PAIRS.index((O.NAMES.index(a), O.NAMES.index(b)))])


@pytest.mark.parametrize("spot", [True, False])
def test_vanna_vs_central_differences_in_the_forward(case, spot):
    """vanna against central differences in F of the first-order parameter rows (the mesh does not depend on F; measured <= 4.3e-9)"""
    which, (p, ttms, fw, df, K, T), (_, grids) = case
    vs, phi = _pinned(p, ttms)
    types = T if spot else [np.array(["IP", "P", "C", "IC", "C"])] * 3
    rows = O.chain_rows(p, phi, grids["log_mgf"], grids["dlog_mgf"], grids["d2log_mgf"], fw, df, K, types, spot)
    for m in range(3):
        h = 1e-5 * fw[m]
        fp, fm = fw.copy(), fw.copy()
        fp[m] += h
        fm[m] -= h
        up = HG.hawkes_chain_greeks(p, ttms, fp, df, K, types, spot, vs)[0][m]
        dn = HG.hawkes_chain_greeks(p, ttms, fm, df, K, types, spot, vs)[0][m]
        assert _rel(rows[m][0], (up[3:] - dn[3:]) / (2 * h)) <= 1e-7, (which, spot, m)


# gap between the scheme-exact Hessian and central differences (step 1e-6 max(1, |x|)) of the first-order rows of the ADAPTIVE oracle
# pricer (mesh re-chosen at every bump, grid pinned): the derivative of the step-size control's mesh choice.  Relative to max(1, max |cd|)
# over all 120 rows and every maturity; measured figure in the comment.  It bounds the GPU check of the public route.
HAWKES_HESSIAN_ADAPTIVE_GAP = {"hawkes": 2e-3,        # measured 7.9e-4 ("alt", spot), 6.2e-4 ("alt", inverse), 1.3e-4 ("dflt")
                               "btc": 4e-3}           # measured 1.5e-3 (default parameters, spot measure)


def adaptive_gap(chain_name, spot=True, which="dflt"):
    """max over rows and maturities of |hessian - cd(first-order rows of the adaptive oracle)| / max(1, |cd|)"""
    p, ttms, fw, df, K, T = _golden_case(which) if chain_name == "hawkes" else _btc_case()
    if not spot:
        T = [np.where(np.asarray(t) == "C", "IC", "IP") for t in T]
    vs = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    out = O.hawkes_chain_hessian(p, ttms, fw, df, K, T, spot, vs)[0]
    gap = 0.0
    for b, nb in enumerate(O.NAMES):
        h = _step(p, nb)
        up, dn = _bump(p, nb, h)
        gu = HG.hawkes_chain_greeks(up, ttms, fw, df, K, T, spot, vs)[0]
        gd = HG.hawkes_chain_greeks(dn, ttms, fw, df, K, T, spot, vs)[0]
        for a in range(len(O.NAMES)):
            r = O.PAIRS.index((min(a, b), max(a, b)))
            for m in range(len(ttms)):
                gap = max(gap, _rel(out[m][2][r], (gu[m][3 + a] - gd[m][3 + a]) / (2 * h)))
    return gap


def test_gap_to_central_differences_of_the_adaptive_pricer():
    assert adaptive_gap("hawkes", which="alt") <= HAWKES_HESSIAN_ADAPTIVE_GAP["hawkes"]


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

    monkeypatch.setattr(engine, "hawkesjd_price_chain_hessian", boom)
    params = sv.HawkesJDParams(risk_premia_gamma=kwargs.pop("risk_premia_gamma", None))
    if "variable_type" in kwargs:
        kwargs = dict(variable_type=sv.VariableType.Q_VAR)
    with pytest.raises(NotImplementedError, match="price_chain_hessian"):
        sv.HawkesJDPricer().price_chain_hessian(_chain(), params, **kwargs)


def test_result_layout_follows_hawkes_greek_params(monkeypatch):
    """a fake engine returns rows whose value encodes their index: the result maps them to HAWKES_GREEK_PARAMS, the upper triangle in that
    order, fills hessian[q][p] with the same arrays as hessian[p][q], and forwards the measure, vol_scaler and the 500-point grid"""
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    names = sv.HAWKES_GREEK_PARAMS
    assert names == O.NAMES
    n, J, seen = len(names), 15, {}

    def fake(params, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, vol_scaler=None, max_phi=None):
        seen.update(vol_scaler=vol_scaler, spot=is_spot_measure, max_phi=max_phi)
        greeks = np.arange(2 + n)[:, None] * 10.0 + np.zeros(J)
        vanna = 100.0 + np.arange(n)[:, None] + np.zeros(J)
        hess = 1000.0 + np.arange(n * (n + 1) // 2)[:, None] + np.arange(J) * 0.001
        return [np.zeros(5)] * 3, greeks, vanna, hess, np.array([0, 5, 10, 15])

    monkeypatch.setattr(engine, "hawkesjd_price_chain_hessian", fake)
    res = sv.HawkesJDPricer().price_chain_hessian(_chain(), sv.HawkesJDParams(), is_spot_measure=False, vol_scaler=0.11)
    assert isinstance(res, sv.FourierChainHessian)
    assert seen == dict(vol_scaler=0.11, spot=False, max_phi=500)
    assert tuple(res.params) == tuple(res.vanna) == tuple(res.hessian) == names
    r = 0
    for i, p in enumerate(names):
        assert np.all(res.params[p][1] == 10.0 * (2 + i)) and np.all(res.vanna[p][2] == 100.0 + i)
        for q in names[i:]:
            assert res.hessian[p][q] is res.hessian[q][p]
            np.testing.assert_array_equal(res.hessian[p][q][1], 1000.0 + r + np.arange(5, 10) * 0.001)
            r += 1
