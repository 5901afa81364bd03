"""CPU checks of the second-order Fourier sensitivities (DESIGN.md §4.4): the numpy forward-over-forward restatement in
mgf_hessian_oracle.py against central differences of the first-order forward mode, the gap to differences of the adaptive pricer, and the
public methods' argument checks and result layout.  The measured adaptive-pricer gaps are quoted next to their bounds."""
import numpy as np
import pytest

import mgf_hessian_oracle as H
from oracle import mgf
from oracle import mgf_greeks as G

Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                 # the quickstart parameters
K = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T = np.array(["P", "P", "C", "C", "C"])
TI = np.array(["IP", "P", "C", "IC", "C"])
HESTON = (0.04, 0.05, 3.0, -0.6, 0.5)
TTMS2, FWD2, DF2 = np.array([0.1, 0.25]), np.array([1.0, 1.02]), np.array([0.99, 0.98])


def _bump(q, i, h):
    qp, qm = list(q), list(q)
    qp[i] += h
    qm[i] -= h
    return qp, qm


def _rel(got, ref):
    return float(np.max(np.abs(got - ref))) / max(float(np.max(np.abs(ref))), 1.0)


def test_hyper_dual_first_parts_are_the_first_order_tangents():
    """the d1 / d2 parts of the hyper-dual replay reproduce oracle.mgf_greeks' tangents on the recorded mesh"""
    vs = mgf.logsv_vol_scaler(Q[0], TTMS2)
    phi = mgf.phi_grid(vs)
    _, grids = G.logsv_chain_greeks(Q, TTMS2, FWD2, DF2, [K, K], [T, T], vol_scaler=vs)
    for p, q in ((1, 4), (0, 3)):
        A = H.logsv_d2_log_mgf(Q, TTMS2, grids["meshes"], phi, p=p, q=q)[1]
        y, y_p = Q[0] - Q[1], {0: 1.0, 1: -1.0}.get(p, 0.0)        # y = sigma0 - theta
        lm1 = sum(A[k].d1 * y ** k + A[k].v * (k * y ** (k - 1) * y_p if k else 0.0) for k in range(5))
        assert _rel(lm1, grids["dlog_mgf"][p, -1]) < 1e-12


# (is_spot_measure, order, etas): both measures, FIRST and SECOND order, eta != 1
ODE_CASES = {"spot": (True, 2, None), "inverse": (False, 2, None), "first_order": (True, 1, None), "eta": (True, 2, np.array([1.3, 0.8])),
             "inverse_eta": (False, 2, np.array([1.3, 0.8]))}


@pytest.mark.parametrize("case", list(ODE_CASES))
def test_second_order_tangents_vs_central_differences_of_first_order_tangents(case):
    """d2 log_mgf of every pair against central differences in q of the first-order tangents (oracle.mgf_greeks.LogsvTangentRhs) stepped
    on the same recorded meshes"""
    spot, order, etas = ODE_CASES[case]
    vs = mgf.logsv_vol_scaler(Q[0], TTMS2)
    phi = mgf.phi_grid(vs, spot)[::10]
    psi = np.zeros_like(phi)
    meshes = []
    a, da = np.zeros((phi.shape[0], mgf.expansion_n(order)), dtype=np.complex128), None
    t0 = 0.0
    for m, ttm in enumerate(TTMS2):      # record the meshes of the thinned grid
        rhs = mgf.LogsvRhs(*Q[1:], phi, psi, spot, order, 1.0 if etas is None else etas[m])
        f = G.logsv_fields(Q, 1.0 if etas is None else etas[m], spot)
        trhs = [G.LogsvTangentRhs(f, d, phi, psi, spot, order) for d in G.logsv_dfields(Q, 1.0 if etas is None else etas[m], spot)]
        da = np.zeros((5,) + a.shape, dtype=np.complex128) if da is None else da
        a, da, _, mesh = G.rk45_grid_tangent(rhs, trhs, a, da, ttm - t0)
        meshes.append(mesh)
        t0 = ttm
    h = 1e-5
    for r, (p, q) in enumerate(H.pairs(6)):
        d2 = H.logsv_d2_log_mgf(Q, TTMS2, meshes, phi, spot, order, etas, p, q)[0]
        qp, qm = _bump(Q, q, h)
        up = H.logsv_tangents_on_meshes(qp, TTMS2, meshes, phi, spot, order, etas)[2]
        dn = H.logsv_tangents_on_meshes(qm, TTMS2, meshes, phi, spot, order, etas)[2]
        cd = (up[p] - dn[p]) / (2 * h)
        assert _rel(d2, cd) < 1e-7, (case, G.LOGSV_NAMES[p], G.LOGSV_NAMES[q], _rel(d2, cd))


def test_heston_hyper_dual_vs_central_differences_of_the_dual_closed_form():
    """d2 log_mgf against central differences of oracle.mgf_greeks.heston_chain_greeks' dlog_mgf"""
    ttms, fwd, df = np.array([0.1, 0.5]), np.array([1.0, 1.02]), np.array([1.0, 0.99])
    strikes, types = [K, K * 1.02], [T, T]
    phi = mgf.phi_grid(0.1)
    h = 1e-6
    for p, q in H.pairs(5):
        d2 = H.heston_d2_log_mgf(HESTON, ttms, phi, p, q)
        qp, qm = _bump(HESTON, q, h)
        up = G.heston_chain_greeks(qp, ttms, fwd, df, strikes, types, vol_scaler=0.1)[1]
        dn = G.heston_chain_greeks(qm, ttms, fwd, df, strikes, types, vol_scaler=0.1)[1]
        assert _rel(d2, (up[p] - dn[p]) / (2 * h)) < 1e-7, (G.HESTON_NAMES[p], G.HESTON_NAMES[q])


@pytest.fixture(scope="module")
def two_maturities():
    vs = mgf.logsv_vol_scaler(Q[0], TTMS2)
    return vs, H.logsv_chain_hessian(Q, TTMS2, FWD2, DF2, [K, K], [T, T], vol_scaler=vs)


def _rows_on_meshes(q, meshes, vs, fwd=FWD2, spot=True, types=(T, T)):
    """first-order rows d price / d p on recorded meshes, through replay_tangent and oracle.mgf_greeks.vanilla_slice_greeks"""
    phi = mgf.phi_grid(vs, spot)
    a, _, dlm = H.logsv_tangents_on_meshes(q, TTMS2, meshes, phi, spot)
    yv = q[0] - q[1]
    ys = np.array([1.0, yv, yv * yv, yv ** 3, yv ** 4]) + 0j
    return [G.vanilla_slice_greeks(a[m] @ ys, dlm[:, m], phi, fwd[m], K, types[m], DF2[m], spot) for m in range(2)]


def test_chain_hessian_vs_central_differences_of_first_order_rows_on_fixed_meshes(two_maturities):
    """every Hessian row against central differences of the first-order parameter rows on the recorded meshes"""
    vs, (out, grids) = two_maturities
    h = 1e-5
    for r, (p, q) in enumerate(H.pairs(6)):
        qp, qm = _bump(Q, q, h)
        up, dn = _rows_on_meshes(qp, grids["meshes"], vs), _rows_on_meshes(qm, grids["meshes"], vs)
        for m in range(2):
            cd = (up[m][3 + p] - dn[m][3 + p]) / (2 * h)
            assert _rel(out[m][2][r], cd) < 1e-7, (G.LOGSV_NAMES[p], G.LOGSV_NAMES[q], m)


def test_the_two_orders_of_a_pair_agree(two_maturities):
    """the hyper-dual replay seeded (p, q) and (q, p), and the sigma0 rows' closed forms against the replay"""
    vs, (out, grids) = two_maturities
    phi = mgf.phi_grid(vs)
    for r, (p, q) in enumerate(H.pairs(6)):
        pq = H.logsv_d2_log_mgf(Q, TTMS2, grids["meshes"], phi, p=p, q=q)[0]
        if p != q:
            assert _rel(H.logsv_d2_log_mgf(Q, TTMS2, grids["meshes"], phi, p=q, q=p)[0], pq) < 1e-12
        assert _rel(grids["d2log_mgf"][r], pq) < 1e-10


@pytest.mark.parametrize("spot", [True, False])
def test_vanna_vs_central_differences_in_the_forward(spot):
    """vanna against central differences in F of the first-order parameter rows (the mesh does not depend on F)"""
    types = (T, T) if spot else (TI, TI)
    vs = mgf.logsv_vol_scaler(Q[0], TTMS2)
    out, grids = H.logsv_chain_hessian(Q, TTMS2, FWD2, DF2, [K, K], list(types), is_spot_measure=spot, vol_scaler=vs)
    for m in range(2):
        h = 1e-5 * FWD2[m]
        fp, fm = FWD2.copy(), FWD2.copy()
        fp[m] += h
        fm[m] -= h
        up = G.logsv_chain_greeks(Q, TTMS2, fp, DF2, [K, K], list(types), spot, vol_scaler=vs)[0][m]
        dn = G.logsv_chain_greeks(Q, TTMS2, fm, DF2, [K, K], list(types), spot, vol_scaler=vs)[0][m]
        assert _rel(out[m][1], (up[3:] - dn[3:]) / (2 * h)) < 1e-7, m


def test_heston_chain_rows_vs_central_differences():
    """Heston vanna and Hessian rows against central differences of the first-order rows (the closed form has no mesh)"""
    ttms, fwd, df = np.array([0.1, 0.5]), np.array([1.0, 1.02]), np.array([1.0, 0.99])
    strikes, types = [K, K * 1.02], [T, T]
    out = H.heston_chain_hessian(HESTON, ttms, fwd, df, strikes, types, vol_scaler=0.1)[0]
    h = 1e-6
    for r, (p, q) in enumerate(H.pairs(5)):
        qp, qm = _bump(HESTON, q, h)
        up = G.heston_chain_greeks(qp, ttms, fwd, df, strikes, types, vol_scaler=0.1)[0]
        dn = G.heston_chain_greeks(qm, ttms, fwd, df, strikes, types, vol_scaler=0.1)[0]
        for m in range(2):
            assert _rel(out[m][2][r], (up[m][3 + p] - dn[m][3 + p]) / (2 * h)) < 1e-7, (p, q, m)
    for m in range(2):
        hh = 1e-5 * fwd[m]
        fp, fm = fwd.copy(), fwd.copy()
        fp[m] += hh
        fm[m] -= hh
        up = G.heston_chain_greeks(HESTON, ttms, fp, df, strikes, types, vol_scaler=0.1)[0][m]
        dn = G.heston_chain_greeks(HESTON, ttms, fm, df, strikes, types, vol_scaler=0.1)[0][m]
        assert _rel(out[m][1], (up[3:] - dn[3:]) / (2 * hh)) < 1e-7, m


# gap between the scheme-exact Hessian and central differences of the first-order rows of the ADAPTIVE pricer (mesh re-chosen at every
# bump, grid pinned): the derivative of the step-size control's mesh choice.  Relative to max(1, max |cd|); measured figure in the comment.
HESSIAN_ADAPTIVE_GAP = {"quickstart": 3e-6,        # measured 6.4e-7
                        "btc": 1e-3}               # measured 3.6e-4 (spot measure), 3.7e-4 (inverse measure)


def _btc():
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS as b, get_btc_test_chain_data
    c = get_btc_test_chain_data()
    return (b.sigma0, b.theta, b.kappa1, b.kappa2, b.beta, b.volvol), c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms


def adaptive_gap(chain_name):
    """max over pairs and maturities of |hessian - cd(first-order rows of the adaptive oracle)| / max(1, |cd|)"""
    if chain_name == "quickstart":
        q, ttms, fwd, df, strikes, types = Q, np.array([0.25]), np.ones(1), np.ones(1), [K], [T]
    else:
        q, ttms, fwd, df, strikes, types = _btc()
    vs = mgf.logsv_vol_scaler(q[0], ttms)
    out = H.logsv_chain_hessian(q, ttms, fwd, df, strikes, types, vol_scaler=vs)[0]
    gap, h = 0.0, 1e-5
    for qi in range(6):
        qp, qm = _bump(q, qi, h)
        up = G.logsv_chain_greeks(qp, ttms, fwd, df, strikes, types, vol_scaler=vs)[0]
        dn = G.logsv_chain_greeks(qm, ttms, fwd, df, strikes, types, vol_scaler=vs)[0]
        for r, (p, qq) in enumerate(H.pairs(6)):
            if qq != qi:
                continue
            for m in range(len(ttms)):
                cd = (up[m][3 + p] - dn[m][3 + p]) / (2 * h)
                gap = max(gap, _rel(out[m][2][r], cd))
    return gap


def test_gap_to_central_differences_of_the_adaptive_pricer_quickstart():
    assert adaptive_gap("quickstart") <= HESSIAN_ADAPTIVE_GAP["quickstart"]


@pytest.mark.parametrize("method", ["price_chain_hessian"])
@pytest.mark.parametrize("kwargs", [dict(is_analytic=True), dict(is_stiff_solver=True), dict(use_rough_mc=True), dict(variable_type=2)])
def test_unsupported_kwargs_raise_before_the_engine(monkeypatch, kwargs, method):
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine

    def boom(*a, **k):
        raise AssertionError("engine called")

    monkeypatch.setattr(engine, "logsv_price_chain_hessian", boom)
    monkeypatch.setattr(engine, "heston_price_chain_hessian", boom)
    chain = sv.OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K], optiontypes_ttms=[T])
    if "variable_type" in kwargs:
        kwargs = dict(variable_type=sv.VariableType.Q_VAR)
    with pytest.raises(NotImplementedError, match=method):
        getattr(sv.LogSVPricer(), method)(chain, sv.LogSvParams(*Q), **kwargs)
    with pytest.raises(NotImplementedError, match=method):
        getattr(sv.HestonPricer(), method)(chain, sv.HestonParams(*HESTON), **kwargs)


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_result_layout_names_upper_triangle_and_symmetric_fill(monkeypatch, model):
    """a fake engine returns rows whose value encodes their index: the result maps them to names, the upper triangle in field order,
    and fills hessian[q][p] with the same arrays as hessian[p][q]"""
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine
    names = engine.LOGSV_GREEK_PARAMS if model == "logsv" else engine.HESTON_GREEK_PARAMS
    n, J = len(names), 7
    offsets = np.array([0, 3, 7])

    def fake(*a, **k):
        prices = [np.arange(3.0), np.arange(3.0, 7.0)]
        greeks = np.arange(2 + n)[:, None] * 10.0 + np.zeros(J)
        vanna = 100.0 + np.arange(n)[:, None] + np.zeros(J)
        hess = 1000.0 + np.arange(n * (n + 1) // 2)[:, None] + np.arange(J) * 0.001
        return prices, greeks, vanna, hess, offsets

    monkeypatch.setattr(engine, f"{model}_price_chain_hessian", fake)
    chain = sv.OptionChain(ttms=np.array([0.25, 0.5]), forwards=np.ones(2), strikes_ttms=[K[:3], K[:4]],
                           optiontypes_ttms=[T[:3], T[:4]])
    if model == "logsv":
        res = sv.LogSVPricer().price_chain_hessian(chain, sv.LogSvParams(*Q))
    else:
        res = sv.HestonPricer().price_chain_hessian(chain, sv.HestonParams(*HESTON))
    assert isinstance(res, sv.FourierChainHessian) and isinstance(res, sv.FourierChainGreeks)
    assert list(res.params) == list(names) and list(res.vanna) == list(names) and list(res.hessian) == list(names)
    assert np.all(res.delta[1] == 0.0) and np.all(res.gamma[0] == 10.0)
    r = 0
    for i, p in enumerate(names):
        assert np.all(res.params[p][1] == 10.0 * (2 + i))
        assert np.all(res.vanna[p][0] == 100.0 + i)
        for q in names[i:]:
            assert res.hessian[p][q] is res.hessian[q][p]
            np.testing.assert_array_equal(res.hessian[p][q][1], 1000.0 + r + np.arange(3, 7) * 0.001)
            r += 1
        assert list(res.hessian[p]) and set(res.hessian[p]) == set(names)
