"""CPU checks of the forward-mode Fourier sensitivities (DESIGN.md §4.2): the numpy restatement in oracle/mgf_greeks.py against central
differences, and the public methods' argument checks.  Measured figures (quickstart slice, 1000-point grid) are quoted next to each bound."""
import numpy as np
import pytest

from oracle import mgf
from oracle import mgf_greeks as G

Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                 # the quickstart parameters
K = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T = np.array(["P", "P", "C", "C", "C"])
TTMS, FWD, DF = np.array([0.25]), np.ones(1), np.ones(1)
HESTON = (0.04, 0.05, 3.0, -0.6, 0.5)


def _bump(q, i, h):
    qp, qm = list(q), list(q)
    qp[i] += h
    qm[i] -= h
    return qp, qm


@pytest.mark.parametrize("spot", [True, False])
@pytest.mark.parametrize("eta", [1.0, 1.3])
def test_model_field_table_vs_central_differences_of_mlh(spot, eta):
    phi = mgf.phi_grid(0.2, spot)[::97]
    psi = np.zeros_like(phi)
    for order in (1, 2):
        n = mgf.expansion_n(order)
        f = G.logsv_fields(Q, eta, spot)
        M0, L0, H0 = G.dense_mlh(f["v2"], f["qv"], f["qv2"], G.coef(f, phi, psi, spot), n)
        Mr, Lr = mgf.logsv_mlh(*Q[1:], phi[3], psi[3], spot, order, eta)[:2]
        assert np.array_equal(M0, Mr) and np.allclose(L0[3], Lr, rtol=1e-15, atol=1e-15)
        for d, df in enumerate(G.logsv_dfields(Q, eta, spot)):
            dM, dL, dH = G.dense_mlh(df["v2"], df["qv"], df["qv2"], G.dcoef(f, df, phi, psi, spot), n)
            h = 1e-6
            qp, qm = _bump(Q, 1 + d, h)
            for p in range(phi.shape[0]):
                Mp, Lp, Hp = mgf.logsv_mlh(*qp[1:], phi[p], psi[p], spot, order, eta)
                Mm, Lm, Hm = mgf.logsv_mlh(*qm[1:], phi[p], psi[p], spot, order, eta)
                for got, cd in ((dM, (Mp - Mm) / (2 * h)), (dL[p], (Lp - Lm) / (2 * h)), (dH[p], (Hp - Hm) / (2 * h))):
                    assert np.allclose(got, cd, rtol=0, atol=1e-7 * max(1.0, np.max(np.abs(cd)))), (d, p)


@pytest.fixture(scope="module")
def quickstart():
    return G.logsv_chain_greeks(Q, TTMS, FWD, DF, [K], [T])


def test_replay_and_tangent_integrator_reproduce_rk45_grid_bit_for_bit(quickstart):
    out, grids = quickstart
    phi = mgf.phi_grid(mgf.logsv_vol_scaler(Q[0], TTMS), True)
    rhs = mgf.LogsvRhs(*Q[1:], phi, np.zeros_like(phi), True, 2, 1.0)
    a0 = np.zeros((phi.shape[0], 5), dtype=np.complex128)
    a_ref, stats = mgf.rk45_grid(rhs, a0, 0.25, return_stats=True)
    assert np.array_equal(grids["a"][0], a_ref)
    assert np.array_equal(grids["nfev"], stats["nfev"])
    assert np.array_equal(G.replay(rhs, a0, grids["meshes"][0]), a_ref)
    assert np.array_equal(out[0][0], mgf.logsv_chain_prices(Q, TTMS, FWD, DF, [K], [T])[0])


def test_tangents_vs_central_differences_on_the_fixed_mesh(quickstart):
    """the exact derivative of the scheme: dA, dlog_mgf and d price agree with central differences of the replay (measured: prices
    2e-11 absolute, dA 1e-9 relative to the row scale)"""
    out, grids = quickstart
    vs = mgf.logsv_vol_scaler(Q[0], TTMS)
    for i in range(6):
        h = 1e-5
        qp, qm = _bump(Q, i, h)
        pp, lp = G.logsv_chain_prices_on_meshes(qp, TTMS, FWD, DF, [K], [T], grids["meshes"], vs)
        pm, lm = G.logsv_chain_prices_on_meshes(qm, TTMS, FWD, DF, [K], [T], grids["meshes"], vs)
        cd = (pp[0] - pm[0]) / (2 * h)
        assert np.max(np.abs(cd - out[0][3 + i])) < 1e-7 * max(1.0, np.max(np.abs(cd))), G.LOGSV_NAMES[i]
        dlm_cd = (lp - lm) / (2 * h)
        scale = np.max(np.abs(dlm_cd))
        assert np.max(np.abs(grids["dlog_mgf"][i] - dlm_cd)) < 1e-7 * max(scale, 1.0), G.LOGSV_NAMES[i]


# gap between the forward-mode sensitivities and central differences of the ADAPTIVE pricer (grid pinned): the derivative of the step-size
# control's mesh choice, which the scheme-exact tangents leave out.  Relative to max(1, max |cd|); the measured figure is in the comment.
ADAPTIVE_GAP = {"quickstart": 3e-7,        # measured 7.8e-8 (theta)
                "btc": 5e-5}               # measured 3.5e-5 (kappa2), 2.1e-5 (volvol), 6.1e-6 (kappa1), <= 1.7e-6 otherwise


def _btc():
    from stochvolmodels_b200 import LOGSV_BTC_PARAMS as b, get_btc_test_chain_data
    c = get_btc_test_chain_data()
    return (b.sigma0, b.theta, b.kappa1, b.kappa2, b.beta, b.volvol), c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms


@pytest.mark.parametrize("chain_name", list(ADAPTIVE_GAP))
def test_tangents_vs_central_differences_of_the_adaptive_pricer(quickstart, chain_name):
    if chain_name == "quickstart":
        q, ttms, fwd, df, strikes, types = Q, TTMS, FWD, DF, [K], [T]
        out = quickstart[0]
    else:
        q, ttms, fwd, df, strikes, types = _btc()
        out = G.logsv_chain_greeks(q, ttms, fwd, df, strikes, types)[0]
    vs = mgf.logsv_vol_scaler(q[0], ttms)
    for i in range(6):
        h = 1e-5
        qp, qm = _bump(q, i, h)
        pp = mgf.logsv_chain_prices(qp, ttms, fwd, df, strikes, types, vol_scaler=vs)
        pm = mgf.logsv_chain_prices(qm, ttms, fwd, df, strikes, types, vol_scaler=vs)
        for m in range(len(ttms)):
            cd = (pp[m] - pm[m]) / (2 * h)
            assert np.max(np.abs(cd - out[m][3 + i])) <= ADAPTIVE_GAP[chain_name] * max(1.0, np.max(np.abs(cd))), (G.LOGSV_NAMES[i], m)


@pytest.mark.parametrize("spot", [True, False])
def test_delta_gamma_vs_central_differences_in_the_forward(spot):
    types = np.array(["P", "P", "C", "C", "C"]) if spot else np.array(["IP", "P", "C", "IC", "C"])
    F, h = 1.05, 1e-4
    out, _ = G.logsv_chain_greeks(Q, TTMS, np.array([F]), np.array([0.97]), [K], [types], is_spot_measure=spot, vol_scaler=0.4)
    price = lambda f: mgf.logsv_chain_prices(Q, TTMS, np.array([f]), np.array([0.97]), [K], [types], spot, vol_scaler=0.4)[0]
    p0, pp, pm = price(F), price(F + h), price(F - h)
    assert np.allclose(out[0][0], p0, rtol=0, atol=1e-15)
    assert np.allclose(out[0][1], (pp - pm) / (2 * h), rtol=0, atol=1e-8)
    assert np.allclose(out[0][2], (pp - 2 * p0 + pm) / (h * h), rtol=0, atol=1e-5)


def test_heston_tangents_vs_central_differences():
    ttms, fwd, df = np.array([0.1, 0.5]), np.array([1.0, 1.02]), np.array([1.0, 0.99])
    strikes, types = [K, K * 1.02], [T, T]
    out, _ = G.heston_chain_greeks(HESTON, ttms, fwd, df, strikes, types, vol_scaler=0.1)
    for i in range(5):
        h = 1e-6
        qp, qm = _bump(HESTON, i, h)
        pp = mgf.heston_chain_prices(qp, ttms, fwd, df, strikes, types, vol_scaler=0.1)
        pm = mgf.heston_chain_prices(qm, ttms, fwd, df, strikes, types, vol_scaler=0.1)
        for m in range(2):
            cd = (pp[m] - pm[m]) / (2 * h)
            assert np.max(np.abs(cd - out[m][3 + i])) < 1e-7 * max(1.0, np.max(np.abs(cd))), (G.HESTON_NAMES[i], m)


@pytest.mark.parametrize("kwargs", [dict(is_analytic=True), dict(is_stiff_solver=True), dict(use_rough_mc=True),
                                    dict(variable_type=2)])
def test_unsupported_kwargs_raise_before_the_engine(monkeypatch, kwargs):
    import stochvolmodels_b200 as sv
    from stochvolmodels_b200 import engine

    def boom(*a, **k):
        raise AssertionError("engine called")

    monkeypatch.setattr(engine, "logsv_price_chain_greeks", boom)
    monkeypatch.setattr(engine, "heston_price_chain_greeks", boom)
    chain = sv.OptionChain(ttms=TTMS, forwards=FWD, strikes_ttms=[K], optiontypes_ttms=[T])
    if "variable_type" in kwargs:
        kwargs = dict(variable_type=sv.VariableType.Q_VAR)
    with pytest.raises(NotImplementedError):
        sv.LogSVPricer().price_chain_greeks(chain, sv.LogSvParams(*Q), **kwargs)
    with pytest.raises(NotImplementedError):
        sv.HestonPricer().price_chain_greeks(chain, sv.HestonParams(*HESTON), **kwargs)
