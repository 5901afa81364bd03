"""CPU: the forward-mode oracle of the rough-vol route's pathwise sensitivities (oracle/rough_greeks.py) against central finite differences
of ``oracle.rough`` on fixed normals, and the argument checks of LogSVPricer.rough_mc_chain_greeks (they raise before any library call)."""
import numpy as np
import pytest

from oracle import mc, rough, rough_greeks as rg

BUMP = 1e-6
FACTORS = {1: (np.array([1.0]), np.array([1e-3])),
           2: (np.array([0.8, 0.35]), np.array([0.0015625, 1.316])),
           3: (np.array([0.97702551, 0.75117174, 1.66711921]), np.array([3.33333333e-02, 6.31209359e+00, 1.01078897e+02]))}
PARAMS = (0.6, 0.5, 2.0, 2.5, -0.4, 1.2)                 # sigma0, theta, kappa1, kappa2, beta, orthog_vol


def _step_h(x):
    return BUMP * max(abs(x), 1e-2)


def _assert_close(a, b, what, rtol=1e-7):
    """relative to the tangent array's scale"""
    scale = max(float(np.max(np.abs(b))), 1e-300)
    assert np.max(np.abs(a - b)) <= rtol * scale, (what, np.max(np.abs(a - b)) / scale)


def _primal(prm, w, x, ls, v, y, h, z0, z1):
    sigma0, theta, kappa1, kappa2, beta, ov = prm
    P = v.shape[1]
    vt = np.sqrt(beta ** 2 + ov ** 2)
    vol, yh, lsh = rough.step(np.repeat(x[:, None], P, axis=1), np.repeat(w[:, None], P, axis=1), np.full(v.shape, sigma0 / np.sum(w)), theta,
                              kappa1, kappa2, ls[None, :], v, y[None, :], beta / vt, vt, h, z0, z1)
    return vol, yh[0], lsh[0]


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("reset", [False, True])
def test_rough_tangent_step_matches_central_differences(n, reset):
    """one step from random states with random input tangents: the tangent = d/deps step(state + eps d, params + eps e_q) for every
    direction q; ``reset`` starts from states whose weighted vol the step drives through zero (reset-to-1e-6 branch, zero factor tangents)"""
    w, x = FACTORS[n]
    P, h = 64, 1.0 / 100
    rs = np.random.RandomState(n + 10 * reset)
    v0 = PARAMS[0] / np.sum(w)
    v = v0 * (0.5 + rs.uniform(size=(n, P)))
    if reset:
        v[:, : P // 2] = -1.0 - rs.uniform(size=(n, P // 2))
    ls, y = 0.1 * rs.normal(size=P), 0.05 * rs.uniform(size=P)
    dv, dls, dy = rs.normal(size=(6, n, P)), rs.normal(size=(6, P)), rs.normal(size=(6, P))
    z0, z1 = rs.normal(size=P), rs.normal(size=P)
    vol, yh, lsh, dvol, dyh, dlsh = rg.step_tangent(x, w, *PARAMS, ls, v, y, dls, dv, dy, h, z0, z1)
    ref = _primal(PARAMS, w, x, ls, v, y, h, z0, z1)
    for a, b in zip((vol, yh, lsh), ref):
        np.testing.assert_array_equal(a, b)                  # the tangent restatement leaves the state to oracle.rough.step
    bad = np.all(vol == 1e-6, axis=0)
    assert (bad.sum() > 0) == reset
    for q, name in enumerate(rg.PARAMS):
        eps = _step_h(PARAMS[q])
        def at(s):
            prm = list(PARAMS)
            prm[q] += s * eps
            return _primal(prm, w, x, ls + s * eps * dls[q], v + s * eps * dv[q], y + s * eps * dy[q], h, z0, z1)
        up, dn = at(1.0), at(-1.0)
        for t, a, b, var in zip((dvol[q], dyh[q], dlsh[q]), up, dn, ("vol", "qv", "log_spot")):
            _assert_close(t, (a - b) / (2 * eps), (name, var, n))
        if reset:
            assert np.all(dvol[q][:, bad] == 0.0)


K4 = np.array([0.85, 0.95, 1.05, 1.15])
TYPES = [np.array(["C", "P", "IC", "IP"]), np.array(["IP", "C", "P", "IC"])]
QK = np.array([0.2, 0.3, 0.4, 0.5])


def _fd_gate(g, se, fd, what):
    """pathwise vs CRN central difference within 0.1 of the sensitivity's standard error (plus fp64 round-off of the difference)"""
    assert np.all(np.abs(g - fd) <= 0.1 * se + 1e-9 * (1.0 + np.abs(g))), (what, g, fd, se)


@pytest.mark.parametrize("variable_type", [mc.LOG_RETURN, mc.Q_VAR])
def test_rough_chain_sensitivities_match_crn_differences(variable_type):
    N, npy = 2000, 100
    ttms, fw, df = np.array([0.1, 0.3]), np.array([1.0, 1.02]), np.array([0.999, 0.99])
    strikes = [QK, QK] if variable_type == mc.Q_VAR else [K4, K4 * 1.02]
    w, x = FACTORS[3]
    Z0, Z1, grids = rough.rough_randoms(ttms, N, npy, 7)
    p, e, g, gse, states = rg.rough_chain_greeks_fixed(ttms, fw, df, strikes, TYPES, Z0, Z1, *PARAMS, w, x, grids, variable_type,
                                                       return_states=True)
    price = lambda prm, f=fw: rough.rough_chain_fixed(ttms, f, df, strikes, TYPES, Z0, Z1, *prm, w, x, grids, variable_type)
    po, eo = price(PARAMS)
    for m in range(2):
        assert not np.any(states[m][6]), "a path resets at some step: the pathwise estimator would omit its mass"
        np.testing.assert_allclose(p[m], po[m], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(e[m], eo[m], rtol=1e-12, atol=1e-15)
    hf = 1e-6
    pu, pd = price(PARAMS, fw * (1 + hf))[0], price(PARAMS, fw * (1 - hf))[0]
    for m in range(2):
        _fd_gate(g[m][0], gse[m][0], (pu[m] - pd[m]) / (2 * hf * fw[m]), ("delta", m))
    for q, name in enumerate(rg.PARAMS):
        eps = _step_h(PARAMS[q])
        up, dn = list(PARAMS), list(PARAMS)
        up[q] += eps
        dn[q] -= eps
        pu, pd = price(up)[0], price(dn)[0]
        for m in range(2):
            _fd_gate(g[m][1 + q], gse[m][1 + q], (pu[m] - pd[m]) / (2 * eps), (name, m))


# ---- argument checks: nothing reaches the library ------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


@pytest.mark.parametrize("kwargs,exc", [(dict(precision="fp32", seed=1), NotImplementedError), (dict(exchange="p2p", seed=1), NotImplementedError),
                                        (dict(exchange="nccl", seed=1), NotImplementedError),
                                        (dict(gauss="fp64_paired", seed=1), NotImplementedError), (dict(), ValueError)])
def test_rough_greeks_rejections_raise_before_the_library(no_library, kwargs, exc):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K4], optiontypes_ttms=[TYPES[0]])
    p = LogSvParams(weights=FACTORS[3][0], nodes=FACTORS[3][1])
    with pytest.raises(exc):
        LogSVPricer().rough_mc_chain_greeks(chain, p, nb_path=1000, nb_steps=100, **kwargs)


def test_model_mc_chain_greeks_points_the_rough_route_to_its_own_method(no_library):
    from stochvolmodels_b200 import LogSvParams, LogSVPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K4], optiontypes_ttms=[TYPES[0]])
    with pytest.raises(NotImplementedError, match="rough_mc_chain_greeks"):
        LogSVPricer().model_mc_chain_greeks(chain, LogSvParams(), nb_path=1000, use_rough_mc=True, seed=1)


def test_oracle_reset_flag_sees_resets_that_do_not_last_to_maturity():
    """the per-path flag of path_tangents is OR-ed over the steps: on a coarse grid with doubled vol shocks paths reset and drift away
    from 1e-6 again, and the flag still counts them"""
    w, x = FACTORS[2]
    ttms = np.array([0.5])
    Z0, Z1, grids = rough.rough_randoms(ttms, 2000, 12, 77)
    st = rg.path_tangents(x, w, 0.5, 0.6, 1.0, 10.0, -0.3, 2.0, grids[0], 2.0 * Z0, Z1)
    terminal = np.all(st[1] == 1e-6, axis=0)
    assert st[6].sum() > terminal.sum() > 0
    assert np.all(st[6][terminal])
