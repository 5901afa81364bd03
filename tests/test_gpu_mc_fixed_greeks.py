"""GPU: pathwise sensitivities of the LogSV chain on fixed normals resident in HBM (``logsv_mc_chain_greeks_fixed_randoms``, DESIGN.md §4.7).

  prices      -- bit-identical to logsv_mc_chain_pricer_fixed_randoms(DeviceRandoms, fast=True); two calls bit-identical
  sensitivity -- every row equals the forward-mode oracle (oracle/mc_greeks.py) on the same normals, and the central difference of the
                 fixed-normal pricer on the same DeviceRandoms
"""
import numpy as np
import pytest

from oracle import mc_greeks as mg

pytestmark = pytest.mark.gpu

PARAMS = (0.6, 0.5, 2.0, 2.5, -0.4, 1.2)
TTMS = np.array([0.1, 0.2, 0.35])
FW = np.array([1.0, 1.01, 1.03])
DF = np.array([0.999, 0.995, 0.99])
ETAS = np.array([0.9, 1.2, 1.1])


def _chain(variable_type):
    """three maturities, the middle one without strikes; all four payoff codes"""
    if variable_type == 2:
        k = np.array([0.2, 0.3, 0.4, 0.5])          # q / ttm ~ sigma^2 ~ 0.36
    else:
        k = np.array([0.85, 0.95, 1.0, 1.05, 1.2])
    t = np.array(["P", "IP", "C", "IC", "C"])[: k.size]
    return [k, np.zeros(0), k * 1.02], [t, np.array([], dtype=t.dtype), t[::-1].copy()]


def _randoms(nb_path, npy=180, seed=5):
    from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_chain_valuation
    return get_randoms_for_chain_valuation(TTMS, nb_path=nb_path, nb_steps_per_year=npy, seed=seed, device=True)


def _greeks(rnd, strikes, types, is_spot, vt, params=PARAMS):
    from stochvolmodels_b200.pricers.logsv_pricer import logsv_mc_chain_greeks_fixed_randoms
    return logsv_mc_chain_greeks_fixed_randoms(TTMS, FW, DF, strikes, types, rnd, v0=params[0], theta=params[1], kappa1=params[2],
                                               kappa2=params[3], beta=params[4], volvol=params[5], vol_backbone_etas=ETAS,
                                               is_spot_measure=is_spot, variable_type=vt)


def _prices(rnd, strikes, types, is_spot, vt, params=PARAMS, forwards=FW):
    from stochvolmodels_b200.pricers.logsv_pricer import logsv_mc_chain_pricer_fixed_randoms
    return logsv_mc_chain_pricer_fixed_randoms(TTMS, forwards, DF, strikes, types, rnd, v0=params[0], theta=params[1], kappa1=params[2],
                                               kappa2=params[3], beta=params[4], volvol=params[5], vol_backbone_etas=ETAS,
                                               is_spot_measure=is_spot, variable_type=vt, fast=True)


def _rows(res, m):
    """[1 + 6, J_m]: delta, then LOGSV_GREEK_PARAMS"""
    return np.vstack([res.delta[m]] + [res.params[n][m] for n in mg.LOGSV_PARAMS])


def _rows_se(res, m):
    return np.vstack([res.delta_se[m]] + [res.params_se[n][m] for n in mg.LOGSV_PARAMS])


CASES = [(True, 1), (False, 1), (True, 2), (False, 2)]


@pytest.mark.parametrize("is_spot,vt", CASES)
@pytest.mark.parametrize("nb_path", [1, 20_000])
def test_prices_equal_the_device_resident_pricer_bitwise(cuda_lib, is_spot, vt, nb_path):
    from stochvolmodels_b200.utils.config import VariableType
    variable_type = VariableType.LOG_RETURN if vt == 1 else VariableType.Q_VAR
    strikes, types = _chain(vt)
    rnd = _randoms(nb_path)
    res = _greeks(rnd, strikes, types, is_spot, variable_type)
    prices, stds = _prices(rnd, strikes, types, is_spot, variable_type)
    assert res.prices[1].size == 0 and res.delta[1].size == 0
    for m in range(3):
        np.testing.assert_array_equal(res.prices[m], prices[m])
        np.testing.assert_array_equal(res.std_errors[m], stds[m])
    again = _greeks(rnd, strikes, types, is_spot, variable_type)
    for m in range(3):
        np.testing.assert_array_equal(_rows(again, m), _rows(res, m))
        np.testing.assert_array_equal(_rows_se(again, m), _rows_se(res, m))
        np.testing.assert_array_equal(again.prices[m], res.prices[m])


def test_host_normals_give_the_device_randoms_results(cuda_lib):
    from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_chain_valuation, logsv_mc_chain_greeks_fixed_randoms
    strikes, types = _chain(1)
    W0s, W1s, dts = get_randoms_for_chain_valuation(TTMS, nb_path=3000, nb_steps_per_year=180, seed=5)
    host = logsv_mc_chain_greeks_fixed_randoms(TTMS, FW, DF, strikes, types, W0s, W1s, dts, *PARAMS, vol_backbone_etas=ETAS)
    dev = _greeks(_randoms(3000), strikes, types, True, 1)
    for m in range(3):
        np.testing.assert_array_equal(host.prices[m], dev.prices[m])
        np.testing.assert_array_equal(_rows(host, m), _rows(dev, m))


@pytest.mark.parametrize("is_spot,vt", CASES)
def test_every_row_matches_the_forward_mode_oracle(cuda_lib, is_spot, vt):
    """the oracle steps the same (downloaded) normals in numpy's strict order, the kernel in the fast stepper's contracted one: states
    differ by ~1e-14 relative, so each per-path term differs by ~1e-13 of its spread at most.  Bound: 1e-10 of the row's scale plus an
    absolute floor of 1e-11 of the term's standard deviation (SE * sqrt(N)), for rows whose mean cancels (e.g. kappa2 on short slices)."""
    N = 20_000
    strikes, types = _chain(vt)
    rnd = _randoms(N)
    res = _greeks(rnd, strikes, types, is_spot, vt)
    Z0s, Z1s = [w.cpu().numpy() for w in rnd.W0s], [w.cpu().numpy() for w in rnd.W1s]
    po, eo, go, _ = mg.logsv_mc_chain_greeks_fixed(PARAMS, TTMS, FW, DF, strikes, types, ETAS, Z0s, Z1s, rnd.dts, is_spot, vt)
    for m in (0, 2):
        np.testing.assert_allclose(res.prices[m], po[m], rtol=1e-12, atol=1e-15)
        got, want, se = _rows(res, m), np.asarray(go[m]), _rows_se(res, m)
        scale = np.max(np.abs(want), axis=1, keepdims=True)
        bound = 1e-10 * scale + 1e-11 * se * np.sqrt(N) + 1e-15
        assert np.all(np.abs(got - want) <= bound), (m, np.max(np.abs(got - want) / bound))


@pytest.mark.parametrize("is_spot,vt", CASES)
def test_every_row_matches_central_differences_of_the_fixed_normal_pricer(cuda_lib, is_spot, vt):
    """central differences of the fixed-normal pricer on the same DeviceRandoms, relative step h = 1e-5 (absolute for beta).  The sample
    price is piecewise smooth in each parameter: truncation is h^2/6 P''' (~1e-10 relative here); each path whose payoff switches branch
    inside [p - h, p + h] adds at most half its own |g| to the quotient and such paths are O(N h) of N, so their share of the mean is O(h)
    -- allowed as 0.1 SE, the gate of the Philox route's CRN test.  The last term is the fp64 round-off of the quotient: the bumped runs
    are one deterministic kernel, so prices carry ~1e-15 relative noise, i.e. 1e-13 |P| / h with margin."""
    from stochvolmodels_b200 import engine
    N = 200_000
    strikes, types = _chain(vt)
    rnd = _randoms(N)
    res = _greeks(rnd, strikes, types, is_spot, vt)

    def gate(m, g, se, up, dn, h, what):
        fd = (up[m] - dn[m]) / (2 * h)
        bound = 0.1 * se + 1e-13 * np.maximum(np.abs(up[m]), np.abs(dn[m])) / h
        assert np.all(np.abs(g - fd) <= bound), (what, m, g, fd, se)

    h = 1e-5
    up = _prices(rnd, strikes, types, is_spot, vt, forwards=FW * (1 + h))[0]
    dn = _prices(rnd, strikes, types, is_spot, vt, forwards=FW * (1 - h))[0]
    for m in (0, 2):
        gate(m, res.delta[m], res.delta_se[m], up, dn, h * FW[m], "delta")
    for k, name in enumerate(engine.LOGSV_GREEK_PARAMS):
        hp = 1e-5 if name == "beta" else 1e-5 * abs(PARAMS[k])
        bump = lambda s: tuple(v + s * hp if i == k else v for i, v in enumerate(PARAMS))
        up = _prices(rnd, strikes, types, is_spot, vt, params=bump(1))[0]
        dn = _prices(rnd, strikes, types, is_spot, vt, params=bump(-1))[0]
        for m in (0, 2):
            gate(m, res.params[name][m], res.params_se[name][m], up, dn, hp, name)
