"""GPU checks of ``HawkesJDPricer.price_chain_greeks`` (forward-mode Fourier sensitivities, DESIGN.md §4.3) against ``price_chain``, the
numpy forward mode of oracle/hawkes_greeks.py and central differences of the public pricer, on both parameter sets and the three carried
maturities of hawkes_fourier.npz."""
import dataclasses

import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes_greeks as H

pytestmark = pytest.mark.gpu


def _case(which):
    from stochvolmodels_b200 import HawkesJDParams, OptionChain
    g = load_golden("hawkes_fourier.npz")
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g[f"{which}_params"])))
    chain = OptionChain(ttms=g["ttms"], forwards=g["forwards"], strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["types"]] * 3,
                        discfactors=g["discfactors"])
    return p, HawkesJDParams(**p), chain


def _rel_close(got, ref, rtol, what):
    scale = max(float(np.max(np.abs(ref))), 1e-300)
    err = float(np.max(np.abs(got - ref))) / scale
    assert err <= rtol, (what, err)


# (parameter set, is_spot_measure, vol_scaler)
CASES = {"dflt_spot": ("dflt", True, None), "dflt_inverse": ("dflt", False, None), "alt_spot": ("alt", True, None),
         "alt_inverse": ("alt", False, None), "alt_pinned_grid": ("alt", True, 0.1)}


@pytest.mark.parametrize("case", list(CASES))
def test_hawkes_greeks_vs_price_chain_and_oracle(cuda_lib, case):
    from stochvolmodels_b200 import HawkesJDPricer, engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    which, spot, vs = CASES[case]
    p, params, chain = _case(which)
    pc = _params_c(**p)
    args = (pc, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    prices, greeks, offsets, dlm, nfev = engine.hawkesjd_price_chain_greeks(*args, is_spot_measure=spot, vol_scaler=vs, return_grids=True)
    again = engine.hawkesjd_price_chain_greeks(*args, is_spot_measure=spot, vol_scaler=vs, return_grids=True)
    ref = HawkesJDPricer().price_chain(chain, params, is_spot_measure=spot, vol_scaler=vs)
    public = HawkesJDPricer().price_chain_greeks(chain, params, is_spot_measure=spot, vol_scaler=vs)
    for m in range(3):
        np.testing.assert_array_equal(prices[m], ref[m])
        np.testing.assert_array_equal(again[0][m], prices[m])
        np.testing.assert_array_equal(public.prices[m], prices[m])
    np.testing.assert_array_equal(again[1], greeks)
    np.testing.assert_array_equal(again[3], dlm)
    np.testing.assert_array_equal(again[4], nfev)
    out, grids = H.hawkes_chain_greeks(p, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                       is_spot_measure=spot, vol_scaler=vs)
    np.testing.assert_array_equal(nfev, grids["nfev"])           # the same mesh at every grid point
    for d in range(15):
        for m in range(3):
            _rel_close(dlm[d, m], grids["dlog_mgf"][d, m], 1e-10, (case, "dlog_mgf", H.HAWKES_NAMES[d], m))
    for m in range(3):
        sl = slice(offsets[m], offsets[m + 1])
        for r in range(17):
            _rel_close(greeks[r, sl], out[m][1 + r], 1e-10, (case, "row", r, m))


def _cd_forward(price, chain, m, h=1e-4):
    from stochvolmodels_b200 import OptionChain

    def bumped(f):
        fw = chain.forwards.copy()
        fw[m] *= f
        return price(OptionChain(ttms=chain.ttms, forwards=fw, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                                 discfactors=chain.discfactors))[m]
    hh = h * chain.forwards[m]
    p0, pp, pm = price(chain)[m], bumped(1 + h), bumped(1 - h)
    return (pp - pm) / (2 * hh), (pp - 2 * p0 + pm) / (hh * hh)


@pytest.mark.parametrize("which,spot", [("dflt", True), ("alt", True), ("alt", False)])
def test_hawkes_public_greeks_vs_central_differences(cuda_lib, which, spot):
    """delta / gamma against central differences of price_chain in the forwards; parameters against central differences with the
    transform grid pinned, within the gap the CPU oracle measures (the derivative of the adaptive mesh choice)"""
    from test_hawkes_greeks_oracle import ADAPTIVE_GAP
    from stochvolmodels_b200 import HawkesJDPricer
    p, params, chain = _case(which)
    pricer = HawkesJDPricer()
    vs = float(np.clip(params.sigma, 0.2, 0.5) * np.sqrt(min(np.min(chain.ttms), 1.0 / 12.0)))
    g = pricer.price_chain_greeks(chain, params, is_spot_measure=spot)
    price = lambda c, q=params: pricer.price_chain(c, q, is_spot_measure=spot, vol_scaler=vs)
    for m in range(3):
        d_cd, g_cd = _cd_forward(price, chain, m)
        np.testing.assert_allclose(g.delta[m], d_cd, rtol=0, atol=1e-7)
        np.testing.assert_allclose(g.gamma[m], g_cd, rtol=0, atol=2e-4 * max(1.0, np.max(np.abs(g_cd))))
    for name in g.params:
        value = getattr(params, name)
        h = 1e-6 * max(1.0, abs(value))
        up = price(chain, dataclasses.replace(params, **{name: value + h}))
        dn = price(chain, dataclasses.replace(params, **{name: value - h}))
        for m in range(3):
            cd = (up[m] - dn[m]) / (2 * h)
            assert np.max(np.abs(g.params[name][m] - cd)) <= ADAPTIVE_GAP * max(1.0, np.max(np.abs(cd))), (name, m)


def test_hawkes_greeks_empty_chain(cuda_lib):
    """a chain without strikes: no sums, the grids still come back and match a chain with strikes"""
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    p, _, chain = _case("dflt")
    pc = _params_c(**p)
    empty = [np.array([])] * 3
    prices, greeks, offsets, dlm, nfev = engine.hawkesjd_price_chain_greeks(pc, chain.ttms, chain.forwards, chain.discfactors, empty, empty,
                                                                           return_grids=True)
    full = engine.hawkesjd_price_chain_greeks(pc, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms,
                                              return_grids=True)
    assert greeks.shape == (17, 0) and all(len(x) == 0 for x in prices)
    np.testing.assert_array_equal(dlm, full[3])
    np.testing.assert_array_equal(nfev, full[4])
