"""GPU pins of the Hawkes Fourier sensitivities, bit for bit: every output with ``return_grids=True`` of
``engine.hawkesjd_price_chain_greeks`` (with and without theta) and ``hawkesjd_price_chain_hessian`` under both measures, and of
``hawkesjd_price_chain_risk_premia_greeks`` / ``hawkesjd_price_chain_risk_premia_hessian`` at gamma in {0.4, -1, 0}, on both parameter
sets of hawkes_fourier.npz, on the BTC chain (default set) and on an empty chain.  That is prices, greeks, theta, vanna, hessian,
dlog_mgf, dlog_norm, d2log_mgf, d2log_norm and nfev.  The grids alone run to tens of megabytes, so the golden file holds, per output, a
sha256 over its dtype, shape and bytes: equal digests are equal arrays, bit for bit.

Run as a script to rewrite tests/golden/hawkes_fourier_sensitivities_pinned.npz."""
import hashlib
import os
import sys

import numpy as np
import pytest

if __name__ == "__main__":                   # run as a script: the package and the test helpers from this tree
    sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__))]

from test_hawkes_risk_premia_greeks_oracle import _golden_case  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hawkes_fourier_sensitivities_pinned.npz")
GAMMAS = (0.4, -1.0, 0.0)


def _chains():
    """(name, params dict, chain arguments) of every pinned chain"""
    from stochvolmodels_b200 import get_btc_test_chain_data
    out = []
    for which in ("dflt", "alt"):
        p, ttms, fw, df, K, T = _golden_case(which)
        out.append((which, p, (ttms, fw, df, K, T)))
    p, ttms, fw, df, _, _ = _golden_case("dflt")
    btc = get_btc_test_chain_data()
    out.append(("btc", p, (btc.ttms, btc.forwards, btc.discfactors, btc.strikes_ttms, btc.optiontypes_ttms)))
    out.append(("empty", p, (ttms, fw, df, [np.array([])] * len(ttms), [np.array([], dtype=str)] * len(ttms))))
    return out


def _flat(key, res, into):
    """every array of an engine result tuple under key|index; a list of per-maturity arrays is concatenated"""
    for i, v in enumerate(res):
        into[f"{key}|{i}"] = np.concatenate(v) if isinstance(v, list) else np.asarray(v)


def _digest(a: np.ndarray) -> np.ndarray:
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


def outputs():
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    out = {}
    for name, p, args in _chains():
        pc = _params_c(**p)
        for spot in (True, False):
            for theta in (False, True):
                _flat(f"{name}|greeks|spot={spot}|theta={theta}", engine.hawkesjd_price_chain_greeks(
                    pc, *args, is_spot_measure=spot, return_grids=True, with_theta=theta), out)
            _flat(f"{name}|hessian|spot={spot}", engine.hawkesjd_price_chain_hessian(pc, *args, is_spot_measure=spot, return_grids=True),
                  out)
        for gamma in GAMMAS:
            _flat(f"{name}|rp_greeks|gamma={gamma}", engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *args, return_grids=True),
                  out)
            _flat(f"{name}|rp_hessian|gamma={gamma}", engine.hawkesjd_price_chain_risk_premia_hessian(pc, gamma, *args, return_grids=True),
                  out)
    return {k: _digest(v) for k, v in out.items()}


@pytest.mark.gpu
def test_hawkes_fourier_sensitivities_pinned(cuda_lib):
    got = outputs()
    with np.load(GOLDEN) as g:
        assert sorted(g.files) == sorted(got)
        changed = [k for k in g.files if not np.array_equal(g[k], got[k])]
    assert not changed, changed


if __name__ == "__main__":
    res = outputs()
    np.savez_compressed(GOLDEN, **res)
    print(f"wrote {len(res)} arrays to {GOLDEN}")
