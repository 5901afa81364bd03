"""GPU: the Black-76 inversion black.cuh::black_implied_vol against the exact implied vol of each fp64 quote (mpmath, 50 digits).

  - 3200 random quotes (|ln F/K| / (vol sqrt T) <= 9, vol in [0.01, 5], T in [3e-4, 10], C / P / IC / IP, D in [0.5, 1], F = 1 and
    67106.44) and constructed edges (K = F, 1 ulp inside each no-arbitrage bound and the bounds themselves, vols either side of the
    bracket [1e-8, 10], T = 1e-6 and 30, quotes down to 1e-300 F, invalid inputs), at the bar of tests/ivol_cases.py, A = 32;
  - NaN if and only if the quote is outside the strict no-arbitrage bounds, decided exactly;
  - the worst iteration count, read through the debug twin of the kernel (b200sv_debug_bsm_implied_vols), below the cap of 64;
  - every fused inversion (the LogSV / Heston Fourier batches, the cooperative and the multi-launch MC chains, the rough batch) returns
    exactly what b200sv_bsm_implied_vols gives for the prices the call returned, on a chain reaching far out-of-the-money puts.
"""
import numpy as np
import pytest

import ivol_cases as ic
from oracle import bsm

pytestmark = pytest.mark.gpu

pytest.importorskip("mpmath")


def _device(c):
    """one quote per slice through the debug twin; the product kernel must agree bit for bit"""
    from stochvolmodels_b200 import engine
    n = c["F"].size
    args = (c["T"], c["F"], c["D"], [c["K"][i:i + 1] for i in range(n)], [c["type"][i:i + 1] for i in range(n)],
            [c["price"][i:i + 1] for i in range(n)])
    iv, it = engine.debug_bsm_implied_vols(*args)
    np.testing.assert_array_equal(np.concatenate(engine.bsm_implied_vols(*args)), iv)
    return iv, it


def _assert_bar(name, iv, c):
    ratio, nan_mismatch, bad = ic.check(iv, c["iv_star"], c["bar"])
    print(f"{name}: {c['F'].size} quotes, {np.isnan(iv).sum()} NaN ({np.isnan(c['iv_star']).sum()} outside the bounds), "
          f"max |iv - iv*| / bar = {ratio:.2f} (A = {ic.A_BAR:g})")
    assert nan_mismatch.size == 0, [(c["type"][i], c["F"][i], c["K"][i], c["T"][i], c["D"][i], c["price"][i], iv[i]) for i in nan_mismatch[:5]]
    assert bad.size == 0, [(c["type"][i], c["F"][i], c["K"][i], c["T"][i], c["price"][i], iv[i], c["iv_star"][i]) for i in bad[:5]]


def test_grid_against_the_exact_implied_vol(cuda_lib):
    g = ic.random_grid()
    g["iv_star"], g["bar"] = ic.reference(g)
    iv, it = _device(g)
    _assert_bar("device, grid", iv, g)
    print(f"iterations: max {it.max()}, mean {it[np.isfinite(iv)].mean():.1f}")
    assert it.max() < bsm.MAX_ITER
    # what the call-side parity used to lose: out-of-the-money puts below 2e-17 F all come back finite
    otm_put = (g["K"] < g["F"]) & np.isin(g["type"], ("P", "IP")) & (g["price"] / g["D"] < 2e-17 * g["F"])
    assert otm_put.sum() >= 50 and np.all(np.isfinite(iv[otm_put]))


def test_constructed_edges(cuda_lib):
    e = ic.edge_cases()
    e["iv_star"], e["bar"] = ic.reference(e, "guess")
    iv, it = _device(e)
    _assert_bar("device, edges", iv, e)
    print(f"iterations: max {it.max()}")
    assert it.max() < bsm.MAX_ITER
    assert np.all(np.isnan(iv[e["tag"] == "invalid"])) and np.all(it[e["tag"] == "invalid"] == 0)
    # a root outside the bracket [1e-8, 10] returns the bracket's nearer end (to the rounding of s / sqrt T)
    out = np.isfinite(e["iv_star"]) & ((e["iv_star"] < bsm.VOL_LO) | (e["iv_star"] > bsm.VOL_HI))
    assert out.sum() >= 20
    np.testing.assert_allclose(iv[out], np.where(e["iv_star"][out] < 1.0, bsm.VOL_LO, bsm.VOL_HI), rtol=1e-15, atol=0)


def test_put_and_call_at_the_same_strike_and_vol_agree(cuda_lib):
    from stochvolmodels_b200 import engine
    pp = ic.parity_pairs()
    n = pp["F"].size
    iv = engine.bsm_implied_vols(pp["T"], pp["F"], pp["D"], [np.full(2, k) for k in pp["K"]], [np.array(["P", "C"])] * n,
                                 [np.array([p, c]) for p, c in zip(pp["put"], pp["call"])])
    for k in range(n):
        iv_star, bar = ic.exact(pp["F"][k], pp["K"][k], pp["T"][k], 1.0, pp["put"][k], "P")
        tol = ic.A_BAR * bar + 4.0 * np.spacing(iv_star)
        assert np.all(np.abs(iv[k] - iv_star) <= tol), (k, iv[k], iv_star, tol)
        assert abs(iv[k][0] - iv[k][1]) <= tol


# ---- the fused inversions --------------------------------------------------------------------------------------------------
TTMS, FW, DF = np.array([0.02, 0.25]), np.array([1.0, 1.03]), np.array([0.999, 0.98])
KS = np.array([0.25, 0.3, 0.4, 0.5, 0.6, 0.8, 0.9, 1.0, 1.1, 1.3, 1.6])
TS = np.array(["P", "P", "P", "IP", "P", "P", "IP", "C", "C", "IC", "C"])
STRIKES, TYPES = [KS, KS * 1.03], [TS, TS]
LOGSV = [(1.0, 1.0, 5.0, 5.0, 0.2, 2.0), (0.4, 0.45, 2.0, 2.5, -0.4, 0.8)]
HESTON = [(0.04, 0.04, 4.0, -0.5, 0.4), (0.09, 0.06, 2.0, -0.3, 0.6)]


def _assert_same_as_separate_inversion(name, prices, ivols, types=TYPES):
    from stochvolmodels_b200 import engine
    offsets = np.cumsum([0] + [k.size for k in STRIKES])
    for b in range(prices.shape[0]):
        split = [prices[b, offsets[m]:offsets[m + 1]] for m in range(len(STRIKES))]
        want = np.concatenate(engine.bsm_implied_vols(TTMS, FW, DF, STRIKES, types, split))
        np.testing.assert_array_equal(ivols[b], want, err_msg=name)
    tiny = (prices > 0) & (prices < 1e-8)
    print(f"{name}: {prices.size} prices, {tiny.sum()} in (0, 1e-8), {np.isfinite(ivols).sum()} finite ivols")


def test_fused_fourier_inversions_equal_the_chain_inversion(cuda_lib):
    from stochvolmodels_b200 import engine
    types = [np.char.replace(t, "I", "") for t in TYPES]           # the spot-measure Fourier routes price C / P only
    p, iv = engine.logsv_price_chain_batch([engine.logsv_params_c(*s) for s in LOGSV], TTMS, FW, DF, None, STRIKES, types)
    _assert_same_as_separate_inversion("logsv fourier batch", p, iv, types)
    p, iv = engine.heston_price_chain_batch([engine.heston_params_c(*s) for s in HESTON], TTMS, FW, DF, STRIKES, types)
    _assert_same_as_separate_inversion("heston fourier batch", p, iv, types)


def test_fused_mc_inversions_equal_the_chain_inversion(cuda_lib):
    """the finalize of the MC chain batches (the cooperative driver at this path count, the multi-launch one when
    B200SV_CHAIN_COOP=0) and the rough batch"""
    from stochvolmodels_b200 import engine
    flags = engine.mc_flags("fp64", "fp32")
    p, _, iv = engine.logsv_mc_chain_batch([engine.logsv_params_c(*s) for s in LOGSV], TTMS, FW, DF, None, STRIKES, TYPES, 50_000, 360,
                                           True, 5, flags)
    _assert_same_as_separate_inversion("logsv mc batch", p, iv)
    p, _, iv = engine.heston_mc_chain_batch([engine.heston_params_c(*s) for s in HESTON], TTMS, FW, DF, STRIKES, TYPES, 50_000, 360, 5, flags)
    _assert_same_as_separate_inversion("heston mc batch", p, iv)
    nsteps = np.maximum(np.round(TTMS * 200).astype(int), 1)
    p, _, iv, _, _ = engine.rough_logsv_mc_chain([engine.logsv_params_c(*s) for s in LOGSV], np.array([0.8, 0.35]), np.array([0.0015625, 1.316]),
                                                 TTMS, FW, DF, STRIKES, TYPES, 20_000, nsteps, TTMS / nsteps, seed=3, flags=flags, with_ivols=True)
    _assert_same_as_separate_inversion("rough mc batch", p, iv)


def test_fused_mc_inversions_on_the_multi_launch_driver(cuda_lib):
    import os
    import subprocess
    import sys
    from conftest import ROOT
    env = dict(os.environ, B200SV_CHAIN_COOP="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", os.path.join("tests", "test_gpu_ivol_edges.py"),
                        "-k", "test_fused_mc_inversions_equal_the_chain_inversion"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "1 passed" in r.stdout, r.stdout[-2000:]
