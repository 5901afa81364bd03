"""Pathwise sensitivities of the rough-vol route against the alternatives (DESIGN.md §3.10, §8): BTC chain with the reference's regression
parameters (H = 0.1, three factors, 360 steps per year), engine level with host buffers, median of 5 calls after one warm-up each:
  greeks   -- engine.rough_logsv_mc_chain_greeks (prices, delta and the 6 parameter rows with standard errors, one pass)
  price    -- engine.rough_logsv_mc_chain with one parameter set (what model_mc_price_chain(use_rough_mc=True) runs)
  crn13    -- engine.rough_logsv_mc_chain with the 13 sets of a central bump-and-reprice (base + 2 x 6 bumps) in one call
Two cases: 1e5 paths on the RandomState normals, 1e6 paths with in-kernel Philox fp32 draws.  Each host-level call uploads its normals
(250 MB in the first case), so next to the wall times the script reports the GPU kernel time of one call (torch.profiler, the host-to-device
copies and memsets excluded): the cost of the three alternatives on normals that are already on the device.  One JSON line per case with
the card name and power limit read in the same run.
   python tools/bench_rough_greeks.py"""
import json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from stochvolmodels_b200 import engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.logsv_pricer import get_randoms_for_rough_vol_chain_valuation
from stochvolmodels_b200.utils.funcs import set_time_grid

# the reference's regression fixture for this route (tests/golden/rough_mc_reference_regression.npz)
PARAMS = (0.377, 0.347, 1.29, 1.93, 2.45, 1.81)
WEIGHTS = np.array([0.77718798, 1.5545139, 8.51550426])
NODES = np.array([7.71995736e-02, 5.19154220e+00, 1.08459557e+02])
NPY, SEED = 360, 10


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def kernel_ms(fn):
    """sum of the GPU kernel durations of one call (copies and memsets excluded), after a warm-up call"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if e.key.startswith("Memcpy") or e.key.startswith("Memset"):
            continue
        us += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    return us / 1e3 if us > 0.0 else None


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


def crn_sets():
    out = [PARAMS]
    for k in range(6):
        for s in (1.0, -1.0):
            p = list(PARAMS)
            p[k] += s * 1e-4 * max(abs(p[k]), 1e-2)
            out.append(tuple(p))
    return [engine.logsv_params_c(*p) for p in out]


def case(chain, nb_path, gauss):
    grids = [set_time_grid(t, NPY)[2] for t in chain.ttms]
    nsteps, hs = [g.size - 1 for g in grids], [float(g[1] - g[0]) for g in grids]
    Z0 = Z1 = None
    if gauss is None:
        Z0, Z1, _ = get_randoms_for_rough_vol_chain_valuation(chain.ttms, nb_path, NPY, SEED)
    flags = engine.mc_flags("fp64", gauss or "fp32")
    pc = engine.logsv_params_c(*PARAMS)
    ch = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    sets = crn_sets()
    calls = {"greeks": lambda: engine.rough_logsv_mc_chain_greeks(pc, WEIGHTS, NODES, *ch, nb_path, nsteps, hs, Z0, Z1, 1, SEED, flags),
             "price": lambda: engine.rough_logsv_mc_chain([pc], WEIGHTS, NODES, *ch, nb_path, nsteps, hs, Z0, Z1, 1, SEED, flags),
             "crn13": lambda: engine.rough_logsv_mc_chain(sets, WEIGHTS, NODES, *ch, nb_path, nsteps, hs, Z0, Z1, 1, SEED, flags)}
    g, p, b = (timed(calls[k]) for k in ("greeks", "price", "crn13"))
    kern = {f"{k}_kernel_ms": kernel_ms(fn) for k, fn in calls.items()}
    return {"workload": f"rough LogSV MC (H = 0.1, 3 factors), BTC chain 4 maturities x 49 strikes, {nb_path:.0e} paths, {NPY} steps/year, "
                        + ("RandomState normals" if gauss is None else f"Philox {gauss}"),
            "greeks_ms": 1e3 * g, "price_ms": 1e3 * p, "crn13_ms": 1e3 * b, "greeks_over_price": g / p, "greeks_over_crn13": g / b, **kern,
            "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}


if __name__ == "__main__":
    chain = get_btc_test_chain_data()
    for nb_path, gauss in ((100_000, None), (1_000_000, "fp32")):
        print(json.dumps(case(chain, nb_path, gauss)), flush=True)
