"""Re-derive HAWKES_MC_ALLOWANCE of tests/test_gpu_hawkes_mc_greeks.py (CPU only, numpy oracles): on the hawkes_mc.npz chain (two maturities,
its parameters, P P C C C strikes scaled by the forwards) the Monte Carlo rows of oracle/hawkes_mc_greeks.py (1800 steps per year, the
route's Euler scheme, pathwise + score) against the exact Fourier sensitivities of oracle/hawkes_greeks.py, on RandomState draws in
batches.  Per row it prints max over the 10 options of |MC - Fourier| + 4 SE: an upper bound on the Euler scheme's bias in that row, which
the GPU gate allows on top of 4.5 SE of its own.
   python tools/hawkes_mc_greeks_allowance.py [paths_per_batch] [batches]        (~10 minutes at the defaults)"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import hawkes, hawkes_greeks as fg, hawkes_mc_greeks as hg        # noqa: E402

NAMES = ("delta",) + hg.PARAMS


def chain():
    g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "hawkes_mc.npz"))
    p = dict(zip(hawkes.KEYS, (float(v) for v in g["chain_params"])))
    ttms, fw, df = g["chain_ttms"], g["chain_forwards"], g["chain_discfactors"]
    return p, ttms, fw, df, [g["chain_strikes"] * f for f in fw], [g["chain_types"]] * ttms.size


def main(n_paths=100_000, batches=4):
    p, ttms, fw, df, K, T = chain()
    four = fg.hawkes_chain_greeks(p, ttms, fw, df, K, T)[0]                   # per maturity [prices, delta, gamma, 15 params] ([18, J])
    runs = []
    for b in range(batches):
        rng, t0, inputs = np.random.RandomState(200 + b), 0.0, []
        for ttm in ttms:
            inputs.append(hawkes.draw_inputs(rng, ttm - t0, n_paths, p["shift_p"], p["mean_p"], p["shift_m"], p["mean_m"]))
            t0 = ttm
        runs.append(hg.chain_greeks_fixed(p, ttms, fw, df, K, T, inputs))
    gap, z = np.zeros(len(NAMES)), np.zeros(len(NAMES))
    for m in range(ttms.size):
        mc = np.mean([r[2][m] for r in runs], axis=0)                           # [16, J]: delta, then the parameters
        se = np.mean([r[3][m] for r in runs], axis=0) / np.sqrt(batches)
        ref = np.vstack([four[m][1]] + [four[m][3 + k] for k in range(hg.NP)])
        gap = np.maximum(gap, np.max(np.abs(mc - ref) + 4.0 * se, axis=1))
        z = np.maximum(z, np.max(np.abs(mc - ref) / se, axis=1))
    for name, g, zz in zip(NAMES, gap, z):
        print(f"{name:9s} max |MC - Fourier| + 4 SE = {g:.3e}   (max |MC - Fourier| / SE = {zz:.2f})")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
