"""Re-derive H05_ALLOWANCE of tests/test_gpu_rough_greeks.py (CPU only, numpy oracles): at H = 1/2 (one node at 1e-3) the rough scheme's
pathwise rows (oracle/rough_greeks.py, 360 steps per year) against the LogSV Fourier sensitivities (oracle/mgf_greeks.py, second-order
expansion) on the chain of the test, 4 batches x 1e5 RandomState paths.  Per row it prints max over the 10 strikes of |MC - Fourier| + SE:
the gap the GPU gate allows on top of 4.5 SE (time-step bias of the Strang / RK4 scheme plus the expansion error of the Fourier route).
   python tools/rough_greeks_h05_allowance.py [paths_per_batch] [batches]        (~2 minutes at the defaults)"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mgf_greeks as fg, rough, rough_greeks as rg        # noqa: E402

TTMS, FW, DF = np.array([0.1, 0.25]), np.ones(2), np.ones(2)
K = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T = np.array(["P", "P", "C", "C", "C"])
PARAMS = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)                 # sigma0, theta, kappa1, kappa2, beta, volvol (the test's LogSvParams)
NAMES = ("delta", "sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")


def main(n_paths=100_000, batches=4, npy=360):
    four = fg.logsv_chain_greeks(PARAMS, TTMS, FW, DF, [K, K], [T, T])
    four = four[0] if isinstance(four, tuple) else four          # per maturity [prices, delta, gamma, d / d params] ([9, J])
    runs = []
    for b in range(batches):
        Z0, Z1, grids = rough.rough_randoms(TTMS, n_paths, npy, 100 + b)
        runs.append(rg.rough_chain_greeks_fixed(TTMS, FW, DF, [K, K], [T, T], Z0, Z1, *PARAMS, np.array([1.0]), np.array([1e-3]), grids, 1))
    gap = np.zeros(len(NAMES))
    for m in range(TTMS.size):
        mc = np.mean([r[2][m] for r in runs], axis=0)                           # [7, J]: delta, then the parameters
        se = np.mean([r[3][m] for r in runs], axis=0) / np.sqrt(batches)
        ref = np.vstack([four[m][1]] + [four[m][3 + k] for k in range(6)])
        gap = np.maximum(gap, np.max(np.abs(mc - ref) + se, axis=1))
    for name, g in zip(NAMES, gap):
        print(f"{name:8s} max |MC - Fourier| + SE = {g:.3e}")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
