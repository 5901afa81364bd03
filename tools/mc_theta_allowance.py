"""Re-derive THETA_ALLOWANCE of tests/test_gpu_mc_theta.py (CPU only, numpy oracles): per chain of that test (quickstart with LogSV at 252
steps per year, g4 with Heston at 360), the Monte Carlo theta of oracle/mc_theta.py against the Fourier theta, here the central difference
of oracle/mgf.py's chain price in ttm_m alone (h = 1e-4), on default_rng draws in batches.  Per chain it prints max over the options of
|MC - Fourier| + 4 SE: an upper bound on the Euler scheme's bias in the theta row, which the GPU check allows on top of 4.5 SE of its own.
   python tools/mc_theta_allowance.py [paths_per_batch] [batches]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mc, mc_theta as ot, mgf        # noqa: E402

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)
CHAINS = {"quickstart": ("logsv", Q, np.array([0.25, 0.5]), 252), "g4": ("heston", HESTON, np.array([0.25, 1.0]), 360)}


def fourier_theta(model, p, ttms, h=1e-4):
    price = (lambda t: mgf.logsv_chain_prices(p, t, np.ones(2), np.ones(2), [K5, K5], [T5, T5])) if model == "logsv" else \
        (lambda t: mgf.heston_chain_prices(p, t, np.ones(2), np.ones(2), [K5, K5], [T5, T5]))
    out = []
    for m in range(len(ttms)):
        up, dn = ttms.copy(), ttms.copy()
        up[m] += h
        dn[m] -= h
        out.append(-(np.asarray(price(up)[m]) - np.asarray(price(dn)[m])) / (2 * h))
    return out


def main(n_paths=100_000, batches=8):
    for name, (model, p, ttms, npy) in CHAINS.items():
        four = fourier_theta(model, p, ttms)
        steps = mc.chain_steps(ttms, npy)
        runs = []
        for b in range(batches):
            rng = np.random.default_rng(400 + b)
            Z0s = [rng.standard_normal((S, n_paths)) for S, _ in steps]
            Z1s = [rng.standard_normal((S, n_paths)) for S, _ in steps]
            dts = [dt for _, dt in steps]
            if model == "logsv":
                runs.append(ot.logsv_mc_chain_theta_fixed(p, ttms, np.ones(2), np.ones(2), [K5, K5], [T5, T5], np.ones(2), Z0s, Z1s, dts))
            else:
                runs.append(ot.heston_mc_chain_theta_fixed(p, ttms, np.ones(2), np.ones(2), [K5, K5], [T5, T5], Z0s, Z1s, dts))
        gap = z = 0.0
        for m in range(len(ttms)):
            t = np.mean([r[2][m] for r in runs], axis=0)
            se = np.sqrt(np.mean([r[3][m] ** 2 for r in runs], axis=0) / batches)
            gap = max(gap, float(np.max(np.abs(t - four[m]) + 4.0 * se)))
            z = max(z, float(np.max(np.abs(t - four[m]) / se)))
        print(f"{name:10s} max |MC - Fourier| + 4 SE = {gap:.3e}   (max |MC - Fourier| / SE = {z:.2f})", flush=True)


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
