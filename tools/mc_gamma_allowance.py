"""Re-derive GAMMA_ALLOWANCE of tests/test_gpu_mc_gamma.py (CPU only, numpy oracles): per chain of that test (quickstart and BTC with
LogSV at 252 steps per year, g4 with Heston at 360), the smoothed Monte Carlo gamma of oracle/mc_gamma.py against the Fourier gamma of
oracle/mgf_greeks.py, on default_rng draws in batches.  Per chain it prints max over the options of |MC - Fourier| + 4 SE: an upper bound
on the Euler scheme's bias in the gamma row, which the GPU gate allows on top of 4.5 SE of its own.
   python tools/mc_gamma_allowance.py [paths_per_batch] [batches]        (a few minutes at the defaults)"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import mc, mc_gamma as og, mgf_greeks as fg        # noqa: E402

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
T5 = np.array(["P", "P", "C", "C", "C"])
Q = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
LOGSV_BTC = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)
HESTON = (0.04, 0.04, 4.0, -0.5, 0.4)


def chains():
    from stochvolmodels_b200 import get_btc_test_chain_data
    btc = get_btc_test_chain_data()
    return {"quickstart": ("logsv", Q, np.array([0.25, 0.5]), np.ones(2), np.ones(2), [K5, K5], [T5, T5], 252),
            "btc": ("logsv", LOGSV_BTC, btc.ttms, btc.forwards, btc.discfactors, list(btc.strikes_ttms), list(btc.optiontypes_ttms), 252),
            "g4": ("heston", HESTON, np.array([0.25, 1.0]), np.ones(2), np.ones(2), [K5, K5], [T5, T5], 360)}


def main(n_paths=100_000, batches=8):
    for name, (model, p, ttms, fw, df, K, T, npy) in chains().items():
        if model == "logsv":
            four = [r[2] for r in fg.logsv_chain_greeks(p, ttms, fw, df, K, T)[0]]
        else:
            four = [r[2] for r in fg.heston_chain_greeks(p, ttms, fw, df, K, T)[0]]
        steps = mc.chain_steps(ttms, npy)
        runs = []
        for b in range(batches):
            rng = np.random.default_rng(300 + b)
            Z0s = [rng.standard_normal((S, n_paths)) for S, _ in steps]
            Z1s = [rng.standard_normal((S, n_paths)) for S, _ in steps]
            dts = [dt for _, dt in steps]
            if model == "logsv":
                runs.append(og.logsv_mc_chain_gamma_fixed(p, ttms, fw, df, K, T, np.ones(len(ttms)), Z0s, Z1s, dts))
            else:
                runs.append(og.heston_mc_chain_gamma_fixed(p, ttms, fw, df, K, T, Z0s, Z1s, dts))
        gap = z = 0.0
        for m in range(len(ttms)):
            g = np.mean([r[2][m] for r in runs], axis=0)
            se = np.sqrt(np.mean([r[3][m] ** 2 for r in runs], axis=0) / batches)
            gap = max(gap, float(np.max(np.abs(g - four[m]) + 4.0 * se)))
            z = max(z, float(np.max(np.abs(g - four[m]) / se)))
        print(f"{name:10s} max |MC - Fourier| + 4 SE = {gap:.3e}   (max |MC - Fourier| / SE = {z:.2f})", flush=True)


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
