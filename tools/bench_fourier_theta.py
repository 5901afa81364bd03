"""Wall-clock of theta (DESIGN.md §4.8) against what it replaces: price_chain_greeks without and with ``with_theta=True``, and the 2 M
single-maturity re-pricings of central differences in ttms[m] (grid pinned, one price_chain call each, on the chain cut after maturity m)
on the BTC chain for LogSV, Heston and Hawkes.  Median of --reps calls after warm-up, the three variants alternated call by call.  Prints
the card and its power limit with the times.
usage: python tools/bench_fourier_theta.py [--reps 30]"""
import argparse, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from stochvolmodels_b200 import (HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer, LOGSV_BTC_PARAMS,
                                 OptionChain, get_btc_test_chain_data)

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=30)
reps = max(20, ap.parse_args().reps)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001 -- the timing does not depend on it
        return f"unknown ({e})"


def alternated(fs):
    for _ in range(3):
        for f in fs:
            f()
    ts = [[] for _ in fs]
    for _ in range(reps):
        for k, f in enumerate(fs):
            t = time.perf_counter()
            f()
            ts[k].append(time.perf_counter() - t)
    return [1e3 * float(np.median(t)) for t in ts]


def cut(chain, m, ttm):
    """the chain's first m + 1 maturities with ttms[m] replaced: what a re-pricing of slice m needs"""
    ttms = chain.ttms[:m + 1].copy()
    ttms[m] = ttm
    return OptionChain(ttms=ttms, forwards=chain.forwards[:m + 1], discfactors=chain.discfactors[:m + 1],
                       strikes_ttms=chain.strikes_ttms[:m + 1], optiontypes_ttms=chain.optiontypes_ttms[:m + 1])


btc = get_btc_test_chain_data()
cases = [("LogSV", LogSVPricer(), LOGSV_BTC_PARAMS, float(LOGSV_BTC_PARAMS.sigma0 * np.sqrt(min(btc.ttms[0], 0.5 / 12.0)))),
         ("Heston", HestonPricer(), HestonParams(v0=0.8, theta=1.0, kappa=2.0, rho=0.0, volvol=2.0), 0.3),
         ("Hawkes", HawkesJDPricer(), HawkesJDParams(), 0.1)]
print(f"card: {card()}; BTC chain {len(btc.ttms)} maturities x {sum(len(k) for k in btc.strikes_ttms)} strikes; median of {reps}")
for name, pricer, params, vs in cases:
    bumped = [(cut(btc, m, btc.ttms[m] + s * 1e-5 * btc.ttms[m])) for m in range(len(btc.ttms)) for s in (1.0, -1.0)]

    def greeks():
        pricer.price_chain_greeks(btc, params, vol_scaler=vs)

    def theta():
        pricer.price_chain_greeks(btc, params, vol_scaler=vs, with_theta=True)

    def repricings():
        for ch in bumped:
            pricer.price_chain(ch, params, vol_scaler=vs)
    t_g, t_t, t_r = alternated([greeks, theta, repricings])
    print(f"{name:7s} price_chain_greeks {t_g:8.3f} ms | with_theta {t_t:8.3f} ms (+{t_t - t_g:.3f}) | "
          f"{len(bumped)} re-pricings {t_r:8.3f} ms")
