"""Wall-clock of the Hawkes second-order Fourier sensitivities against the alternatives they replace, on the hawkes_fourier.npz 3x5 chain and
the BTC 4x49 chain, default parameters, vol_scaler pinned: price_chain_greeks, price_chain_hessian, the 2 n^2 + 1 = 451 sets of central
second differences in one engine.hawkesjd_price_chain_batch call, and the 2n = 30 price_chain_greeks calls of first-order differences.
The four are alternated call by call after warm-up; medians.  Prints the card and its power limit with the times.
usage: python tools/bench_hawkes_hessian.py [--reps 20]"""
import argparse, dataclasses, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
reps = ap.parse_args().reps


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001 -- the timing does not depend on it
        return f"unknown ({e})"


def second_difference_sets(values, h=1e-4):
    """the base point, x +- h e_i (diagonal) and x +- h e_i +- h e_j for i < j (mixed): 2 n^2 + 1 sets"""
    n, sets = len(values), [list(values)]
    for i in range(n):
        for s in (1.0, -1.0):
            v = list(values)
            v[i] += s * h
            sets.append(v)
    for i in range(n):
        for j in range(i + 1, n):
            for si in (1.0, -1.0):
                for sj in (1.0, -1.0):
                    v = list(values)
                    v[i] += si * h
                    v[j] += sj * h
                    sets.append(v)
    return sets


def timed_alternating(fs):
    for f in fs:
        for _ in range(3):
            f()
    ts = [[] for _ in fs]
    for _ in range(reps):
        for k, f in enumerate(fs):
            t = time.perf_counter()
            f()
            ts[k].append(time.perf_counter() - t)
    return [1e3 * float(np.median(t)) for t in ts]


g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "hawkes_fourier.npz"))
small = OptionChain(ttms=g["ttms"], forwards=g["forwards"], strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["types"]] * 3,
                    discfactors=g["discfactors"])
print(f"card: {card()}", flush=True)
params = HawkesJDParams()
names = engine.HAWKES_GREEK_PARAMS
base = {k: v for k, v in params.to_dict().items() if k != "risk_premia_gamma"}
for label, chain in (("hawkes_fourier 3x5", small), ("btc 4x49", get_btc_test_chain_data())):
    pricer = HawkesJDPricer()
    vs = float(np.clip(params.sigma, 0.2, 0.5) * np.sqrt(min(np.min(chain.ttms), 1.0 / 12.0)))
    sets = [_params_c(**{**base, **dict(zip(names, s))}) for s in second_difference_sets([base[n] for n in names])]
    bumps = [dataclasses.replace(params, **{n: getattr(params, n) + s * 1e-6 * max(1.0, abs(getattr(params, n)))}) for n in names for s in (1, -1)]
    fs = [lambda: pricer.price_chain_greeks(chain, params, vol_scaler=vs),
          lambda: pricer.price_chain_hessian(chain, params, vol_scaler=vs),
          lambda: engine.hawkesjd_price_chain_batch(sets, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                    chain.optiontypes_ttms, vol_scaler=vs, max_phi=500, with_ivols=False),
          lambda: [pricer.price_chain_greeks(chain, b, vol_scaler=vs) for b in bumps]]
    t_g, t_h, t_b, t_f = timed_alternating(fs)
    print(f"{label:18s} price_chain_greeks {t_g:8.3f} ms   price_chain_hessian {t_h:8.3f} ms   {len(sets)}-set central-difference batch "
          f"{t_b:8.3f} ms   {len(bumps)} price_chain_greeks {t_f:8.3f} ms", flush=True)
