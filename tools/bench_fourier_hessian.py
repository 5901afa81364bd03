"""Wall-clock of the second-order Fourier sensitivities against the alternative they replace: median of repeated calls after warm-up of
price_chain_greeks, price_chain_hessian and the central-difference batch of second differences (engine.*_price_chain_batch, grid pinned:
the 2 n^2 + 1 sets of the diagonal and mixed central second differences) on the BTC chain and BASELINE config 3 (5 maturities x 21
strikes), LogSV and Heston.  Prints the card and its power limit with the times.
usage: python tools/bench_fourier_hessian.py [--reps 30]"""
import argparse, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from stochvolmodels_b200 import HestonParams, HestonPricer, LogSvParams, LogSVPricer, LOGSV_BTC_PARAMS, OptionChain, engine, get_btc_test_chain_data

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=30)
reps = ap.parse_args().reps


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001 -- the timing does not depend on it
        return f"unknown ({e})"


def timed(f):
    for _ in range(3):
        f()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t)
    return 1e3 * float(np.median(ts))


def second_difference_sets(values, h=1e-4):
    """the base point, x +- h e_i (diagonal) and x +- h e_i +- h e_j for i < j (mixed): 1 + 2n + 4 n (n - 1) / 2 = 2 n^2 + 1 sets"""
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


K21 = np.linspace(0.5, 1.5, 21)
T21 = np.where(K21 >= 1.0, "C", "P")
c3 = OptionChain(ttms=np.array([1.0 / 12.0, 0.25, 0.5, 0.75, 1.0]), forwards=np.ones(5), strikes_ttms=[K21] * 5, optiontypes_ttms=[T21] * 5)
btc = get_btc_test_chain_data()
print(f"card: {card()}", flush=True)
for name, chain, params in (("logsv btc 4x49", btc, LOGSV_BTC_PARAMS), ("logsv c3 5x21", c3, LogSvParams(1.0, 1.0, 5.0, 5.0, 0.2, 2.0))):
    pricer = LogSVPricer()
    q = (params.sigma0, params.theta, params.kappa1, params.kappa2, params.beta, params.volvol)
    vs = float(params.sigma0 * np.sqrt(min(np.min(chain.ttms), 0.5 / 12.0)))
    sets = [engine.logsv_params_c(*s) for s in second_difference_sets(q)]
    batch = lambda: engine.logsv_price_chain_batch(sets, chain.ttms, chain.forwards, chain.discfactors, None, chain.strikes_ttms,
                                                   chain.optiontypes_ttms, vol_scaler=vs, with_ivols=False)
    t_g = timed(lambda: pricer.price_chain_greeks(chain, params))
    t_h = timed(lambda: pricer.price_chain_hessian(chain, params))
    t_b = timed(batch)
    print(f"{name:16s} price_chain_greeks {t_g:8.3f} ms   price_chain_hessian {t_h:8.3f} ms   {len(sets)}-set central-difference batch "
          f"{t_b:8.3f} ms", flush=True)
hp = HestonParams()
q = (hp.v0, hp.theta, hp.kappa, hp.rho, hp.volvol)
for name, chain in (("heston btc 4x49", btc), ("heston c3 5x21", c3)):
    pricer = HestonPricer()
    vs = float(min(0.3, np.sqrt(hp.v0 * chain.ttms[0])))
    sets = [engine.heston_params_c(*s) for s in second_difference_sets(q)]
    batch = lambda: engine.heston_price_chain_batch(sets, chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms,
                                                    chain.optiontypes_ttms, vol_scaler=vs, with_ivols=False)
    t_g = timed(lambda: pricer.price_chain_greeks(chain, hp))
    t_h = timed(lambda: pricer.price_chain_hessian(chain, hp))
    t_b = timed(batch)
    print(f"{name:16s} price_chain_greeks {t_g:8.3f} ms   price_chain_hessian {t_h:8.3f} ms   {len(sets)}-set central-difference batch "
          f"{t_b:8.3f} ms", flush=True)
