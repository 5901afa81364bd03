"""K chains calibrated one after the other (calibrate_model_params_to_chain) against the same K fits in lock-step
(calibrate_model_params_to_chains: one multi-chain library call per optimizer round), for LogSV PARAMS5 and Heston.

The chains are the BTC sample chain's quotes and synthetic model markets on its strikes and maturities at parameters drifting from one
chain to the next (a stand-in for a series of daily chains).  Every lock-step fit is checked to equal its sequential fit bit for bit.
Wall times are medians over --reps alternating runs; "library" is the part of it spent inside the batched pricer calls (marshalling, GPU
work and the copy back), the rest is host work: SLSQP, the parameter codec, the objective and, in lock-step, the hand-over between threads.
Prints one line per (model, K) and writes them as JSON to --out.   python tools/bench_calibration_chains.py [--ks 1 4 16 64] [--out f]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from stochvolmodels_b200 import (BTC_HESTON_PARAMS, LOGSV_BTC_PARAMS, HestonParams, HestonPricer, LogSvParams, LogSVPricer, OptionChain,
                                 engine, get_btc_test_chain_data)

LIBRARY_S = [0.0]          # wall time inside the batched pricers (marshalling + GPU + copy back), accumulated by timed()


def timed(fn):
    def wrapper(*args, **kwargs):
        t = time.perf_counter()
        try:
            return fn(*args, **kwargs)
        finally:
            LIBRARY_S[0] += time.perf_counter() - t
    return wrapper


for _name in ("logsv_price_chain_batch", "heston_price_chain_batch", "logsv_price_chains_batch", "heston_price_chains_batch"):
    setattr(engine, _name, timed(getattr(engine, _name)))


def markets(K: int, model: str):
    """K chains: the BTC quotes, then model markets at drifting parameters on the BTC strikes and maturities"""
    btc = get_btc_test_chain_data()
    out = [btc]
    for i in range(1, K):
        s = i / max(K - 1, 1)
        if model == "logsv":
            p, pricer = LOGSV_BTC_PARAMS, LogSVPricer()
            truth = LogSvParams(sigma0=p.sigma0 * (0.85 + 0.3 * s), theta=p.theta * (1.1 - 0.2 * s), kappa1=p.kappa1, kappa2=p.kappa2,
                                beta=p.beta + 0.2 * (s - 0.5), volvol=p.volvol * (0.9 + 0.2 * s))
            vols = pricer.compute_model_ivols_for_chain(btc, truth, vol_scaler=pricer.set_vol_scaler(btc))
        else:
            p = BTC_HESTON_PARAMS
            truth = HestonParams(v0=p.v0 * (0.8 + 0.4 * s), theta=p.theta * (1.1 - 0.2 * s), kappa=p.kappa, rho=p.rho * (0.8 + 0.4 * s),
                                 volvol=p.volvol * (0.9 + 0.2 * s))
            vols = HestonPricer().compute_model_ivols_for_chain(btc, truth)
        vols = [np.asarray(v) for v in vols]
        out.append(OptionChain(ttms=btc.ttms, forwards=btc.forwards, discfactors=btc.discfactors, strikes_ttms=btc.strikes_ttms,
                               optiontypes_ttms=btc.optiontypes_ttms, ids=btc.ids, bid_ivs=[v - 0.005 for v in vols],
                               ask_ivs=[v + 0.005 for v in vols]))
    return out


def run(model: str, K: int, reps: int):
    chains = markets(K, model)
    if model == "logsv":
        pricer, start = LogSVPricer(), LogSvParams(sigma0=0.7, theta=0.9, kappa1=LOGSV_BTC_PARAMS.kappa1, kappa2=LOGSV_BTC_PARAMS.kappa2,
                                                   beta=0.0, volvol=1.4)
    else:
        pricer, start = HestonPricer(), HestonParams(v0=0.6, theta=0.6, kappa=3.0, rho=-0.1, volvol=1.5)
    seq_t, lock_t, seq_lib, lock_lib = [], [], [], []
    for _ in range(reps):                # alternate the two so that host noise hits both alike
        torch.cuda.synchronize()
        LIBRARY_S[0] = 0.0
        t = time.perf_counter()
        seq = [pricer.calibrate_model_params_to_chain(c, start, return_info=True) for c in chains]
        torch.cuda.synchronize()
        seq_t.append(time.perf_counter() - t)
        seq_lib.append(LIBRARY_S[0])
        LIBRARY_S[0] = 0.0
        t = time.perf_counter()
        fits, infos = pricer.calibrate_model_params_to_chains(chains, start, return_info=True)
        torch.cuda.synchronize()
        lock_t.append(time.perf_counter() - t)
        lock_lib.append(LIBRARY_S[0])
    for (f, i), j in zip(seq, infos):
        assert np.array_equal(i["x"], j["x"]) and i["fun"] == j["fun"] and i["nit"] == j["nit"], "lock-step fit differs"
    seq_calls = sum(i["nb_batches"] for _, i in seq)
    rounds = infos[0]["rounds"]
    sets_total = sum(i["nb_batches"] for i in infos) * (len(infos[0]["x"]) + 1)      # difference objective: n + 1 sets per batch
    return dict(model=model, K=K, sequential_s=float(np.median(seq_t)), lockstep_s=float(np.median(lock_t)),
                speedup=float(np.median(seq_t) / np.median(lock_t)), sequential_library_s=float(np.median(seq_lib)),
                lockstep_library_s=float(np.median(lock_lib)), sequential_calls=seq_calls, lockstep_calls=rounds,
                sets_per_lockstep_call=sets_total / rounds, sets_per_sequential_call=sets_total / seq_calls,
                nb_batches_max=max(i["nb_batches"] for i in infos), nb_batches_min=min(i["nb_batches"] for i in infos))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--models", nargs="+", default=["logsv", "heston"])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"# {gpu}")
    for model in a.models:                # warm-up: module load, first allocations
        run(model, 2, 1)
    rows = []
    for model in a.models:
        for K in a.ks:
            r = run(model, K, a.reps)
            rows.append(r)
            print(f"{model:6s} K={K:3d}  sequential {r['sequential_s']:7.3f} s ({r['sequential_library_s']:7.3f} s in {r['sequential_calls']:5d} "
                  f"calls of {r['sets_per_sequential_call']:.1f} sets) | lock-step {r['lockstep_s']:7.3f} s ({r['lockstep_library_s']:7.3f} s in "
                  f"{r['lockstep_calls']:4d} calls of {r['sets_per_lockstep_call']:.1f} sets) | x{r['speedup']:.2f}", flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
