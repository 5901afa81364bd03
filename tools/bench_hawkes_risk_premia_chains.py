"""K risk-premia fits of the Hawkes jump-diffusion one after the other (HawkesJDPricer.calibrate_risk_premia_gamma_to_chain, the loop of
the reference's calibrate_risk_premia_at_dates) against the same K fits in lock-step (calibrate_risk_premia_gamma_to_chains: one
risk-kernel multi-chain library call per optimizer round).

The series is the BTC sample chain followed by risk-kernel markets on the synthetic 3 x 12 strikes of tools/bench_hawkes_calibration.py
(the risk-premia market of tests/test_gpu_hawkes.py), priced at sigma and gamma drifting from one chain to the next (a stand-in for a
series of daily chains); each chain starts from its own (lambda_p, lambda_m, sigma, gamma), as each date does
in the reference.  Every lock-step fit is checked to equal its sequential fit bit for bit.  Also one gradient round alone: K chains x 2
sets with gammas through hawkesjd_price_chains_batch against K hawkesjd_price_chain_batch calls.  Wall times are medians over --reps
alternating runs after a warm-up; "library" is the time inside the batched pricer calls.  The card and its power limit are read in the
same run.   python tools/bench_hawkes_risk_premia_chains.py [--ks 1 4 16 64] [--reps 3] [--out f]"""
import argparse
import importlib.util
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

_spec = importlib.util.spec_from_file_location("bench_hawkes_calibration", os.path.join(ROOT, "tools", "bench_hawkes_calibration.py"))
single = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(single)

LIBRARY_S = [0.0]


def timed(fn):
    def wrapper(*args, **kwargs):
        t = time.perf_counter()
        try:
            return fn(*args, **kwargs)
        finally:
            LIBRARY_S[0] += time.perf_counter() - t
    return wrapper


for _name in ("hawkesjd_price_chain_batch", "hawkesjd_price_chains_batch"):
    setattr(engine, _name, timed(getattr(engine, _name)))


def series(base: OptionChain, K: int):
    """``base`` and K - 1 risk-kernel markets on the 3 x 12 strikes of tools/bench_hawkes_calibration.py at drifting (sigma, gamma), with
    one start per chain"""
    pricer, chains = HawkesJDPricer(), [base]
    flat, _ = single.synthetic_market()
    for k in range(1, K):
        truth = HawkesJDParams(sigma=0.42 + 0.08 * np.sin(0.7 * k), risk_premia_gamma=0.4 + 0.2 * np.sin(0.5 * k))
        vols = pricer.compute_model_ivols_for_chain(flat, truth)
        vols = [np.where(np.isfinite(v), v, 0.5) for v in vols]           # a quote needs a finite vol
        chains.append(OptionChain(ttms=flat.ttms, forwards=flat.forwards, discfactors=flat.discfactors, strikes_ttms=flat.strikes_ttms,
                                  optiontypes_ttms=flat.optiontypes_ttms, bid_ivs=vols, ask_ivs=[v.copy() for v in vols]))
    starts = [HawkesJDParams(sigma=0.45 + 0.02 * np.cos(k), lambda_p=6.55 + 0.1 * np.sin(k), lambda_m=8.5 + 0.1 * np.cos(k),
                             risk_premia_gamma=0.2 + 0.1 * np.sin(0.5 * k)) for k in range(K)]
    return chains, starts


def run_fits(label: str, base: OptionChain, K: int, reps: int):
    pricer = HawkesJDPricer()
    chains, starts = series(base, K)

    def sequential():
        return [pricer.calibrate_risk_premia_gamma_to_chain(c, s, print_iter=False, return_info=True) for c, s in zip(chains, starts)]

    def lockstep():
        return pricer.calibrate_risk_premia_gamma_to_chains(chains, starts, return_info=True)

    seq, lock = sequential(), lockstep()                   # warm-up, and the bit-for-bit check
    for (fit, info), lf, li in zip(seq, *lock):
        assert fit == lf and np.array_equal(info["x"], li["x"]) and info["fun"] == li["fun"] and info["nit"] == li["nit"], label
    ts, tl, ls, ll = [], [], [], []
    for _ in range(reps):
        for fn, t_out, l_out in ((sequential, ts, ls), (lockstep, tl, ll)):
            LIBRARY_S[0] = 0.0
            t = time.perf_counter()
            fn()
            t_out.append(time.perf_counter() - t)
            l_out.append(LIBRARY_S[0])
    row = {"case": "fits", "chain": label, "K": K, "seq_s": statistics.median(ts), "seq_library_s": statistics.median(ls),
           "lock_s": statistics.median(tl), "lock_library_s": statistics.median(ll), "seq_calls": sum(i["nb_batches"] for _, i in seq),
           "lock_calls": lock[1][0]["rounds"], "nit": [i["nit"] for _, i in seq], "same_fits": True}
    row["speedup"] = row["seq_s"] / row["lock_s"]
    return row


def run_round(label: str, base: OptionChain, K: int, reps: int):
    """one gradient round: K chains x 2 sets (the difference neighbours of a risk-premia point), one multi-chain call against K
    single-chain calls"""
    chains, starts = series(base, K)
    sets, gammas = [], []
    for s in starts:
        d = {k: v for k, v in s.to_dict().items() if k != "risk_premia_gamma"}
        sets.append([_params_c(**{**d, "sigma": s.sigma + 0.025}), _params_c(**d)])
        gammas.append([s.risk_premia_gamma, s.risk_premia_gamma + 8.0 * 0.025])
    args = [(c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms) for c in chains]

    def old():
        return [engine.hawkesjd_price_chain_batch(s, *a, max_phi=500, gammas=g) for s, a, g in zip(sets, args, gammas)]

    def new():
        return engine.hawkesjd_price_chains_batch([p for s in sets for p in s], np.repeat(np.arange(K), 2), args, max_phi=500,
                                                  gammas=[x for g in gammas for x in g])

    o, n = old(), new()
    for k in range(K):
        for i in range(2):
            assert np.array_equal(o[k][0][i], n[0][2 * k + i], equal_nan=True), label
            assert np.array_equal(o[k][1][i], n[1][2 * k + i], equal_nan=True), label
    t_old, t_new = single.alternate(old, new, reps)
    return {"case": "round", "chain": label, "K": K, "sets": 2 * K, "single_calls_ms": 1e3 * t_old, "multi_chain_ms": 1e3 * t_new,
            "speedup": t_old / t_new}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--round-reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool times the GPU")
    card = {"name": torch.cuda.get_device_name(0), "power_limit_w": single.power_limit_w()}
    print(json.dumps(card), flush=True)
    rows = []
    base = get_btc_test_chain_data()
    for K in a.ks:
        rows.append(run_round("btc", base, K, a.round_reps))
        print(json.dumps(rows[-1]), flush=True)
    for K in a.ks:
        rows.append(run_fits("btc", base, K, a.reps))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
