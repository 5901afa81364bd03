"""K Hawkes jump-diffusion chains calibrated one after the other (HawkesJDPricer.calibrate_model_params_to_chain) against the same K fits in
lock-step (calibrate_model_params_to_chains: one multi-chain library call per optimizer round, each chain's sets in one Riccati launch).

Two series: the BTC sample chain followed by model markets on its strikes, and the synthetic 3 x 12 market of
tools/bench_hawkes_calibration.py followed by model markets on its strikes; the model markets are priced at parameters drifting from one
chain to the next (a stand-in for a series of daily chains).  Every lock-step fit is checked to equal its sequential fit bit for bit.
Also one round's library call alone: K x 9 sets through hawkesjd_price_chains_batch against K hawkesjd_price_chain_batch calls.
Wall times are medians over --reps alternating runs after a warm-up; "library" is the time inside the batched pricer calls.  The card
and its power limit are read in the same run.   python tools/bench_hawkes_calibration_chains.py [--ks 1 4 16 64] [--reps 3] [--out f]"""
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
    """``base`` and K - 1 model markets on its strikes at drifting parameters"""
    pricer, out = HawkesJDPricer(), [base]
    for k in range(1, K):
        truth = HawkesJDParams(sigma=0.4 + 0.15 * np.sin(0.7 * k), mean_p=0.03 + 0.01 * np.cos(k), theta_p=6.0 + 0.05 * k, kappa_p=24.0 + 0.1 * k,
                               kappa_m=24.0 + 0.1 * k)
        vols = pricer.compute_model_ivols_for_chain(base, truth)
        out.append(OptionChain(ttms=base.ttms, forwards=base.forwards, discfactors=base.discfactors, strikes_ttms=base.strikes_ttms,
                               optiontypes_ttms=base.optiontypes_ttms, bid_ivs=vols, ask_ivs=[v.copy() for v in vols]))
    return out


def run_fits(label: str, base: OptionChain, K: int, reps: int):
    pricer = HawkesJDPricer()
    chains = series(base, K)

    def sequential():
        return [pricer.calibrate_model_params_to_chain(c, single.START, return_info=True) for c in chains]

    def lockstep():
        return pricer.calibrate_model_params_to_chains(chains, single.START, return_info=True)

    seq, lock = sequential(), lockstep()                   # warm-up, and the bit-for-bit check
    for (fit, info), lf, li in zip(seq, *lock):
        assert np.array_equal(info["x"], li["x"]) and info["fun"] == li["fun"] and info["nit"] == li["nit"], label
    ts, tl, ls, ll = [], [], [], []
    for _ in range(reps):
        for fn, t_out, l_out in ((sequential, ts, ls), (lockstep, tl, ll)):
            LIBRARY_S[0] = 0.0
            t = time.perf_counter()
            fn()
            t_out.append(time.perf_counter() - t)
            l_out.append(LIBRARY_S[0])
    batches = sum(i["nb_batches"] for _, i in seq)
    row = {"case": "fits", "chain": label, "K": K, "seq_s": statistics.median(ts), "seq_library_s": statistics.median(ls),
           "lock_s": statistics.median(tl), "lock_library_s": statistics.median(ll), "seq_calls": batches, "lock_calls": lock[1][0]["rounds"]}
    row["speedup"] = row["seq_s"] / row["lock_s"]
    return row


def run_round(label: str, base: OptionChain, K: int, reps: int):
    """one gradient round: K chains x 9 sets, one multi-chain call against K single-chain calls"""
    chains = series(base, K)
    sets = [[_params_c(**p.to_dict()) for p in single.neighbours(single.START, 8)] for _ in range(K)]
    args = [(c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms) for c in chains]

    def old():
        return [engine.hawkesjd_price_chain_batch(s, *a, max_phi=500) for s, a in zip(sets, args)]

    def new():
        return engine.hawkesjd_price_chains_batch([p for s in sets for p in s], np.repeat(np.arange(K), 9), args, max_phi=500)

    o, n = old(), new()
    for k in range(K):
        for i in range(9):
            assert np.array_equal(o[k][1][i], n[1][9 * k + i], equal_nan=True), label
    t_old, t_new = single.alternate(old, new, reps)
    return {"case": "round", "chain": label, "K": K, "sets": 9 * K, "single_calls_ms": 1e3 * t_old, "multi_chain_ms": 1e3 * t_new,
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
    bases = (("btc", get_btc_test_chain_data()), ("synthetic_3x12", single.synthetic_market()[0]))
    for label, base in bases:
        for K in a.ks:
            rows.append(run_round(label, base, K, a.round_reps))
            print(json.dumps(rows[-1]), flush=True)
    for label, base in bases:
        for K in a.ks:
            rows.append(run_fits(label, base, K, a.reps))
            print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
