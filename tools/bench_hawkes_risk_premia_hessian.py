"""One call of the Hawkes risk-kernel second order (engine.hawkesjd_price_chain_risk_premia_hessian: prices, delta, gamma, the 16 rows,
vanna and the 136 Hessian rows of HAWKES_RISK_PREMIA_GREEK_PARAMS) against what it replaces: one price_chain_risk_premia_greeks call for
scale, the 1 + 32 + 480 = 513-set central-difference batch of the second order (the base, +-h in each of the 16 parameters, and the four
corners +-h_p +-h_q of each of the 120 pairs p < q), each set priced under its own risk kernel in one
engine.hawkesjd_price_chain_batch(..., gammas=...) call, and 32 first-order calls (differences of the first-order rows, +-h in each
parameter).  On the BTC sample chain and the hawkes_fourier.npz chain, at gamma = 0.4, with the grid scale pinned (the difference batch
needs one grid for every set).  Medians over --reps alternating calls after a warm-up; each call ends in the library's own
synchronisation.  The card and its power limit are read in the same run.
    python tools/bench_hawkes_risk_premia_hessian.py [--reps 10] [--out f]"""
import argparse
import importlib.util
import itertools
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from stochvolmodels_b200 import engine
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

_spec = importlib.util.spec_from_file_location("bench_hawkes_risk_premia_greeks",
                                               os.path.join(ROOT, "tools", "bench_hawkes_risk_premia_greeks.py"))
first = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(first)

VOL_SCALER = first.VOL_SCALER
GAMMA = 0.4


def _moved(p: dict, gamma: float, steps):
    """(params, gamma) moved by the (name, sign) steps, each 1e-6 max(1, |value|)"""
    q, g = dict(p), gamma
    for name, s in steps:
        if name == "risk_premia_gamma":
            g += s * 1e-6 * max(1.0, abs(gamma))
        else:
            q[name] += s * 1e-6 * max(1.0, abs(p[name]))
    return q, g


def second_order_sets(p: dict, gamma: float):
    """the 1 + 32 + 480 (params, gamma) of second-order central differences in HAWKES_RISK_PREMIA_GREEK_PARAMS"""
    names = engine.HAWKES_RISK_PREMIA_GREEK_PARAMS
    moves = [[]] + [[(n, s)] for n in names for s in (1.0, -1.0)]
    moves += [[(a, sa), (b, sb)] for a, b in itertools.combinations(names, 2) for sa in (1.0, -1.0) for sb in (1.0, -1.0)]
    sets = [_moved(p, gamma, mv) for mv in moves]
    return [_params_c(**q) for q, _ in sets], np.array([g for _, g in sets])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    p, _, cs = first.chains()
    card = {"name": torch.cuda.get_device_name(0), "power_limit_w": first.single.power_limit_w()}
    pc = _params_c(**p)
    params_list, gammas = second_order_sets(p, GAMMA)
    bumps = [(_params_c(**q), g) for q, g in (_moved(p, GAMMA, [(n, s)]) for n in engine.HAWKES_RISK_PREMIA_GREEK_PARAMS for s in (1.0, -1.0))]
    results = {"card": card, "gamma": GAMMA, "vol_scaler": VOL_SCALER, "reps": args.reps, "chains": {}}
    for label, c in cs.items():
        ch = (c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms)
        hessian = lambda: engine.hawkesjd_price_chain_risk_premia_hessian(pc, GAMMA, *ch, vol_scaler=VOL_SCALER)
        greeks = lambda: engine.hawkesjd_price_chain_risk_premia_greeks(pc, GAMMA, *ch, vol_scaler=VOL_SCALER)
        batch = lambda: engine.hawkesjd_price_chain_batch(params_list, *ch, vol_scaler=VOL_SCALER, gammas=gammas, with_ivols=False)

        def greeks_32():
            for q, g in bumps:
                engine.hawkesjd_price_chain_risk_premia_greeks(q, g, *ch, vol_scaler=VOL_SCALER)

        fns = {"hessian_ms": hessian, "greeks_ms": greeks, "difference_batch_ms": batch, "first_order_differences_ms": greeks_32}
        for _ in range(2):
            for fn in fns.values():
                fn()
        times = {k: [] for k in fns}
        for _ in range(args.reps):
            for k, fn in fns.items():
                t = time.perf_counter()
                fn()
                times[k].append(time.perf_counter() - t)
        row = {"strikes": int(sum(len(k) for k in c.strikes_ttms)), "maturities": len(c.ttms), "difference_sets": len(params_list)}
        row.update({k: 1e3 * statistics.median(v) for k, v in times.items()})
        results["chains"][label] = row
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
