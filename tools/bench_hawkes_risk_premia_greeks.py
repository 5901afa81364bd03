"""One call of the Hawkes risk-kernel sensitivities (engine.hawkesjd_price_chain_risk_premia_greeks: prices, delta, gamma and the 16 rows
of HAWKES_RISK_PREMIA_GREEK_PARAMS) against the central-difference batch it replaces: 1 + 2 x 16 parameter sets, each priced under its own
risk kernel, in one engine.hawkesjd_price_chain_batch(..., gammas=...) call.  On the BTC sample chain and the hawkes_fourier.npz chain, at
the fixture's gamma, with the grid scale pinned (the difference batch needs one grid for every set).  Medians over --reps alternating
calls after a warm-up; each call ends in the library's own synchronisation.  The card and its power limit are read in the same run.
    python tools/bench_hawkes_risk_premia_greeks.py [--reps 30] [--out f]"""
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

from stochvolmodels_b200 import OptionChain, engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

_spec = importlib.util.spec_from_file_location("bench_hawkes_calibration", os.path.join(ROOT, "tools", "bench_hawkes_calibration.py"))
single = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(single)

VOL_SCALER = 0.1


def chains():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hawkes_fourier.npz"))
    p = dict(zip([str(k) for k in g["keys"]], (float(v) for v in g["dflt_params"])))
    fixture = OptionChain(ttms=g["ttms"], forwards=g["forwards"], strikes_ttms=[g["strikes"]] * 3, optiontypes_ttms=[g["types"]] * 3,
                          discfactors=g["discfactors"])
    return p, float(g["gamma"]), {"btc": get_btc_test_chain_data(), "hawkes_fourier": fixture}


def difference_sets(p: dict, gamma: float):
    """the 1 + 2 x 16 (params, gamma) of central differences in HAWKES_RISK_PREMIA_GREEK_PARAMS, steps 1e-6 max(1, |value|)"""
    sets, gammas = [dict(p)], [gamma]
    for name in engine.HAWKES_RISK_PREMIA_GREEK_PARAMS:
        for s in (1.0, -1.0):
            q, g = dict(p), gamma
            if name == "risk_premia_gamma":
                g += s * 1e-6 * max(1.0, abs(gamma))
            else:
                q[name] += s * 1e-6 * max(1.0, abs(q[name]))
            sets.append(q)
            gammas.append(g)
    return [_params_c(**q) for q in sets], np.array(gammas)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    p, gamma, cs = chains()
    card = {"name": torch.cuda.get_device_name(0), "power_limit_w": single.power_limit_w()}
    pc = _params_c(**p)
    params_list, gammas = difference_sets(p, gamma)
    results = {"card": card, "gamma": gamma, "vol_scaler": VOL_SCALER, "reps": args.reps, "chains": {}}
    for label, c in cs.items():
        ch = (c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms)
        greeks = lambda: engine.hawkesjd_price_chain_risk_premia_greeks(pc, gamma, *ch, vol_scaler=VOL_SCALER)
        batch = lambda: engine.hawkesjd_price_chain_batch(params_list, *ch, vol_scaler=VOL_SCALER, gammas=gammas, with_ivols=False)
        for _ in range(3):
            greeks()
            batch()
        tg, tb = [], []
        for _ in range(args.reps):
            for fn, acc in ((greeks, tg), (batch, tb)):
                t = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t)
        results["chains"][label] = {"strikes": int(sum(len(k) for k in c.strikes_ttms)), "maturities": len(c.ttms),
                                    "greeks_ms": 1e3 * statistics.median(tg), "difference_batch_ms": 1e3 * statistics.median(tb),
                                    "difference_sets": len(params_list)}
    line = json.dumps(results)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
