"""Calibration drivers with the forward-difference gradient (default) against the exact gradient (``gradient="exact"``, DESIGN.md §4.6),
per fit: wall time, SLSQP iterations, library calls and final objective.  Fits: the calib_logsv_params4 golden (PARAMS4), the
calib_logsv_varswap golden's chain (PARAMS5), the calib_heston golden, the BTC chain (PARAMS5) and a Hawkes chain generated from known
parameters plus fixed vol noise.  The two modes alternate fit by fit after one warm-up fit of each; medians over the repeats.  Prints the
card and its power limit with the results, and writes them as JSON to --out when given.
usage: python tools/bench_ivol_calibration.py [--reps 3] [--out results.json]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from stochvolmodels_b200 import (HawkesJDParams, HawkesJDPricer, HestonParams, HestonPricer, LogSvParams, LogSVPricer, LogsvModelCalibrationType,
                                 OptionChain, get_btc_test_chain_data)

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--out", default=None)
args = ap.parse_args()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001 -- the timing does not depend on it
        return f"unknown ({e})"


def golden_chain(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name))
    vols = [np.asarray(v) for v in g["market_vols"]]
    M = len(g["ttms"])
    return g, OptionChain(ttms=g["ttms"], ids=np.array([f"{t:0.2f}" for t in g["ttms"]]), forwards=g["forwards"], strikes_ttms=[g["strikes"]] * M,
                          optiontypes_ttms=[g["types"]] * M, bid_ivs=vols, ask_ivs=[v.copy() for v in vols])


def hawkes_case():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hawkes_fourier.npz"))
    unpack = lambda x: HawkesJDParams(mu=0.0, sigma=x[0], shift_p=0.06, mean_p=x[1], shift_m=-0.06, mean_m=x[2], lambda_p=6.55, theta_p=x[3],
                                      kappa_p=x[5], beta1_p=x[6], beta2_p=-x[6], lambda_m=8.5, theta_m=x[4], kappa_m=x[5], beta1_m=x[7],
                                      beta2_m=-x[7])
    strikes = [np.linspace(0.8, 1.2, 9) * f for f in g["forwards"]]
    types = [np.where(k >= f, "C", "P") for k, f in zip(strikes, g["forwards"])]
    grid = OptionChain(ttms=g["ttms"], forwards=g["forwards"], discfactors=g["discfactors"], strikes_ttms=strikes, optiontypes_ttms=types)
    vols = HawkesJDPricer().compute_model_ivols_for_chain(grid, unpack(np.array([0.7, 0.03, -0.03, 6.55, 8.5, 25.0, 70.0, 100.0])))
    rng = np.random.RandomState(4)
    noisy = [v + rng.uniform(-2e-3, 2e-3, v.size) for v in vols]
    chain = OptionChain(ttms=g["ttms"], forwards=g["forwards"], discfactors=g["discfactors"], strikes_ttms=strikes, optiontypes_ttms=types,
                        ids=np.array(["a", "b", "c"]), bid_ivs=noisy, ask_ivs=[v.copy() for v in noisy])
    return chain, unpack(np.array([0.8, 0.05, -0.05, 8.0, 7.0, 30.0, 60.0, 90.0]))


def fits():
    g4, c4 = golden_chain("calib_logsv_params4.npz")
    gv, cv = golden_chain("calib_logsv_varswap.npz")
    gh, ch = golden_chain("calib_heston.npz")
    btc = get_btc_test_chain_data()
    hk_chain, hk_start = hawkes_case()
    P4, P5 = LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5
    btc_start = LogSvParams(sigma0=0.7, theta=0.9, kappa1=3.1844, kappa2=None, beta=0.0, volvol=1.4)
    return {
        "logsv_params4_golden": lambda mode: LogSVPricer().calibrate_model_params_to_chain(c4, LogSvParams(*g4["start"]), model_calibration_type=P4,
                                                                                           return_info=True, gradient=mode)[1],
        "logsv_params5_varswap_golden_chain": lambda mode: LogSVPricer().calibrate_model_params_to_chain(
            cv, LogSvParams(*gv["start"][:3], None, *gv["start"][4:]), model_calibration_type=P5, return_info=True, gradient=mode)[1],
        "heston_golden": lambda mode: HestonPricer().calibrate_model_params_to_chain(ch, HestonParams(*gh["start"]), return_info=True,
                                                                                      gradient=mode)[1],
        "logsv_params5_btc": lambda mode: LogSVPricer().calibrate_model_params_to_chain(btc, btc_start, model_calibration_type=P5,
                                                                                        return_info=True, gradient=mode)[1],
        "hawkes_generated": lambda mode: HawkesJDPricer().calibrate_model_params_to_chain(hk_chain, hk_start, return_info=True, gradient=mode)[1],
    }


def main():
    results = {"card": card(), "reps": args.reps, "fits": {}}
    print(f"card, power limit: {results['card']}", flush=True)
    for name, fit in fits().items():
        runs = {"difference": [], "exact": []}
        for mode in runs:                                    # warm-up: module loads, pools, first-call set-up
            fit(mode)
        for _ in range(args.reps):
            for mode in ("difference", "exact"):
                t0 = time.perf_counter()
                info = fit(mode)                             # every driver call ends in a synchronised D2H copy
                runs[mode].append((time.perf_counter() - t0, info))
        row = {}
        for mode, rs in runs.items():
            wall = float(np.median([r[0] for r in rs]))
            info = rs[-1][1]
            row[mode] = {"wall_s": wall, "nit": int(info["nit"]), "library_calls": int(info["nb_batches"]), "fun": float(info["fun"]),
                         "ms_per_iteration": 1e3 * wall / max(int(info["nit"]), 1)}
        results["fits"][name] = row
        d, e = row["difference"], row["exact"]
        print(f"{name:38s} difference: {1e3 * d['wall_s']:9.1f} ms nit {d['nit']:3d} calls {d['library_calls']:4d} fun {d['fun']:.6e} | "
              f"exact: {1e3 * e['wall_s']:9.1f} ms nit {e['nit']:3d} calls {e['library_calls']:4d} fun {e['fun']:.6e} | "
              f"ms/it {d['ms_per_iteration']:.2f} vs {e['ms_per_iteration']:.2f}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
