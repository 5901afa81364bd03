"""Exact event-driven route of the Hawkes jump-diffusion Monte Carlo against the Euler route (DESIGN.md §3.13): BTC chain and the
hawkes_mc.npz chain, default HawkesJDParams, 1e6 and 1e7 paths, engine level, the two routes alternated in one process, median of 7 calls
after two warm-up calls each.  Per configuration and route:
  wall_ms      host clock around the synchronous library call
  gpu_ms       CUDA events around the call on the library's stream (every launch and copy of the call)
  slice_ms     the slice kernel's own time per call (hawkes_slice_kernel / hawkes_exact_slice_kernel), from a torch.profiler pass of its own
  max_z        max over strikes of |MC - Fourier| / SE at that path count
and for the exact route the candidates per path over the chain (mean, max) and the mean over warps of 32 consecutive paths of the warp's
largest per-maturity candidate count, summed over maturities, from the events hook on the first 1e5 paths.  One JSON line per
configuration, with the card name and power limit read in the same run.
   python tools/bench_hawkes_exact.py [--paths 1e6,1e7] [--reps 7]"""
import argparse, json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine, get_btc_test_chain_data
from stochvolmodels_b200 import _capi as C
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

SEED = 10


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def mc_chain():
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    g = np.load(os.path.join(here, "tests", "golden", "hawkes_mc.npz"))
    M = g["chain_ttms"].shape[0]
    return OptionChain(ttms=g["chain_ttms"], forwards=g["chain_forwards"], discfactors=g["chain_discfactors"],
                       strikes_ttms=[g["chain_strikes"] * f for f in g["chain_forwards"]], optiontypes_ttms=[g["chain_types"]] * M)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", default="1e6,1e7")
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    params = HawkesJDParams()
    d = params.to_dict()
    d.pop("risk_premia_gamma")
    pc = _params_c(**d)
    flags = engine.mc_flags("fp64", "fp32")
    name = card()
    for label, chain in (("btc", get_btc_test_chain_data()), ("hawkes_mc", mc_chain())):
        four = HawkesJDPricer().price_chain(chain, params)
        a = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
        _, _, _, ev = engine.hawkesjd_mc_chain_exact(pc, *a, 100_000, C.LOG_RETURN, SEED, n_paths_out=100_000)
        cand = ev[:, 2, :]                                              # [M, n]
        warp_max = cand.reshape(cand.shape[0], -1, 32).max(axis=2).sum(axis=0)
        for n in (int(float(s)) for s in args.paths.split(",")):
            routes = {"euler": lambda: engine.hawkesjd_mc_chain(pc, *a, n, C.LOG_RETURN, SEED, flags),
                      "exact": lambda: engine.hawkesjd_mc_chain_exact(pc, *a, n, C.LOG_RETURN, SEED)[:2]}
            wall, gpu, z = {k: [] for k in routes}, {k: [] for k in routes}, {}
            for k, fn in routes.items():
                for _ in range(2):
                    p, e = fn()
                z[k] = float(max(np.max(np.abs((p[m] - four[m]) / e[m])) for m in range(len(p))))
            for _ in range(args.reps):
                for k, fn in routes.items():
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    ev0.record()
                    fn()
                    ev1.record()
                    torch.cuda.synchronize()
                    wall[k].append(1e3 * (time.perf_counter() - t))
                    gpu[k].append(ev0.elapsed_time(ev1))
            slice_ms = {}
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for k, fn in routes.items():
                    fn()
                torch.cuda.synchronize()
            for e in prof.key_averages():
                if e.key.startswith("_ZN6b200sv25hawkes_exact_slice_kernel") or "hawkes_exact_slice_kernel" in e.key:
                    slice_ms["exact"] = slice_ms.get("exact", 0.0) + e.device_time_total / 1e3
                elif "hawkes_slice_kernel" in e.key:
                    slice_ms["euler"] = slice_ms.get("euler", 0.0) + e.device_time_total / 1e3
            row = {"chain": label, "nb_path": n, "card": name,
                   **{f"{k}_wall_ms": round(statistics.median(wall[k]), 2) for k in routes},
                   **{f"{k}_gpu_ms": round(statistics.median(gpu[k]), 2) for k in routes},
                   **{f"{k}_slice_ms": round(v, 2) for k, v in slice_ms.items()},
                   **{f"{k}_max_z": round(z[k], 2) for k in routes},
                   "exact_over_euler_wall": round(statistics.median(wall["exact"]) / statistics.median(wall["euler"]), 3),
                   "candidates_mean": round(float(cand.sum(axis=0).mean()), 2), "candidates_max": int(cand.sum(axis=0).max()),
                   "warp_max_candidates_mean": round(float(warp_max.mean()), 2),
                   "events_mean": round(float((ev[:, 0] + ev[:, 1]).sum(axis=0).mean()), 2)}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
