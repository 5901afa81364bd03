"""Cost of the Monte Carlo theta (DESIGN.md §3.12): LogSV and Heston MC on the BTC chain, 1e7 paths (LogSV 252 steps, nb_steps_per_year=582;
Heston at 360 steps per year), public API with host buffers, median of 5 calls after one warm-up each, the variants alternated call by
call.  Times the greeks pass without and with theta, and the 2 M common-random-number pricings (each maturity moved alone, both ways) a
bumped theta needs; on the rough-LogSV route (1e6 paths, 360 steps per year) the 2 pricings with every maturity moved at once.  One JSON line per model with the times, the theta overhead, and the card name and power limit they were measured at.
   python tools/bench_mc_theta.py"""
import json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from stochvolmodels_b200 import LOGSV_BTC_PARAMS, HestonParams, HestonPricer, LogSVPricer, OptionChain, get_btc_test_chain_data


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


chain = get_btc_test_chain_data()
bumped = []
for m in range(len(chain.ttms)):
    for s in (1.0, -1.0):
        t = np.array(chain.ttms, dtype=np.float64)
        t[m] += s * 1e-4
        bumped.append(OptionChain(ttms=t, forwards=chain.forwards, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                                  discfactors=chain.discfactors))
cases = {"logsv": (LogSVPricer(), LOGSV_BTC_PARAMS, dict(nb_path=10_000_000, nb_steps=582, seed=10)),
         "heston": (HestonPricer(), HestonParams(), dict(nb_path=10_000_000, seed=10))}
for model, (pricer, params, kw) in cases.items():
    variants = {"greeks": lambda: pricer.model_mc_chain_greeks(chain, params, **kw),
                "greeks_theta": lambda: pricer.model_mc_chain_greeks(chain, params, with_theta=True, **kw),
                "crn_2m_pricings": lambda: [pricer.model_mc_price_chain(c, params, **kw) for c in bumped]}
    times = {k: [] for k in variants}
    for fn in variants.values():
        fn()
    for _ in range(5):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            t = time.perf_counter(); fn(); times[k].append(time.perf_counter() - t)
    ms = {k: 1e3 * statistics.median(v) for k, v in times.items()}
    print(json.dumps({"workload": f"{model} MC, BTC chain {len(chain.ttms)} maturities, 1e7 paths", **{f"{k}_ms": v for k, v in ms.items()},
                      "theta_overhead": ms["greeks_theta"] / ms["greeks"] - 1.0,
                      "spread_ms": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in times.items()},
                      "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}), flush=True)

# rough-LogSV: the reference's H = 0.1 three-factor fixture, 1e6 Philox paths at 360 steps per year; every maturity restarts at t = 0, so a
# bumped theta needs 2 pricings (all ttms moved at once)
from stochvolmodels_b200 import LogSvParams
g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "rough_mc_reference_regression.npz"))
sigma0, theta, kappa1, kappa2, beta, volvol, H = g["params"]
rp = LogSvParams(sigma0=sigma0, theta=theta, kappa1=kappa1, kappa2=kappa2, beta=beta, volvol=volvol, H=H, weights=g["weights"], nodes=g["nodes"])
pricer, kw = LogSVPricer(), dict(nb_path=1_000_000, nb_steps=360, seed=10, gauss="fp32")
moved = [OptionChain(ttms=chain.ttms + s * 1e-4, forwards=chain.forwards, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                     discfactors=chain.discfactors) for s in (1.0, -1.0)]
variants = {"greeks": lambda: pricer.rough_mc_chain_greeks(chain, rp, **kw),
            "greeks_theta": lambda: pricer.rough_mc_chain_greeks(chain, rp, with_theta=True, **kw),
            "crn_2_pricings": lambda: [pricer.model_mc_price_chain(c, rp, use_rough_mc=True, distributed=False, **kw) for c in moved]}
times = {k: [] for k in variants}
for fn in variants.values():
    fn()
for _ in range(5):
    for k, fn in variants.items():
        torch.cuda.synchronize()
        t = time.perf_counter(); fn(); times[k].append(time.perf_counter() - t)
ms = {k: 1e3 * statistics.median(v) for k, v in times.items()}
print(json.dumps({"workload": f"rough-LogSV MC (3 factors, H = 0.1), BTC chain {len(chain.ttms)} maturities, 1e6 paths, 360 steps/yr",
                  **{f"{k}_ms": v for k, v in ms.items()}, "theta_overhead": ms["greeks_theta"] / ms["greeks"] - 1.0,
                  "spread_ms": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in times.items()},
                  "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}), flush=True)
