"""Cost of the Monte Carlo gamma (DESIGN.md §3.9): LogSV MC on the BTC chain, 1e7 paths x 252 steps (nb_steps_per_year=582), public API
with host buffers, median of 5 calls after one warm-up each, the variants alternated call by call.  Times the greeks pass without and with
gamma, and the three common-random-number pricings (forward at 1 and 1 +- h) a bumped gamma needs.  One JSON line with the times, the
gamma overhead, and the card name and power limit the numbers were measured at.
   python tools/bench_mc_gamma.py"""
import json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, OptionChain, get_btc_test_chain_data


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


chain, pricer = get_btc_test_chain_data(), LogSVPricer()
kw = dict(nb_path=10_000_000, nb_steps=582, seed=10)
bumped = [OptionChain(ttms=chain.ttms, forwards=chain.forwards * f, strikes_ttms=chain.strikes_ttms, optiontypes_ttms=chain.optiontypes_ttms,
                      discfactors=chain.discfactors) for f in (1.01, 1.0, 0.99)]
variants = {"greeks": lambda: pricer.model_mc_chain_greeks(chain, LOGSV_BTC_PARAMS, **kw),
            "greeks_gamma": lambda: pricer.model_mc_chain_greeks(chain, LOGSV_BTC_PARAMS, with_gamma=True, **kw),
            "crn_3_pricings": lambda: [pricer.model_mc_price_chain(c, LOGSV_BTC_PARAMS, **kw) for c in bumped]}
times = {k: [] for k in variants}
for fn in variants.values():
    fn()
for _ in range(5):
    for k, fn in variants.items():
        t = time.perf_counter(); fn(); times[k].append(time.perf_counter() - t)
ms = {k: 1e3 * statistics.median(v) for k, v in times.items()}
print(json.dumps({"workload": "LogSV MC, BTC chain 4 maturities x 49 strikes, 1e7 paths x 252 steps", **{f"{k}_ms": v for k, v in ms.items()},
                  "gamma_overhead": ms["greeks_gamma"] / ms["greeks"] - 1.0, "spread_ms": {k: [1e3 * min(v), 1e3 * max(v)] for k, v in times.items()},
                  "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}))
