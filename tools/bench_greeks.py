"""Pathwise sensitivities against a price-only chain (DESIGN.md §3.9, §8): LogSV MC on the BTC chain, 1e7 paths x 252 steps
(nb_steps_per_year=582 -> 25+34+57+136), public API with host buffers, median of 3 calls after one warm-up each.  One JSON line with both wall
times, their ratio, and the card name and power limit the numbers were measured at.
   python tools/bench_greeks.py"""
import json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from stochvolmodels_b200 import LOGSV_BTC_PARAMS, LogSVPricer, get_btc_test_chain_data


def timed(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts), out


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


chain, pricer = get_btc_test_chain_data(), LogSVPricer()
kw = dict(nb_path=10_000_000, nb_steps=582, seed=10)
secs_p, _ = timed(lambda: pricer.model_mc_price_chain(chain, LOGSV_BTC_PARAMS, **kw))
secs_g, res = timed(lambda: pricer.model_mc_chain_greeks(chain, LOGSV_BTC_PARAMS, **kw))
print(json.dumps({"workload": "LogSV MC, BTC chain 4 maturities x 49 strikes, 1e7 paths x 252 steps", "greeks_ms": 1e3 * secs_g,
                  "price_ms": 1e3 * secs_p, "ratio": secs_g / secs_p, "n_sensitivities": 1 + len(res.params),
                  "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}))
