"""Monte Carlo sensitivities of the Hawkes jump-diffusion chain against the alternatives (DESIGN.md §3.11): BTC chain, default
HawkesJDParams, fp32 draws, engine level, median of 3 calls after one warm-up each:
  greeks   -- engine.hawkesjd_mc_chain_greeks (prices, delta and the 15 parameter rows with standard errors, one pass)
  price    -- engine.hawkesjd_mc_chain (what model_mc_price_chain runs)
  crn31    -- 31 engine.hawkesjd_mc_chain calls on the same seed (base + 2 x 15 bumps: central bump-and-reprice)
at 1e6 and 1e7 paths.  One JSON line per case with the card name and power limit read in the same run.
   python tools/bench_hawkes_greeks.py"""
import json, os, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from stochvolmodels_b200 import HawkesJDParams, engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c

SEED = 10


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


def case(chain, nb_path):
    d = HawkesJDParams().to_dict()
    d.pop("risk_premia_gamma")
    flags = engine.mc_flags("fp64", "fp32")
    args = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms, nb_path, 1, SEED, flags)
    sets = [d] + [{**d, k: d[k] + s * 0.01 * max(abs(d[k]), 0.05)} for k in engine.HAWKES_GREEK_PARAMS for s in (1.0, -1.0)]
    greeks = timed(lambda: engine.hawkesjd_mc_chain_greeks(_params_c(**d), *args))
    price = timed(lambda: engine.hawkesjd_mc_chain(_params_c(**d), *args))
    crn = timed(lambda: [engine.hawkesjd_mc_chain(_params_c(**p), *args) for p in sets])
    return {"nb_path": nb_path, "greeks_ms": 1e3 * greeks, "price_ms": 1e3 * price, "crn31_ms": 1e3 * crn,
            "greeks_over_price": greeks / price, "crn31_over_greeks": crn / greeks,
            "card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}}


if __name__ == "__main__":
    chain = get_btc_test_chain_data()
    for nb_path in (1_000_000, 10_000_000):
        print(json.dumps(case(chain, nb_path)), flush=True)
