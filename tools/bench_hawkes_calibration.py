"""The Hawkes calibration objective on the batched chain pricer against the sequential one (DESIGN.md §8), on the BTC chain (4 x 49) and on
the 3 x 12 synthetic market of tests/test_gpu_hawkes.py.  Every case is warmed up, then old and new alternate in the same process and the
median of 30 calls of each is reported:
  point  -- a point and its difference neighbours: B = 9 sets (model parameters) or B = 3 with gammas (risk premia), one
            hawkesjd_price_chain_batch call against B sequential compute_model_ivols_for_chain calls
  batch  -- hawkesjd_price_chain_batch alone (prices and fused implied vols) at B = 1, 9, 33, 129, both routes
  fit    -- one calibrate_model_params_to_chain (maxiter = 60) and one calibrate_risk_premia_gamma_to_chain, against the sequential oracle
            (scipy differencing the one-set objective; tests/hawkes_sequential.py), with a check that both return the same parameters
One JSON line per case with the card name and power limit read in the same run.
   python tools/bench_hawkes_calibration.py"""
import json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain, engine, get_btc_test_chain_data
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
import hawkes_sequential as seq

REPS = 30


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


CARD = None


def emit(row):
    print(json.dumps({**row, "card": CARD}), flush=True)


def alternate(old, new, reps=REPS):
    """medians (s) of ``reps`` calls of each, old and new alternating, after one warm-up call of each; every call ends in a host copy"""
    old(), new()
    to, tn = [], []
    for _ in range(reps):
        t = time.perf_counter(); old(); to.append(time.perf_counter() - t)
        t = time.perf_counter(); new(); tn.append(time.perf_counter() - t)
    return statistics.median(to), statistics.median(tn)


def timed(fn, reps=REPS):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def synthetic_market():
    K = np.linspace(0.75, 1.3, 12)
    ttms, fw = np.array([0.08, 0.25, 0.5]), np.ones(3)
    mk = lambda vols: OptionChain(ttms=ttms, forwards=fw, strikes_ttms=[K] * 3, optiontypes_ttms=[np.where(K >= 1.0, "C", "P")] * 3,
                                  ids=np.array(["1m", "3m", "6m"]), bid_ivs=vols, ask_ivs=[v.copy() for v in vols])
    pricer = HawkesJDPricer()
    true = HawkesJDParams(sigma=0.4, mean_p=0.04, mean_m=-0.05, theta_p=6.0, theta_m=8.0, kappa_p=25.0, kappa_m=25.0, beta1_p=30.0, beta2_p=-30.0,
                          beta1_m=40.0, beta2_m=-40.0)
    flat = mk([0.5 * np.ones_like(K)] * 3)
    return mk(pricer.compute_model_ivols_for_chain(flat, true)), mk(pricer.compute_model_ivols_for_chain(flat, HawkesJDParams(sigma=0.42, risk_premia_gamma=0.5)))


START = HawkesJDParams(sigma=0.45, mean_p=0.03, mean_m=-0.04, theta_p=7.0, theta_m=7.0, kappa_p=22.0, kappa_m=28.0, beta1_p=33.0, beta2_p=-33.0,
                       beta1_m=36.0, beta2_m=-36.0)
START_G = HawkesJDParams(sigma=0.45, risk_premia_gamma=0.2)


def neighbours(base, n, gamma=None):
    """n + 1 parameter sets: base and n small moves of it (a difference batch)"""
    d = {k: v for k, v in base.to_dict().items() if k != "risk_premia_gamma"}
    keys = ["sigma", "mean_p", "mean_m", "theta_p", "theta_m", "kappa_p", "beta1_p", "beta1_m"]
    out = [HawkesJDParams(**d, risk_premia_gamma=gamma)]
    for i in range(n):
        k = keys[i % len(keys)]
        out.append(HawkesJDParams(**{**d, k: d[k] * (1.0 + 1e-6 * (1 + i // len(keys)))}, risk_premia_gamma=None if gamma is None else gamma + 1e-3 * i))
    return out


def run_chain(label, chain, chain_g):
    pricer = HawkesJDPricer()
    args = (chain.ttms, chain.forwards, chain.discfactors, chain.strikes_ttms, chain.optiontypes_ttms)
    J = sum(len(k) for k in chain.strikes_ttms)
    for B, gamma in ((9, None), (3, 0.3)):
        sets = neighbours(START if gamma is None else START_G, B - 1, gamma)
        pcs = [_params_c(**s.to_dict()) for s in sets]
        gammas = None if gamma is None else [s.risk_premia_gamma for s in sets]
        seq_rows = np.vstack([np.concatenate(pricer.compute_model_ivols_for_chain(chain, s)) for s in sets])
        same = bool(np.array_equal(engine.hawkesjd_price_chain_batch(pcs, *args, gammas=gammas)[1], seq_rows, equal_nan=True))
        old, new = alternate(lambda: [pricer.compute_model_ivols_for_chain(chain, s) for s in sets],
                             lambda: engine.hawkesjd_price_chain_batch(pcs, *args, gammas=gammas))
        emit({"case": "point", "chain": label, "M": len(chain.ttms), "J": J, "B": B, "risk_kernel": gamma is not None, "sequential_ms": 1e3 * old,
              "batch_ms": 1e3 * new, "speedup": old / new, "bitwise_equal": same})
    for gamma in (None, 0.3):
        for B in (1, 9, 33, 129):
            sets = neighbours(START if gamma is None else START_G, B - 1, gamma)
            pcs = [_params_c(**s.to_dict()) for s in sets]
            gammas = None if gamma is None else [s.risk_premia_gamma for s in sets]
            t = timed(lambda: engine.hawkesjd_price_chain_batch(pcs, *args, gammas=gammas))
            emit({"case": "batch", "chain": label, "J": J, "B": B, "risk_kernel": gamma is not None, "batch_ms": 1e3 * t,
                  "per_set_us": 1e6 * t / B})
    fits = {}

    def model_old():
        fits["old"] = seq.calibrate_model_params(pricer, chain, START, maxiter=60)

    def model_new():
        fits["new"] = pricer.calibrate_model_params_to_chain(chain, START, maxiter=60, return_info=True)
    old, new = alternate(model_old, model_new)
    (ref, res), (fit, info) = fits["old"], fits["new"]
    emit({"case": "fit_model_params", "chain": label, "sequential_ms": 1e3 * old, "batched_ms": 1e3 * new, "speedup": old / new,
          "nit": info["nit"], "nb_batches": info["nb_batches"], "same_fit": bool(fit == ref and np.array_equal(info["x"], res.x))})

    def gamma_old():
        fits["old"] = seq.calibrate_risk_premia_gamma(pricer, chain_g, START_G, print_iter=False)

    def gamma_new():
        fits["new"] = pricer.calibrate_risk_premia_gamma_to_chain(chain_g, START_G, print_iter=False, return_info=True)
    old, new = alternate(gamma_old, gamma_new)
    (ref, res), (fit, info) = fits["old"], fits["new"]
    emit({"case": "fit_risk_premia_gamma", "chain": label, "sequential_ms": 1e3 * old, "batched_ms": 1e3 * new, "speedup": old / new,
          "nit": info["nit"], "nb_batches": info["nb_batches"], "same_fit": bool(fit == ref and np.array_equal(info["x"], res.x))})


if __name__ == "__main__":
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing to measure")
    CARD = {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    btc = get_btc_test_chain_data()
    run_chain("btc_4x49", btc, btc)
    run_chain("synthetic_3x12", *synthetic_market())
