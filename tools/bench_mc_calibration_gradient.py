"""Cost of the calibration gradient on the Monte Carlo engines (DESIGN.md §4.7): SLSQP's forward difference (n + 1 = 6 pricings per
evaluation for PARAMS5) against gradient='pathwise' (one tangent pass).  Workload: the BTC sample chain, PARAMS5, 1e5 paths; MC with the
RandomState normals resident in HBM ('numpy') and with Philox ('philox') at 360 steps per year, ROUGH_MC at H = 0.45 (the two-node kernel
of tests/test_gpu_rough.py) at 120 steps per year.  Per route: the median over 7 of one objective + gradient evaluation at a fresh point
(host clock around a call that ends in a device synchronise, after 2 warm-up evaluations), then one full fit per gradient with nit,
nb_batches, wall time and the final objective.  One JSON line, with the card name and power limit the numbers were measured at.
   python tools/bench_mc_calibration_gradient.py"""
import json, os, statistics, subprocess, sys, time
from types import SimpleNamespace
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from stochvolmodels_b200 import CalibrationEngine, LogSvParams, LogSVPricer, LogsvModelCalibrationType, get_btc_test_chain_data
from stochvolmodels_b200.pricers import calibration


def power_limit_w():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                           timeout=10)
        return float(q.stdout.strip().splitlines()[0])
    except Exception:
        return None


W2, X2 = np.array([0.80082171, 0.34941995]), np.array([0.0015625, 1.31611315])
ROUTES = {"mc_numpy": dict(calibration_engine=CalibrationEngine.MC, mc_randoms="numpy", nb_steps=360),
          "mc_philox": dict(calibration_engine=CalibrationEngine.MC, mc_randoms="philox", nb_steps=360),
          "rough_mc_h045": dict(calibration_engine=CalibrationEngine.ROUGH_MC, mc_randoms="numpy", nb_steps=120)}
chain, pricer = get_btc_test_chain_data(), LogSVPricer()
start = LogSvParams(sigma0=0.8, theta=1.0, kappa1=3.0, kappa2=None, beta=0.1, volvol=1.8, H=0.45, weights=W2, nodes=X2)
common = dict(model_calibration_type=LogsvModelCalibrationType.PARAMS5, nb_path=100_000, seed=10, return_info=True)
run_slsqp = calibration.run_slsqp


def objective(route, gradient):
    """the objective calibrate_logsv hands SLSQP, taken at that call (the optimizer is not run)"""
    seen = {}

    def capture(obj, p0, bounds, constraints=None, disp=False):
        seen.update(obj=obj, p0=np.asarray(p0, dtype=float))
        return np.asarray(p0, dtype=float), SimpleNamespace(fun=np.nan, nit=0)

    calibration.run_slsqp = capture
    try:
        pricer.calibrate_model_params_to_chain(chain, start, gradient=gradient, **ROUTES[route], **common)
    finally:
        calibration.run_slsqp = run_slsqp
    return seen["obj"], seen["p0"]


def evaluation_ms(obj, p0, reps=7, warmup=2):
    times = []
    for r in range(warmup + reps):
        x = p0 * (1.0 + 1e-9 * (r + 1))            # a fresh point: the objective memoises the last one
        torch.cuda.synchronize()
        t = time.perf_counter()
        obj.fun(x)
        obj.jac(x)
        torch.cuda.synchronize()
        if r >= warmup:
            times.append(1e3 * (time.perf_counter() - t))
    return statistics.median(times)


out = {"card": {"name": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}, "evaluation_ms": {}, "fit": {}}
for route in ROUTES:
    out["evaluation_ms"][route] = {g: round(evaluation_ms(*objective(route, g)), 3) for g in ("difference", "pathwise")}
    for gradient in ("difference", "pathwise"):
        torch.cuda.synchronize()
        t = time.perf_counter()
        _, info = pricer.calibrate_model_params_to_chain(chain, start, gradient=gradient, **ROUTES[route], **common)
        torch.cuda.synchronize()
        out["fit"][f"{route}/{gradient}"] = {"nit": info["nit"], "nb_batches": info["nb_batches"], "wall_s": round(time.perf_counter() - t, 3),
                                             "fun": info["fun"]}
print(json.dumps(out))
