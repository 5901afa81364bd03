"""The Hawkes calibration drivers as they were before the batched pricer: scipy SLSQP differences a one-set-at-a-time objective
(``compute_model_ivols_for_chain`` per point) itself.  The tests hold the batched drivers to this oracle bit for bit."""
import numpy as np
from scipy.optimize import minimize

from stochvolmodels_b200 import HawkesJDParams
from stochvolmodels_b200.pricers.hawkes_jd_pricer import _KEYS


def vol_objective(pricer, option_chain, unpack, is_vega_weighted=True, is_unit_ttm_vega=False, scale=1.0):
    market = np.concatenate([np.asarray(v, dtype=float) for v in option_chain.get_mid_vols()])
    if is_vega_weighted:
        weights = np.concatenate([v / np.sum(v) for v in option_chain.get_chain_vegas(is_unit_ttm_vega=is_unit_ttm_vega)])
    else:
        weights = np.ones_like(market)

    def objective(pars, *_):
        model = np.concatenate(pricer.compute_model_ivols_for_chain(option_chain=option_chain, params=unpack(pars)))
        return float(np.nansum(scale * weights * np.square(model - market)))
    return objective


MODEL_BOUNDS = ((0.10, 2.0), (0.01, 0.99), (-0.99, -0.01), (0.01, 100.0), (0.01, 100.0), (1.0, 100.0), (1.0, 100.0), (1.0, 100.0))
GAMMA_BOUNDS = ((0.01, 1.5), (-1.0, 1.0))


def model_unpack(params0):
    def unpack(x):
        return HawkesJDParams(mu=0.0, sigma=x[0], shift_p=params0.shift_p, mean_p=x[1], shift_m=params0.shift_m, mean_m=x[2],
                              lambda_p=params0.lambda_p, theta_p=x[3], kappa_p=x[5], beta1_p=x[6], beta2_p=-x[6], lambda_m=params0.lambda_m,
                              theta_m=x[4], kappa_m=x[5], beta1_m=x[7], beta2_m=-x[7])
    return unpack


def calibrate_model_params(pricer, option_chain, params0, maxiter=None):
    """-> (fit, scipy result)"""
    p0 = np.array([params0.sigma, params0.mean_p, params0.mean_m, params0.theta_p, params0.theta_m, 0.5 * (params0.kappa_p + params0.kappa_m),
                   0.5 * (params0.beta1_p - params0.beta2_p), 0.5 * (params0.beta2_p - params0.beta2_m)])
    unpack = model_unpack(params0)
    stationary = {"type": "ineq", "fun": lambda x: unpack(x).jump1_cond + unpack(x).jump2_cond}
    options = {"disp": False, "ftol": 1e-8}
    if maxiter is not None:
        options["maxiter"] = int(maxiter)
    res = minimize(vol_objective(pricer, option_chain, unpack), p0, args=None, method="SLSQP", constraints=stationary, bounds=MODEL_BOUNDS,
                   options=options)
    return unpack(res.x), res


def calibrate_risk_premia_gamma(pricer, option_chain, params0, maxiter=100, print_iter=True):
    """-> (fit, scipy result)"""
    gamma_scaler = 8.0
    fixed = {k: v for k, v in params0.to_dict().items() if k in _KEYS}

    def unpack(x):
        if print_iter:
            print(f"unpack_pars: sigma={x[0]}, gamma={gamma_scaler * x[1]}")
        return HawkesJDParams(**{**fixed, "sigma": float(x[0])}, risk_premia_gamma=float(gamma_scaler * x[1]))

    p0 = np.array([params0.sigma, (params0.risk_premia_gamma or 0.0) / gamma_scaler])
    res = minimize(vol_objective(pricer, option_chain, unpack, scale=10000.0), p0, args=None, method="SLSQP", bounds=GAMMA_BOUNDS,
                   options={"disp": False, "ftol": 1e-16, "maxiter": maxiter, "eps": 0.025}, tol=1e-16)
    return unpack(res.x), res


def batches(res, n):
    """pricing calls of the batched objective for the same run: one per point SLSQP asked the value of (every evaluation minus the n
    difference points of each gradient), one per gradient"""
    return res.nfev - n * res.njev + res.njev
