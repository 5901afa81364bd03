"""Calibration drivers on top of the batched GPU chain pricers (SURVEY.md §8f "next" #2).

Mirrors ``LogSVPricer.calibrate_model_params_to_chain`` (reference pricers/logsv_pricer.py:441-558 with the codec :103-193, the
weights :196-207, the objective :222-294 and the constraints :297-330) and ``HestonPricer.calibrate_model_params_to_chain``
(pricers/heston_pricer.py:111-180): same arguments, bounds, objective (vega-weighted squared implied-vol errors, ``nansum``), SLSQP
with ``ftol=1e-8``, result validation and return type.

What is different is how the optimizer gets its numbers.  The reference lets scipy difference the objective: n+1 sequential chain
pricings (~2 s each on the CPU) per SLSQP iteration.  Here every evaluation point x is priced TOGETHER with its n forward-difference
neighbours x + h e_i as ONE batch of n+1 parameter sets (``b200sv_logsv_price_chain_batch``: (n+1) x 1000 ODE threads, Fourier sums
and the Black inversion fused, one launch pair, one D2H copy), so the objective and its gradient cost one ~1 ms GPU call.  The step is
SLSQP's own default (``eps = 1.4901161193847656e-08``, absolute, flipped at an upper bound), so the gradient is the number scipy would
have computed from the same objective.

The MC engine (:251-266) has two sources of fixed normals: ``mc_randoms="numpy"`` (default) draws them exactly as the reference does
(``np.random.RandomState(seed)``, :1051-1074), keeps them resident in HBM (``DeviceRandoms``) and prices each of the n+1 sets with the
fixed-random stepper -- the same objective values as the reference for the same seed; ``mc_randoms="philox"`` prices the n+1 sets in one
``b200sv_logsv_mc_chain_batch`` call in which the counter-based generator re-draws identical normals for every set (nothing stored or
streamed; statistically equivalent objective, different sample).

``gradient='exact'`` (ANALYTIC engine) and ``gradient='pathwise'`` (MC and ROUGH_MC engines) replace the difference by one sensitivity call
per point through ``ExactGradientObjective``: the Fourier implied-vol sensitivities (DESIGN.md §4.6), resp. the pathwise Monte Carlo
sensitivities on the fit's fixed normals mapped to implied-vol rows (§4.7) -- the exact derivative of the sample objective the difference
route approximates, with no step size.

Quotes whose model price falls outside the no-arbitrage bounds have no implied vol: the GPU inversion returns NaN for them and the
objective's ``nansum`` (the reference's own reduction, :292-294) leaves them out of that evaluation, exactly as the reference does with the NaNs
of its third-party inverter.  Which quotes that inverter would flag is not pinned (the package is absent, DESIGN.md 2); ``BatchedObjective``
counts the skipped quotes per evaluation in ``nan_quotes`` so that a caller can see when a fit was driven by a shrinking set of quotes.
"""
from __future__ import annotations

import threading
from dataclasses import dataclass
from enum import Enum
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from .. import engine
from ..utils.funcs import to_flat_np_array

SLSQP_EPS = 1.4901161193847656e-08      # scipy.optimize._slsqp_py default `eps` (sqrt of the double epsilon)


class LogsvModelCalibrationType(Enum):
    """which parameters the calibration solves for (reference logsv_pricer.py:56-68)."""
    PARAMS4 = 1                  # sigma0, theta, beta, volvol; kappa1, kappa2 fixed
    PARAMS5 = 2                  # sigma0, theta, kappa1, beta, volvol; kappa2 = kappa1 / theta
    PARAMS6 = 3
    PARAMS_WITH_VARSWAP_FIT = 4  # beta, volvol; the eta backbone is re-fitted to the chain's variance-swap strikes at every point


class ConstraintsType(Enum):
    """parameter constraints (reference :71-90)."""
    UNCONSTRAINT = 1
    MMA_MARTINGALE = 2               # kappa2 >= beta
    INVERSE_MARTINGALE = 3           # kappa2 >= 2 beta
    MMA_MARTINGALE_MOMENT4 = 4       # + kappa >= 1.5 vartheta^2
    INVERSE_MARTINGALE_MOMENT4 = 5


class CalibrationEngine(Enum):
    """how model vols are produced inside the objective (reference :93-102)."""
    ANALYTIC = 1
    MC = 2
    ROUGH_MC = 3                     # rough-LogSV multi-factor MC with fixed normals (reference logsv_pricer.py:266-289)


class CalibrationError(RuntimeError):
    """raised when the optimizer fails or returns an unusable vector (reference pricers/model_pricer.py:44-80)."""


def validate_optimization_result(result, bounds) -> np.ndarray:
    """the optimizer's vector as float64[len(bounds)], or ``CalibrationError`` naming what is wrong with it.

    Same acceptance rule and error wording as the reference's guard (pricers/model_pricer.py:48-80: success flag, numeric 1-d vector
    of the right length, finite, inside the bounds up to 1e-10) -- callers match on the message text."""
    note = str(getattr(result, "message", "no optimizer message"))

    def reject(what: str, cause=None):
        raise CalibrationError(f"Calibration {what}: {note}") from cause

    if not getattr(result, "success", False):
        reject("failed")
    x = getattr(result, "x", None)
    if x is None:
        reject("returned no parameter vector")
    try:
        x = np.array(x, dtype=np.float64, copy=True)
    except (TypeError, ValueError) as exc:
        reject("returned a non-numeric parameter vector", exc)
    if x.shape != (len(bounds),):
        reject("returned a parameter vector with the wrong shape")
    if not np.isfinite(x).all():
        reject("returned non-finite parameters")
    slack = 1.0e-10
    lo = np.array([-np.inf if b[0] is None else b[0] for b in bounds], dtype=np.float64)
    hi = np.array([np.inf if b[1] is None else b[1] for b in bounds], dtype=np.float64)
    if (x < lo - slack).any():
        reject("returned parameters below bounds")
    if (x > hi + slack).any():
        reject("returned parameters above bounds")
    return x


def calibration_weights(option_chain, market_vols: np.ndarray, is_vega_weighted: bool, is_unit_ttm_vega: bool) -> np.ndarray:
    """flattened objective weights: per-slice normalised Black vegas or ones (reference logsv_pricer.py:196-207)."""
    if not is_vega_weighted:
        return np.ones_like(market_vols)
    vegas_ttms = option_chain.get_chain_vegas(is_unit_ttm_vega=is_unit_ttm_vega)
    return to_flat_np_array([v / sum(v) for v in vegas_ttms])


@dataclass
class BatchedObjective:
    """objective + forward-difference gradient from ONE batched evaluation, memoised on the last point so that SLSQP's separate
    ``fun(x)`` / ``jac(x)`` calls share it.  ``batch_vols(points [B, n]) -> model vols [B, J]``."""
    batch_vols: Callable[[np.ndarray], np.ndarray]
    market_vols: np.ndarray
    weights: np.ndarray
    bounds: Sequence[Tuple[float, float]]
    eps: float = SLSQP_EPS
    nb_batches: int = 0
    nan_quotes: int = 0          # quotes without an implied vol at the LAST evaluation point (dropped there by nansum, as in the reference)
    _x: Optional[np.ndarray] = None
    _f: float = np.nan
    _g: Optional[np.ndarray] = None

    def steps(self, x: np.ndarray) -> np.ndarray:
        """+eps, or -eps where x + eps would leave the box (scipy approx_derivative's one-sided bound handling)."""
        ub = np.array([np.inf if b[1] is None else b[1] for b in self.bounds], dtype=float)
        return np.where(x + self.eps > ub, -self.eps, self.eps)

    def values(self, vols: np.ndarray) -> np.ndarray:
        return np.nansum(self.weights[None, :] * np.square(vols - self.market_vols[None, :]), axis=1)

    def _evaluate(self, x: np.ndarray) -> None:
        x = np.asarray(x, dtype=float)
        if self._x is not None and np.array_equal(x, self._x):
            return
        h = self.steps(x)
        pts = np.vstack([x[None, :], x[None, :] + np.diag(h)])
        vols = self.batch_vols(pts)
        f = self.values(vols)
        self.nb_batches += 1
        self.nan_quotes = int(np.count_nonzero(np.isnan(vols[0])))
        self._x, self._f, self._g = x.copy(), float(f[0]), (f[1:] - f[0]) / h

    def fun(self, x: np.ndarray, *args) -> float:
        self._evaluate(x)
        return self._f

    def jac(self, x: np.ndarray, *args) -> np.ndarray:
        self._evaluate(x)
        return self._g.copy()


def scipy_difference_steps(x: np.ndarray, eps: float, bounds) -> np.ndarray:
    """the steps h of scipy's 2-point ``approx_derivative(abs_step=eps, bounds=bounds)`` -- what SLSQP differences an objective with when it
    is given no ``jac``: eps, a relative step sqrt(machine eps) sign(x) max(1, |x|) where x + eps == x, then the one-sided bound handling of
    ``_adjust_scheme_to_bounds``: flipped where x + h leaves the box and -h fits, else the distance to the farther bound."""
    lb = np.array([-np.inf if b[0] is None else b[0] for b in bounds], dtype=float)
    ub = np.array([np.inf if b[1] is None else b[1] for b in bounds], dtype=float)
    sign = (x >= 0).astype(x.dtype) * 2 - 1
    h = np.where(((x + eps) - x) == 0, SLSQP_EPS * sign * np.maximum(1.0, np.abs(x)), eps).astype(x.dtype)
    if np.all((lb == -np.inf) & (ub == np.inf)):
        return h
    lower, upper = x - lb, ub - x
    xh = x + h
    fitting = np.abs(h) <= np.maximum(lower, upper)
    h[((xh < lb) | (xh > ub)) & fitting] *= -1
    forward = (upper >= lower) & ~fitting
    h[forward] = upper[forward]
    backward = (upper < lower) & ~fitting
    h[backward] = -lower[backward]
    return h


@dataclass
class ScipyDifferenceObjective:
    """objective + the gradient scipy would difference from it (scipy_difference_steps), memoised on the last point.  ``fun(x)`` prices x
    alone; ``jac(x)`` prices its n neighbours x + h_i e_i together in ONE batch, so a point SLSQP only asks the value of (a line-search
    trial) costs one set, and every set is priced once.  Each row is reduced with the sequential objective's own expression
    (``nansum(weights * (vols - market)^2)``, ``weights`` with any scale folded in), the neighbours are built as scipy builds them (a copy of
    x with one coordinate moved) and the divisor is dx = (x + h) - x, so ``fun`` / ``jac`` return bit for bit what SLSQP computes from a
    one-set-at-a-time objective.  ``on_point(x)``, if given, sees the points in the order that objective would have been evaluated: x on
    ``fun``, its neighbours on ``jac``.  ``batch_vols(points [B, n]) -> model vols [B, J]``; ``nb_batches`` counts its calls."""
    batch_vols: Callable[[np.ndarray], np.ndarray]
    market_vols: np.ndarray
    weights: np.ndarray
    bounds: Sequence[Tuple[float, float]]
    eps: float = SLSQP_EPS
    on_point: Optional[Callable[[np.ndarray], None]] = None
    nb_batches: int = 0
    nan_quotes: int = 0          # quotes without an implied vol at the LAST point priced by fun (dropped there by nansum, as in the reference)
    _x: Optional[np.ndarray] = None
    _f: float = np.nan
    _g: Optional[np.ndarray] = None

    def _values(self, pts: np.ndarray) -> np.ndarray:
        vols = self.batch_vols(pts)
        self.nb_batches += 1
        return vols, [float(np.nansum(self.weights * np.square(v - self.market_vols))) for v in vols]

    def _value(self, x: np.ndarray) -> None:
        if self._x is not None and np.array_equal(x, self._x):
            return
        vols, f = self._values(x[None, :].copy())
        self.nan_quotes = int(np.count_nonzero(np.isnan(vols[0])))
        self._x, self._f, self._g = x.copy(), f[0], None

    def fun(self, x: np.ndarray, *args) -> float:
        x = np.asarray(x, dtype=float)
        self._value(x)
        if self.on_point is not None:
            self.on_point(x)
        return self._f

    def jac(self, x: np.ndarray, *args) -> np.ndarray:
        x = np.asarray(x, dtype=float)
        if self._x is None or not np.array_equal(x, self._x):
            self.fun(x)                                          # the one-set objective evaluates x before differencing at it
        if self._g is None:
            h = scipy_difference_steps(x, self.eps, self.bounds)
            pts = np.repeat(x[None, :], x.size, axis=0)
            for i in range(x.size):
                pts[i, i] = x[i] + h[i]
            if self.on_point is not None:
                for p in pts:
                    self.on_point(p)
            _, f = self._values(pts)
            self._g = np.array([(f[i] - self._f) / ((x[i] + h[i]) - x[i]) for i in range(x.size)])
        return self._g.copy()


GRADIENTS = ("difference", "exact", "pathwise")


def check_gradient(gradient: str, pathwise: bool = False) -> str:
    """the ``gradient`` argument of the calibration drivers: 'difference' (default: SLSQP's forward difference, priced as one batch),
    'exact' (ExactGradientObjective on the Fourier sensitivities) or 'pathwise' (ExactGradientObjective on the Monte Carlo sensitivities of
    the fixed normals; only drivers with a Monte Carlo engine pass ``pathwise=True``, the others reject it before any library call)"""
    if gradient not in GRADIENTS:
        raise ValueError("gradient must be 'difference', 'exact' or 'pathwise'")
    if gradient == "pathwise" and not pathwise:
        raise NotImplementedError("gradient='pathwise' covers LogSVPricer.calibrate_model_params_to_chain with CalibrationEngine.MC or ROUGH_MC "
                                  "(PARAMS4 / PARAMS5) only")
    return gradient


@dataclass
class ExactGradientObjective:
    """objective and its exact gradient from ONE implied-vol sensitivity evaluation, memoised on the last point so that SLSQP's ``fun(x)``
    and ``jac(x)`` share it (DESIGN.md §4.6).  ``ivol_greeks(x) -> (vols [J], dvols [F, J])``: the model vols at x and their derivatives
    in the pricer's F model fields (ModelPricer.compute_chain_ivol_greeks on a pinned transform grid); ``field_jacobian(x) -> D [F, n]``:
    d fields / d x of the parameter codec.  fun(x) = nansum(w (vol - market)^2); jac(x) = sum over the quotes with a finite vol of
    2 w (vol - market) D^T dvols.  ``nb_batches`` counts library calls (two per evaluation: the price sensitivities and their
    implied-vol transform)."""
    ivol_greeks: Callable[[np.ndarray], Tuple[np.ndarray, np.ndarray]]
    field_jacobian: Callable[[np.ndarray], np.ndarray]
    market_vols: np.ndarray
    weights: np.ndarray
    nb_batches: int = 0
    nan_quotes: int = 0          # quotes without an implied vol at the LAST evaluation point (dropped there by nansum, as in the reference)
    _x: Optional[np.ndarray] = None
    _f: float = np.nan
    _g: Optional[np.ndarray] = None

    CALLS_PER_EVALUATION = 2

    def _evaluate(self, x: np.ndarray) -> None:
        x = np.asarray(x, dtype=float)
        if self._x is not None and np.array_equal(x, self._x):
            return
        vols, dvols = self.ivol_greeks(x)
        self.nb_batches += self.CALLS_PER_EVALUATION
        finite = np.isfinite(vols)
        self.nan_quotes = int(np.count_nonzero(~finite))
        resid = vols - self.market_vols
        f = float(np.nansum(self.weights * np.square(resid)))
        g_fields = dvols[:, finite] @ (2.0 * self.weights[finite] * resid[finite])
        self._x, self._f, self._g = x.copy(), f, self.field_jacobian(x).T @ g_fields

    def fun(self, x: np.ndarray, *args) -> float:
        self._evaluate(x)
        return self._f

    def jac(self, x: np.ndarray, *args) -> np.ndarray:
        self._evaluate(x)
        return self._g.copy()


def flat_ivol_rows(sens, names: Sequence[str]) -> Tuple[np.ndarray, np.ndarray]:
    """ChainIvolGreeks -> (vols [J], d vols / d names [len(names), J]) flat in chain order"""
    return (to_flat_np_array(sens.ivols), np.vstack([to_flat_np_array(sens.params[n]) for n in names]))


def run_slsqp(objective: BatchedObjective, p0: np.ndarray, bounds, constraints=None, disp: bool = False):
    """``scipy.optimize.minimize(method='SLSQP', options={'ftol': 1e-8})`` as in the reference (:543-555), with the batched gradient."""
    from scipy.optimize import minimize      # host-side optimizer; scipy is already a dependency of the reference
    kwargs = dict(method="SLSQP", jac=objective.jac, bounds=bounds, options={"disp": disp, "ftol": 1e-8})
    if constraints is not None:
        kwargs["constraints"] = constraints
    result = minimize(objective.fun, np.asarray(p0, dtype=float), **kwargs)
    return validate_optimization_result(result, bounds), result


# ---- LogSV ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class LogSvParameterCodec:
    """optimizer vector <-> LogSvParams (reference _LogSvParameterCodec, :103-193)."""
    params0: "LogSvParams"
    params_min: "LogSvParams"
    params_max: "LogSvParams"
    calibration_type: LogsvModelCalibrationType
    varswap_strikes: object = None          # pandas Series (PARAMS_WITH_VARSWAP_FIT only)

    def parse(self, pars: np.ndarray):
        from .logsv.vol_moments import fit_vol_backbone_to_varswaps
        from .logsv_pricer import LogSvParams
        p0 = self.params0
        rough = dict(H=getattr(p0, "H", 0.5), nodes=getattr(p0, "nodes", None), weights=getattr(p0, "weights", None))   # reference :125-127
        if self.calibration_type == LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT:
            out = LogSvParams(sigma0=p0.sigma0, theta=p0.theta, kappa1=p0.kappa1, kappa2=p0.kappa2, beta=pars[0], volvol=pars[1], **rough)
            out.set_vol_backbone(fit_vol_backbone_to_varswaps(out, self.varswap_strikes))     # reference :145-160
            return out
        if self.calibration_type == LogsvModelCalibrationType.PARAMS4:
            out = LogSvParams(sigma0=pars[0], theta=pars[1], kappa1=p0.kappa1, kappa2=p0.kappa2, beta=pars[2], volvol=pars[3], **rough)
        elif self.calibration_type == LogsvModelCalibrationType.PARAMS5:
            out = LogSvParams(sigma0=pars[0], theta=pars[1], kappa1=pars[2], kappa2=None, beta=pars[3], volvol=pars[4], **rough)
        else:
            raise NotImplementedError(f"{self.calibration_type}")
        # no vol_backbone on the trial point: the reference codec (logsv_pricer.py:112-137) builds PARAMS4 / PARAMS5 candidates without
        # one, so eta = 1 during the fit and the fitted object carries none, whatever params0 holds
        return out

    def initial_and_bounds(self) -> Tuple[np.ndarray, Tuple[Tuple[float, float], ...]]:
        p0, lo, hi = self.params0, self.params_min, self.params_max
        if self.calibration_type == LogsvModelCalibrationType.PARAMS4:
            names = ("sigma0", "theta", "beta", "volvol")
        elif self.calibration_type == LogsvModelCalibrationType.PARAMS5:
            names = ("sigma0", "theta", "kappa1", "beta", "volvol")
        elif self.calibration_type == LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT:
            names = ("beta", "volvol")
        else:
            raise NotImplementedError(f"{self.calibration_type}")
        return (np.array([getattr(p0, n) for n in names], dtype=float),
                tuple((getattr(lo, n), getattr(hi, n)) for n in names))

    def field_jacobian(self, pars: np.ndarray) -> np.ndarray:
        """D [6, n] = d (sigma0, theta, kappa1, kappa2, beta, volvol) / d pars (engine.LOGSV_GREEK_PARAMS order), the chain rule of the
        exact gradient.  PARAMS5 sets kappa2 = kappa1 / theta while the price sensitivities hold kappa2 fixed, so d/d theta picks up
        -kappa1 / theta^2 d/d kappa2 and d/d kappa1 picks up d/d kappa2 / theta."""
        D = np.zeros((6, len(pars)))
        if self.calibration_type == LogsvModelCalibrationType.PARAMS4:
            for col, field in enumerate((0, 1, 4, 5)):
                D[field, col] = 1.0
        elif self.calibration_type == LogsvModelCalibrationType.PARAMS5:
            for col, field in enumerate((0, 1, 2, 4, 5)):
                D[field, col] = 1.0
            theta, kappa1 = pars[1], pars[2]
            D[3, 1] = -kappa1 / (theta * theta)
            D[3, 2] = 1.0 / theta
        else:
            raise NotImplementedError(f"exact gradient for {self.calibration_type}")
        return D


def build_logsv_constraints(codec: LogSvParameterCodec, constraints_type: ConstraintsType):
    """SLSQP inequality constraints of Theorem 3.7 (reference :297-330)."""
    def martingale_measure(pars):
        p = codec.parse(pars)
        return p.kappa2 - p.beta

    def inverse_measure(pars):
        p = codec.parse(pars)
        return p.kappa2 - 2.0 * p.beta

    def vol_4thmoment_finite(pars):
        p = codec.parse(pars)
        return (p.kappa1 + p.kappa2 * p.theta) - 1.5 * p.vartheta2

    if constraints_type == ConstraintsType.UNCONSTRAINT:
        return None
    if constraints_type == ConstraintsType.MMA_MARTINGALE:
        return {"type": "ineq", "fun": martingale_measure}
    if constraints_type == ConstraintsType.INVERSE_MARTINGALE:
        return {"type": "ineq", "fun": inverse_measure}
    if constraints_type == ConstraintsType.MMA_MARTINGALE_MOMENT4:
        return ({"type": "ineq", "fun": martingale_measure}, {"type": "ineq", "fun": vol_4thmoment_finite})
    if constraints_type == ConstraintsType.INVERSE_MARTINGALE_MOMENT4:
        return ({"type": "ineq", "fun": inverse_measure}, {"type": "ineq", "fun": vol_4thmoment_finite})
    raise NotImplementedError(f"{constraints_type}")


def calibrate_logsv(pricer, option_chain, params0, params_min, params_max, is_vega_weighted: bool, is_unit_ttm_vega: bool,
                    model_calibration_type: LogsvModelCalibrationType, constraints_type: ConstraintsType,
                    calibration_engine: CalibrationEngine, nb_path: int, nb_steps: int, seed: int, is_spot_measure: bool = True,
                    disp: bool = False, return_info: bool = False, fd_step: Optional[float] = None, mc_randoms: str = "numpy",
                    gradient: str = "difference", price_batch: Optional[Callable] = None):
    """``price_batch``: what the ANALYTIC difference objective prices its points with, engine.logsv_price_chain_batch (None) or a
    callable with its arguments and return value (the lock-step drivers of calibrate_chains_lockstep)"""
    if check_gradient(gradient, pathwise=True) == "exact":
        if calibration_engine != CalibrationEngine.ANALYTIC:
            raise NotImplementedError(f"gradient='exact' covers CalibrationEngine.ANALYTIC only, not {calibration_engine} "
                                      "(the Monte Carlo engines have gradient='pathwise')")
        if model_calibration_type not in (LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5):
            raise NotImplementedError(f"gradient='exact' covers PARAMS4 and PARAMS5 only, not {model_calibration_type} (the eta backbone "
                                      "of PARAMS_WITH_VARSWAP_FIT is refitted at every point and is not differentiated)")
    if gradient == "pathwise":
        if calibration_engine not in (CalibrationEngine.MC, CalibrationEngine.ROUGH_MC):
            raise NotImplementedError(f"gradient='pathwise' covers CalibrationEngine.MC and ROUGH_MC only, not {calibration_engine} "
                                      "(the ANALYTIC engine has gradient='exact')")
        if model_calibration_type not in (LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5):
            raise NotImplementedError(f"gradient='pathwise' covers PARAMS4 and PARAMS5 only, not {model_calibration_type} (the eta backbone "
                                      "of PARAMS_WITH_VARSWAP_FIT is refitted at every point and is not differentiated)")
    from ..multi_gpu import _fixed_randoms_chain_device
    from .fourier_greeks import to_chain_ivol_sensitivities
    from .logsv_pricer import DeviceRandoms, _params_c, get_randoms_for_chain_valuation, logsv_mc_chain_greeks_fixed_randoms
    from .mc_greeks import to_mc_chain_greeks
    vol_scaler = pricer.set_vol_scaler(option_chain=option_chain)
    _, market_vols_ttms = option_chain.get_chain_data_as_xy()
    market_vols = to_flat_np_array(market_vols_ttms)
    weights = calibration_weights(option_chain, market_vols, is_vega_weighted, is_unit_ttm_vega)
    varswap_strikes = (option_chain.get_slice_varswap_strikes(floor_with_atm_vols=True)
                       if model_calibration_type == LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT else None)
    codec = LogSvParameterCodec(params0, params_min, params_max, model_calibration_type, varswap_strikes)
    p0, bounds = codec.initial_and_bounds()
    ttms = option_chain.ttms
    resets = np.zeros(len(ttms), dtype=np.int64)       # ROUGH_MC pathwise: per maturity, the most paths any evaluation saw reset

    def mc_ivol_rows(res):
        """engine.*_mc_chain_greeks output -> (vols [J], d vols / d LOGSV_GREEK_PARAMS [6, J])"""
        sens = to_chain_ivol_sensitivities(option_chain, to_mc_chain_greeks(res, engine.LOGSV_GREEK_PARAMS))
        return flat_ivol_rows(sens, engine.LOGSV_GREEK_PARAMS)

    if gradient == "exact":
        # one compute_chain_ivol_greeks call per point, on the grid the difference route pins too (set_vol_scaler above)
        def ivol_greeks(x: np.ndarray):
            sens = pricer.compute_chain_ivol_greeks(option_chain, codec.parse(x), is_spot_measure=is_spot_measure, vol_scaler=vol_scaler)
            return flat_ivol_rows(sens, engine.LOGSV_GREEK_PARAMS)

        objective = ExactGradientObjective(ivol_greeks=ivol_greeks, field_jacobian=codec.field_jacobian, market_vols=market_vols,
                                           weights=weights)
    elif calibration_engine == CalibrationEngine.ANALYTIC:
        def batch_vols(points: np.ndarray) -> np.ndarray:
            sets = [codec.parse(p) for p in points]
            etas = np.array([s.get_vol_backbone_etas(ttms=ttms) for s in sets], dtype=float)
            _, ivols = (price_batch or engine.logsv_price_chain_batch)([_params_c(s) for s in sets], ttms, option_chain.forwards,
                                                                       option_chain.discfactors, etas, option_chain.strikes_ttms,
                                                                       option_chain.optiontypes_ttms, is_spot_measure=is_spot_measure,
                                                                       vol_scaler=vol_scaler)
            return ivols
    elif calibration_engine == CalibrationEngine.MC and mc_randoms == "philox":
        flags = engine.mc_flags("fp64", "fp32")

        def batch_vols(points: np.ndarray) -> np.ndarray:
            sets = [codec.parse(p) for p in points]
            etas = np.array([s.get_vol_backbone_etas(ttms=ttms) for s in sets], dtype=float)
            _, _, ivols = engine.logsv_mc_chain_batch([_params_c(s) for s in sets], ttms, option_chain.forwards, option_chain.discfactors, etas,
                                                      option_chain.strikes_ttms, option_chain.optiontypes_ttms, nb_path, nb_steps,
                                                      is_spot_measure, seed, flags)
            return ivols

        def ivol_greeks(x: np.ndarray):
            # the vols are the batch pricer's, so that the objective is the difference route's bit for bit; the sensitivity pass prices
            # the same paths with another reduction order (~1e-13 apart) and supplies only the derivatives
            s = codec.parse(x)
            res = engine.logsv_mc_chain_greeks(_params_c(s), ttms, option_chain.forwards, option_chain.discfactors,
                                               s.get_vol_backbone_etas(ttms=ttms), option_chain.strikes_ttms, option_chain.optiontypes_ttms,
                                               nb_path, nb_steps, is_spot_measure, 1, seed, flags)
            return batch_vols(x[None, :])[0], mc_ivol_rows(res)[1]
    elif calibration_engine == CalibrationEngine.MC:
        if mc_randoms != "numpy":
            raise ValueError("mc_randoms must be 'numpy' or 'philox'")
        rnd = get_randoms_for_chain_valuation(ttms=ttms, nb_path=nb_path, nb_steps_per_year=nb_steps, seed=seed, device=True)
        assert isinstance(rnd, DeviceRandoms)

        def batch_vols(points: np.ndarray) -> np.ndarray:
            rows = []
            for p in points:
                s = codec.parse(p)
                prices, _ = _fixed_randoms_chain_device(rnd, ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
                                                        option_chain.optiontypes_ttms, _params_c(s), s.get_vol_backbone_etas(ttms=ttms),
                                                        is_spot_measure, 1, True)
                rows.append(to_flat_np_array(option_chain.compute_model_ivols_from_chain_data(model_prices=prices)))
            return np.vstack(rows)

        def ivol_greeks(x: np.ndarray):
            s = codec.parse(x)
            res = logsv_mc_chain_greeks_fixed_randoms(ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
                                                      option_chain.optiontypes_ttms, rnd, v0=s.sigma0, theta=s.theta, kappa1=s.kappa1,
                                                      kappa2=s.kappa2, beta=s.beta, volvol=s.volvol,
                                                      vol_backbone_etas=s.get_vol_backbone_etas(ttms=ttms), is_spot_measure=is_spot_measure)
            return flat_ivol_rows(to_chain_ivol_sensitivities(option_chain, res), engine.LOGSV_GREEK_PARAMS)
    elif calibration_engine == CalibrationEngine.ROUGH_MC:
        # reference :528-533 + :266-289: fixed normals of get_randoms_for_rough_vol_chain_valuation; here the n + 1 finite-difference
        # parameter sets of an optimizer step share ONE upload of them (or none: mc_randoms="philox" draws in-kernel on a fixed seed)
        from .logsv_pricer import get_randoms_for_rough_vol_chain_valuation
        if mc_randoms not in ("numpy", "philox"):
            raise ValueError("mc_randoms must be 'numpy' or 'philox'")
        if params0.weights is None or params0.nodes is None:
            raise ValueError("ROUGH_MC needs params0.weights / params0.nodes (LogSvParams.approximate_kernel)")
        Z0, Z1, grids = get_randoms_for_rough_vol_chain_valuation(ttms=ttms, nb_path=nb_path, nb_steps_per_year=nb_steps, seed=seed)
        if mc_randoms == "philox":
            Z0 = Z1 = None
        nsteps = [int(g.size) - 1 for g in grids]
        hs = [float(g[1] - g[0]) for g in grids]
        flags = engine.mc_flags("fp64", "fp32")

        def batch_vols(points: np.ndarray) -> np.ndarray:
            sets = [codec.parse(p) for p in points]
            _, _, ivols, _, _ = engine.rough_logsv_mc_chain([_params_c(s) for s in sets], params0.weights, params0.nodes, ttms, option_chain.forwards,
                                                            option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms,
                                                            nb_path, nsteps, hs, Z0, Z1, 1, seed, flags, with_ivols=True)
            return ivols

        def ivol_greeks(x: np.ndarray):
            res = engine.rough_logsv_mc_chain_greeks(_params_c(codec.parse(x)), params0.weights, params0.nodes, ttms, option_chain.forwards,
                                                     option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms,
                                                     nb_path, nsteps, hs, Z0, Z1, 1, seed, flags)
            np.maximum(resets, res[7], out=resets)
            return mc_ivol_rows(res[:5])
    else:
        raise NotImplementedError(f"{calibration_engine}")

    if gradient == "difference":
        objective = BatchedObjective(batch_vols=batch_vols, market_vols=market_vols, weights=weights, bounds=bounds, eps=fd_step or SLSQP_EPS)
    elif gradient == "pathwise":
        objective = ExactGradientObjective(ivol_greeks=ivol_greeks, field_jacobian=codec.field_jacobian, market_vols=market_vols,
                                           weights=weights)
        if calibration_engine == CalibrationEngine.MC and mc_randoms == "philox":
            objective.CALLS_PER_EVALUATION = 3       # the batch pricer's vols as well (ivol_greeks above)
    x, result = run_slsqp(objective, p0, bounds, build_logsv_constraints(codec, constraints_type), disp=disp)
    fit = codec.parse(x)
    if return_info:
        info = {"fun": float(result.fun), "nit": int(result.nit), "nb_batches": objective.nb_batches, "x": x, "nan_quotes": objective.nan_quotes}
        if gradient == "pathwise" and calibration_engine == CalibrationEngine.ROUGH_MC:
            info["reset_paths"] = resets
        return fit, info
    return fit


# ---- Heston -----------------------------------------------------------------------------------------------------------------
HESTON_BOUNDS = ((0.01, 2.0), (0.01, 2.0), (0.1, 30.0), (-0.99, 0.99), (0.1, 5.0))      # heston_pricer.py:127


def heston_default_vol_scaler(v0: float, ttm0: float) -> float:
    """the transform-grid scaler the Heston chain pricers use when given none, min(0.3, sqrt(v0 T0)) with T0 the first maturity (the
    library's default, to the bit)"""
    return float(min(0.3, np.sqrt(v0 * ttm0)))


def calibrate_heston(pricer, option_chain, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, disp: bool = False,
                     return_info: bool = False, fd_step: Optional[float] = None, gradient: str = "difference",
                     price_batch: Optional[Callable] = None):
    """``price_batch``: engine.heston_price_chain_batch (None) or a callable with its arguments and return value, as for calibrate_logsv"""
    from .heston_pricer import HestonParams, _params_c
    check_gradient(gradient)
    p0 = (np.array([params0.v0, params0.theta, params0.kappa, params0.rho, params0.volvol], dtype=float) if params0 is not None
          else np.array([0.1, 0.1, 2.0, -0.2, 1.0]))
    _, market_vols_ttms = option_chain.get_chain_data_as_xy()
    market_vols = to_flat_np_array(market_vols_ttms)
    weights = calibration_weights(option_chain, market_vols, is_vega_weighted, is_unit_ttm_vega)

    if gradient == "exact":
        # the grid is pinned at the start point's default scaler; the difference route re-grids every set (the default depends on v0)
        vol_scaler = heston_default_vol_scaler(p0[0], float(option_chain.ttms[0]))

        def ivol_greeks(x: np.ndarray):
            sens = pricer.compute_chain_ivol_greeks(option_chain, HestonParams(*x), vol_scaler=vol_scaler)
            return flat_ivol_rows(sens, engine.HESTON_GREEK_PARAMS)

        objective = ExactGradientObjective(ivol_greeks=ivol_greeks, field_jacobian=lambda x: np.eye(5), market_vols=market_vols,
                                           weights=weights)

    def batch_vols(points: np.ndarray) -> np.ndarray:
        sets = [_params_c(*p) for p in points]
        _, ivols = (price_batch or engine.heston_price_chain_batch)(sets, option_chain.ttms, option_chain.forwards, option_chain.discfactors,
                                                                    option_chain.strikes_ttms, option_chain.optiontypes_ttms)
        return ivols

    def feller(pars):                     # 2 kappa theta - volvol^2 >= 0 (heston_pricer.py:152-160)
        return 2.0 * pars[2] * pars[1] - pars[4] * pars[4]

    if gradient == "difference":
        objective = BatchedObjective(batch_vols=batch_vols, market_vols=market_vols, weights=weights, bounds=HESTON_BOUNDS,
                                     eps=fd_step or SLSQP_EPS)
    x, result = run_slsqp(objective, p0, HESTON_BOUNDS, {"type": "ineq", "fun": feller}, disp=disp)
    fit = HestonParams(v0=x[0], theta=x[1], kappa=x[2], rho=x[3], volvol=x[4])
    if return_info:
        return fit, {"fun": float(result.fun), "nit": int(result.nit), "nb_batches": objective.nb_batches, "x": x}
    return fit


# ---- several chains in lock-step ------------------------------------------------------------------------------------------------
class _LockStep:
    """rendezvous of K fits run in threads and the caller's thread, which prices their points: a fit's ``post(k, request)`` blocks until
    the round it belongs to has been priced.  A round closes once every live fit has posted or left, so each round holds one request per
    live fit and the rounds of a run are max_k nb_batches_k.  Only the caller's thread waits on the condition and each fit on an event
    of its own, so a round wakes each thread once."""

    def __init__(self, n: int):
        self._cv = threading.Condition()
        self._live = n
        self._posted = {}
        self._answers = {}
        self._ready = [threading.Event() for _ in range(n)]
        self._closed: Optional[BaseException] = None

    def post(self, k: int, request):
        with self._cv:
            if self._closed is not None:
                raise self._closed
            self._posted[k] = request
            if len(self._posted) == self._live:
                self._cv.notify()
        self._ready[k].wait()
        self._ready[k].clear()
        answer = self._answers.pop(k)
        if isinstance(answer, BaseException):
            raise answer
        return answer

    def leave(self) -> None:
        with self._cv:
            self._live -= 1
            if len(self._posted) == self._live:
                self._cv.notify()

    def _answer(self, pending: dict, answers: dict) -> None:
        """hand answers[k] to every fit k of ``pending``; a fit leaves ``pending`` once woken, so after an interrupt part-way through,
        ``pending`` holds exactly the fits still waiting"""
        for k in list(pending):
            self._answers[k] = answers[k]
            self._ready[k].set()
            del pending[k]

    def serve(self, price_round: Callable[[dict], Tuple[dict, int]]) -> int:
        """price rounds until every fit has left -> the number of library calls.  ``price_round({k: request}) -> ({k: rows}, calls)``;
        an exception it raises is the answer of every fit of that round.  A BaseException that is not an Exception (KeyboardInterrupt,
        SystemExit) raised anywhere in here -- inside ``price_round`` too -- is handed to every fit still waiting, the round in flight
        included, closes the rendezvous to later posts and is re-raised, so that every fit thread ends."""
        calls = 0
        in_flight: dict = {}
        try:
            while True:
                with self._cv:
                    self._cv.wait_for(lambda: len(self._posted) == self._live)
                    if self._live == 0:
                        return calls
                    in_flight, self._posted = self._posted, {}
                try:
                    answers, n = price_round(in_flight)
                    calls += n
                except Exception as exc:              # noqa: BLE001 (handed to the fits of the round)
                    answers = {k: exc for k in in_flight}
                self._answer(in_flight, answers)
        except BaseException as exc:                  # no fit may wait for a round that never comes
            with self._cv:
                self._closed = exc
                pending = {**in_flight, **self._posted}
                self._posted = {}
            self._answer(pending, {k: exc for k in pending})
            raise


def _pack(posted: dict, max_sets_per_call: Optional[int]) -> List[List[int]]:
    """the fits of a round split into library calls of at most ``max_sets_per_call`` sets, in chain order; a fit's sets are never split (its
    rows must come from one group of one call to equal the single-chain call's)"""
    calls, sets = [], 0
    for k in sorted(posted):
        n = len(posted[k][0])
        if not calls or (max_sets_per_call is not None and sets + n > max_sets_per_call):
            calls.append([])
            sets = 0
        calls[-1].append(k)
        sets += n
    return calls


def calibrate_chains_lockstep(fit: Callable[[int, Callable], object], n: int, price_call: Callable, max_sets_per_call: Optional[int],
                              return_exceptions: bool):
    """K = n single-chain fits in lock-step.  ``fit(k, price_batch)`` runs fit k (calibrate_logsv / calibrate_heston with ``price_batch``
    injected and ``return_info=True``) and returns its (fit, info); ``price_call(requests) -> [ivols [B_i, J_i]]`` prices the requests
    (price_batch's positional arguments, keyword arguments) of several fits in one library call.  Each fit runs in a thread of its own; the caller's thread, whose
    CUDA stream the library calls keep (b200sv_set_stream is per thread), prices every round and waits for all threads before it returns.
    -> (fits, infos), ``rounds`` (library calls of the whole run) added to every info dict; a failed fit's slot holds its exception (info
    None) with ``return_exceptions``, else the lowest-index exception is raised."""
    lock = _LockStep(n)
    results = [None] * n

    def run(k: int) -> None:
        try:
            results[k] = fit(k, lambda *args, **kw: (None, lock.post(k, (args[0], args, kw))))
        except BaseException as exc:                  # noqa: BLE001 (reported per chain below)
            results[k] = exc
        finally:
            lock.leave()

    def price_round(posted: dict):
        answers = {}
        calls = _pack(posted, max_sets_per_call)
        for ks in calls:
            for k, rows in zip(ks, price_call([posted[k][1:] for k in ks])):
                answers[k] = rows
        return answers, len(calls)

    threads = [threading.Thread(target=run, args=(k,), name=f"calibrate-chain-{k}") for k in range(n)]
    for t in threads:
        t.start()
    try:
        rounds = lock.serve(price_round)
    finally:
        for t in threads:
            t.join()
    if not return_exceptions:
        for r in results:
            if isinstance(r, BaseException):
                raise r
    fits, infos = [], []
    for r in results:
        if isinstance(r, BaseException):
            fits.append(r)
            infos.append(None)
        else:
            fits.append(r[0])
            infos.append(dict(r[1], rounds=rounds))
    return fits, infos


def per_chain(value, n: int, name: str) -> list:
    """one value for every chain, or a list / tuple of exactly one per chain"""
    if isinstance(value, (list, tuple)):
        if len(value) != n:
            raise ValueError(f"{name} must be one value or one per chain ({n}), not {len(value)}")
        return list(value)
    return [value] * n


def check_lockstep_args(option_chains, max_sets_per_call, gradient: str) -> int:
    """the checks every lock-step driver makes before any library call -> the number of chains"""
    if gradient != "difference":
        if gradient in GRADIENTS:
            raise NotImplementedError(f"calibrate_model_params_to_chains has gradient='difference' only, not {gradient!r}")
        check_gradient(gradient)
    n = len(option_chains)
    if n == 0:
        raise ValueError("option_chains is empty")
    if max_sets_per_call is not None and int(max_sets_per_call) < 1:
        raise ValueError("max_sets_per_call must be at least 1")
    return n


def calibrate_logsv_chains(pricer, option_chains, params0, params_min, params_max, is_vega_weighted: bool, is_unit_ttm_vega: bool,
                           model_calibration_type: LogsvModelCalibrationType, constraints_type: ConstraintsType,
                           calibration_engine: CalibrationEngine, is_spot_measure: bool = True, disp: bool = False, return_info: bool = False,
                           fd_step: Optional[float] = None, gradient: str = "difference", return_exceptions: bool = False,
                           max_sets_per_call: Optional[int] = None):
    """calibrate_logsv on every chain, ANALYTIC engine, in lock-step: one engine.logsv_price_chains_batch call per optimizer round"""
    n = check_lockstep_args(option_chains, max_sets_per_call, gradient)
    if calibration_engine != CalibrationEngine.ANALYTIC:
        raise NotImplementedError(f"calibrate_model_params_to_chains covers CalibrationEngine.ANALYTIC only, not {calibration_engine}")
    if model_calibration_type not in (LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5,
                                      LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT):
        raise NotImplementedError(f"{model_calibration_type}")
    p0s, los, his = (per_chain(v, n, name) for v, name in ((params0, "params0"), (params_min, "params_min"), (params_max, "params_max")))

    def fit(k: int, price_batch):
        return calibrate_logsv(pricer, option_chains[k], p0s[k], los[k], his[k], is_vega_weighted, is_unit_ttm_vega, model_calibration_type,
                               constraints_type, calibration_engine, 0, 0, 0,          # nb_path, nb_steps, seed: Monte Carlo engines only
                               is_spot_measure=is_spot_measure, disp=disp, return_info=True,
                               fd_step=fd_step, price_batch=price_batch)

    def price_call(requests):
        # request = (args, kwargs) of engine.logsv_price_chain_batch(params_list, ttms, forwards, discfactors, etas, strikes, types, ...)
        params, chain_of_set, chains, etas, scalers = [], [], [], [], []
        for i, (args, kw) in enumerate(requests):
            sets, ttms, forwards, discfactors, e, strikes_ttms, optiontypes_ttms = args
            params += list(sets)
            chain_of_set += [i] * len(sets)
            chains.append((ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms))
            etas += list(e)
            scalers.append(kw["vol_scaler"])
        _, ivols = engine.logsv_price_chains_batch(params, chain_of_set, chains, etas, scalers, is_spot_measure=is_spot_measure)
        return _rows_by_request(ivols, chain_of_set, len(requests))

    out = calibrate_chains_lockstep(fit, n, price_call, max_sets_per_call, return_exceptions)
    return out if return_info else out[0]


def calibrate_heston_chains(pricer, option_chains, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, disp: bool = False,
                            return_info: bool = False, fd_step: Optional[float] = None, gradient: str = "difference",
                            return_exceptions: bool = False, max_sets_per_call: Optional[int] = None):
    """calibrate_heston on every chain in lock-step: one engine.heston_price_chains_batch call per optimizer round"""
    n = check_lockstep_args(option_chains, max_sets_per_call, gradient)
    p0s = per_chain(params0, n, "params0")

    def fit(k: int, price_batch):
        return calibrate_heston(pricer, option_chains[k], p0s[k], is_vega_weighted, is_unit_ttm_vega, disp=disp, return_info=True,
                                fd_step=fd_step, price_batch=price_batch)

    def price_call(requests):
        # request = (args, kwargs) of engine.heston_price_chain_batch(params_list, ttms, forwards, discfactors, strikes, types)
        params, chain_of_set, chains = [], [], []
        for i, (args, _) in enumerate(requests):
            params += list(args[0])
            chain_of_set += [i] * len(args[0])
            chains.append(tuple(args[1:6]))
        _, ivols = engine.heston_price_chains_batch(params, chain_of_set, chains)
        return _rows_by_request(ivols, chain_of_set, len(requests))

    out = calibrate_chains_lockstep(fit, n, price_call, max_sets_per_call, return_exceptions)
    return out if return_info else out[0]


def _rows_by_request(ivols, chain_of_set, n: int) -> List[np.ndarray]:
    """the B rows of a multi-chain call -> one [B_i, J_i] array per request (request i's sets are the i-th run of chain_of_set)"""
    ends = np.cumsum(np.bincount(chain_of_set, minlength=n)).tolist()
    return [np.vstack(ivols[a:b]) for a, b in zip([0] + ends[:-1], ends)]
