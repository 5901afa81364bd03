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


def calibration_weights(option_chain, market_vols: np.ndarray, is_vega_weighted: bool, is_unit_ttm_vega: bool,
                        slice_sum: Callable = sum) -> np.ndarray:
    """flattened objective weights: the Black vegas of each slice divided by their ``slice_sum``, or ones (reference
    logsv_pricer.py:196-207).  The LogSV and Heston drivers normalise with the builtin ``sum`` (left to right), the Hawkes drivers with
    ``np.sum`` (pairwise from 8 quotes a slice) -- the two differ in the last bit, so each driver names its own."""
    if not is_vega_weighted:
        return np.ones_like(market_vols)
    vegas_ttms = option_chain.get_chain_vegas(is_unit_ttm_vega=is_unit_ttm_vega)
    return to_flat_np_array([v / slice_sum(v) for v in vegas_ttms])


def market_and_weights(option_chain, is_vega_weighted: bool, is_unit_ttm_vega: bool, slice_sum: Callable = sum
                       ) -> Tuple[np.ndarray, np.ndarray]:
    """(mid vols, calibration_weights) flat in chain order: what every driver's objective compares the model vols with"""
    _, mid_vols = option_chain.get_chain_data_as_xy()
    market = to_flat_np_array(mid_vols)
    return market, calibration_weights(option_chain, market, is_vega_weighted, is_unit_ttm_vega, slice_sum)


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


def run_slsqp(objective, p0: np.ndarray, bounds, constraints=None, disp: bool = False, tol: Optional[float] = None, validate: bool = True,
              **options):
    """``scipy.optimize.minimize(method='SLSQP', options={'ftol': 1e-8})`` as in the reference (:543-555), with the objective's own
    gradient -> (x, result).  ``options`` (``maxiter``, ``eps``, another ``ftol``) and ``tol`` go to SLSQP as given.  ``validate``: x is
    the vector validate_optimization_result accepts (the LogSV and Heston drivers, as the reference's), else ``result.x`` unchecked (the
    Hawkes drivers, as the reference's hawkes_jd_pricer.py:296-298)."""
    from scipy.optimize import minimize      # host-side optimizer; scipy is already a dependency of the reference
    result = minimize(objective.fun, np.asarray(p0, dtype=float), method="SLSQP", jac=objective.jac, bounds=bounds,
                      constraints=() if constraints is None else constraints, tol=tol, options={"disp": disp, "ftol": 1e-8, **options})
    return (validate_optimization_result(result, bounds) if validate else result.x), result


def fit_info(result, x: np.ndarray, objective, **extra) -> dict:
    """the ``return_info`` dict of a fit: SLSQP's last value and iterations, the library calls of the objective, the fitted vector"""
    return {"fun": float(result.fun), "nit": int(result.nit), "nb_batches": objective.nb_batches, "x": x, **extra}


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
    """``params_min`` / ``params_max``: None for the default bounds.  ``price_batch``: what the ANALYTIC difference objective prices its
    points with, engine.logsv_price_chain_batch (None) or a callable with its arguments and return value (calibrate_chains_lockstep)"""
    routes = {"exact": ((CalibrationEngine.ANALYTIC,), "CalibrationEngine.ANALYTIC only", "the Monte Carlo engines have gradient='pathwise'"),
              "pathwise": ((CalibrationEngine.MC, CalibrationEngine.ROUGH_MC), "CalibrationEngine.MC and ROUGH_MC only",
                           "the ANALYTIC engine has gradient='exact'")}
    if check_gradient(gradient, pathwise=True) in routes:
        engines, covered, other = routes[gradient]
        if calibration_engine not in engines:
            raise NotImplementedError(f"gradient={gradient!r} covers {covered}, not {calibration_engine} ({other})")
        if model_calibration_type not in (LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5):
            raise NotImplementedError(f"gradient={gradient!r} covers PARAMS4 and PARAMS5 only, not {model_calibration_type} (the eta "
                                      "backbone of PARAMS_WITH_VARSWAP_FIT is refitted at every point and is not differentiated)")
    from ..multi_gpu import _fixed_randoms_chain_device
    from .fourier_greeks import to_chain_ivol_sensitivities
    from .logsv_pricer import (DeviceRandoms, LogSvParams, _params_c, get_randoms_for_chain_valuation,
                               logsv_mc_chain_greeks_fixed_randoms)
    from .mc_greeks import to_mc_chain_greeks
    params_min = params_min or LogSvParams(sigma0=0.1, theta=0.1, kappa1=0.25, kappa2=0.25, beta=-3.0, volvol=0.2)
    params_max = params_max or LogSvParams(sigma0=1.5, theta=1.5, kappa1=10.0, kappa2=10.0, beta=3.0, volvol=3.0)
    vol_scaler = pricer.set_vol_scaler(option_chain=option_chain)
    market_vols, weights = market_and_weights(option_chain, is_vega_weighted, is_unit_ttm_vega)
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
        info = fit_info(result, x, objective, nan_quotes=objective.nan_quotes)
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
    market_vols, weights = market_and_weights(option_chain, is_vega_weighted, is_unit_ttm_vega)

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
    return (fit, fit_info(result, x, objective)) if return_info else fit


# ---- Hawkes jump-diffusion --------------------------------------------------------------------------------------------------
def calibrate_hawkes(pricer, option_chain, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, return_info: bool = False,
                     price_batch: Optional[Callable] = None, **kwargs):
    """HawkesJDPricer.calibrate_model_params_to_chain (reference hawkes_jd_pricer.py:230-300).  ``price_batch``: what the difference
    objective prices its points with, engine.hawkesjd_price_chain_batch (None) or a callable with its arguments and return value, as for
    calibrate_logsv"""
    from .hawkes_jd_pricer import HawkesJDParams, set_vol_scaler
    gradient = check_gradient(kwargs.get("gradient", "difference"))
    p0 = np.array([params0.sigma, params0.mean_p, params0.mean_m, params0.theta_p, params0.theta_m, 0.5 * (params0.kappa_p + params0.kappa_m),
                   0.5 * (params0.beta1_p - params0.beta2_p), 0.5 * (params0.beta2_p - params0.beta2_m)])
    bounds = ((0.10, 2.0), (0.01, 0.99), (-0.99, -0.01), (0.01, 100.0), (0.01, 100.0), (1.0, 100.0), (1.0, 100.0), (1.0, 100.0))

    def unpack(x: np.ndarray):
        return HawkesJDParams(mu=0.0, sigma=x[0], shift_p=params0.shift_p, mean_p=x[1], shift_m=params0.shift_m, mean_m=x[2],
                              lambda_p=params0.lambda_p, theta_p=x[3], kappa_p=x[5], beta1_p=x[6], beta2_p=-x[6], lambda_m=params0.lambda_m,
                              theta_m=x[4], kappa_m=x[5], beta1_m=x[7], beta2_m=-x[7])

    stationary = {"type": "ineq", "fun": lambda x: unpack(x).jump1_cond + unpack(x).jump2_cond}
    if gradient == "exact":
        objective = _exact_vol_objective(pricer, option_chain, unpack, is_vega_weighted, is_unit_ttm_vega,
                                         set_vol_scaler(params0.sigma, float(option_chain.ttms[0])))
    else:
        objective = _batched_vol_objective(option_chain, unpack, is_vega_weighted, is_unit_ttm_vega, bounds, SLSQP_EPS,
                                           price_batch=price_batch)
    x, result = run_slsqp(objective, p0, bounds, stationary, disp=bool(kwargs.get("disp", False)), validate=False,
                          **({"maxiter": int(kwargs["maxiter"])} if "maxiter" in kwargs else {}))
    fit = unpack(x)
    return (fit, fit_info(result, x, objective, nan_quotes=objective.nan_quotes)) if return_info else fit


def calibrate_hawkes_risk_premia(option_chain, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, maxiter: int = 100,
                                 print_iter: bool = True, return_info: bool = False, price_batch: Optional[Callable] = None,
                                 line_sink: Callable[[str], None] = print, **kwargs):
    """HawkesJDPricer.calibrate_risk_premia_gamma_to_chain (reference hawkes_jd_pricer.py:303-357): (sigma, gamma / 8) with the rest of
    ``params0`` fixed, weights x 1e4, SLSQP with difference step 0.025 and ftol = tol = 1e-16.  ``price_batch`` as for calibrate_hawkes;
    ``line_sink`` receives the ``print_iter`` lines (the lock-step driver collects each chain's)"""
    from .hawkes_jd_pricer import _KEYS, HawkesJDParams
    if check_gradient(kwargs.get("gradient", "difference")) == "exact":
        raise NotImplementedError("gradient='exact' does not cover calibrate_risk_premia_gamma_to_chain: the risk-kernel pricer has no "
                                  "sensitivities")
    gamma_scaler = 8.0
    fixed = {k: v for k, v in params0.to_dict().items() if k in _KEYS}
    bounds = ((0.01, 1.5), (-1.0, 1.0))

    def announce(x: np.ndarray) -> None:
        line_sink(f"unpack_pars: sigma={x[0]}, gamma={gamma_scaler * x[1]}")

    def to_params(x: np.ndarray):
        return HawkesJDParams(**{**fixed, "sigma": float(x[0])}, risk_premia_gamma=float(gamma_scaler * x[1]))

    p0 = np.array([params0.sigma, (params0.risk_premia_gamma or 0.0) / gamma_scaler])
    objective = _batched_vol_objective(option_chain, to_params, is_vega_weighted, is_unit_ttm_vega, bounds, 0.025, scale=10000.0,
                                       on_point=announce if print_iter else None, price_batch=price_batch)
    x, result = run_slsqp(objective, p0, bounds, disp=bool(kwargs.get("disp", False)), tol=1e-16, validate=False, ftol=1e-16,
                          maxiter=maxiter, eps=0.025)
    if print_iter:
        announce(x)
    fit = to_params(x)
    return (fit, fit_info(result, x, objective, nan_quotes=objective.nan_quotes)) if return_info else fit


# d HAWKES_GREEK_PARAMS / d x of calibrate_hawkes's x = (sigma, mean_p, mean_m, theta_p, theta_m, kappa, beta_p, beta_m): kappa feeds
# kappa_p and kappa_m, beta_p feeds beta1_p = +x and beta2_p = -x, beta_m feeds beta1_m = +x and beta2_m = -x
_HAWKES_FIT_FIELDS = ((("sigma", 1.0),), (("mean_p", 1.0),), (("mean_m", 1.0),), (("theta_p", 1.0),), (("theta_m", 1.0),),
                      (("kappa_p", 1.0), ("kappa_m", 1.0)), (("beta1_p", 1.0), ("beta2_p", -1.0)), (("beta1_m", 1.0), ("beta2_m", -1.0)))


def hawkes_fit_jacobian() -> np.ndarray:
    D = np.zeros((len(engine.HAWKES_GREEK_PARAMS), len(_HAWKES_FIT_FIELDS)))
    for col, fields in enumerate(_HAWKES_FIT_FIELDS):
        for name, sign in fields:
            D[engine.HAWKES_GREEK_PARAMS.index(name), col] = sign
    return D


def _exact_vol_objective(pricer, option_chain, to_params, is_vega_weighted: bool, is_unit_ttm_vega: bool,
                         vol_scaler: float) -> ExactGradientObjective:
    """the Hawkes objective with its exact gradient: one compute_chain_ivol_greeks call per point on the grid of ``vol_scaler``"""
    market, weights = market_and_weights(option_chain, is_vega_weighted, is_unit_ttm_vega, slice_sum=np.sum)
    D = hawkes_fit_jacobian()

    def ivol_greeks(x: np.ndarray):
        sens = pricer.compute_chain_ivol_greeks(option_chain, to_params(x), vol_scaler=vol_scaler)
        return flat_ivol_rows(sens, engine.HAWKES_GREEK_PARAMS)
    return ExactGradientObjective(ivol_greeks=ivol_greeks, field_jacobian=lambda x: D, market_vols=market, weights=weights)


def _batched_vol_objective(option_chain, to_params, is_vega_weighted: bool, is_unit_ttm_vega: bool, bounds, eps: float,
                           scale: float = 1.0, on_point=None, price_batch=None) -> ScipyDifferenceObjective:
    """the Hawkes drivers' objective: weighted squared difference of model and mid implied vols, nansum over the chain (quotes whose model
    price leaves the no-arbitrage bounds drop out), with the weights of the reference (per-slice normalised vegas, times ``scale``).  The
    model vols of a point, and of its difference neighbours together, come from hawkesjd_price_chain_batch, on the risk-kernel route when
    the parameter sets carry a risk_premia_gamma -- the same prices and vols as compute_model_ivols_for_chain per set.  ``price_batch``: a
    callable with hawkesjd_price_chain_batch's arguments and return value in its place (the lock-step driver)."""
    from .hawkes_jd_pricer import MAX_PHI, _params_c
    market, weights = market_and_weights(option_chain, is_vega_weighted, is_unit_ttm_vega, slice_sum=np.sum)

    def batch_vols(points: np.ndarray) -> np.ndarray:
        sets = [to_params(p) for p in points]
        gammas = None if sets[0].risk_premia_gamma is None else [s.risk_premia_gamma for s in sets]
        _, ivols = (price_batch or engine.hawkesjd_price_chain_batch)([_params_c(**s.to_dict()) for s in sets], option_chain.ttms,
                                                                      option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
                                                                      option_chain.optiontypes_ttms, max_phi=MAX_PHI, gammas=gammas)
        return ivols
    return ScipyDifferenceObjective(batch_vols=batch_vols, market_vols=market, weights=scale * weights, bounds=bounds, eps=eps,
                                    on_point=on_point)


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


def calibrate_chains_lockstep(fit: Callable, option_chains, price_chains: Callable, gradient: str, max_sets_per_call: Optional[int],
                              return_exceptions: bool, return_info: bool, extras: Optional[Callable] = None,
                              method: str = "calibrate_model_params_to_chains", **per_chain_args):
    """one single-chain fit per chain of ``option_chains``, in lock-step.  Before any library call: ``gradient`` ('difference' only),
    ``option_chains`` (not empty), ``max_sets_per_call`` (None or at least 1), then per_chain on each of ``per_chain_args`` in turn.
    ``fit(option_chain, price_batch, **args)`` runs the fit of one chain on its values of ``per_chain_args`` (calibrate_logsv /
    calibrate_heston / calibrate_hawkes with ``price_batch`` injected and ``return_info=True``) and returns its (fit, info).  The requests
    of the fits priced together -- price_batch's (positional arguments, keyword arguments) -- go to ``price_chains(params, chain_of_set,
    chains, *args, **kwargs)``, the model's engine.*_price_chains_batch, with each fit's sets, its chain's arrays and ``(args, kwargs) =
    extras(requests)``, the model's other arguments (none without ``extras``).  Each fit runs in a thread of its own; the caller's thread,
    whose CUDA stream the library calls keep (b200sv_set_stream is per thread), prices every round and waits for all threads before it
    returns.  -> the fits, with ``return_info`` (fits, infos) whose info dicts add ``rounds`` (library calls of the whole run); a failed
    fit's slot holds its exception (info None) with ``return_exceptions``, else the lowest-index exception is raised.  ``method`` names the
    caller in the ``gradient`` rejection."""
    if gradient != "difference":
        if gradient in GRADIENTS:
            raise NotImplementedError(f"{method} has gradient='difference' only, not {gradient!r}")
        check_gradient(gradient)
    n = len(option_chains)
    if n == 0:
        raise ValueError("option_chains is empty")
    if max_sets_per_call is not None and int(max_sets_per_call) < 1:
        raise ValueError("max_sets_per_call must be at least 1")
    columns = {name: per_chain(value, n, name) for name, value in per_chain_args.items()}
    lock = _LockStep(n)
    results = [None] * n

    def run(k: int) -> None:
        try:
            results[k] = fit(option_chains[k], lambda *args, **kw: (None, lock.post(k, (args[0], args, kw))),
                             **{name: values[k] for name, values in columns.items()})
        except BaseException as exc:                  # noqa: BLE001 (reported per chain below)
            results[k] = exc
        finally:
            lock.leave()

    def price_round(posted: dict):
        answers, calls = {}, _pack(posted, max_sets_per_call)
        for ks in calls:
            params, chain_of_set, chains = [], [], []
            for i, k in enumerate(ks):
                c = option_chains[k]                  # the arrays fit k hands price_batch
                params += list(posted[k][0])
                chain_of_set += [i] * len(posted[k][0])
                chains.append((c.ttms, c.forwards, c.discfactors, c.strikes_ttms, c.optiontypes_ttms))
            args, kw = extras([posted[k][1:] for k in ks]) if extras is not None else ((), {})
            _, ivols = price_chains(params, chain_of_set, chains, *args, **kw)
            answers.update(zip(ks, _rows_by_request(ivols, chain_of_set, len(ks))))
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
    fits = [r if isinstance(r, BaseException) else r[0] for r in results]
    if not return_info:
        return fits
    return fits, [None if isinstance(r, BaseException) else dict(r[1], rounds=rounds) for r in results]


def per_chain(value, n: int, name: str) -> list:
    """one value for every chain, or a list / tuple of exactly one per chain"""
    if isinstance(value, (list, tuple)):
        if len(value) != n:
            raise ValueError(f"{name} must be one value or one per chain ({n}), not {len(value)}")
        return list(value)
    return [value] * n


def calibrate_logsv_chains(pricer, option_chains, params0, params_min, params_max, is_vega_weighted: bool, is_unit_ttm_vega: bool,
                           model_calibration_type: LogsvModelCalibrationType, constraints_type: ConstraintsType,
                           calibration_engine: CalibrationEngine, is_spot_measure: bool = True, disp: bool = False, return_info: bool = False,
                           fd_step: Optional[float] = None, gradient: str = "difference", return_exceptions: bool = False,
                           max_sets_per_call: Optional[int] = None):
    """calibrate_logsv on every chain, ANALYTIC engine, in lock-step: one engine.logsv_price_chains_batch call per optimizer round"""
    if calibration_engine != CalibrationEngine.ANALYTIC:
        raise NotImplementedError(f"calibrate_model_params_to_chains covers CalibrationEngine.ANALYTIC only, not {calibration_engine}")
    if model_calibration_type not in (LogsvModelCalibrationType.PARAMS4, LogsvModelCalibrationType.PARAMS5,
                                      LogsvModelCalibrationType.PARAMS_WITH_VARSWAP_FIT):
        raise NotImplementedError(f"{model_calibration_type}")

    def fit(option_chain, price_batch, params0, params_min, params_max):
        return calibrate_logsv(pricer, option_chain, params0, params_min, params_max, is_vega_weighted, is_unit_ttm_vega, model_calibration_type,
                               constraints_type, calibration_engine, 0, 0, 0,          # nb_path, nb_steps, seed: Monte Carlo engines only
                               is_spot_measure=is_spot_measure, disp=disp, return_info=True, fd_step=fd_step, price_batch=price_batch)

    def extras(requests):
        # request = (args, kwargs) of engine.logsv_price_chain_batch(params_list, ttms, forwards, discfactors, etas, strikes, types, ...,
        # vol_scaler=): the eta row of every set, the grid scaler of every chain
        return ([row for args, _ in requests for row in args[4]], [kw["vol_scaler"] for _, kw in requests]), {"is_spot_measure": is_spot_measure}

    return calibrate_chains_lockstep(fit, option_chains, engine.logsv_price_chains_batch, gradient, max_sets_per_call, return_exceptions,
                                     return_info, extras, params0=params0, params_min=params_min, params_max=params_max)


def calibrate_heston_chains(pricer, option_chains, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, disp: bool = False,
                            return_info: bool = False, fd_step: Optional[float] = None, gradient: str = "difference",
                            return_exceptions: bool = False, max_sets_per_call: Optional[int] = None):
    """calibrate_heston on every chain in lock-step: one engine.heston_price_chains_batch call per optimizer round"""
    def fit(option_chain, price_batch, params0):
        return calibrate_heston(pricer, option_chain, params0, is_vega_weighted, is_unit_ttm_vega, disp=disp, return_info=True,
                                fd_step=fd_step, price_batch=price_batch)

    return calibrate_chains_lockstep(fit, option_chains, engine.heston_price_chains_batch, gradient, max_sets_per_call, return_exceptions,
                                     return_info, params0=params0)


def calibrate_hawkes_chains(pricer, option_chains, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, return_info: bool = False,
                            gradient: str = "difference", return_exceptions: bool = False, max_sets_per_call: Optional[int] = None, **kwargs):
    """calibrate_hawkes on every chain in lock-step: one engine.hawkesjd_price_chains_batch call per optimizer round"""
    from .hawkes_jd_pricer import MAX_PHI

    def fit(option_chain, price_batch, params0):
        return calibrate_hawkes(pricer, option_chain, params0, is_vega_weighted, is_unit_ttm_vega, return_info=True, price_batch=price_batch,
                                **kwargs)

    return calibrate_chains_lockstep(fit, option_chains, engine.hawkesjd_price_chains_batch, gradient, max_sets_per_call, return_exceptions,
                                     return_info, lambda requests: ((), {"max_phi": MAX_PHI}), params0=params0)


def calibrate_hawkes_risk_premia_chains(option_chains, params0, is_vega_weighted: bool, is_unit_ttm_vega: bool, maxiter: int = 100,
                                        print_iter: bool = False, return_info: bool = False, gradient: str = "difference",
                                        return_exceptions: bool = False, max_sets_per_call: Optional[int] = None, **kwargs):
    """calibrate_hawkes_risk_premia on every chain in lock-step: one risk-kernel engine.hawkesjd_price_chains_batch call per optimizer
    round.  ``print_iter``: each chain's lines are collected and printed as one block per chain, in chain order, once every fit has ended"""
    from .hawkes_jd_pricer import MAX_PHI
    lines: List[List[str]] = [[] for _ in option_chains]

    def fit(option_chain, price_batch, params0, line_sink):
        return calibrate_hawkes_risk_premia(option_chain, params0, is_vega_weighted, is_unit_ttm_vega, maxiter=maxiter, print_iter=print_iter,
                                            return_info=True, price_batch=price_batch, line_sink=line_sink, **kwargs)

    def extras(requests):
        # request = (args, kwargs) of engine.hawkesjd_price_chain_batch(params_list, ..., max_phi=, gammas=): every set's gamma, in call order
        return (), {"max_phi": MAX_PHI, "gammas": [g for _, kw in requests for g in kw["gammas"]]}

    try:
        return calibrate_chains_lockstep(fit, option_chains, engine.hawkesjd_price_chains_batch, gradient, max_sets_per_call, return_exceptions,
                                         return_info, extras, method="calibrate_risk_premia_gamma_to_chains", params0=params0,
                                         line_sink=[chain_lines.append for chain_lines in lines])
    finally:
        for chain_lines in lines:
            for line in chain_lines:
                print(line)


def _rows_by_request(ivols, chain_of_set, n: int) -> List[np.ndarray]:
    """the B rows of a multi-chain call -> one [B_i, J_i] array per request (request i's sets are the i-th run of chain_of_set)"""
    ends = np.cumsum(np.bincount(chain_of_set, minlength=n)).tolist()
    return [np.vstack(ivols[a:b]) for a, b in zip([0] + ends[:-1], ends)]
