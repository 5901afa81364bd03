"""HawkesJDPricer on H100: the reference's ``pricers/hawkes_jd_pricer.py`` (SURVEY.md §8f #4), Monte Carlo and Fourier routes.

* ``HawkesJDParams``                          (hawkes_jd_pricer.py:41-119)
* ``HawkesJDPricer.model_mc_price_chain``     (:156-171) -> ``hawkesjd_mc_chain_pricer`` (:644-715); ``model_mc_chain_greeks`` adds Monte Carlo
  sensitivities (DESIGN.md §3.11); ``scheme="exact"`` opts into the exact event-driven route (DESIGN.md §3.13, not in the reference)
* ``HawkesJDPricer.simulate_terminal_values`` (:193-224) -> ``simulate_hawkesjd_terminal`` (:718-779)
* ``HawkesJDPricer.price_chain``              (:125-155) -> ``hawkesjd_chain_pricer`` (:365-417) / ``hawkesjd_chain_pricer_with_risk_premia`` (:420-484),
  ``hawkesjd_forwards_under_risk_kernel`` (:487-515), ``compute_hawkes_a_mgf_grid`` / ``solve_a_ode_grid`` (:518-579)
* ``HawkesJDPricer.calibrate_model_params_to_chain`` (:230-300), ``calibrate_risk_premia_gamma_to_chain`` (:303-357): host SLSQP loops around the
  batched GPU chain pricer (``b200sv_hawkesjd_price_chain_batch``), fits bit-identical to SLSQP differencing the one-set objective (pricers/calibration.py);
  their ``*_to_chains`` twins fit a series of chains in lock-step on ``b200sv_hawkesjd_price_chains_batch{,_gamma}``

Monte Carlo: the reference draws every random input from numpy's process-global generator; here they are drawn in-kernel from the Philox
stream keyed by an explicit ``seed`` (default: the ``set_seed`` stream or OS entropy).  ``simulate_hawkesjd_terminal`` additionally accepts the five
input blocks (``W0, U_P, U_M, J_P, J_M`` in the reference's own form) and then reproduces the reference arithmetic operation by operation.
Fourier: the 3-equation Riccati system per transform point goes through the same SciPy-RK45 clone as the LogSV coefficient ODEs
(csrc/mgf_kernels.cu, ``hawkes_mgf_kernel``); its stiff (BDF) variant is not built and raises.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from .. import _capi as C
from .. import engine
from ..data.option_chain import OptionChain
from ..multi_gpu import _shared_seed, _use_distributed, mc_chain_distributed
from ..utils.config import VariableType
from ..utils.funcs import set_time_grid, timer
from .calibration import calibrate_hawkes, calibrate_hawkes_chains, calibrate_hawkes_risk_premia, calibrate_hawkes_risk_premia_chains
from .calibration import _batched_vol_objective, hawkes_fit_jacobian  # noqa: F401  (imported from this module by callers)
from .model_pricer import ModelParams, ModelPricer

_KEYS = tuple(k for k, _ in C.HawkesParamsC._fields_)
STEPS_PER_YEAR = 5 * 360          # hawkes_jd_pricer.py:752 "need small dt step for large intensities"


@dataclass
class HawkesJDParams(ModelParams):
    """parameters of the 2-factor Hawkes jump-diffusion, annualised (reference :41-65, same defaults)"""
    mu: float = 0.0
    sigma: float = 0.45
    shift_p: float = 0.06
    mean_p: float = 0.03
    shift_m: float = -0.06
    mean_m: float = -0.03
    lambda_p: float = 6.55
    theta_p: float = 6.55
    kappa_p: float = 22.29
    beta1_p: float = 76.0
    beta2_p: float = -67.58
    lambda_m: float = 8.50
    theta_m: float = 8.50
    kappa_m: float = 29.0
    beta1_m: float = 104.55
    beta2_m: float = -109.6
    risk_premia_gamma: Optional[float] = None

    def __post_init__(self):
        self.compensator_p = np.exp(self.shift_p) / (1.0 - self.mean_p) - 1.0
        self.compensator_m = np.exp(self.shift_m) / (1.0 - self.mean_m) - 1.0

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    @property
    def exp_jump_p(self) -> float:
        return self.shift_p + self.mean_p

    @property
    def exp_jump_m(self) -> float:
        return self.shift_m + self.mean_m

    @property
    def jump1_cond(self) -> float:
        """stationarity margin of the positive-jump intensity (:87-96)"""
        return self.kappa_p - self.beta1_p * self.exp_jump_p - self.beta2_p * self.exp_jump_m

    @property
    def jump2_cond(self) -> float:
        return self.kappa_m - self.beta2_m * self.exp_jump_m - self.beta1_m * self.exp_jump_p


def _params_c(**kw) -> C.HawkesParamsC:
    return C.HawkesParamsC(*[float(kw[k]) for k in _KEYS])


SCHEMES = ("euler", "exact")
# the exact route refuses a parameter set whose bound on the expected events per path over the simulated horizon exceeds this
HAWKES_EXACT_MAX_EXPECTED_EVENTS = 5000.0


def _is_exact(scheme) -> bool:
    """'euler' (default: the reference's 1800-steps-per-year scheme, the numbers the goldens pin) | 'exact' (opt-in event-driven simulation
    of the continuous-time model without a grid, DESIGN.md §3.13; not in the reference)"""
    if scheme not in SCHEMES:
        raise ValueError("scheme must be 'euler' or 'exact'")
    return scheme == "exact"


def hawkes_expected_events_bound(horizon: float, lambda_p: float, lambda_m: float, shift_p: float, mean_p: float, shift_m: float, mean_m: float,
                                 theta_p: float, kappa_p: float, beta1_p: float, beta2_p: float, theta_m: float, kappa_m: float, beta1_m: float,
                                 beta2_m: float, **_) -> float:
    """an upper bound on the expected number of events per path over [0, horizon], for any sign of the parameters: the integral of
    m_p + m_m from the comparison system d m / dt = |K theta| - K m + B m, m(0) = |lambda(0)|, B_ij = |beta_ij| (|shift_j| + |mean_j|).
    Between events d|lambda|/dt <= |kappa theta| - kappa |lambda|, a jump adds at most |beta| |J| at the rate max(lambda_j, 0) <= |lambda_j|,
    and the system is cooperative, so m >= E|lambda| >= E[max(lambda, 0)], the firing rate (DESIGN.md §3.13).  inf where the bound does not
    exist in floating point."""
    from scipy.linalg import expm
    ej_p, ej_m = abs(shift_p) + abs(mean_p), abs(shift_m) + abs(mean_m)
    a = np.zeros((4, 4))
    a[0, :2] = (abs(beta1_p) * ej_p - kappa_p, abs(beta2_p) * ej_m)
    a[1, :2] = (abs(beta1_m) * ej_p, abs(beta2_m) * ej_m - kappa_m)
    a[:2, 2] = (abs(kappa_p * theta_p), abs(kappa_m * theta_m))
    a[3, :2] = 1.0
    with np.errstate(all="ignore"):
        y = expm(a * float(horizon)) @ np.array([abs(lambda_p), abs(lambda_m), 1.0, 0.0])
    return float(y[3]) if np.isfinite(y[3]) else float("inf")


def _check_exact_events(horizon: float, kw) -> None:
    """refuse, before any GPU work, a parameter set the exact route would spend a runaway number of events on"""
    bound = hawkes_expected_events_bound(horizon, **kw)
    if not bound <= HAWKES_EXACT_MAX_EXPECTED_EVENTS:
        raise ValueError(f"scheme='exact': up to {bound:.4g} expected events per path over {horizon} years exceeds the limit "
                         f"{HAWKES_EXACT_MAX_EXPECTED_EVENTS:g} (HAWKES_EXACT_MAX_EXPECTED_EVENTS)")


def _check_risk_premia_greeks(option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool, kwargs, method: str) -> float:
    """what the risk-kernel sensitivities reject, before any library call; returns gamma"""
    from .fourier_greeks import _check_fourier_kwargs
    gamma = params.risk_premia_gamma
    if gamma is None:
        raise ValueError(f"{method} needs params.risk_premia_gamma; price_chain_greeks covers the pricer without a risk kernel")
    if not np.isfinite(gamma):
        raise ValueError(f"{method}: risk_premia_gamma must be finite, got {gamma}")
    if kwargs.get("with_theta"):
        raise NotImplementedError(f"{method} does not cover theta (with_theta) under the risk kernel")
    _check_fourier_kwargs(kwargs, method)
    if not is_spot_measure or any(str(t) not in ("C", "P") for types in option_chain.optiontypes_ttms for t in types):
        raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318, as price_chain
    return float(gamma)


class HawkesJDPricer(ModelPricer):
    """ModelPricer for the Hawkes jump-diffusion model: Fourier and Monte Carlo routes on the GPU."""

    def price_chain(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True, **kwargs) -> List[np.ndarray]:
        """Fourier prices of the chain (reference :125-155): the risk-kernel pricer when ``params.risk_premia_gamma`` is set, else the plain one"""
        pricer = hawkesjd_chain_pricer if params.risk_premia_gamma is None else hawkesjd_chain_pricer_with_risk_premia
        return pricer(model_params=params, ttms=option_chain.ttms, forwards=option_chain.forwards, discfactors=option_chain.discfactors,
                      strikes_ttms=option_chain.strikes_ttms, optiontypes_ttms=option_chain.optiontypes_ttms, is_spot_measure=is_spot_measure, **kwargs)

    def price_chain_greeks(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True, with_theta: bool = False,
                           **kwargs):
        """Fourier prices (bit-identical to ``price_chain`` with the same arguments) plus forward-mode sensitivities in one call ->
        ``FourierChainGreeks``: delta and gamma in the slice forward and d price / d HAWKES_GREEK_PARAMS (every field but ``mu``, which the
        Fourier route does not read, and ``risk_premia_gamma``).  The compensators are differentiated through ``shift`` and ``mean``.  Takes
        ``vol_scaler`` like ``price_chain``; the transform grid is held fixed, so the dependence of the default ``vol_scaler`` on ``sigma``
        (through clip(sigma, 0.2, 0.5)) is not differentiated, nor are the discount factors.  A risk kernel (``risk_premia_gamma``), the BDF
        branch and Q_VAR raise NotImplementedError.  ``with_theta``: also ``theta`` = -d price / d ttm per maturity (DESIGN.md §4.8), exact on
        the solver's accepted mesh with the earlier maturities and the grid held; every other output bit for bit."""
        from .fourier_greeks import check_fourier_greeks_kwargs, to_fourier_chain_greeks
        if params.risk_premia_gamma is not None:
            raise NotImplementedError("price_chain_greeks does not cover the risk-kernel pricer (risk_premia_gamma)")
        check_fourier_greeks_kwargs(kwargs)
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        out = engine.hawkesjd_price_chain_greeks(
            _params_c(**d), option_chain.ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
            option_chain.optiontypes_ttms, is_spot_measure=is_spot_measure, vol_scaler=kwargs.get("vol_scaler"), max_phi=MAX_PHI,
            **({"with_theta": True} if with_theta else {}))
        return to_fourier_chain_greeks(*out[:3], engine.HAWKES_GREEK_PARAMS, *out[3:])

    def price_chain_hessian(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True, **kwargs):
        """``price_chain_greeks`` (bit for bit) plus the second order in one call -> ``FourierChainHessian``: vanna (d^2 price / d forward
        d parameter) and the symmetric Hessian d^2 price / d p d q over HAWKES_GREEK_PARAMS, the exact second derivatives of the scheme on
        the adaptive solver's own mesh (DESIGN.md §4.5).  Same conventions and the same rejections as ``price_chain_greeks``."""
        from .fourier_greeks import check_fourier_hessian_kwargs, to_fourier_chain_hessian
        if params.risk_premia_gamma is not None:
            raise NotImplementedError("price_chain_hessian does not cover the risk-kernel pricer (risk_premia_gamma)")
        check_fourier_hessian_kwargs(kwargs)
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        prices, greeks, vanna, hessian, offsets = engine.hawkesjd_price_chain_hessian(
            _params_c(**d), option_chain.ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
            option_chain.optiontypes_ttms, is_spot_measure=is_spot_measure, vol_scaler=kwargs.get("vol_scaler"), max_phi=MAX_PHI)
        return to_fourier_chain_hessian(prices, greeks, vanna, hessian, offsets, engine.HAWKES_GREEK_PARAMS)

    def price_chain_risk_premia_greeks(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True, **kwargs):
        """Fourier prices under the risk kernel exp(-gamma x), gamma = ``params.risk_premia_gamma`` (bit-identical to ``price_chain``
        with the same arguments), plus forward-mode sensitivities in one call -> ``FourierChainGreeks`` keyed by
        HAWKES_RISK_PREMIA_GREEK_PARAMS: delta and gamma in the slice forward, d price / d HAWKES_GREEK_PARAMS and d price /
        d risk_premia_gamma, through the grid (which sits on Re phi = -1/2 - gamma), the two normaliser solves and K^(1 + gamma)
        (DESIGN.md §4.12).  Exact on the solver's own meshes with the grid's imaginary parts held fixed: pin ``vol_scaler`` to compare
        against re-pricings, since the default's dependence on ``sigma`` is not differentiated.  Rejects, before any GPU work: no
        ``risk_premia_gamma`` (ValueError: ``price_chain_greeks`` covers the plain pricer), a non-finite one (ValueError), the BDF
        branch, Q_VAR and ``with_theta`` (NotImplementedError), another measure or types other than 'C' / 'P' (ValueError, as
        ``price_chain``)."""
        from .fourier_greeks import to_fourier_chain_greeks
        gamma = _check_risk_premia_greeks(option_chain, params, is_spot_measure, kwargs, "price_chain_risk_premia_greeks")
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        out = engine.hawkesjd_price_chain_risk_premia_greeks(
            _params_c(**d), gamma, option_chain.ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
            option_chain.optiontypes_ttms, vol_scaler=kwargs.get("vol_scaler"), max_phi=MAX_PHI)
        return to_fourier_chain_greeks(*out, engine.HAWKES_RISK_PREMIA_GREEK_PARAMS)

    def compute_chain_risk_premia_ivol_greeks(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True,
                                              **kwargs):
        """implied-vol sensitivities under the risk kernel -> ``ChainIvolGreeks`` keyed by HAWKES_RISK_PREMIA_GREEK_PARAMS, among them
        d ivol / d risk_premia_gamma: ``price_chain_risk_premia_greeks`` mapped by the Black-76 transform (DESIGN.md §4.6).  The ivols are
        bit-identical to ``compute_chain_prices_with_vols`` with the same arguments; same rejections as ``price_chain_risk_premia_greeks``."""
        from .fourier_greeks import to_chain_ivol_sensitivities
        _check_risk_premia_greeks(option_chain, params, is_spot_measure, kwargs, "compute_chain_risk_premia_ivol_greeks")
        return to_chain_ivol_sensitivities(option_chain, self.price_chain_risk_premia_greeks(option_chain, params, is_spot_measure, **kwargs))

    def price_chain_risk_premia_hessian(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True, **kwargs):
        """``price_chain_risk_premia_greeks`` (bit for bit) plus the second order in one call -> ``FourierChainHessian`` keyed by
        HAWKES_RISK_PREMIA_GREEK_PARAMS: vanna (d^2 price / d forward d parameter) and the symmetric Hessian d^2 price / d p d q, the
        curvature in ``risk_premia_gamma`` included, through the grid, the two normaliser solves and K^(1 + gamma) (DESIGN.md §4.13).  The
        exact second derivatives of the scheme on the solver's own meshes with the grid's imaginary parts held fixed; same conventions and
        the same rejections as ``price_chain_risk_premia_greeks``."""
        from .fourier_greeks import to_fourier_chain_hessian
        gamma = _check_risk_premia_greeks(option_chain, params, is_spot_measure, kwargs, "price_chain_risk_premia_hessian")
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        prices, greeks, vanna, hessian, offsets = engine.hawkesjd_price_chain_risk_premia_hessian(
            _params_c(**d), gamma, option_chain.ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms,
            option_chain.optiontypes_ttms, vol_scaler=kwargs.get("vol_scaler"), max_phi=MAX_PHI)
        return to_fourier_chain_hessian(prices, greeks, vanna, hessian, offsets, engine.HAWKES_RISK_PREMIA_GREEK_PARAMS)

    def compute_chain_risk_premia_ivol_hessian(self, option_chain: OptionChain, params: HawkesJDParams, is_spot_measure: bool = True,
                                               **kwargs):
        """implied-vol second order under the risk kernel -> ``ChainIvolHessian`` keyed by HAWKES_RISK_PREMIA_GREEK_PARAMS:
        ``price_chain_risk_premia_hessian`` mapped by the Black-76 transform (DESIGN.md §4.6, §4.13).  The ivols are bit-identical to
        ``compute_chain_prices_with_vols`` with the same arguments; same rejections as ``price_chain_risk_premia_greeks``."""
        from .fourier_greeks import to_chain_ivol_sensitivities
        _check_risk_premia_greeks(option_chain, params, is_spot_measure, kwargs, "compute_chain_risk_premia_ivol_hessian")
        return to_chain_ivol_sensitivities(option_chain, self.price_chain_risk_premia_hessian(option_chain, params, is_spot_measure, **kwargs))

    @timer
    def model_mc_price_chain(self, option_chain: OptionChain, params: HawkesJDParams, nb_path: int = 100000, scheme: str = "euler", **kwargs
                             ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """MC prices and standard errors of the chain (reference :156-171).  ``scheme``: 'euler' (default, the reference's scheme) or
        'exact', the event-driven simulation of the continuous-time model the Fourier route prices (DESIGN.md §3.13); see
        ``hawkesjd_mc_chain_pricer``."""
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        return hawkesjd_mc_chain_pricer(ttms=option_chain.ttms, forwards=option_chain.forwards, discfactors=option_chain.discfactors,
                                        strikes_ttms=option_chain.strikes_ttms, optiontypes_ttms=option_chain.optiontypes_ttms, nb_path=nb_path,
                                        seed=kwargs.get("seed"), gauss=kwargs.get("gauss", "fp32"),
                                        variable_type=kwargs.get("variable_type", VariableType.LOG_RETURN),
                                        distributed=kwargs.get("distributed", True), exchange=kwargs.get("exchange"), scheme=scheme,
                                        max_candidates=kwargs.get("max_candidates"), **d)

    @timer
    def model_mc_chain_greeks(self, option_chain: OptionChain, params: HawkesJDParams, nb_path: int = 100000, seed: Optional[int] = None,
                              gauss: str = "fp32", scheme: str = "euler", **kwargs):
        """MC prices and standard errors bit-identical to ``model_mc_price_chain`` with the same ``nb_path`` / ``seed`` / ``gauss`` (one GPU),
        plus the forward delta and d price / d HAWKES_GREEK_PARAMS (the Fourier route's 15 names and order; ``mu`` is excluded there too),
        each with its standard error df std(g) / sqrt(N) -> ``McChainGreeks``.  Pathwise with the firing decisions frozen plus the
        likelihood-ratio score of the decisions (DESIGN.md §3.11): unbiased for the discretised scheme the pricer simulates.  LOG_RETURN,
        fp64 state, ``gauss`` 'fp32' / 'fp64'; Q_VAR, ``exchange``, another ``precision`` or a set ``risk_premia_gamma`` raise
        NotImplementedError, ``mean_p == 0`` or ``mean_m == 0`` (degenerate jump sizes) ValueError.  Under torch.distributed every rank prices all paths (replicated, bit-identical results).
        ``scheme``: 'euler' only; 'exact' (no sensitivities on that route) raises NotImplementedError, another value ValueError."""
        from .mc_greeks import check_hawkes_mc_greeks_kwargs, check_no_gamma, check_no_theta, to_mc_chain_greeks
        if _is_exact(scheme):
            raise NotImplementedError("model_mc_chain_greeks covers scheme='euler' only: the exact route has no sensitivities")
        check_no_gamma(kwargs, "HawkesJDPricer.model_mc_chain_greeks")
        check_no_theta(kwargs, "HawkesJDPricer.model_mc_chain_greeks",
                       "the firing clock's dt enters through the likelihood-ratio score and the dt*(1 +- 1e-9) comparison constants; "
                       "price_chain_greeks(with_theta=True) has the Fourier theta")
        check_hawkes_mc_greeks_kwargs(kwargs, gauss, params)
        d = params.to_dict()
        d.pop("risk_premia_gamma", None)
        res = engine.hawkesjd_mc_chain_greeks(_params_c(**d), option_chain.ttms, option_chain.forwards, option_chain.discfactors,
                                              option_chain.strikes_ttms, option_chain.optiontypes_ttms, nb_path, C.LOG_RETURN, _shared_seed(seed),
                                              engine.mc_flags("fp64", gauss))
        return to_mc_chain_greeks(res[:5], engine.HAWKES_GREEK_PARAMS)

    # ---- calibration drivers (reference :230-357): SLSQP on the host around the batched GPU Fourier chain pricer ---------------------
    @timer
    def calibrate_model_params_to_chain(self, option_chain: OptionChain, params0: HawkesJDParams, is_vega_weighted: bool = True,
                                        is_unit_ttm_vega: bool = False, return_info: bool = False, **kwargs):
        """fit (sigma, mean_p, mean_m, theta_p, theta_m, kappa, beta_p, beta_m) to the chain's mid vols with shifts and initial intensities
        fixed at ``params0``'s; kappa is shared by the two intensities and beta_p / beta_m enter as +beta / -beta pairs (reference :230-300, same
        start vector -- including its beta_m start 0.5 (beta2_p - beta2_m) --, bounds, stationarity constraint and SLSQP options).
        ``disp`` / ``maxiter`` (extras) are handed to SLSQP.  The 8 difference neighbours of a point whose gradient SLSQP asks for are priced
        in one ``hawkesjd_price_chain_batch`` call; objective and gradient are bit for bit what SLSQP differences from the one-set objective,
        so the fit is too.  ``return_info``: (fit, {"fun", "nit", "nb_batches", "x", "nan_quotes"}).  ``gradient='exact'`` hands SLSQP the
        exact gradient from one ``compute_chain_ivol_greeks`` call per point, on ``params0``'s default grid (DESIGN.md §4.6)."""
        return calibrate_hawkes(self, option_chain, params0, is_vega_weighted, is_unit_ttm_vega, return_info, **kwargs)

    def calibrate_model_params_to_chains(self, option_chains: List[OptionChain], params0, is_vega_weighted: bool = True,
                                         is_unit_ttm_vega: bool = False, return_info: bool = False, gradient: str = "difference",
                                         return_exceptions: bool = False, max_sets_per_call: Optional[int] = None, **kwargs):
        """``calibrate_model_params_to_chain`` on every chain of ``option_chains``, in lock-step: one ``engine.hawkesjd_price_chains_batch``
        call per optimizer round, each chain's parameter sets in one Riccati launch, every fit bit for bit the single-chain driver's
        (DESIGN.md §4.10).  ``params0``: one HawkesJDParams or a list of one per chain (``risk_premia_gamma`` ignored, as by the single-chain
        fit); ``gradient='difference'`` only; ``disp`` / ``maxiter`` (extras) as there.  -> list of fits, with ``return_info`` (fits, infos)
        whose info dicts add ``rounds`` (library calls of the run).  ``return_exceptions``: a failed fit's slot holds its exception instead
        of raising the first one after all fits have ended.  ``max_sets_per_call`` splits a round into calls of at most that many sets
        (never one fit's sets).  Every chain runs in a thread of its own while the caller's thread prices."""
        return calibrate_hawkes_chains(self, option_chains, params0, is_vega_weighted, is_unit_ttm_vega, return_info=return_info,
                                       gradient=gradient, return_exceptions=return_exceptions, max_sets_per_call=max_sets_per_call, **kwargs)

    @timer
    def calibrate_risk_premia_gamma_to_chain(self, option_chain: OptionChain, params0: HawkesJDParams, is_vega_weighted: bool = True,
                                             is_unit_ttm_vega: bool = False, maxiter: int = 100, print_iter: bool = True, return_info: bool = False,
                                             **kwargs):
        """fit (sigma, risk_premia_gamma) with every other parameter of ``params0`` fixed (reference :303-357: gamma scaled by 8 into (-1, 1),
        weights x 1e4, SLSQP with finite-difference step 0.025, ftol = tol = 1e-16).  Returns a new object; the reference mutates ``params0``.
        The 2 difference neighbours of a point whose gradient SLSQP asks for are priced in one risk-kernel ``hawkesjd_price_chain_batch``
        call, with the fit of the one-set objective bit for bit; ``print_iter`` prints a line per point in the order that objective would (the neighbours
        only when SLSQP asks for the gradient).  ``return_info``: (fit, {"fun", "nit", "nb_batches", "x", "nan_quotes"}).  The risk kernel
        has no sensitivities, so ``gradient='exact'`` raises NotImplementedError."""
        return calibrate_hawkes_risk_premia(option_chain, params0, is_vega_weighted, is_unit_ttm_vega, maxiter=maxiter, print_iter=print_iter,
                                            return_info=return_info, **kwargs)

    def calibrate_risk_premia_gamma_to_chains(self, option_chains: List[OptionChain], params0, is_vega_weighted: bool = True,
                                              is_unit_ttm_vega: bool = False, maxiter: int = 100, print_iter: bool = False,
                                              return_info: bool = False, gradient: str = "difference", return_exceptions: bool = False,
                                              max_sets_per_call: Optional[int] = None, **kwargs):
        """``calibrate_risk_premia_gamma_to_chain`` on every chain of ``option_chains``, in lock-step: one risk-kernel
        ``engine.hawkesjd_price_chains_batch`` call per optimizer round, every fit bit for bit the single-chain driver's (DESIGN.md §4.11).
        ``params0``: one HawkesJDParams or a list of one per chain, each with its own start (sigma, gamma; a ``None`` gamma starts at 0) and
        fixed fields.  ``print_iter``: each chain's lines, exactly what the single-chain driver prints, as one block per chain in chain order
        once every fit has ended.  ``gradient='difference'`` only.  ``return_info``, ``return_exceptions`` and ``max_sets_per_call`` as for
        ``calibrate_model_params_to_chains``, and the info dicts add ``rounds``."""
        return calibrate_hawkes_risk_premia_chains(option_chains, params0, is_vega_weighted, is_unit_ttm_vega, maxiter=maxiter,
                                                   print_iter=print_iter, return_info=return_info, gradient=gradient,
                                                   return_exceptions=return_exceptions, max_sets_per_call=max_sets_per_call, **kwargs)

    @timer
    def simulate_terminal_values(self, params: HawkesJDParams, ttm: float = 1.0, nb_path: int = 100000, is_spot_measure: bool = True,
                                 scheme: str = "euler", **kwargs) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """terminal (x, lambda_p, lambda_m) from (0, lambda_p, lambda_m) (reference :193-224); ``scheme`` as in ``model_mc_price_chain``"""
        d = {k: v for k, v in params.to_dict().items() if k in _KEYS and k not in ("lambda_p", "lambda_m")}
        return simulate_hawkesjd_terminal(ttm=ttm, x0=np.zeros(1), lambda_p0=params.lambda_p * np.ones(1), lambda_m0=params.lambda_m * np.ones(1),
                                          nb_path=nb_path, seed=kwargs.get("seed"), gauss=kwargs.get("gauss", "fp32"), scheme=scheme,
                                          max_candidates=kwargs.get("max_candidates"), **d)


def hawkesjd_mc_chain_pricer(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, lambda_p: float, lambda_m: float, mu: float, sigma: float,
                             shift_p: float, mean_p: float, shift_m: float, mean_m: float, theta_p: float, kappa_p: float, beta1_p: float,
                             beta2_p: float, theta_m: float, kappa_m: float, beta1_m: float, beta2_m: float, risk_premia_gamma: float = 0.0,
                             nb_path: int = 100000, variable_type: VariableType = VariableType.LOG_RETURN, seed: Optional[int] = None,
                             gauss: str = "fp32", distributed: bool = True, exchange: Optional[str] = None, scheme: str = "euler",
                             max_candidates: Optional[int] = None) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """chain prices and standard errors by simulating the jump-diffusion (reference :644-715): the terminal (x, lambda_p, lambda_m) of slice m
    seeds slice m+1; payoffs are forward-recentred on x (utils/mc_payoffs.py).  Under an initialised torch.distributed world ``nb_path`` is
    the TOTAL path count, sharded over the ranks by global path id (the LogSV chain's two exchanges per maturity, multi_gpu.py).

    ``scheme``: 'euler' (default) steps the reference's scheme at 1800 steps per year, the route whose numbers the reference pins.
    'exact' simulates the continuous-time model event by event by thinning, with no time grid and no discretisation bias (DESIGN.md
    §3.13): where the intensities cannot become negative it is the model the Fourier route prices.  The two are different discretisations,
    not two implementations of one result.  On the exact route ``gauss`` is not consulted (its draws are fp64), a parameter set whose bound
    on the expected events per path over the chain exceeds HAWKES_EXACT_MAX_EXPECTED_EVENTS raises ValueError before any GPU work, and
    ``max_candidates`` (default engine.HAWKES_EXACT_DEFAULT_BUDGET) caps the candidates per path and maturity: a path that reaches it fails
    the call with B200svError(-6), never with biased prices."""
    exact = _is_exact(scheme)
    vt = engine.variable_code(variable_type)
    pc = _params_c(**locals())
    if exact:
        _check_exact_events(float(np.max(ttms)), {k: getattr(pc, k) for k in _KEYS})
        budget = engine.HAWKES_EXACT_DEFAULT_BUDGET if max_candidates is None else int(max_candidates)
        flags = engine.mc_flags("fp64")
        seed = _shared_seed(seed)
        if _use_distributed({"distributed": distributed, "nb_path": nb_path, "exchange": exchange}):
            t = np.asarray(ttms, dtype=np.float64)
            grid = [(1, float(t[m] - (t[m - 1] if m > 0 else 0.0))) for m in range(t.shape[0])]
            return mc_chain_distributed("hawkes_exact", pc, ttms, forwards, discfactors, None, strikes_ttms, optiontypes_ttms, nb_path,
                                        STEPS_PER_YEAR, True, vt, seed, flags, exchange=exchange, grid=grid, max_candidates=budget)
        return engine.hawkesjd_mc_chain_exact(pc, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path, vt, seed, flags, budget)[:2]
    seed = _shared_seed(seed)
    if _use_distributed({"distributed": distributed, "nb_path": nb_path, "exchange": exchange}):
        return mc_chain_distributed("hawkes", pc, ttms, forwards, discfactors, None, strikes_ttms, optiontypes_ttms, nb_path, STEPS_PER_YEAR,
                                    True, vt, seed, engine.mc_flags("fp64", gauss), exchange=exchange)
    return engine.hawkesjd_mc_chain(pc, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path, vt, seed, engine.mc_flags("fp64", gauss))


def simulate_hawkesjd_terminal(ttm: float, x0: np.ndarray, lambda_p0: np.ndarray, lambda_m0: np.ndarray, mu: float, sigma: float, shift_p: float,
                               mean_p: float, shift_m: float, mean_m: float, theta_p: float, kappa_p: float, beta1_p: float, beta2_p: float,
                               theta_m: float, kappa_m: float, beta1_m: float, beta2_m: float, nb_path: int = 100000, seed: Optional[int] = None,
                               gauss: str = "fp32", slice_index: int = 0, inputs=None, scheme: str = "euler", max_candidates: Optional[int] = None
                               ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """terminal (log-return, lambda_p, lambda_m) with both Hawkes intensities evolving jointly (reference :718-779).  Length-1 initial
    arrays broadcast as in the reference (:742-750: x0 -> zeros, intensities -> constants).  ``inputs = (W0, U_P, U_M, J_P, J_M)`` (extra;
    [nb_steps, nb_path] each, in the form :753-757 builds them) runs the strict kernel on caller-supplied draws.  ``scheme``, ``gauss``
    and ``max_candidates`` as in ``hawkesjd_mc_chain_pricer``; ``inputs`` are Euler draws, so ``scheme='exact'`` with ``inputs`` raises
    ValueError."""
    exact = _is_exact(scheme)
    if exact and inputs is not None:
        raise ValueError("inputs= feeds the Euler scheme's strict kernel: it cannot be combined with scheme='exact'")
    x0, lambda_p0, lambda_m0 = np.atleast_1d(x0), np.atleast_1d(lambda_p0), np.atleast_1d(lambda_m0)
    for a in (x0, lambda_p0, lambda_m0):
        assert a.shape[0] in (1, nb_path)
    x = np.zeros(nb_path) if x0.shape[0] == 1 else np.array(x0, dtype=np.float64)
    lp = lambda_p0 * np.ones(nb_path) if lambda_p0.shape[0] == 1 else np.array(lambda_p0, dtype=np.float64)
    lm = lambda_m0 * np.ones(nb_path) if lambda_m0.shape[0] == 1 else np.array(lambda_m0, dtype=np.float64)
    x, lp, lm = (np.ascontiguousarray(a, dtype=np.float64) for a in (x, lp, lm))
    pc = _params_c(lambda_p=float(lp[0]), lambda_m=float(lm[0]), **{k: v for k, v in locals().items() if k in _KEYS})
    nb_steps, dt, _ = set_time_grid(ttm=ttm, nb_steps_per_year=STEPS_PER_YEAR)
    if inputs is not None:
        blocks = [C.f64(b) for b in inputs]
        if len(blocks) != 5 or any(b.shape != (nb_steps, nb_path) for b in blocks):
            raise ValueError(f"inputs must be five arrays of shape ({nb_steps}, {nb_path})")
        return engine.hawkesjd_step_fixed(x, lp, lm, blocks, nb_steps, nb_path, dt, pc)
    const_start = x0.shape[0] == 1 and lambda_p0.shape[0] == 1 and lambda_m0.shape[0] == 1
    if exact:
        kw = {k: getattr(pc, k) for k in _KEYS}
        _check_exact_events(float(ttm), {**kw, "lambda_p": float(np.max(np.abs(lp))), "lambda_m": float(np.max(np.abs(lm)))})
        return engine.hawkesjd_terminal_exact(pc, ttm, x, lp, lm, engine.fresh_seed() if seed is None else int(seed), slice_index, not const_start,
                                              engine.HAWKES_EXACT_DEFAULT_BUDGET if max_candidates is None else int(max_candidates))
    return engine.hawkesjd_terminal(pc, ttm, x, lp, lm, engine.fresh_seed() if seed is None else int(seed), engine.mc_flags("fp64", gauss),
                                    slice_index, not const_start)


def hawkesjd_device_draws(seed: int, path0: int, n: int, slice_index: int, ttm: float, gauss: str = "fp32", **params):
    """(W0, U_P, U_M, J_P, J_M, dt): what the in-kernel generator draws for paths [path0, path0 + n) of a slice of length ``ttm``, in the
    reference's form (test / diagnostics hook)."""
    pc = _params_c(**{**{k: 0.0 for k in _KEYS}, **params})
    S, dt, _ = set_time_grid(ttm=ttm, nb_steps_per_year=STEPS_PER_YEAR)
    return (*engine.hawkesjd_device_draws(seed, path0, n, slice_index, S, dt, pc, engine.mc_flags("fp64", gauss)), dt)


MAX_PHI = 500           # transform grid size of the Fourier route (reference :37)


def set_vol_scaler(sigma0: float, ttm: float) -> float:
    """grid scaler of the Fourier route (reference :360-362)"""
    return float(np.clip(sigma0, 0.2, 0.5) * np.sqrt(np.minimum(ttm, 1.0 / 12.0)))


def _fourier_chain(model_params: HawkesJDParams, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_stiff_solver, is_spot_measure,
                   variable_type, vol_scaler, gamma, return_grids=False):
    if getattr(variable_type, "value", variable_type) != VariableType.LOG_RETURN.value:
        raise NotImplementedError           # reference :413-414
    if is_stiff_solver:
        raise NotImplementedError("is_stiff_solver: the Hawkes Fourier route runs SciPy's RK45 control law on the GPU; its BDF variant is not built")
    if gamma is None:
        engine._check_fourier_types(optiontypes_ttms, bool(is_spot_measure))
    elif not is_spot_measure or any(str(t) not in ("C", "P") for types in optiontypes_ttms for t in types):
        raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318
    d = model_params.to_dict()
    d.pop("risk_premia_gamma", None)
    return engine.hawkesjd_price_chain(_params_c(**d), ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_spot_measure, vol_scaler,
                                       MAX_PHI, gamma, return_grids)


def hawkesjd_chain_pricer(model_params: HawkesJDParams, ttms: np.ndarray, forwards: np.ndarray, discfactors: np.ndarray, strikes_ttms, optiontypes_ttms,
                          is_stiff_solver: bool = False, is_spot_measure: bool = True, variable_type: VariableType = VariableType.LOG_RETURN,
                          vol_scaler: float = None, return_grids: bool = False) -> List[np.ndarray]:
    """Fourier chain prices of the Hawkes jump-diffusion (reference :365-417): Riccati ODEs for (a0, a_p, a_m) on a 500-point transform grid
    with SciPy's RK45 control law per point, carried over the maturities, then the vanilla slice pricer -- one GPU call"""
    return _fourier_chain(model_params, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_stiff_solver, is_spot_measure, variable_type,
                          vol_scaler, None, return_grids)


def hawkesjd_chain_pricer_with_risk_premia(model_params: HawkesJDParams, ttms: np.ndarray, forwards: np.ndarray, discfactors: np.ndarray, strikes_ttms,
                                           optiontypes_ttms, is_stiff_solver: bool = False, is_spot_measure: bool = True,
                                           variable_type: VariableType = VariableType.LOG_RETURN, vol_scaler: float = None,
                                           return_grids: bool = False) -> List[np.ndarray]:
    """Fourier chain prices under the risk kernel exp(-gamma x) (reference :420-484; grid on Re = -1/2 - gamma, normalisers and forwards under the
    kernel from two single-point solves per maturity, gamma slice pricer without discounting -- all as in the reference)"""
    return _fourier_chain(model_params, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_stiff_solver, is_spot_measure, variable_type,
                          vol_scaler, model_params.risk_premia_gamma, return_grids)


def hawkesjd_forwards_under_risk_kernel(model_params: HawkesJDParams, risk_premia_gamma: float, ttms: np.ndarray, forwards: np.ndarray,
                                        is_stiff_solver: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """(normalizers, gamma_forwards) per maturity (reference :487-515)"""
    ttms, forwards = np.asarray(ttms, dtype=float), np.asarray(forwards, dtype=float)
    one = [np.ones(1) for _ in ttms]
    p = HawkesJDParams(**{**model_params.to_dict(), "risk_premia_gamma": float(risk_premia_gamma)})
    _, _, _, norm, gfw = _fourier_chain(p, ttms, forwards, np.ones_like(ttms), one, [np.array(["C"]) for _ in ttms], is_stiff_solver, True,
                                        VariableType.LOG_RETURN, None, float(risk_premia_gamma), return_grids=True)
    return norm, gfw


def compute_hawkes_a_mgf_grid(ttm: float, phi_grid: np.ndarray, model_params: HawkesJDParams, psi_grid: Optional[np.ndarray] = None,
                              a_t0: Optional[np.ndarray] = None, is_stiff_solver: bool = False, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
    """(a_t1 [P, 3], log_mgf [P]) over a caller-supplied transform grid (reference :518-547): A(ttm) from A(0) = ``a_t0`` (zeros by default) and
    log-MGF = a0 + a_p lambda_p + a_m lambda_m"""
    if is_stiff_solver:
        raise NotImplementedError("is_stiff_solver: the Hawkes Fourier route runs SciPy's RK45 control law on the GPU; its BDF variant is not built")
    phi = C.c128(phi_grid)
    psi = None if psi_grid is None else C.c128(psi_grid)
    a = np.zeros((phi.shape[0], 3), dtype=np.complex128) if a_t0 is None else np.ascontiguousarray(a_t0, dtype=np.complex128).copy()
    if a.shape != (phi.shape[0], 3):
        raise ValueError("a_t0 must have shape (len(phi_grid), 3)")
    d = model_params.to_dict()
    d.pop("risk_premia_gamma", None)
    return a, engine.hawkesjd_mgf_grid(phi, psi, ttm, a, _params_c(**d))


def solve_a_ode_grid(phi_grid: np.ndarray, ttm: float, model_params: HawkesJDParams, psi_grid: Optional[np.ndarray] = None,
                     a_t0: Optional[np.ndarray] = None, is_stiff_solver: bool = False) -> np.ndarray:
    """A(ttm) per transform point (reference :550-579)"""
    return compute_hawkes_a_mgf_grid(ttm, phi_grid, model_params, psi_grid=psi_grid, a_t0=a_t0, is_stiff_solver=is_stiff_solver)[0]
