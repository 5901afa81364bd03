"""LogSVPricer on H100: drop-in for the two hot paths of the reference ``pricers/logsv_pricer.py``.

Same public names, argument meaning, defaults, return shapes and exception classes as the reference:

* ``LogSVPricer.price_chain``                 (logsv_pricer.py:345-366)  -> ``logsv_chain_pricer`` (:669-739)
* ``LogSVPricer.model_mc_price_chain``        (:369-427)                -> ``logsv_mc_chain_pricer`` (:806-867)
* ``LogSVPricer.simulate_terminal_values``    (:590-611)                -> ``simulate_logsv_x_vol_terminal`` (:950-1047)
* ``logsv_mc_chain_pricer_fixed_randoms``     (:1100-1162), ``get_randoms_for_chain_valuation`` (:1051-1074)
* inherited ``compute_chain_prices_with_vols`` / ``price_slice`` / ``price_vanilla`` / ``compute_mc_chain_implied_vols``

Extra OPTIONAL kwargs (all default to reference behaviour where one exists): ``seed`` (the reference draws from Numba's global
RNG and exposes no seed; default = OS entropy), ``precision`` ('fp64' | 'fp32'), ``gauss`` ('fp32' | 'fp64'), ``distributed``
(shard ``nb_path`` over the ranks of an initialised ``torch.distributed`` world; default True when one exists).
Unknown kwargs are accepted and ignored on both routes, as in the reference (:349, :376, :681).

``LogSVPricer.calibrate_model_params_to_chain`` (:441-558) runs on the batched GPU chain pricer (pricers/calibration.py); the
rough-vol route (``use_rough_mc=True``, :1164-1232 -> rough_logsv/split_simulation.py) runs on csrc/rough_kernels.cuh.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from .. import _capi as C
from .. import engine
from ..data.option_chain import OptionChain
from ..multi_gpu import CudaMcEngine, _fixed_randoms_chain_device, _shared_seed, _use_distributed, mc_chain_distributed, shard_paths
from ..multi_gpu import _fixed_randoms_chain_greeks_device
from ..multi_gpu import SHARD_MIN_PATHS  # noqa: F401  (the MC routing policy lives in multi_gpu; this name stays importable from here)
from ..utils.config import VariableType
from ..utils.funcs import set_time_grid, timer
from .calibration import CalibrationEngine, ConstraintsType, LogsvModelCalibrationType, calibrate_logsv
from .logsv.affine_expansion import ExpansionOrder, _order_code
from .model_pricer import ModelParams, ModelPricer


@dataclass
class LogSvParams(ModelParams):
    """the six parameters of the log-normal SV model with quadratic drift (reference pricers/logsv/logsv_params.py:35-83),
    plus the optional ``vol_backbone`` term structure (a pandas Series of eta indexed by maturity)."""
    sigma0: float = 0.2
    theta: float = 0.2
    kappa1: float = 1.0
    kappa2: Optional[float] = 2.5
    beta: float = -1.0
    volvol: float = 1.0
    vol_backbone: Any = None
    H: float = 0.5                  # Hurst exponent of the rough extension (logsv_params.py:81); 1/2 = the article's model
    weights: Any = None             # quadrature weights / nodes of the Markovian lift of the rough kernel (:82-83)
    nodes: Any = None

    def __post_init__(self):
        if self.kappa2 is None:              # logsv_params.py:92-93
            self.kappa2 = self.kappa1 / self.theta
        assert 1e-4 < self.H <= 0.5          # :94

    def approximate_kernel(self, T: float) -> None:
        """nodes / weights of the Markovian approximation of the rough kernel (logsv_params.py:96-118).  H in (0.49, 1/2] is the single
        node 1e-3 with weight 1 (the non-rough dynamics).  Smaller H needs the reference's 'European' quadrature optimiser
        (rough_logsv/rough_kernel.py:927, a 1200-line scipy optimisation outside the Monte Carlo hot path): it is not rebuilt here --
        set ``weights`` / ``nodes`` from it (or any other quadrature rule) yourself."""
        if 0.49 < self.H <= 0.5:
            self.weights = np.array([1.0])
            self.nodes = np.array([1e-3])
            return
        raise NotImplementedError("approximate_kernel for H <= 0.49 needs the reference's european_rule optimiser (out of the hot path): "
                                  "assign params.weights / params.nodes directly")

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)

    def to_str(self) -> str:
        return (f"sigma0={self.sigma0:0.2f}, theta={self.theta:0.2f}, kappa1={self.kappa1:0.2f}, kappa2={self.kappa2:0.2f}, "
                f"beta={self.beta:0.2f}, volvol={self.volvol:0.2f}")

    def set_vol_backbone(self, vol_backbone) -> None:
        self.vol_backbone = vol_backbone

    def get_vol_backbone_eta(self, tau: float) -> float:
        """eta at the nearest quoted maturity at or beyond tau; 1.0 without a backbone (logsv_params.py:140-151)."""
        if self.vol_backbone is None:
            return 1.0
        index = np.asarray(self.vol_backbone.index, dtype=float)
        return float(np.asarray(self.vol_backbone)[np.searchsorted(index, tau, side="left")])

    def get_vol_backbone_etas(self, ttms: np.ndarray) -> np.ndarray:
        return np.array([self.get_vol_backbone_eta(tau) for tau in ttms], dtype=float)

    @property
    def kappa(self) -> float:
        return self.kappa1 + self.kappa2 * self.theta

    @property
    def theta2(self) -> float:
        return self.theta * self.theta

    @property
    def vartheta2(self) -> float:
        return self.beta * self.beta + self.volvol * self.volvol

    @property
    def gamma(self) -> float:
        """kappa1 / theta: the quadratic mean-reversion rate of the pure quadratic drift (logsv_params.py:189-196)"""
        return self.kappa1 / self.theta

    @property
    def eta(self) -> float:
        """exponent of the steady-state (generalised inverse Gaussian) vol density, 2 (kappa2 theta - kappa1) / vartheta^2 - 1 (:198-207)"""
        return 2.0 * (self.kappa2 * self.theta - self.kappa1) / self.vartheta2 - 1.0

    # spatial grids for the densities of logsv_pdfs (logsv_params.py:209-267): n points; width set by the average of sigma0^2 and theta^2
    def get_x_grid(self, ttm: float = 1.0, n_stdevs: float = 3.0, n: int = 200) -> np.ndarray:
        total_vol = np.sqrt(0.5 * ttm * (self.sigma0 ** 2 + self.theta ** 2))
        centre, half_width = -0.5 * total_vol * total_vol, (n_stdevs + 1) * total_vol
        return np.linspace(centre - half_width, centre + half_width, n)

    def get_sigma_grid(self, ttm: float = 1.0, n_stdevs: float = 3.0, n: int = 200) -> np.ndarray:
        level = np.sqrt(0.5 * (self.sigma0 ** 2 + self.theta ** 2))
        return np.linspace(0.0, level + n_stdevs * 0.5 * np.sqrt(self.vartheta2 * ttm), n)

    def get_qvar_grid(self, ttm: float = 1.0, n_stdevs: float = 3.0, n: int = 200) -> np.ndarray:
        level = np.sqrt(ttm * (self.sigma0 ** 2 + self.theta ** 2))
        return np.linspace(0.0, level + n_stdevs * np.sqrt(self.vartheta2) * ttm, n)

    def get_variable_space_grid(self, variable_type: VariableType = VariableType.LOG_RETURN, ttm: float = 1.0, n_stdevs: float = 3,
                                n: int = 200) -> np.ndarray:
        code = getattr(variable_type, "value", variable_type)            # by value: the reference's own enum duck-types
        grid = {VariableType.LOG_RETURN.value: self.get_x_grid, VariableType.SIGMA.value: self.get_sigma_grid,
                VariableType.Q_VAR.value: self.get_qvar_grid}.get(code)
        if grid is None:
            raise NotImplementedError
        return grid(ttm=ttm, n_stdevs=n_stdevs, n=n)

    def get_vol_moments_lambda(self, n_terms: int = 4) -> np.ndarray:
        """generator Lambda^(1,k*) of the truncated vol-moment system, Eq. (3.48) (logsv_params.py:269-323)"""
        from .logsv.vol_moments import vol_moments_generator
        return vol_moments_generator(self, n_terms=n_terms)

    def assert_vol_moments_stability(self, n_terms: int = 4):
        """prints (does not assert, as in the reference :325-335) whether every eigenvalue of Lambda has a negative real part"""
        stable = bool(np.all(np.linalg.eigvals(self.get_vol_moments_lambda(n_terms)).real < 0.0))
        print(f"vol moments stable = {stable}")

    def print_vol_moments_stability(self, n_terms: int = 4) -> None:
        for order, label in ((2, "con2"), (3, "con3"), (4, "cond4")):       # diagonal conditions c(n) - n kappa (:337-357)
            print(f"{label}:\n{0.5 * self.vartheta2 * order * (order - 1.0) - order * self.kappa}")
        lam = self.get_vol_moments_lambda(n_terms)
        w = np.linalg.eigvals(lam)
        print(f"lambda_m:\n{lam}")
        print(f"eigenvalues w:\n{w}")
        print(f"vol moments stable = {bool(np.all(w.real < 0.0))}")


LOGSV_BTC_PARAMS = LogSvParams(sigma0=0.8376, theta=1.0413, kappa1=3.1844, kappa2=3.058, beta=0.1514, volvol=1.8458)   # logsv_pricer.py:102


def _params_c(params) -> C.LogsvParamsC:
    kappa2 = params.kappa2 if params.kappa2 is not None else params.kappa1 / params.theta
    return engine.logsv_params_c(params.sigma0, params.theta, params.kappa1, kappa2, params.beta, params.volvol)


class LogSVPricer(ModelPricer):
    """ModelPricer for the log-normal SV model, Fourier + Monte Carlo routes on the GPU."""

    def price_chain(self, option_chain: OptionChain, params: LogSvParams, is_spot_measure: bool = True, **kwargs) -> List[np.ndarray]:
        """Fourier prices of the chain (MMA measure Eqs. (5.4)/(5.9); inverse measure (5.13)/(5.16))."""
        kwargs.pop("vol_backbone_etas", None)
        return logsv_chain_pricer(params=params, ttms=option_chain.ttms, forwards=option_chain.forwards,
                                  discfactors=option_chain.discfactors, strikes_ttms=option_chain.strikes_ttms,
                                  optiontypes_ttms=option_chain.optiontypes_ttms, is_spot_measure=is_spot_measure, **kwargs)

    def price_chain_greeks(self, option_chain: OptionChain, params: LogSvParams, is_spot_measure: bool = True, with_theta: bool = False,
                           **kwargs):
        """Fourier prices (bit-identical to ``price_chain`` with the same arguments) plus forward-mode sensitivities in one call ->
        ``FourierChainGreeks``: delta and gamma in the slice forward and d price / d (sigma0, theta, kappa1, kappa2, beta, volvol).  Takes
        ``expansion_order``, ``vol_scaler`` and ``max_phi`` like ``price_chain``; ``kappa2`` is the value after ``__post_init__`` and is held
        fixed when kappa1 or theta moves; the vol backbone, the discount factors and the transform grid are not differentiated.  The
        semi-analytic and BDF branches, Q_VAR and the rough-vol route raise NotImplementedError.  ``with_theta``: also ``theta`` = -d price /
        d ttm per maturity (DESIGN.md §4.8), exact on the solver's accepted mesh with the earlier maturities, the backbone and the grid held;
        every other output bit for bit as without it."""
        from .fourier_greeks import check_fourier_greeks_kwargs, to_fourier_chain_greeks
        check_fourier_greeks_kwargs(kwargs)
        out = engine.logsv_price_chain_greeks(
            _params_c(params), option_chain.ttms, option_chain.forwards, option_chain.discfactors,
            params.get_vol_backbone_etas(ttms=option_chain.ttms), option_chain.strikes_ttms, option_chain.optiontypes_ttms,
            is_spot_measure=is_spot_measure, expansion_order=_order_code(kwargs.get("expansion_order", ExpansionOrder.SECOND)),
            vol_scaler=kwargs.get("vol_scaler"), max_phi=kwargs.get("max_phi"), **({"with_theta": True} if with_theta else {}))
        return to_fourier_chain_greeks(*out[:3], engine.LOGSV_GREEK_PARAMS, *out[3:])

    def price_chain_hessian(self, option_chain: OptionChain, params: LogSvParams, is_spot_measure: bool = True, **kwargs):
        """``price_chain_greeks`` (bit for bit) plus the second-order sensitivities in one call -> ``FourierChainHessian``: vanna
        d^2 price / d forward d p and the symmetric Hessian d^2 price / d p d q over (sigma0, theta, kappa1, kappa2, beta, volvol), exact
        second derivatives of the scheme on the adaptive solver's accepted steps.  Same arguments, conventions and rejections as
        ``price_chain_greeks``."""
        from .fourier_greeks import check_fourier_hessian_kwargs, to_fourier_chain_hessian
        check_fourier_hessian_kwargs(kwargs)
        prices, greeks, vanna, hessian, offsets = engine.logsv_price_chain_hessian(
            _params_c(params), option_chain.ttms, option_chain.forwards, option_chain.discfactors,
            params.get_vol_backbone_etas(ttms=option_chain.ttms), option_chain.strikes_ttms, option_chain.optiontypes_ttms,
            is_spot_measure=is_spot_measure, expansion_order=_order_code(kwargs.get("expansion_order", ExpansionOrder.SECOND)),
            vol_scaler=kwargs.get("vol_scaler"), max_phi=kwargs.get("max_phi"))
        return to_fourier_chain_hessian(prices, greeks, vanna, hessian, offsets, engine.LOGSV_GREEK_PARAMS)

    def set_vol_scaler(self, option_chain: OptionChain) -> float:
        """transform-grid scaler from the first slice's ATM vol (reference :436-439)."""
        return set_vol_scaler(sigma0=option_chain.get_chain_atm_vols()[0], ttm=option_chain.ttms[0])

    @timer
    def calibrate_model_params_to_chain(self, option_chain: OptionChain, params0: LogSvParams,
                                        params_min: Optional[LogSvParams] = None, params_max: Optional[LogSvParams] = None,
                                        is_vega_weighted: bool = True, is_unit_ttm_vega: bool = False,
                                        model_calibration_type: LogsvModelCalibrationType = LogsvModelCalibrationType.PARAMS5,
                                        constraints_type: ConstraintsType = ConstraintsType.UNCONSTRAINT,
                                        calibration_engine: CalibrationEngine = CalibrationEngine.ANALYTIC,
                                        nb_path: int = 100000, nb_steps: int = 360, seed: int = 10, **kwargs) -> LogSvParams:
        """fit model parameters to the chain's mid implied vols: vega-weighted squared vol errors (Eq. (6.3)) minimised by SLSQP under
        ``constraints_type`` (reference :441-558; same arguments, bounds and return type).  The objective and its finite-difference
        gradient are ONE batched GPU call per optimizer evaluation (pricers/calibration.py).  ``return_info=True`` also returns
        {fun, nit, nb_batches, x}.  ``gradient='exact'`` (ANALYTIC engine, PARAMS4 / PARAMS5) hands SLSQP the exact gradient of the
        objective from one ``compute_chain_ivol_greeks`` call per point instead of the forward difference (DESIGN.md §4.6).
        ``gradient='pathwise'`` (MC engine with either ``mc_randoms``, ROUGH_MC; PARAMS4 / PARAMS5) hands SLSQP the pathwise derivative of the
        sample objective on the fit's fixed normals from one Monte Carlo sensitivity pass per point (DESIGN.md §4.7); it is the derivative
        of the sample objective, not of the model.  A ROUGH_MC pathwise fit's ``return_info`` adds ``reset_paths``: per maturity, the most
        paths any evaluation saw take the reset-to-1e-6 branch; where it is non-zero the gradient misses the mass those paths move across
        that switch."""
        return calibrate_logsv(self, option_chain, params0, params_min, params_max, is_vega_weighted, is_unit_ttm_vega,
                               model_calibration_type, constraints_type, calibration_engine, nb_path, nb_steps, seed,
                               is_spot_measure=kwargs.get("is_spot_measure", True), disp=bool(kwargs.get("disp", False)),
                               return_info=bool(kwargs.get("return_info", False)), fd_step=kwargs.get("fd_step"),
                               mc_randoms=kwargs.get("mc_randoms", "numpy"), gradient=kwargs.get("gradient", "difference"))

    def calibrate_model_params_to_chains(self, option_chains: List[OptionChain], params0, params_min=None, params_max=None,
                                         is_vega_weighted: bool = True, is_unit_ttm_vega: bool = False,
                                         model_calibration_type: LogsvModelCalibrationType = LogsvModelCalibrationType.PARAMS5,
                                         constraints_type: ConstraintsType = ConstraintsType.UNCONSTRAINT,
                                         calibration_engine: CalibrationEngine = CalibrationEngine.ANALYTIC, return_exceptions: bool = False,
                                         max_sets_per_call: Optional[int] = None, **kwargs):
        """``calibrate_model_params_to_chain`` on every chain of ``option_chains`` (a series of daily chains, say), the fits run in
        lock-step: each optimizer round prices the pending points of every fit in one ``engine.logsv_price_chains_batch`` call, and every
        fit equals, bit for bit, the single-chain driver's on its chain (DESIGN.md §4.9).  ``params0`` / ``params_min`` / ``params_max``:
        one LogSvParams for all chains or a list of one per chain.  ANALYTIC engine, ``gradient='difference'``; PARAMS4, PARAMS5 and
        PARAMS_WITH_VARSWAP_FIT.  ``max_sets_per_call`` caps the parameter sets of one library call (a round then takes several; a fit's
        n + 1 sets always share one); without it a round is one call of about (n + 1) K sets, ~320 kB of ODE state per set on a
        four-maturity chain, so pass it for long series.  Every chain gets a thread.  Not faster than fitting the chains one after the
        other on the H100 measured so far: the Python optimizer work dominates (DESIGN.md §4.9).  Returns the list of fits, with ``return_info=True`` also the list of info dicts, each with
        ``rounds``, the library calls of the whole run.  A fit that fails raises its error after all fits have ended (the lowest chain
        index first), or with ``return_exceptions=True`` takes the exception's place in the list (its info is None)."""
        from .calibration import calibrate_logsv_chains
        return calibrate_logsv_chains(self, option_chains, params0, params_min, params_max, is_vega_weighted, is_unit_ttm_vega,
                                      model_calibration_type, constraints_type, calibration_engine,
                                      is_spot_measure=kwargs.get("is_spot_measure", True), disp=bool(kwargs.get("disp", False)),
                                      return_info=bool(kwargs.get("return_info", False)), fd_step=kwargs.get("fd_step"),
                                      gradient=kwargs.get("gradient", "difference"), return_exceptions=return_exceptions,
                                      max_sets_per_call=max_sets_per_call)

    @timer
    def model_mc_price_chain(self, option_chain: OptionChain, params: LogSvParams, is_spot_measure: bool = True,
                             variable_type: VariableType = VariableType.LOG_RETURN, nb_path: int = 100000,
                             nb_steps: Optional[int] = None, **kwargs) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """MC prices and standard errors, one array per maturity.  ``nb_steps`` is a PER-YEAR rate whose default is
        ``int(360*max(ttms)) + 1`` (reference quirk, logsv_pricer.py:427)."""
        if kwargs.get("use_rough_mc"):          # reference :395-411 (needs `seed`; `nb_steps` is passed through as given)
            assert "seed" in kwargs
            gauss = kwargs.get("gauss")        # None: the reference's host-drawn RandomState normals; 'fp32' / 'fp64': in-kernel Philox
            if gauss is None:
                Z0, Z1, grid_ttms = get_randoms_for_rough_vol_chain_valuation(ttms=option_chain.ttms, nb_path=nb_path, nb_steps_per_year=nb_steps,
                                                                              seed=kwargs["seed"])
            else:
                Z0 = Z1 = None
                grid_ttms = [set_time_grid(ttm, nb_steps)[2] for ttm in option_chain.ttms]
            return rough_logsv_mc_chain_pricer_fixed_randoms(ttms=option_chain.ttms, forwards=option_chain.forwards,
                                                             discfactors=option_chain.discfactors, strikes_ttms=option_chain.strikes_ttms,
                                                             optiontypes_ttms=option_chain.optiontypes_ttms, Z0=Z0, Z1=Z1, sigma0=params.sigma0,
                                                             theta=params.theta, kappa1=params.kappa1, kappa2=params.kappa2, beta=params.beta,
                                                             orthog_vol=params.volvol, weights=params.weights, nodes=params.nodes,
                                                             timegrids=grid_ttms, variable_type=variable_type, nb_path=nb_path,
                                                             seed=kwargs["seed"], gauss=gauss or "fp32",
                                                             distributed=kwargs.get("distributed", True), exchange=kwargs.get("exchange"))
        vol_backbone_etas = params.get_vol_backbone_etas(ttms=option_chain.ttms)
        return logsv_mc_chain_pricer(v0=params.sigma0, theta=params.theta, kappa1=params.kappa1, kappa2=params.kappa2,
                                     beta=params.beta, volvol=params.volvol, vol_backbone_etas=vol_backbone_etas,
                                     ttms=option_chain.ttms, forwards=option_chain.forwards, discfactors=option_chain.discfactors,
                                     strikes_ttms=option_chain.strikes_ttms, optiontypes_ttms=option_chain.optiontypes_ttms,
                                     is_spot_measure=is_spot_measure, variable_type=variable_type, nb_path=nb_path,
                                     nb_steps_per_year=nb_steps or int(360 * np.max(option_chain.ttms)) + 1,
                                     seed=kwargs.get("seed"), precision=kwargs.get("precision", "fp64"),
                                     gauss=kwargs.get("gauss", "fp32"), distributed=kwargs.get("distributed", True),
                                     exchange=kwargs.get("exchange"))

    @timer
    def model_mc_chain_greeks(self, option_chain: OptionChain, params: LogSvParams, is_spot_measure: bool = True,
                              variable_type: VariableType = VariableType.LOG_RETURN, nb_path: int = 100000,
                              nb_steps: Optional[int] = None, with_gamma: bool = False, with_theta: bool = False, **kwargs):
        """MC prices and standard errors as ``model_mc_price_chain`` (same defaults, ``seed`` / ``gauss`` kwargs, same numbers on the same
        seed) plus pathwise sensitivities in the same pass: the forward delta and d price / d (sigma0, theta, kappa1, kappa2, beta, volvol),
        each with its standard error -> ``McChainGreeks``.  ``kappa2`` is the value after ``__post_init__`` and is held fixed when kappa1 or
        theta moves; the vol backbone and discount factors are not differentiated.  fp64 state only; no ``exchange``; the rough-vol route has its own ``rough_mc_chain_greeks``.
        ``with_gamma=True`` also fills ``gamma`` / ``gamma_se`` (d^2 price / d forward^2 by conditional smoothing of the last step,
        DESIGN.md §3.9) and leaves every other number unchanged.
        ``with_theta=True`` also fills ``theta`` / ``theta_se`` (-d price / d ttm per year, pathwise in each slice's step length with the
        step count, forward, discount factor and vol backbone held, DESIGN.md §3.12), alone or with ``with_gamma``, and leaves every other
        number unchanged.
        Under torch.distributed every rank prices all paths (replicated, bit-identical results)."""
        from .mc_greeks import check_greeks_kwargs, to_mc_chain_greeks
        check_greeks_kwargs(kwargs)
        vt = engine.variable_code(variable_type)
        flags = engine.mc_flags("fp64", kwargs.get("gauss", "fp32"))
        args = (_params_c(params), option_chain.ttms, option_chain.forwards, option_chain.discfactors,
                params.get_vol_backbone_etas(ttms=option_chain.ttms), option_chain.strikes_ttms, option_chain.optiontypes_ttms, nb_path,
                nb_steps or int(360 * np.max(option_chain.ttms)) + 1, is_spot_measure, vt, _shared_seed(kwargs.get("seed")), flags)
        if with_theta:
            res = engine.logsv_mc_chain_greeks_theta(*args, with_gamma=with_gamma)
        else:
            res = (engine.logsv_mc_chain_greeks_gamma if with_gamma else engine.logsv_mc_chain_greeks)(*args)
        return to_mc_chain_greeks(res, engine.LOGSV_GREEK_PARAMS)

    @timer
    def rough_mc_chain_greeks(self, option_chain: OptionChain, params: LogSvParams, nb_path: int = 100000, nb_steps: Optional[int] = None,
                              variable_type: VariableType = VariableType.LOG_RETURN, with_theta: bool = False, **kwargs):
        """pathwise sensitivities of the rough-vol route (DESIGN.md §3.10): prices and "std errors" equal to
        ``model_mc_price_chain(use_rough_mc=True)`` with the same arguments (``seed`` required; ``gauss=None`` the RandomState normals of
        get_randoms_for_rough_vol_chain_valuation, 'fp32' / 'fp64' in-kernel Philox; ``nb_steps`` passed through as given), plus the forward
        delta and d price / d (sigma0, theta, kappa1, kappa2, beta, volvol) with standard errors -> ``McChainGreeks``.  ``volvol`` is the
        orthogonal vol-of-vol, as on the price route; ``params.weights`` / ``params.nodes`` are inputs, not differentiated.  ``reset_paths``
        counts, per maturity, the paths that hit the reset-to-1e-6 branch (their mass across it is not in the rows).  fp64 only, no
        ``exchange``; under torch.distributed every rank prices all paths (replicated, bit-identical results).
        ``with_theta=True`` also fills ``theta`` / ``theta_se``: -d price / d ttm per year, pathwise in each maturity's step length with its
        step count held (every maturity restarts at t = 0 on its own grid, DESIGN.md §3.12); ``reset_paths`` describes the theta row too."""
        from .mc_greeks import check_no_gamma, check_rough_greeks_kwargs, to_mc_chain_greeks
        check_no_gamma(kwargs, "rough_mc_chain_greeks")
        check_rough_greeks_kwargs(kwargs)
        vt = engine.variable_code(variable_type)
        gauss, seed = kwargs.get("gauss"), int(kwargs["seed"])
        if gauss is None:
            Z0, Z1, grids = get_randoms_for_rough_vol_chain_valuation(ttms=option_chain.ttms, nb_path=nb_path, nb_steps_per_year=nb_steps, seed=seed)
        else:
            Z0 = Z1 = None
            grids = [set_time_grid(ttm, nb_steps)[2] for ttm in option_chain.ttms]
        weights, nodes = np.asarray(params.weights, dtype=np.float64), np.asarray(params.nodes, dtype=np.float64)
        res = engine.rough_logsv_mc_chain_greeks(engine.logsv_params_c(params.sigma0, params.theta, params.kappa1, params.kappa2, params.beta,
                                                                       params.volvol), weights, nodes, option_chain.ttms, option_chain.forwards,
                                                 option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms, nb_path,
                                                 [g.size - 1 for g in grids], [float(g[1] - g[0]) for g in grids], Z0, Z1, vt, seed,
                                                 engine.mc_flags("fp64", gauss or "fp32"), with_theta=with_theta)
        out = to_mc_chain_greeks(res[:5], engine.LOGSV_GREEK_PARAMS)
        out.reset_paths = res[7]
        if with_theta:
            out.theta, out.theta_se = C.split_chain(res[8], res[4]), C.split_chain(res[9], res[4])
        return out

    @timer
    def simulate_vol_paths(self, params: LogSvParams, brownians: np.ndarray = None, ttm: float = 1.0, nb_path: int = 100000,
                           is_spot_measure: bool = True, nb_steps: int = None, year_days: int = 360, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """volatility paths on the time grid, ``(sigma_t [nb_steps+1, nb_path], grid_t)`` (reference :561-587): note the reference
        passes ``nb_steps or ceil(year_days*ttm)`` as the PER-YEAR rate of ``set_time_grid`` -- reproduced."""
        nb_steps = nb_steps or int(np.ceil(year_days * ttm))
        return simulate_vol_paths(ttm=ttm, v0=params.sigma0, theta=params.theta, kappa1=params.kappa1, kappa2=params.kappa2,
                                  beta=params.beta, volvol=params.volvol, nb_path=nb_path, is_spot_measure=is_spot_measure,
                                  nb_steps_per_year=nb_steps, brownians=brownians, seed=kwargs.get("seed"))

    @timer
    def simulate_terminal_values(self, params: LogSvParams, ttm: float = 1.0, nb_path: int = 100000, is_spot_measure: bool = True,
                                 **kwargs) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """terminal (log-return, vol, quadratic variance), float64[nb_path] each; 360 steps/year and eta = 1 as in the
        reference (:600-610).  Under an initialised ``torch.distributed`` world (one process per GPU) every rank simulates and returns ITS
        contiguous shard of the ``nb_path`` global path ids (SURVEY.md 8e: no collective; concatenating the shards in rank order gives the
        single-GPU arrays); ``path_range=(offset, n_local)`` selects a shard explicitly, ``distributed=False`` switches sharding off."""
        path_range = kwargs.get("path_range")
        if path_range is None and _use_distributed(kwargs):
            import torch.distributed as dist
            n_local, offset = shard_paths(nb_path, dist.get_world_size(), dist.get_rank())
            path_range = (offset, n_local)
        if path_range is not None:
            return _terminal_values_shard(params, ttm, int(path_range[0]), int(path_range[1]), is_spot_measure,
                                          kwargs.get("nb_steps_per_year", 360), kwargs.get("seed"), kwargs.get("gauss", "fp32"))
        return simulate_logsv_x_vol_terminal(ttm=ttm, x0=np.zeros(1), sigma0=params.sigma0 * np.ones(1), qvar0=np.zeros(1),
                                             theta=params.theta, kappa1=params.kappa1, kappa2=params.kappa2, beta=params.beta,
                                             volvol=params.volvol, nb_path=nb_path, is_spot_measure=is_spot_measure,
                                             nb_steps_per_year=kwargs.get("nb_steps_per_year", 360), seed=kwargs.get("seed"),
                                             gauss=kwargs.get("gauss", "fp32"))

    def logsv_pdfs(self, params: LogSvParams, ttm: float, space_grid: np.ndarray, **kwargs) -> np.ndarray:
        """model density of log-return / quadratic variance / volatility on ``space_grid`` (reference :613-637)."""
        return logsv_pdfs(params=params, ttm=ttm, space_grid=space_grid, **kwargs)


def set_vol_scaler(sigma0: float, ttm: float) -> float:
    """transform-grid scaler sigma0*sqrt(min(min ttm, 0.5/12)) (logsv_pricer.py:664-666)."""
    return sigma0 * np.sqrt(np.minimum(np.min(ttm), 0.5 / 12.0))


def logsv_chain_pricer(params: LogSvParams, ttms: np.ndarray, forwards: np.ndarray, discfactors: np.ndarray,
                       strikes_ttms: List[np.ndarray], optiontypes_ttms: List[np.ndarray], is_stiff_solver: bool = False,
                       is_analytic: bool = False, is_spot_measure: bool = True,
                       expansion_order: ExpansionOrder = ExpansionOrder.SECOND,
                       variable_type: VariableType = VariableType.LOG_RETURN, vol_scaler: float = None, **kwargs) -> List[np.ndarray]:
    """Fourier chain pricer (reference :669-739): one fused GPU call for the whole chain -- transform grid, RK45 ODE solves of the
    affine expansion carried across maturities, log-MGF, Simpson sums.  ``return_grids=True`` additionally returns
    (a_t1 [M,P,n], log_mgf [M,P])."""
    vt = getattr(variable_type, "value", variable_type)
    if vt not in (1, 2):
        raise NotImplementedError       # SIGMA: the reference raises too (:733-734)
    order = _order_code(expansion_order)
    if is_analytic or is_stiff_solver:
        return _logsv_chain_pricer_branch(params, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_spot_measure, expansion_order,
                                          variable_type, vol_scaler, bool(kwargs.get("return_grids", False)), is_analytic, is_stiff_solver)
    etas = np.array([params.get_vol_backbone_eta(tau=ttm) for ttm in ttms], dtype=float)
    return engine.logsv_price_chain(_params_c(params), ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                                    is_spot_measure=is_spot_measure, expansion_order=order, vol_scaler=vol_scaler,
                                    max_phi=kwargs.get("max_phi"), return_grids=bool(kwargs.get("return_grids", False)), variable_type=vt)


def _logsv_chain_pricer_branch(params, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_spot_measure, expansion_order, variable_type,
                               vol_scaler, return_grids, is_analytic, is_stiff_solver):
    """the chain loop of the reference (:699-737) on its two non-default ODE branches (``is_analytic=True``: semi-analytic scheme;
    ``is_stiff_solver=True``: SciPy's BDF control law): per maturity one grid solve carried on ``a_t0`` and one Fourier sum, both on the
    GPU.  Not fused into a single call like the default RK45 branch."""
    from ..utils import mgf_pricer as mgfp
    from .logsv.affine_expansion import compute_logsv_a_mgf_grid, get_expansion_n
    if vol_scaler is None:
        vol_scaler = set_vol_scaler(sigma0=params.sigma0, ttm=np.min(ttms))
    phi_grid, psi_grid, theta_grid = mgfp.get_transform_var_grid(variable_type=variable_type, is_spot_measure=is_spot_measure, vol_scaler=vol_scaler)
    a_t0 = np.zeros((phi_grid.shape[0], get_expansion_n(expansion_order)), dtype=np.complex128)
    ttm0, prices, grids = 0.0, [], []
    vt = getattr(variable_type, "value", variable_type)
    for ttm, forward, strikes, types, discfactor in zip(ttms, forwards, strikes_ttms, optiontypes_ttms, discfactors):
        a_t0, log_mgf = compute_logsv_a_mgf_grid(ttm=ttm - ttm0, phi_grid=phi_grid, psi_grid=psi_grid, theta_grid=theta_grid, a_t0=a_t0,
                                                 is_analytic=is_analytic, is_stiff_solver=is_stiff_solver, expansion_order=expansion_order,
                                                 is_spot_measure=is_spot_measure, sigma0=params.sigma0, theta=params.theta, kappa1=params.kappa1,
                                                 kappa2=params.kappa2, beta=params.beta, volvol=params.volvol, variable_type=variable_type,
                                                 vol_backbone_eta=params.get_vol_backbone_eta(tau=ttm))
        if vt == 1:
            prices.append(mgfp.vanilla_slice_pricer_with_mgf_grid(log_mgf_grid=log_mgf, phi_grid=phi_grid, forward=forward, strikes=strikes,
                                                                  optiontypes=types, discfactor=discfactor, is_spot_measure=is_spot_measure))
        else:
            prices.append(mgfp.slice_qvar_pricer_with_a_grid(log_mgf_grid=log_mgf, psi_grid=psi_grid, ttm=ttm, forward=forward, strikes=strikes,
                                                             optiontypes=types, discfactor=discfactor, is_spot_measure=is_spot_measure))
        if not np.all(np.isfinite(log_mgf)):
            # the branch's unchecked fixed-point sweeps have diverged on part of the grid (the reference: quickstart / BTC parameters at
            # SECOND order).  The reference's Fourier sum is an njit(fastmath=True) nansum, which does not skip the NaNs it is fed and
            # returns NaN for every strike; a NaN-skipping sum over the surviving grid points would be a finite but meaningless number.
            prices[-1] = np.full(np.asarray(strikes).shape, np.nan)
        grids.append((a_t0, log_mgf))
        ttm0 = ttm
    return (prices, grids) if return_grids else prices


def logsv_pdfs(params: LogSvParams, ttm: float, space_grid: np.ndarray, is_stiff_solver: bool = False, is_analytic: bool = False,
               is_spot_measure: bool = True, expansion_order: ExpansionOrder = ExpansionOrder.SECOND,
               variable_type: VariableType = VariableType.LOG_RETURN, vol_scaler: float = None) -> np.ndarray:
    """model density of the log-return, the quadratic variance or the volatility on ``space_grid`` (reference :742-803): ODE grid
    solve on the GPU from the variable's initial condition, then the Fourier density sums on the GPU."""
    from ..utils import mgf_pricer as mgfp
    from .logsv.affine_expansion import compute_logsv_a_mgf_grid
    if vol_scaler is None:
        vol_scaler = set_vol_scaler(sigma0=params.sigma0, ttm=ttm)
    phi_grid, psi_grid, theta_grid = mgfp.get_transform_var_grid(variable_type=variable_type, is_spot_measure=is_spot_measure,
                                                                 vol_scaler=vol_scaler)
    _, log_mgf_grid = compute_logsv_a_mgf_grid(ttm=ttm, phi_grid=phi_grid, psi_grid=psi_grid, theta_grid=theta_grid, sigma0=params.sigma0,
                                               theta=params.theta, kappa1=params.kappa1, kappa2=params.kappa2, beta=params.beta,
                                               volvol=params.volvol, variable_type=variable_type, expansion_order=expansion_order,
                                               is_stiff_solver=is_stiff_solver, is_analytic=is_analytic, is_spot_measure=is_spot_measure)
    vt = getattr(variable_type, "value", variable_type)
    if vt == 1:
        grid, shift, scale = phi_grid, 0.0, 1.0
    elif vt == 2:
        grid, shift, scale = psi_grid, 0.0, 1.0 / ttm          # scaled by ttm (:785-788)
    elif vt == 3:
        grid, shift, scale = theta_grid, params.theta, 1.0
    else:
        raise NotImplementedError
    return mgfp.pdf_with_mgf_grid(log_mgf_grid=log_mgf_grid, transform_var_grid=grid, space_grid=space_grid, shift=shift, scale=scale) / scale


def logsv_mc_chain_pricer(ttms: np.ndarray, forwards: np.ndarray, discfactors: np.ndarray, strikes_ttms, optiontypes_ttms,
                          v0: float, theta: float, kappa1: float, kappa2: float, beta: float, volvol: float,
                          vol_backbone_etas: np.ndarray, is_spot_measure: bool = True, nb_path: int = 100000,
                          nb_steps_per_year: int = 360, variable_type: VariableType = VariableType.LOG_RETURN,
                          seed: Optional[int] = None, precision: str = "fp64", gauss: str = "fp32", distributed: bool = True,
                          exchange: Optional[str] = None) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """chain MC (reference :806-867): every maturity is simulated from the terminal state of the previous one by the fused
    stepper, followed by forward-recentred payoff moments.  Under an initialised torch.distributed world ``nb_path`` is the
    TOTAL path count, sharded over the ranks (two fp64 all-reduces per maturity)."""
    params_c = engine.logsv_params_c(v0, theta, kappa1, kappa2, beta, volvol)
    flags = engine.mc_flags(precision, gauss)
    seed = _shared_seed(seed)
    if _use_distributed({"distributed": distributed, "nb_path": nb_path, "exchange": exchange}):
        return mc_chain_distributed("logsv", params_c, ttms, forwards, discfactors, vol_backbone_etas, strikes_ttms,
                                    optiontypes_ttms, nb_path, nb_steps_per_year, is_spot_measure,
                                    engine.variable_code(variable_type), seed, flags, exchange=exchange)
    return engine.logsv_mc_chain(params_c, ttms, forwards, discfactors, vol_backbone_etas, strikes_ttms, optiontypes_ttms, nb_path,
                                 nb_steps_per_year, is_spot_measure, variable_type, seed, flags)


def simulate_vol_paths(ttm: float, v0: float, theta: float, kappa1: float, kappa2: float, beta: float, volvol: float,
                       is_spot_measure: bool = True, nb_path: int = 100000, nb_steps_per_year: int = 360, brownians: np.ndarray = None,
                       seed: Optional[int] = None, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
    """full volatility paths (reference :870-947) on the GPU; ``brownians`` = pre-drawn SCALED increments [nb_steps, nb_path]."""
    seed = engine.fresh_seed() if seed is None else int(seed)
    return engine.logsv_vol_paths(engine.logsv_params_c(v0, theta, kappa1, kappa2, beta, volvol), ttm, nb_path, nb_steps_per_year,
                                  is_spot_measure, seed, brownians)


def _terminal_values_shard(params, ttm, offset, n_local, is_spot_measure, nb_steps_per_year, seed, gauss):
    """paths [offset, offset + n_local) of the global Philox stream on the current CUDA device (device-level slice call, state copied back)"""
    if seed is None:
        raise ValueError("a sharded simulation needs an explicit seed (every rank must draw from the same stream)")
    if n_local == 0:
        return np.zeros(0), np.zeros(0), np.zeros(0)
    eng = CudaMcEngine("logsv", _params_c(params), n_local, offset, engine.mc_flags("fp64", gauss), 1)
    nb_steps, dt, _ = set_time_grid(ttm, nb_steps_per_year)
    eng.simulate_slice(0, True, nb_steps, dt, 1.0, is_spot_measure, 1.0, int(seed))
    host = eng.state.cpu().numpy()
    return host[0].copy(), host[1].copy(), host[2].copy()


def simulate_logsv_x_vol_terminal(ttm: float, x0: np.ndarray, sigma0: np.ndarray, qvar0: np.ndarray, theta: float, kappa1: float,
                                  kappa2: float, beta: float, volvol: float, vol_backbone_eta: float = 1.0,
                                  is_spot_measure: bool = True, nb_path: int = 100000, nb_steps_per_year: int = 360,
                                  W0: Optional[np.ndarray] = None, W1: Optional[np.ndarray] = None, dt: Optional[float] = None,
                                  seed: Optional[int] = None, gauss: str = "fp32", slice_index: int = 0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """terminal (x, sigma, qvar) after ``ttm`` (reference :950-1047).

    With ``W0, W1, dt`` (unit normals [nb_steps, nb_path]) the strict fixed-random kernel reproduces the reference arithmetic
    (fp64, reference evaluation order, no FMA contraction).  Without them the fused Philox kernel draws the normals; the initial state is
    either the length-1 broadcast form or per-path arrays of length ``nb_path``, as in the reference (:1007-1020).  ``slice_index`` (extra)
    selects the Philox sub-stream so that a chain of calls on one seed does not reuse normals."""
    if W0 is not None or W1 is not None:
        if W0 is None or W1 is None or dt is None:
            raise ValueError("W0, W1 and dt must be supplied together")
        params_c = engine.logsv_params_c(1.0, theta, kappa1, kappa2, beta, volvol)
        return engine.logsv_step_fixed(x0, sigma0, qvar0, W0, W1, dt, params_c, vol_backbone_eta, is_spot_measure)
    x0, sigma0, qvar0 = np.atleast_1d(x0), np.atleast_1d(sigma0), np.atleast_1d(qvar0)
    for a in (x0, sigma0, qvar0):
        assert a.shape[0] in (1, nb_path)            # :1007-1020
    seed = engine.fresh_seed() if seed is None else int(seed)
    flags = engine.mc_flags("fp64", gauss)
    x_bcast = x0.shape[0] == 1 or not np.any(x0)         # a length-1 x0 / qvar0 is replaced by zeros in the reference (:1007-1015)
    q_bcast = qvar0.shape[0] == 1 or not np.any(qvar0)
    if x_bcast and q_bcast and np.all(sigma0 == sigma0[0]):
        # the form the reference's own callers use: every path starts from (0, sigma0, 0) -- no state upload
        params_c = engine.logsv_params_c(float(sigma0[0]), theta, kappa1, kappa2, beta, volvol)
        return engine.logsv_terminal(params_c, ttm, nb_path, nb_steps_per_year, is_spot_measure, vol_backbone_eta, seed, flags)
    # per-path initial state (:1007-1020): length-1 inputs broadcast as the reference does (x0 -> zeros, qvar0 -> zeros, sigma0 -> constant)
    xs = np.zeros(nb_path) if x0.shape[0] == 1 else x0
    qs = np.zeros(nb_path) if qvar0.shape[0] == 1 else qvar0
    ss = sigma0 * np.ones(nb_path) if sigma0.shape[0] == 1 else sigma0
    params_c = engine.logsv_params_c(float(ss[0]), theta, kappa1, kappa2, beta, volvol)
    return engine.logsv_terminal_from_state(params_c, xs, ss, qs, ttm, nb_steps_per_year, is_spot_measure, vol_backbone_eta, seed, flags, slice_index)


class DeviceRandoms:
    """Fixed unit normals of a chain kept RESIDENT in HBM (float64 CUDA tensors W0s[m], W1s[m] of shape [S_m, nb_path]) so that the
    calibration inner loop (reference :235-294 -> :1100-1162) re-prices with new parameters without re-uploading 16 B per path-step.
    torch is used for device memory only."""

    def __init__(self, W0s, W1s, dts, device=None):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("DeviceRandoms needs a CUDA device; stochvolmodels_b200 has no CPU fallback")
        self.device = torch.device(f"cuda:{torch.cuda.current_device()}" if device is None or device is True else device)
        up = lambda w: w.to(self.device, torch.float64).contiguous() if torch.is_tensor(w) else torch.as_tensor(np.ascontiguousarray(w, dtype=np.float64)).to(self.device)
        self.W0s, self.W1s, self.dts = [up(w) for w in W0s], [up(w) for w in W1s], [float(d) for d in dts]
        self.nb_path = int(self.W0s[0].shape[1])
        for a, b in zip(self.W0s, self.W1s):
            if a.shape != b.shape or a.shape[1] != self.nb_path:
                raise ValueError("W0s and W1s must be lists of [nb_steps, nb_path] arrays of equal shapes")

    def nbytes(self) -> int:
        return sum(w.numel() * 8 for w in self.W0s + self.W1s)


def get_randoms_for_chain_valuation(ttms: np.ndarray, nb_path: int = 100000, nb_steps_per_year: int = 360, seed: int = 10,
                                    device=None):
    """fixed unit normals per maturity from a LOCAL legacy generator: per slice W0 then W1, never touching numpy's global state
    (reference :1051-1074).  ``device="cuda"`` returns the same numbers as a :class:`DeviceRandoms` resident in HBM."""
    rng = np.random.RandomState(seed)
    W0s, W1s, dts = [], [], []
    ttm0 = 0.0
    for ttm in ttms:
        nb_steps_, dt, _ = set_time_grid(ttm=ttm - ttm0, nb_steps_per_year=nb_steps_per_year)
        W0s.append(rng.normal(0, 1, size=(nb_steps_, nb_path)))
        W1s.append(rng.normal(0, 1, size=(nb_steps_, nb_path)))
        dts.append(dt)
        ttm0 = ttm
    if device is not None:
        return DeviceRandoms(W0s, W1s, dts, device)
    return W0s, W1s, dts


def get_randoms_for_rough_vol_chain_valuation(ttms: np.ndarray, nb_path: int = 100000, nb_steps_per_year: int = 360, seed: int = 10):
    """(Z0, Z1, per-maturity time grids) of the rough-vol chain valuation (reference :1076-1097): one block of unit normals of the LAST
    maturity's length from a local ``RandomState(seed)`` -- Z0 then Z1 -- whose first S_m rows every maturity m consumes."""
    rng = np.random.RandomState(seed)
    grid_ttms, nb_steps = [], 0
    for ttm in ttms:
        nb_steps, _, grid_t = set_time_grid(ttm, nb_steps_per_year)
        grid_ttms.append(grid_t)
    Z0 = rng.normal(0, 1, size=(nb_steps, nb_path))
    Z1 = rng.normal(0, 1, size=(nb_steps, nb_path))
    return Z0, Z1, grid_ttms


def rough_logsv_mc_chain_pricer_fixed_randoms(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, Z0, Z1, sigma0: float, theta: float,
                                              kappa1: float, kappa2: float, beta: float, orthog_vol: float, weights: np.ndarray, nodes: np.ndarray,
                                              timegrids: List[np.ndarray], variable_type: VariableType = VariableType.LOG_RETURN,
                                              debug: bool = False, nb_path: Optional[int] = None, seed: Optional[int] = None, gauss: str = "fp32",
                                              return_states: bool = False, distributed: bool = True, exchange: Optional[str] = None):
    """rough-LogSV chain prices by the multi-factor Strang-splitting scheme with caller-supplied normals (reference :1164-1232 ->
    rough_logsv/split_simulation.py:466): every maturity restarts at t = 0 on ITS grid and uses the first rows of ``Z0`` / ``Z1``.
    Returned "standard errors" are, as in the reference on this route, discfactor * nanstd(payoff) without the 1/sqrt(nb_path).
    ``Z0 = Z1 = None`` (extra): the normals are drawn in-kernel (Philox stream keyed by ``seed``; ``nb_path`` required); in that mode, under
    an initialised torch.distributed world, ``nb_path`` is the TOTAL path count sharded over the ranks by global path id (multi_gpu.py).
    Caller-supplied normals are not sharded: every rank prices all of them."""
    weights, nodes = np.asarray(weights, dtype=np.float64), np.asarray(nodes, dtype=np.float64)
    assert weights.shape == nodes.shape and weights.ndim == 1            # :1188
    if Z0 is not None:
        nb_path = Z0.shape[1]
    elif nb_path is None:
        raise ValueError("nb_path is required when the normals are drawn in-kernel")
    nsteps = [int(np.asarray(g).size) - 1 for g in timegrids]
    hs = [float(np.asarray(g)[1] - np.asarray(g)[0]) for g in timegrids]             # split_simulation.py:346
    params_c = engine.logsv_params_c(sigma0, theta, kappa1, kappa2, beta, orthog_vol)
    if Z0 is None and not (return_states or debug) and _use_distributed({"distributed": distributed, "nb_path": nb_path, "exchange": exchange}):
        return mc_chain_distributed("rough", params_c, ttms, forwards, discfactors, None, strikes_ttms, optiontypes_ttms, nb_path, 0, True,
                                    engine.variable_code(variable_type), _shared_seed(seed),
                                    engine.mc_flags("fp64", gauss), exchange=exchange, grid=list(zip(nsteps, hs)), factors=(weights, nodes),
                                    se_paths=1)
    prices, stds, _, states, offsets = engine.rough_logsv_mc_chain([params_c], weights, nodes, ttms, forwards, discfactors, strikes_ttms,
                                                                   optiontypes_ttms, nb_path, nsteps, hs, Z0, Z1, variable_type,
                                                                   engine.fresh_seed() if seed is None else int(seed),
                                                                   engine.mc_flags("fp64", gauss), return_states=return_states or debug)
    if debug:            # the reference's per-slice diagnostics (:1218-1220)
        for m in range(len(nsteps)):
            vol = weights @ states[m, 1:-1]
            print(f"Number of paths with negative vol: {np.sum(vol < 0.0)}, nan vol: {np.count_nonzero(np.isnan(vol))}")
            print(f"Mean spot Strand: {np.mean(np.exp(states[m, 0]))}, nan spots: {np.count_nonzero(np.isnan(states[m, 0]))}")
    out = (C.split_chain(prices[0], offsets), C.split_chain(stds[0], offsets))
    return out + (states,) if return_states else out


def logsv_mc_chain_pricer_fixed_randoms(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, W0s, W1s=None, dts=None,
                                        v0: float = None, theta: float = None, kappa1: float = None, kappa2: float = None,
                                        beta: float = None, volvol: float = None, vol_backbone_etas: np.ndarray = None,
                                        is_spot_measure: bool = True, variable_type: VariableType = VariableType.LOG_RETURN,
                                        return_states: bool = False, fast: bool = True):
    """chain valuation with caller-supplied unit normals (reference :1100-1162).  Host arrays go through the strict-arithmetic
    stepper (reference evaluation order).  ``W0s`` may be a :class:`DeviceRandoms` (then ``W1s`` / ``dts`` are taken from it, nothing
    is uploaded, and ``fast`` selects the throughput stepper, which agrees with the strict one to ~1e-14)."""
    params_c = engine.logsv_params_c(v0, theta, kappa1, kappa2, beta, volvol)
    if vol_backbone_etas is None:
        vol_backbone_etas = np.ones(len(ttms))
    if isinstance(W0s, DeviceRandoms):
        if return_states:
            raise NotImplementedError("return_states is only available with host arrays")
        return _fixed_randoms_chain_device(W0s, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, params_c, vol_backbone_etas,
                                           is_spot_measure, variable_type, fast)
    nb_path = W0s[0].shape[1]
    x, q, s = np.zeros(nb_path), np.zeros(nb_path), v0 * np.ones(nb_path)
    prices, stds, states = [], [], []
    for ttm, forward, discfactor, strikes, types, eta, W0, W1, dt in zip(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                                                                         vol_backbone_etas, W0s, W1s, dts):
        x, s, q = engine.logsv_step_fixed(x, s, q, W0, W1, dt, params_c, eta, is_spot_measure)
        p, e = engine.mc_payoffs(x, q, ttm, forward, strikes, types, discfactor, variable_type)
        prices.append(p)
        stds.append(e)
        if return_states:
            states.append((x.copy(), s.copy(), q.copy()))
    return (prices, stds, states) if return_states else (prices, stds)


def logsv_mc_chain_greeks_fixed_randoms(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, W0s, W1s=None, dts=None,
                                        v0: float = None, theta: float = None, kappa1: float = None, kappa2: float = None,
                                        beta: float = None, volvol: float = None, vol_backbone_etas: np.ndarray = None,
                                        is_spot_measure: bool = True, variable_type: VariableType = VariableType.LOG_RETURN):
    """``logsv_mc_chain_pricer_fixed_randoms`` plus pathwise sensitivities in the same pass (DESIGN.md §4.7) -> ``McChainGreeks``: the forward
    delta and d price / d (sigma0, theta, kappa1, kappa2, beta, volvol) with standard errors.  ``kappa2`` is held fixed when kappa1 or
    theta moves; the vol backbone and the discount factors are not differentiated.  On fixed normals the sensitivities are the exact
    derivatives of the sample prices, the limit a common-random-number difference approximates.

    ``W0s`` may be a :class:`DeviceRandoms`, used in place; host arrays ``W0s``, ``W1s``, ``dts`` are uploaded once into one.  Prices and std
    errors are bit-identical to ``logsv_mc_chain_pricer_fixed_randoms(DeviceRandoms, fast=True)`` on the same normals; they agree with the
    strict host-array stepper only to ~1e-14."""
    from .mc_greeks import to_mc_chain_greeks
    params_c = engine.logsv_params_c(v0, theta, kappa1, kappa2, beta, volvol)
    if vol_backbone_etas is None:
        vol_backbone_etas = np.ones(len(ttms))
    rnd = W0s if isinstance(W0s, DeviceRandoms) else DeviceRandoms(W0s, W1s, dts)
    res = _fixed_randoms_chain_greeks_device(rnd, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, params_c, vol_backbone_etas,
                                             is_spot_measure, variable_type)
    return to_mc_chain_greeks(res, engine.LOGSV_GREEK_PARAMS)


def v0_implied(atm: float, beta: float, volvol: float, theta: float, kappa1: float, ttm: float) -> float:
    """short-maturity approximation of the initial volatility sigma0 from an ATM vol (reference logsv_pricer.py:638-661; host scalar helper).
    Regular expansion ``atm - vartheta^2 ttm / 4`` when |beta| > 1 or beta ~ 0; otherwise the positive root of the quadratic in sigma0 the
    reference solves."""
    b2, vartheta2 = beta * beta, beta * beta + volvol * volvol
    regular = atm - vartheta2 * ttm / 4.0
    lead = 12.0 * beta * ttm
    if abs(beta) > 1.0 or abs(lead) <= 1e-10:
        return regular
    half_b = 24.0 + b2 * ttm + 2.0 * vartheta2 * ttm - 12.0 * kappa1 * ttm
    disc = half_b * half_b - 288.0 * beta * ttm * (theta * kappa1 * ttm - 2.0 * atm)
    return (np.sqrt(disc) - half_b) / lead
