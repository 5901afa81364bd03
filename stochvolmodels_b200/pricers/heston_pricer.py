"""HestonPricer on H100: drop-in for the hot paths of the reference ``pricers/heston_pricer.py``.

* ``HestonPricer.price_chain``               (heston_pricer.py:52-66)   -> ``heston_chain_pricer`` (:217-282), closed-form MGF (:183-214)
* ``HestonPricer.model_mc_price_chain``      (:68-87)                   -> ``heston_mc_chain_pricer`` (:285-331)
* ``HestonPricer.simulate_terminal_values``  (:90-108)                  -> ``simulate_heston_x_vol_terminal`` (:334-381, floor-Euler)

The reference hard-wires 360 steps per year in the MC (:344, not forwarded at :76-87); ``nb_steps_per_year`` is an optional kwarg
here (default 360).  Calibration (:111-180) is a caller of the hot path and out of scope.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

from .. import _capi as C
from .. import engine
from ..data.option_chain import OptionChain
from ..multi_gpu import _shared_seed, _use_distributed, mc_chain_distributed
from ..utils.config import VariableType
from ..utils.funcs import timer
from .model_pricer import ModelParams, ModelPricer


@dataclass
class HestonParams(ModelParams):
    """dv = kappa (theta - v) dt + volvol sqrt(v) dW, corr(dS, dv) = rho (reference heston_pricer.py:27-41)."""
    v0: float = 0.04
    theta: float = 0.04
    kappa: float = 4.0
    rho: float = -0.5
    volvol: float = 0.4


BTC_HESTON_PARAMS = HestonParams(v0=0.8, theta=1.0, kappa=2.0, rho=0.0, volvol=2.0)


def _params_c(v0, theta, kappa, rho, volvol) -> C.HestonParamsC:
    return engine.heston_params_c(v0, theta, kappa, rho, volvol)


def _scheme_code(scheme) -> int:
    """'euler_floor' (default = the reference's scheme) | 'qe' (opt-in Andersen quadratic-exponential; not in the reference)."""
    codes = {"euler_floor": C.HESTON_EULER_FLOOR, "qe": C.HESTON_QE, C.HESTON_EULER_FLOOR: C.HESTON_EULER_FLOOR, C.HESTON_QE: C.HESTON_QE}
    if scheme not in codes:
        raise ValueError("scheme must be 'euler_floor' or 'qe'")
    return codes[scheme]


class HestonPricer(ModelPricer):
    """ModelPricer for the Heston model, Fourier + Monte Carlo routes on the GPU."""

    def price_chain(self, option_chain: OptionChain, params: HestonParams, **kwargs) -> List[np.ndarray]:
        """Fourier prices; ``variable_type`` and other unknown kwargs are accepted and ignored as in the reference (:52-66)."""
        return heston_chain_pricer(v0=params.v0, theta=params.theta, kappa=params.kappa, volvol=params.volvol, rho=params.rho,
                                   ttms=option_chain.ttms, forwards=option_chain.forwards, discfactors=option_chain.discfactors,
                                   strikes_ttms=option_chain.strikes_ttms, optiontypes_ttms=option_chain.optiontypes_ttms,
                                   vol_scaler=kwargs.get("vol_scaler"))

    def price_chain_greeks(self, option_chain: OptionChain, params: HestonParams, with_theta: bool = False, **kwargs):
        """Fourier prices (bit-identical to ``price_chain`` with the same ``vol_scaler``) plus forward-mode sensitivities in one call ->
        ``FourierChainGreeks``: delta and gamma in the slice forward and d price / d (v0, theta, kappa, rho, volvol), exact derivatives of
        the closed form on a fixed transform grid.  Q_VAR raises NotImplementedError.  ``with_theta``: also ``theta`` = -d price / d ttm per
        maturity (DESIGN.md §4.8), exact in the slice length with the earlier maturities and the grid held; every other output bit for bit."""
        from .fourier_greeks import check_fourier_greeks_kwargs, to_fourier_chain_greeks
        check_fourier_greeks_kwargs(kwargs)
        out = engine.heston_price_chain_greeks(
            _params_c(params.v0, params.theta, params.kappa, params.rho, params.volvol), option_chain.ttms, option_chain.forwards,
            option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms, vol_scaler=kwargs.get("vol_scaler"),
            **({"with_theta": True} if with_theta else {}))
        return to_fourier_chain_greeks(*out[:3], engine.HESTON_GREEK_PARAMS, *out[3:])

    def price_chain_hessian(self, option_chain: OptionChain, params: HestonParams, **kwargs):
        """``price_chain_greeks`` (bit for bit) plus vanna and the symmetric Hessian over (v0, theta, kappa, rho, volvol) in one call ->
        ``FourierChainHessian``: second derivatives of the closed form through hyper-dual numbers on a fixed transform grid.  Q_VAR
        raises NotImplementedError."""
        from .fourier_greeks import check_fourier_hessian_kwargs, to_fourier_chain_hessian
        check_fourier_hessian_kwargs(kwargs)
        prices, greeks, vanna, hessian, offsets = engine.heston_price_chain_hessian(
            _params_c(params.v0, params.theta, params.kappa, params.rho, params.volvol), option_chain.ttms, option_chain.forwards,
            option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms, vol_scaler=kwargs.get("vol_scaler"))
        return to_fourier_chain_hessian(prices, greeks, vanna, hessian, offsets, engine.HESTON_GREEK_PARAMS)

    @timer
    def calibrate_model_params_to_chain(self, option_chain: OptionChain, params0: HestonParams = None, is_vega_weighted: bool = True,
                                        is_unit_ttm_vega: bool = False, **kwargs) -> HestonParams:
        """fit (v0, theta, kappa, rho, volvol) to the chain's mid vols by SLSQP under the Feller constraint (reference :111-180); the
        objective and its gradient are one batched GPU call per evaluation (pricers/calibration.py).  ``gradient='exact'`` hands SLSQP
        the exact gradient from one ``compute_chain_ivol_greeks`` call per point, on the start point's default grid (DESIGN.md §4.6)."""
        from .calibration import calibrate_heston
        return calibrate_heston(self, option_chain, params0, is_vega_weighted, is_unit_ttm_vega, disp=bool(kwargs.get("disp", False)),
                                return_info=bool(kwargs.get("return_info", False)), fd_step=kwargs.get("fd_step"),
                                gradient=kwargs.get("gradient", "difference"))

    def calibrate_model_params_to_chains(self, option_chains: List[OptionChain], params0=None, is_vega_weighted: bool = True,
                                         is_unit_ttm_vega: bool = False, return_exceptions: bool = False,
                                         max_sets_per_call: Optional[int] = None, **kwargs):
        """``calibrate_model_params_to_chain`` on every chain of ``option_chains``, in lock-step: one ``engine.heston_price_chains_batch``
        call per optimizer round, every fit bit for bit the single-chain driver's (DESIGN.md §4.9).  ``params0``: None, one HestonParams
        or a list of one per chain; ``gradient='difference'`` only.  Return value, ``return_info``, ``return_exceptions`` and
        ``max_sets_per_call`` as LogSVPricer.calibrate_model_params_to_chains.  Slower than fitting the chains one after the other on the H100
        measured so far (DESIGN.md §4.9)."""
        from .calibration import calibrate_heston_chains
        return calibrate_heston_chains(self, option_chains, params0, is_vega_weighted, is_unit_ttm_vega, disp=bool(kwargs.get("disp", False)),
                                       return_info=bool(kwargs.get("return_info", False)), fd_step=kwargs.get("fd_step"),
                                       gradient=kwargs.get("gradient", "difference"), return_exceptions=return_exceptions,
                                       max_sets_per_call=max_sets_per_call)

    def model_mc_price_chain(self, option_chain: OptionChain, params: HestonParams, nb_path: int = 100000,
                             variable_type: VariableType = VariableType.LOG_RETURN, **kwargs) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        return heston_mc_chain_pricer(v0=params.v0, theta=params.theta, kappa=params.kappa, rho=params.rho, volvol=params.volvol,
                                      ttms=option_chain.ttms, forwards=option_chain.forwards, discfactors=option_chain.discfactors,
                                      strikes_ttms=option_chain.strikes_ttms, optiontypes_ttms=option_chain.optiontypes_ttms,
                                      nb_path=nb_path, variable_type=variable_type,
                                      nb_steps_per_year=kwargs.get("nb_steps_per_year", 360), seed=kwargs.get("seed"),
                                      precision=kwargs.get("precision", "fp64"), gauss=kwargs.get("gauss", "fp32"),
                                      distributed=kwargs.get("distributed", True), scheme=kwargs.get("scheme", "euler_floor"),
                                      exchange=kwargs.get("exchange"))

    def model_mc_chain_greeks(self, option_chain: OptionChain, params: HestonParams, nb_path: int = 100000,
                              variable_type: VariableType = VariableType.LOG_RETURN, with_gamma: bool = False, with_theta: bool = False,
                              **kwargs):
        """MC prices and standard errors as ``model_mc_price_chain`` (same defaults and kwargs, same numbers on the same seed) plus pathwise
        sensitivities in the same pass: the forward delta and d price / d (v0, theta, kappa, rho, volvol), each with its standard error ->
        ``McChainGreeks``.  ``with_gamma=True`` also fills ``gamma`` / ``gamma_se`` (DESIGN.md §3.9) and leaves every other number unchanged.
        ``with_theta=True`` also fills ``theta`` / ``theta_se`` (-d price / d ttm per year, pathwise in each slice's step length with its
        step count held, DESIGN.md §3.12), alone or with ``with_gamma``, and leaves every other number unchanged.
        Floor-Euler scheme and fp64 state only; no ``exchange``.  Under torch.distributed every rank prices all paths (replicated,
        bit-identical results)."""
        from .mc_greeks import check_greeks_kwargs, to_mc_chain_greeks
        check_greeks_kwargs(kwargs)
        if _scheme_code(kwargs.get("scheme", "euler_floor")) != C.HESTON_EULER_FLOOR:
            raise NotImplementedError("model_mc_chain_greeks needs scheme='euler_floor'")
        vt = engine.variable_code(variable_type)
        flags = engine.mc_flags("fp64", kwargs.get("gauss", "fp32"))
        args = (_params_c(params.v0, params.theta, params.kappa, params.rho, params.volvol), option_chain.ttms, option_chain.forwards,
                option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms, nb_path,
                kwargs.get("nb_steps_per_year", 360), vt, _shared_seed(kwargs.get("seed")), flags)
        if with_theta:
            res = engine.heston_mc_chain_greeks_theta(*args, with_gamma=with_gamma)
        else:
            res = (engine.heston_mc_chain_greeks_gamma if with_gamma else engine.heston_mc_chain_greeks)(*args)
        return to_mc_chain_greeks(res, engine.HESTON_GREEK_PARAMS)

    @timer
    def simulate_terminal_values(self, params: HestonParams, ttm: float = 1.0, nb_path: int = 100000, x0: float = 0.0, **kwargs
                                 ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """terminal (log-return, variance, quadratic variance); ``x0`` is ignored exactly as in the reference (:90-108)."""
        return simulate_heston_x_vol_terminal(ttm=ttm, x0=np.zeros(1), var0=params.v0 * np.ones(1), qvar0=np.zeros(1),
                                              theta=params.theta, kappa=params.kappa, rho=params.rho, volvol=params.volvol,
                                              nb_path=nb_path, nb_steps_per_year=kwargs.get("nb_steps_per_year", 360),
                                              seed=kwargs.get("seed"), gauss=kwargs.get("gauss", "fp32"), scheme=kwargs.get("scheme", "euler_floor"))


def compute_heston_mgf_grid(v0: float, theta: float, kappa: float, volvol: float, rho: float, ttm: float, phi_grid: np.ndarray,
                            psi_grid: np.ndarray, a_t0: np.ndarray = None, b_t0: np.ndarray = None):
    """closed-form Heston log-MGF over the grid, (log_mgf, a_t1, b_t1) (reference :183-214), on the GPU."""
    return engine.heston_mgf_grid(phi_grid, psi_grid, ttm, a_t0, b_t0, _params_c(v0, theta, kappa, rho, volvol))


def heston_chain_pricer(v0: float, theta: float, kappa: float, volvol: float, rho: float, ttms: np.ndarray, forwards: np.ndarray,
                        strikes_ttms, optiontypes_ttms, discfactors: np.ndarray,
                        variable_type: VariableType = VariableType.LOG_RETURN, vol_scaler: float = None, **kwargs) -> List[np.ndarray]:
    """Fourier chain pricer (reference :217-282), one fused GPU call for the chain."""
    vt = getattr(variable_type, "value", variable_type)
    if vt not in (1, 2):
        raise NotImplementedError(f"variable_type={variable_type}")      # heston_pricer.py:276-277
    return engine.heston_price_chain(_params_c(v0, theta, kappa, rho, volvol), ttms, forwards, discfactors, strikes_ttms,
                                     optiontypes_ttms, vol_scaler=vol_scaler, max_phi=kwargs.get("max_phi"),
                                     return_grids=bool(kwargs.get("return_grids", False)), variable_type=vt)


def heston_mc_chain_pricer(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, v0: float, theta: float, kappa: float,
                           rho: float, volvol: float, nb_path: int = 100000, variable_type: VariableType = VariableType.LOG_RETURN,
                           nb_steps_per_year: int = 360, seed: Optional[int] = None, precision: str = "fp64", gauss: str = "fp32",
                           distributed: bool = True, scheme="euler_floor", exchange: Optional[str] = None) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """chain MC under Heston (reference :285-331)."""
    params_c = _params_c(v0, theta, kappa, rho, volvol)
    flags = engine.mc_flags(precision, gauss)
    seed = _shared_seed(seed)
    if _use_distributed({"distributed": distributed, "nb_path": nb_path, "exchange": exchange}):
        return mc_chain_distributed("heston", params_c, ttms, forwards, discfactors, None, strikes_ttms, optiontypes_ttms, nb_path,
                                    nb_steps_per_year, True, engine.variable_code(variable_type), seed, flags, scheme=_scheme_code(scheme), exchange=exchange)
    return engine.heston_mc_chain(params_c, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path, nb_steps_per_year,
                                  variable_type, seed, flags, _scheme_code(scheme))


def simulate_heston_x_vol_terminal(ttm: float, x0: np.ndarray, var0: np.ndarray, qvar0: np.ndarray, theta: float, kappa: float,
                                   rho: float, volvol: float, nb_path: int = 100000, nb_steps_per_year: int = 360,
                                   W0: Optional[np.ndarray] = None, W1: Optional[np.ndarray] = None, dt: Optional[float] = None,
                                   seed: Optional[int] = None, gauss: str = "fp32", scheme="euler_floor"):
    """terminal (x, variance, qvar) by floor-Euler (reference :334-381; ``scheme="qe"`` opts into Andersen's QE).  ``W0, W1, dt`` (an extension: the reference has no
    fixed-random Heston entry) select the strict-arithmetic kernel."""
    if W0 is not None or W1 is not None:
        if W0 is None or W1 is None or dt is None:
            raise ValueError("W0, W1 and dt must be supplied together")
        return engine.heston_step_fixed(x0, var0, qvar0, W0, W1, dt, _params_c(1.0, theta, kappa, rho, volvol))
    x0, var0, qvar0 = np.atleast_1d(x0), np.atleast_1d(var0), np.atleast_1d(qvar0)
    for a in (x0, var0, qvar0):
        assert a.shape[0] in (1, nb_path)
    x_ok = x0.shape[0] == 1 or not np.any(x0)
    q_ok = qvar0.shape[0] == 1 or not np.any(qvar0)
    if not (x_ok and q_ok and np.all(var0 == var0[0])):
        raise NotImplementedError("the fused kernel starts every path from (0, v0, 0); pass W0/W1/dt for per-path initial states")
    seed = engine.fresh_seed() if seed is None else int(seed)
    return engine.heston_terminal(_params_c(float(var0[0]), theta, kappa, rho, volvol), ttm, nb_path, nb_steps_per_year, seed,
                                  engine.mc_flags("fp64", gauss), _scheme_code(scheme))


def v0_implied(v0: float, volvol: float, ttm: float) -> float:
    """the reference's placeholder short-maturity adjustment of the initial variance (heston_pricer.py:384-390)"""
    return v0 - volvol * volvol * ttm / 8.0
