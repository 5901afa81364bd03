"""Monte Carlo sensitivities of the chain pricers (DESIGN.md §3.9-3.11): the result type and the argument checks of
``LogSVPricer.model_mc_chain_greeks``, ``HestonPricer.model_mc_chain_greeks``, ``LogSVPricer.rough_mc_chain_greeks`` and
``HawkesJDPricer.model_mc_chain_greeks``.

One GPU pass returns, for every strike and maturity, the price and its standard error (identical to ``model_mc_price_chain`` on the same
seed), the forward delta and the derivative with respect to every model parameter, each with its own standard error.  The estimators are
unbiased for the discretised scheme the pricer simulates.

Under an initialised ``torch.distributed`` world the call is REPLICATED, not sharded: every rank prices all ``nb_path`` paths on its own
GPU.  The Philox counter is the global path id, so every rank returns bit-identical results.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np

from .. import _capi as C


@dataclass
class McChainGreeks:
    """prices / std errors / delta / delta_se: one array per maturity.  ``params`` / ``params_se``: parameter name (dataclass field,
    after ``__post_init__``) -> one array per maturity of d price / d parameter and its standard error.  ``reset_paths`` (rough-vol route
    only, else None): per maturity, the number of paths that took the reset-to-1e-6 branch at any step; the pathwise rows omit the price
    mass such paths move across that switch, so they are unbiased for the scheme only where it is 0.  ``gamma`` / ``gamma_se`` (LogSV and
    Heston with ``with_gamma=True``, else None): one array per maturity of d^2 price / d forward^2 by conditional smoothing of the
    last step (DESIGN.md §3.9) and its standard error.  ``theta`` / ``theta_se`` (LogSV and Heston with ``with_theta=True``, else None):
    one array per maturity of -d price / d ttm per year, pathwise in the slice's step length with its step count held (DESIGN.md §3.12),
    and its standard error; named as ``FourierChainGreeks.theta``.  ``params["theta"]`` stays d price / d theta."""
    prices: List[np.ndarray]
    std_errors: List[np.ndarray]
    delta: List[np.ndarray]
    delta_se: List[np.ndarray]
    params: Dict[str, List[np.ndarray]]
    params_se: Dict[str, List[np.ndarray]]
    reset_paths: Optional[np.ndarray] = None
    gamma: Optional[List[np.ndarray]] = None
    gamma_se: Optional[List[np.ndarray]] = None
    theta: Optional[List[np.ndarray]] = None
    theta_se: Optional[List[np.ndarray]] = None


def check_greeks_kwargs(kwargs, precision_default: str = "fp64") -> None:
    """reject what the pathwise route does not cover before any GPU work"""
    if kwargs.get("precision", precision_default) != "fp64":
        raise NotImplementedError("model_mc_chain_greeks needs precision='fp64'")
    if kwargs.get("use_rough_mc"):
        raise NotImplementedError("model_mc_chain_greeks does not cover the rough-vol route (use_rough_mc): use LogSVPricer.rough_mc_chain_greeks")
    if kwargs.get("exchange") is not None:
        raise NotImplementedError("model_mc_chain_greeks is single-GPU per rank (replicated under torch.distributed): no exchange")
    if kwargs.get("gauss", "fp32") not in ("fp32", "fp64"):
        raise NotImplementedError("model_mc_chain_greeks supports gauss='fp32' or 'fp64'")


def check_rough_greeks_kwargs(kwargs) -> None:
    """what LogSVPricer.rough_mc_chain_greeks rejects before any GPU work"""
    if kwargs.get("precision", "fp64") != "fp64":
        raise NotImplementedError("rough_mc_chain_greeks needs precision='fp64'")
    if kwargs.get("exchange") is not None:
        raise NotImplementedError("rough_mc_chain_greeks is single-GPU per rank (replicated under torch.distributed): no exchange")
    if kwargs.get("gauss") not in (None, "fp32", "fp64"):
        raise NotImplementedError("rough_mc_chain_greeks supports gauss=None (RandomState normals), 'fp32' or 'fp64'")
    if kwargs.get("seed") is None:
        raise ValueError("rough_mc_chain_greeks needs a seed, like model_mc_price_chain(use_rough_mc=True)")


def check_hawkes_mc_greeks_kwargs(kwargs, gauss, params) -> None:
    """what HawkesJDPricer.model_mc_chain_greeks rejects before any GPU work"""
    if kwargs.get("precision", "fp64") != "fp64":
        raise NotImplementedError("model_mc_chain_greeks needs precision='fp64'")
    if kwargs.get("exchange") is not None:
        raise NotImplementedError("model_mc_chain_greeks is single-GPU per rank (replicated under torch.distributed): no exchange")
    if gauss not in ("fp32", "fp64"):
        raise NotImplementedError("model_mc_chain_greeks supports gauss='fp32' or 'fp64'")
    vt = kwargs.get("variable_type", C.LOG_RETURN)
    if getattr(vt, "value", vt) != C.LOG_RETURN:
        raise NotImplementedError("the Hawkes Monte Carlo sensitivities cover variable_type=LOG_RETURN only")
    if params.risk_premia_gamma is not None:
        raise NotImplementedError("the Hawkes Monte Carlo sensitivities do not cover a risk kernel (risk_premia_gamma)")
    if params.mean_p == 0.0 or params.mean_m == 0.0:
        # d J / d mean is the jump's unit exponential, recovered as (J - shift) / mean: undefined for a degenerate jump size
        raise ValueError("the Hawkes Monte Carlo sensitivities need mean_p != 0 and mean_m != 0")


def check_no_gamma(kwargs, method: str) -> None:
    """the routes without a Monte Carlo gamma reject ``with_gamma=True`` before any GPU work"""
    if kwargs.get("with_gamma"):
        raise NotImplementedError(f"{method} has no Monte Carlo gamma: with_gamma=True covers LogSVPricer and HestonPricer.model_mc_chain_greeks")


def check_no_theta(kwargs, method: str, reason: str) -> None:
    """the routes without a Monte Carlo theta reject ``with_theta=True`` before any GPU work"""
    if kwargs.get("with_theta"):
        raise NotImplementedError(f"{method} has no Monte Carlo theta: {reason}")


def to_mc_chain_greeks(result, names: Sequence[str]) -> McChainGreeks:
    """engine.*_mc_chain_greeks output -> McChainGreeks; engine.*_mc_chain_greeks_gamma output (gamma and gamma_se after the offsets) fills
    ``gamma`` / ``gamma_se`` as well; engine.*_mc_chain_greeks_theta output (gamma, gamma_se -- None without gamma --, theta, theta_se, dtheta
    after the offsets) fills ``theta`` / ``theta_se`` and, where given, ``gamma`` / ``gamma_se``"""
    prices, stds, greeks, greeks_se, offsets = result[:5]
    split = lambda row: None if row is None else C.split_chain(row, offsets)
    out = McChainGreeks(prices=prices, std_errors=stds, delta=split(greeks[0]), delta_se=split(greeks_se[0]),
                        params={n: split(greeks[1 + k]) for k, n in enumerate(names)},
                        params_se={n: split(greeks_se[1 + k]) for k, n in enumerate(names)})
    if len(result) > 5:
        out.gamma, out.gamma_se = split(result[5]), split(result[6])
    if len(result) > 9:
        out.theta, out.theta_se = split(result[7]), split(result[8])
    return out
