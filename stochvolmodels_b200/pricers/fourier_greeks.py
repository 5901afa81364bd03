"""Forward-mode sensitivities of the LogSV / Heston / Hawkes Fourier chain pricers (DESIGN.md §4.2, §4.3): the result type and the checks
shared by ``LogSVPricer.price_chain_greeks``, ``HestonPricer.price_chain_greeks`` and ``HawkesJDPricer.price_chain_greeks``.

One call returns, for every strike and maturity, the price (bit-identical to ``price_chain`` with the same arguments), delta and gamma
with respect to the slice forward, and the derivative with respect to every model parameter.  The parameter sensitivities are the exact
derivative of the scheme the pricer runs: the coefficient ODEs are differentiated on the adaptive solver's own accepted steps, and the
transform grid is held fixed.  No step size to choose.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence

import numpy as np

from .. import _capi as C


@dataclass
class FourierChainGreeks:
    """prices / delta (d price / d forward) / gamma (d^2 price / d forward^2): one array per maturity.  ``params``: parameter name
    (dataclass field, after ``__post_init__``) -> one array per maturity of d price / d parameter."""
    prices: List[np.ndarray]
    delta: List[np.ndarray]
    gamma: List[np.ndarray]
    params: Dict[str, List[np.ndarray]]


def check_fourier_greeks_kwargs(kwargs) -> None:
    """reject what the forward-mode route does not cover before any GPU work"""
    if kwargs.get("is_analytic"):
        raise NotImplementedError("price_chain_greeks does not cover the semi-analytic branch (is_analytic)")
    if kwargs.get("is_stiff_solver"):
        raise NotImplementedError("price_chain_greeks does not cover the BDF branch (is_stiff_solver)")
    if kwargs.get("use_rough_mc"):
        raise NotImplementedError("price_chain_greeks does not cover the rough-vol route (use_rough_mc)")
    vt = kwargs.get("variable_type")
    if vt is not None and getattr(vt, "value", vt) != C.LOG_RETURN:
        raise NotImplementedError("price_chain_greeks covers variable_type=LOG_RETURN only")


def to_fourier_chain_greeks(prices, greeks, offsets, names: Sequence[str]) -> FourierChainGreeks:
    """engine.*_price_chain_greeks output -> FourierChainGreeks"""
    split = lambda row: C.split_chain(row, offsets)
    return FourierChainGreeks(prices=prices, delta=split(greeks[0]), gamma=split(greeks[1]),
                              params={n: split(greeks[2 + k]) for k, n in enumerate(names)})
