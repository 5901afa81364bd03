"""Pathwise Monte Carlo sensitivities of the LogSV / Heston chain pricers (DESIGN.md §3.9): the result type and the checks shared by
``LogSVPricer.model_mc_chain_greeks`` and ``HestonPricer.model_mc_chain_greeks``.

One GPU pass returns, for every strike and maturity, the price and its standard error (identical to ``model_mc_price_chain`` on the same
seed), the forward delta and the derivative with respect to every model parameter, each with its own standard error.  The estimators are
unbiased for the discretised scheme the pricer simulates.

Under an initialised ``torch.distributed`` world the call is REPLICATED, not sharded: every rank prices all ``nb_path`` paths on its own
GPU.  The Philox counter is the global path id, so every rank returns bit-identical results.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence

import numpy as np

from .. import _capi as C


@dataclass
class McChainGreeks:
    """prices / std errors / delta / delta_se: one array per maturity.  ``params`` / ``params_se``: parameter name (dataclass field,
    after ``__post_init__``) -> one array per maturity of d price / d parameter and its standard error."""
    prices: List[np.ndarray]
    std_errors: List[np.ndarray]
    delta: List[np.ndarray]
    delta_se: List[np.ndarray]
    params: Dict[str, List[np.ndarray]]
    params_se: Dict[str, List[np.ndarray]]


def check_greeks_kwargs(kwargs, precision_default: str = "fp64") -> None:
    """reject what the pathwise route does not cover before any GPU work"""
    if kwargs.get("precision", precision_default) != "fp64":
        raise NotImplementedError("model_mc_chain_greeks needs precision='fp64'")
    if kwargs.get("use_rough_mc"):
        raise NotImplementedError("model_mc_chain_greeks does not cover the rough-vol route (use_rough_mc)")
    if kwargs.get("exchange") is not None:
        raise NotImplementedError("model_mc_chain_greeks is single-GPU per rank (replicated under torch.distributed): no exchange")
    if kwargs.get("gauss", "fp32") not in ("fp32", "fp64"):
        raise NotImplementedError("model_mc_chain_greeks supports gauss='fp32' or 'fp64'")


def to_mc_chain_greeks(result, names: Sequence[str]) -> McChainGreeks:
    """engine.*_mc_chain_greeks output -> McChainGreeks"""
    prices, stds, greeks, greeks_se, offsets = result
    split = lambda row: C.split_chain(row, offsets)
    return McChainGreeks(prices=prices, std_errors=stds, delta=split(greeks[0]), delta_se=split(greeks_se[0]),
                         params={n: split(greeks[1 + k]) for k, n in enumerate(names)},
                         params_se={n: split(greeks_se[1 + k]) for k, n in enumerate(names)})
