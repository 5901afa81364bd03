"""Forward-mode sensitivities of the LogSV / Heston / Hawkes Fourier chain pricers (DESIGN.md §4.2, §4.3): the result type and the checks
shared by ``LogSVPricer.price_chain_greeks``, ``HestonPricer.price_chain_greeks`` and ``HawkesJDPricer.price_chain_greeks``.

One call returns, for every strike and maturity, the price (bit-identical to ``price_chain`` with the same arguments), delta and gamma
with respect to the slice forward, and the derivative with respect to every model parameter.  The parameter sensitivities are the exact
derivative of the scheme the pricer runs: the coefficient ODEs are differentiated on the adaptive solver's own accepted steps, and the
transform grid is held fixed.  No step size to choose.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from .. import _capi as C


@dataclass
class FourierChainGreeks:
    """prices / delta (d price / d forward) / gamma (d^2 price / d forward^2): one array per maturity.  ``params``: parameter name
    (dataclass field, after ``__post_init__``) -> one array per maturity of d price / d parameter.  ``theta`` (with ``with_theta=True``,
    else None): one array per maturity of -d price / d ttm per year, DESIGN.md §4.8."""
    prices: List[np.ndarray]
    delta: List[np.ndarray]
    gamma: List[np.ndarray]
    params: Dict[str, List[np.ndarray]]
    theta: Optional[List[np.ndarray]] = field(default=None, kw_only=True)


@dataclass
class FourierChainHessian(FourierChainGreeks):
    """``FourierChainGreeks`` (bit-identical to ``price_chain_greeks``) plus the second order, one array per maturity:
    ``vanna``: parameter name -> d^2 price / d forward d parameter; ``hessian``: name -> name -> d^2 price / d p d q, symmetric
    (``hessian[p][q]`` and ``hessian[q][p]`` are the same arrays)."""
    vanna: Dict[str, List[np.ndarray]]
    hessian: Dict[str, Dict[str, List[np.ndarray]]]


@dataclass
class ChainIvolGreeks:
    """implied-vol sensitivities of a chain (DESIGN.md §4.6), one array per maturity: ``ivols`` (bit-identical to
    ``compute_chain_prices_with_vols`` with the same arguments), ``delta`` / ``gamma`` (d ivol / d forward, d^2 ivol / d forward^2, sticky
    strike) and ``params``: parameter name -> d ivol / d parameter.  NaN where the ivol is NaN, 0 where it is an end of the inversion
    bracket (1e-8 or 10).  ``gamma`` is None for Monte Carlo sensitivities without a gamma row.  ``theta`` (with ``with_theta=True``, else
    None): -d ivol / d ttm per year at fixed forward and discount factor, under the same NaN / bracket-end rules (DESIGN.md §4.8)."""
    ivols: List[np.ndarray]
    delta: List[np.ndarray]
    gamma: Optional[List[np.ndarray]]
    params: Dict[str, List[np.ndarray]]
    theta: Optional[List[np.ndarray]] = field(default=None, kw_only=True)


@dataclass
class ChainIvolHessian(ChainIvolGreeks):
    """``ChainIvolGreeks`` plus ``vanna``: name -> d^2 ivol / d forward d parameter, and ``hessian``: name -> name -> d^2 ivol / d p d q,
    symmetric (``hessian[p][q]`` and ``hessian[q][p]`` are the same arrays)."""
    vanna: Dict[str, List[np.ndarray]]
    hessian: Dict[str, Dict[str, List[np.ndarray]]]


_MAX_IVOL_ROWS = 15     # parameter rows per b200sv_bsm_implied_vol_sensitivities call


def _flat(rows_ttms) -> np.ndarray:
    return np.concatenate([np.asarray(r, dtype=np.float64).ravel() for r in rows_ttms])


def to_chain_ivol_sensitivities(option_chain, greeks: FourierChainGreeks):
    """``FourierChainGreeks`` -> ``ChainIvolGreeks``, ``FourierChainHessian`` -> ``ChainIvolHessian``: the price rows mapped to implied-vol
    rows on the chain's forwards and discount factors by one engine.bsm_implied_vol_sensitivities call.  A Monte Carlo ``McChainGreeks``
    maps the same way (its standard errors are not carried over); without a gamma row (``gamma`` None) the transform gets zeros in its place
    and the result has ``gamma=None``, the other rows being independent of it.  A ``theta`` row is mapped by a second call,
    engine.bsm_implied_vol_theta, on the same prices (the same ivols, bit for bit).  Past the transform's 15 parameter rows, further calls
    on the same prices map the remaining rows, first or second order (DESIGN.md §4.12, §4.13)."""
    from .. import engine
    names = list(greeks.params)
    delta = _flat(greeks.delta)
    gamma = np.zeros_like(delta) if greeks.gamma is None else _flat(greeks.gamma)
    rows = np.vstack([delta, gamma, *(_flat(greeks.params[n]) for n in names)])
    second = isinstance(greeks, FourierChainHessian)
    head = names[:_MAX_IVOL_ROWS]
    tri = lambda group: np.vstack([_flat(greeks.hessian[p][q]) for i, p in enumerate(group) for q in group[i:]])
    vanna = np.vstack([_flat(greeks.vanna[n]) for n in head]) if second else None
    hessian = tri(head) if second else None
    chain = (option_chain.ttms, option_chain.forwards, option_chain.discfactors, option_chain.strikes_ttms, option_chain.optiontypes_ttms)
    ivols, g, v, h = engine.bsm_implied_vol_sensitivities(*chain, greeks.prices, rows[:2 + _MAX_IVOL_ROWS], vanna, hessian)
    pair_rows = {(p, q): h[r] for r, (p, q) in enumerate((p, q) for i, p in enumerate(head) for q in head[i:])} if second else None
    if rows.shape[0] > 2 + _MAX_IVOL_ROWS and not second:
        # a first-order parameter row maps on its own (d ivol / d p = d price / d p / vega): the rows past the transform's limit go through
        # a further call on the same prices, with delta and gamma again in front
        for r0 in range(2 + _MAX_IVOL_ROWS, rows.shape[0], _MAX_IVOL_ROWS):
            more = engine.bsm_implied_vol_sensitivities(*chain, greeks.prices, np.vstack([rows[:2], rows[r0:r0 + _MAX_IVOL_ROWS]]))[1]
            g = np.vstack([g, more[2:]])
    elif rows.shape[0] > 2 + _MAX_IVOL_ROWS:
        # second order past the limit: sigma_pq = (P_pq - B_ss sigma_p sigma_q) / B_s and vanna_p need only the rows of p and q, so each
        # further name e goes through calls on the same prices with e first and at most 14 of the names before it, [e, p1..p14], [e, p15],
        # ...; e's first-order row, vanna and (e, e) come from its first call, each (e, q) from the call that holds q
        v = list(v)
        for i in range(_MAX_IVOL_ROWS, len(names)):
            e = names[i]
            for c0 in range(0, i, _MAX_IVOL_ROWS - 1):
                group = [e] + names[c0:min(i, c0 + _MAX_IVOL_ROWS - 1)]
                sel = [names.index(n) for n in group]
                _, mg, mv, mh = engine.bsm_implied_vol_sensitivities(*chain, greeks.prices, np.vstack([rows[:2], rows[[2 + k for k in sel]]]),
                                                                     np.vstack([_flat(greeks.vanna[n]) for n in group]), tri(group))
                if c0 == 0:
                    g, v = np.vstack([g, mg[2:3]]), v + [mv[0]]
                    pair_rows[(e, e)] = mh[0]
                for k, q in enumerate(group[1:], 1):
                    pair_rows[(q, e)] = mh[k]
    offsets = np.zeros(len(ivols) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([a.size for a in ivols])
    split = lambda row: C.split_chain(row, offsets)
    theta = None
    if getattr(greeks, "theta", None) is not None:
        theta = split(engine.bsm_implied_vol_theta(option_chain.ttms, option_chain.forwards, option_chain.discfactors,
                                                   option_chain.strikes_ttms, option_chain.optiontypes_ttms, greeks.prices,
                                                   _flat(greeks.theta))[1])
    first = ChainIvolGreeks(ivols=ivols, delta=split(g[0]), gamma=None if greeks.gamma is None else split(g[1]),
                            params={n: split(g[2 + k]) for k, n in enumerate(names)}, theta=theta)
    if not second:
        return first
    hess: Dict[str, Dict[str, List[np.ndarray]]] = {n: {} for n in names}
    for i, p in enumerate(names):
        for q in names[i:]:
            hess[p][q] = hess[q][p] = split(pair_rows[(p, q)])
    return ChainIvolHessian(ivols=first.ivols, delta=first.delta, gamma=first.gamma, params=first.params,
                            vanna={n: split(v[k]) for k, n in enumerate(names)}, hessian=hess)


def _check_fourier_kwargs(kwargs, method: str) -> None:
    if kwargs.get("is_analytic"):
        raise NotImplementedError(f"{method} does not cover the semi-analytic branch (is_analytic)")
    if kwargs.get("is_stiff_solver"):
        raise NotImplementedError(f"{method} does not cover the BDF branch (is_stiff_solver)")
    if kwargs.get("use_rough_mc"):
        raise NotImplementedError(f"{method} does not cover the rough-vol route (use_rough_mc)")
    vt = kwargs.get("variable_type")
    if vt is not None and getattr(vt, "value", vt) != C.LOG_RETURN:
        raise NotImplementedError(f"{method} covers variable_type=LOG_RETURN only")


def check_fourier_greeks_kwargs(kwargs) -> None:
    """reject what the forward-mode route does not cover before any GPU work"""
    _check_fourier_kwargs(kwargs, "price_chain_greeks")


def check_fourier_hessian_kwargs(kwargs) -> None:
    """the same rejections for ``price_chain_hessian``, which has no theta (second-order time terms are not covered)"""
    if kwargs.get("with_theta"):
        raise NotImplementedError("price_chain_hessian does not cover theta (with_theta): use price_chain_greeks(with_theta=True)")
    _check_fourier_kwargs(kwargs, "price_chain_hessian")


def to_fourier_chain_greeks(prices, greeks, offsets, names: Sequence[str], theta=None) -> FourierChainGreeks:
    """engine.*_price_chain_greeks output -> FourierChainGreeks; ``theta`` [J] (with_theta) or None"""
    split = lambda row: C.split_chain(row, offsets)
    return FourierChainGreeks(prices=prices, delta=split(greeks[0]), gamma=split(greeks[1]),
                              params={n: split(greeks[2 + k]) for k, n in enumerate(names)}, theta=None if theta is None else split(theta))


def to_fourier_chain_hessian(prices, greeks, vanna, hessian, offsets, names: Sequence[str]) -> FourierChainHessian:
    """engine.*_price_chain_hessian output -> FourierChainHessian; hessian rows are the upper triangle p <= q, row-major in ``names``"""
    split = lambda row: C.split_chain(row, offsets)
    first = to_fourier_chain_greeks(prices, greeks, offsets, names)
    hess: Dict[str, Dict[str, List[np.ndarray]]] = {n: {} for n in names}
    r = 0
    for i, p in enumerate(names):
        for q in names[i:]:
            hess[p][q] = hess[q][p] = split(hessian[r])
            r += 1
    return FourierChainHessian(prices=first.prices, delta=first.delta, gamma=first.gamma, params=first.params,
                               vanna={n: split(vanna[k]) for k, n in enumerate(names)}, hessian=hess)
