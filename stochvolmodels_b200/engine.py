"""numpy <-> C-ABI marshalling for the host-level entry points of libb200sv (include/b200sv.h).

Thin by design: validation that the reference does in Python (exception classes, messages) lives here; all arithmetic is in
the CUDA library.  No function in this module computes a price on the CPU.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import byref
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _capi as C
from .utils.config import VariableType


_SEED_STREAM = None          # set_seed(): a deterministic stream of per-call Philox seeds; None: OS entropy


def set_seed(value) -> None:
    """the reference's ``set_seed`` (utils/funcs.py:51-60) seeds Numba's process-global generator so that the Monte Carlo calls that follow
    are reproducible.  Here every MC call takes an explicit ``seed``; calls WITHOUT one draw theirs from a process-global stream that this
    function (re)starts, so `set_seed(8); price(); price()` gives the same two results in every run, as with the reference.  ``None``
    returns to OS entropy."""
    global _SEED_STREAM
    _SEED_STREAM = None if value is None else np.random.Generator(np.random.Philox(int(value)))


def fresh_seed() -> int:
    """seed of an MC call that was not given one: next value of the set_seed() stream, else OS entropy."""
    if _SEED_STREAM is not None:
        return int(_SEED_STREAM.integers(0, 1 << 63))
    return int.from_bytes(os.urandom(8), "little")


def mc_flags(precision: str = "fp64", gauss: str = "fp32") -> int:
    """precision: 'fp64' (default) | 'fp32' state arithmetic; gauss: 'fp32' (default, SFU Box-Muller) | 'fp64' (fp64 Box-Muller on
    52-bit uniforms) | 'fp64_paired' (check mode: the default stream's 32-bit uniforms through the fp64 Box-Muller)."""
    if precision not in ("fp64", "fp32"):
        raise ValueError("precision must be 'fp64' or 'fp32'")
    if gauss not in ("fp32", "fp64", "fp64_paired"):
        raise ValueError("gauss must be 'fp32', 'fp64' or 'fp64_paired'")
    return (C.STATE_F32 if precision == "fp32" else C.STATE_F64) | {"fp32": C.GAUSS_F32, "fp64": C.GAUSS_F64, "fp64_paired": C.GAUSS_F64_PAIRED}[gauss]


def variable_code(variable_type) -> int:
    v = variable_type.value if isinstance(variable_type, VariableType) or hasattr(variable_type, "value") else int(variable_type)
    if v not in (C.LOG_RETURN, C.Q_VAR):
        raise NotImplementedError        # utils/mc_payoffs.py:69-70, pricers/logsv_pricer.py:733-734
    return v


def logsv_params_c(sigma0, theta, kappa1, kappa2, beta, volvol) -> C.LogsvParamsC:
    return C.LogsvParamsC(float(sigma0), float(theta), float(kappa1), float(kappa2), float(beta), float(volvol))


def heston_params_c(v0, theta, kappa, rho, volvol) -> C.HestonParamsC:
    return C.HestonParamsC(float(v0), float(theta), float(kappa), float(rho), float(volvol))


class _Chain(NamedTuple):
    M: int
    ttms: np.ndarray
    forwards: np.ndarray
    discfactors: np.ndarray
    offsets: np.ndarray
    strikes: np.ndarray
    types: np.ndarray


def _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms) -> _Chain:
    ttms, forwards, discfactors = C.f64(ttms), C.f64(forwards), C.f64(discfactors)
    M = ttms.shape[0]
    if not (forwards.shape[0] == discfactors.shape[0] == len(strikes_ttms) == len(optiontypes_ttms) == M):
        raise ValueError("ttms, forwards, discfactors, strikes_ttms, and optiontypes_ttms must have the same length")
    offsets, strikes, types = C.flatten_chain(strikes_ttms, optiontypes_ttms)
    return _Chain(M, ttms, forwards, discfactors, offsets, strikes, types)


def _backbone(etas, M: int):
    """the etas slot of a single-set chain call: [vol backbone [M], ones when None] on the LogSV routes, [] (passed as ()) on the others"""
    return [C.f64(np.ones(M) if e is None else e) for e in etas]


# ---- Monte Carlo --------------------------------------------------------------------------------------------------------
def _mc_chain(symbol: str, params, chain, etas, head, variable_type, seed: int, flags: int, tail=(), n_greeks: int = 0, post=()):
    """the single-set chain MC entry points: C arguments (params, chain block, *head, variable type, seed, flags, *tail, prices, stds
    [, greeks, greeks_se], *post).  ``etas`` = (LogSV vol backbone or None,) or ().  With ``n_greeks`` returns (prices, std errors,
    greeks [1+P, J], greeks_se [1+P, J], offsets), else (prices, std errors)."""
    vt = variable_code(variable_type)
    ch = _chain_arrays(*chain)
    etas = _backbone(etas, ch.M)
    J = ch.strikes.shape[0]
    prices, stds = np.empty(J), np.empty(J)
    greeks = [np.empty((1 + n_greeks, J)), np.empty((1 + n_greeks, J))] if n_greeks else []
    C.call(symbol, byref(params), *C.chain_ptrs(ch, *etas), *head, vt, C.seed64(seed), int(flags), *tail, C.dptr(prices), C.dptr(stds),
           *map(C.dptr, greeks), *post)
    prices, stds = C.split_chain(prices, ch.offsets), C.split_chain(stds, ch.offsets)
    return (prices, stds, *greeks, ch.offsets) if n_greeks else (prices, stds)


def logsv_mc_chain(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                   nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int
                   ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    return _mc_chain("b200sv_logsv_mc_chain", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (etas,),
                     (int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure))), variable_type, seed, flags)


def heston_mc_chain(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                    nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR
                    ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    return _mc_chain("b200sv_heston_mc_chain", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (),
                     (int(nb_path), int(nb_steps_per_year)), variable_type, seed, flags, (int(scheme),))


def hawkesjd_mc_chain(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int, variable_type,
                      seed: int, flags: int) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """chain MC of the Hawkes jump-diffusion (b200sv_hawkesjd_mc_chain; its time grid is fixed by the library)"""
    return _mc_chain("b200sv_hawkesjd_mc_chain", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (), (int(nb_path),),
                     variable_type, seed, flags)


HAWKES_EXACT_DEFAULT_BUDGET = 1 << 20      # candidates per path and maturity interval of the exact route (include/b200sv.h)


def hawkesjd_mc_chain_exact(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int, variable_type,
                            seed: int, flags: int = 0, max_candidates: int = HAWKES_EXACT_DEFAULT_BUDGET, n_paths_out: int = 0):
    """chain MC of the Hawkes jump-diffusion on the exact event-driven route (b200sv_hawkesjd_mc_chain_exact; DESIGN.md §3.13).  Returns
    (prices, std errors, states, events): with ``n_paths_out`` > 0 states [M, 3, n_paths_out] = (x, lambda_p, lambda_m) and events
    [M, 3, n_paths_out] = (accepted '+', accepted '-', candidates) of the first paths per maturity, else None.  A path that draws more than
    ``max_candidates`` candidates in one interval fails the call (B200svError -6)."""
    M, n_out = C.f64(ttms).shape[0], int(n_paths_out)
    states = np.empty((M, 3, n_out)) if n_out else None
    events = np.empty((M, 3, n_out)) if n_out else None
    prices, stds = _mc_chain("b200sv_hawkesjd_mc_chain_exact", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (),
                             (int(nb_path),), variable_type, seed, flags, post=(int(max_candidates), n_out, C.dptr(states), C.dptr(events)))
    return prices, stds, states, events


LOGSV_GREEK_PARAMS = ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")
HESTON_GREEK_PARAMS = ("v0", "theta", "kappa", "rho", "volvol")
# HawkesJDParams fields in dataclass order without mu (the Fourier route never reads it) and risk_premia_gamma (not covered)
HAWKES_GREEK_PARAMS = ("sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p",
                       "lambda_m", "theta_m", "kappa_m", "beta1_m", "beta2_m")
# the rows of the risk-kernel pricer's sensitivities (DESIGN.md §4.12)
HAWKES_RISK_PREMIA_GREEK_PARAMS = HAWKES_GREEK_PARAMS + ("risk_premia_gamma",)


def logsv_mc_chain_greeks(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                          nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int):
    """prices, std errors and pathwise sensitivities of the chain in one pass (b200sv_logsv_mc_chain_greeks).  Returns (prices, std errors,
    greeks [1+6, J], greeks_se [1+6, J], offsets): row 0 the forward delta, then LOGSV_GREEK_PARAMS; J runs over the flattened chain."""
    return _mc_chain("b200sv_logsv_mc_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (etas,),
                     (int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure))), variable_type, seed, flags,
                     n_greeks=len(LOGSV_GREEK_PARAMS))


def heston_mc_chain_greeks(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                           nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR):
    """Heston twin of logsv_mc_chain_greeks (b200sv_heston_mc_chain_greeks): greeks rows = forward delta, then HESTON_GREEK_PARAMS."""
    return _mc_chain("b200sv_heston_mc_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (),
                     (int(nb_path), int(nb_steps_per_year)), variable_type, seed, flags, (int(scheme),), n_greeks=len(HESTON_GREEK_PARAMS))


def _mc_chain_greeks_gamma(symbol: str, params, chain, etas, head, variable_type, seed: int, flags: int, tail, n_greeks: int,
                           n_paths_out: int):
    M, J, n_out = len(chain[3]), sum(len(s) for s in chain[3]), int(n_paths_out)
    gamma, gamma_se = np.empty(J), np.empty(J)
    laststep = np.empty((M, 2, n_out)) if n_out else None
    res = _mc_chain(symbol, params, chain, etas, head, variable_type, seed, flags, tail, n_greeks=n_greeks,
                    post=(C.dptr(gamma), C.dptr(gamma_se), n_out, C.dptr(laststep)))
    return (*res, gamma, gamma_se, laststep)


def logsv_mc_chain_greeks_gamma(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                                nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int, n_paths_out: int = 0):
    """logsv_mc_chain_greeks plus the Monte Carlo gamma by conditional smoothing of the last step (b200sv_logsv_mc_chain_greeks_gamma;
    DESIGN.md §3.9).  Returns (prices, std errors, greeks [1+6, J], greeks_se [1+6, J], offsets, gamma [J], gamma_se [J], laststep): the
    first five bit-identical to logsv_mc_chain_greeks; with ``n_paths_out`` > 0, laststep [M, 2, n_paths_out] = (s, mu) of the first paths'
    last step after each maturity (x = mu + s z0), else None."""
    return _mc_chain_greeks_gamma("b200sv_logsv_mc_chain_greeks_gamma", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                  (etas,), (int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure))), variable_type, seed, flags, (),
                                  len(LOGSV_GREEK_PARAMS), n_paths_out)


def heston_mc_chain_greeks_gamma(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                                 nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR,
                                 n_paths_out: int = 0):
    """Heston twin of logsv_mc_chain_greeks_gamma (b200sv_heston_mc_chain_greeks_gamma)."""
    return _mc_chain_greeks_gamma("b200sv_heston_mc_chain_greeks_gamma", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                  (), (int(nb_path), int(nb_steps_per_year)), variable_type, seed, flags, (int(scheme),),
                                  len(HESTON_GREEK_PARAMS), n_paths_out)


def _mc_chain_greeks_theta(symbol: str, params, chain, etas, head, variable_type, seed: int, flags: int, tail, n_greeks: int,
                           with_gamma: bool, n_paths_out: int):
    M, J, n_out = len(chain[3]), sum(len(s) for s in chain[3]), int(n_paths_out)
    gamma, gamma_se = (np.empty(J), np.empty(J)) if with_gamma else (None, None)
    theta, theta_se = np.empty(J), np.empty(J)
    dtheta = np.empty((M, 2, n_out)) if n_out else None
    res = _mc_chain(symbol, params, chain, etas, head, variable_type, seed, flags, tail, n_greeks=n_greeks,
                    post=(C.dptr(gamma), C.dptr(gamma_se), n_out, None, C.dptr(theta), C.dptr(theta_se), C.dptr(dtheta)))
    return (*res, gamma, gamma_se, theta, theta_se, dtheta)


def logsv_mc_chain_greeks_theta(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                                nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int, with_gamma: bool = False,
                                n_paths_out: int = 0):
    """logsv_mc_chain_greeks (with_gamma: logsv_mc_chain_greeks_gamma) plus the Monte Carlo theta -d price / d ttm per year, pathwise in
    each slice's step length with its step count held (b200sv_logsv_mc_chain_greeks_theta; DESIGN.md §3.12).  Returns (prices, std errors,
    greeks [1+6, J], greeks_se [1+6, J], offsets, gamma [J] | None, gamma_se [J] | None, theta [J], theta_se [J], dtheta): the rest
    bit-identical to the call without theta; with ``n_paths_out`` > 0, dtheta [M, 2, n_paths_out] = (dx, dq) / d dt of the first paths after
    each maturity, else None."""
    return _mc_chain_greeks_theta("b200sv_logsv_mc_chain_greeks_theta", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                  (etas,), (int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure))), variable_type, seed, flags, (),
                                  len(LOGSV_GREEK_PARAMS), with_gamma, n_paths_out)


def heston_mc_chain_greeks_theta(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                                 nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR,
                                 with_gamma: bool = False, n_paths_out: int = 0):
    """Heston twin of logsv_mc_chain_greeks_theta (b200sv_heston_mc_chain_greeks_theta)."""
    return _mc_chain_greeks_theta("b200sv_heston_mc_chain_greeks_theta", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                  (), (int(nb_path), int(nb_steps_per_year)), variable_type, seed, flags, (int(scheme),),
                                  len(HESTON_GREEK_PARAMS), with_gamma, n_paths_out)


def hawkesjd_mc_chain_greeks(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int, variable_type,
                             seed: int, flags: int, n_paths_out: int = 0):
    """chain MC of the Hawkes jump-diffusion with Monte Carlo sensitivities (b200sv_hawkesjd_mc_chain_greeks; DESIGN.md §3.11).  Returns
    (prices, std errors, greeks [1+15, J], greeks_se [1+15, J], offsets, states, tangents): greeks row 0 the forward delta, then
    HAWKES_GREEK_PARAMS.  With ``n_paths_out`` > 0, states [M, 3, n_paths_out] = (x, lambda_p, lambda_m) and tangents [M, 4, 15, n_paths_out]
    = (dx, dlambda_p, dlambda_m, accumulated score) of the first paths after each maturity, else None."""
    M, P, n_out = C.f64(ttms).shape[0], len(HAWKES_GREEK_PARAMS), int(n_paths_out)
    states = np.empty((M, 3, n_out)) if n_out else None
    tangents = np.empty((M, 4, P, n_out)) if n_out else None
    res = _mc_chain("b200sv_hawkesjd_mc_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (), (int(nb_path),),
                    variable_type, seed, flags, n_greeks=P, post=(n_out, C.dptr(states), C.dptr(tangents)))
    return (*res, states, tangents)


def _tangent_terminal(symbol: str, params, ttm: float, nb_path: int, nb_steps_per_year: int, model_args, seed: int, flags: int,
                      slice_index: int, path_offset: int, n_params: int):
    out = [np.empty(nb_path) for _ in range(3)] + [np.empty((n_params, nb_path)) for _ in range(3)]
    C.call(symbol, byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), *model_args, C.seed64(seed), int(flags), int(slice_index),
           int(path_offset), *map(C.dptr, out))
    return tuple(out)


def logsv_tangent_terminal(params: C.LogsvParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                           seed: int, flags: int, slice_index: int = 0, path_offset: int = 0):
    """one slice of the tangent stepper from (0, sigma0, 0): (x, sigma, qvar, dx [6, n], dsigma [6, n], dqvar [6, n])"""
    return _tangent_terminal("b200sv_logsv_tangent_terminal", params, ttm, nb_path, nb_steps_per_year, (int(bool(is_spot_measure)), float(eta)),
                             seed, flags, slice_index, path_offset, len(LOGSV_GREEK_PARAMS))


def heston_tangent_terminal(params: C.HestonParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, seed: int, flags: int,
                            slice_index: int = 0, path_offset: int = 0):
    """one slice of the Heston tangent stepper from (0, v0, 0): (x, var, qvar, dx [5, n], dvar [5, n], dqvar [5, n])"""
    return _tangent_terminal("b200sv_heston_tangent_terminal", params, ttm, nb_path, nb_steps_per_year, (), seed, flags, slice_index,
                             path_offset, len(HESTON_GREEK_PARAMS))


def _chain_batch(symbol: str, struct, params_list, chain, etas, args, n_out: int, with_ivols: bool):
    """the batched chain entry points: C arguments (params [B], B, chain block with ``etas`` = (LogSV [B, M] or None,) or (), *args, n_out
    outputs [B, J], ivols [B, J] | NULL) -> (*outputs, ivols | None)"""
    ch = _chain_arrays(*chain)
    B = len(params_list)
    arr = (struct * B)(*params_list)
    etas = [C.batch_etas(e, B, ch.M) for e in etas]
    outs = [np.empty((B, ch.strikes.shape[0])) for _ in range(n_out)]
    ivols = np.empty((B, ch.strikes.shape[0])) if with_ivols else None
    C.call(symbol, arr, B, *C.chain_ptrs(ch, *etas), *args, *map(C.dptr, outs), C.dptr(ivols))
    return (*outs, ivols)


def logsv_mc_chain_batch(params_list: Sequence[C.LogsvParamsC], ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                         nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, seed: int, flags: int, with_ivols: bool = True):
    """B parameter sets through the fused chain MC on the SAME seed in one call -> (prices, std errors, ivols | None), each [B, J]."""
    return _chain_batch("b200sv_logsv_mc_chain_batch", C.LogsvParamsC, params_list, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                        (etas,), (int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)), C.seed64(seed), int(flags)), 2, with_ivols)


def heston_mc_chain_batch(params_list: Sequence[C.HestonParamsC], ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                          nb_path: int, nb_steps_per_year: int, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR,
                          with_ivols: bool = True):
    return _chain_batch("b200sv_heston_mc_chain_batch", C.HestonParamsC, params_list, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                        (), (int(nb_path), int(nb_steps_per_year), C.seed64(seed), int(flags), int(scheme)), 2, with_ivols)


def _rough_grid_normals(M: int, nb_path: int, nsteps, hs, Z0, Z1):
    """the per-maturity grids and the optional host normals of the rough-vol entry points -> (nsteps, hs, Z0, Z1, z_rows)"""
    nsteps = np.ascontiguousarray(nsteps, dtype=np.int32)
    hs = C.f64(hs)
    if nsteps.shape[0] != M or hs.shape[0] != M:
        raise ValueError("nsteps and hs must have one entry per maturity")
    z_rows = 0
    if Z0 is not None or Z1 is not None:
        if Z0 is None or Z1 is None:
            raise ValueError("Z0 and Z1 must be supplied together")
        Z0, Z1 = C.f64(Z0), C.f64(Z1)
        if Z0.ndim != 2 or Z0.shape != Z1.shape or Z0.shape[1] != nb_path:
            raise ValueError("Z0 and Z1 must be 2-d arrays [nb_steps, nb_path] of the same shape")
        z_rows = Z0.shape[0]
        if z_rows < int(nsteps.max()):
            raise ValueError("Z0 / Z1 have fewer rows than the longest time grid")
        if z_rows > int(nsteps.max()):          # the library uploads exactly max(nsteps) rows
            Z0, Z1 = np.ascontiguousarray(Z0[: int(nsteps.max())]), np.ascontiguousarray(Z1[: int(nsteps.max())])
            z_rows = int(nsteps.max())
    return nsteps, hs, Z0, Z1, z_rows


def rough_logsv_mc_chain_greeks(params: C.LogsvParamsC, weights, nodes, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                                nb_path: int, nsteps, hs, Z0=None, Z1=None, variable_type=1, seed: int = 0, flags: int = 0,
                                return_states: bool = False, return_tangents: bool = False, with_theta: bool = False, n_paths_out: int = 0):
    """one parameter set through the rough-LogSV chain MC with pathwise sensitivities (b200sv_rough_logsv_mc_chain_greeks).  Arguments as
    rough_logsv_mc_chain with ``weights`` / ``nodes`` [n].  Returns (prices, std errors, greeks [1+6, J], greeks_se [1+6, J], offsets,
    states [M, n + 2, nb_path] | None, tangents [M, 6, n + 2, nb_path] | None, resets [M]): greeks row 0 the forward delta, then
    LOGSV_GREEK_PARAMS; resets[m] = the number of paths that took the reset-to-1e-6 branch at any step of maturity m's grid.
    ``with_theta`` (b200sv_rough_logsv_mc_chain_greeks_theta; DESIGN.md §3.12) appends (theta [J], theta_se [J], dtheta): -d price / d ttm
    per year, pathwise in each maturity's step length with its step count held, the rest bit-identical; with ``n_paths_out`` > 0, dtheta
    [M, 2, n_paths_out] = (d log_spot, d qv) / d h of the first paths at each maturity, else None."""
    vt = variable_code(variable_type)
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    weights, nodes = C.f64(weights), C.f64(nodes)
    if weights.shape != nodes.shape or weights.ndim != 1:
        raise ValueError("weights and nodes must be 1-d arrays of the same length")
    n = weights.shape[0]
    nsteps, hs, Z0, Z1, z_rows = _rough_grid_normals(ch.M, nb_path, nsteps, hs, Z0, Z1)
    J, P = ch.strikes.shape[0], len(LOGSV_GREEK_PARAMS)
    prices, stds, greeks, greeks_se = np.empty(J), np.empty(J), np.empty((1 + P, J)), np.empty((1 + P, J))
    states = np.empty((ch.M, n + 2, int(nb_path))) if return_states else None
    tangents = np.empty((ch.M, P, n + 2, int(nb_path))) if return_tangents else None
    resets = np.empty(ch.M)
    args = (byref(params), n, C.dptr(weights), C.dptr(nodes), *C.chain_ptrs(ch), int(nb_path), C.iptr(nsteps), C.dptr(hs), C.dptr(Z0), C.dptr(Z1),
            int(z_rows), vt, C.seed64(seed), int(flags), C.dptr(prices), C.dptr(stds), C.dptr(greeks), C.dptr(greeks_se), C.dptr(states),
            C.dptr(tangents), C.dptr(resets))
    if with_theta:
        n_out = int(n_paths_out)
        theta, theta_se = np.empty(J), np.empty(J)
        dtheta = np.empty((ch.M, 2, n_out)) if n_out else None
        C.call("b200sv_rough_logsv_mc_chain_greeks_theta", *args, C.dptr(theta), C.dptr(theta_se), n_out, C.dptr(dtheta))
    else:
        C.call("b200sv_rough_logsv_mc_chain_greeks", *args)
    res = (C.split_chain(prices, ch.offsets), C.split_chain(stds, ch.offsets), greeks, greeks_se, ch.offsets, states, tangents,
           resets.astype(np.int64))
    return (*res, theta, theta_se, dtheta) if with_theta else res


def rough_logsv_mc_chain(params_list, weights, nodes, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int, nsteps, hs,
                         Z0=None, Z1=None, variable_type=1, seed: int = 0, flags: int = 0, with_ivols: bool = False, return_states: bool = False):
    """B parameter sets through the rough-LogSV multi-factor chain MC (b200sv_rough_logsv_mc_chain).  ``weights`` / ``nodes``: [n] (shared)
    or [B, n]; ``Z0`` / ``Z1``: host unit normals [rows >= max(nsteps), nb_path] or None (in-kernel Philox draws).
    Returns (prices [B, J], std [B, J], ivols [B, J] | None, states [M, n + 2, nb_path] | None)."""
    vt = variable_code(variable_type)
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    M = ch.M
    B = len(params_list)
    arr = (C.LogsvParamsC * B)(*params_list)
    weights, nodes = np.atleast_2d(C.f64(weights)), np.atleast_2d(C.f64(nodes))
    if weights.shape != nodes.shape or weights.ndim != 2:
        raise ValueError("weights and nodes must have the same 1-d (or [B, n]) shape")
    n = weights.shape[1]
    if weights.shape[0] == 1 and B > 1:
        weights, nodes = np.repeat(weights, B, axis=0), np.repeat(nodes, B, axis=0)
    if weights.shape[0] != B:
        raise ValueError(f"weights / nodes must have {B} rows")
    weights, nodes = np.ascontiguousarray(weights), np.ascontiguousarray(nodes)
    nsteps, hs, Z0, Z1, z_rows = _rough_grid_normals(M, nb_path, nsteps, hs, Z0, Z1)
    J = ch.strikes.shape[0]
    prices, stds = np.empty((B, J)), np.empty((B, J))
    ivols = np.empty((B, J)) if with_ivols else None
    states = np.empty((M, n + 2, int(nb_path))) if return_states else None
    C.call("b200sv_rough_logsv_mc_chain", arr, B, n, C.dptr(weights), C.dptr(nodes), *C.chain_ptrs(ch), int(nb_path), C.iptr(nsteps), C.dptr(hs),
           C.dptr(Z0), C.dptr(Z1), int(z_rows), vt, C.seed64(seed), int(flags), C.dptr(prices), C.dptr(stds), C.dptr(ivols), C.dptr(states))
    return prices, stds, ivols, states, ch.offsets


def logsv_terminal(params: C.LogsvParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                   seed: int, flags: int):
    x, s, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    C.call("b200sv_logsv_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)),
           float(eta), C.seed64(seed), int(flags), C.dptr(x), C.dptr(s), C.dptr(q))
    return x, s, q


def logsv_terminal_from_state(params: C.LogsvParamsC, x0, sigma0, qvar0, ttm: float, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                              seed: int, flags: int, slice_index: int = 0):
    """fused Philox stepper from PER-PATH initial arrays (b200sv_logsv_terminal_from_state); returns fresh (x, sigma, qvar) arrays."""
    x, s, q = (np.array(a, dtype=np.float64, copy=True, order="C") for a in (x0, sigma0, qvar0))
    if not (x.shape == s.shape == q.shape and x.ndim == 1):
        raise ValueError("x0, sigma0, qvar0 must be 1-d arrays of one length")
    C.call("b200sv_logsv_terminal_from_state", byref(params), float(ttm), int(x.shape[0]), int(nb_steps_per_year), int(bool(is_spot_measure)),
           float(eta), C.seed64(seed), int(flags), int(slice_index), C.dptr(x), C.dptr(s), C.dptr(q))
    return x, s, q


def set_stream(stream) -> None:
    """CUDA stream (int / ctypes pointer / torch.cuda.Stream) for this thread's host-level library calls; None = the default stream."""
    ptr = getattr(stream, "cuda_stream", stream)
    C.call("b200sv_set_stream", ptr)


def heston_terminal(params: C.HestonParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, seed: int, flags: int,
                    scheme: int = C.HESTON_EULER_FLOOR):
    x, v, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    C.call("b200sv_heston_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year),
           C.seed64(seed), int(flags), int(scheme), C.dptr(x), C.dptr(v), C.dptr(q))
    return x, v, q


def hawkesjd_terminal(params: C.HawkesParamsC, ttm: float, x, lambda_p, lambda_m, seed: int, flags: int, slice_index: int, per_path: bool):
    """fused Philox stepper of the Hawkes jump-diffusion (b200sv_hawkesjd_terminal), in place on the float64 arrays (x, lambda_p, lambda_m);
    without ``per_path`` every path starts from (0, params.lambda_p, params.lambda_m)"""
    C.call("b200sv_hawkesjd_terminal", byref(params), float(ttm), int(x.shape[0]), C.seed64(seed), flags, int(slice_index), 1 if per_path else 0,
           C.dptr(x), C.dptr(lambda_p), C.dptr(lambda_m))
    return x, lambda_p, lambda_m


def hawkesjd_terminal_exact(params: C.HawkesParamsC, ttm: float, x, lambda_p, lambda_m, seed: int, slice_index: int, per_path: bool,
                            max_candidates: int = HAWKES_EXACT_DEFAULT_BUDGET, flags: int = 0):
    """the exact event-driven twin of hawkesjd_terminal over one interval of length ``ttm`` (b200sv_hawkesjd_terminal_exact), in place"""
    C.call("b200sv_hawkesjd_terminal_exact", byref(params), float(ttm), int(x.shape[0]), C.seed64(seed), int(flags), int(slice_index),
           1 if per_path else 0, int(max_candidates), C.dptr(x), C.dptr(lambda_p), C.dptr(lambda_m))
    return x, lambda_p, lambda_m


def hawkesjd_step_fixed(x, lambda_p, lambda_m, blocks, nb_steps: int, nb_path: int, dt: float, params: C.HawkesParamsC):
    """strict Hawkes stepper on caller-supplied draws ``blocks`` = (W0, U_P, U_M, J_P, J_M) (b200sv_hawkesjd_step_fixed), in place"""
    C.call("b200sv_hawkesjd_step_fixed", C.dptr(x), C.dptr(lambda_p), C.dptr(lambda_m), *map(C.dptr, blocks), nb_steps, nb_path, dt,
           byref(params))
    return x, lambda_p, lambda_m


def hawkesjd_device_draws(seed: int, path0: int, n: int, slice_index: int, nb_steps: int, dt: float, params: C.HawkesParamsC, flags: int):
    """[W0, U_P, U_M, J_P, J_M], each [nb_steps, n]: what the Hawkes stepper draws in-kernel (b200sv_hawkesjd_device_draws)"""
    out = [np.empty((nb_steps, n)) for _ in range(5)]
    C.call("b200sv_hawkesjd_device_draws", C.seed64(seed), int(path0), int(n), int(slice_index), nb_steps, dt, byref(params), flags,
           *map(C.dptr, out))
    return out


def _fixed_inputs(x0, v0, q0, W0, W1):
    """length-1 initial values broadcast like pricers/logsv_pricer.py:1007-1020 (x0 -> zeros, qvar0 -> zeros, sigma0 -> const)."""
    W0, W1 = C.f64(W0), C.f64(W1)
    if W0.ndim != 2 or W0.shape != W1.shape:
        raise ValueError("W0 and W1 must be 2-d arrays [nb_steps, nb_path] of the same shape")
    S, N = W0.shape

    def bcast(a, kind):
        a = np.atleast_1d(np.asarray(a, dtype=np.float64))
        if a.shape[0] == 1:
            return np.full(N, a[0]) if kind == "v" else np.zeros(N)
        assert a.shape[0] == N
        return np.array(a, dtype=np.float64, copy=True)

    return bcast(x0, "x"), bcast(v0, "v"), bcast(q0, "q"), W0, W1, S, N


def logsv_step_fixed(x0, sigma0, qvar0, W0, W1, dt: float, params: C.LogsvParamsC, eta: float, is_spot_measure: bool):
    x, s, q, W0, W1, S, N = _fixed_inputs(x0, sigma0, qvar0, W0, W1)
    C.call("b200sv_logsv_step_fixed", C.dptr(x), C.dptr(s), C.dptr(q), C.dptr(W0), C.dptr(W1), S, N, float(dt), byref(params),
           float(eta), int(bool(is_spot_measure)))
    return x, s, q


def heston_step_fixed(x0, var0, qvar0, W0, W1, dt: float, params: C.HestonParamsC):
    x, v, q, W0, W1, S, N = _fixed_inputs(x0, var0, qvar0, W0, W1)
    C.call("b200sv_heston_step_fixed", C.dptr(x), C.dptr(v), C.dptr(q), C.dptr(W0), C.dptr(W1), S, N, float(dt), byref(params))
    return x, v, q


def mc_payoffs(x, qvar, ttm, forward, strikes, optiontypes, discfactor=1.0, variable_type=VariableType.LOG_RETURN):
    vt = variable_code(variable_type)
    x = C.f64(x)
    q = C.f64(qvar) if qvar is not None else None
    strikes = C.f64(strikes)
    types = C.encode_types(optiontypes)
    J = strikes.shape[0]
    prices, stds = np.empty(J), np.empty(J)
    C.call("b200sv_mc_payoffs", C.dptr(x), C.dptr(q), x.shape[0], float(ttm), float(forward), C.dptr(strikes), C.i8ptr(types), J,
           float(discfactor), vt, C.dptr(prices), C.dptr(stds))
    return prices, stds


def device_normals(seed: int, path0: int, n: int, slice_idx: int, nsteps: int, flags: int):
    z0, z1 = np.empty((nsteps, n)), np.empty((nsteps, n))
    C.call("b200sv_device_normals", C.seed64(seed), int(path0), int(n), int(slice_idx), int(nsteps), int(flags), C.dptr(z0), C.dptr(z1))
    return z0, z1


def debug_exp_pair(L):
    L = C.f64(L)
    out = np.empty(2 * L.shape[0])
    C.call("b200sv_debug_exp_pair", C.dptr(L), L.shape[0], C.dptr(out))
    return out[0::2].copy(), out[1::2].copy()


def logsv_ode_terms(phi_grid, psi_grid, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, order: int):
    """dense (M [P,n,n,n], L [P,n,n], H [P,n]) of the coefficient ODEs over a transform grid (b200sv_logsv_ode_terms)."""
    phi = C.c128(np.atleast_1d(phi_grid))
    psi = None if psi_grid is None else C.c128(np.atleast_1d(psi_grid))
    P, n = phi.shape[0], (3 if order == 1 else 5)
    M, L, H = np.empty((P, n, n, n), np.complex128), np.empty((P, n, n), np.complex128), np.empty((P, n), np.complex128)
    C.call("b200sv_logsv_ode_terms", C.dptr(phi), C.dptr(psi), P, byref(params), float(eta), int(bool(is_spot_measure)),
           int(order), C.dptr(M), C.dptr(L), C.dptr(H))
    return M, L, H


def logsv_ode_rhs(phi_grid, psi_grid, A, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, order: int):
    """right-hand side A'MA + LA + H at A [P, n] through the production device function (b200sv_logsv_ode_rhs)."""
    phi, A = C.c128(np.atleast_1d(phi_grid)), C.c128(np.atleast_2d(A))
    psi = None if psi_grid is None else C.c128(np.atleast_1d(psi_grid))
    out = np.empty_like(A)
    C.call("b200sv_logsv_ode_rhs", C.dptr(phi), C.dptr(psi), phi.shape[0], C.dptr(A), byref(params), float(eta),
           int(bool(is_spot_measure)), int(order), C.dptr(out))
    return out


def ode_rhs_dense(A, M, L, H):
    """func_rhs with caller-supplied dense tensors: A [P, n] (or [n]) -> rhs of the same shape (b200sv_ode_rhs_dense)."""
    A0 = C.c128(A)
    A2, M, L, H = np.atleast_2d(A0), C.c128(M), C.c128(L), C.c128(H)
    n = A2.shape[1]
    if M.shape != (n, n, n) or L.shape != (n, n) or H.shape != (n,):
        raise ValueError("M, L, H must have shapes (n, n, n), (n, n), (n,)")
    out = np.empty_like(A2)
    C.call("b200sv_ode_rhs_dense", C.dptr(A2), A2.shape[0], n, C.dptr(M), C.dptr(L), C.dptr(H), C.dptr(out))
    return out.reshape(A0.shape)


def debug_exp_pair_scaled(Ls):
    """(exp(Ls ln2/256), exp(-Ls ln2/256)) through the variant the fp64 stepper runs on its table-unit log-vol state."""
    Ls = C.f64(Ls)
    out = np.empty(2 * Ls.shape[0])
    C.call("b200sv_debug_exp_pair_scaled", C.dptr(Ls), Ls.shape[0], C.dptr(out))
    return out[0::2].copy(), out[1::2].copy()


def debug_box_muller(words, flags: int):
    """the device Box-Muller on Philox output words [n, 4] (uint32) -> [n, 4] float64 normals (b200sv_debug_box_muller)."""
    w = np.ascontiguousarray(np.asarray(words, dtype=np.uint32).reshape(-1, 4))
    out = np.empty((w.shape[0], 4))
    C.call("b200sv_debug_box_muller", w.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), w.shape[0], int(flags), C.dptr(out))
    return out


def debug_fastmath(op: int, a, b=None):
    """op(a, b) through one of the fp64 device helpers, op = C.DEBUG_* (b200sv_debug_fastmath)."""
    a = C.f64(np.atleast_1d(a))
    b = None if b is None else C.f64(np.broadcast_to(b, a.shape))
    out = np.empty_like(a)
    C.call("b200sv_debug_fastmath", int(op), C.dptr(a), C.dptr(b), a.shape[0], C.dptr(out))
    return out


def debug_hawkes_clocks(words, lam, dt: float, params: C.HawkesParamsC):
    """the Hawkes stepper's jump-clock functions on 32-bit words against intensities (b200sv_debug_hawkes_clocks) -> [n, 6] float64:
    u, clock -ln(u)/dt, size_p, size_m, candidate flag, fused firing decision."""
    w = np.ascontiguousarray(np.asarray(words, dtype=np.uint32).ravel())
    lam = C.f64(np.broadcast_to(np.asarray(lam, dtype=np.float64), w.shape))
    out = np.empty((w.shape[0], 6))
    C.call("b200sv_debug_hawkes_clocks", w.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), C.dptr(lam), w.shape[0], float(dt), byref(params),
           C.dptr(out))
    return out


# ---- Fourier / MGF --------------------------------------------------------------------------------------------------------
def _check_fourier_types(optiontypes_ttms, is_spot_measure: bool):
    for types in optiontypes_ttms:
        for t in types:
            t = str(t)
            if t not in C.TYPE_CODES or (is_spot_measure and t in ("IC", "IP")):
                raise ValueError("not implemented")       # utils/mgf_pricer.py:206-219


def _check_qvar_types(optiontypes_ttms):
    for types in optiontypes_ttms:
        for t in types:
            if str(t) != "C":
                raise ValueError("not implemented")       # utils/mgf_pricer.py:349-358


def _price_chain(symbol: str, params, chain, etas, is_spot_measure: bool, head, variable_type: int, vol_scaler, max_phi, return_grids: bool,
                 coefs: Tuple[int, ...]):
    """the fused Fourier chain entry points: C arguments (params, chain block, *head, vol_scaler, max_phi, prices[, a [M, P, n] for n in
    ``coefs``], log_mgf [M, P])"""
    if variable_type == C.Q_VAR:
        _check_qvar_types(chain[4])
    else:
        _check_fourier_types(chain[4], is_spot_measure)
    max_phi = int(max_phi) if max_phi else (40000 if variable_type == C.Q_VAR else 1000)
    ch = _chain_arrays(*chain)
    etas = _backbone(etas, ch.M)
    prices = np.empty(ch.strikes.shape[0])
    grids = [np.empty((ch.M, max_phi, n), dtype=np.complex128) if return_grids else None for n in coefs]
    grids.append(np.empty((ch.M, max_phi), dtype=np.complex128) if return_grids else None)
    C.call(symbol, byref(params), *C.chain_ptrs(ch, *etas), *head, C.vol_scaler_arg(vol_scaler), max_phi, C.dptr(prices), *map(C.dptr, grids))
    out = C.split_chain(prices, ch.offsets)
    return (out, *grids) if return_grids else out


def logsv_price_chain(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                      is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                      max_phi: Optional[int] = None, return_grids: bool = False, variable_type: int = C.LOG_RETURN):
    return _price_chain("b200sv_logsv_price_chain", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (etas,),
                        is_spot_measure, (int(bool(is_spot_measure)), int(variable_type), int(expansion_order)), variable_type, vol_scaler,
                        max_phi, return_grids, (3 if expansion_order == C.ORDER_FIRST else 5,))


def heston_price_chain(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                       vol_scaler: Optional[float] = None, max_phi: Optional[int] = None, return_grids: bool = False,
                       variable_type: int = C.LOG_RETURN):
    return _price_chain("b200sv_heston_price_chain", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (), True,
                        (int(variable_type),), variable_type, vol_scaler, max_phi, return_grids, ())


def hawkesjd_price_chain(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, is_spot_measure: bool,
                         vol_scaler: Optional[float], max_phi: int, gamma: Optional[float], return_grids: bool = False):
    """Fourier prices of the Hawkes chain (b200sv_hawkesjd_price_chain), under the risk kernel exp(-gamma x) unless ``gamma`` is None.
    ``return_grids`` adds (a [M, P, 3], log_mgf [M, P], normalizers [M], gamma_forwards [M])."""
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = np.empty(ch.strikes.shape[0])
    a = np.empty((ch.M, max_phi, 3), dtype=np.complex128) if return_grids else None
    lm = np.empty((ch.M, max_phi), dtype=np.complex128) if return_grids else None
    norm, gfw = np.empty(ch.M), np.empty(ch.M)
    C.call("b200sv_hawkesjd_price_chain", byref(params), *C.chain_ptrs(ch), int(bool(is_spot_measure)), C.vol_scaler_arg(vol_scaler), max_phi,
           float("nan") if gamma is None else float(gamma), C.dptr(prices), C.dptr(a), C.dptr(lm), C.dptr(norm), C.dptr(gfw))
    out = C.split_chain(prices, ch.offsets)
    return (out, a, lm, norm, gfw) if return_grids else out


def _price_chain_greeks(symbol: str, params, chain, etas, is_spot_measure: bool, head, vol_scaler, max_phi: int, return_grids: bool, names,
                        with_nfev: bool, with_theta: bool = False):
    """the Fourier greeks entry points: C arguments (params, chain block, *head, vol_scaler, max_phi, prices, greeks [2 + P, J],
    dlog_mgf [P, M, max_phi][, nfev [max_phi]]) -> (prices per maturity, greeks, offsets[, dlog_mgf[, nfev]]).  ``with_theta``: the
    symbol's _theta twin, which also takes theta [J], dlog_mgf_theta [M, max_phi][, theta_nfev [max_phi]], returned after the rest as
    (theta[, dlog_mgf_theta[, theta_nfev]])"""
    _check_fourier_types(chain[4], is_spot_measure)
    ch = _chain_arrays(*chain)
    etas = _backbone(etas, ch.M)
    n, J = len(names), ch.strikes.shape[0]
    prices, greeks = np.empty(J), np.empty((2 + n, J))
    grids = (np.empty((n, ch.M, max_phi), dtype=np.complex128) if return_grids else None,)
    if with_nfev:
        grids += (np.empty(max_phi, dtype=np.int32) if return_grids else None,)
    theta_args, theta_out = (), ()
    if with_theta:
        symbol += "_theta"
        theta_out = (np.empty(J), np.empty((ch.M, max_phi), dtype=np.complex128) if return_grids else None)
        if with_nfev:
            theta_out += (np.empty(max_phi, dtype=np.int32) if return_grids else None,)
        theta_args = (C.dptr(theta_out[0]), C.dptr(theta_out[1]), *map(C.iptr, theta_out[2:]))
    C.call(symbol, byref(params), *C.chain_ptrs(ch, *etas), *head, C.vol_scaler_arg(vol_scaler), max_phi, C.dptr(prices), C.dptr(greeks),
           C.dptr(grids[0]), *map(C.iptr, grids[1:]), *theta_args)
    out = (C.split_chain(prices, ch.offsets), greeks, ch.offsets) + (grids if return_grids else ())
    return out + (theta_out if return_grids else theta_out[:1])


def logsv_price_chain_greeks(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                             is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                             max_phi: Optional[int] = None, return_grids: bool = False, with_theta: bool = False):
    """Fourier prices and forward-mode sensitivities of the chain (b200sv_logsv_price_chain_greeks).  Returns (prices per maturity,
    greeks [2 + 6, J], offsets) -- greeks rows: delta, gamma, then LOGSV_GREEK_PARAMS -- and with ``return_grids`` also
    (dlog_mgf [6, M, P], nfev [P]).  ``with_theta`` (b200sv_logsv_price_chain_greeks_theta, the rest bit for bit) appends theta [J] and,
    with ``return_grids``, (dlog_mgf_theta [M, P], theta_nfev [P])."""
    return _price_chain_greeks("b200sv_logsv_price_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (etas,),
                               is_spot_measure, (int(bool(is_spot_measure)), C.LOG_RETURN, int(expansion_order)), vol_scaler,
                               int(max_phi or 1000), return_grids, LOGSV_GREEK_PARAMS, True, with_theta)


def heston_price_chain_greeks(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                              vol_scaler: Optional[float] = None, max_phi: Optional[int] = None, return_grids: bool = False,
                              with_theta: bool = False):
    """Heston twin of logsv_price_chain_greeks (b200sv_heston_price_chain_greeks): greeks rows = delta, gamma, then HESTON_GREEK_PARAMS;
    ``return_grids`` adds dlog_mgf [5, M, P]; ``with_theta`` appends theta [J] (and dlog_mgf_theta [M, P] with ``return_grids``)."""
    return _price_chain_greeks("b200sv_heston_price_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (),
                               True, (C.LOG_RETURN,), vol_scaler, int(max_phi or 1000), return_grids, HESTON_GREEK_PARAMS, False, with_theta)


def _price_chain_hessian(symbol: str, params, chain, etas, is_spot_measure: bool, head, vol_scaler, max_phi: int, return_grids: bool, names,
                         with_nfev: bool):
    """the second-order Fourier entry points: the arguments of _price_chain_greeks, then vanna [P, J], hessian [P(P+1)/2, J],
    d2log_mgf [P(P+1)/2, M, max_phi] -> (prices per maturity, greeks, vanna, hessian, offsets[, dlog_mgf, d2log_mgf])"""
    _check_fourier_types(chain[4], is_spot_measure)
    ch = _chain_arrays(*chain)
    etas = _backbone(etas, ch.M)
    n, J = len(names), ch.strikes.shape[0]
    nh = n * (n + 1) // 2
    prices, greeks, vanna, hessian = np.empty(J), np.empty((2 + n, J)), np.empty((n, J)), np.empty((nh, J))
    dlm = np.empty((n, ch.M, max_phi), dtype=np.complex128) if return_grids else None
    d2lm = np.empty((nh, ch.M, max_phi), dtype=np.complex128) if return_grids else None
    C.call(symbol, byref(params), *C.chain_ptrs(ch, *etas), *head, C.vol_scaler_arg(vol_scaler), max_phi, C.dptr(prices), C.dptr(greeks),
           C.dptr(dlm), *((None,) if with_nfev else ()), C.dptr(vanna), C.dptr(hessian), C.dptr(d2lm))
    out = (C.split_chain(prices, ch.offsets), greeks, vanna, hessian, ch.offsets)
    return out + (dlm, d2lm) if return_grids else out


def logsv_price_chain_hessian(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                              is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                              max_phi: Optional[int] = None, return_grids: bool = False):
    """logsv_price_chain_greeks plus the second-order sensitivities (b200sv_logsv_price_chain_hessian).  Returns (prices per maturity,
    greeks [2 + 6, J], vanna [6, J], hessian [21, J], offsets): greeks as logsv_price_chain_greeks (bit for bit), vanna rows in
    LOGSV_GREEK_PARAMS order, hessian rows the upper triangle (p <= q) row-major in that order; ``return_grids`` adds
    (dlog_mgf [6, M, P], d2log_mgf [21, M, P])."""
    return _price_chain_hessian("b200sv_logsv_price_chain_hessian", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                (etas,), is_spot_measure, (int(bool(is_spot_measure)), C.LOG_RETURN, int(expansion_order)), vol_scaler,
                                int(max_phi or 1000), return_grids, LOGSV_GREEK_PARAMS, True)


def heston_price_chain_hessian(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                               vol_scaler: Optional[float] = None, max_phi: Optional[int] = None, return_grids: bool = False):
    """Heston twin of logsv_price_chain_hessian (b200sv_heston_price_chain_hessian): vanna [5, J], hessian [15, J] over
    HESTON_GREEK_PARAMS; ``return_grids`` adds (dlog_mgf [5, M, P], d2log_mgf [15, M, P])."""
    return _price_chain_hessian("b200sv_heston_price_chain_hessian", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                (), True, (C.LOG_RETURN,), vol_scaler, int(max_phi or 1000), return_grids, HESTON_GREEK_PARAMS, False)


def hawkesjd_price_chain_greeks(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                                is_spot_measure: bool = True, vol_scaler: Optional[float] = None, max_phi: Optional[int] = None,
                                return_grids: bool = False, with_theta: bool = False):
    """Hawkes twin of logsv_price_chain_greeks without a risk kernel (b200sv_hawkesjd_price_chain_greeks): greeks rows = delta, gamma, then
    HAWKES_GREEK_PARAMS; ``return_grids`` adds (dlog_mgf [15, M, P], nfev [P]).  P defaults to the route's 500 points.  ``with_theta`` as
    for logsv_price_chain_greeks."""
    return _price_chain_greeks("b200sv_hawkesjd_price_chain_greeks", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), (),
                               is_spot_measure, (int(bool(is_spot_measure)),), vol_scaler, int(max_phi or 500), return_grids,
                               HAWKES_GREEK_PARAMS, True, with_theta)


def hawkesjd_price_chain_hessian(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                                 is_spot_measure: bool = True, vol_scaler: Optional[float] = None, max_phi: Optional[int] = None,
                                 return_grids: bool = False):
    """hawkesjd_price_chain_greeks plus the second-order sensitivities (b200sv_hawkesjd_price_chain_hessian): vanna [15, J], hessian
    [120, J] over HAWKES_GREEK_PARAMS (upper triangle, row-major); ``return_grids`` adds (dlog_mgf [15, M, P], d2log_mgf [120, M, P]).
    P defaults to the route's 500 points."""
    return _price_chain_hessian("b200sv_hawkesjd_price_chain_hessian", params, (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms),
                                (), is_spot_measure, (int(bool(is_spot_measure)),), vol_scaler, int(max_phi or 500), return_grids,
                                HAWKES_GREEK_PARAMS, True)


def _hawkesjd_risk_premia(symbol: str, params, gamma: float, chain, vol_scaler, max_phi: Optional[int], return_grids: bool, second: bool):
    """the risk-kernel sensitivity entry points: C arguments (params, chain block, spot measure, vol_scaler, max_phi, gamma, prices,
    greeks [2 + n, J], dlog_mgf [n, M, P], dlog_norm [n, M, 2], nfev [P][, vanna [n, J], hessian [nh, J], d2log_mgf [nh, M, P],
    d2log_norm [nh, M, 2]]) -> (prices per maturity, greeks[, vanna, hessian], offsets) and with ``return_grids`` the grids in that order"""
    ch = _chain_arrays(*chain)
    max_phi, n, J = int(max_phi or 500), len(HAWKES_RISK_PREMIA_GREEK_PARAMS), ch.strikes.shape[0]
    nh = n * (n + 1) // 2
    prices, greeks = np.empty(J), np.empty((2 + n, J))
    rows = (np.empty((n, J)), np.empty((nh, J))) if second else ()
    grids = (np.empty((n, ch.M, max_phi), dtype=np.complex128), np.empty((n, ch.M, 2)), np.empty(max_phi, dtype=np.int32))
    if second:
        grids += (np.empty((nh, ch.M, max_phi), dtype=np.complex128), np.empty((nh, ch.M, 2)))
    if not return_grids:
        grids = (None,) * len(grids)
    C.call(symbol, byref(params), *C.chain_ptrs(ch), 1, C.vol_scaler_arg(vol_scaler), max_phi, float(gamma), C.dptr(prices),
           C.dptr(greeks), C.dptr(grids[0]), C.dptr(grids[1]), C.iptr(grids[2]), *map(C.dptr, rows), *map(C.dptr, grids[3:]))
    out = (C.split_chain(prices, ch.offsets), greeks, *rows, ch.offsets)
    return out + grids if return_grids else out


def hawkesjd_price_chain_risk_premia_greeks(params: C.HawkesParamsC, gamma: float, ttms, forwards, discfactors, strikes_ttms,
                                            optiontypes_ttms, vol_scaler: Optional[float] = None, max_phi: Optional[int] = None,
                                            return_grids: bool = False):
    """Fourier prices and forward-mode sensitivities of the Hawkes chain under the risk kernel exp(-gamma x)
    (b200sv_hawkesjd_price_chain_risk_premia_greeks; spot measure, calls and puts, DESIGN.md §4.12).  Returns (prices per maturity,
    greeks [18, J], offsets) -- greeks rows: delta, gamma, then HAWKES_RISK_PREMIA_GREEK_PARAMS -- and with ``return_grids`` also
    (dlog_mgf [16, M, P], dlog_norm [16, M, 2], nfev [P]); dlog_norm holds the derivatives of Re log-MGF at -gamma and -gamma - 1.  The
    prices are bit-identical to hawkesjd_price_chain with the same gamma.  P defaults to the route's 500 points."""
    return _hawkesjd_risk_premia("b200sv_hawkesjd_price_chain_risk_premia_greeks", params, gamma,
                                 (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), vol_scaler, max_phi, return_grids, False)


def hawkesjd_price_chain_risk_premia_hessian(params: C.HawkesParamsC, gamma: float, ttms, forwards, discfactors, strikes_ttms,
                                             optiontypes_ttms, vol_scaler: Optional[float] = None, max_phi: Optional[int] = None,
                                             return_grids: bool = False):
    """hawkesjd_price_chain_risk_premia_greeks plus the second-order sensitivities (b200sv_hawkesjd_price_chain_risk_premia_hessian,
    DESIGN.md §4.13): vanna [16, J] and hessian [136, J] over HAWKES_RISK_PREMIA_GREEK_PARAMS (upper triangle, row-major).  Returns
    (prices per maturity, greeks [18, J], vanna, hessian, offsets) and with ``return_grids`` also (dlog_mgf [16, M, P], dlog_norm [16, M, 2],
    nfev [P], d2log_mgf [136, M, P], d2log_norm [136, M, 2]); d2log_norm holds the second derivatives of Re log-MGF at -gamma and
    -gamma - 1.  The first-order outputs are bit-identical to hawkesjd_price_chain_risk_premia_greeks."""
    return _hawkesjd_risk_premia("b200sv_hawkesjd_price_chain_risk_premia_hessian", params, gamma,
                                 (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms), vol_scaler, max_phi, return_grids, True)


def logsv_price_chain_batch(params_list: Sequence[C.LogsvParamsC], ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                            is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                            max_phi: int = 1000, with_ivols: bool = True):
    """B parameter sets on one chain in one pass -> (prices [B, J], ivols [B, J] | None); ``etas`` is [B, M] or None."""
    _check_fourier_types(optiontypes_ttms, bool(is_spot_measure))
    return _chain_batch("b200sv_logsv_price_chain_batch", C.LogsvParamsC, params_list, (ttms, forwards, discfactors, strikes_ttms,
                        optiontypes_ttms), (etas,), (int(bool(is_spot_measure)), int(expansion_order), C.vol_scaler_arg(vol_scaler),
                        int(max_phi)), 1, with_ivols)


def heston_price_chain_batch(params_list: Sequence[C.HestonParamsC], ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                             vol_scaler: Optional[float] = None, max_phi: int = 1000, with_ivols: bool = True):
    """B Heston parameter sets on one chain in one pass -> (prices [B, J], ivols [B, J] | None)."""
    _check_fourier_types(optiontypes_ttms, True)
    return _chain_batch("b200sv_heston_price_chain_batch", C.HestonParamsC, params_list, (ttms, forwards, discfactors, strikes_ttms,
                        optiontypes_ttms), (), (C.vol_scaler_arg(vol_scaler), int(max_phi)), 1, with_ivols)


def _chains_batch(symbol: str, struct, params_list, chain_of_set, chains, etas, vol_scalers, is_spot_measure: bool, head, tail,
                  with_ivols: bool, lead=()):
    """the multi-chain batched entry points: C arguments (params [B], *lead, B, chain_of_set [B], K, Ms [K], concatenated ttms / forwards /
    discfactors, [etas,] per-chain offsets, strikes, types, *head, vol_scalers [K], *tail, prices, ivols | NULL) -> (prices, ivols | None),
    each a list of B rows, row b of length J of chain chain_of_set[b].  ``etas`` = (LogSV per-set backbones or None,) or ()."""
    B, K = len(params_list), len(chains)
    if B < 1 or K < 1:
        raise ValueError("need at least one parameter set and one chain")
    cos = np.asarray(chain_of_set)
    if cos.shape != (B,) or (B and cos.dtype.kind not in "iu"):
        raise ValueError(f"chain_of_set must hold {B} chain indices")
    if cos.min() < 0 or cos.max() >= K:
        raise ValueError(f"chain_of_set must lie in [0, {K})")
    cos = np.ascontiguousarray(cos, dtype=np.int32)
    if vol_scalers is None:
        vol_scalers = [None] * K
    if len(vol_scalers) != K:
        raise ValueError(f"vol_scalers must hold one value per chain ({K})")
    scalers = C.f64([C.vol_scaler_arg(v) for v in vol_scalers])
    chs = [_chain_arrays(*c) for c in chains]
    types = np.ascontiguousarray(np.concatenate([c.types for c in chs]), dtype=np.int8)
    if is_spot_measure and (types >= C.INV_CALL).any():
        raise ValueError("not implemented")       # _check_fourier_types on the encoded types (unknown codes raised in _chain_arrays)
    flat_etas = []
    for e in etas:
        if e is not None:
            if len(e) != B:
                raise ValueError(f"etas must hold one backbone per set ({B})")
            e = [C.f64(x) for x in e]
            if any(x.shape != (chs[k].M,) for x, k in zip(e, cos)):
                raise ValueError("etas[b] must hold one value per maturity of set b's chain")
            e = C.f64(np.concatenate(e))
        flat_etas.append(e)
    Ms = np.array([c.M for c in chs], dtype=np.int32)
    starts = np.cumsum([0] + [c.strikes.shape[0] for c in chs])
    offsets = np.ascontiguousarray(np.concatenate([c.offsets + s for c, s in zip(chs, starts)]), dtype=np.int32)
    cat = [C.f64(np.concatenate([getattr(c, f) for c in chs])) for f in ("ttms", "forwards", "discfactors", "strikes")]
    J = np.array([chs[k].strikes.shape[0] for k in cos])
    prices = np.empty(int(J.sum()))
    ivols = np.empty_like(prices) if with_ivols else None
    C.call(symbol, (struct * B)(*params_list), *lead, B, C.iptr(cos), K, C.iptr(Ms), *map(C.dptr, cat[:3]), *map(C.dptr, flat_etas),
           C.iptr(offsets), C.dptr(cat[3]), C.i8ptr(types), *head, C.dptr(scalers), *tail, C.dptr(prices), C.dptr(ivols))
    ends = np.cumsum(J).tolist()
    spans = list(zip([0] + ends[:-1], ends))
    return [prices[a:b] for a, b in spans], ([ivols[a:b] for a, b in spans] if with_ivols else None)


def logsv_price_chains_batch(params_list: Sequence[C.LogsvParamsC], chain_of_set, chains, etas=None, vol_scalers=None,
                             is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, max_phi: int = 1000, with_ivols: bool = True):
    """B parameter sets over K chains in one pass -> (prices, ivols | None), each a list of B rows in chain order.  ``chains[k]`` =
    (ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms); set b is priced on chains[chain_of_set[b]].  ``etas``: None or one vol
    backbone per set over its own chain's maturities; ``vol_scalers``: None or one per chain (None / <= 0: each set's default grid).  Row b
    is bit for bit row b of logsv_price_chain_batch on its chain with the sets of this call on that chain, in order."""
    return _chains_batch("b200sv_logsv_price_chains_batch", C.LogsvParamsC, params_list, chain_of_set, chains, (etas,), vol_scalers,
                         is_spot_measure, (int(bool(is_spot_measure)), int(expansion_order)), (int(max_phi),), with_ivols)


def heston_price_chains_batch(params_list: Sequence[C.HestonParamsC], chain_of_set, chains, vol_scalers=None, max_phi: int = 1000,
                              with_ivols: bool = True):
    """B Heston parameter sets over K chains in one pass -> (prices, ivols | None); arguments as logsv_price_chains_batch."""
    return _chains_batch("b200sv_heston_price_chains_batch", C.HestonParamsC, params_list, chain_of_set, chains, (), vol_scalers, True, (),
                         (int(max_phi),), with_ivols)


def hawkesjd_price_chain_batch(params_list: Sequence[C.HawkesParamsC], ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                               is_spot_measure: bool = True, vol_scaler: Optional[float] = None, max_phi: int = 500, gammas=None,
                               with_ivols: bool = True):
    """B Hawkes parameter sets on one chain in one pass -> (prices [B, J], ivols [B, J] | None).  ``gammas``: None (no risk kernel) or [B]
    risk_premia_gamma per set, every set then priced under its risk kernel.  Row b is bit-identical to hawkesjd_price_chain of set b."""
    if gammas is None:
        _check_fourier_types(optiontypes_ttms, bool(is_spot_measure))
    else:
        if not is_spot_measure or any(str(t) not in ("C", "P") for types in optiontypes_ttms for t in types):
            raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318
        gammas = C.f64(gammas)
        if gammas.shape != (len(params_list),):
            raise ValueError(f"gammas must have shape ({len(params_list)},)")
    return _chain_batch("b200sv_hawkesjd_price_chain_batch", C.HawkesParamsC, params_list, (ttms, forwards, discfactors, strikes_ttms,
                        optiontypes_ttms), (), (int(bool(is_spot_measure)), C.vol_scaler_arg(vol_scaler), int(max_phi), C.dptr(gammas)), 1,
                        with_ivols)


def hawkesjd_price_chains_batch(params_list: Sequence[C.HawkesParamsC], chain_of_set, chains, vol_scalers=None, is_spot_measure: bool = True,
                                max_phi: int = 500, with_ivols: bool = True, gammas=None):
    """B Hawkes parameter sets over K chains in one pass -> (prices, ivols | None); arguments as logsv_price_chains_batch.  ``gammas``: None
    (no risk kernel) or [B] risk_premia_gamma per set, every set then priced under its risk kernel (b200sv_hawkesjd_price_chains_batch_gamma).
    Row b is bit for bit row b of hawkesjd_price_chain_batch (with the same gammas) on its chain with the sets of this call on that chain,
    in order."""
    if gammas is not None:
        if not is_spot_measure or any(str(t) not in ("C", "P") for chain in chains for types in chain[4] for t in types):
            raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318
        gammas = C.f64(gammas)
        if gammas.shape != (len(params_list),):
            raise ValueError(f"gammas must have shape ({len(params_list)},)")
        return _chains_batch("b200sv_hawkesjd_price_chains_batch_gamma", C.HawkesParamsC, params_list, chain_of_set, chains, (), vol_scalers,
                             is_spot_measure, (int(bool(is_spot_measure)),), (int(max_phi),), with_ivols, lead=(C.dptr(gammas),))
    return _chains_batch("b200sv_hawkesjd_price_chains_batch", C.HawkesParamsC, params_list, chain_of_set, chains, (), vol_scalers,
                         is_spot_measure, (int(bool(is_spot_measure)),), (int(max_phi),), with_ivols)


def _logsv_mgf_grid(symbol: str, phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, expansion_order: int, args):
    """the three LogSV grid solvers: C arguments (phi, psi, P, dtau, a, params, *args, log_mgf) -> (a_t1 [P, n], log_mgf [P])"""
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    n = 3 if expansion_order == C.ORDER_FIRST else 5
    a = np.array(C.c128(a_t0), copy=True)
    if a.shape != (P, n):
        raise ValueError(f"a_t0 must have shape ({P}, {n})")
    lm = np.empty(P, dtype=np.complex128)
    C.call(symbol, C.dptr(phi), C.dptr(psi), P, float(dtau), C.dptr(a), byref(params), *args, C.dptr(lm))
    return a, lm


def logsv_mgf_grid(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, expansion_order: int):
    return _logsv_mgf_grid("b200sv_logsv_mgf_grid", phi, psi, dtau, a_t0, params, expansion_order,
                           (float(eta), int(bool(is_spot_measure)), int(expansion_order)))


def logsv_mgf_grid_bdf(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, expansion_order: int):
    """stiff branch (is_stiff_solver=True: SciPy's BDF control law) over a transform grid: (a_t1 [P, n], log_mgf [P])"""
    return _logsv_mgf_grid("b200sv_logsv_mgf_grid_bdf", phi, psi, dtau, a_t0, params, expansion_order,
                           (float(eta), int(bool(is_spot_measure)), int(expansion_order)))


def logsv_mgf_grid_analytic(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, is_spot_measure: bool, expansion_order: int, year_days: int = 260):
    """semi-analytic branch (is_analytic=True) over a transform grid: (a_t1 [P, n], log_mgf [P])"""
    return _logsv_mgf_grid("b200sv_logsv_mgf_grid_analytic", phi, psi, dtau, a_t0, params, expansion_order,
                           (int(bool(is_spot_measure)), int(expansion_order), int(year_days)))


def heston_mgf_grid(phi, psi, dtau: float, a_t0, b_t0, params: C.HestonParamsC):
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    a = np.array(C.c128(a_t0), copy=True) if a_t0 is not None else np.zeros(P, dtype=np.complex128)
    b = np.array(C.c128(b_t0), copy=True) if b_t0 is not None else np.zeros(P, dtype=np.complex128)
    lm = np.empty(P, dtype=np.complex128)
    C.call("b200sv_heston_mgf_grid", C.dptr(phi), C.dptr(psi), P, float(dtau), C.dptr(a), C.dptr(b), byref(params), C.dptr(lm))
    return lm, a, b


def hawkesjd_mgf_grid(phi, psi, dtau: float, a, params: C.HawkesParamsC):
    """Hawkes log-MGF over a transform grid (b200sv_hawkesjd_mgf_grid): complex128 ``a`` [P, 3] holds A(0) and receives A(dtau);
    returns log_mgf [P]"""
    lm = np.empty(phi.shape[0], dtype=np.complex128)
    C.call("b200sv_hawkesjd_mgf_grid", C.dptr(phi), C.dptr(psi), phi.shape[0], float(dtau), C.dptr(a), byref(params), C.dptr(lm))
    return lm


def fourier_vanilla(log_mgf, phi, forward, strikes, optiontypes, discfactor=1.0, is_spot_measure=True):
    _check_fourier_types([optiontypes], is_spot_measure)
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    J = strikes.shape[0]
    prices = np.empty(J)
    C.call("b200sv_fourier_vanilla", C.dptr(log_mgf), C.dptr(phi), phi.shape[0], float(forward),
           C.dptr(strikes), C.i8ptr(types), J, float(discfactor), int(bool(is_spot_measure)), C.dptr(prices))
    return prices


def fourier_gamma(log_mgf, phi, risk_premia_gamma, forward, normalizer, gamma_forward, strikes, optiontypes, is_spot_measure=True):
    if not is_spot_measure or any(str(t) not in ("C", "P") for t in optiontypes):
        raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_gamma", C.dptr(log_mgf), C.dptr(phi), phi.shape[0], float(risk_premia_gamma), float(forward),
           float(normalizer), float(gamma_forward), C.dptr(strikes), C.i8ptr(types), strikes.shape[0], 1, C.dptr(prices))
    return prices


def fourier_qvar(log_mgf, psi, ttm, strikes, optiontypes, discfactor=1.0):
    _check_qvar_types([optiontypes])
    log_mgf, psi, strikes = C.c128(log_mgf), C.c128(psi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_qvar", C.dptr(log_mgf), C.dptr(psi), psi.shape[0], float(ttm), C.dptr(strikes),
           C.i8ptr(types), strikes.shape[0], float(discfactor), C.dptr(prices))
    return prices


def fourier_pdf_sums(log_mgf, grid, z):
    log_mgf, grid, z = C.c128(log_mgf), C.c128(grid), C.f64(z)
    out = np.empty(z.shape[0])
    C.call("b200sv_fourier_pdf", C.dptr(log_mgf), C.dptr(grid), grid.shape[0], C.dptr(z), z.shape[0], C.dptr(out))
    return out


def fourier_digital(log_mgf, phi, forward, strikes, optiontypes, discfactor=1.0):
    for t in optiontypes:
        if str(t) not in ("C", "P"):
            raise ValueError("not implemented")           # utils/mgf_pricer.py:265-266
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_digital", C.dptr(log_mgf), C.dptr(phi), phi.shape[0], float(forward), C.dptr(strikes),
           C.i8ptr(types), strikes.shape[0], float(discfactor), C.dptr(prices))
    return prices


def bsm_implied_vols(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms):
    """Black-76 implied vols of a whole chain in one kernel launch."""
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = C.f64(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in prices_ttms]))
    if prices.shape[0] != ch.strikes.shape[0]:
        raise ValueError("model prices and strikes must have the same length")
    ivols = np.empty(ch.strikes.shape[0])
    C.call("b200sv_bsm_implied_vols", *C.chain_ptrs(ch), C.dptr(prices), C.dptr(ivols))
    return C.split_chain(ivols, ch.offsets)


def debug_bsm_implied_vols(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms):
    """bsm_implied_vols through the debug twin of its kernel -> (ivols, iterations), both flat in chain order (b200sv_debug_bsm_implied_vols)"""
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = C.f64(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in prices_ttms]))
    if prices.shape[0] != ch.strikes.shape[0]:
        raise ValueError("model prices and strikes must have the same length")
    ivols, iterations = np.empty(ch.strikes.shape[0]), np.empty(ch.strikes.shape[0], dtype=np.int32)
    C.call("b200sv_debug_bsm_implied_vols", *C.chain_ptrs(ch), C.dptr(prices), C.dptr(ivols), C.iptr(iterations))
    return ivols, iterations


def bsm_implied_vol_sensitivities(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms, greeks, vanna=None, hessian=None):
    """implied vols of the model prices and their sensitivities in one kernel launch (b200sv_bsm_implied_vol_sensitivities; DESIGN.md
    §4.6).  ``greeks`` [2 + P, J]: d price / d forward, d^2 price / d forward^2, d price / d p, as the *_price_chain_greeks entry points
    return it; ``vanna`` [P, J] and ``hessian`` [P(P+1)/2, J] as the *_price_chain_hessian ones do, both or neither.  Returns (ivols per
    maturity, ivol_greeks [2 + P, J], ivol_vanna [P, J] | None, ivol_hessian [P(P+1)/2, J] | None) -- the same derivatives of the implied
    vol; the ivols bit-identical to bsm_implied_vols."""
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = C.f64(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in prices_ttms]))
    J = ch.strikes.shape[0]
    if prices.shape[0] != J:
        raise ValueError("model prices and strikes must have the same length")
    greeks = C.f64(greeks)
    if greeks.ndim != 2 or greeks.shape[1] != J or not 1 <= greeks.shape[0] - 2 <= 15:
        raise ValueError(f"greeks must have shape (2 + P, {J}) with P in 1..15")
    P = greeks.shape[0] - 2
    if (vanna is None) != (hessian is None):
        raise ValueError("vanna and hessian are given together or not at all")
    second = vanna is not None
    if second:
        vanna, hessian = C.f64(vanna), C.f64(hessian)
        if vanna.shape != (P, J) or hessian.shape != (P * (P + 1) // 2, J):
            raise ValueError(f"vanna must have shape ({P}, {J}) and hessian ({P * (P + 1) // 2}, {J})")
    ivols, ivol_greeks = np.empty(J), np.empty((2 + P, J))
    ivol_vanna = np.empty((P, J)) if second else None
    ivol_hessian = np.empty((P * (P + 1) // 2, J)) if second else None
    C.call("b200sv_bsm_implied_vol_sensitivities", *C.chain_ptrs(ch), C.dptr(prices), P, C.dptr(greeks), C.dptr(vanna), C.dptr(hessian),
           C.dptr(ivols), C.dptr(ivol_greeks), C.dptr(ivol_vanna), C.dptr(ivol_hessian))
    return C.split_chain(ivols, ch.offsets), ivol_greeks, ivol_vanna, ivol_hessian


def bsm_implied_vol_theta(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms, theta):
    """implied vols of the model prices and their theta in one kernel launch (b200sv_bsm_implied_vol_theta; DESIGN.md §4.8).  ``theta`` [J]:
    -d price / d ttm as the *_price_chain_greeks entry points return it with ``with_theta``.  Returns (ivols per maturity, ivol_theta [J]) --
    -d ivol / d ttm at fixed forward and discount factor; the ivols bit-identical to bsm_implied_vols."""
    ch = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = C.f64(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in prices_ttms]))
    J = ch.strikes.shape[0]
    theta = C.f64(theta)
    if prices.shape[0] != J or theta.shape != (J,):
        raise ValueError(f"model prices and theta must have {J} entries, one per strike")
    ivols, ivol_theta = np.empty(J), np.empty(J)
    C.call("b200sv_bsm_implied_vol_theta", *C.chain_ptrs(ch), C.dptr(prices), C.dptr(theta), C.dptr(ivols), C.dptr(ivol_theta))
    return C.split_chain(ivols, ch.offsets), ivol_theta


def infer_bsm_ivols_from_model_chain_prices(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, model_prices_ttms):
    """the chain inversion the reference delegates to its third-party Black package (data/option_chain.py:340-345), keyword for keyword"""
    return bsm_implied_vols(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, model_prices_ttms)


def infer_bsm_ivols_from_slice_prices(ttm: float, forward: float, strikes, optiontypes, model_prices, discfactor: float = 1.0) -> np.ndarray:
    """Black-76 implied vols of one slice on the GPU (NaN where a price is outside the no-arbitrage bounds) -- the slice form of the same
    third-party call, used by ModelPricer.price_slice-style callers"""
    return bsm_implied_vols(np.array([ttm]), np.array([forward]), np.array([discfactor]), [np.asarray(strikes, dtype=np.float64)],
                            [np.asarray(optiontypes)], [np.asarray(model_prices, dtype=np.float64)])[0]


def logsv_vol_paths(params: C.LogsvParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, seed: int,
                    brownians=None):
    from .utils.funcs import set_time_grid
    nb_steps, _, grid_t = set_time_grid(ttm, nb_steps_per_year)
    if brownians is not None:
        brownians = C.f64(brownians)
        if brownians.shape != (nb_steps, nb_path):
            raise ValueError(f"brownians must have shape ({nb_steps}, {nb_path})")
    sigma_t = np.empty((nb_steps + 1, nb_path))
    C.call("b200sv_logsv_vol_paths", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)),
           C.seed64(seed), C.dptr(brownians), C.dptr(sigma_t))
    return sigma_t, grid_t
