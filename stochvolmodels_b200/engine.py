"""numpy <-> C-ABI marshalling for the host-level entry points of libb200sv (include/b200sv.h).

Thin by design: validation that the reference does in Python (exception classes, messages) lives here; all arithmetic is in
the CUDA library.  No function in this module computes a price on the CPU.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import byref
from typing import List, Optional, Sequence, Tuple

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


def _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms):
    ttms, forwards, discfactors = C.f64(ttms), C.f64(forwards), C.f64(discfactors)
    M = ttms.shape[0]
    if not (forwards.shape[0] == discfactors.shape[0] == len(strikes_ttms) == len(optiontypes_ttms) == M):
        raise ValueError("ttms, forwards, discfactors, strikes_ttms, and optiontypes_ttms must have the same length")
    offsets, strikes, types = C.flatten_chain(strikes_ttms, optiontypes_ttms)
    return M, ttms, forwards, discfactors, offsets, strikes, types


# ---- Monte Carlo --------------------------------------------------------------------------------------------------------
def logsv_mc_chain(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                   nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int
                   ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    vt = variable_code(variable_type)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    etas = C.f64(np.ones(M) if etas is None else etas)
    prices, stds = np.empty(strikes.shape[0]), np.empty(strikes.shape[0])
    C.call("b200sv_logsv_mc_chain", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.dptr(etas),
           C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)), vt,
           int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), C.dptr(prices), C.dptr(stds))
    return C.split_chain(prices, offsets), C.split_chain(stds, offsets)


def heston_mc_chain(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                    nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR
                    ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    vt = variable_code(variable_type)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices, stds = np.empty(strikes.shape[0]), np.empty(strikes.shape[0])
    C.call("b200sv_heston_mc_chain", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), int(nb_path), int(nb_steps_per_year), vt, int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags),
           int(scheme), C.dptr(prices), C.dptr(stds))
    return C.split_chain(prices, offsets), C.split_chain(stds, offsets)


LOGSV_GREEK_PARAMS = ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")
HESTON_GREEK_PARAMS = ("v0", "theta", "kappa", "rho", "volvol")
# HawkesJDParams fields in dataclass order without mu (the Fourier route never reads it) and risk_premia_gamma (not covered)
HAWKES_GREEK_PARAMS = ("sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p",
                       "lambda_m", "theta_m", "kappa_m", "beta1_m", "beta2_m")


def _greeks_result(prices, stds, greeks, greeks_se, offsets):
    """flat library outputs -> (prices, std errors, greeks [1+P, J], greeks_se [1+P, J], offsets)"""
    return C.split_chain(prices, offsets), C.split_chain(stds, offsets), greeks, greeks_se, offsets


def logsv_mc_chain_greeks(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                          nb_steps_per_year: int, is_spot_measure: bool, variable_type, seed: int, flags: int):
    """prices, std errors and pathwise sensitivities of the chain in one pass (b200sv_logsv_mc_chain_greeks).  Returns (prices, std errors,
    greeks [1+6, J], greeks_se [1+6, J], offsets): row 0 the forward delta, then LOGSV_GREEK_PARAMS; J runs over the flattened chain."""
    vt = variable_code(variable_type)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    etas = C.f64(np.ones(M) if etas is None else etas)
    J = strikes.shape[0]
    prices, stds = np.empty(J), np.empty(J)
    greeks, greeks_se = np.empty((1 + len(LOGSV_GREEK_PARAMS), J)), np.empty((1 + len(LOGSV_GREEK_PARAMS), J))
    C.call("b200sv_logsv_mc_chain_greeks", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.dptr(etas),
           C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)), vt,
           int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), C.dptr(prices), C.dptr(stds), C.dptr(greeks), C.dptr(greeks_se))
    return _greeks_result(prices, stds, greeks, greeks_se, offsets)


def heston_mc_chain_greeks(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int,
                           nb_steps_per_year: int, variable_type, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR):
    """Heston twin of logsv_mc_chain_greeks (b200sv_heston_mc_chain_greeks): greeks rows = forward delta, then HESTON_GREEK_PARAMS."""
    vt = variable_code(variable_type)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    J = strikes.shape[0]
    prices, stds = np.empty(J), np.empty(J)
    greeks, greeks_se = np.empty((1 + len(HESTON_GREEK_PARAMS), J)), np.empty((1 + len(HESTON_GREEK_PARAMS), J))
    C.call("b200sv_heston_mc_chain_greeks", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), int(nb_path), int(nb_steps_per_year), vt, int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags),
           int(scheme), C.dptr(prices), C.dptr(stds), C.dptr(greeks), C.dptr(greeks_se))
    return _greeks_result(prices, stds, greeks, greeks_se, offsets)


def logsv_tangent_terminal(params: C.LogsvParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                           seed: int, flags: int, slice_index: int = 0, path_offset: int = 0):
    """one slice of the tangent stepper from (0, sigma0, 0): (x, sigma, qvar, dx [6, n], dsigma [6, n], dqvar [6, n])"""
    P = len(LOGSV_GREEK_PARAMS)
    x, s, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    dx, ds, dq = np.empty((P, nb_path)), np.empty((P, nb_path)), np.empty((P, nb_path))
    C.call("b200sv_logsv_tangent_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)),
           float(eta), int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), int(slice_index), int(path_offset), C.dptr(x), C.dptr(s), C.dptr(q),
           C.dptr(dx), C.dptr(ds), C.dptr(dq))
    return x, s, q, dx, ds, dq


def heston_tangent_terminal(params: C.HestonParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, seed: int, flags: int,
                            slice_index: int = 0, path_offset: int = 0):
    """one slice of the Heston tangent stepper from (0, v0, 0): (x, var, qvar, dx [5, n], dvar [5, n], dqvar [5, n])"""
    P = len(HESTON_GREEK_PARAMS)
    x, v, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    dx, dv, dq = np.empty((P, nb_path)), np.empty((P, nb_path)), np.empty((P, nb_path))
    C.call("b200sv_heston_tangent_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), int(seed) & 0xFFFFFFFFFFFFFFFF,
           int(flags), int(slice_index), int(path_offset), C.dptr(x), C.dptr(v), C.dptr(q), C.dptr(dx), C.dptr(dv), C.dptr(dq))
    return x, v, q, dx, dv, dq


def logsv_mc_chain_batch(params_list: Sequence[C.LogsvParamsC], ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                         nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, seed: int, flags: int, with_ivols: bool = True):
    """B parameter sets through the fused chain MC on the SAME seed in one call -> (prices, std errors, ivols | None), each [B, J]."""
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    B = len(params_list)
    arr = (C.LogsvParamsC * B)(*params_list)
    etas_c = None
    if etas is not None:
        etas_c = np.ascontiguousarray(etas, dtype=np.float64)
        if etas_c.shape != (B, M):
            raise ValueError(f"etas must have shape ({B}, {M})")
    J = strikes.shape[0]
    prices, stds = np.empty((B, J)), np.empty((B, J))
    ivols = np.empty((B, J)) if with_ivols else None
    C.call("b200sv_logsv_mc_chain_batch", arr, B, M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors),
           C.dptr(etas_c) if etas_c is not None else None, C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(nb_path),
           int(nb_steps_per_year), int(bool(is_spot_measure)), int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), C.dptr(prices), C.dptr(stds),
           C.dptr(ivols) if with_ivols else None)
    return prices, stds, ivols


def heston_mc_chain_batch(params_list: Sequence[C.HestonParamsC], ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                          nb_path: int, nb_steps_per_year: int, seed: int, flags: int, scheme: int = C.HESTON_EULER_FLOOR,
                          with_ivols: bool = True):
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    B = len(params_list)
    arr = (C.HestonParamsC * B)(*params_list)
    J = strikes.shape[0]
    prices, stds = np.empty((B, J)), np.empty((B, J))
    ivols = np.empty((B, J)) if with_ivols else None
    C.call("b200sv_heston_mc_chain_batch", arr, B, M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets), C.dptr(strikes),
           C.i8ptr(types), int(nb_path), int(nb_steps_per_year), int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), int(scheme), C.dptr(prices),
           C.dptr(stds), C.dptr(ivols) if with_ivols else None)
    return prices, stds, ivols


def rough_logsv_mc_chain(params_list, weights, nodes, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, nb_path: int, nsteps, hs,
                         Z0=None, Z1=None, variable_type=1, seed: int = 0, flags: int = 0, with_ivols: bool = False, return_states: bool = False):
    """B parameter sets through the rough-LogSV multi-factor chain MC (b200sv_rough_logsv_mc_chain).  ``weights`` / ``nodes``: [n] (shared)
    or [B, n]; ``Z0`` / ``Z1``: host unit normals [rows >= max(nsteps), nb_path] or None (in-kernel Philox draws).
    Returns (prices [B, J], std [B, J], ivols [B, J] | None, states [M, n + 2, nb_path] | None)."""
    vt = variable_code(variable_type)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
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
    J = strikes.shape[0]
    prices, stds = np.empty((B, J)), np.empty((B, J))
    ivols = np.empty((B, J)) if with_ivols else None
    states = np.empty((M, n + 2, int(nb_path))) if return_states else None
    C.call("b200sv_rough_logsv_mc_chain", arr, B, n, C.dptr(weights), C.dptr(nodes), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors),
           C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(nb_path), nsteps.ctypes.data_as(C._ip), C.dptr(hs),
           C.dptr(Z0) if Z0 is not None else None, C.dptr(Z1) if Z1 is not None else None, int(z_rows), vt, int(seed) & 0xFFFFFFFFFFFFFFFF,
           int(flags), C.dptr(prices), C.dptr(stds), C.dptr(ivols) if with_ivols else None, C.dptr(states) if return_states else None)
    return prices, stds, ivols, states, offsets


def logsv_terminal(params: C.LogsvParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                   seed: int, flags: int):
    x, s, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    C.call("b200sv_logsv_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year), int(bool(is_spot_measure)),
           float(eta), int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), C.dptr(x), C.dptr(s), C.dptr(q))
    return x, s, q


def logsv_terminal_from_state(params: C.LogsvParamsC, x0, sigma0, qvar0, ttm: float, nb_steps_per_year: int, is_spot_measure: bool, eta: float,
                              seed: int, flags: int, slice_index: int = 0):
    """fused Philox stepper from PER-PATH initial arrays (b200sv_logsv_terminal_from_state); returns fresh (x, sigma, qvar) arrays."""
    x, s, q = (np.array(a, dtype=np.float64, copy=True, order="C") for a in (x0, sigma0, qvar0))
    if not (x.shape == s.shape == q.shape and x.ndim == 1):
        raise ValueError("x0, sigma0, qvar0 must be 1-d arrays of one length")
    C.call("b200sv_logsv_terminal_from_state", byref(params), float(ttm), int(x.shape[0]), int(nb_steps_per_year), int(bool(is_spot_measure)),
           float(eta), int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), int(slice_index), C.dptr(x), C.dptr(s), C.dptr(q))
    return x, s, q


def set_stream(stream) -> None:
    """CUDA stream (int / ctypes pointer / torch.cuda.Stream) for this thread's host-level library calls; None = the default stream."""
    ptr = getattr(stream, "cuda_stream", stream)
    C.call("b200sv_set_stream", ptr)


def heston_terminal(params: C.HestonParamsC, ttm: float, nb_path: int, nb_steps_per_year: int, seed: int, flags: int,
                    scheme: int = C.HESTON_EULER_FLOOR):
    x, v, q = np.empty(nb_path), np.empty(nb_path), np.empty(nb_path)
    C.call("b200sv_heston_terminal", byref(params), float(ttm), int(nb_path), int(nb_steps_per_year),
           int(seed) & 0xFFFFFFFFFFFFFFFF, int(flags), int(scheme), C.dptr(x), C.dptr(v), C.dptr(q))
    return x, v, q


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
    C.call("b200sv_device_normals", int(seed) & 0xFFFFFFFFFFFFFFFF, int(path0), int(n), int(slice_idx), int(nsteps), int(flags),
           C.dptr(z0), C.dptr(z1))
    return z0, z1


def debug_exp_pair(L):
    L = C.f64(L)
    out = np.empty(2 * L.shape[0])
    C.call("b200sv_debug_exp_pair", C.dptr(L), L.shape[0], C.dptr(out))
    return out[0::2].copy(), out[1::2].copy()


def _c128(a):
    return np.ascontiguousarray(a, dtype=np.complex128)


def logsv_ode_terms(phi_grid, psi_grid, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, order: int):
    """dense (M [P,n,n,n], L [P,n,n], H [P,n]) of the coefficient ODEs over a transform grid (b200sv_logsv_ode_terms)."""
    phi = _c128(np.atleast_1d(phi_grid))
    psi = None if psi_grid is None else _c128(np.atleast_1d(psi_grid))
    P, n = phi.shape[0], (3 if order == 1 else 5)
    M, L, H = np.empty((P, n, n, n), np.complex128), np.empty((P, n, n), np.complex128), np.empty((P, n), np.complex128)
    as_d = lambda a: a.view(np.float64).ctypes.data_as(C._dp)
    C.call("b200sv_logsv_ode_terms", as_d(phi), as_d(psi) if psi is not None else None, P, byref(params), float(eta), int(bool(is_spot_measure)),
           int(order), as_d(M), as_d(L), as_d(H))
    return M, L, H


def logsv_ode_rhs(phi_grid, psi_grid, A, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, order: int):
    """right-hand side A'MA + LA + H at A [P, n] through the production device function (b200sv_logsv_ode_rhs)."""
    phi, A = _c128(np.atleast_1d(phi_grid)), _c128(np.atleast_2d(A))
    psi = None if psi_grid is None else _c128(np.atleast_1d(psi_grid))
    out = np.empty_like(A)
    as_d = lambda a: a.view(np.float64).ctypes.data_as(C._dp)
    C.call("b200sv_logsv_ode_rhs", as_d(phi), as_d(psi) if psi is not None else None, phi.shape[0], as_d(A), byref(params), float(eta),
           int(bool(is_spot_measure)), int(order), as_d(out))
    return out


def ode_rhs_dense(A, M, L, H):
    """func_rhs with caller-supplied dense tensors: A [P, n] (or [n]) -> rhs of the same shape (b200sv_ode_rhs_dense)."""
    A0 = _c128(A)
    A2, M, L, H = np.atleast_2d(A0), _c128(M), _c128(L), _c128(H)
    n = A2.shape[1]
    if M.shape != (n, n, n) or L.shape != (n, n) or H.shape != (n,):
        raise ValueError("M, L, H must have shapes (n, n, n), (n, n), (n,)")
    out = np.empty_like(A2)
    as_d = lambda a: a.view(np.float64).ctypes.data_as(C._dp)
    C.call("b200sv_ode_rhs_dense", as_d(A2), A2.shape[0], n, as_d(M), as_d(L), as_d(H), as_d(out))
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


def logsv_price_chain(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                      is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                      max_phi: Optional[int] = None, return_grids: bool = False, variable_type: int = C.LOG_RETURN):
    if variable_type == C.Q_VAR:
        _check_qvar_types(optiontypes_ttms)
    else:
        _check_fourier_types(optiontypes_ttms, is_spot_measure)
    max_phi = int(max_phi) if max_phi else (40000 if variable_type == C.Q_VAR else 1000)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    etas = C.f64(np.ones(M) if etas is None else etas)
    n = 3 if expansion_order == C.ORDER_FIRST else 5
    prices = np.empty(strikes.shape[0])
    a_out = np.empty((M, max_phi, n), dtype=np.complex128) if return_grids else None
    lm_out = np.empty((M, max_phi), dtype=np.complex128) if return_grids else None
    C.call("b200sv_logsv_price_chain", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.dptr(etas),
           C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(bool(is_spot_measure)), int(variable_type), int(expansion_order),
           float(vol_scaler) if vol_scaler is not None else -1.0, int(max_phi), C.dptr(prices),
           a_out.ctypes.data_as(C._dp) if return_grids else None, lm_out.ctypes.data_as(C._dp) if return_grids else None)
    out = C.split_chain(prices, offsets)
    return (out, a_out, lm_out) if return_grids else out


def heston_price_chain(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                       vol_scaler: Optional[float] = None, max_phi: Optional[int] = None, return_grids: bool = False,
                       variable_type: int = C.LOG_RETURN):
    if variable_type == C.Q_VAR:
        _check_qvar_types(optiontypes_ttms)
    else:
        _check_fourier_types(optiontypes_ttms, True)
    max_phi = int(max_phi) if max_phi else (40000 if variable_type == C.Q_VAR else 1000)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = np.empty(strikes.shape[0])
    lm_out = np.empty((M, max_phi), dtype=np.complex128) if return_grids else None
    C.call("b200sv_heston_price_chain", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), int(variable_type), float(vol_scaler) if vol_scaler is not None else -1.0, int(max_phi),
           C.dptr(prices), lm_out.ctypes.data_as(C._dp) if return_grids else None)
    out = C.split_chain(prices, offsets)
    return (out, lm_out) if return_grids else out


def logsv_price_chain_greeks(params: C.LogsvParamsC, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                             is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                             max_phi: Optional[int] = None, return_grids: bool = False):
    """Fourier prices and forward-mode sensitivities of the chain (b200sv_logsv_price_chain_greeks).  Returns (prices per maturity,
    greeks [2 + 6, J], offsets) -- greeks rows: delta, gamma, then LOGSV_GREEK_PARAMS -- and with ``return_grids`` also
    (dlog_mgf [6, M, P], nfev [P])."""
    _check_fourier_types(optiontypes_ttms, is_spot_measure)
    max_phi = int(max_phi) if max_phi else 1000
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    etas = C.f64(np.ones(M) if etas is None else etas)
    n = len(LOGSV_GREEK_PARAMS)
    prices, greeks = np.empty(strikes.shape[0]), np.empty((2 + n, strikes.shape[0]))
    dlm = np.empty((n, M, max_phi), dtype=np.complex128) if return_grids else None
    nfev = np.empty(max_phi, dtype=np.int32) if return_grids else None
    C.call("b200sv_logsv_price_chain_greeks", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.dptr(etas),
           C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(bool(is_spot_measure)), C.LOG_RETURN, int(expansion_order),
           float(vol_scaler) if vol_scaler is not None else -1.0, max_phi, C.dptr(prices), C.dptr(greeks),
           dlm.ctypes.data_as(C._dp) if return_grids else None, C.iptr(nfev) if return_grids else None)
    out = (C.split_chain(prices, offsets), greeks, offsets)
    return out + (dlm, nfev) if return_grids else out


def heston_price_chain_greeks(params: C.HestonParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                              vol_scaler: Optional[float] = None, max_phi: Optional[int] = None, return_grids: bool = False):
    """Heston twin of logsv_price_chain_greeks (b200sv_heston_price_chain_greeks): greeks rows = delta, gamma, then HESTON_GREEK_PARAMS;
    ``return_grids`` adds dlog_mgf [5, M, P]."""
    _check_fourier_types(optiontypes_ttms, True)
    max_phi = int(max_phi) if max_phi else 1000
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    n = len(HESTON_GREEK_PARAMS)
    prices, greeks = np.empty(strikes.shape[0]), np.empty((2 + n, strikes.shape[0]))
    dlm = np.empty((n, M, max_phi), dtype=np.complex128) if return_grids else None
    C.call("b200sv_heston_price_chain_greeks", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), C.LOG_RETURN, float(vol_scaler) if vol_scaler is not None else -1.0, max_phi, C.dptr(prices),
           C.dptr(greeks), dlm.ctypes.data_as(C._dp) if return_grids else None)
    out = (C.split_chain(prices, offsets), greeks, offsets)
    return out + (dlm,) if return_grids else out


def hawkesjd_price_chain_greeks(params: C.HawkesParamsC, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                                is_spot_measure: bool = True, vol_scaler: Optional[float] = None, max_phi: Optional[int] = None,
                                return_grids: bool = False):
    """Hawkes twin of logsv_price_chain_greeks without a risk kernel (b200sv_hawkesjd_price_chain_greeks): greeks rows = delta, gamma, then
    HAWKES_GREEK_PARAMS; ``return_grids`` adds (dlog_mgf [15, M, P], nfev [P]).  P defaults to the route's 500 points."""
    _check_fourier_types(optiontypes_ttms, is_spot_measure)
    max_phi = int(max_phi) if max_phi else 500
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    n = len(HAWKES_GREEK_PARAMS)
    prices, greeks = np.empty(strikes.shape[0]), np.empty((2 + n, strikes.shape[0]))
    dlm = np.empty((n, M, max_phi), dtype=np.complex128) if return_grids else None
    nfev = np.empty(max_phi, dtype=np.int32) if return_grids else None
    C.call("b200sv_hawkesjd_price_chain_greeks", byref(params), M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), int(bool(is_spot_measure)), float(vol_scaler) if vol_scaler is not None else 0.0, max_phi,
           C.dptr(prices), C.dptr(greeks), dlm.ctypes.data_as(C._dp) if return_grids else None, C.iptr(nfev) if return_grids else None)
    out = (C.split_chain(prices, offsets), greeks, offsets)
    return out + (dlm, nfev) if return_grids else out


def logsv_price_chain_batch(params_list: Sequence[C.LogsvParamsC], ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms,
                            is_spot_measure: bool = True, expansion_order: int = C.ORDER_SECOND, vol_scaler: Optional[float] = None,
                            max_phi: int = 1000, with_ivols: bool = True):
    """B parameter sets on one chain in one pass -> (prices [B, J], ivols [B, J] | None); ``etas`` is [B, M] or None."""
    _check_fourier_types(optiontypes_ttms, bool(is_spot_measure))
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    B = len(params_list)
    arr = (C.LogsvParamsC * B)(*params_list)
    etas_c = None
    if etas is not None:
        etas_c = np.ascontiguousarray(etas, dtype=np.float64)
        if etas_c.shape != (B, M):
            raise ValueError(f"etas must have shape ({B}, {M})")
    prices = np.empty((B, strikes.shape[0]))
    ivols = np.empty((B, strikes.shape[0])) if with_ivols else None
    C.call("b200sv_logsv_price_chain_batch", arr, B, M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors),
           C.dptr(etas_c) if etas_c is not None else None, C.iptr(offsets), C.dptr(strikes), C.i8ptr(types), int(bool(is_spot_measure)),
           int(expansion_order), float(vol_scaler) if vol_scaler is not None else -1.0, int(max_phi), C.dptr(prices),
           C.dptr(ivols) if with_ivols else None)
    return prices, ivols


def heston_price_chain_batch(params_list: Sequence[C.HestonParamsC], ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms,
                             vol_scaler: Optional[float] = None, max_phi: int = 1000, with_ivols: bool = True):
    """B Heston parameter sets on one chain in one pass -> (prices [B, J], ivols [B, J] | None)."""
    _check_fourier_types(optiontypes_ttms, True)
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    B = len(params_list)
    arr = (C.HestonParamsC * B)(*params_list)
    prices = np.empty((B, strikes.shape[0]))
    ivols = np.empty((B, strikes.shape[0])) if with_ivols else None
    C.call("b200sv_heston_price_chain_batch", arr, B, M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets),
           C.dptr(strikes), C.i8ptr(types), float(vol_scaler) if vol_scaler is not None else -1.0, int(max_phi), C.dptr(prices),
           C.dptr(ivols) if with_ivols else None)
    return prices, ivols


def logsv_mgf_grid(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, expansion_order: int):
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    n = 3 if expansion_order == C.ORDER_FIRST else 5
    a = np.array(C.c128(a_t0), copy=True)
    if a.shape != (P, n):
        raise ValueError(f"a_t0 must have shape ({P}, {n})")
    lm = np.empty(P, dtype=np.complex128)
    C.call("b200sv_logsv_mgf_grid", phi.ctypes.data_as(C._dp), psi.ctypes.data_as(C._dp) if psi is not None else None, P, float(dtau),
           a.ctypes.data_as(C._dp), byref(params), float(eta), int(bool(is_spot_measure)), int(expansion_order), lm.ctypes.data_as(C._dp))
    return a, lm


def logsv_mgf_grid_bdf(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, eta: float, is_spot_measure: bool, expansion_order: int):
    """stiff branch (is_stiff_solver=True: SciPy's BDF control law) over a transform grid: (a_t1 [P, n], log_mgf [P])"""
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    n = 3 if expansion_order == C.ORDER_FIRST else 5
    a = np.array(C.c128(a_t0), copy=True)
    if a.shape != (P, n):
        raise ValueError(f"a_t0 must have shape ({P}, {n})")
    lm = np.empty(P, dtype=np.complex128)
    C.call("b200sv_logsv_mgf_grid_bdf", phi.ctypes.data_as(C._dp), psi.ctypes.data_as(C._dp) if psi is not None else None, P, float(dtau),
           a.ctypes.data_as(C._dp), byref(params), float(eta), int(bool(is_spot_measure)), int(expansion_order), lm.ctypes.data_as(C._dp))
    return a, lm


def logsv_mgf_grid_analytic(phi, psi, dtau: float, a_t0, params: C.LogsvParamsC, is_spot_measure: bool, expansion_order: int, year_days: int = 260):
    """semi-analytic branch (is_analytic=True) over a transform grid: (a_t1 [P, n], log_mgf [P])"""
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    n = 3 if expansion_order == C.ORDER_FIRST else 5
    a = np.array(C.c128(a_t0), copy=True)
    if a.shape != (P, n):
        raise ValueError(f"a_t0 must have shape ({P}, {n})")
    lm = np.empty(P, dtype=np.complex128)
    C.call("b200sv_logsv_mgf_grid_analytic", phi.ctypes.data_as(C._dp), psi.ctypes.data_as(C._dp) if psi is not None else None, P, float(dtau),
           a.ctypes.data_as(C._dp), byref(params), int(bool(is_spot_measure)), int(expansion_order), int(year_days), lm.ctypes.data_as(C._dp))
    return a, lm


def heston_mgf_grid(phi, psi, dtau: float, a_t0, b_t0, params: C.HestonParamsC):
    phi = C.c128(phi)
    psi = C.c128(psi) if psi is not None else None
    P = phi.shape[0]
    a = np.array(C.c128(a_t0), copy=True) if a_t0 is not None else np.zeros(P, dtype=np.complex128)
    b = np.array(C.c128(b_t0), copy=True) if b_t0 is not None else np.zeros(P, dtype=np.complex128)
    lm = np.empty(P, dtype=np.complex128)
    C.call("b200sv_heston_mgf_grid", phi.ctypes.data_as(C._dp), psi.ctypes.data_as(C._dp) if psi is not None else None, P, float(dtau),
           a.ctypes.data_as(C._dp), b.ctypes.data_as(C._dp), byref(params), lm.ctypes.data_as(C._dp))
    return lm, a, b


def fourier_vanilla(log_mgf, phi, forward, strikes, optiontypes, discfactor=1.0, is_spot_measure=True):
    _check_fourier_types([optiontypes], is_spot_measure)
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    J = strikes.shape[0]
    prices = np.empty(J)
    C.call("b200sv_fourier_vanilla", log_mgf.ctypes.data_as(C._dp), phi.ctypes.data_as(C._dp), phi.shape[0], float(forward),
           C.dptr(strikes), C.i8ptr(types), J, float(discfactor), int(bool(is_spot_measure)), C.dptr(prices))
    return prices


def fourier_gamma(log_mgf, phi, risk_premia_gamma, forward, normalizer, gamma_forward, strikes, optiontypes, is_spot_measure=True):
    if not is_spot_measure or any(str(t) not in ("C", "P") for t in optiontypes):
        raise ValueError("not implemented")           # utils/mgf_pricer.py:310-318
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_gamma", log_mgf.ctypes.data_as(C._dp), phi.ctypes.data_as(C._dp), phi.shape[0], float(risk_premia_gamma), float(forward),
           float(normalizer), float(gamma_forward), C.dptr(strikes), C.i8ptr(types), strikes.shape[0], 1, C.dptr(prices))
    return prices


def fourier_qvar(log_mgf, psi, ttm, strikes, optiontypes, discfactor=1.0):
    _check_qvar_types([optiontypes])
    log_mgf, psi, strikes = C.c128(log_mgf), C.c128(psi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_qvar", log_mgf.ctypes.data_as(C._dp), psi.ctypes.data_as(C._dp), psi.shape[0], float(ttm), C.dptr(strikes),
           C.i8ptr(types), strikes.shape[0], float(discfactor), C.dptr(prices))
    return prices


def fourier_pdf_sums(log_mgf, grid, z):
    log_mgf, grid, z = C.c128(log_mgf), C.c128(grid), C.f64(z)
    out = np.empty(z.shape[0])
    C.call("b200sv_fourier_pdf", log_mgf.ctypes.data_as(C._dp), grid.ctypes.data_as(C._dp), grid.shape[0], C.dptr(z), z.shape[0], C.dptr(out))
    return out


def fourier_digital(log_mgf, phi, forward, strikes, optiontypes, discfactor=1.0):
    for t in optiontypes:
        if str(t) not in ("C", "P"):
            raise ValueError("not implemented")           # utils/mgf_pricer.py:265-266
    log_mgf, phi, strikes = C.c128(log_mgf), C.c128(phi), C.f64(strikes)
    types = C.encode_types(optiontypes)
    prices = np.empty(strikes.shape[0])
    C.call("b200sv_fourier_digital", log_mgf.ctypes.data_as(C._dp), phi.ctypes.data_as(C._dp), phi.shape[0], float(forward), C.dptr(strikes),
           C.i8ptr(types), strikes.shape[0], float(discfactor), C.dptr(prices))
    return prices


def bsm_implied_vols(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, prices_ttms):
    """Black-76 implied vols of a whole chain in one kernel launch."""
    M, ttms, forwards, discfactors, offsets, strikes, types = _chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    prices = C.f64(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in prices_ttms]))
    if prices.shape[0] != strikes.shape[0]:
        raise ValueError("model prices and strikes must have the same length")
    ivols = np.empty(strikes.shape[0])
    C.call("b200sv_bsm_implied_vols", M, C.dptr(ttms), C.dptr(forwards), C.dptr(discfactors), C.iptr(offsets), C.dptr(strikes),
           C.i8ptr(types), C.dptr(prices), C.dptr(ivols))
    return C.split_chain(ivols, offsets)


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
           int(seed) & 0xFFFFFFFFFFFFFFFF, C.dptr(brownians) if brownians is not None else None, C.dptr(sigma_t))
    return sigma_t, grid_t
