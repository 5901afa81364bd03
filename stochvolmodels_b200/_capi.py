"""ctypes binding of ``libb200sv.so`` (C ABI: ``include/b200sv.h``).

There is NO CPU fallback: if the library is missing or fails to load, importing the product path raises.  Symbols are
bound lazily on first use so that CPU-only environments can import the package (e.g. to build the library or to run the
host-logic tests) but cannot compute.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_int, c_int8, c_longlong, c_uint64, c_void_p

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200SV_LIB") or os.path.join(_PKG, "lib", "libb200sv.so")   # B200SV_LIB: tuning builds only

# enums of include/b200sv.h
CALL, PUT, INV_CALL, INV_PUT = 0, 1, 2, 3
LOG_RETURN, Q_VAR, SIGMA = 1, 2, 3
ORDER_FIRST, ORDER_SECOND = 1, 2
STATE_F64, STATE_F32, GAUSS_F32, GAUSS_F64, GAUSS_F64_PAIRED = 0, 1, 0, 2, 4
HESTON_EULER_FLOOR, HESTON_QE = 0, 1
DEBUG_FAST_DIV, DEBUG_FAST_SQRT, DEBUG_FAST_SQRT_POS, DEBUG_NEG2_LOG, DEBUG_EXP_TABLE = 0, 1, 2, 3, 4
TYPE_CODES = {"C": CALL, "P": PUT, "IC": INV_CALL, "IP": INV_PUT}


class LogsvParamsC(Structure):
    _fields_ = [(n, c_double) for n in ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")]


class HestonParamsC(Structure):
    _fields_ = [(n, c_double) for n in ("v0", "theta", "kappa", "rho", "volvol")]


class B200svError(RuntimeError):
    """error reported by libb200sv (code, message)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"libb200sv error {code}: {message}")
        self.code = code
        self.message = message


class HawkesParamsC(ctypes.Structure):
    """b200sv_hawkes_params"""
    _fields_ = [(k, c_double) for k in ("mu", "sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p",
                                        "lambda_m", "theta_m", "kappa_m", "beta1_m", "beta2_m")]


_dp = POINTER(c_double)
_ip = POINTER(c_int)
_i8p = POINTER(c_int8)
_lp = POINTER(LogsvParamsC)
_hp = POINTER(HestonParamsC)
_kp = POINTER(HawkesParamsC)

# name -> argtypes; every symbol declared in include/b200sv.h must be listed here (tests/test_capi_symbols.py checks it)
SIGNATURES = {
    "b200sv_logsv_mc_chain": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_int, c_uint64, c_int, _dp, _dp],
    "b200sv_heston_mc_chain": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_uint64, c_int, c_int, _dp, _dp],
    "b200sv_logsv_mc_chain_batch": [_lp, c_int, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_uint64, c_int, _dp, _dp, _dp],
    "b200sv_heston_mc_chain_batch": [_hp, c_int, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_uint64, c_int, c_int, _dp, _dp, _dp],
    "b200sv_logsv_mc_chain_greeks": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_int, c_uint64, c_int, _dp, _dp,
                                     _dp, _dp],
    "b200sv_heston_mc_chain_greeks": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_uint64, c_int, c_int, _dp, _dp,
                                      _dp, _dp],
    "b200sv_logsv_mc_chain_greeks_gamma": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_int, c_uint64, c_int, _dp,
                                           _dp, _dp, _dp, _dp, _dp, c_longlong, _dp],
    "b200sv_heston_mc_chain_greeks_gamma": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_uint64, c_int, c_int, _dp, _dp,
                                            _dp, _dp, _dp, _dp, c_longlong, _dp],
    "b200sv_logsv_mc_chain_greeks_theta": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_int, c_uint64, c_int, _dp,
                                           _dp, _dp, _dp, _dp, _dp, c_longlong, _dp, _dp, _dp, _dp],
    "b200sv_heston_mc_chain_greeks_theta": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_int, c_uint64, c_int, c_int, _dp, _dp,
                                            _dp, _dp, _dp, _dp, c_longlong, _dp, _dp, _dp, _dp],
    "b200sv_logsv_tangent_terminal": [_lp, c_double, c_longlong, c_int, c_int, c_double, c_uint64, c_int, c_int, c_longlong, _dp, _dp, _dp,
                                      _dp, _dp, _dp],
    "b200sv_heston_tangent_terminal": [_hp, c_double, c_longlong, c_int, c_uint64, c_int, c_int, c_longlong, _dp, _dp, _dp, _dp, _dp, _dp],
    "b200sv_logsv_terminal": [_lp, c_double, c_longlong, c_int, c_int, c_double, c_uint64, c_int, _dp, _dp, _dp],
    "b200sv_logsv_terminal_from_state": [_lp, c_double, c_longlong, c_int, c_int, c_double, c_uint64, c_int, c_int, _dp, _dp, _dp],
    "b200sv_set_stream": [c_void_p],
    "b200sv_heston_terminal": [_hp, c_double, c_longlong, c_int, c_uint64, c_int, c_int, _dp, _dp, _dp],
    "b200sv_logsv_step_fixed": [_dp, _dp, _dp, _dp, _dp, c_int, c_longlong, c_double, _lp, c_double, c_int],
    "b200sv_heston_step_fixed": [_dp, _dp, _dp, _dp, _dp, c_int, c_longlong, c_double, _hp],
    "b200sv_logsv_vol_paths": [_lp, c_double, c_longlong, c_int, c_int, c_uint64, _dp, _dp],
    "b200sv_mc_payoffs": [_dp, _dp, c_longlong, c_double, c_double, _dp, _i8p, c_int, c_double, c_int, _dp, _dp],
    "b200sv_rough_logsv_mc_chain": [_lp, c_int, c_int, _dp, _dp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, _ip, _dp, _dp, _dp, c_longlong,
                                    c_int, c_uint64, c_int, _dp, _dp, _dp, _dp],
    "b200sv_rough_logsv_mc_chain_greeks": [_lp, c_int, _dp, _dp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, _ip, _dp, _dp, _dp, c_longlong,
                                           c_int, c_uint64, c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp],
    "b200sv_rough_logsv_mc_chain_greeks_theta": [_lp, c_int, _dp, _dp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, _ip, _dp, _dp, _dp,
                                                 c_longlong, c_int, c_uint64, c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, c_longlong, _dp],
    "b200sv_hawkesjd_mc_chain": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_uint64, c_int, _dp, _dp],
    "b200sv_hawkesjd_mc_chain_greeks": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_uint64, c_int, _dp, _dp, _dp, _dp,
                                        c_longlong, _dp, _dp],
    "b200sv_hawkesjd_mc_chain_exact": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_longlong, c_int, c_uint64, c_int, _dp, _dp, c_longlong,
                                       c_longlong, _dp, _dp],
    "b200sv_hawkesjd_terminal_exact": [_kp, c_double, c_longlong, c_uint64, c_int, c_int, c_int, c_longlong, _dp, _dp, _dp],
    "b200sv_hawkesjd_price_chain": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, c_double, _dp, _dp, _dp, _dp, _dp],
    "b200sv_hawkesjd_mgf_grid": [_dp, _dp, c_int, c_double, _dp, _kp, _dp],
    "b200sv_fourier_gamma": [_dp, _dp, c_int, c_double, c_double, c_double, c_double, _dp, _i8p, c_int, c_int, _dp],
    "b200sv_hawkesjd_terminal": [_kp, c_double, c_longlong, c_uint64, c_int, c_int, c_int, _dp, _dp, _dp],
    "b200sv_hawkesjd_step_fixed": [_dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, c_int, c_longlong, c_double, _kp],
    "b200sv_hawkesjd_device_draws": [c_uint64, c_longlong, c_longlong, c_int, c_int, c_double, _kp, c_int, _dp, _dp, _dp, _dp, _dp],
    "b200sv_device_normals": [c_uint64, c_longlong, c_longlong, c_int, c_int, c_int, _dp, _dp],
    "b200sv_dev_logsv_slice": [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_int, _lp, c_double, c_int, c_int, c_double,
                               c_int, c_double, c_uint64, c_int, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_heston_slice": [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_int, _hp, c_int, c_double, c_int, c_double,
                                c_uint64, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_payoff_sums": [c_void_p, c_void_p, c_longlong, c_int, c_double, c_double, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_void_p, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_payoff_finalize": [c_void_p, c_int, c_double, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p],
    "b200sv_p2p_create": [c_int, c_int, c_int, POINTER(c_void_p), POINTER(ctypes.c_ubyte)],
    "b200sv_p2p_connect": [c_void_p, POINTER(ctypes.c_ubyte)],
    "b200sv_p2p_destroy": [c_void_p],
    "b200sv_p2p_set_spin_limit": [c_void_p, ctypes.c_uint],
    "b200sv_p2p_status": [c_void_p, POINTER(ctypes.c_uint), c_void_p],
    "b200sv_debug_p2p_lose_publish": [c_void_p],
    "b200sv_dev_p2p_publish": [c_void_p, c_void_p, c_int, c_void_p],
    "b200sv_dev_p2p_gather": [c_void_p, c_int, c_void_p, c_void_p],
    "b200sv_dev_logsv_step_fixed": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_double, _lp, c_double,
                                    c_int, c_int, c_void_p],
    "b200sv_dev_heston_step_fixed": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_double, _hp, c_void_p],
    "b200sv_dev_logsv_mc_chain_greeks_fixed": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, POINTER(c_void_p), POINTER(c_void_p), _ip, _dp,
                                               c_longlong, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_spot_moments": [c_void_p, c_longlong, c_double, c_void_p, c_void_p],
    "b200sv_dev_hawkesjd_slice": [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_int, _kp, c_int, c_double, c_int, c_double, c_uint64,
                                  c_int, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_hawkesjd_exact_slice": [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_int, _kp, c_double, c_int, c_double, c_uint64,
                                        c_longlong, c_void_p, c_void_p, c_void_p, c_void_p],
    "b200sv_dev_rough_logsv_slice": [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, _lp, c_int, _dp, _dp, c_int, c_double, c_double,
                                     c_uint64, c_int, c_void_p, c_void_p, c_void_p],
    "b200sv_debug_exp_pair": [_dp, c_longlong, _dp],
    "b200sv_debug_exp_pair_scaled": [_dp, c_longlong, _dp],
    "b200sv_debug_box_muller": [POINTER(ctypes.c_uint32), c_longlong, c_int, _dp],
    "b200sv_debug_fastmath": [c_int, _dp, _dp, c_longlong, _dp],
    "b200sv_debug_hawkes_clocks": [POINTER(ctypes.c_uint32), _dp, c_longlong, c_double, _kp, _dp],
    "b200sv_logsv_price_chain": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, c_int, c_double, c_int, _dp, _dp, _dp],
    "b200sv_heston_price_chain": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp],
    "b200sv_logsv_price_chain_greeks": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, c_int, c_double, c_int, _dp, _dp, _dp, _ip],
    "b200sv_heston_price_chain_greeks": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp],
    "b200sv_hawkesjd_price_chain_greeks": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp, _ip],
    "b200sv_hawkesjd_price_chain_risk_premia_greeks": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, c_double, _dp, _dp,
                                                       _dp, _dp, _ip],
    "b200sv_hawkesjd_price_chain_risk_premia_hessian": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, c_double, _dp, _dp,
                                                        _dp, _dp, _ip, _dp, _dp, _dp, _dp],
    "b200sv_logsv_price_chain_greeks_theta": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, c_int, c_double, c_int, _dp, _dp, _dp,
                                              _ip, _dp, _dp, _ip],
    "b200sv_heston_price_chain_greeks_theta": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp, _dp, _dp],
    "b200sv_hawkesjd_price_chain_greeks_theta": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp, _ip, _dp, _dp,
                                                 _ip],
    "b200sv_logsv_price_chain_hessian": [_lp, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, c_int, c_double, c_int, _dp, _dp, _dp, _ip,
                                         _dp, _dp, _dp],
    "b200sv_heston_price_chain_hessian": [_hp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp, _dp, _dp, _dp],
    "b200sv_hawkesjd_price_chain_hessian": [_kp, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp, _ip, _dp, _dp,
                                            _dp],
    "b200sv_logsv_price_chain_batch": [_lp, c_int, c_int, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, c_double, c_int, _dp, _dp],
    "b200sv_heston_price_chain_batch": [_hp, c_int, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_double, c_int, _dp, _dp],
    "b200sv_logsv_price_chains_batch": [_lp, c_int, _ip, c_int, _ip, _dp, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_int, _dp, c_int, _dp, _dp],
    "b200sv_heston_price_chains_batch": [_hp, c_int, _ip, c_int, _ip, _dp, _dp, _dp, _ip, _dp, _i8p, _dp, c_int, _dp, _dp],
    "b200sv_hawkesjd_price_chain_batch": [_kp, c_int, c_int, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, c_double, c_int, _dp, _dp, _dp],
    "b200sv_hawkesjd_price_chains_batch": [_kp, c_int, _ip, c_int, _ip, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, _dp, c_int, _dp, _dp],
    "b200sv_hawkesjd_price_chains_batch_gamma": [_kp, _dp, c_int, _ip, c_int, _ip, _dp, _dp, _dp, _ip, _dp, _i8p, c_int, _dp, c_int, _dp, _dp],
    "b200sv_fourier_qvar": [_dp, _dp, c_int, c_double, _dp, _i8p, c_int, c_double, _dp],
    "b200sv_fourier_pdf": [_dp, _dp, c_int, _dp, c_int, _dp],
    "b200sv_fourier_digital": [_dp, _dp, c_int, c_double, _dp, _i8p, c_int, c_double, _dp],
    "b200sv_bsm_implied_vols": [c_int, _dp, _dp, _dp, _ip, _dp, _i8p, _dp, _dp],
    "b200sv_debug_bsm_implied_vols": [c_int, _dp, _dp, _dp, _ip, _dp, _i8p, _dp, _dp, _ip],
    "b200sv_bsm_implied_vol_sensitivities": [c_int, _dp, _dp, _dp, _ip, _dp, _i8p, _dp, c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp],
    "b200sv_bsm_implied_vol_theta": [c_int, _dp, _dp, _dp, _ip, _dp, _i8p, _dp, _dp, _dp, _dp],
    "b200sv_logsv_mgf_grid": [_dp, _dp, c_int, c_double, _dp, _lp, c_double, c_int, c_int, _dp],
    "b200sv_logsv_mgf_grid_analytic": [_dp, _dp, c_int, c_double, _dp, _lp, c_int, c_int, c_int, _dp],
    "b200sv_logsv_mgf_grid_bdf": [_dp, _dp, c_int, c_double, _dp, _lp, c_double, c_int, c_int, _dp],
    "b200sv_logsv_ode_terms": [_dp, _dp, c_int, _lp, c_double, c_int, c_int, _dp, _dp, _dp],
    "b200sv_logsv_ode_rhs": [_dp, _dp, c_int, _dp, _lp, c_double, c_int, c_int, _dp],
    "b200sv_ode_rhs_dense": [_dp, c_int, c_int, _dp, _dp, _dp, _dp],
    "b200sv_heston_mgf_grid": [_dp, _dp, c_int, c_double, _dp, _dp, _hp, _dp],
    "b200sv_fourier_vanilla": [_dp, _dp, c_int, c_double, _dp, _i8p, c_int, c_double, c_int, _dp],
}
_MISC = {
    "b200sv_last_error": ([], c_char_p),
    "b200sv_version": ([], c_int),
    "b200sv_launch_count": ([], c_longlong),
    "b200sv_reset_launch_count": ([], None),
    "b200sv_get_stream": ([], c_void_p),
}

_lib = None


def load_library() -> ctypes.CDLL:
    """dlopen the in-tree CUDA library; raise (never fall back) if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m stochvolmodels_b200._build` (needs nvcc). "
            "stochvolmodels_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int
    for name, (args, res) in _MISC.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = res
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load_library().b200sv_last_error()
        raise B200svError(rc, msg.decode() if msg else "unknown")


def call(name: str, *args) -> None:
    check(getattr(load_library(), name)(*args))


# ---- numpy helpers --------------------------------------------------------------------------------------------------------
def f64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float64)


def c128(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.complex128)


def dptr(a: np.ndarray):
    """double* of a float64 array, or of a complex128 one (interleaved re, im); None -> NULL"""
    return a.ctypes.data_as(_dp) if a is not None else None


def iptr(a: np.ndarray):
    """int* of an int32 array; None -> NULL"""
    return a.ctypes.data_as(_ip) if a is not None else None


def i8ptr(a: np.ndarray):
    return a.ctypes.data_as(_i8p)


def seed64(seed) -> int:
    """a Philox key as the library's uint64: Python ints of any sign or size wrap modulo 2^64"""
    return int(seed) & 0xFFFFFFFFFFFFFFFF


DEFAULT_VOL_SCALER = -1.0       # the Fourier chain entry points read every vol_scaler <= 0 as "the model's default transform grid"


def vol_scaler_arg(vol_scaler) -> float:
    return DEFAULT_VOL_SCALER if vol_scaler is None else float(vol_scaler)


def batch_etas(etas, B: int, M: int):
    """per-set vol backbones [B, M] as float64, or None (the library then uses ones)"""
    if etas is None:
        return None
    etas = np.ascontiguousarray(etas, dtype=np.float64)
    if etas.shape != (B, M):
        raise ValueError(f"etas must have shape ({B}, {M})")
    return etas


def chain_ptrs(chain, *etas):
    """the chain block of a chain entry point, (M, ttms, forwards, discfactors, [etas,] offsets, strikes, types), from engine._chain_arrays;
    the LogSV entry points take their etas array (None -> NULL) between the discount factors and the offsets"""
    return (chain.M, dptr(chain.ttms), dptr(chain.forwards), dptr(chain.discfactors), *(dptr(e) for e in etas), iptr(chain.offsets),
            dptr(chain.strikes), i8ptr(chain.types))


def encode_types(optiontypes) -> np.ndarray:
    """'C','P','IC','IP' -> int8 codes; unknown code -> ValueError like utils/mc_payoffs.py:83-84 / utils/mgf_pricer.py:212.
    Vectorised (four array comparisons): the marshalling of a 49-strike chain is part of the latency of a small MC call."""
    a = np.asarray(optiontypes)
    if a.dtype.kind != "U":
        a = np.array([str(t) for t in np.atleast_1d(a).ravel()], dtype="U8").reshape(np.shape(a))
    out = np.full(a.shape, -1, dtype=np.int8)
    for name, code in TYPE_CODES.items():
        out[a == name] = code
    if out.size and out.min() < 0:
        raise ValueError("unknown option payoff code")
    return out


def flatten_chain(strikes_ttms, optiontypes_ttms):
    """ragged per-maturity lists -> (offsets int32[M+1], strikes f64[sum J], types int8[sum J])."""
    sizes = [len(s) for s in strikes_ttms]
    offsets = np.zeros(len(sizes) + 1, dtype=np.int32)
    offsets[1:] = np.cumsum(sizes)
    strikes = f64(np.concatenate([np.asarray(s, dtype=np.float64).ravel() for s in strikes_ttms])) if sizes else np.zeros(0)
    types = encode_types(np.concatenate([np.asarray(t).ravel() for t in optiontypes_ttms])) if sizes else np.zeros(0, dtype=np.int8)
    if strikes.shape[0] != types.shape[0]:
        raise ValueError("strikes and option types must have the same length")
    return offsets, strikes, np.ascontiguousarray(types, dtype=np.int8)


def split_chain(flat: np.ndarray, offsets: np.ndarray):
    return [flat[offsets[m]:offsets[m + 1]].copy() for m in range(len(offsets) - 1)]
