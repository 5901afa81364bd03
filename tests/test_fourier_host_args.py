"""Argument checks of every Fourier / MGF entry point of libb200sv.  Each case below has exactly one defect; the call must return the
error code and message before its first stream operation, so this file needs the library but no GPU."""
import ctypes
import math

import numpy as np
import pytest

from stochvolmodels_b200 import _capi as C

NULL = (-1, "invalid argument: null pointer")
TTMS = (-1, "invalid argument: ttms must be positive and strictly increasing")
MP = (-1, "invalid argument: M >= 1, P >= 3")
BMP = (-1, "invalid argument: 1 <= B <= 65535, M >= 1, P >= 3")
STRIKE = (-1, "invalid argument: strikes must be positive")
EMPTY = (-1, "invalid argument: the chain has no strikes")
NOT_IMPL = (-5, "not implemented")
ORDER = (-4, "expansion_order not implemented")
VTYPE = (-4, "variable_type not implemented")
VTYPE_GREEKS = (-4, "variable_type not implemented: sensitivities cover LOG_RETURN only")
GRID = (-1, "invalid argument: P >= 1, dtau > 0")
GRID_AN = (-1, "invalid argument: P >= 1, dtau > 0, year_days >= 1")
GRID_P = (-1, "invalid argument: P >= 1")
DENSE = (-1, "invalid argument: P >= 1, 1 <= n <= 16")
SUM = (-1, "invalid argument: P >= 3, J >= 1")
SUM_QVAR = (-1, "invalid argument: P >= 3, J >= 1, ttm > 0")

LP = C.LogsvParamsC(1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
HP = C.HestonParamsC(0.04, 0.04, 4.0, -0.5, 0.5)
KP = C.HawkesParamsC(0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5)
IC = C.INV_CALL
SINGLE = ("logsv", "heston", "logsv_greeks", "heston_greeks", "hawkes")
BATCH = ("logsv_batch", "heston_batch")
LOGSV = ("logsv", "logsv_greeks", "logsv_batch")


def _valid_chain():
    return dict(M=2, ttms=[0.25, 0.5], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2, spot=1,
                vt=C.LOG_RETURN, order=C.ORDER_SECOND, P=0, B=2, gamma=math.nan)


def _call_chain(route, c):
    lib = C.load_library()
    M, B, P, spot, vt, order = c["M"], c["B"], c["P"], c["spot"], c["vt"], c["order"]
    ttms, fw, df = C.f64(c["ttms"]), np.ones(2), np.ones(2)
    off = np.asarray(c["offsets"], dtype=np.int32)
    strikes = None if c["strikes"] is None else C.f64(c["strikes"])
    types = None if c["types"] is None else np.asarray(c["types"], dtype=np.int8)
    t, fw_, df_, o, k = C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(off), C.dptr(strikes)
    ty = None if types is None else C.i8ptr(types)
    out, greeks = np.zeros(64), np.zeros(512)
    pr, g = C.dptr(out), C.dptr(greeks)
    lps, hps = (C.LogsvParamsC * 2)(LP, LP), (C.HestonParamsC * 2)(HP, HP)
    if route == "logsv":
        return lib.b200sv_logsv_price_chain(ctypes.byref(LP), M, t, fw_, df_, None, o, k, ty, spot, vt, order, -1.0, P, pr, None, None)
    if route == "heston":
        return lib.b200sv_heston_price_chain(ctypes.byref(HP), M, t, fw_, df_, o, k, ty, vt, -1.0, P, pr, None)
    if route == "logsv_greeks":
        return lib.b200sv_logsv_price_chain_greeks(ctypes.byref(LP), M, t, fw_, df_, None, o, k, ty, spot, vt, order, -1.0, P, pr, g, None, None)
    if route == "heston_greeks":
        return lib.b200sv_heston_price_chain_greeks(ctypes.byref(HP), M, t, fw_, df_, o, k, ty, vt, -1.0, P, pr, g, None)
    if route == "logsv_batch":
        return lib.b200sv_logsv_price_chain_batch(lps, B, M, t, fw_, df_, None, o, k, ty, spot, order, -1.0, P, pr, None)
    if route == "heston_batch":
        return lib.b200sv_heston_price_chain_batch(hps, B, M, t, fw_, df_, o, k, ty, -1.0, P, pr, None)
    assert route == "hawkes"
    return lib.b200sv_hawkesjd_price_chain(ctypes.byref(KP), M, t, fw_, df_, o, k, ty, spot, -1.0, P, c["gamma"], pr, None, None, None, None)


def _chain_cases():
    """(routes, one-field change of the valid chain, expected (code, message))"""
    bad_type = [C.PUT, 4, C.CALL] * 2
    inverse = [C.PUT, IC, C.CALL] * 2
    table = [
        (SINGLE + BATCH, dict(ttms=[0.5, 0.25]), TTMS),
        (SINGLE, dict(M=0), MP),
        (SINGLE, dict(P=2), MP),
        (BATCH, dict(M=0), BMP),
        (BATCH, dict(P=2), BMP),
        (("logsv", "heston", "logsv_greeks", "heston_greeks") + BATCH, dict(strikes=[0.9, 1.0, 1.1, 0.9, 0.0, 1.1]), STRIKE),
        (SINGLE + BATCH, dict(types=bad_type), NOT_IMPL),
        (SINGLE + BATCH, dict(types=inverse), NOT_IMPL),
        (("logsv", "heston"), dict(vt=C.Q_VAR), NOT_IMPL),
        (LOGSV, dict(order=7), ORDER),
        (("logsv", "heston"), dict(vt=C.SIGMA), VTYPE),
        (("logsv_greeks", "heston_greeks"), dict(vt=C.SIGMA), VTYPE_GREEKS),
        (("logsv_greeks", "heston_greeks"), dict(vt=C.Q_VAR), VTYPE_GREEKS),
        (BATCH, dict(B=0), BMP),
        (BATCH, dict(offsets=[0, 0, 0]), EMPTY),
        (("hawkes",), dict(gamma=0.5, spot=0), NOT_IMPL),
        (("hawkes",), dict(gamma=0.5, types=inverse), NOT_IMPL),
        (SINGLE + BATCH, dict(strikes=None), NULL),
        (SINGLE + BATCH, dict(types=None), NULL),
    ]
    for routes, change, expected in table:
        name = "-".join(f"{k}={'null' if v is None else v}" for k, v in change.items())
        for r in routes:
            yield pytest.param(r, change, expected, id=f"{r}-{name}")


def _check(rc, expected):
    msg = C.load_library().b200sv_last_error().decode()
    assert (rc, msg) == expected


@pytest.mark.parametrize("route,change,expected", list(_chain_cases()))
def test_chain_entry_points_reject(route, change, expected):
    c = _valid_chain()
    c.update(change)
    _check(_call_chain(route, c), expected)


def _call_grid(route, P=8, dtau=0.25, order=C.ORDER_SECOND, n=5, J=3, ttm=0.25, spot=1, types=(C.PUT, C.CALL, C.CALL)):
    lib = C.load_library()
    buf = [np.zeros(2 * 5 ** 3 * max(P, 1) + 64) for _ in range(6)]
    b = [C.dptr(x) for x in buf]
    strikes, ty = C.f64([0.9, 1.0, 1.1]), np.asarray(types, dtype=np.int8)
    k, t = C.dptr(strikes), C.i8ptr(ty)
    calls = {
        "hawkesjd_mgf_grid": lambda: lib.b200sv_hawkesjd_mgf_grid(b[0], None, P, dtau, b[1], ctypes.byref(KP), b[2]),
        "logsv_mgf_grid": lambda: lib.b200sv_logsv_mgf_grid(b[0], None, P, dtau, b[1], ctypes.byref(LP), 1.0, spot, order, b[2]),
        "logsv_mgf_grid_bdf": lambda: lib.b200sv_logsv_mgf_grid_bdf(b[0], None, P, dtau, b[1], ctypes.byref(LP), 1.0, spot, order, b[2]),
        "logsv_mgf_grid_analytic": lambda: lib.b200sv_logsv_mgf_grid_analytic(b[0], None, P, dtau, b[1], ctypes.byref(LP), spot, order, 260, b[2]),
        "heston_mgf_grid": lambda: lib.b200sv_heston_mgf_grid(b[0], None, P, dtau, b[1], b[2], ctypes.byref(HP), b[3]),
        "logsv_ode_terms": lambda: lib.b200sv_logsv_ode_terms(b[0], None, P, ctypes.byref(LP), 1.0, spot, order, b[1], b[2], b[3]),
        "logsv_ode_rhs": lambda: lib.b200sv_logsv_ode_rhs(b[0], None, P, b[1], ctypes.byref(LP), 1.0, spot, order, b[2]),
        "ode_rhs_dense": lambda: lib.b200sv_ode_rhs_dense(b[0], P, n, b[1], b[2], b[3], b[4]),
        "fourier_vanilla": lambda: lib.b200sv_fourier_vanilla(b[0], b[1], P, 1.0, k, t, J, 1.0, spot, b[2]),
        "fourier_gamma": lambda: lib.b200sv_fourier_gamma(b[0], b[1], P, 0.5, 1.0, 1.0, 1.0, k, t, J, spot, b[2]),
        "fourier_qvar": lambda: lib.b200sv_fourier_qvar(b[0], b[1], P, ttm, k, t, J, 1.0, b[2]),
        "fourier_pdf": lambda: lib.b200sv_fourier_pdf(b[0], b[1], P, k, J, b[2]),
        "fourier_digital": lambda: lib.b200sv_fourier_digital(b[0], b[1], P, 1.0, k, t, J, 1.0, b[2]),
    }
    return calls[route]()


GRID_CASES = [
    *[(r, dict(dtau=0.0), GRID) for r in ("hawkesjd_mgf_grid", "logsv_mgf_grid", "logsv_mgf_grid_bdf", "heston_mgf_grid")],
    *[(r, dict(P=0), GRID) for r in ("hawkesjd_mgf_grid", "logsv_mgf_grid", "logsv_mgf_grid_bdf", "heston_mgf_grid")],
    ("logsv_mgf_grid_analytic", dict(dtau=0.0), GRID_AN),
    ("logsv_mgf_grid_analytic", dict(P=0), GRID_AN),
    *[(r, dict(order=7), ORDER) for r in ("logsv_mgf_grid", "logsv_mgf_grid_bdf", "logsv_mgf_grid_analytic", "logsv_ode_terms", "logsv_ode_rhs")],
    ("logsv_ode_terms", dict(P=0), GRID_P),
    ("logsv_ode_rhs", dict(P=0), GRID_P),
    ("ode_rhs_dense", dict(P=0), DENSE),
    ("ode_rhs_dense", dict(n=17), DENSE),
    *[(r, dict(P=0), SUM) for r in ("fourier_vanilla", "fourier_gamma", "fourier_pdf", "fourier_digital")],
    *[(r, dict(J=0), SUM) for r in ("fourier_vanilla", "fourier_gamma", "fourier_pdf", "fourier_digital")],
    ("fourier_qvar", dict(P=0), SUM_QVAR),
    ("fourier_qvar", dict(ttm=0.0), SUM_QVAR),
    ("fourier_qvar", dict(types=(C.CALL, C.PUT, C.CALL)), NOT_IMPL),
    ("fourier_vanilla", dict(types=(C.PUT, 4, C.CALL)), NOT_IMPL),
    ("fourier_vanilla", dict(types=(C.PUT, IC, C.CALL)), NOT_IMPL),
    ("fourier_gamma", dict(spot=0), NOT_IMPL),
    ("fourier_gamma", dict(types=(C.PUT, IC, C.CALL)), NOT_IMPL),
    ("fourier_digital", dict(types=(C.PUT, IC, C.CALL)), NOT_IMPL),
]


@pytest.mark.parametrize("route,change,expected", [pytest.param(r, ch, e, id=f"{r}-{'-'.join(f'{k}={v}' for k, v in ch.items())}")
                                                   for r, ch, e in GRID_CASES])
def test_grid_and_sum_entry_points_reject(route, change, expected):
    _check(_call_grid(route, **change), expected)
