"""Argument checks of the host-level Monte Carlo entry points of libb200sv.  Each case below has exactly one defect; the call must return the
error code and message before its first stream operation, so this file needs the library but no GPU."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

from stochvolmodels_b200 import _capi as C

NULL = (-1, "invalid argument: null pointer")
M_ERR = (-1, "invalid argument: M must be >= 1")
B_ERR = (-1, "invalid argument: B must be >= 1")
NB_PATH = (-1, "invalid argument: nb_path must be >= 1")
STEPS = (-1, "invalid argument: nb_steps_per_year must be >= 1")
TTMS = (-1, "invalid argument: ttms must be positive and strictly increasing")
OFFSETS = (-1, "invalid argument: offsets must be non-decreasing")
PAYOFF = (-3, "unknown option payoff code")
VTYPE = (-4, "variable_type not implemented")
SCHEME = (-1, "invalid argument: unknown Heston scheme")
SCHEME_GREEKS = (-1, "invalid argument: pathwise sensitivities need scheme = B200SV_HESTON_EULER_FLOOR")
GAUSS_GREEKS = (-1, "invalid argument: pathwise sensitivities support B200SV_GAUSS_F32 and B200SV_GAUSS_F64")
F32_GREEKS = (-1, "invalid argument: pathwise sensitivities need fp64 state (B200SV_STATE_F64)")
TERMINAL = (-1, "invalid argument: nb_path, ttm, nb_steps_per_year must be positive")
SLICE = (-1, "invalid argument: slice_index and path_offset must be >= 0")
HAWKES_F32 = (-1, "invalid argument: the Hawkes route is float64 only")
ROUGH_FACTORS = (-1, "invalid argument: B >= 1 and 1 <= n_factors <= 8")
ROUGH_GREEKS_FACTORS = (-1, "invalid argument: 1 <= n_factors <= 8")
ROUGH_PAIR = (-1, "invalid argument: Z0 and Z1 must be supplied together")
ROUGH_STATES = (-1, "invalid argument: terminal states are returned for a single parameter set")
ROUGH_GAUSS = (-1, "invalid argument: gauss flags")
ROUGH_F32 = (-1, "invalid argument: the rough-vol route is float64 only")
ROUGH_STEPS = (-1, "invalid argument: nsteps / h must be positive")
ROUGH_ZROWS = (-1, "invalid argument: Z0 / Z1 have fewer rows than the longest grid")

LP = C.LogsvParamsC(1.0, 1.0, 5.0, 5.0, 0.2, 2.0)
HP = C.HestonParamsC(0.04, 0.04, 4.0, -0.5, 0.5)
KP = C.HawkesParamsC(0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5)
PAIRED, CONTRADICTORY = C.GAUSS_F64_PAIRED, C.GAUSS_F64 | C.GAUSS_F64_PAIRED

PRICING = ("logsv", "heston", "logsv_batch", "heston_batch")
GREEKS = ("logsv_greeks", "heston_greeks")
TANGENT = ("logsv_tangent", "heston_tangent")
ROUGH = ("rough", "rough_greeks")
CHAIN = PRICING + GREEKS + ROUGH + ("hawkes",)
VT_ROUTES = ("logsv", "heston") + GREEKS + ROUGH + ("hawkes",)


def _valid():
    return dict(M=2, ttms=[0.25, 0.5], offsets=[0, 3, 6], strikes=[0.9, 1.0, 1.1] * 2, types=[C.PUT, C.CALL, C.CALL] * 2, B=2, nb_path=16,
                steps=12, vt=C.LOG_RETURN, flags=0, scheme=C.HESTON_EULER_FLOOR, ttm=0.25, slice=0, path_offset=0, x=True,
                n=2, weights=True, nsteps=[4, 8], hs=[0.0625, 0.0625], z0=False, z1=False, z_rows=0, states=False, rough_B=1)


def _f64(a):
    return None if a is None else C.f64(a)


def _call(route, c):
    lib = C.load_library()
    a = SimpleNamespace(**c)
    ttms, fw, df = _f64(a.ttms), np.ones(2), np.ones(2)
    off = np.asarray(a.offsets, dtype=np.int32)
    strikes = _f64(a.strikes)
    types = None if a.types is None else np.asarray(a.types, dtype=np.int8)
    t, fw_, df_, o, k = C.dptr(ttms), C.dptr(fw), C.dptr(df), C.iptr(off), C.dptr(strikes)
    ty = None if types is None else C.i8ptr(types)
    buf = np.zeros(4096)
    out = C.dptr(buf)
    lps, hps = (C.LogsvParamsC * 2)(LP, LP), (C.HestonParamsC * 2)(HP, HP)
    w = C.f64(np.full(2 * max(a.n, 1), 0.5)) if a.weights else None
    nodes = C.f64(np.full(2 * max(a.n, 1), 1.0))
    nsteps, hs = np.asarray(a.nsteps, dtype=np.int32), C.f64(a.hs)
    z = C.f64(np.zeros(8 * a.nb_path + 1))
    z0, z1 = (C.dptr(z) if a.z0 else None), (C.dptr(z) if a.z1 else None)
    x = out if a.x else None
    if route == "logsv":
        return lib.b200sv_logsv_mc_chain(ctypes.byref(LP), a.M, t, fw_, df_, None, o, k, ty, a.nb_path, a.steps, 1, a.vt, 0, a.flags, out, out)
    if route == "heston":
        return lib.b200sv_heston_mc_chain(ctypes.byref(HP), a.M, t, fw_, df_, o, k, ty, a.nb_path, a.steps, a.vt, 0, a.flags, a.scheme, out, out)
    if route == "logsv_batch":
        return lib.b200sv_logsv_mc_chain_batch(lps, a.B, a.M, t, fw_, df_, None, o, k, ty, a.nb_path, a.steps, 1, 0, a.flags, out, out, None)
    if route == "heston_batch":
        return lib.b200sv_heston_mc_chain_batch(hps, a.B, a.M, t, fw_, df_, o, k, ty, a.nb_path, a.steps, 0, a.flags, a.scheme, out, out, None)
    if route == "logsv_greeks":
        return lib.b200sv_logsv_mc_chain_greeks(ctypes.byref(LP), a.M, t, fw_, df_, None, o, k, ty, a.nb_path, a.steps, 1, a.vt, 0, a.flags,
                                                out, out, out, out)
    if route == "heston_greeks":
        return lib.b200sv_heston_mc_chain_greeks(ctypes.byref(HP), a.M, t, fw_, df_, o, k, ty, a.nb_path, a.steps, a.vt, 0, a.flags, a.scheme,
                                                 out, out, out, out)
    if route == "logsv_tangent":
        return lib.b200sv_logsv_tangent_terminal(ctypes.byref(LP), a.ttm, a.nb_path, a.steps, 1, 1.0, 0, a.flags, a.slice, a.path_offset, x, out,
                                                 out, out, out, out)
    if route == "heston_tangent":
        return lib.b200sv_heston_tangent_terminal(ctypes.byref(HP), a.ttm, a.nb_path, a.steps, 0, a.flags, a.slice, a.path_offset, x, out, out,
                                                  out, out, out)
    if route == "rough":
        return lib.b200sv_rough_logsv_mc_chain(lps, a.rough_B, a.n, C.dptr(w), C.dptr(nodes), a.M, t, fw_, df_, o, k, ty, a.nb_path,
                                               C.iptr(nsteps), C.dptr(hs), z0, z1, a.z_rows, a.vt, 0, a.flags, out, out, None,
                                               out if a.states else None)
    if route == "rough_greeks":
        return lib.b200sv_rough_logsv_mc_chain_greeks(ctypes.byref(LP), a.n, C.dptr(w), C.dptr(nodes), a.M, t, fw_, df_, o, k, ty, a.nb_path,
                                                      C.iptr(nsteps), C.dptr(hs), z0, z1, a.z_rows, a.vt, 0, a.flags, out, out, out, out, None,
                                                      None, None)
    assert route == "hawkes"
    return lib.b200sv_hawkesjd_mc_chain(ctypes.byref(KP), a.M, t, fw_, df_, o, k, ty, a.nb_path, a.vt, 0, a.flags, out, out)


def _cases():
    """(routes, one-field change of the valid arguments, expected (code, message))"""
    table = [
        (CHAIN, dict(M=0), M_ERR),
        (("logsv_batch", "heston_batch"), dict(B=0), B_ERR),
        (("rough",), dict(rough_B=0), ROUGH_FACTORS),
        (CHAIN, dict(nb_path=0), NB_PATH),
        (PRICING + GREEKS, dict(steps=0), STEPS),
        (TANGENT, dict(nb_path=0), TERMINAL),
        (TANGENT, dict(steps=0), TERMINAL),
        (TANGENT, dict(ttm=0.0), TERMINAL),
        (TANGENT, dict(slice=-1), SLICE),
        (TANGENT, dict(path_offset=-1), SLICE),
        (CHAIN, dict(ttms=[0.5, 0.25]), TTMS),
        (CHAIN, dict(ttms=[0.0, 0.5]), TTMS),
        (CHAIN, dict(offsets=[0, 4, 3]), OFFSETS),
        (CHAIN, dict(types=[C.PUT, 4, C.CALL] * 2), PAYOFF),
        (CHAIN, dict(types=[C.PUT, -1, C.CALL] * 2), PAYOFF),
        (VT_ROUTES, dict(vt=C.SIGMA), VTYPE),
        (("heston", "heston_batch"), dict(scheme=7), SCHEME),
        (("heston_greeks",), dict(scheme=C.HESTON_QE), SCHEME_GREEKS),
        (GREEKS + TANGENT, dict(flags=CONTRADICTORY), GAUSS_GREEKS),
        (GREEKS + TANGENT, dict(flags=PAIRED), GAUSS_GREEKS),
        (GREEKS + TANGENT, dict(flags=C.STATE_F32), F32_GREEKS),
        (ROUGH, dict(flags=CONTRADICTORY), ROUGH_GAUSS),
        (ROUGH, dict(flags=PAIRED), ROUGH_GAUSS),
        (ROUGH, dict(flags=C.STATE_F32), ROUGH_F32),
        (("hawkes",), dict(flags=C.STATE_F32), HAWKES_F32),
        (("rough",), dict(n=0), ROUGH_FACTORS),
        (("rough",), dict(n=9), ROUGH_FACTORS),
        (("rough_greeks",), dict(n=0), ROUGH_GREEKS_FACTORS),
        (("rough_greeks",), dict(n=9), ROUGH_GREEKS_FACTORS),
        (ROUGH, dict(z0=True), ROUGH_PAIR),
        (ROUGH, dict(z1=True), ROUGH_PAIR),
        (ROUGH, dict(z0=True, z1=True, z_rows=7), ROUGH_ZROWS),
        (ROUGH, dict(nsteps=[0, 8]), ROUGH_STEPS),
        (ROUGH, dict(hs=[0.0625, 0.0]), ROUGH_STEPS),
        (("rough",), dict(rough_B=2, states=True), ROUGH_STATES),
        (CHAIN, dict(ttms=None), NULL),
        (ROUGH, dict(weights=False), NULL),
        (TANGENT, dict(x=False), NULL),
        (CHAIN, dict(strikes=None), NULL),
        (CHAIN, dict(types=None), NULL),
    ]
    for routes, change, expected in table:
        name = "-".join(f"{k}={'null' if v is None else v}" for k, v in change.items())
        for r in routes:
            yield pytest.param(r, change, expected, id=f"{r}-{name}")


@pytest.mark.parametrize("route,change,expected", list(_cases()))
def test_mc_entry_points_reject(route, change, expected):
    c = _valid()
    c.update(change)
    rc = _call(route, c)
    assert (rc, C.load_library().b200sv_last_error().decode()) == expected
