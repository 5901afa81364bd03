"""oracle.rough_greeks -- numpy forward-mode (tangent-linear) restatement of ``oracle.rough``: the rough-LogSV multi-factor step with its
per-step tangents, and the chain's pathwise sensitivities through ``oracle.mc_greeks.mc_payoff_greeks``.  TEST INFRASTRUCTURE ONLY;
written from DESIGN.md §3.10, not from the kernel.

Directions in ``PARAMS`` order (LOGSV_GREEK_PARAMS of the package; ``orthog_vol`` is the ``volvol`` field on this route).  With W = sum w,
v0 = sigma0 / W, vartheta = sqrt(beta^2 + orthog_vol^2), rho = beta / vartheta, the step is differentiated operation by operation: RK4 stage
tangents combined like the stages, the exact log-normal step through its exponent, zero factor tangents on a path that takes the
reset-to-1e-6 branch, and the log-spot / quadratic-variation increments through term1 and term2.
State arrays are (n, P) / (P,), tangents (6, n, P) / (6, P).
"""
from __future__ import annotations

import numpy as np

from . import mc as _mc
from .mc_greeks import mc_payoff_greeks

PARAMS = ("sigma0", "theta", "kappa1", "kappa2", "beta", "orthog_vol")


def tangent_consts(weights, sigma0, beta, orthog_vol):
    """per-direction derivatives of the step's constants: dict of (6,) arrays"""
    W = float(np.sum(weights))
    vt = np.sqrt(beta ** 2 + orthog_vol ** 2)
    rho = beta / vt
    rho_comp = np.sqrt(1.0 - rho * rho)
    e = np.eye(6)
    dvt = e[4] * beta / vt + e[5] * orthog_vol / vt
    drho = (e[4] - rho * dvt) / vt
    return dict(dv0=e[0] / W, dtheta=e[1], dk1=e[2], dk2=e[3], dvt=dvt, dvv=W * dvt, drho=drho,
                drho_comp=-rho * drho / rho_comp if rho_comp > 0.0 else 0.0 * drho)


def drift_rk4_tangent(nodes, weight, v0, dv0, theta, dtheta, kappa1, dk1, kappa2, dk2, z0, dz0, h):
    """``oracle.rough.drift_rk4`` and its tangent: nodes / weight (n, 1), z0 (n, P), dz0 (6, n, P) -> (z_h, dz_h)"""
    def slope(z, dz):
        zw = np.sum(weight * z, axis=0)
        dzw = np.sum(weight * dz, axis=1)
        g = (kappa1 + kappa2 * zw) * (theta - zw)
        dg = (dk1[:, None] + dk2[:, None] * zw + kappa2 * dzw) * (theta - zw) + (kappa1 + kappa2 * zw) * (dtheta[:, None] - dzw)
        return -nodes * (z - v0) + g, -nodes * (dz - dv0[:, None, None]) + dg[:, None, :]
    s1, d1 = slope(z0, dz0)
    s2, d2 = slope(z0 + 0.5 * h * s1, dz0 + 0.5 * h * d1)
    s3, d3 = slope(z0 + 0.5 * h * s2, dz0 + 0.5 * h * d2)
    s4, d4 = slope(z0 + h * s3, dz0 + h * d3)
    return z0 + (h / 6.0) * (s1 + 2.0 * s2 + 2.0 * s3 + s4), dz0 + (h / 6.0) * (d1 + 2.0 * d2 + 2.0 * d3 + d4)


def step_tangent(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, log_s, v, y, dls, dv, dy, h, z0, z1):
    """``oracle.rough.step`` (same operations, same state) with tangents.  nodes / weights (n,), v (n, P), dv (6, n, P), dls / dy (6, P).
    Returns (vol_h, y_h, log_spot_h, dvol_h, dy_h, dls_h)."""
    weights, nodes = np.asarray(weights, dtype=float), np.asarray(nodes, dtype=float)
    k = tangent_consts(weights, sigma0, beta, orthog_vol)
    w, x = weights[:, None], nodes[:, None]
    W = np.sum(weights)
    v0 = sigma0 / W
    volvol = np.sqrt(beta ** 2 + orthog_vol ** 2)
    rho = beta / volvol
    vv = volvol * W
    D, dD = drift_rk4_tangent(x, w, v0, k["dv0"], theta, k["dtheta"], kappa1, k["dk1"], kappa2, k["dk2"], v, dv, 0.5 * h)
    # diffusion_exact: Yh = yw e^ex, shared shift (Yh - yw) / W
    yw = np.sum(w * D, axis=0)
    dyw = np.sum(w * dD, axis=1)
    ee = np.exp(-0.5 * vv ** 2 * h + vv * (z0 * np.sqrt(h)))
    dex = k["dvv"][:, None] * (np.sqrt(h) * z0 - vv * h)
    S = D + (1.0 / W * (yw * ee - yw))[None, :]
    dS = dD + ((ee * (dyw + yw * dex) - dyw) / W)[:, None, :]
    vol_h, dvol_h = drift_rk4_tangent(x, w, v0, k["dv0"], theta, k["dtheta"], kappa1, k["dk1"], kappa2, k["dk2"], S, dS, 0.5 * h)
    w_vol_h = np.sum(w * vol_h, axis=0)
    bad = np.isnan(w_vol_h) | (w_vol_h <= 0.0)
    vol_h[:, bad] = 1e-6
    dvol_h[:, :, bad] = 0.0
    wlam = w * x
    vw, volw_h = np.sum(w * v, axis=0), np.sum(w * vol_h, axis=0)
    dvw, dvhw = np.sum(w * dv, axis=1), np.sum(w * dvol_h, axis=1)
    dwlv, dwlvh = np.sum(wlam * dv, axis=1), np.sum(wlam * dvol_h, axis=1)
    w_inv = 1.0 / W
    rho_comp = np.sqrt(1.0 - rho * rho)
    w_lam_v0 = np.sum(wlam * v0)
    dwlv0 = np.sum(wlam) * k["dv0"]
    A = (((volw_h - vw) / h + 0.5 * np.sum(wlam * v, axis=0) + 0.5 * np.sum(wlam * vol_h, axis=0) - w_lam_v0) * w_inv
         - kappa1 * theta + (kappa1 - kappa2 * theta) * (0.5 * vw + 0.5 * volw_h) + kappa2 * (0.5 * vw ** 2 + 0.5 * volw_h ** 2))
    dk1, dk2, dth = k["dk1"][:, None], k["dk2"][:, None], k["dtheta"][:, None]
    dA = (((dvhw - dvw) / h + 0.5 * dwlv + 0.5 * dwlvh - dwlv0[:, None]) * w_inv - (dk1 * theta + kappa1 * dth)
          + (dk1 - dk2 * theta - kappa2 * dth) * (0.5 * vw + 0.5 * volw_h) + (kappa1 - kappa2 * theta) * (0.5 * dvw + 0.5 * dvhw)
          + dk2 * (0.5 * vw ** 2 + 0.5 * volw_h ** 2) + kappa2 * (vw * dvw + volw_h * dvhw))
    term1 = 1.0 / volvol * A * h
    dterm1 = (-k["dvt"][:, None] / volvol ** 2) * A * h + dA * h / volvol
    term2 = 0.5 * h * vw ** 2 + 0.5 * h * volw_h ** 2
    dterm2 = h * (vw * dvw + volw_h * dvhw)
    sq = np.sqrt(term2)
    with np.errstate(divide="ignore", invalid="ignore"):
        dsq = np.where(term2 > 0.0, dterm2 / (2.0 * sq), 0.0)
    vol_r, y_h, log_spot_h = _step_primal(nodes, weights, v0, theta, kappa1, kappa2, log_s, v, y, rho, volvol, h, z0, z1)
    dls_h = dls - 0.5 * dterm2 + k["drho"][:, None] * term1 + rho * dterm1 + (k["drho_comp"][:, None] * sq + rho_comp * dsq) * z1
    return vol_r, y_h, log_spot_h, dvol_h, dy + dterm2, dls_h


def _step_primal(nodes, weights, v0, theta, kappa1, kappa2, log_s, v, y, rho, volvol, h, z0, z1):
    """the state itself through ``oracle.rough.step`` unchanged"""
    from . import rough
    P = v.shape[1]
    n_vec, w_vec = np.repeat(nodes[:, None], P, axis=1), np.repeat(weights[:, None], P, axis=1)
    vol_h, y_h, ls_h = rough.step(n_vec, w_vec, np.full((nodes.size, P), v0), theta, kappa1, kappa2, np.atleast_2d(log_s), v,
                                  np.atleast_2d(y), rho, volvol, h, z0, z1)
    return vol_h, y_h[0], ls_h[0]


def path_tangents(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, grid, Z0, Z1):
    """one maturity from t = 0 on its own grid: (log_spot (P,), vol (n, P), qv (P,), dls (6, P), dvol (6, n, P), dqv (6, P), reset (P,)),
    reset = the path took the reset-to-1e-6 branch at some step of the grid"""
    weights, nodes = np.asarray(weights, dtype=float), np.asarray(nodes, dtype=float)
    n, P = nodes.size, Z0.shape[1]
    h = grid[1] - grid[0]
    W = np.sum(weights)
    k = tangent_consts(weights, sigma0, beta, orthog_vol)
    v = np.full((n, P), sigma0 / W)
    dv = np.repeat(np.repeat(k["dv0"][:, None, None], n, axis=1), P, axis=2)
    ls, y, dls, dy = np.zeros(P), np.zeros(P), np.zeros((6, P)), np.zeros((6, P))
    reset = np.zeros(P, dtype=bool)
    for s in range(grid.size - 1):
        v, y, ls, dv, dy, dls = step_tangent(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, ls, v, y, dls, dv, dy, h,
                                             Z0[s], Z1[s])
        reset |= np.all(v == 1e-6, axis=0)
    return ls, v, y, dls, dv, dy, reset


def rough_chain_greeks_fixed(ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0, Z1, sigma0, theta, kappa1, kappa2, beta, orthog_vol,
                             weights, nodes, timegrids, variable_type: int = 1, return_states: bool = False):
    """``oracle.rough.rough_chain_fixed`` with pathwise sensitivities: (prices, route "stds", greeks [7, J], greeks_se [7, J]) per maturity,
    the stds un-normalised like the route's (discfactor * nanstd(payoff)); with ``return_states`` also the path_tangents tuple per maturity."""
    P = Z0.shape[1]
    out = ([], [], [], [])
    states = []
    for ttm, fwd, df, K, T, grid in zip(ttms, forwards, discfactors, strikes_ttms, types_ttms, timegrids):
        S = grid.size - 1
        st = path_tangents(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, grid, Z0[:S], Z1[:S])
        ls, _, qv, dls, _, dqv, _ = st
        p, e, g, gse = mc_payoff_greeks(ls, qv, dls, dqv, ttm, fwd, K, T, df, variable_type)
        for acc, r in zip(out, (p, e * np.sqrt(P), g, gse)):
            acc.append(r)
        states.append(st)
    return out + (states,) if return_states else out
