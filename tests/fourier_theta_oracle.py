"""Numpy restatement of the theta of the Fourier chain pricers (DESIGN.md §4.8).  TEST INFRASTRUCTURE ONLY.

theta = -d price / d ttm_m with the slice forward and discount factor, the earlier maturities, the vol backbone and the transform grid held.
The adaptive routes hold the accepted mesh of slice m and move its last step only (dh_K / dT_m = 1):

* ``last_step_theta``: Dormand-Prince replayed on a recorded mesh, plus the derivative of every step in its length at a fixed start,
  G_s = k_s + h dk_s, dY_s = sum_{j<s} a_sj G_j, dk_s = J(Y_s) dY_s, dy = sum_j b_j G_j; the last step of each point writes last;
* ``bump_last_step``: the same mesh with the last step of every point lengthened by eps (the central differences of the tests);
* ``logsv_chain_theta`` / ``hawkes_chain_theta`` / ``heston_chain_theta``: theta per maturity, d log_mgf / d T_m and the meshes;
* ``black_ivol_theta``: the implied-vol transform (theta + B_T) / vega with the NaN / bracket-end rules of the sensitivity rows.
"""
from __future__ import annotations

import numpy as np
from scipy.stats import norm

from oracle import hawkes, mgf
from oracle import hawkes_greeks as H
from oracle import mgf_greeks as G


def last_step_theta(rhs, jvp, y0, mesh):
    """(y, dy): y as mgf_greeks.replay(rhs, y0, mesh) (bit for bit), dy = d y / d (length of each point's last step)"""
    y = y0.astype(np.complex128).copy()
    dy = np.zeros_like(y)
    n = y.shape[1]
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya = y[ja]
        K = np.zeros((6, ja.shape[0], n), dtype=np.complex128)
        Gs = np.zeros((6, ja.shape[0], n), dtype=np.complex128)
        K[0] = rhs(ya, ja)
        Gs[0] = K[0]
        for s in range(1, 6):
            Ys = ya + G._stage_sum(K, mgf._A[s], s) * h[:, None]
            K[s] = rhs(Ys, ja)
            Gs[s] = K[s] + h[:, None] * jvp(Ys, G._stage_sum(Gs, mgf._A[s], s), ja)
        y[ja] = ya + h[:, None] * sum(K[j] * mgf._B[j] for j in range(6))
        dy[ja] = sum(Gs[j] * mgf._B[j] for j in range(6))
    return y, dy


def bump_last_step(mesh, eps):
    """the mesh with the last accepted step of every point lengthened by eps (shortened for eps < 0)"""
    out = [(ja, h.copy()) for ja, h in mesh]
    last = {}
    for i, (ja, _) in enumerate(mesh):
        for k, p in enumerate(ja):
            last[int(p)] = (i, k)
    for i, k in last.values():
        out[i][1][k] += eps
    return out


def _theta_rows(lm, dlm_t, phi, forward, strikes, types, discfactor, spot):
    """theta [J] of one slice: -(d price / d T) from the parameter-row formula with S_T = sum w Re(e^z d_T lm)"""
    return -G.vanilla_slice_greeks(lm, dlm_t[None], phi, forward, strikes, types, discfactor, spot)[3]


def _adaptive_chain_theta(rhs_of, jvp_of, lm_of, y0, ttms, forwards, discfactors, strikes_ttms, types_ttms, phi, spot):
    a = y0
    theta, dlm, lms, meshes = [], [], [], []
    t0 = 0.0
    for m, ttm in enumerate(ttms):
        rhs, jvp = rhs_of(m), jvp_of(m)
        a_start = a
        a, _, _, mesh = G.rk45_grid_tangent(rhs, [jvp], a, np.zeros((1,) + a.shape, dtype=np.complex128), ttm - t0)
        a_re, da = last_step_theta(rhs, jvp, a_start, mesh)
        assert np.array_equal(a_re, a)
        lm, d = lm_of(a), lm_of(da)
        theta.append(_theta_rows(lm, d, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], spot))
        dlm.append(d)
        lms.append(lm)
        meshes.append(mesh)
        t0 = ttm
    return theta, dict(dlog_mgf_theta=np.array(dlm), log_mgf=np.array(lms), meshes=meshes, phi=phi)


def logsv_jvp(params6, eta, phi, psi, spot, order):
    """J(A) dA of the LogSV coefficient ODEs: mgf_greeks.LogsvTangentRhs with every field derivative zero"""
    f = G.logsv_fields(params6, eta, spot)
    return G.LogsvTangentRhs(f, dict.fromkeys(G.FIELDS, 0.0), phi, psi, spot, order)


def logsv_chain_theta(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, order=2, etas=None,
                      vol_scaler=None):
    """theta per maturity ([J_m] each) and dict(dlog_mgf_theta [M, P], log_mgf [M, P], meshes, phi, vol_scaler)"""
    if vol_scaler is None:
        vol_scaler = mgf.logsv_vol_scaler(params6[0], ttms)
    phi = mgf.phi_grid(vol_scaler, is_spot_measure)
    psi = np.zeros_like(phi)
    n = mgf.expansion_n(order)
    etas = np.ones(len(ttms)) if etas is None else etas
    yv = params6[0] - params6[1]
    ys = np.array([1.0, yv, yv * yv, yv * yv * yv, (yv * yv) * (yv * yv)])[:n] + 0j
    theta, grids = _adaptive_chain_theta(lambda m: mgf.LogsvRhs(*params6[1:], phi, psi, is_spot_measure, order, etas[m]),
                                         lambda m: logsv_jvp(params6, etas[m], phi, psi, is_spot_measure, order), lambda a: a @ ys,
                                         np.zeros((phi.shape[0], n), dtype=np.complex128), ttms, forwards, discfactors, strikes_ttms,
                                         types_ttms, phi, is_spot_measure)
    grids["vol_scaler"] = vol_scaler
    return theta, grids


def hawkes_jvp(p, phi, psi):
    """J(A) dA of the Hawkes Riccati system: hawkes_greeks.HawkesTangentRhs with every constant derivative zero"""
    j = H.HawkesTangentRhs(p, H.ODE_NAMES[0], phi, psi)
    j.d = dict.fromkeys(j.d, 0.0)
    j.dcomp_p = j.dcomp_m = 0.0
    return j


def hawkes_chain_theta(p: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, vol_scaler=None):
    """the Hawkes twin of logsv_chain_theta (no risk kernel)"""
    if vol_scaler is None:
        vol_scaler = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    phi = mgf.phi_grid(vol_scaler, True, hawkes.MAX_PHI)
    psi = np.zeros_like(phi)
    rhs, jvp = hawkes.HawkesRhs(p, phi, psi), hawkes_jvp(p, phi, psi)
    theta, grids = _adaptive_chain_theta(lambda m: rhs, lambda m: jvp, lambda a: a[:, 0] + a[:, 1] * p["lambda_p"] + a[:, 2] * p["lambda_m"],
                                         np.zeros((phi.shape[0], 3), dtype=np.complex128), ttms, forwards, discfactors, strikes_ttms,
                                         types_ttms, phi, is_spot_measure)
    grids["vol_scaler"] = vol_scaler
    return theta, grids


def heston_chain_theta(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None):
    """the Heston closed form on dual numbers in the slice length (derivatives of (a, b) zeroed at every slice start): theta per maturity
    and dlog_mgf_theta [M, P]"""
    v0, theta_, kappa, rho, volvol = params5
    if vol_scaler is None:
        vol_scaler = mgf.heston_vol_scaler(v0, ttms)
    phi = mgf.phi_grid(vol_scaler, True)
    vv2 = volvol * volvol
    b1 = kappa + rho * volvol * phi
    zeta = np.sqrt(b1 * b1 - 2.0 * (0.5 * phi * (phi + 1.0)) * vv2)
    psi_p, psi_m = -b1 + zeta, b1 + zeta
    a, b = np.zeros_like(phi), np.zeros_like(phi)
    out, dlm = [], []
    t0 = 0.0
    for m, ttm in enumerate(ttms):
        tau = G._Dual(ttm - t0, 1.0)
        bd = G._Dual(b)
        ez = (-(tau * zeta)).exp()
        c_p, c_m = (psi_p + vv2 * bd) / (2.0 * zeta), (psi_m - vv2 * bd) / (2.0 * zeta)
        bn = -(-psi_m * c_p * ez + psi_p * c_m) / (vv2 * (c_p * ez + c_m))
        an = -(theta_ * kappa / vv2) * (tau * psi_p + 2.0 * (c_p * ez + c_m).log()) + G._Dual(a)
        a, b = an.v, bn.v
        d = an.d + bn.d * v0
        out.append(_theta_rows(a + b * v0, d, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], True))
        dlm.append(d)
        t0 = ttm
    return out, np.array(dlm)


# ---- the Black-76 transform ----------------------------------------------------------------------------------------------------------
VOL_LO, VOL_HI = 1e-8, 10.0


def black_price(forward, strike, ttm, vol, is_call, discfactor=1.0):
    s = vol * np.sqrt(ttm)
    d1 = np.log(forward / strike) / s + 0.5 * s
    d2 = d1 - s
    c = forward * norm.cdf(d1) - strike * norm.cdf(d2)
    return discfactor * (c if is_call else c - forward + strike)


def black_vega(forward, strike, ttm, vol, discfactor=1.0):
    s = vol * np.sqrt(ttm)
    d1 = np.log(forward / strike) / s + 0.5 * s
    return discfactor * forward * norm.pdf(d1) * np.sqrt(ttm)


def black_ivol_theta(forward, strike, ttm, discfactor, vol, theta):
    """-d ivol / d ttm = (theta + B_T) / vega, B_T = vega vol / (2 ttm); NaN for a NaN ivol, 0 at an end of the bracket"""
    if vol != vol:
        return np.nan
    if vol <= VOL_LO * (1.0 + 1e-10) or vol >= VOL_HI * (1.0 - 1e-10):
        return 0.0
    vega = black_vega(forward, strike, ttm, vol, discfactor)
    return (theta + vega * vol / (2.0 * ttm)) / vega
