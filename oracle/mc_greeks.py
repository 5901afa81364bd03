"""oracle.mc_greeks -- numpy forward-mode (tangent-linear) restatement of the fixed-normal steppers of ``oracle.mc`` and of the
pathwise payoff sensitivities with forward re-centring.  TEST INFRASTRUCTURE ONLY; written from DESIGN.md §3.9, not from the kernel.

Parameters are differentiated in dataclass field order:
  LogSV  ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")   kappa2 held fixed when kappa1 / theta move
  Heston ("v0", "theta", "kappa", "rho", "volvol")
Tangent arrays are [P, N].  Greeks arrays are [1 + P, J]: row 0 = d price / d forward, then the parameters.
"""
from __future__ import annotations

import numpy as np

from .mc import LOG_RETURN, Q_VAR

LOGSV_PARAMS = ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")
HESTON_PARAMS = ("v0", "theta", "kappa", "rho", "volvol")


def logsv_tangent_step_fixed(x, sigma, qvar, dx, dsigma, dq, Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, eta=1.0,
                             is_spot_measure=True):
    """``oracle.mc.logsv_step_fixed`` with its tangents.  dx, dsigma, dq: [6, N] tangents of the initial state.
    Returns (x, sigma, qvar, dx, dsigma, dq) at the end of the steps."""
    x, sigma, qvar = (np.array(a, dtype=np.float64, copy=True) for a in (x, sigma, qvar))
    dx, dq = (np.array(a, dtype=np.float64, copy=True) for a in (dx, dq))
    sdt = np.sqrt(dt)
    alpha, adj, dadj_dbeta = (-1.0, 0.0, 0.0) if is_spot_measure else (1.0, beta * eta, eta)
    vartheta2 = beta * beta + volvol * volvol
    eta2 = eta * eta
    L = np.log(sigma)
    dL = np.asarray(dsigma, dtype=np.float64) / sigma                 # d log sigma
    for z0, z1 in zip(Z0, Z1):
        w0, w1 = sdt * z0, sdt * z1
        s2dt = eta2 * sigma * sigma * dt
        x = x + alpha * 0.5 * s2dt + eta * sigma * w0
        dx = dx + (alpha * s2dt + eta * sigma * w0) * dL             # d/dL of alpha/2 eta^2 e^{2L} dt + eta e^L w0
        drift = (kappa1 * theta / sigma - kappa1) + kappa2 * (theta - sigma) + adj * sigma - 0.5 * vartheta2
        jac = 1.0 + (-kappa1 * theta / sigma - kappa2 * sigma + adj * sigma) * dt
        drive = np.stack([np.zeros_like(sigma),                                   # sigma0
                          (kappa1 / sigma + kappa2) * dt,                         # theta
                          (theta / sigma - 1.0) * dt,                             # kappa1
                          (theta - sigma) * dt,                                   # kappa2
                          (dadj_dbeta * sigma - beta) * dt + w0,                  # beta
                          -volvol * dt + w1])                                     # volvol
        L = L + drift * dt + beta * w0 + volvol * w1
        dL_new = jac * dL + drive
        sigma_new = np.exp(L)
        qvar = qvar + 0.5 * (s2dt + eta2 * sigma_new * sigma_new * dt)
        dq = dq + s2dt * dL + eta2 * sigma_new * sigma_new * dt * dL_new
        sigma, dL = sigma_new, dL_new
    return x, sigma, qvar, dx, sigma * dL, dq


def heston_tangent_step_fixed(x, var, qvar, dx, dvar, dq, Z0, Z1, dt, theta, kappa, rho, volvol):
    """``oracle.mc.heston_step_fixed`` (floor-Euler) with its tangents; a step on which the floor binds has a zero variance tangent."""
    x, var, qvar = (np.array(a, dtype=np.float64, copy=True) for a in (x, var, qvar))
    dx, dv, dq = (np.array(a, dtype=np.float64, copy=True) for a in (dx, dvar, dq))
    sdt = np.sqrt(dt)
    rho_1 = np.sqrt(1.0 - rho * rho)
    for z0, z1 in zip(Z0, Z1):
        w0, w1 = sdt * z0, sdt * z1
        sig = np.sqrt(var)
        vdt = var * dt
        x = x - 0.5 * vdt + sig * w0
        dx = dx + (-0.5 * dt + w0 / (2.0 * sig)) * dv
        qvar = qvar + vdt
        dq = dq + dt * dv
        noise = rho * w0 + rho_1 * w1
        vn = var + kappa * (theta - var) * dt + sig * volvol * noise
        jac = 1.0 - kappa * dt + volvol * noise / (2.0 * sig)
        drive = np.stack([np.zeros_like(var),                                     # v0
                          kappa * dt * np.ones_like(var),                         # theta
                          (theta - var) * dt,                                     # kappa
                          sig * volvol * (w0 - rho / rho_1 * w1),                 # rho
                          sig * noise])                                           # volvol
        dv = np.where(vn > 1e-4, jac * dv + drive, 0.0)
        var = np.maximum(vn, 1e-4)
    return x, var, qvar, dx, dv, dq


def mc_payoff_greeks(x, qvar, dx, dq, ttm, forward, strikes, types, discfactor=1.0, variable_type=LOG_RETURN):
    """``oracle.mc.mc_payoffs`` plus pathwise sensitivities: (prices, std errors, greeks [1+P, J], greeks_se [1+P, J]).

    S_i = F e^{x_i} - (nanmean_j F e^{x_j} - F); dS_i/dp = F e^{x_i} dx_i - nanmean_j(F e^{x_j} dx_j); dS_i/dF = S_i/F.
    U = S (LOG_RETURN) or q/ttm (Q_VAR, dU/dp = dq/ttm, dU/dF = 0).  pay = h(U) for C/P, h(U)/S for IC/IP with h = (U-K)^+ / (K-U)^+;
    g = h'(U) dU, resp. (h'(U) dU - pay dS)/S.  Paths with a NaN payoff are skipped for the price and its sensitivities."""
    fe = forward * np.exp(x)
    spots = fe - (np.nanmean(fe) - forward)
    valid = ~np.isnan(fe)
    mean_d = np.array([np.mean((fe * d)[valid]) for d in dx])
    dS = np.vstack([spots / forward, fe * dx - mean_d[:, None]])
    if variable_type == LOG_RETURN:
        under, dU = spots, dS
    elif variable_type == Q_VAR:
        under = qvar / ttm
        dU = np.vstack([np.zeros_like(x), np.asarray(dq) / ttm])
    else:
        raise NotImplementedError
    N, J = x.shape[0], len(strikes)
    prices, stds = np.zeros(J), np.zeros(J)
    greeks, greeks_se = np.zeros((dS.shape[0], J)), np.zeros((dS.shape[0], J))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        ty = str(ty)
        if ty not in ("C", "P", "IC", "IP"):
            raise ValueError("unknown option payoff code")
        put = ty in ("P", "IP")
        with np.errstate(invalid="ignore"):
            itm = under < k if put else under > k
        h = np.where(itm, (k - under) if put else (under - k), 0.0)
        hp = np.where(itm, -1.0 if put else 1.0, 0.0)
        g = np.where(itm, hp * dU, 0.0)
        if ty in ("IC", "IP"):
            pay = h / spots
            g = (g - pay * dS) / spots
        else:
            pay = h
        ok = ~np.isnan(pay)
        prices[j] = discfactor * np.mean(pay[ok])
        stds[j] = discfactor * np.std(pay[ok])
        greeks[:, j] = discfactor * np.mean(g[:, ok], axis=1)
        greeks_se[:, j] = discfactor * np.std(g[:, ok], axis=1)
    return prices, stds / np.sqrt(N), greeks, greeks_se / np.sqrt(N)


def logsv_mc_chain_greeks_fixed(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, etas, Z0s, Z1s, dts,
                                is_spot_measure=True, variable_type=LOG_RETURN):
    """``oracle.mc.logsv_mc_chain_fixed`` with pathwise sensitivities: (prices, stds, greeks, greeks_se), one entry per maturity."""
    sigma0, theta, kappa1, kappa2, beta, volvol = params6
    n = Z0s[0].shape[1]
    x, q, s = np.zeros(n), np.zeros(n), sigma0 * np.ones(n)
    dx, dq, ds = np.zeros((6, n)), np.zeros((6, n)), np.zeros((6, n))
    ds[0] = 1.0
    out = ([], [], [], [])
    for m, ttm in enumerate(ttms):
        x, s, q, dx, ds, dq = logsv_tangent_step_fixed(x, s, q, dx, ds, dq, Z0s[m], Z1s[m], dts[m], theta, kappa1, kappa2, beta, volvol,
                                                       etas[m], is_spot_measure)
        for acc, r in zip(out, mc_payoff_greeks(x, q, dx, dq, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)):
            acc.append(r)
    return out


def heston_mc_chain_greeks_fixed(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type=LOG_RETURN):
    """``oracle.mc.heston_mc_chain_fixed`` with pathwise sensitivities: (prices, stds, greeks, greeks_se), one entry per maturity."""
    v0, theta, kappa, rho, volvol = params5
    n = Z0s[0].shape[1]
    x, q, v = np.zeros(n), np.zeros(n), v0 * np.ones(n)
    dx, dq, dv = np.zeros((5, n)), np.zeros((5, n)), np.zeros((5, n))
    dv[0] = 1.0
    out = ([], [], [], [])
    for m, ttm in enumerate(ttms):
        x, v, q, dx, dv, dq = heston_tangent_step_fixed(x, v, q, dx, dv, dq, Z0s[m], Z1s[m], dts[m], theta, kappa, rho, volvol)
        for acc, r in zip(out, mc_payoff_greeks(x, q, dx, dq, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)):
            acc.append(r)
    return out
