"""oracle.mc_gamma -- numpy restatement of the Monte Carlo gamma of the LogSV / Heston chain pricers by conditional smoothing of the
log-spot's last step.  TEST INFRASTRUCTURE ONLY; written from DESIGN.md §3.9, not from the kernel, on top of ``oracle.mc``.

Given the state before the last step of a slice, the log-spot's last step is Gaussian, x_S = mu + s Z:
  LogSV   s = eta sqrt(dt) sigma_{S-1}        Heston  s = sqrt(v_{S-1} dt)
and mu = x_S - s z0_S.  With the other paths held fixed, the re-centred spot S_i = Y_i - (mean_j Y_j - F), Y = F e^x, is
S_i = (1 - 1/n) F e^{mu_i + s_i Z} - c_i, c_i = (sum_{j != i} Y_j)/n - F, with density f_i(k) = phi(d) / ((k + c_i) s_i),
d = ln((k + c_i) / A_i) / s_i, A_i = (1 - 1/n) F e^{mu_i} (0 where k + c_i <= 0).  Per-path gamma terms:
  LOG_RETURN  C, P: (K/F)^2 f_i(K)    IC: (K/F^2) f_i(K) - 2K/(F^2 S_i) 1{S_i > K}    IP: (K/F^2) f_i(K) + 2K/(F^2 S_i) 1{S_i < K}
  Q_VAR       C, P: 0                  IC, IP: 2 pay_i / F^2
"""
from __future__ import annotations

import numpy as np

from .mc import LOG_RETURN, Q_VAR, heston_step_fixed, logsv_step_fixed, mc_payoffs


def logsv_step_fixed_laststep(x, sigma, qvar, Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, eta=1.0, is_spot_measure=True):
    """``oracle.mc.logsv_step_fixed`` that also returns the last step's (s, mu): (x, sigma, qvar, s, mu)"""
    x, sigma, qvar = logsv_step_fixed(x, sigma, qvar, Z0[:-1], Z1[:-1], dt, theta, kappa1, kappa2, beta, volvol, eta, is_spot_measure)
    s = eta * np.sqrt(dt) * sigma
    x, sigma, qvar = logsv_step_fixed(x, sigma, qvar, Z0[-1:], Z1[-1:], dt, theta, kappa1, kappa2, beta, volvol, eta, is_spot_measure)
    return x, sigma, qvar, s, x - s * Z0[-1]


def heston_step_fixed_laststep(x, var, qvar, Z0, Z1, dt, theta, kappa, rho, volvol):
    """``oracle.mc.heston_step_fixed`` (floor-Euler) that also returns the last step's (s, mu): (x, var, qvar, s, mu)"""
    x, var, qvar = heston_step_fixed(x, var, qvar, Z0[:-1], Z1[:-1], dt, theta, kappa, rho, volvol)
    s = np.sqrt(var * dt)
    x, var, qvar = heston_step_fixed(x, var, qvar, Z0[-1:], Z1[-1:], dt, theta, kappa, rho, volvol)
    return x, var, qvar, s, x - s * Z0[-1]


def mc_payoff_gamma(x, qvar, s, mu, ttm, forward, strikes, types, discfactor=1.0, variable_type=LOG_RETURN):
    """(gamma [J], gamma_se [J]): discfactor * mean / std(per-path term) over the paths with a non-NaN payoff, std / sqrt(len(x))"""
    fe = forward * np.exp(x)
    valid = ~np.isnan(fe)
    n = np.count_nonzero(valid)
    corr = np.mean(fe[valid]) - forward
    spots = fe - corr
    c = corr - fe / n                                             # (sum_{j != i} Y_j)/n - F
    log_a = np.log((1.0 - 1.0 / n) * forward) + mu
    if variable_type == LOG_RETURN:
        under = spots
    elif variable_type == Q_VAR:
        under = qvar / ttm
    else:
        raise NotImplementedError
    gamma, gamma_se = np.zeros(len(strikes)), np.zeros(len(strikes))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        ty = str(ty)
        if ty not in ("C", "P", "IC", "IP"):
            raise ValueError("unknown option payoff code")
        put, inverse = ty in ("P", "IP"), ty in ("IC", "IP")
        with np.errstate(invalid="ignore", divide="ignore"):
            itm = under < k if put else under > k
            h = np.where(itm, (k - under) if put else (under - k), 0.0)
            pay = h / spots if inverse else h
            kc = k + c
            d = (np.log(np.where(kc > 0.0, kc, 1.0)) - log_a) / s
            dens = np.where(kc > 0.0, np.exp(-0.5 * d * d) / (np.sqrt(2.0 * np.pi) * kc * s), 0.0)
            if variable_type == Q_VAR:
                g = 2.0 * pay / forward ** 2 if inverse else np.zeros_like(pay)
            elif inverse:
                g = k / forward ** 2 * dens + np.where(itm, (2.0 if put else -2.0) * k / (forward ** 2 * spots), 0.0)
            else:
                g = (k / forward) ** 2 * dens
        ok = ~np.isnan(pay)
        gamma[j] = discfactor * np.mean(g[ok])
        gamma_se[j] = discfactor * np.std(g[ok])
    return gamma, gamma_se / np.sqrt(x.shape[0])


def logsv_mc_chain_gamma_fixed(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, etas, Z0s, Z1s, dts, is_spot_measure=True,
                               variable_type=LOG_RETURN, return_states=False):
    """``oracle.mc.logsv_mc_chain_fixed`` with the smoothed gamma: (prices, stds, gamma, gamma_se[, states]) per maturity, states =
    (x, sigma, qvar, s, mu)"""
    sigma0, theta, kappa1, kappa2, beta, volvol = params6
    n = Z0s[0].shape[1]
    x, q, v = np.zeros(n), np.zeros(n), sigma0 * np.ones(n)
    out = ([], [], [], [], [])
    for m, ttm in enumerate(ttms):
        x, v, q, s, mu = logsv_step_fixed_laststep(x, v, q, Z0s[m], Z1s[m], dts[m], theta, kappa1, kappa2, beta, volvol, etas[m], is_spot_measure)
        _accumulate(out, x, v, q, s, mu, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
    return out if return_states else out[:4]


def heston_mc_chain_gamma_fixed(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type=LOG_RETURN,
                                return_states=False):
    """``oracle.mc.heston_mc_chain_fixed`` with the smoothed gamma, as logsv_mc_chain_gamma_fixed"""
    v0, theta, kappa, rho, volvol = params5
    n = Z0s[0].shape[1]
    x, q, v = np.zeros(n), np.zeros(n), v0 * np.ones(n)
    out = ([], [], [], [], [])
    for m, ttm in enumerate(ttms):
        x, v, q, s, mu = heston_step_fixed_laststep(x, v, q, Z0s[m], Z1s[m], dts[m], theta, kappa, rho, volvol)
        _accumulate(out, x, v, q, s, mu, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
    return out if return_states else out[:4]


def _accumulate(out, x, v, q, s, mu, ttm, forward, strikes, types, discfactor, variable_type):
    p, e = mc_payoffs(x, q, ttm, forward, strikes, types, discfactor, variable_type)
    g, ge = mc_payoff_gamma(x, q, s, mu, ttm, forward, strikes, types, discfactor, variable_type)
    for acc, r in zip(out, (p, e, g, ge, (x.copy(), v.copy(), q.copy(), s, mu))):
        acc.append(r)
