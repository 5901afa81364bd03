"""oracle.hawkes_mc_greeks -- numpy restatement of the Hawkes jump-diffusion Monte Carlo sensitivities: the tangent-linear recursion of
``oracle.hawkes.step_fixed`` with the firing decisions frozen, the likelihood-ratio score of the decisions, and the payoff estimator with
forward re-centring.  TEST INFRASTRUCTURE ONLY; written from DESIGN.md §3.11, not from the kernel: full [15, N] tangents of x and of both
intensities and the score are updated at every step (no running sums, no sparsity).

Inputs are the reference-form draws (W0, U_P, U_M, J_P, J_M) of ``oracle.hawkes``: a clock fires when lambda > U (U = -ln(u)/dt), so
P(fire) = 1 - exp(-lambda dt) for lambda > 0 and 0 otherwise.  A firing step adds dlambda dt / expm1(lambda dt) to the score, a silent step
with lambda > 0 adds -dt dlambda, lambda taken at the step start.  Directions in ``PARAMS`` order (HAWKES_GREEK_PARAMS of the package).
"""
from __future__ import annotations

import numpy as np

PARAMS = ("sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p", "lambda_m", "theta_m",
          "kappa_m", "beta1_m", "beta2_m")
NP = len(PARAMS)


def _e(name):
    e = np.zeros((NP, 1))
    e[PARAMS.index(name)] = 1.0
    return e


def initial_tangents(nb_path):
    """(dx, dlp, dlm, score) at t = 0: only lambda_p(0) / lambda_m(0) move the intensities"""
    dlp, dlm = np.zeros((NP, nb_path)), np.zeros((NP, nb_path))
    dlp[PARAMS.index("lambda_p")] = 1.0
    dlm[PARAMS.index("lambda_m")] = 1.0
    return np.zeros((NP, nb_path)), dlp, dlm, np.zeros((NP, nb_path))


def tangent_step_fixed(x, lp, lm, dx, dlp, dlm, score, W0, U_P, U_M, J_P, J_M, dt, mu, sigma, shift_p, mean_p, shift_m, mean_m, theta_p, kappa_p,
                       beta1_p, beta2_p, theta_m, kappa_m, beta1_m, beta2_m, return_fires=False, **_):
    """``oracle.hawkes.step_fixed`` (same operations, same state) with tangents dx, dlp, dlm and the score, each [15, N].
    Returns (x, lp, lm, dx, dlp, dlm, score), plus the decisions fires [S, 2, N] with ``return_fires``."""
    comp_p = dt * (np.exp(shift_p) / (1.0 - mean_p) - 1.0)
    comp_m = dt * (np.exp(shift_m) / (1.0 - mean_m) - 1.0)
    gp, gm = dt * np.exp(shift_p) / (1.0 - mean_p), dt * np.exp(shift_m) / (1.0 - mean_m)
    dcomp_p = gp * _e("shift_p") + gp / (1.0 - mean_p) * _e("mean_p")
    dcomp_m = gm * _e("shift_m") + gm / (1.0 - mean_m) * _e("mean_m")
    drift_dt = (mu - 0.5 * sigma * sigma) * dt
    x, lp, lm = x.copy(), lp.copy(), lm.copy()
    dx, dlp, dlm, score = dx.copy(), dlp.copy(), dlm.copy(), score.copy()
    fires = []
    for w0, u_p, u_m, j_p, j_m in zip(W0, U_P, U_M, J_P, J_M):
        fire_p, fire_m = lp > u_p, lm > u_m
        fires.append((fire_p, fire_m))
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            wp = np.where(fire_p, dt / np.expm1(lp * dt), np.where(lp > 0.0, -dt, 0.0))
            wm = np.where(fire_m, dt / np.expm1(lm * dt), np.where(lm > 0.0, -dt, 0.0))
        score = score + wp * dlp + wm * dlm
        jump_p = np.where(fire_p, j_p, 0.0)
        jump_m = np.where(fire_m, j_m, 0.0)
        dJp = np.where(fire_p, _e("shift_p") + _e("mean_p") * ((j_p - shift_p) / mean_p), 0.0)      # J = shift + mean E
        dJm = np.where(fire_m, _e("shift_m") + _e("mean_m") * ((j_m - shift_m) / mean_m), 0.0)
        dx = (dx - dcomp_p * lp - comp_p * dlp - dcomp_m * lm - comp_m * dlm + _e("sigma") * (w0 - sigma * dt) + dJp + dJm)
        dload_p = _e("beta1_p") * jump_p + beta1_p * dJp + _e("beta2_p") * jump_m + beta2_p * dJm
        dload_m = _e("beta1_m") * jump_p + beta1_m * dJp + _e("beta2_m") * jump_m + beta2_m * dJm
        dlp = dlp + (_e("kappa_p") * (theta_p - lp) + kappa_p * (_e("theta_p") - dlp)) * dt + dload_p
        dlm = dlm + (_e("kappa_m") * (theta_m - lm) + kappa_m * (_e("theta_m") - dlm)) * dt + dload_m
        # the primal exactly as oracle.hawkes.step_fixed
        diffusion = drift_dt - comp_p * lp - comp_m * lm + sigma * w0
        x = x + diffusion + jump_p + jump_m
        load_p = beta1_p * jump_p + beta2_p * jump_m
        load_m = beta1_m * jump_p + beta2_m * jump_m
        lp = lp + kappa_p * (theta_p - lp) * dt + load_p
        lm = lm + kappa_m * (theta_m - lm) * dt + load_m
    out = (x, lp, lm, dx, dlp, dlm, score)
    return out + (np.array(fires),) if return_fires else out


def payoff_greeks(x, dx, score, forward, strikes, types, discfactor=1.0):
    """LOG_RETURN payoffs of ``oracle.mc.mc_payoffs`` with the mixed estimator: (prices, std errors, greeks [16, J], greeks_se [16, J]).

    S_i = F e^{x_i} - (mean_j F e^{x_j} - F); the re-centring differentiates its expectation: dS_i = F e^{x_i} dx_i - mean_j F e^{x_j}
    (dx_j + score_j); dS/dF = S/F (delta is pathwise).  pay = h(S) (C/P) or h(S)/S (IC/IP); g_p = (pathwise g of DESIGN §3.9) + pay score_p."""
    fe = forward * np.exp(x)
    spots = fe - (np.nanmean(fe) - forward)
    valid = ~np.isnan(fe)
    mean_d = np.array([np.mean((fe * (d + s))[valid]) for d, s in zip(dx, score)])
    dS = np.vstack([spots / forward, fe * dx - mean_d[:, None]])
    lr = np.vstack([np.zeros_like(x), score])
    N, J = x.shape[0], len(strikes)
    prices, stds = np.zeros(J), np.zeros(J)
    greeks, greeks_se = np.zeros((1 + NP, J)), np.zeros((1 + NP, J))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        ty = str(ty)
        if ty not in ("C", "P", "IC", "IP"):
            raise ValueError("unknown option payoff code")
        put = ty in ("P", "IP")
        with np.errstate(invalid="ignore"):
            itm = spots < k if put else spots > k
        h = np.where(itm, (k - spots) if put else (spots - k), 0.0)
        g = np.where(itm, (-1.0 if put else 1.0) * dS, 0.0)
        if ty in ("IC", "IP"):
            pay = h / spots
            g = (g - pay * dS) / spots
        else:
            pay = h
        g = g + pay * lr
        ok = ~np.isnan(pay)
        prices[j] = discfactor * np.mean(pay[ok])
        stds[j] = discfactor * np.std(pay[ok])
        greeks[:, j] = discfactor * np.mean(g[:, ok], axis=1)
        greeks_se[:, j] = discfactor * np.std(g[:, ok], axis=1)
    return prices, stds / np.sqrt(N), greeks, greeks_se / np.sqrt(N)


def chain_greeks_fixed(params: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, inputs, return_paths=False):
    """``oracle.hawkes.chain_prices`` on the per-slice draws ``inputs`` (W0, U_P, U_M, J_P, J_M, dt) with sensitivities: (prices, stds,
    greeks, greeks_se), one entry per maturity; with ``return_paths`` also per maturity (x, lp, lm, dx, dlp, dlm, score)."""
    n = inputs[0][0].shape[1]
    x, lp, lm = np.zeros(n), params["lambda_p"] * np.ones(n), params["lambda_m"] * np.ones(n)
    dx, dlp, dlm, score = initial_tangents(n)
    kw = {k: v for k, v in params.items() if k not in ("lambda_p", "lambda_m")}
    out, paths = ([], [], [], []), []
    for m, (fwd, df, K, T) in enumerate(zip(forwards, discfactors, strikes_ttms, types_ttms)):
        x, lp, lm, dx, dlp, dlm, score = tangent_step_fixed(x, lp, lm, dx, dlp, dlm, score, *inputs[m], **kw)
        for acc, r in zip(out, payoff_greeks(x, dx, score, fwd, K, T, df)):
            acc.append(r)
        paths.append((x, lp, lm, dx, dlp, dlm, score))
    return out + (paths,) if return_paths else out
