"""oracle.mc_theta -- numpy restatement of the Monte Carlo theta of the LogSV, Heston and rough-LogSV chain pricers: the tangent of each slice in its
step length dt with the step count S held.  TEST INFRASTRUCTURE ONLY; written from DESIGN.md §3.12, not from the kernel, on top of
``oracle.mc`` and ``oracle.mc_greeks``.

Slice m runs S_m steps of dt_m = (ttm_m - ttm_{m-1}) / S_m, so d/d ttm_m = (1/S_m) d/d dt_m.  The tangent is 0 at the slice's start and
does not carry into the next slice.  Every step constant is proportional to dt or sqrt(dt):
  LogSV   dL' = dL (1 - a1/sigma + a2 sigma) + (a0 + a1/sigma + a2 sigma)/dt + (b0 z0 + b1 z1)/(2 dt)          (0 through a clamp)
          dx += (2 cx sigma^2 + ce sigma z0) dL + (cx sigma^2 + ce sigma z0 / 2)/dt                          (old sigma)
          dq += 2 cq (sigma^2 dL + sigma'^2 dL') + cq (sigma^2 + sigma'^2)/dt
  Heston  dv' = dv (1 - kappa dt) + kappa (theta - v) + dv (c0 z0 + c1 z1)/(2 sqrt v) + sqrt(v) (c0 z0 + c1 z1)/(2 dt)   (0 at the floor)
          dx += (-dt/2 + sqrt(dt) z0 / (2 sqrt v)) dv - v/2 + sqrt(v) z0 / (2 sqrt dt);   dq += dt dv + v       (old v)
with a0..a2, cx, cq proportional to dt and b0, b1, ce, c0, c1 to sqrt(dt).  The payoff is differentiated as for the parameter rows with
the forward held; under Q_VAR the underlying q/ttm gives dU/d dt = (dq - S q / ttm) / ttm.  theta = -df mean(g) / S, se = df std(g) / (S sqrt N).
"""
from __future__ import annotations

import numpy as np

from .mc import LOG_RETURN, mc_payoffs
from .mc_greeks import mc_payoff_greeks


def logsv_theta_step_fixed(x, sigma, qvar, Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, eta=1.0, is_spot_measure=True):
    """``oracle.mc.logsv_step_fixed`` over one slice with the d/d dt tangent started at 0: (x, sigma, qvar, dx, dq)"""
    x, sigma, qvar = (np.array(a, dtype=np.float64, copy=True) for a in (x, sigma, qvar))
    sdt = np.sqrt(dt)
    alpha, adj = (-1.0, 0.0) if is_spot_measure else (1.0, beta * eta)
    cx, ce, cq = alpha * 0.5 * eta * eta * dt, eta * sdt, 0.5 * eta * eta * dt
    a0 = (-kappa1 + kappa2 * theta - 0.5 * (beta * beta + volvol * volvol)) * dt
    a1, a2 = kappa1 * theta * dt, (adj - kappa2) * dt
    b0, b1 = beta * sdt, volvol * sdt
    L = np.log(sigma)
    dx, dL, dq = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
    for z0, z1 in zip(Z0, Z1):
        so = sigma
        dx = dx + (2.0 * cx * so * so + ce * so * z0) * dL + (cx * so * so + 0.5 * ce * so * z0) / dt
        dLn = dL * (1.0 - a1 / so + a2 * so) + (a0 + a1 / so + a2 * so) / dt + (b0 * z0 + b1 * z1) / (2.0 * dt)
        L = L + a0 + a1 / so + a2 * so + b0 * z0 + b1 * z1
        sigma = np.exp(L)
        x = x + cx * so * so + ce * so * z0
        qvar = qvar + cq * (so * so + sigma * sigma)
        dq = dq + 2.0 * cq * (so * so * dL + sigma * sigma * dLn) + cq * (so * so + sigma * sigma) / dt
        dL = dLn
    return x, sigma, qvar, dx, dq


def heston_theta_step_fixed(x, var, qvar, Z0, Z1, dt, theta, kappa, rho, volvol):
    """``oracle.mc.heston_step_fixed`` (floor-Euler) over one slice with the d/d dt tangent started at 0: (x, var, qvar, dx, dq)"""
    x, var, qvar = (np.array(a, dtype=np.float64, copy=True) for a in (x, var, qvar))
    sdt = np.sqrt(dt)
    c0, c1 = volvol * rho * sdt, volvol * np.sqrt(1.0 - rho * rho) * sdt
    dx, dv, dq = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
    for z0, z1 in zip(Z0, Z1):
        sig = np.sqrt(var)
        noise = c0 * z0 + c1 * z1
        dx = dx + (-0.5 * dt + sdt * z0 / (2.0 * sig)) * dv - 0.5 * var + sig * z0 / (2.0 * sdt)
        dq = dq + dt * dv + var
        x = x - 0.5 * dt * var + sdt * sig * z0
        qvar = qvar + dt * var
        vn = var + kappa * dt * (theta - var) + sig * noise
        dv = np.where(vn > 1e-4, dv * (1.0 - kappa * dt) + kappa * (theta - var) + dv * noise / (2.0 * sig) + sig * noise / (2.0 * dt), 0.0)
        var = np.maximum(vn, 1e-4)
    return x, var, qvar, dx, dq


def mc_payoff_theta(x, qvar, dx, dq, S, ttm, forward, strikes, types, discfactor=1.0, variable_type=LOG_RETURN):
    """(theta [J], theta_se [J]) of one maturity from its state and its d/d dt tangents (dx, dq) over a slice of S steps"""
    dq_pay = np.asarray(dq) - S * np.asarray(qvar) / ttm
    _, _, g, ge = mc_payoff_greeks(x, qvar, np.asarray(dx)[None, :], dq_pay[None, :], ttm, forward, strikes, types, discfactor, variable_type)
    return -g[1] / S, ge[1] / S


def _chain(step, params, v0, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type, return_states):
    n = Z0s[0].shape[1]
    x, v, q = np.zeros(n), v0 * np.ones(n), np.zeros(n)
    out = ([], [], [], [], [])
    for m, ttm in enumerate(ttms):
        x, v, q, dx, dq = step(m, x, v, q, Z0s[m], Z1s[m], dts[m], params)
        S = Z0s[m].shape[0]
        p, e = mc_payoffs(x, q, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
        th, se = mc_payoff_theta(x, q, dx, dq, S, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
        for acc, r in zip(out, (p, e, th, se, (x.copy(), v.copy(), q.copy(), dx, dq))):
            acc.append(r)
    return out if return_states else out[:4]


def logsv_mc_chain_theta_fixed(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, etas, Z0s, Z1s, dts, is_spot_measure=True,
                               variable_type=LOG_RETURN, return_states=False):
    """``oracle.mc.logsv_mc_chain_fixed`` with the theta row: (prices, stds, theta, theta_se[, states]) per maturity, states =
    (x, sigma, qvar, dx, dq) with the d/d dt tangents of the maturity's slice"""
    sigma0, theta, kappa1, kappa2, beta, volvol = params6
    step = lambda m, x, v, q, Z0, Z1, dt, p: logsv_theta_step_fixed(x, v, q, Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, etas[m],
                                                                    is_spot_measure)
    return _chain(step, params6, sigma0, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type, return_states)


def heston_mc_chain_theta_fixed(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type=LOG_RETURN,
                                return_states=False):
    """``oracle.mc.heston_mc_chain_fixed`` with the theta row, as logsv_mc_chain_theta_fixed"""
    v0, theta, kappa, rho, volvol = params5
    step = lambda m, x, v, q, Z0, Z1, dt, p: heston_theta_step_fixed(x, v, q, Z0, Z1, dt, theta, kappa, rho, volvol)
    return _chain(step, params5, v0, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts, variable_type, return_states)



# ---- rough-LogSV: every maturity restarts at t = 0 on its own grid h = ttm / S, so d/d ttm = (1/S) d/d h over the whole path ------------
#   RK4 half-steps (hh = h/2): the stage tangents chained with the explicit hh-dependence of the stage points and of the combination;
#   exponent ex = vv z0 sqrt(h) - vv^2 h / 2: d ex / d h = vv z0 / (2 sqrt h) - vv^2 / 2;  term1 = (1/vartheta) ((volw_h - vw) / W + h rest),
#   term2 = h/2 (vw^2 + volw_h^2) and y are proportional to h; the reset branch has zero factor tangents.
def rough_theta_step(nodes, weights, v0, theta, kappa1, kappa2, rho, volvol, h, log_s, v, y, dls, dv, dy, z0, z1):
    """one step of ``oracle.rough.step`` with its h-tangent: (log_s, v, y, dls, dv, dy, reset); v, dv: (n, P)"""
    from . import rough
    x, w = np.asarray(nodes, dtype=float)[:, None], np.asarray(weights, dtype=float)[:, None]
    W = float(np.sum(weights))

    def slope(z):
        zw = np.sum(w * z, axis=0)
        return -x * (z - v0) + (kappa1 + kappa2 * zw) * (theta - zw)

    def dslope(z, dz):
        zw, dzw = np.sum(w * z, axis=0), np.sum(w * dz, axis=0)
        return -x * dz + dzw * (kappa2 * (theta - zw) - (kappa1 + kappa2 * zw))

    def drift(z, dz, hh, dhh):
        s1, d1 = slope(z), dslope(z, dz)
        t, dt = z + 0.5 * hh * s1, dz + 0.5 * hh * d1 + 0.5 * dhh * s1
        s2, d2 = slope(t), dslope(t, dt)
        t, dt = z + 0.5 * hh * s2, dz + 0.5 * hh * d2 + 0.5 * dhh * s2
        s3, d3 = slope(t), dslope(t, dt)
        t, dt = z + hh * s3, dz + hh * d3 + dhh * s3
        s4, d4 = slope(t), dslope(t, dt)
        S, dS = s1 + 2.0 * s2 + 2.0 * s3 + s4, d1 + 2.0 * d2 + 2.0 * d3 + d4
        return z + hh / 6.0 * S, dz + hh / 6.0 * dS + dhh / 6.0 * S

    P = v.shape[1]
    vol_h, y_h, ls_h = rough.step(np.repeat(x, P, axis=1), np.repeat(w, P, axis=1), np.full(v.shape, v0), theta, kappa1, kappa2,
                                  np.atleast_2d(log_s), v, np.atleast_2d(y), rho, volvol, h, z0, z1)
    D, dD = drift(v, dv, 0.5 * h, 0.5)
    vv = volvol * W
    yw, dyw = np.sum(w * D, axis=0), np.sum(w * dD, axis=0)
    e = np.exp(-0.5 * vv ** 2 * h + vv * z0 * np.sqrt(h))
    dex = vv * z0 / (2.0 * np.sqrt(h)) - 0.5 * vv ** 2
    Sv, dSv = D + (yw * e - yw) / W, dD + (e * (dyw + yw * dex) - dyw) / W
    _, dvh = drift(Sv, dSv, 0.5 * h, 0.5)
    reset = np.all(vol_h == 1e-6, axis=0)
    dvh[:, reset] = 0.0
    vw, vhw = np.sum(w * v, axis=0), np.sum(w * vol_h, axis=0)
    dvw, dvhw = np.sum(w * dv, axis=0), np.sum(w * dvh, axis=0)
    wl = w * x
    wlv, wlvh, wlv0 = np.sum(wl * v, axis=0), np.sum(wl * vol_h, axis=0), float(np.sum(wl)) * v0
    dwlv, dwlvh = np.sum(wl * dv, axis=0), np.sum(wl * dvh, axis=0)
    a_mean, a_sq, dsum = 0.5 * (vw + vhw), 0.5 * (vw ** 2 + vhw ** 2), vw * dvw + vhw * dvhw
    rest = (0.5 * wlv + 0.5 * wlvh - wlv0) / W - kappa1 * theta + (kappa1 - kappa2 * theta) * a_mean + kappa2 * a_sq
    drest = (0.5 * dwlv + 0.5 * dwlvh) / W + (kappa1 - kappa2 * theta) * 0.5 * (dvw + dvhw) + kappa2 * dsum
    dterm1 = ((dvhw - dvw) / W + rest + h * drest) / volvol
    term2 = 0.5 * h * (vw ** 2 + vhw ** 2)
    dterm2 = a_sq + h * dsum
    dls = dls - 0.5 * dterm2 + rho * dterm1 + np.sqrt(1.0 - rho * rho) * z1 * dterm2 / (2.0 * np.sqrt(term2))
    return ls_h[0], vol_h, y_h[0], dls, dvh, dy + dterm2, reset


def rough_theta_path(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, S, h, Z0, Z1):
    """one maturity from t = 0 on S steps of h: (log_spot, vol (n, P), qv, dls, dqv, reset) with the d/d h tangents"""
    weights, nodes = np.asarray(weights, dtype=float), np.asarray(nodes, dtype=float)
    n, P = nodes.size, Z0.shape[1]
    volvol = np.sqrt(beta ** 2 + orthog_vol ** 2)
    rho = beta / volvol
    v0 = sigma0 / np.sum(weights)
    v, dv = np.full((n, P), v0), np.zeros((n, P))
    ls, y, dls, dy = np.zeros(P), np.zeros(P), np.zeros(P), np.zeros(P)
    reset = np.zeros(P, dtype=bool)
    for s in range(S):
        ls, v, y, dls, dv, dy, r = rough_theta_step(nodes, weights, v0, theta, kappa1, kappa2, rho, volvol, h, ls, v, y, dls, dv, dy, Z0[s], Z1[s])
        reset |= r
    return ls, v, y, dls, dy, reset


def rough_chain_theta_fixed(ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0, Z1, sigma0, theta, kappa1, kappa2, beta, orthog_vol,
                            weights, nodes, nsteps, hs, variable_type=LOG_RETURN):
    """(theta, theta_se, states) per maturity of the rough chain, states = rough_theta_path's tuple; maturity m uses the first nsteps[m] rows"""
    out = ([], [], [])
    for m, ttm in enumerate(ttms):
        S = int(nsteps[m])
        st = rough_theta_path(nodes, weights, sigma0, theta, kappa1, kappa2, beta, orthog_vol, S, hs[m], Z0[:S], Z1[:S])
        th, se = mc_payoff_theta(st[0], st[2], st[3], st[4], S, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
        for acc, r in zip(out, (th, se, st)):
            acc.append(r)
    return out
