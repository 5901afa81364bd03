"""oracle.mgf_greeks -- numpy forward-mode restatement of the Fourier chain sensitivities (DESIGN.md §4.2).  TEST INFRASTRUCTURE ONLY.

Written from the maths, next to ``oracle.mgf``:

* ``logsv_dfields``: d(model field)/d(parameter) -- the table the library builds on the host;
* ``dense_mlh``: dense M / L / H from the model fields and the coefficient table, so that the derivative table can be checked against
  central differences of ``oracle.mgf.logsv_mlh``;
* ``rk45_grid_tangent``: the control law of ``oracle.mgf.rk45_grid`` with forward-mode tangents stepped on the primal's attempts (the
  error norm sees the primal only), returning the accepted mesh; ``replay`` steps Dormand-Prince on a recorded mesh;
* ``logsv_chain_greeks`` / ``heston_chain_greeks``: prices, delta, gamma and d price / d parameter of a chain;
* ``vanilla_slice_greeks``: the Fourier sums S, S_x, S_xx, S_p and their assembly.
"""
from __future__ import annotations

import numpy as np

from . import mgf

LOGSV_NAMES = ("sigma0", "theta", "kappa1", "kappa2", "beta", "volvol")
HESTON_NAMES = ("v0", "theta", "kappa", "rho", "volvol")
FIELDS = ("theta", "th2", "v2", "qv", "qv2", "lam", "k2p", "kp", "beta_eta")


# --------------------------------------------------------------------------------------------
# model fields, their parameter derivatives, coefficient tables
# --------------------------------------------------------------------------------------------
def logsv_fields(params6, eta=1.0, is_spot_measure=True):
    """the phi-independent reals of affine_expansion.py:121-135 (LogsvModel of the CUDA library)"""
    _, theta, kappa1, kappa2, beta, volvol = params6
    v2 = beta * beta + volvol * volvol
    f = dict(theta=theta, th2=theta * theta, v2=v2, qv=theta * v2, qv2=theta * theta * v2, beta_eta=beta * eta, eta2=eta * eta)
    if is_spot_measure:
        f.update(lam=0.0, k2p=kappa2, kp=kappa1 + kappa2 * theta)
    else:
        f.update(lam=beta * theta * theta * eta, k2p=kappa2 - beta * eta, kp=kappa1 + kappa2 * theta - 2 * beta * theta * eta)
    return f


def logsv_dfields(params6, eta=1.0, is_spot_measure=True):
    """d(field)/d(theta, kappa1, kappa2, beta, volvol): list of 5 dicts (kappa2 held fixed when kappa1 or theta moves; eta2 constant)"""
    _, theta, kappa1, kappa2, beta, volvol = params6
    v2, th2, spot = beta * beta + volvol * volvol, theta * theta, is_spot_measure
    z = dict.fromkeys(FIELDS, 0.0)
    d_theta = dict(z, theta=1.0, th2=2 * theta, qv=v2, qv2=2 * theta * v2, lam=0.0 if spot else 2 * beta * theta * eta,
                   kp=kappa2 if spot else kappa2 - 2 * beta * eta)
    d_kappa1 = dict(z, kp=1.0)
    d_kappa2 = dict(z, k2p=1.0, kp=theta)
    d_beta = dict(z, v2=2 * beta, qv=2 * beta * theta, qv2=2 * beta * th2, lam=0.0 if spot else th2 * eta, k2p=0.0 if spot else -eta,
                  kp=0.0 if spot else -2 * theta * eta, beta_eta=eta)
    d_volvol = dict(z, v2=2 * volvol, qv=2 * volvol * theta, qv2=2 * volvol * th2)
    return [d_theta, d_kappa1, d_kappa2, d_beta, d_volvol]


def _h_factor(phi, psi, spot):
    return phi * (phi + 1.0) - 2.0 * psi if spot else phi * (phi - 1.0) - 2.0 * psi


def coef(f, phi, psi, spot):
    """the 14 phi-dependent entries of L and H (affine_expansion.py:166-183) from the model fields"""
    b = f["beta_eta"] * phi
    th2, th = f["th2"], f["theta"]
    r = _h_factor(phi, psi, spot)
    return dict(l01=f["lam"] - th2 * b, l11=-f["kp"] - 2.0 * th * b, l12=2.0 * (f["lam"] + f["qv"] - th2 * b), l21=-f["k2p"] - b,
                l22=f["v2"] - 2.0 * f["kp"] - 4.0 * th * b, l23=3.0 * (2.0 * f["qv"] - th2 * b), l32=-2.0 * (f["k2p"] + b),
                l33=3.0 * (f["v2"] - f["kp"] - 2.0 * th * b), l34=4.0 * (3.0 * f["qv"] - th2 * b), l43=-3.0 * (f["k2p"] + b),
                l44=2.0 * (f["v2"] - 2.0 * f["kp"] - 4.0 * th * b),
                h0=0.5 * th2 * f["eta2"] * r, h1=th * f["eta2"] * r, h2=0.5 * f["eta2"] * r)


def dcoef(f, df, phi, psi, spot):
    """coef() differentiated in one direction (product rule on th2 b, theta b, th2 eta2, theta eta2)"""
    b, db = f["beta_eta"] * phi, df["beta_eta"] * phi
    dtb = df["th2"] * b + f["th2"] * db
    d1b = df["theta"] * b + f["theta"] * db
    r = _h_factor(phi, psi, spot)
    zero = 0.0 * phi
    return dict(l01=df["lam"] - dtb, l11=-df["kp"] - 2.0 * d1b, l12=2.0 * (df["lam"] + df["qv"] - dtb), l21=-df["k2p"] - db,
                l22=df["v2"] - 2.0 * df["kp"] - 4.0 * d1b, l23=3.0 * (2.0 * df["qv"] - dtb), l32=-2.0 * (df["k2p"] + db),
                l33=3.0 * (df["v2"] - df["kp"] - 2.0 * d1b), l34=4.0 * (3.0 * df["qv"] - dtb), l43=-3.0 * (df["k2p"] + db),
                l44=2.0 * (df["v2"] - 2.0 * df["kp"] - 4.0 * d1b),
                h0=0.5 * df["th2"] * f["eta2"] * r, h1=df["theta"] * f["eta2"] * r, h2=zero)


def dense_mlh(v2, qv, qv2, c, n):
    """dense M [n,n,n], L [P,n,n], H [P,n] of one grid vector from (v2, qv, qv2) and a coefficient table -- the layout of logsv_mlh,
    linear in its inputs, so it assembles the derivatives from (dv2, dqv, dqv2, dcoef) as well"""
    P = np.atleast_1d(c["l01"]).shape[0]
    M = np.zeros((n, n, n), dtype=np.complex128)
    diag = [(0, 1, 0.5 * qv2), (1, 1, qv), (2, 1, 0.5 * v2), (2, 2, 2.0 * qv2)]
    sym = [(1, 1, 2, qv2), (2, 1, 2, 2.0 * qv)]
    if n == 5:
        diag += [(3, 2, 4.0 * qv), (4, 2, 2.0 * v2), (4, 3, 4.5 * qv2)]
        sym += [(2, 1, 3, 1.5 * qv2), (3, 1, 2, v2), (3, 1, 3, 3.0 * qv), (3, 1, 4, 2.0 * qv2), (3, 2, 3, 3.0 * qv2),
                (4, 1, 3, 1.5 * v2), (4, 1, 4, 4.0 * qv), (4, 2, 3, 6.0 * qv), (4, 2, 4, 4.0 * qv2)]
    for k, i, val in diag:
        M[k, i, i] = val
    for k, i, j, val in sym:
        M[k, i, j] = M[k, j, i] = val
    g = lambda key: np.broadcast_to(c[key], (P,))
    L = np.zeros((P, n, n), dtype=np.complex128)
    L[:, 0, 1], L[:, 0, 2] = g("l01"), qv2
    L[:, 1, 1], L[:, 1, 2] = g("l11"), g("l12")
    L[:, 2, 1], L[:, 2, 2] = g("l21"), g("l22")
    if n == 5:
        L[:, 1, 3] = 3.0 * qv2
        L[:, 2, 3], L[:, 2, 4] = g("l23"), 6.0 * qv2
        L[:, 3, 2], L[:, 3, 3], L[:, 3, 4] = g("l32"), g("l33"), g("l34")
        L[:, 4, 3], L[:, 4, 4] = g("l43"), g("l44")
    H = np.zeros((P, n), dtype=np.complex128)
    H[:, 0], H[:, 1], H[:, 2] = g("h0"), g("h1"), g("h2")
    return M, L, H


# --------------------------------------------------------------------------------------------
# right-hand side and its tangent (the rows of oracle.mgf.LogsvRhs with products q and linear inputs u)
# --------------------------------------------------------------------------------------------
def _rows(q, u, v2, qv, qv2, c, with_h, n, idx):
    g = lambda key: c[key][idx] if isinstance(c[key], np.ndarray) else c[key]
    h = (lambda key: g(key)) if with_h else (lambda key: 0.0)
    out = np.empty_like(u)
    out[:, 0] = 0.5 * qv2 * q["11"] + g("l01") * u[:, 1] + qv2 * u[:, 2] + h("h0")
    if n == 5:
        out[:, 1] = qv * q["11"] + 2.0 * qv2 * q["12"] + g("l11") * u[:, 1] + g("l12") * u[:, 2] + 3.0 * qv2 * u[:, 3] + h("h1")
        out[:, 2] = (0.5 * v2 * q["11"] + 2.0 * qv2 * q["22"] + 4.0 * qv * q["12"] + 3.0 * qv2 * q["13"] + g("l21") * u[:, 1]
                     + g("l22") * u[:, 2] + g("l23") * u[:, 3] + 6.0 * qv2 * u[:, 4] + h("h2"))
        out[:, 3] = (4.0 * qv * q["22"] + 2.0 * v2 * q["12"] + 6.0 * qv * q["13"] + 4.0 * qv2 * q["14"] + 6.0 * qv2 * q["23"]
                     + g("l32") * u[:, 2] + g("l33") * u[:, 3] + g("l34") * u[:, 4])
        out[:, 4] = (2.0 * v2 * q["22"] + 4.5 * qv2 * q["33"] + 3.0 * v2 * q["13"] + 8.0 * qv * q["14"] + 12.0 * qv * q["23"]
                     + 8.0 * qv2 * q["24"] + g("l43") * u[:, 3] + g("l44") * u[:, 4])
    else:
        out[:, 1] = qv * q["11"] + 2.0 * qv2 * q["12"] + g("l11") * u[:, 1] + g("l12") * u[:, 2] + h("h1")
        out[:, 2] = 0.5 * v2 * q["11"] + 2.0 * qv2 * q["22"] + 4.0 * qv * q["12"] + g("l21") * u[:, 1] + g("l22") * u[:, 2] + h("h2")
    return out


_PAIRS = ("11", "12", "22", "13", "14", "23", "24", "33")


class LogsvTangentRhs:
    """d f(A) = J(A) dA + d_p f(A) for one parameter direction: J(A) dA = rows(A_i dA_j + dA_i A_j, dA; fields, coef, no H),
    d_p f(A) = rows(A_i A_j, A; d fields, d coef, with d H)"""

    def __init__(self, f, df, phi, psi, is_spot_measure, order):
        self.n = mgf.expansion_n(order)
        self.f, self.df = f, df
        self.c = coef(f, phi, psi, is_spot_measure)
        self.dc = dcoef(f, df, phi, psi, is_spot_measure)

    def __call__(self, A, dA, idx=slice(None)):
        q = {p: A[:, int(p[0])] * A[:, int(p[1])] for p in _PAIRS if max(int(p[0]), int(p[1])) < self.n}
        dq = {p: A[:, int(p[0])] * dA[:, int(p[1])] + dA[:, int(p[0])] * A[:, int(p[1])] for p in q}
        f, df = self.f, self.df
        return (_rows(dq, dA, f["v2"], f["qv"], f["qv2"], self.c, False, self.n, idx)
                + _rows(q, A, df["v2"], df["qv"], df["qv2"], self.dc, True, self.n, idx))


# --------------------------------------------------------------------------------------------
# RK45 with tangents on the primal's attempts, and the replay of a recorded mesh
# --------------------------------------------------------------------------------------------
def _stage_sum(K, coefs, s):
    return sum(K[j] * coefs[j] for j in range(s))


def rk45_grid_tangent(rhs, trhs, y0, dy0, t_bound):
    """oracle.mgf.rk45_grid (same control law, same arithmetic for y) plus D tangents dy [D, P, n]: each stage dY_s = dy + h sum_j a_sj dK_j,
    dK_s = trhs[d](Y_s, dY_s), committed with the primal's acceptance.  Returns (y, dy, nfev [P], mesh: list of (point indices, h))."""
    P, n = y0.shape
    D = len(trhs)
    y = y0.astype(np.complex128).copy()
    dy = np.array(dy0, dtype=np.complex128).copy()
    t = np.zeros(P)
    f = rhs(y)
    scale = mgf.ATOL + np.abs(y) * mgf.RTOL
    d0, d1 = mgf._rms(y / scale), mgf._rms(f / scale)
    with np.errstate(divide="ignore", invalid="ignore"):
        h0 = np.where((d0 < 1e-5) | (d1 < 1e-5), 1e-6, 0.01 * d0 / d1)
    h0 = np.minimum(h0, t_bound)
    f1 = rhs(y + h0[:, None] * f)
    d2 = mgf._rms((f1 - f) / scale) / h0
    with np.errstate(divide="ignore"):
        h1 = np.where((d1 <= 1e-15) & (d2 <= 1e-15), np.maximum(1e-6, h0 * 1e-3), (0.01 / np.maximum(d1, d2)) ** (1 / 5))
    h_abs = np.minimum(np.minimum(100 * h0, h1), t_bound)
    nfev = np.full(P, 2)
    df0 = np.array([trhs[d](y, dy[d]) for d in range(D)])
    active = t < t_bound
    rejected = np.zeros(P, dtype=bool)
    new_step = np.ones(P, dtype=bool)
    mesh = []
    while np.any(active):
        ia = np.nonzero(active)[0]
        ta, ya = t[ia], y[ia]
        min_step = 10 * np.abs(np.nextafter(ta, np.inf) - ta)
        ha = h_abs[ia]
        ha = np.where(new_step[ia] & (ha < min_step), min_step, ha)
        t_new = ta + ha
        t_new = np.where((t_new - t_bound) > 0, t_bound, t_new)
        h = t_new - ta
        ha = np.abs(h)
        K = np.zeros((7, ia.shape[0], n), dtype=np.complex128)
        dK = np.zeros((7, D, ia.shape[0], n), dtype=np.complex128)
        K[0], dK[0] = f[ia], df0[:, ia]
        for s in range(1, 6):
            Ys = ya + _stage_sum(K, mgf._A[s], s) * h[:, None]
            K[s] = rhs(Ys, ia)
            for d in range(D):
                dK[s, d] = trhs[d](Ys, dy[d, ia] + _stage_sum(dK[:, d], mgf._A[s], s) * h[:, None], ia)
        y_new = ya + h[:, None] * sum(K[j] * mgf._B[j] for j in range(6))
        dy_new = np.array([dy[d, ia] + h[:, None] * sum(dK[j, d] * mgf._B[j] for j in range(6)) for d in range(D)])
        f_new = rhs(y_new, ia)
        K[6] = f_new
        df_new = np.array([trhs[d](y_new, dy_new[d], ia) for d in range(D)])
        nfev[ia] += 6
        scale = mgf.ATOL + np.maximum(np.abs(ya), np.abs(y_new)) * mgf.RTOL
        err = mgf._rms(sum(K[j] * mgf._E[j] for j in range(7)) * h[:, None] / scale)
        acc = err < 1
        with np.errstate(divide="ignore"):
            fac_acc = np.where(err == 0, mgf.MAX_FACTOR, np.minimum(mgf.MAX_FACTOR, mgf.SAFETY * err ** -0.2))
            fac_acc = np.where(rejected[ia], np.minimum(1.0, fac_acc), fac_acc)
            fac_rej = np.maximum(mgf.MIN_FACTOR, mgf.SAFETY * err ** -0.2)
        h_abs[ia] = ha * np.where(acc, fac_acc, fac_rej)
        ja = ia[acc]
        mesh.append((ja, h[acc]))
        t[ja], y[ja], f[ja] = t_new[acc], y_new[acc], f_new[acc]
        dy[:, ja], df0[:, ja] = dy_new[:, acc], df_new[:, acc]
        rejected[ja], new_step[ja] = False, True
        jr = ia[~acc]
        rejected[jr], new_step[jr] = True, False
        active = t < t_bound
    return y, dy, nfev, mesh


def replay(rhs, y0, mesh):
    """Dormand-Prince on a recorded mesh (no step-size control): with the parameters the mesh was recorded at, the result is
    oracle.mgf.rk45_grid's bit for bit; with perturbed parameters it is the scheme whose derivative rk45_grid_tangent steps"""
    y = y0.astype(np.complex128).copy()
    n = y.shape[1]
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya = y[ja]
        K = np.zeros((7, ja.shape[0], n), dtype=np.complex128)
        K[0] = rhs(ya, ja)
        for s in range(1, 6):
            K[s] = rhs(ya + _stage_sum(K, mgf._A[s], s) * h[:, None], ja)
        y[ja] = ya + h[:, None] * sum(K[j] * mgf._B[j] for j in range(6))
    return y


# --------------------------------------------------------------------------------------------
# Fourier sums and their derivatives
# --------------------------------------------------------------------------------------------
def vanilla_slice_greeks(log_mgf, dlog_mgf, phi, forward, strikes, types, discfactor=1.0, is_spot_measure=True):
    """|Re phi| = 1/2 branch of oracle.mgf.vanilla_slice_prices: (prices, delta, gamma, dprice [NP, J]) with dlog_mgf [NP, P]"""
    p = np.imag(phi)
    w = (mgf.legacy_simpson_weights(phi) / np.pi) / (p * p + 0.25)
    J = len(strikes)
    out = np.zeros((3 + dlog_mgf.shape[0], J))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        x = np.log(forward / k)
        e = np.exp(-x * phi + log_mgf)
        keep = ~np.isnan(np.real((w + 0j) * e))
        S = np.sum(np.real(w * e)[keep])
        Sx = np.sum((w * np.real(-phi * e))[keep])
        Sxx = np.sum((w * np.real(phi * phi * e))[keep])
        Sp = np.array([np.sum((w * np.real(e * d))[keep]) for d in dlog_mgf])
        ty, F, df = str(ty), forward, discfactor
        call = ty in ("C", "IC")
        if is_spot_measure:
            price = df * (F - k * S) if call else df * (k - k * S)
            delta = df * (1.0 - k * Sx / F) if call else -df * k * Sx / F
            gamma = -df * k * (Sxx - Sx) / (F * F)
            dp = -df * k * Sp
        else:
            price = F * df * (1.0 - S) if call else F * df * (np.exp(-x) - S)
            delta = df * (1.0 - S - Sx) if call else -df * (S + Sx)
            gamma = -df * (Sx + Sxx) / F
            dp = -F * df * Sp
        out[0, j], out[1, j], out[2, j], out[3:, j] = price, delta, gamma, dp
    return out


# --------------------------------------------------------------------------------------------
# chains
# --------------------------------------------------------------------------------------------
def logsv_chain_greeks(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, order=2, etas=None,
                       vol_scaler=None):
    """forward mode through the LogSV chain: per maturity [prices, delta, gamma, d price / d LOGSV_NAMES] ([9, J]), plus the grids
    dict(dlog_mgf [6, M, P], log_mgf [M, P], a [M, P, n], da [5, M, P, n], nfev [P], meshes)"""
    sigma0, theta = params6[0], params6[1]
    if vol_scaler is None:
        vol_scaler = mgf.logsv_vol_scaler(sigma0, ttms)
    phi = mgf.phi_grid(vol_scaler, is_spot_measure)
    psi = np.zeros_like(phi)
    n, P = mgf.expansion_n(order), phi.shape[0]
    etas = np.ones(len(ttms)) if etas is None else etas
    a = np.zeros((P, n), dtype=np.complex128)
    da = np.zeros((5, P, n), dtype=np.complex128)
    yv = sigma0 - theta
    ys = np.array([1.0, yv, yv * yv, yv * yv * yv, (yv * yv) * (yv * yv)])[:n]
    dys = np.array([0.0, 1.0, 2.0 * yv, 3.0 * yv * yv, 4.0 * yv * yv * yv])[:n]
    dy_dp = np.array([-1.0, 0.0, 0.0, 0.0, 0.0])
    out, grids = [], dict(dlog_mgf=[], log_mgf=[], a=[], da=[], meshes=[])
    nfev = np.zeros(P, dtype=int)
    t0 = 0.0
    for m, ttm in enumerate(ttms):
        rhs = mgf.LogsvRhs(*params6[1:], phi, psi, is_spot_measure, order, etas[m])
        f = logsv_fields(params6, etas[m], is_spot_measure)
        trhs = [LogsvTangentRhs(f, dfd, phi, psi, is_spot_measure, order) for dfd in logsv_dfields(params6, etas[m], is_spot_measure)]
        a, da, nf, mesh = rk45_grid_tangent(rhs, trhs, a, da, ttm - t0)
        nfev += nf
        lm = a @ (ys + 0j)
        dlm = np.empty((6, P), dtype=np.complex128)
        dlm[0] = a @ (dys + 0j)
        for d in range(5):
            dlm[1 + d] = da[d] @ (ys + 0j) + a @ (dys * dy_dp[d] + 0j)
        out.append(vanilla_slice_greeks(lm, dlm, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], is_spot_measure))
        for key, val in (("dlog_mgf", dlm), ("log_mgf", lm), ("a", a.copy()), ("da", da.copy()), ("meshes", mesh)):
            grids[key].append(val)
        t0 = ttm
    grids["dlog_mgf"] = np.stack(grids["dlog_mgf"], axis=1)
    grids["nfev"] = nfev
    return out, grids


def logsv_chain_prices_on_meshes(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, meshes, vol_scaler, is_spot_measure=True,
                                 order=2, etas=None):
    """logsv_chain_prices with every maturity's ODE stepped on a recorded mesh (the scheme whose exact derivative the tangents are)"""
    sigma0, theta = params6[0], params6[1]
    phi = mgf.phi_grid(vol_scaler, is_spot_measure)
    psi = np.zeros_like(phi)
    n = mgf.expansion_n(order)
    etas = np.ones(len(ttms)) if etas is None else etas
    a = np.zeros((phi.shape[0], n), dtype=np.complex128)
    yv = sigma0 - theta
    ys = np.array([1.0, yv, yv * yv, yv * yv * yv, (yv * yv) * (yv * yv)])[:n]
    prices, lms = [], []
    for m in range(len(ttms)):
        rhs = mgf.LogsvRhs(*params6[1:], phi, psi, is_spot_measure, order, etas[m])
        a = replay(rhs, a, meshes[m])
        lm = a @ (ys + 0j)
        lms.append(lm)
        prices.append(mgf.vanilla_slice_prices(lm, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], is_spot_measure))
    return prices, np.array(lms)


class _Dual:
    """complex dual number (value, derivative) over numpy arrays"""
    __array_ufunc__ = None          # ndarray (op) _Dual defers to the _Dual's reflected operator

    def __init__(self, v, d=0.0):
        self.v, self.d = np.asarray(v, dtype=np.complex128), np.asarray(d, dtype=np.complex128)

    @staticmethod
    def lift(x):
        return x if isinstance(x, _Dual) else _Dual(x)

    def __add__(self, o):
        o = _Dual.lift(o)
        return _Dual(self.v + o.v, self.d + o.d)

    __radd__ = __add__

    def __sub__(self, o):
        o = _Dual.lift(o)
        return _Dual(self.v - o.v, self.d - o.d)

    def __rsub__(self, o):
        return _Dual.lift(o) - self

    def __neg__(self):
        return _Dual(-self.v, -self.d)

    def __mul__(self, o):
        o = _Dual.lift(o)
        return _Dual(self.v * o.v, self.d * o.v + self.v * o.d)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _Dual.lift(o)
        q = self.v / o.v
        return _Dual(q, (self.d - q * o.d) / o.v)

    def __rtruediv__(self, o):
        return _Dual.lift(o) / self

    def sqrt(self):
        s = np.sqrt(self.v)
        return _Dual(s, self.d / (2.0 * s))

    def exp(self):
        e = np.exp(self.v)
        return _Dual(e, e * self.d)

    def log(self):
        return _Dual(np.log(self.v), self.d / self.v)


def heston_chain_greeks(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None):
    """forward mode through the Heston closed form (oracle.mgf.heston_mgf_grid) with (a, b) and their tangents carried over the
    maturities: per maturity [prices, delta, gamma, d price / d HESTON_NAMES] ([8, J]), and dlog_mgf [5, M, P]"""
    v0 = params5[0]
    if vol_scaler is None:
        vol_scaler = mgf.heston_vol_scaler(v0, ttms)
    phi = mgf.phi_grid(vol_scaler, True)
    M, P = len(ttms), phi.shape[0]
    dlm = np.empty((5, M, P), dtype=np.complex128)
    lms = []
    for d in range(4):
        theta, kappa, rho, volvol = (_Dual(params5[1 + k], 1.0 if k == d else 0.0) for k in range(4))
        vv2 = volvol * volvol
        b1 = kappa + rho * volvol * phi
        b0 = 0.5 * phi * (phi + 1.0)
        zeta = (b1 * b1 - 2.0 * b0 * vv2).sqrt()
        psi_p, psi_m = -b1 + zeta, b1 + zeta
        a, b = _Dual(np.zeros(P)), _Dual(np.zeros(P))
        t0 = 0.0
        for m, ttm in enumerate(ttms):
            dtau = ttm - t0
            ez = (-zeta * dtau).exp()
            c_p, c_m = (psi_p + vv2 * b) / (2.0 * zeta), (psi_m - vv2 * b) / (2.0 * zeta)
            b = -(-psi_m * c_p * ez + psi_p * c_m) / (vv2 * (c_p * ez + c_m))
            a = -(theta * kappa / vv2) * (psi_p * dtau + 2.0 * (c_p * ez + c_m).log()) + a
            dlm[1 + d, m] = a.d + b.d * v0
            if d == 0:
                dlm[0, m] = b.v
                lms.append(a.v + b.v * v0)
            t0 = ttm
    out = [vanilla_slice_greeks(lms[m], dlm[:, m], phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], True) for m in range(M)]
    return out, dlm
