"""Numpy forward-over-forward restatement of the second-order Fourier chain sensitivities (DESIGN.md §4.4).  TEST INFRASTRUCTURE ONLY.

Written from the maths, next to ``oracle.mgf_greeks``:

* ``Hyper``: complex hyper-dual numbers (value, d/dp, d/dq, d2/dp dq) over numpy arrays;
* ``logsv_chain_hessian``: every parameter pair of LOGSV_NAMES seeded as a hyper-dual pair and pushed through the model fields, the
  coefficient table (``oracle.mgf_greeks.coef``), Dormand-Prince replayed on the meshes ``oracle.mgf_greeks.logsv_chain_greeks`` recorded,
  and lm = sum_k A_k (sigma0 - theta)^k -- the exact second derivative of the scheme on that mesh (the chain function takes the sigma0
  rows, which need no ODE work, in closed form from the recorded A and dA);
* ``heston_chain_hessian``: the Heston closed form of ``oracle.mgf_greeks.heston_chain_greeks`` in hyper-dual numbers;
* ``replay_tangent``: first-order tangents (``oracle.mgf_greeks.LogsvTangentRhs``) stepped on a recorded mesh, which the tests difference;
* ``vanilla_slice_hessian``: the Fourier sums S_p, S_xp, S_pq and the vanna / Hessian assembly.
"""
from __future__ import annotations

import numpy as np

from oracle import mgf
from oracle import mgf_greeks as G


def pairs(n):
    """the upper triangle p <= q, row-major: the row order of the hessian outputs"""
    return [(p, q) for p in range(n) for q in range(p, n)]


class Hyper:
    """complex hyper-dual number (v, d1, d2, d12) over numpy arrays"""
    __array_ufunc__ = None

    def __init__(self, v, d1=0.0, d2=0.0, d12=0.0):
        c = lambda x: np.asarray(x, dtype=np.complex128)
        self.v, self.d1, self.d2, self.d12 = c(v), c(d1), c(d2), c(d12)

    @staticmethod
    def lift(x):
        return x if isinstance(x, Hyper) else Hyper(x)

    def parts(self):
        return self.v, self.d1, self.d2, self.d12

    def __getitem__(self, idx):
        return Hyper(*(np.broadcast_to(x, self.v.shape)[idx] for x in self.parts()))

    def __add__(self, o):
        o = Hyper.lift(o)
        return Hyper(self.v + o.v, self.d1 + o.d1, self.d2 + o.d2, self.d12 + o.d12)

    __radd__ = __add__

    def __neg__(self):
        return Hyper(-self.v, -self.d1, -self.d2, -self.d12)

    def __sub__(self, o):
        return self + (-Hyper.lift(o))

    def __rsub__(self, o):
        return Hyper.lift(o) - self

    def __mul__(self, o):
        o = Hyper.lift(o)
        return Hyper(self.v * o.v, self.d1 * o.v + self.v * o.d1, self.d2 * o.v + self.v * o.d2,
                     self.d12 * o.v + self.d1 * o.d2 + self.d2 * o.d1 + self.v * o.d12)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Hyper.lift(o)
        q = self.v / o.v
        q1, q2 = (self.d1 - q * o.d1) / o.v, (self.d2 - q * o.d2) / o.v
        return Hyper(q, q1, q2, (self.d12 - q1 * o.d2 - q2 * o.d1 - q * o.d12) / o.v)

    def __rtruediv__(self, o):
        return Hyper.lift(o) / self

    def sqrt(self):
        s = np.sqrt(self.v)
        s1, s2 = self.d1 / (2.0 * s), self.d2 / (2.0 * s)
        return Hyper(s, s1, s2, (self.d12 - 2.0 * s1 * s2) / (2.0 * s))

    def exp(self):
        e = np.exp(self.v)
        return Hyper(e, e * self.d1, e * self.d2, e * (self.d12 + self.d1 * self.d2))

    def log(self):
        l1, l2 = self.d1 / self.v, self.d2 / self.v
        return Hyper(np.log(self.v), l1, l2, (self.d12 - l1 * self.d2) / self.v)


def seeded(values, p, q):
    """the parameters as hyper-dual numbers with d1 along parameter p and d2 along parameter q"""
    return [Hyper(x, 1.0 if k == p else 0.0, 1.0 if k == q else 0.0) for k, x in enumerate(values)]


# --------------------------------------------------------------------------------------------
# LogSV
# --------------------------------------------------------------------------------------------
def _logsv_rhs(A, f, c, n):
    """the right-hand side f(A) = A^T M A + L A + H row by row (the sparse list of oracle.mgf_greeks._rows with q = A_i A_j, u = A);
    A: list of n columns, f: model fields, c: coefficient table -- any arithmetic type"""
    qv, qv2, v2 = f["qv"], f["qv2"], f["v2"]
    a1, a2 = A[1], A[2]
    out = [0.5 * qv2 * a1 * a1 + c["l01"] * a1 + qv2 * a2 + c["h0"]]
    if n == 5:
        a3, a4 = A[3], A[4]
        out.append(qv * a1 * a1 + 2.0 * qv2 * a1 * a2 + c["l11"] * a1 + c["l12"] * a2 + 3.0 * qv2 * a3 + c["h1"])
        out.append(0.5 * v2 * a1 * a1 + 2.0 * qv2 * a2 * a2 + 4.0 * qv * a1 * a2 + 3.0 * qv2 * a1 * a3 + c["l21"] * a1 + c["l22"] * a2
                   + c["l23"] * a3 + 6.0 * qv2 * a4 + c["h2"])
        out.append(4.0 * qv * a2 * a2 + 2.0 * v2 * a1 * a2 + 6.0 * qv * a1 * a3 + 4.0 * qv2 * a1 * a4 + 6.0 * qv2 * a2 * a3
                   + c["l32"] * a2 + c["l33"] * a3 + c["l34"] * a4)
        out.append(2.0 * v2 * a2 * a2 + 4.5 * qv2 * a3 * a3 + 3.0 * v2 * a1 * a3 + 8.0 * qv * a1 * a4 + 12.0 * qv * a2 * a3
                   + 8.0 * qv2 * a2 * a4 + c["l43"] * a3 + c["l44"] * a4)
    else:
        out.append(qv * a1 * a1 + 2.0 * qv2 * a1 * a2 + c["l11"] * a1 + c["l12"] * a2 + c["h1"])
        out.append(0.5 * v2 * a1 * a1 + 2.0 * qv2 * a2 * a2 + 4.0 * qv * a1 * a2 + c["l21"] * a1 + c["l22"] * a2 + c["h2"])
    return out


def _take(x, idx):
    if isinstance(x, Hyper):
        return x[idx] if x.v.ndim else x
    return x[idx] if np.ndim(x) else x


def _replay_columns(rhs, A, mesh):
    """Dormand-Prince on a recorded mesh (oracle.mgf_greeks.replay) with the state as a list of columns of any arithmetic type"""
    A = list(A)
    n = len(A)
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya = [_take(a, ja) for a in A]
        K = [rhs(ya, ja)]
        for s in range(1, 6):
            K.append(rhs([ya[k] + sum(K[j][k] * mgf._A[s][j] for j in range(s)) * h for k in range(n)], ja))
        yn = [ya[k] + h * sum(K[j][k] * mgf._B[j] for j in range(6)) for k in range(n)]
        for k in range(n):
            A[k] = _scatter(A[k], ja, yn[k])
    return A


def _scatter(a, ja, val):
    if isinstance(val, Hyper):
        a = Hyper.lift(a)
        parts = []
        for x, y in zip(a.parts(), val.parts()):
            x = np.array(np.broadcast_to(x, val.v.shape[:0] + a.v.shape), dtype=np.complex128)
            x[ja] = y
            parts.append(x)
        return Hyper(*parts)
    a = np.array(a, dtype=np.complex128)
    a[ja] = val
    return a


def logsv_d2_log_mgf(params6, ttms, meshes, phi, is_spot_measure=True, order=2, etas=None, p=0, q=0):
    """d2 lm / d p d q [M, P] (and the hyper-dual a of the last maturity) on recorded meshes; p, q index LOGSV_NAMES"""
    n, P = mgf.expansion_n(order), phi.shape[0]
    etas = np.ones(len(ttms)) if etas is None else etas
    par = seeded(params6, p, q)
    psi = np.zeros_like(phi)
    A = [Hyper(np.zeros(P)) for _ in range(n)]
    y = par[0] - par[1]
    ys = [Hyper(1.0)]
    for _ in range(1, n):
        ys.append(ys[-1] * y)
    out = np.empty((len(ttms), P), dtype=np.complex128)
    for m in range(len(ttms)):
        f = G.logsv_fields(par, etas[m], is_spot_measure)
        c = G.coef(f, phi, psi, is_spot_measure)
        rhs = lambda Y, idx, f=f, c=c: _logsv_rhs(Y, f, {k: _take(v, idx) for k, v in c.items()}, n)
        A = _replay_columns(rhs, A, meshes[m])
        lm = sum((A[k] * ys[k] for k in range(n)), Hyper(np.zeros(P)))
        out[m] = lm.d12
    return out, A


def replay_tangent(rhs, trhs, y0, dy0, mesh):
    """oracle.mgf_greeks.replay plus first-order tangents dy [D, P, n] stepped with trhs[d] on the same recorded mesh"""
    y, dy = y0.astype(np.complex128).copy(), np.array(dy0, dtype=np.complex128).copy()
    n, D = y.shape[1], len(trhs)
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya, dya = y[ja], dy[:, ja]
        K = np.zeros((7, ja.shape[0], n), dtype=np.complex128)
        dK = np.zeros((7, D, ja.shape[0], n), dtype=np.complex128)
        K[0] = rhs(ya, ja)
        dK[0] = [trhs[d](ya, dya[d], ja) for d in range(D)]
        for s in range(1, 6):
            Ys = ya + G._stage_sum(K, mgf._A[s], s) * h[:, None]
            K[s] = rhs(Ys, ja)
            for d in range(D):
                dK[s, d] = trhs[d](Ys, dya[d] + G._stage_sum(dK[:, d], mgf._A[s], s) * h[:, None], ja)
        y[ja] = ya + h[:, None] * sum(K[j] * mgf._B[j] for j in range(6))
        dy[:, ja] = np.array([dya[d] + h[:, None] * sum(dK[j, d] * mgf._B[j] for j in range(6)) for d in range(D)])
    return y, dy


def logsv_tangents_on_meshes(params6, ttms, meshes, phi, is_spot_measure=True, order=2, etas=None):
    """first-order tangents of the five ODE directions on recorded meshes: (a [M, P, n], da [M, 5, P, n], dlog_mgf [6, M, P])"""
    n, P = mgf.expansion_n(order), phi.shape[0]
    etas = np.ones(len(ttms)) if etas is None else etas
    psi = np.zeros_like(phi)
    a, da = np.zeros((P, n), dtype=np.complex128), np.zeros((5, P, n), dtype=np.complex128)
    yv = params6[0] - params6[1]
    ys = np.array([1.0, yv, yv * yv, yv ** 3, yv ** 4])[:n] + 0j
    dys = np.array([0.0, 1.0, 2.0 * yv, 3.0 * yv * yv, 4.0 * yv ** 3])[:n] + 0j
    As, dAs, dlm = [], [], np.empty((6, len(ttms), P), dtype=np.complex128)
    for m in range(len(ttms)):
        rhs = mgf.LogsvRhs(*params6[1:], phi, psi, is_spot_measure, order, etas[m])
        f = G.logsv_fields(params6, etas[m], is_spot_measure)
        trhs = [G.LogsvTangentRhs(f, d, phi, psi, is_spot_measure, order) for d in G.logsv_dfields(params6, etas[m], is_spot_measure)]
        a, da = replay_tangent(rhs, trhs, a, da, meshes[m])
        As.append(a.copy())
        dAs.append(da.copy())
        dlm[0, m] = a @ dys
        for d in range(5):
            dlm[1 + d, m] = da[d] @ ys - (a @ dys if d == 0 else 0.0)
    return np.array(As), np.array(dAs), dlm


# --------------------------------------------------------------------------------------------
# Fourier sums
# --------------------------------------------------------------------------------------------
def vanilla_slice_hessian(log_mgf, dlog_mgf, d2log_mgf, phi, forward, strikes, types, discfactor=1.0, is_spot_measure=True):
    """(vanna [NP, J], hessian [NP (NP + 1) / 2, J]) from lm [P], dlm [NP, P], d2lm [NH, P] (pairs() order)"""
    p = np.imag(phi)
    w = (mgf.legacy_simpson_weights(phi) / np.pi) / (p * p + 0.25)
    NP = dlog_mgf.shape[0]
    pr = pairs(NP)
    vanna, hess = np.zeros((NP, len(strikes))), np.zeros((len(pr), len(strikes)))
    F, df = forward, discfactor
    for j, k in enumerate(strikes):
        x = np.log(F / k)
        e = np.exp(-x * phi + log_mgf)
        keep = ~np.isnan(np.real((w + 0j) * e))
        S = lambda z: np.sum((w * np.real(z))[keep])
        Sp = np.array([S(e * d) for d in dlog_mgf])
        Sxp = np.array([S(-phi * e * d) for d in dlog_mgf])
        Spq = np.array([S(e * (d2log_mgf[r] + dlog_mgf[a] * dlog_mgf[b])) for r, (a, b) in enumerate(pr)])
        if is_spot_measure:
            vanna[:, j], hess[:, j] = -df * k * Sxp / F, -df * k * Spq
        else:
            vanna[:, j], hess[:, j] = -df * (Sp + Sxp), -F * df * Spq
    return vanna, hess


# --------------------------------------------------------------------------------------------
# chains
# --------------------------------------------------------------------------------------------
def logsv_chain_hessian(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, order=2, etas=None,
                        vol_scaler=None):
    """per maturity (first-order rows [9, J] of oracle.mgf_greeks.logsv_chain_greeks, vanna [6, J], hessian [21, J]), and the grids of
    logsv_chain_greeks plus d2log_mgf [21, M, P]"""
    if vol_scaler is None:
        vol_scaler = mgf.logsv_vol_scaler(params6[0], ttms)
    out1, grids = G.logsv_chain_greeks(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure, order, etas,
                                       vol_scaler)
    phi = mgf.phi_grid(vol_scaler, is_spot_measure)
    pr = pairs(6)
    d2lm = np.empty((len(pr), len(ttms), phi.shape[0]), dtype=np.complex128)
    # sigma0 enters only through y = sigma0 - theta: its rows are closed forms in the recorded A and dA (y_sigma0 = 1, y_theta = -1),
    # d2lm / dsigma0 dq = sum_k dA_q,k k y^(k-1) + A_k k (k-1) y^(k-2) y_q
    n, yv = mgf.expansion_n(order), params6[0] - params6[1]
    d1 = np.array([k * yv ** (k - 1) if k else 0.0 for k in range(n)]) + 0j
    d2 = np.array([k * (k - 1) * yv ** (k - 2) if k > 1 else 0.0 for k in range(n)]) + 0j
    for r, (p, q) in enumerate(pr):
        if p == 0:
            for m in range(len(ttms)):
                y_q = -1.0 if q == 1 else 0.0
                d2lm[r, m] = grids["a"][m] @ d2 if q == 0 else grids["da"][m][q - 1] @ d1 + y_q * (grids["a"][m] @ d2)
        else:
            d2lm[r] = logsv_d2_log_mgf(params6, ttms, grids["meshes"], phi, is_spot_measure, order, etas, p, q)[0]
    grids["d2log_mgf"] = d2lm
    out = []
    for m in range(len(ttms)):
        v, h = vanilla_slice_hessian(grids["log_mgf"][m], grids["dlog_mgf"][:, m], d2lm[:, m], phi, forwards[m], strikes_ttms[m],
                                     types_ttms[m], discfactors[m], is_spot_measure)
        out.append((out1[m], v, h))
    return out, grids


def heston_d2_log_mgf(params5, ttms, phi, p, q):
    """d2 lm / d p d q [M, P] of the Heston closed form (oracle.mgf_greeks.heston_chain_greeks) in hyper-dual numbers"""
    v0, theta, kappa, rho, volvol = seeded(params5, p, q)
    vv2 = volvol * volvol
    b1 = kappa + rho * volvol * phi
    b0 = 0.5 * phi * (phi + 1.0)
    zeta = (b1 * b1 - 2.0 * b0 * vv2).sqrt()
    psi_p, psi_m = -b1 + zeta, b1 + zeta
    a, b = Hyper(np.zeros(phi.shape[0])), Hyper(np.zeros(phi.shape[0]))
    out, t0 = np.empty((len(ttms), phi.shape[0]), dtype=np.complex128), 0.0
    for m, ttm in enumerate(ttms):
        dtau = ttm - t0
        ez = (-zeta * dtau).exp()
        c_p, c_m = (psi_p + vv2 * b) / (2.0 * zeta), (psi_m - vv2 * b) / (2.0 * zeta)
        b = -(-psi_m * c_p * ez + psi_p * c_m) / (vv2 * (c_p * ez + c_m))
        a = -(theta * kappa / vv2) * (psi_p * dtau + 2.0 * (c_p * ez + c_m).log()) + a
        out[m] = (a + b * v0).d12
        t0 = ttm
    return out


def heston_chain_hessian(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None):
    """per maturity (first-order rows [8, J], vanna [5, J], hessian [15, J]), dlog_mgf [5, M, P], d2log_mgf [15, M, P]"""
    if vol_scaler is None:
        vol_scaler = mgf.heston_vol_scaler(params5[0], ttms)
    out1, dlm = G.heston_chain_greeks(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler)
    phi = mgf.phi_grid(vol_scaler, True)
    pr = pairs(5)
    d2lm = np.array([heston_d2_log_mgf(params5, ttms, phi, p, q) for p, q in pr])
    grids = mgf.heston_chain_prices(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=vol_scaler, return_grids=True)[1]
    out = []
    for m in range(len(ttms)):
        v, h = vanilla_slice_hessian(grids[m][0], dlm[:, m], d2lm[:, m], phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], True)
        out.append((out1[m], v, h))
    return out, dlm, d2lm
