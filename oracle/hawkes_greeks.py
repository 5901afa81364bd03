"""oracle.hawkes_greeks -- numpy forward-mode restatement of the Hawkes Fourier chain sensitivities (DESIGN.md §4.3).  TEST INFRASTRUCTURE
ONLY.

Written from the maths, next to ``oracle.hawkes.HawkesRhs``:

* ``HawkesTangentRhs``: d f(A) = J(A) dA + d_p f(A) of the Riccati system for one parameter direction;
* ``hawkes_chain_greeks``: prices, delta, gamma and d price / d HAWKES_NAMES of a chain, driving ``mgf_greeks.rk45_grid_tangent`` and
  ``mgf_greeks.vanilla_slice_greeks`` over the carried maturities;
* ``hawkes_chain_prices_on_meshes``: the chain prices with every maturity stepped on a recorded mesh (``mgf_greeks.replay``).
"""
from __future__ import annotations

import numpy as np

from . import hawkes, mgf
from . import mgf_greeks as G

# HawkesJDParams fields in dataclass order without mu (never read by the Fourier route) and risk_premia_gamma
HAWKES_NAMES = ("sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p", "lambda_m",
                "theta_m", "kappa_m", "beta1_m", "beta2_m")
ODE_NAMES = tuple(n for n in HAWKES_NAMES if n not in ("lambda_p", "lambda_m"))


def _djump(z, dz, s, m, ds, dm):
    """d E(z) of E(z) = exp(-s z) / (1 + m z) along (dz, ds, dm)"""
    r = 1.0 / (1.0 + m * z)
    e = np.exp(-s * z) * r
    return e * (-(s + m * r) * dz - z * (ds + dm * r))


class HawkesTangentRhs:
    """tangent of oracle.hawkes.HawkesRhs in the direction of one parameter (``name``, one of ODE_NAMES):
    d rhs0 = k_p th_p da_p + k_m th_m da_m + d(k_p th_p) a_p + d(k_m th_m) a_m + 2 sigma dsigma ((phi + 1) phi / 2 - psi)
    d rhs1 = E_p'(z_p) dz_p + d_s E_p ds_p + d_m E_p dm_p - k_p da_p - dk_p a_p + dcomp_p phi,  dz_p = -b1_p da_p - b1_m da_m - db1_p a_p - db1_m a_m
    d rhs2 likewise with (shift_m, mean_m, beta2_p, beta2_m, kappa_m); comp = e^shift / (1 - mean) - 1 is differentiated through shift, mean."""

    def __init__(self, p: dict, name: str, phi: np.ndarray, psi: np.ndarray):
        assert name in ODE_NAMES, name
        self.p, self.phi, self.psi = p, np.asarray(phi, dtype=np.complex128), np.asarray(psi, dtype=np.complex128)
        self.d = {k: (1.0 if k == name else 0.0) for k in hawkes.KEYS}
        ep, em = np.exp(p["shift_p"]) / (1.0 - p["mean_p"]), np.exp(p["shift_m"]) / (1.0 - p["mean_m"])
        self.dcomp_p = ep * self.d["shift_p"] + ep / (1.0 - p["mean_p"]) * self.d["mean_p"]
        self.dcomp_m = em * self.d["shift_m"] + em / (1.0 - p["mean_m"]) * self.d["mean_m"]

    def __call__(self, A: np.ndarray, dA: np.ndarray, rows=None) -> np.ndarray:
        p, d = self.p, self.d
        phi, psi = (self.phi, self.psi) if rows is None else (self.phi[rows], self.psi[rows])
        a1, a2, da1, da2 = A[:, 1], A[:, 2], dA[:, 1], dA[:, 2]
        zp = phi - p["beta1_p"] * a1 - p["beta1_m"] * a2
        zm = phi - p["beta2_p"] * a1 - p["beta2_m"] * a2
        dzp = -(p["beta1_p"] * da1 + p["beta1_m"] * da2 + d["beta1_p"] * a1 + d["beta1_m"] * a2)
        dzm = -(p["beta2_p"] * da1 + p["beta2_m"] * da2 + d["beta2_p"] * a1 + d["beta2_m"] * a2)
        dkt_p = d["kappa_p"] * p["theta_p"] + p["kappa_p"] * d["theta_p"]
        dkt_m = d["kappa_m"] * p["theta_m"] + p["kappa_m"] * d["theta_m"]
        out = np.empty_like(A)
        out[:, 0] = (p["kappa_p"] * p["theta_p"] * da1 + p["kappa_m"] * p["theta_m"] * da2 + dkt_p * a1 + dkt_m * a2
                     + 2.0 * p["sigma"] * d["sigma"] * (0.5 * (phi + 1.0) * phi - psi))
        out[:, 1] = (_djump(zp, dzp, p["shift_p"], p["mean_p"], d["shift_p"], d["mean_p"]) - p["kappa_p"] * da1 - d["kappa_p"] * a1
                     + self.dcomp_p * phi)
        out[:, 2] = (_djump(zm, dzm, p["shift_m"], p["mean_m"], d["shift_m"], d["mean_m"]) - p["kappa_m"] * da2 - d["kappa_m"] * a2
                     + self.dcomp_m * phi)
        return out


def _grid(p, ttms, vol_scaler):
    if vol_scaler is None:
        vol_scaler = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    return mgf.phi_grid(vol_scaler, True, hawkes.MAX_PHI)           # Re phi = -1/2 under both measures (the pricer's grid)


def hawkes_chain_greeks(p: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, vol_scaler=None):
    """forward mode through the Hawkes chain (no risk kernel): per maturity [prices, delta, gamma, d price / d HAWKES_NAMES] ([18, J]), plus
    the grids dict(dlog_mgf [15, M, P], log_mgf [M, P], a [M, P, 3], nfev [P], meshes)"""
    phi = _grid(p, ttms, vol_scaler)
    psi = np.zeros_like(phi)
    P = phi.shape[0]
    rhs = hawkes.HawkesRhs(p, phi, psi)
    trhs = [HawkesTangentRhs(p, name, phi, psi) for name in ODE_NAMES]
    rows = [HAWKES_NAMES.index(name) for name in ODE_NAMES]
    a = np.zeros((P, 3), dtype=np.complex128)
    da = np.zeros((len(ODE_NAMES), P, 3), dtype=np.complex128)
    out, grids = [], dict(dlog_mgf=[], log_mgf=[], a=[], meshes=[])
    nfev = np.zeros(P, dtype=int)
    t0 = 0.0
    for m, ttm in enumerate(ttms):
        a, da, nf, mesh = G.rk45_grid_tangent(rhs, trhs, a, da, ttm - t0)
        nfev += nf
        lm = a[:, 0] + a[:, 1] * p["lambda_p"] + a[:, 2] * p["lambda_m"]
        dlm = np.empty((len(HAWKES_NAMES), P), dtype=np.complex128)
        for d, r in enumerate(rows):
            dlm[r] = da[d, :, 0] + da[d, :, 1] * p["lambda_p"] + da[d, :, 2] * p["lambda_m"]
        dlm[HAWKES_NAMES.index("lambda_p")], dlm[HAWKES_NAMES.index("lambda_m")] = a[:, 1], a[:, 2]
        out.append(G.vanilla_slice_greeks(lm, dlm, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], is_spot_measure))
        for key, val in (("dlog_mgf", dlm), ("log_mgf", lm), ("a", a.copy()), ("meshes", mesh)):
            grids[key].append(val)
        t0 = ttm
    grids["dlog_mgf"] = np.stack(grids["dlog_mgf"], axis=1)
    grids["log_mgf"] = np.array(grids["log_mgf"])
    grids["nfev"] = nfev
    return out, grids


def hawkes_chain_prices_on_meshes(p: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, meshes, vol_scaler, is_spot_measure=True):
    """the Hawkes chain prices with every maturity's ODE stepped on a recorded mesh (the scheme whose exact derivative the tangents are);
    returns (prices per maturity, log_mgf [M, P])"""
    phi = mgf.phi_grid(vol_scaler, True, hawkes.MAX_PHI)
    rhs = hawkes.HawkesRhs(p, phi, np.zeros_like(phi))
    a = np.zeros((phi.shape[0], 3), dtype=np.complex128)
    prices, lms = [], []
    for m in range(len(ttms)):
        a = G.replay(rhs, a, meshes[m])
        lm = a[:, 0] + a[:, 1] * p["lambda_p"] + a[:, 2] * p["lambda_m"]
        lms.append(lm)
        prices.append(mgf.vanilla_slice_prices(lm, phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], is_spot_measure))
    return prices, np.array(lms)
