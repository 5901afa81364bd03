"""oracle.hawkes_rp_greeks -- numpy forward-mode restatement of the Hawkes Fourier chain sensitivities under the risk kernel exp(-gamma x)
(DESIGN.md §4.12).  TEST INFRASTRUCTURE ONLY.

Written from the maths, next to ``oracle.hawkes_greeks`` (left as it is):

* ``HawkesPhiTangentRhs``: J(A) dA + dphi d f(A) / d phi of the Riccati system, the direction of the transform variable;
* ``gamma_slice_greeks``: the risk-kernel slice sums of ``oracle.hawkes.gamma_slice_prices`` and their derivatives;
* ``hawkes_rp_chain_greeks``: prices, delta, gamma and d price / d RP_NAMES of a chain, with the restarted normaliser tangents at -gamma and
  -gamma - 1 and the carried grid tangents, driving ``mgf_greeks.rk45_grid_tangent``;
* ``hawkes_rp_chain_prices_on_meshes``: the chain prices with every solve stepped on a recorded mesh (``mgf_greeks.replay``), the scheme
  whose exact derivative the tangents are.
"""
from __future__ import annotations

import numpy as np

from . import hawkes, mgf
from . import mgf_greeks as G
from .hawkes_greeks import HAWKES_NAMES, ODE_NAMES, HawkesTangentRhs

RP_NAMES = HAWKES_NAMES + ("risk_premia_gamma",)
_ODE_ROWS = [HAWKES_NAMES.index(n) for n in ODE_NAMES]


class HawkesPhiTangentRhs:
    """tangent of oracle.hawkes.HawkesRhs along a move ``dphi`` of every transform point (psi fixed), plus J(A) dA:
    d rhs0 = k_p th_p da_p + k_m th_m da_m + sigma^2 (phi + 1/2) dphi
    d rhs1 = E_p'(z_p) dz_p - k_p da_p + comp_p dphi,  dz_p = dphi - b1_p da_p - b1_m da_m
    d rhs2 likewise with (shift_m, mean_m, beta2_p, beta2_m, kappa_m).  risk_premia_gamma moves every point by dphi = -1."""

    def __init__(self, p: dict, phi: np.ndarray, psi: np.ndarray, dphi: float = 1.0):
        self.p, self.phi, self.dphi = p, np.asarray(phi, dtype=np.complex128), float(dphi)
        self.comp_p = np.exp(p["shift_p"]) / (1.0 - p["mean_p"]) - 1.0
        self.comp_m = np.exp(p["shift_m"]) / (1.0 - p["mean_m"]) - 1.0

    def __call__(self, A: np.ndarray, dA: np.ndarray, rows=None) -> np.ndarray:
        p, dphi = self.p, self.dphi
        phi = self.phi if rows is None else self.phi[rows]
        a1, a2, da1, da2 = A[:, 1], A[:, 2], dA[:, 1], dA[:, 2]
        zp = phi - p["beta1_p"] * a1 - p["beta1_m"] * a2
        zm = phi - p["beta2_p"] * a1 - p["beta2_m"] * a2
        dzp = dphi - (p["beta1_p"] * da1 + p["beta1_m"] * da2)
        dzm = dphi - (p["beta2_p"] * da1 + p["beta2_m"] * da2)
        rp = 1.0 / (1.0 + p["mean_p"] * zp)
        rm = 1.0 / (1.0 + p["mean_m"] * zm)
        ep = np.exp(-p["shift_p"] * zp) * rp
        em = np.exp(-p["shift_m"] * zm) * rm
        out = np.empty_like(A)
        out[:, 0] = p["kappa_p"] * p["theta_p"] * da1 + p["kappa_m"] * p["theta_m"] * da2 + np.square(p["sigma"]) * (phi + 0.5) * dphi
        out[:, 1] = -ep * (p["shift_p"] + p["mean_p"] * rp) * dzp - p["kappa_p"] * da1 + self.comp_p * dphi
        out[:, 2] = -em * (p["shift_m"] + p["mean_m"] * rm) * dzm - p["kappa_m"] * da2 + self.comp_m * dphi
        return out


def _tangent_rhs(p, phi):
    psi = np.zeros_like(phi)
    return [HawkesTangentRhs(p, name, phi, psi) for name in ODE_NAMES] + [HawkesPhiTangentRhs(p, phi, psi, -1.0)]


def _log_mgf_rows(p, a, da):
    """log_mgf [P] and its 16 derivative rows [16, P] from A [P, 3] and the 14 tangents da [14, P, 3]"""
    lam = lambda y: y[..., 0] + y[..., 1] * p["lambda_p"] + y[..., 2] * p["lambda_m"]
    dlm = np.empty((len(RP_NAMES), a.shape[0]), dtype=np.complex128)
    dlm[_ODE_ROWS] = lam(da[:len(ODE_NAMES)])
    dlm[HAWKES_NAMES.index("lambda_p")], dlm[HAWKES_NAMES.index("lambda_m")] = a[:, 1], a[:, 2]
    dlm[-1] = lam(da[-1])
    return lam(a), dlm


def rp_grid(p: dict, gamma: float, ttms, vol_scaler=None) -> np.ndarray:
    """the pricer's grid under the risk kernel: Re phi = -1/2 - gamma, the imaginary parts of the plain grid"""
    if vol_scaler is None:
        vol_scaler = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    return (-0.5 - gamma) + 1j * np.imag(mgf.phi_grid(vol_scaler, True, hawkes.MAX_PHI))


def _weights(phi, gamma):
    """the weights of oracle.hawkes.gamma_slice_prices (fast branch at gamma = -1/2 only)"""
    dp = mgf.legacy_simpson_weights(phi)
    if np.all(np.abs(np.real(phi) - (0.5 + gamma)) < 1e-10):
        return (dp / np.pi) / (np.imag(phi) ** 2 + 0.25) + 0j
    return -(dp / np.pi) / ((phi + gamma + 1.0) * (phi + gamma))


def gamma_slice_greeks(log_mgf, dlog_mgf, phi, gamma, forward, normalizer, gamma_forward, dnorm, strikes, types):
    """(prices, delta, gamma, dprice [16, J]) of the risk-kernel slice: call G - n K^(1+g) S, put K - n K^(1+g) S with n = e^{-l0},
    G = F e^{l1} n; dlog_mgf [16, P] the log-MGF rows, dnorm [16, 2] the derivatives of (l0, l1).  The gamma row adds the grid's move
    (S_g = sum Re(w e (x + dlm_g))) and d K^(1+g) / d g = ln K K^(1+g)."""
    w = _weights(phi, gamma)
    prices = hawkes.gamma_slice_prices(log_mgf, phi, gamma, forward, normalizer, gamma_forward, strikes, types)
    out = np.zeros((3 + len(RP_NAMES), len(strikes)))
    l0, l1 = dnorm[:, 0], dnorm[:, 1]
    for j, (k, ty) in enumerate(zip(strikes, types)):
        x = np.log(forward / k)
        e = np.exp(-x * phi + log_mgf)
        term = w * e
        keep = ~np.isnan(np.real(term))
        ssum = lambda v: np.sum(np.real(v)[keep])
        S, Sx, Sxx = ssum(term), ssum(-w * phi * e), ssum(w * phi * phi * e)
        Sp = np.array([ssum(term * d) for d in dlog_mgf[:-1]] + [ssum(term * (x + dlog_mgf[-1]))])
        ngk = normalizer * np.power(k, 1.0 + gamma)
        call = str(ty) == "C"
        ln_k = np.zeros(len(RP_NAMES))
        ln_k[-1] = np.log(k) * S
        out[0, j] = prices[j]
        out[1, j] = (gamma_forward / forward if call else 0.0) - ngk * Sx / forward
        out[2, j] = -ngk * (Sxx - Sx) / forward ** 2
        out[3:, j] = (gamma_forward * (l1 - l0) if call else 0.0) - ngk * (Sp - l0 * S + ln_k)
    return out


def hawkes_rp_chain_greeks(p: dict, gamma: float, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None):
    """forward mode through the Hawkes chain under the risk kernel: per maturity [prices, delta, gamma, d price / d RP_NAMES] ([19, J]),
    plus the grids dict(dlog_mgf [16, M, P], dlog_norm [16, M, 2], log_mgf [M, P], normalizers [M], gamma_forwards [M], nfev [P],
    meshes, norm_meshes).  discfactors are not applied (as in the pricer)."""
    phi = rp_grid(p, gamma, ttms, vol_scaler)
    P = phi.shape[0]
    two = np.array([-gamma, -gamma - 1.0], dtype=np.complex128)
    rhs2, trhs2 = hawkes.HawkesRhs(p, two, np.zeros(2, dtype=np.complex128)), _tangent_rhs(p, two)
    rhs, trhs = hawkes.HawkesRhs(p, phi, np.zeros_like(phi)), _tangent_rhs(p, phi)
    a = np.zeros((P, 3), dtype=np.complex128)
    da = np.zeros((len(trhs), P, 3), dtype=np.complex128)
    out, nfev, t0 = [], np.zeros(P, dtype=int), 0.0
    grids = dict(dlog_mgf=[], dlog_norm=[], log_mgf=[], normalizers=[], gamma_forwards=[], meshes=[], norm_meshes=[])
    for m, ttm in enumerate(ttms):
        a2, da2, _, mesh2 = G.rk45_grid_tangent(rhs2, trhs2, np.zeros((2, 3), dtype=np.complex128),
                                                np.zeros((len(trhs2), 2, 3), dtype=np.complex128), float(ttm))
        lm2, dlm2 = _log_mgf_rows(p, a2, da2)
        norm = 1.0 / np.exp(lm2[0].real)
        gfw = forwards[m] * np.exp(lm2[1].real) * norm
        dnorm = np.real(dlm2)
        a, da, nf, mesh = G.rk45_grid_tangent(rhs, trhs, a, da, ttm - t0)
        nfev += nf
        lm, dlm = _log_mgf_rows(p, a, da)
        out.append(gamma_slice_greeks(lm, dlm, phi, gamma, forwards[m], norm, gfw, dnorm, strikes_ttms[m], types_ttms[m]))
        for key, val in (("dlog_mgf", dlm), ("dlog_norm", dnorm), ("log_mgf", lm), ("normalizers", norm), ("gamma_forwards", gfw),
                         ("meshes", mesh), ("norm_meshes", mesh2)):
            grids[key].append(val)
        t0 = ttm
    grids["dlog_mgf"] = np.stack(grids["dlog_mgf"], axis=1)
    grids["dlog_norm"] = np.stack(grids["dlog_norm"], axis=1)
    grids["log_mgf"] = np.array(grids["log_mgf"])
    grids["nfev"] = nfev
    return out, grids


def hawkes_rp_chain_prices_on_meshes(p: dict, gamma: float, ttms, forwards, strikes_ttms, types_ttms, meshes, norm_meshes, vol_scaler):
    """the risk-kernel chain prices with every solve (grid carried over the maturities, normaliser points restarted) stepped on a
    recorded mesh; returns (prices per maturity, log_mgf [M, P], Re log-MGF at the normaliser points [M, 2])"""
    phi = rp_grid(p, gamma, ttms, vol_scaler)
    two = np.array([-gamma, -gamma - 1.0], dtype=np.complex128)
    rhs, rhs2 = hawkes.HawkesRhs(p, phi, np.zeros_like(phi)), hawkes.HawkesRhs(p, two, np.zeros(2, dtype=np.complex128))
    lam = lambda y: y[:, 0] + y[:, 1] * p["lambda_p"] + y[:, 2] * p["lambda_m"]
    a = np.zeros((phi.shape[0], 3), dtype=np.complex128)
    prices, lms, l2s = [], [], []
    for m in range(len(ttms)):
        l2 = np.real(lam(G.replay(rhs2, np.zeros((2, 3), dtype=np.complex128), norm_meshes[m])))
        norm = 1.0 / np.exp(l2[0])
        a = G.replay(rhs, a, meshes[m])
        lm = lam(a)
        prices.append(hawkes.gamma_slice_prices(lm, phi, gamma, forwards[m], norm, forwards[m] * np.exp(l2[1]) * norm, strikes_ttms[m],
                                                types_ttms[m]))
        lms.append(lm)
        l2s.append(l2)
    return prices, np.array(lms), np.array(l2s)
