"""Numpy forward-over-forward restatement of the Hawkes second-order Fourier chain sensitivities under the risk kernel exp(-gamma x)
(DESIGN.md §4.13).  TEST INFRASTRUCTURE ONLY.

Written from the maths, on ``hawkes_hessian_oracle`` (the hyper-dual Riccati right-hand side) and ``oracle.hawkes_rp_greeks`` (the
first-order risk-kernel scheme), both left as they are:

* ``rp_d2_log_mgf``: every pair of RP_NAMES seeded as a hyper-dual pair, the transform variable among the seeded variables (dphi = -1 on
  risk_premia_gamma), Dormand-Prince replayed on recorded meshes -- carried over the maturities on the grid, restarted at every maturity at
  the normaliser points -- and lm = a0 + a_p lambda_p + a_m lambda_m: the exact second derivative of the scheme on those meshes;
* ``rp_tangents_on_meshes``: the first-order rows of ``oracle.hawkes_rp_greeks`` with every solve stepped on a recorded mesh, which the
  tests difference;
* ``rp_slice_hessian``: the risk-kernel sums S_x, S_xp, S_pq and the vanna / Hessian assembly of DESIGN.md §4.13;
* ``hawkes_rp_chain_hessian``: the chain rows on the meshes ``oracle.hawkes_rp_greeks.hawkes_rp_chain_greeks`` recorded.
"""
from __future__ import annotations

import numpy as np

import hawkes_hessian_oracle as HH
import mgf_hessian_oracle as MH
from mgf_hessian_oracle import Hyper
from oracle import hawkes, mgf
from oracle import hawkes_rp_greeks as R

NAMES = R.RP_NAMES
G = len(NAMES) - 1                      # the index of risk_premia_gamma
PAIRS = MH.pairs(len(NAMES))            # the 136 hessian rows


def seeded_phi(phi, pairs):
    """the transform points as hyper-dual numbers over the pair axis: dphi / dgamma = -1, no second part (phi is linear in gamma)"""
    full = (len(pairs), phi.shape[0])
    d1 = np.array([-1.0 if a == G else 0.0 for a, _ in pairs])[:, None]
    d2 = np.array([-1.0 if b == G else 0.0 for _, b in pairs])[:, None]
    return Hyper(np.broadcast_to(phi, full), np.broadcast_to(d1, full), np.broadcast_to(d2, full), np.zeros(full))


def tan2_rhs(p: dict, a: int, b: int, phi, A, dAa, dAb, d2A):
    """(d_a f, d_b f, d_ab f) [P, 3] of the pair (a, b) of RP_NAMES at A [P, 3] with the tangents dA_a, dA_b and d2A, phi seeded"""
    par = {k: Hyper(v.v, v.d1[0, 0], v.d2[0, 0]) for k, v in HH.seeded(p, [(a, b)]).items()}
    ph = seeded_phi(phi, [(a, b)])[0]
    out = HH.rhs([Hyper(A[:, k], dAa[:, k], dAb[:, k], d2A[:, k]) for k in range(3)], par, ph)
    return tuple(np.stack([getattr(o, part) * np.ones(phi.shape[0]) for o in out], axis=1) for part in ("d1", "d2", "d12"))


def replay(A, par, phi, mesh):
    """hawkes_hessian_oracle.replay with phi hyper-dual over the pair axis too"""
    A = list(A)
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya, ph = [HH._cols(a, ja) for a in A], HH._cols(phi, ja)
        K = [HH.rhs(ya, par, ph)]
        for s in range(1, 6):
            K.append(HH.rhs([ya[k] + sum(K[j][k] * mgf._A[s][j] for j in range(s)) * h for k in range(3)], par, ph))
        for k in range(3):
            A[k] = HH._set(A[k], ja, ya[k] + h * sum(K[j][k] * mgf._B[j] for j in range(6)))
    return A


def rp_d2_log_mgf(p: dict, meshes, phi, restart=False, pairs=PAIRS):
    """(d2 lm [npairs, M, P], d lm along each pair's first name [npairs, M, P]) on recorded meshes; ``restart``: every maturity from A = 0
    (the normaliser points, meshes over the full ttms)"""
    par, ph = HH.seeded(p, pairs), seeded_phi(phi, pairs)
    full = (len(pairs), phi.shape[0])
    zero = lambda: [Hyper(np.zeros(full), np.zeros(full), np.zeros(full), np.zeros(full)) for _ in range(3)]
    A = zero()
    d2 = np.empty((len(pairs), len(meshes), phi.shape[0]), dtype=np.complex128)
    d1 = np.empty_like(d2)
    for m, mesh in enumerate(meshes):
        A = replay(zero() if restart else A, par, ph, mesh)
        lm = A[0] + A[1] * par["lambda_p"] + A[2] * par["lambda_m"]
        d2[:, m], d1[:, m] = lm.d12, lm.d1
    return d2, d1


def rp_tangents_on_meshes(p: dict, gamma: float, ttms, forwards, strikes_ttms, types_ttms, meshes, norm_meshes, vol_scaler):
    """the first-order risk-kernel rows of oracle.hawkes_rp_greeks with every solve stepped on a recorded mesh (grid carried, normaliser
    points restarted): (per maturity [prices, delta, gamma, d price / d RP_NAMES] [19, J], dlog_mgf [16, M, P], dlog_norm [16, M, 2])"""
    phi = R.rp_grid(p, gamma, ttms, vol_scaler)
    two = np.array([-gamma, -gamma - 1.0], dtype=np.complex128)
    rhs, trhs = hawkes.HawkesRhs(p, phi, np.zeros_like(phi)), R._tangent_rhs(p, phi)
    rhs2, trhs2 = hawkes.HawkesRhs(p, two, np.zeros(2, dtype=np.complex128)), R._tangent_rhs(p, two)
    a, da = np.zeros((phi.shape[0], 3), dtype=np.complex128), np.zeros((len(trhs), phi.shape[0], 3), dtype=np.complex128)
    out, dlms, dnorms = [], [], []
    for m in range(len(ttms)):
        a2, da2 = MH.replay_tangent(rhs2, trhs2, np.zeros((2, 3)), np.zeros((len(trhs2), 2, 3)), norm_meshes[m])
        lm2, dlm2 = R._log_mgf_rows(p, a2, da2)
        norm = 1.0 / np.exp(lm2[0].real)
        gfw = forwards[m] * np.exp(lm2[1].real) * norm
        a, da = MH.replay_tangent(rhs, trhs, a, da, meshes[m])
        lm, dlm = R._log_mgf_rows(p, a, da)
        out.append(R.gamma_slice_greeks(lm, dlm, phi, gamma, forwards[m], norm, gfw, np.real(dlm2), strikes_ttms[m], types_ttms[m]))
        dlms.append(dlm)
        dnorms.append(np.real(dlm2))
    return out, np.stack(dlms, axis=1), np.stack(dnorms, axis=1)


def rp_slice_hessian(log_mgf, dlog_mgf, d2log_mgf, phi, gamma, forward, normalizer, gamma_forward, dnorm, d2norm, strikes, types):
    """(vanna [16, J], hessian [136, J]) of the risk-kernel slice (DESIGN.md §4.13): with T_p = dlm_p (T_gamma = dlm_gamma + x),
    T_pq = d2lm_pq, c = n K^(1+g), c_p = -l0_p [+ ln K], c_pq = -l0_pq, g = l1 - l0,
      hessian_pq = [C] G (g_p g_q + g_pq) - c (S_pq + c_p S_q + c_q S_p + (c_p c_q + c_pq) S),
      vanna_p = ([C] G g_p - c (S_xp + c_p S_x)) / F."""
    w = R._weights(phi, gamma)
    n = len(NAMES)
    l0, l1, l0pq, l1pq = dnorm[:, 0], dnorm[:, 1], d2norm[:, 0], d2norm[:, 1]
    vanna, hess = np.zeros((n, len(strikes))), np.zeros((len(PAIRS), len(strikes)))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        x = np.log(forward / k)
        e = np.exp(-x * phi + log_mgf)
        term = w * e
        keep = ~np.isnan(np.real(term))
        ssum = lambda v: np.sum(np.real(v)[keep])
        T = dlog_mgf.copy()
        T[G] = T[G] + x
        S, Sx = ssum(term), ssum(-w * phi * e)
        Sp = np.array([ssum(term * T[a]) for a in range(n)])
        Sxp = np.array([ssum(term * (-phi * T[a] + (1.0 if a == G else 0.0))) for a in range(n)])
        c = normalizer * np.power(k, 1.0 + gamma)
        cp = -l0 + np.where(np.arange(n) == G, np.log(k), 0.0)
        call = str(ty) == "C"
        vanna[:, j] = ((gamma_forward * (l1 - l0) if call else 0.0) - c * (Sxp + cp * Sx)) / forward
        for r, (a, b) in enumerate(PAIRS):
            Sab = ssum(term * (T[a] * T[b] + d2log_mgf[r]))
            gpq = l1pq[r] - l0pq[r]
            hess[r, j] = ((gamma_forward * ((l1[a] - l0[a]) * (l1[b] - l0[b]) + gpq)) if call else 0.0) - \
                c * (Sab + cp[a] * Sp[b] + cp[b] * Sp[a] + (cp[a] * cp[b] - l0pq[r]) * S)
    return vanna, hess


def hawkes_rp_chain_hessian(p: dict, gamma: float, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler=None):
    """per maturity (first-order rows [19, J] of oracle.hawkes_rp_greeks.hawkes_rp_chain_greeks, vanna [16, J], hessian [136, J]), and the
    grids of hawkes_rp_chain_greeks plus d2log_mgf [136, M, P] and d2log_norm [136, M, 2] (Re parts)"""
    if vol_scaler is None:
        vol_scaler = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    out1, grids = R.hawkes_rp_chain_greeks(p, gamma, ttms, forwards, discfactors, strikes_ttms, types_ttms, vol_scaler)
    phi = R.rp_grid(p, gamma, ttms, vol_scaler)
    two = np.array([-gamma, -gamma - 1.0], dtype=np.complex128)
    grids["d2log_mgf"] = rp_d2_log_mgf(p, grids["meshes"], phi)[0]
    grids["d2log_norm"] = np.real(rp_d2_log_mgf(p, grids["norm_meshes"], two, restart=True)[0])
    rows = []
    for m in range(len(ttms)):
        v, h = rp_slice_hessian(grids["log_mgf"][m], grids["dlog_mgf"][:, m], grids["d2log_mgf"][:, m], phi, gamma, forwards[m],
                                grids["normalizers"][m], grids["gamma_forwards"][m], grids["dlog_norm"][:, m], grids["d2log_norm"][:, m],
                                strikes_ttms[m], types_ttms[m])
        rows.append((out1[m], v, h))
    return rows, grids
