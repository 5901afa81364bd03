"""Numpy forward-over-forward restatement of the Hawkes second-order Fourier chain sensitivities (DESIGN.md §4.5).  TEST INFRASTRUCTURE
ONLY.

Written from the maths, next to ``oracle.hawkes_greeks`` and on the helpers of ``mgf_hessian_oracle``:

* ``rhs``: the Riccati right-hand side of ``oracle.hawkes.HawkesRhs`` on columns of any arithmetic type; with the parameters and A as
  hyper-dual numbers (``mgf_hessian_oracle.Hyper``) its mixed part is the second-order right-hand side
  J(A) d2A + f_AA(dA_p, dA_q) + d_p J dA_q + d_q J dA_p + d_pq f (``tan2_rhs``);
* ``hawkes_d2_log_mgf``: every pair of HAWKES_NAMES seeded as a hyper-dual pair along a leading pair axis, Dormand-Prince replayed on the
  meshes ``oracle.hawkes_greeks.hawkes_chain_greeks`` recorded, lm = a0 + a_p lambda_p + a_m lambda_m -- the exact second derivative of
  the scheme on that mesh, the lambda rows included (no special case: lm is hyper-dual in the lambdas too);
* ``hawkes_tangents_on_meshes``: first-order tangents (``oracle.hawkes_greeks.HawkesTangentRhs``) stepped on recorded meshes
  (``mgf_hessian_oracle.replay_tangent``), which the tests difference;
* ``hawkes_chain_hessian``: the chain rows through ``mgf_hessian_oracle.vanilla_slice_hessian``.
"""
from __future__ import annotations

import numpy as np

import mgf_hessian_oracle as MH
from mgf_hessian_oracle import Hyper
from oracle import hawkes, mgf
from oracle import hawkes_greeks as HG

NAMES = HG.HAWKES_NAMES
PAIRS = MH.pairs(len(NAMES))            # the 120 hessian rows


def rhs(A, par, phi):
    """oracle.hawkes.HawkesRhs (psi = 0) on the columns A = [a0, a_p, a_m] with parameters ``par`` (name -> Hyper)"""
    zp = phi - par["beta1_p"] * A[1] - par["beta1_m"] * A[2]
    zm = phi - par["beta2_p"] * A[1] - par["beta2_m"] * A[2]
    jp = (-(par["shift_p"] * zp)).exp() / (1.0 + par["mean_p"] * zp) - 1.0
    jm = (-(par["shift_m"] * zm)).exp() / (1.0 + par["mean_m"] * zm) - 1.0
    comp_p = par["shift_p"].exp() / (1.0 - par["mean_p"]) - 1.0
    comp_m = par["shift_m"].exp() / (1.0 - par["mean_m"]) - 1.0
    return [par["kappa_p"] * par["theta_p"] * A[1] + par["kappa_m"] * par["theta_m"] * A[2] + par["sigma"] * par["sigma"] * (0.5 * (phi + 1.0) * phi),
            jp - par["kappa_p"] * A[1] + comp_p * phi,
            jm - par["kappa_m"] * A[2] + comp_m * phi]


def seeded(p: dict, pairs):
    """the parameters as hyper-dual numbers over a leading pair axis: d1 along the pair's first name, d2 along its second"""
    out = {}
    for k, name in enumerate(NAMES):
        d1 = np.array([1.0 if a == k else 0.0 for a, _ in pairs])[:, None]
        d2 = np.array([1.0 if b == k else 0.0 for _, b in pairs])[:, None]
        out[name] = Hyper(p[name], d1, d2)
    return out


def tan2_rhs(p: dict, a: int, b: int, phi, A, dAa, dAb, d2A):
    """(d_a f, d_b f, d_ab f) [P, 3] of the pair (a, b) of HAWKES_NAMES at A [P, 3] with the tangents dA_a, dA_b and d2A"""
    par = {k: Hyper(v.v, v.d1[0, 0], v.d2[0, 0]) for k, v in seeded(p, [(a, b)]).items()}
    out = rhs([Hyper(A[:, k], dAa[:, k], dAb[:, k], d2A[:, k]) for k in range(3)], par, phi)
    return tuple(np.stack([getattr(o, part) * np.ones(phi.shape[0]) for o in out], axis=1) for part in ("d1", "d2", "d12"))


def _cols(a, ja):
    return a[..., ja]


def _set(a, ja, val):
    parts = []
    for x, y in zip(a.parts(), val.parts()):
        x = np.array(np.broadcast_to(x, a.v.shape), dtype=np.complex128)
        x[..., ja] = y
        parts.append(x)
    return Hyper(*parts)


def replay(A, par, phi, mesh):
    """oracle.mgf_greeks.replay on the hyper-dual columns A [npairs, P] (the pair axis leads, the mesh indexes the points)"""
    A = list(A)
    for ja, h in mesh:
        if ja.shape[0] == 0:
            continue
        ya, ph = [_cols(a, ja) for a in A], phi[ja]
        K = [rhs(ya, par, ph)]
        for s in range(1, 6):
            K.append(rhs([ya[k] + sum(K[j][k] * mgf._A[s][j] for j in range(s)) * h for k in range(3)], par, ph))
        for k in range(3):
            A[k] = _set(A[k], ja, ya[k] + h * sum(K[j][k] * mgf._B[j] for j in range(6)))
    return A


def hawkes_d2_log_mgf(p: dict, meshes, phi, pairs=PAIRS):
    """(d2 lm [npairs, M, P], d lm along each pair's first name [npairs, M, P]) on recorded meshes"""
    par = seeded(p, pairs)
    full = (len(pairs), phi.shape[0])
    A = [Hyper(np.zeros(full), np.zeros(full), np.zeros(full), np.zeros(full)) for _ in range(3)]
    d2 = np.empty((len(pairs), len(meshes), phi.shape[0]), dtype=np.complex128)
    d1 = np.empty_like(d2)
    for m, mesh in enumerate(meshes):
        A = replay(A, par, phi, mesh)
        lm = A[0] + A[1] * par["lambda_p"] + A[2] * par["lambda_m"]
        d2[:, m], d1[:, m] = lm.d12, lm.d1
    return d2, d1


def hawkes_tangents_on_meshes(p: dict, meshes, phi):
    """first-order tangents of the 13 ODE directions on recorded meshes -> (a [M, P, 3], dlog_mgf [15, M, P])"""
    psi = np.zeros_like(phi)
    f = hawkes.HawkesRhs(p, phi, psi)
    trhs = [HG.HawkesTangentRhs(p, name, phi, psi) for name in HG.ODE_NAMES]
    a, da = np.zeros((phi.shape[0], 3), dtype=np.complex128), np.zeros((len(trhs), phi.shape[0], 3), dtype=np.complex128)
    As, dlm = [], np.empty((len(NAMES), len(meshes), phi.shape[0]), dtype=np.complex128)
    for m, mesh in enumerate(meshes):
        a, da = MH.replay_tangent(f, trhs, a, da, mesh)
        As.append(a.copy())
        for d, name in enumerate(HG.ODE_NAMES):
            dlm[NAMES.index(name), m] = da[d, :, 0] + da[d, :, 1] * p["lambda_p"] + da[d, :, 2] * p["lambda_m"]
        dlm[NAMES.index("lambda_p"), m], dlm[NAMES.index("lambda_m"), m] = a[:, 1], a[:, 2]
    return np.array(As), dlm


def chain_rows(p: dict, phi, lm, dlm, d2lm, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True):
    """per maturity (vanna [15, J], hessian [120, J]) from the grids"""
    return [MH.vanilla_slice_hessian(lm[m], dlm[:, m], d2lm[:, m], phi, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m],
                                     is_spot_measure) for m in range(lm.shape[0])]


def hawkes_chain_hessian(p: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure=True, vol_scaler=None):
    """per maturity (first-order rows [18, J] of oracle.hawkes_greeks.hawkes_chain_greeks, vanna [15, J], hessian [120, J]), and the
    grids of hawkes_chain_greeks plus d2log_mgf [120, M, P]"""
    if vol_scaler is None:
        vol_scaler = hawkes.fourier_vol_scaler(p["sigma"], float(np.min(ttms)))
    out1, grids = HG.hawkes_chain_greeks(p, ttms, forwards, discfactors, strikes_ttms, types_ttms, is_spot_measure, vol_scaler)
    phi = mgf.phi_grid(vol_scaler, True, hawkes.MAX_PHI)
    grids["d2log_mgf"] = hawkes_d2_log_mgf(p, grids["meshes"], phi)[0]
    rows = chain_rows(p, phi, grids["log_mgf"], grids["dlog_mgf"], grids["d2log_mgf"], forwards, discfactors, strikes_ttms, types_ttms,
                      is_spot_measure)
    return [(out1[m], v, h) for m, (v, h) in enumerate(rows)], grids
