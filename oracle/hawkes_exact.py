"""CPU restatement (numpy) of the exact event-driven route of the Hawkes jump-diffusion Monte Carlo (DESIGN.md §3.13,
csrc/hawkes_kernels.cuh ``hawkes_exact_slice_kernel``).  TEST INFRASTRUCTURE ONLY (oracle/__init__.py).

The continuous-time limit of the Euler step of ``oracle.hawkes.step_fixed``, simulated without a grid by thinning (Ogata).  Per path and
maturity interval of length T, from the carried state (x, lambda_p, lambda_m):
  bound      at each candidate's start s, per intensity the largest value of its monotone deterministic path on [s, T]: max(lambda, theta, 0)
             for kappa >= 0, max(lambda, lambda(T), 0) for kappa < 0 (growing away from theta); Lbar = their sum; Lbar = 0: advance to T
  candidate  d = E / Lbar with E = -ln(u53); s + d >= T: advance to T; else advance by d and accept '+' if v Lbar < max(lambda_p, 0), '-' if
             v Lbar < max(lambda_p, 0) + max(lambda_m, 0), else reject
  segment    lambda <- theta + (lambda - theta) e^{-kappa d},  int lambda += theta d + (lambda - theta) (1 - e^{-kappa d}) / kappa  (d at kappa = 0)
  jump       J = shift + mean E_J; '+' adds (J, beta1_p J, beta1_m J) to (x, lambda_p, lambda_m), '-' adds (J, beta2_p J, beta2_m J)
  end        x += (mu - sigma^2/2) T - c_p int lambda_p - c_m int lambda_m + sigma sqrt(T) z,  c = e^shift / (1 - mean) - 1

Draws, from the same Philox4x32-10 as the device (oracle.mc.philox4x32_10), key = (seed_lo, seed_hi), counter = (path_lo, path_hi, call,
maturity index | 0xC0000000):
  call = k, candidate k of the interval:  (r0, r1) -> u53 = (((r0:r1) >> 11) + 1) 2^-53 in (0, 1], the waiting time's uniform;
                                          r2 -> v = (r2 + 1/2) 2^-32, the thinning uniform;
                                          r3 -> E_J = -ln((r3 + 1/2) 2^-32), the jump size's unit exponential (used when accepted)
  call = 0xFFFFFFFF:                      z = Z0 of the fp64 Box-Muller on the block (oracle.mc.device_normals, gauss="f64")
"""
from __future__ import annotations

import numpy as np

from . import mc as _mc
from .hawkes import KEYS  # noqa: F401  (parameter order of the golden sets)

STREAM = 0xC0000000
NORMAL_CALL = 0xFFFFFFFF
DEFAULT_BUDGET = 1 << 20


class BudgetExhausted(RuntimeError):
    """a path drew more candidates in one interval than the budget allows (the device returns -6)"""


def _u53(hi, lo):
    b = ((hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)) >> np.uint64(11)
    return (b + np.uint64(1)).astype(np.float64) * 2.0 ** -53


def _u32(r):
    return (r.astype(np.float64) + 0.5) * 2.0 ** -32


def _decay(lam, integral, theta, kappa, d):
    """one deterministic segment of length d: (lambda at its end, integral + the integral over it)"""
    em = np.expm1(-kappa * d)
    g = -em / kappa if kappa != 0.0 else d
    dev = lam - theta
    return theta + dev * (1.0 + em), integral + (theta * d + dev * g)


def _rate_bound(lam, theta, kappa, rest):
    """the largest firing rate of one intensity on its deterministic path from the candidate's start to the interval end"""
    far = theta if kappa >= 0.0 else theta + (lam - theta) * np.exp(-kappa * rest)
    return np.maximum(np.maximum(lam, far), 0.0)


def normals(seed: int, path_ids, slice_idx: int):
    """the interval's unit normal z per path"""
    path_ids = np.asarray(path_ids, dtype=np.uint64)
    r0, r1, r2, r3 = _mc.philox4x32_10(path_ids & _mc._MASK, path_ids >> np.uint64(32), np.uint64(NORMAL_CALL), np.uint64(STREAM | slice_idx),
                                       seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u1 = 2.0 - _mc._u52(r0, r1 | np.uint32(1))
    u2 = _mc._u52(r2, r3) - 1.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def interval(x, lp, lm, T: float, p: dict, seed: int, slice_idx: int, path_ids, budget: int = DEFAULT_BUDGET):
    """one maturity interval of length T on the given global path ids -> (x, lambda_p, lambda_m, events [3, n]) with events = (accepted '+',
    accepted '-', candidates)"""
    x, lp, lm = (np.array(a, dtype=np.float64, copy=True) for a in (x, lp, lm))
    path_ids = np.asarray(path_ids, dtype=np.uint64)
    n = x.shape[0]
    plo, phi = path_ids & _mc._MASK, path_ids >> np.uint64(32)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    tag = np.uint64(STREAM | slice_idx)
    s, ip, im = np.zeros(n), np.zeros(n), np.zeros(n)
    k, n_p, n_m = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
    idx = np.arange(n)
    while idx.size:
        rest = T - s[idx]
        bound = _rate_bound(lp[idx], p["theta_p"], p["kappa_p"], rest) + _rate_bound(lm[idx], p["theta_m"], p["kappa_m"], rest)
        r0, r1, r2, r3 = _mc.philox4x32_10(plo[idx], phi[idx], k[idx].astype(np.uint64), tag, k0, k1)
        with np.errstate(divide="ignore", invalid="ignore"):
            dc = -np.log(_u53(r0, r1)) / bound
        cand = (bound > 0.0) & (s[idx] + dc < T)
        if np.any(cand & (k[idx] >= budget)):
            raise BudgetExhausted(f"a path drew more than {budget} candidates")
        d = np.where(cand, dc, T - s[idx])
        lp[idx], ip[idx] = _decay(lp[idx], ip[idx], p["theta_p"], p["kappa_p"], d)
        lm[idx], im[idx] = _decay(lm[idx], im[idx], p["theta_m"], p["kappa_m"], d)
        j = idx[cand]
        s[j] += d[cand]
        k[j] += 1
        v = _u32(r2[cand]) * bound[cand]
        pp = np.maximum(lp[j], 0.0)
        fire_p = v < pp
        fire_m = ~fire_p & (v < pp + np.maximum(lm[j], 0.0))
        e = -np.log(_u32(r3[cand]))
        jp = p["shift_p"] + p["mean_p"] * e
        jm = p["shift_m"] + p["mean_m"] * e
        for fire, jump, b_p, b_m, cnt in ((fire_p, jp, p["beta1_p"], p["beta1_m"], n_p), (fire_m, jm, p["beta2_p"], p["beta2_m"], n_m)):
            jj, jv = j[fire], jump[fire]
            x[jj] += jv
            lp[jj] += b_p * jv
            lm[jj] += b_m * jv
            cnt[jj] += 1
        idx = j
    c_p = np.exp(p["shift_p"]) / (1.0 - p["mean_p"]) - 1.0
    c_m = np.exp(p["shift_m"]) / (1.0 - p["mean_m"]) - 1.0
    drift = p["mu"] - 0.5 * p["sigma"] * p["sigma"]
    z = normals(seed, path_ids, slice_idx)
    x += ((drift * T - c_p * ip) - c_m * im) + p["sigma"] * np.sqrt(T) * z
    return x, lp, lm, np.stack([n_p, n_m, k]).astype(np.float64)


def terminal(p: dict, ttm: float, nb_path: int, seed: int, slice_idx: int = 0, path0: int = 0, budget: int = DEFAULT_BUDGET):
    """b200sv_hawkesjd_terminal_exact from (0, lambda_p, lambda_m): (x, lambda_p, lambda_m, events)"""
    n = int(nb_path)
    return interval(np.zeros(n), np.full(n, p["lambda_p"]), np.full(n, p["lambda_m"]), float(ttm), p, seed, slice_idx,
                    np.arange(path0, path0 + n, dtype=np.uint64), budget)


def chain(p: dict, ttms, forwards, discfactors, strikes_ttms, types_ttms, nb_path: int, seed: int, budget: int = DEFAULT_BUDGET):
    """b200sv_hawkesjd_mc_chain_exact: (prices, std errors, states [M][3][n], events [M][3][n]); the state of maturity m seeds m + 1 and
    the payoffs are the Euler chain's (oracle.mc.mc_payoffs on x)"""
    n = int(nb_path)
    x, lp, lm = np.zeros(n), np.full(n, p["lambda_p"]), np.full(n, p["lambda_m"])
    ids = np.arange(n, dtype=np.uint64)
    prices, stds, states, events = [], [], [], []
    for m, ttm in enumerate(ttms):
        T = ttms[m] - (ttms[m - 1] if m > 0 else 0.0)
        x, lp, lm, ev = interval(x, lp, lm, float(T), p, seed, m, ids, budget)
        pr, se = _mc.mc_payoffs(x, x, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m])
        prices.append(pr)
        stds.append(se)
        states.append(np.stack([x, lp, lm]))
        events.append(ev)
    return prices, stds, np.array(states), np.array(events)


def mean_equations(p: dict, T: float):
    """closed forms of the linear mean equations d m / dt = K (theta - m) + B m, B_ij = beta_ij E[J_j], exact where the intensities cannot
    become negative: (E[lambda_p(T)], E[lambda_m(T)], E[N_p(T)], E[N_m(T)]) from (lambda_p, lambda_m) at 0"""
    from scipy.linalg import expm
    ej_p, ej_m = p["shift_p"] + p["mean_p"], p["shift_m"] + p["mean_m"]
    a = np.zeros((5, 5))
    a[0, :2] = (p["beta1_p"] * ej_p - p["kappa_p"], p["beta2_p"] * ej_m)
    a[1, :2] = (p["beta1_m"] * ej_p, p["beta2_m"] * ej_m - p["kappa_m"])
    a[:2, 2] = (p["kappa_p"] * p["theta_p"], p["kappa_m"] * p["theta_m"])
    a[3, 0] = a[4, 1] = 1.0
    y = expm(a * float(T)) @ np.array([p["lambda_p"], p["lambda_m"], 1.0, 0.0, 0.0])
    return y[0], y[1], y[3], y[4]
