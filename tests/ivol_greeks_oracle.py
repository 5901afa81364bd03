"""numpy restatement of the implied-vol sensitivity transform (csrc/ivol_kernels.cu, black_ivol_sensitivities_kernel; DESIGN.md §4.6).
TEST INFRASTRUCTURE ONLY.

The model ivol sigma(F, p) is defined by B(F, sigma) = P(F, p), B the discounted Black-76 price.  Given the ivols (from any inversion) and
the price rows in the layout of the *_price_chain_greeks / *_price_chain_hessian entry points, ``ivol_sensitivities`` returns the ivol rows
by the implicit-function rule, with the kernel's conventions: NaN ivol -> NaN rows, ivol at an end of the inversion bracket -> zero rows.

``black_in_model`` builds the inputs of a "Black-in" model, P = B(F, g(F, p)) with a known smooth g, whose price rows are written
analytically: the transform must give back g's derivatives.
"""
from __future__ import annotations

import numpy as np
from scipy.special import ndtr

from oracle import bsm as obsm

_INV_SQRT_2PI = 0.3989422804014327


def is_call_type(optiontypes) -> np.ndarray:
    return np.isin(np.asarray(optiontypes), ("C", "IC"))


def black_partials(F, K, T, D, vol, is_call):
    """(B_vol, B_F, B_FF, B_Fvol, B_volvol) of the discounted Black-76 price, in vol"""
    srt = np.sqrt(T)
    s = vol * srt
    d1 = np.log(F / K) / s + 0.5 * s
    d2 = d1 - s
    n = _INV_SQRT_2PI * np.exp(-0.5 * d1 * d1)
    vega = D * F * n * srt
    dF = D * np.where(is_call, ndtr(d1), -ndtr(-d1))
    dFF = D * n / (F * s)
    dFv = -D * n * d2 / vol
    dvv = vega * d1 * d2 / vol
    return vega, dF, dFF, dFv, dvv


def at_bracket_end(vol) -> np.ndarray:
    return (vol <= obsm.VOL_LO * (1.0 + 1e-10)) | (vol >= obsm.VOL_HI * (1.0 - 1e-10))


def ivol_sensitivities(F, K, T, D, vol, is_call, greeks, vanna=None, hessian=None):
    """ivol rows from price rows, all arrays flat over J quotes.  greeks [2 + P, J]; vanna [P, J] and hessian [P(P+1)/2, J] (upper
    triangle, row-major) or None.  -> (ivol_greeks [2 + P, J], ivol_vanna | None, ivol_hessian | None)"""
    greeks = np.asarray(greeks, float)
    P = greeks.shape[0] - 2
    with np.errstate(all="ignore"):
        vega, dF, dFF, dFv, dvv = black_partials(F, K, T, D, vol, is_call)
        sF = (greeks[0] - dF) / vega
        sFF = (greeks[1] - dFF - 2.0 * dFv * sF - dvv * sF * sF) / vega
        sp = greeks[2:] / vega
        g = np.vstack([sF, sFF, sp])
        v = h = None
        if vanna is not None:
            v = (np.asarray(vanna, float) - (dFv + dvv * sF) * sp) / vega
            idx = [(a, c) for a in range(P) for c in range(a, P)]
            h = np.vstack([(np.asarray(hessian, float)[r] - dvv * sp[a] * sp[c]) / vega for r, (a, c) in enumerate(idx)])
    nan, end = np.isnan(vol), at_bracket_end(vol)
    for rows in (g, v, h):
        if rows is not None:
            rows[:, end] = 0.0
            rows[:, nan] = np.nan
    return g, v, h


# ---- the Black-in model: g(F, p) = sigma0 exp(u), u = a.p + b L + p.Q.p / 2 + L e.p, L = ln(F / F0) --------------------------------
def black_in_vol(F, p, F0, sigma0, a, b, Q, e):
    """g and its exact derivatives (g, g_F, g_FF, g_p [P], g_Fp [P], g_pq [P, P]) for scalar F and parameter vector p"""
    L = np.log(F / F0)
    u = a @ p + b * L + 0.5 * p @ Q @ p + L * (e @ p)
    g = sigma0 * np.exp(u)
    u_p = a + Q @ p + L * e
    u_L = b + e @ p
    g_p = g * u_p
    g_pq = g * (np.outer(u_p, u_p) + Q)
    g_F = g * u_L / F
    g_FF = g * (u_L * u_L - u_L) / (F * F)
    g_Fp = g * (u_p * u_L + e) / F
    return g, g_F, g_FF, g_p, g_Fp, g_pq


def black_in_model(F, K, T, D, types, p, F0, sigma0, a, b, Q, e):
    """price P = B(F, g) of every quote (one slice, forward F) and its analytic rows: greeks [2 + P, J], vanna [P, J], hessian [P(P+1)/2, J];
    plus the vol derivatives they encode, as a dict of the same layouts (the answer the transform must give)"""
    K = np.asarray(K, float)
    is_call = is_call_type(types)
    g, g_F, g_FF, g_p, g_Fp, g_pq = black_in_vol(F, p, F0, sigma0, a, b, Q, e)
    vol = np.full(K.shape, g)
    itm = np.where(is_call, K < F, K > F)              # out-of-the-money side to its relative precision, plus the intrinsic value
    price = D * (obsm.otm_black_price(F, K, vol * np.sqrt(T)) + np.where(itm, np.abs(F - K), 0.0))
    vega, dF, dFF, dFv, dvv = black_partials(F, K, T, D, vol, is_call)
    n = len(p)
    idx = [(i, j) for i in range(n) for j in range(i, n)]
    greeks = np.vstack([dF + vega * g_F, dFF + 2.0 * dFv * g_F + dvv * g_F ** 2 + vega * g_FF, *(vega * g_p[k] for k in range(n))])
    vanna = np.vstack([dFv * g_p[k] + dvv * g_F * g_p[k] + vega * g_Fp[k] for k in range(n)])
    hessian = np.vstack([dvv * g_p[i] * g_p[j] + vega * g_pq[i, j] for i, j in idx])
    ones = np.ones(K.shape)
    want = {"ivol": g * ones, "greeks": np.vstack([g_F * ones, g_FF * ones, *(g_p[k] * ones for k in range(n))]),
            "vanna": np.vstack([g_Fp[k] * ones for k in range(n)]), "hessian": np.vstack([g_pq[i, j] * ones for i, j in idx])}
    return price, greeks, vanna, hessian, want


def strikes_for_d1(F, T, vol, d1s):
    """strikes at which the Black d1 of total vol vol sqrt T takes the values d1s"""
    s = vol * np.sqrt(T)
    return F * np.exp(-(np.asarray(d1s, float) - 0.5 * s) * s)


def default_black_in(n: int, seed: int = 7):
    """a fixed smooth Black-in model with n parameters: (p, sigma0, a, b, Q, e)"""
    rng = np.random.RandomState(seed)
    p = rng.uniform(-0.5, 0.5, n)
    a = rng.uniform(-0.3, 0.3, n)
    Qh = rng.uniform(-0.2, 0.2, (n, n))
    Q = 0.5 * (Qh + Qh.T)
    e = rng.uniform(-0.4, 0.4, n)
    return p, 0.35, a, -0.15, Q, e
