"""oracle.bsm -- Black-76 prices and implied-volatility inversion on the host (numpy).  TEST INFRASTRUCTURE ONLY: the checker of
``black_implied_vol`` (stochvolmodels_b200/csrc/black.cuh), which every GPU inversion runs.

Two inversions, both on the out-of-the-money side of the quote (the put for K < F, the call for K >= F):
  * ``infer_bsm_implied_vol``: an independent 80-step bisection;
  * ``black_implied_vol_newton``: a numpy restatement of the kernel's safeguarded Newton iteration, step for step, with its
    iteration count.
An in-the-money quote is turned into its out-of-the-money twin by parity, q = p / D - |F - K|, with the rounding errors of the
division and of the subtraction carried along (``otm_quote``), so the time value is kept to its own relative precision instead of
the absolute precision of p.

In the reference this step is third-party: ``vanilla_option_pricers.infer_bsm_ivols_from_model_chain_prices`` called from
``data/option_chain.py:327-346``; that package is not part of the reference tree and is absent here, so bit-level parity
with it is UNPINNED (SURVEY.md §8c).  What the reference pins is satisfied by any correct inversion: the quickstart
implied vols 0.999577 / 0.995757 (examples/getting_started/quickstart.py:44,46, rtol 5e-6) and flat-vol round trips.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
from scipy.special import erfcx, ndtr

VOL_LO, VOL_HI = 1e-8, 10.0          # the inversion bracket (annualised vol); roots outside it return its nearer end
MAX_ITER = 64                        # iteration cap of the kernel's Newton loop
_SQRT_2PI = 2.5066282746310002
_INV_SQRT_2PI = 0.3989422804014327


def compute_bsm_vanilla_price(forward, strike, ttm, vol, optiontype="C", discfactor=1.0):
    """undiscounted-forward Black-76 price times discfactor; 'IC'/'IP' are quoted in the same units as 'C'/'P'."""
    forward, strike, vol = np.asarray(forward, float), np.asarray(strike, float), np.asarray(vol, float)
    sdev = vol * np.sqrt(ttm)
    with np.errstate(divide="ignore", invalid="ignore"):
        d1 = np.log(forward / strike) / sdev + 0.5 * sdev
    d2 = d1 - sdev
    call = forward * ndtr(d1) - strike * ndtr(d2)
    is_call = np.isin(np.asarray(optiontype), ("C", "IC"))
    return discfactor * np.where(is_call, call, call - (forward - strike))


def otm_black_price(forward, strike, sdev):
    """undiscounted Black-76 price of the out-of-the-money option at total vol ``sdev``: the put K N(-d2) - F N(-d1) for K < F, else
    the call F N(d1) - K N(d2).  Each is a small difference of small terms, so it keeps its relative precision deep in the tails."""
    forward, strike, sdev = np.broadcast_arrays(*(np.asarray(a, float) for a in (forward, strike, sdev)))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return _otm_terms(forward, strike, np.log(forward / strike), sdev)[0]


def _otm_terms(F, K, x, s):
    """-> (price, t1, t2, vega) of the out-of-the-money side at total vol s, x = ln(F/K): price = t1 - t2 with the rounding of d1 and d2
    carried to first order (two-sum errors e1, e2 of xs +- s/2; F phi(d1) = K phi(d2) = vega), as black.cuh evaluates it."""
    xs, hs = x / s, 0.5 * s
    d1, d2 = xs + hs, xs - hs
    bb = d1 - xs
    e1 = (xs - (d1 - bb)) + (hs - bb)
    bb = d2 - xs
    e2 = (xs - (d2 - bb)) + (-hs - bb)
    put_side = K < F
    t1 = np.where(put_side, K * _ncdf(-d2), F * _ncdf(d1))
    t2 = np.where(put_side, F * _ncdf(-d1), K * _ncdf(d2))
    vega = F * _INV_SQRT_2PI * np.exp(-0.5 * d1 * d1)
    return (t1 - t2) + vega * (e1 - e2), t1, t2, vega


def _ncdf(z):
    """N(z) to a few ulp over the whole range, as the device's normcdf (documented to 5 ulp).  scipy's ndtr forms exp(-z^2 / 2) from
    a rounded z^2, which costs z^2 ulp in the lower tail; here z^2 is split exactly and the scaled erfcx carries the rest."""
    z = np.asarray(z, float)
    with np.errstate(all="ignore"):
        hi, lo = _two_prod(z, z)
        tail = 0.5 * erfcx(-z / np.sqrt(2.0)) * np.exp(-0.5 * hi) * (1.0 - 0.5 * lo)
    return np.where(z < -1.0, tail, ndtr(z))


# ---- error-free transformations (what fma gives the kernel) -------------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _fma(a, b, c):
    """a b + c rounded once, where c - a b is small against c (a quotient's remainder) or only its sign is used."""
    p, e = _two_prod(a, b)
    return (p + c) + e


def otm_quote(forward, strike, discfactor, price, is_call):
    """-> (q, valid): the undiscounted price of the out-of-the-money option that the quote implies by parity, and whether the quote is
    strictly inside the no-arbitrage bounds (F, K, D > 0, finite, 0 < time value, p / D < F for a call and < K for a put).  For an
    in-the-money quote q = p / D - |F - K| is formed from the exact remainder of the division and the exact error of F - K."""
    F, K, D, p = np.broadcast_arrays(*(np.asarray(a, float) for a in (forward, strike, discfactor, price)))
    is_call = np.broadcast_to(np.asarray(is_call, bool), F.shape)
    with np.errstate(all="ignore"):
        r = p / D
        rr = _fma(-r, D, p) / D                                  # p / D = r + rr (to a few units of eps^2 r)
        upper_room = _fma(D, np.where(is_call, F, K), -p)        # sign of D F - p (call) or D K - p (put), exactly
        itm = np.where(is_call, K < F, K > F)
        s, t = _two_sum(np.where(is_call, F, K), -np.where(is_call, K, F))    # |F - K| = s + t exactly on the in-the-money side
        q = np.where(itm, (r - s) + (rr - t), r)
        valid = ((F > 0) & (K > 0) & (D > 0) & np.isfinite(F) & np.isfinite(K) & np.isfinite(D) & np.isfinite(p)
                 & (q > 0) & (upper_room > 0))
    return q, valid


def infer_bsm_implied_vol(forward, ttm, strikes, given_prices, optiontypes, discfactor=1.0, lo=VOL_LO, hi=VOL_HI):
    """implied vols of one slice by bracketed bisection (80 halvings => ~1e-23 bracket) of the out-of-the-money price -- robust for
    deep OTM, independent of the kernel's Newton iteration."""
    strikes = np.asarray(strikes, float)
    is_call = np.isin(np.asarray(optiontypes), ("C", "IC"))
    q, ok = otm_quote(forward, strikes, discfactor, given_prices, is_call)
    ok &= np.asarray(ttm, float) > 0
    a = np.full(strikes.shape, lo)
    b = np.full(strikes.shape, hi)
    with np.errstate(invalid="ignore"):
        srt = np.sqrt(ttm)
    for _ in range(80):
        mid = 0.5 * (a + b)
        up = otm_black_price(forward, strikes, mid * srt) < q
        a = np.where(up, mid, a)
        b = np.where(up, b, mid)
    vol = 0.5 * (a + b)
    return np.where(ok, vol, np.nan)


def black_implied_vol_newton(forward, strike, ttm, discfactor, price, optiontype, max_iter=MAX_ITER):
    """numpy restatement of black.cuh::black_implied_vol, elementwise (broadcast) -> (vols, iterations).  Safeguarded Newton in total
    vol s = vol sqrt(T) on the out-of-the-money price, from the inflection point sqrt(2 |ln F/K|) (Brenner-Subrahmanyam at the money),
    inside the bracket [1e-8, 10] sqrt(T) kept up to date by the sign of every residual.  Where the model price is above twice the
    target the step is Newton's on ln(price) against ln(s); a step that leaves the bracket moves 4x towards an untried end, else to
    the geometric midpoint.  The rounding of d1, d2 is carried to first order.  Stops when the residual is within 4 ulp of the two
    terms (after one last Newton step), or the step or the bracket is within 2 ulp of s."""
    shape = np.broadcast_shapes(*(np.shape(a) for a in (forward, strike, ttm, discfactor, price, optiontype)))
    F, K, T, D, p, is_call = (np.broadcast_to(a, shape).ravel() for a in (
        *(np.asarray(a, float) for a in (forward, strike, ttm, discfactor, price)), np.isin(np.asarray(optiontype), ("C", "IC"))))
    q, ok = otm_quote(F, K, D, p, is_call)
    ok &= (T > 0) & np.isfinite(T)
    vol = np.full(F.size, np.nan)
    iters = np.zeros(F.size, dtype=np.int64)
    idx = np.flatnonzero(ok)
    F, K, T, q = F[idx], K[idx], T[idx], q[idx]
    srt = np.sqrt(T)
    x = np.log(F / K)
    a0, b0 = VOL_LO * srt, VOL_HI * srt
    a, b = a0.copy(), b0.copy()
    s = np.sqrt(2.0 * np.abs(x))
    s = np.where((s > a) & (s < b), s, np.minimum(np.maximum(_SQRT_2PI * q / F, 2.0 * a), 0.5 * b))
    live = np.ones(idx.size, bool)
    it_done = np.zeros(idx.size, dtype=np.int64)
    with np.errstate(all="ignore"):
        for it in range(max_iter):
            if not live.any():
                break
            it_done = np.where(live, it + 1, it_done)
            f, t1, t2, vega = _otm_terms(F, K, x, s)
            conv = live & (np.abs(f - q) <= 8.9e-16 * (t1 + t2)) & (vega > 0.0)
            s = np.where(conv, s - (f - q) / vega, s)
            live &= ~conv
            below = f < q
            a = np.where(live & below, s, a)
            b = np.where(live & ~below, s, b)
            sn = np.where(f > 2.0 * q, s * np.exp(-np.log(f / q) * f / (s * vega)), s - (f - q) / vega)
            sn = np.where((sn > a) & (sn < b), sn,
                          np.where((sn >= b) & (b == b0), np.minimum(4.0 * s, b),
                                   np.where((sn <= a) & (a == a0), np.maximum(0.25 * s, a), np.sqrt(a * b))))
            step = np.abs(sn - s)
            s = np.where(live, sn, s)
            live &= ~((step <= 4.5e-16 * s) | (b - a <= 4.5e-16 * b))
    vol[idx] = s / srt
    iters[idx] = it_done
    return vol.reshape(shape), iters.reshape(shape)


def infer_bsm_ivols_from_model_chain_prices(ttms, forwards, discfactors, strikes_ttms: Sequence[np.ndarray],
                                            optiontypes_ttms: Sequence[np.ndarray], model_prices_ttms: Sequence[np.ndarray]
                                            ) -> List[np.ndarray]:
    """same call shape as the third-party function used at data/option_chain.py:340-345."""
    out = []
    for ttm, forward, df, strikes, types, prices in zip(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, model_prices_ttms):
        out.append(infer_bsm_implied_vol(forward, ttm, strikes, prices, types, df))
    return out
