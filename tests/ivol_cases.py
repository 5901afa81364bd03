"""Quotes and the exact reference shared by the Black-76 inversion tests (tests/test_bsm_oracle_edges.py on the CPU restatement,
tests/test_gpu_ivol_edges.py on the device).

Reference: the exact implied vol iv* of the fp64 quote AS GIVEN (not the vol that generated it), by a bracketed Newton in mpmath at
50 digits; whether the quote is inside the strict no-arbitrage bounds is decided exactly there too.
Bar: |iv - iv*| <= A eps (F N(+-d1) + K N(+-d2) + q) / vega_sigma + 4 ulp(iv*), the two terms those of the out-of-the-money side
at iv*, q its price and vega_sigma = F phi(d1) sqrt(T): the backward error of evaluating that side's formula in fp64.  Where the terms
are subnormal (a quote of a few times 2^-1074) their absolute precision 2^-1074 (F + K) joins eps (...) in the numerator.  A root
outside the bracket [1e-8, 10] must come back as the bracket's nearer end.
"""
from __future__ import annotations

import numpy as np

from oracle import bsm

EPS = 2.0 ** -52
TINY = 2.0 ** -1074           # N(-d) below 2^-1022 is subnormal: its absolute precision, times F or K, joins the bar
# A of the bar.  On the CPU the restatement of the kernel reaches 4.6 on the grid below and 2.4 on the edges, the bisection 8.4
# (tests/test_bsm_oracle_edges.py prints them); the device's normcdf is documented to 5 ulp where the restatement's N is to ~2, so the
# device gets the same A with that much room.
A_BAR = 32.0
TYPES = np.array(["C", "P", "IC", "IP"])
F_BTC = 67106.44


def _mp():
    import mpmath
    return mpmath.mp


def quote(F, K, T, vol, optiontype, D):
    """fp64 quote of a Black-76 option: the out-of-the-money price from its own formula (so it keeps its relative precision however
    deep), the in-the-money one by parity from it -- the way a careful pricer rounds both."""
    F, K, T, vol, D = (np.asarray(a, float) for a in (F, K, T, vol, D))
    q = bsm.otm_black_price(F, K, vol * np.sqrt(T))
    is_call = np.isin(np.asarray(optiontype), ("C", "IC"))
    itm = np.where(is_call, K < F, K > F)
    return D * np.where(itm, q + np.abs(F - K), q)


def exact(F, K, T, D, price, optiontype, guess=None, dps=50):
    """-> (iv*, bar_without_A) of one quote, or (nan, nan) if the quote is outside the strict no-arbitrage bounds.
    ``guess``: a total-vol start for Newton (a vol near the root, e.g. the one that generated the quote); the answer does not depend
    on it.  bar_without_A = eps (F N(+-d1) + K N(+-d2) + q) / vega_sigma; the caller adds A x it + 4 ulp(iv*)."""
    mp = _mp()
    vals = [float(F), float(K), float(T), float(D), float(price)]
    if not all(np.isfinite(vals)) or min(vals[:4]) <= 0.0:
        return np.nan, np.nan
    is_call = str(optiontype) in ("C", "IC")
    with mp.workdps(dps):
        F, K, T, D, P = (mp.mpf(v) for v in vals)
        intrinsic = max(F - K, 0) if is_call else max(K - F, 0)
        upper = F if is_call else K
        if not (P > D * intrinsic and P < D * upper):            # products of doubles are exact at this precision
            return np.nan, np.nan
        # out-of-the-money twin by parity: time value of the quote
        q = P / D - intrinsic
        put_side = K < F
        x = mp.log(F / K)

        def otm(s):
            d1 = x / s + s / 2
            d2 = d1 - s
            if x == 0:                                  # at the money: F (2 N(s/2) - 1) without the cancellation (s may be 1e-300)
                return F * mp.erf(s / (2 * mp.sqrt(2))), F * mp.npdf(d1), F * mp.ncdf(d1) + K * mp.ncdf(d2)
            if put_side:
                return K * mp.ncdf(-d2) - F * mp.ncdf(-d1), F * mp.npdf(d1), F * mp.ncdf(-d1) + K * mp.ncdf(-d2)
            return F * mp.ncdf(d1) - K * mp.ncdf(d2), F * mp.npdf(d1), F * mp.ncdf(d1) + K * mp.ncdf(d2)

        lo, hi = mp.mpf(0), mp.inf
        s = mp.mpf(guess) if guess is not None and guess > 0 else (mp.sqrt(2 * abs(x)) if x != 0 else mp.sqrt(2 * mp.pi) * q / F)
        tol = mp.mpf(10) ** (-(dps - 8))
        for _ in range(400):
            f, vega, _t = otm(s)
            if f < q:
                lo = s
            else:
                hi = s
            # Newton on ln(price) (the tails are exponential in s), safeguarded by the bracket; geometric bisection otherwise
            sn = s - mp.log(f / q) * f / vega if f > 0 and vega > 0 else mp.nan
            if not (lo < sn < hi):
                sn = mp.sqrt(lo * hi) if lo > 0 and hi < mp.inf else (s / 4 if lo == 0 else s * 4)
            step = abs(sn - s)
            s = sn
            if step <= tol * s:
                break
        else:
            raise RuntimeError("mpmath reference did not converge")
        f, vega, terms = otm(s)
        iv = s / mp.sqrt(T)
        bar = (EPS * (terms + q) + TINY * (F + K)) / (vega * mp.sqrt(T))
        return float(iv), float(bar)


def allowed(iv_star, bar, A=A_BAR):
    """the bar at each quote, and the value expected there: iv* inside the bracket, else its nearer end"""
    iv_star, bar = np.asarray(iv_star, float), np.asarray(bar, float)
    want = np.clip(iv_star, bsm.VOL_LO, bsm.VOL_HI)
    tol = np.where((iv_star >= bsm.VOL_LO) & (iv_star <= bsm.VOL_HI), A * bar + 4.0 * np.spacing(np.abs(iv_star)),
                   4.0 * np.spacing(want))
    return want, tol


def random_grid(n=3200, seed=11):
    """n quotes: z = ln(F/K)/(vol sqrt T) in [-9, 9], vol in [0.01, 5] and T in [3e-4, 10] (log-uniform), all four codes, D in
    [0.5, 1], F = 1 and the BTC chain's scale.  -> dict of arrays F, K, T, D, type, vol (the generating vol), price."""
    rs = np.random.RandomState(seed)
    F = np.where(rs.rand(n) < 0.5, 1.0, F_BTC)
    z = rs.uniform(-9.0, 9.0, n)
    vol = np.exp(rs.uniform(np.log(0.01), np.log(5.0), n))
    T = np.exp(rs.uniform(np.log(3e-4), np.log(10.0), n))
    K = F * np.exp(-z * vol * np.sqrt(T))
    D = rs.uniform(0.5, 1.0, n)
    ty = TYPES[rs.randint(0, 4, n)]
    return dict(F=F, K=K, T=T, D=D, type=ty, vol=vol, price=quote(F, K, T, vol, ty, D))


def edge_cases():
    """constructed quotes -> dict of arrays F, K, T, D, type, price, guess (total vol or nan), tag"""
    rows = []

    def add(tag, F, K, T, D, ty, price, vol=np.nan):
        rows.append((tag, float(F), float(K), float(T), float(D), ty, float(price), float(vol) * np.sqrt(T) if np.isfinite(vol) else np.nan))

    for F in (1.0, F_BTC):
        for ty in TYPES:
            # K = F exactly, a range of vols and maturities
            for vol, T in ((0.2, 0.25), (1.0, 1.0), (0.01, 3e-4), (3.0, 10.0)):
                add("atm", F, F, T, 0.97, ty, quote(F, F, T, vol, ty, 0.97), vol)
            # T = 1e-6 and T = 30
            for T, z in ((1e-6, 0.5), (1e-6, -3.0), (30.0, 2.0), (30.0, -6.0)):
                K = F * np.exp(-z * 0.4 * np.sqrt(T))
                add("ttm", F, K, T, 0.9, ty, quote(F, K, T, 0.4, ty, 0.9), 0.4)
            # vols just inside and just outside the bracket [1e-8, 10], at the money and off it
            for vol in (1.0001e-8, 0.9999e-8, 9.99, 10.01, 20.0):
                for K in (F, 1.05 * F, 0.95 * F):
                    if vol < 1e-6 and K != F:
                        continue
                    add("bracket", F, K, 1.0, 1.0, ty, quote(F, K, 1.0, vol, ty, 1.0), vol)
        # out-of-the-money quotes down to 1e-300 (x F): a put below the forward and a call above, given directly as the price
        for p in (1e-12, 1e-17, 1e-30, 1e-100, 1e-200, 1e-300):
            for T in (0.02, 1.0):
                add("tiny", F, 0.6 * F, T, 1.0, "P", p * F)
                add("tiny", F, 1.6 * F, T, 1.0, "C", p * F)
                add("tiny", F, 0.6 * F, T, 0.8, "IP", p * F)
                add("tiny", F, 1.6 * F, T, 0.8, "IC", p * F)
        # intrinsic + 1 ulp and the upper bound - 1 ulp (valid), and both bounds themselves (NaN)
        for K in (0.9 * F, F, 1.1 * F):
            for D in (1.0, 0.93):
                for ty in TYPES:
                    is_call = ty in ("C", "IC")
                    intr = D * max(F - K, 0.0) if is_call else D * max(K - F, 0.0)
                    up = D * (F if is_call else K)
                    add("lower+1ulp", F, K, 0.5, D, ty, np.nextafter(intr, np.inf))
                    add("upper-1ulp", F, K, 0.5, D, ty, np.nextafter(up, 0.0))
                    add("at-lower", F, K, 0.5, D, ty, intr)
                    add("at-upper", F, K, 0.5, D, ty, up)
    # invalid inputs: NaN whatever the price
    for F, K, T, D, p in ((0.0, 1.0, 1.0, 1.0, 0.1), (-1.0, 1.0, 1.0, 1.0, 0.1), (1.0, 0.0, 1.0, 1.0, 0.1), (1.0, -1.0, 1.0, 1.0, 0.1),
                          (1.0, 1.0, 0.0, 1.0, 0.1), (1.0, 1.0, -1.0, 1.0, 0.1), (1.0, 1.0, 1.0, 0.0, 0.1), (1.0, 1.0, 1.0, -0.5, 0.1),
                          (1.0, 1.0, 1.0, 1.0, np.nan), (1.0, 1.0, 1.0, 1.0, np.inf), (1.0, 1.0, 1.0, 1.0, -np.inf), (1.0, 1.0, 1.0, 1.0, 0.0),
                          (1.0, 1.0, 1.0, 1.0, -1e-3), (np.inf, 1.0, 1.0, 1.0, 0.1), (1.0, 1.0, np.nan, 1.0, 0.1)):
        for ty in TYPES:
            rows.append(("invalid", F, K, T, D, ty, p, np.nan))
    tag, F, K, T, D, ty, price, guess = zip(*rows)
    return dict(tag=np.array(tag), F=np.array(F), K=np.array(K), T=np.array(T), D=np.array(D), type=np.array(ty), price=np.array(price),
                guess=np.array(guess))


def parity_pairs():
    """(put, call) quotes at the same (K, vol) with exact parity c = p + (F - K) in fp64 (F - K is a power of two, p is rounded onto the
    grid of c), so both have the same iv*: the in-the-money call must come back with the put's vol.  And the mirror pair above F.
    -> dict of arrays F, K, T, D(=1), put_price, call_price, vol"""
    rows = []
    for K, vol, T in ((0.75, 0.2, 0.5), (0.75, 0.6, 0.25), (0.5, 0.9, 2.0), (0.5, 1.5, 1.0), (0.875, 0.05, 1.0), (1.25, 0.3, 1.0),
                      (1.5, 0.8, 0.5), (2.0, 1.2, 3.0)):
        F = 1.0
        otm = float(bsm.otm_black_price(F, K, vol * np.sqrt(T)))
        if K < F:
            call = (F - K) + otm
            put = call - (F - K)
        else:
            put = (K - F) + otm
            call = put - (K - F)
        rows.append((F, K, T, 1.0, put, call, vol))
    F, K, T, D, p, c, v = (np.array(a) for a in zip(*rows))
    return dict(F=F, K=K, T=T, D=D, put=p, call=c, vol=v)


def reference(cases, guess_key="vol"):
    """iv*, bar (without A) of each quote of a case dict"""
    g = cases.get(guess_key)
    out = [exact(cases["F"][i], cases["K"][i], cases["T"][i], cases["D"][i], cases["price"][i], cases["type"][i],
                 None if g is None or not np.isfinite(g[i]) else (g[i] * np.sqrt(cases["T"][i]) if guess_key == "vol" else g[i]))
           for i in range(cases["F"].size)]
    iv, bar = (np.array(a) for a in zip(*out))
    return iv, bar


def check(iv, iv_star, bar, A=A_BAR):
    """-> (ratio, nan_mismatch, bad): max |iv - iv*| / bar over the quotes inside the bracket, the quotes whose NaN-ness differs from
    the exact verdict, and the indices over the bar"""
    iv = np.asarray(iv, float)
    valid = np.isfinite(iv_star)
    nan_mismatch = np.flatnonzero(np.isfinite(iv) != valid)
    want, tol = allowed(iv_star[valid], bar[valid], A)
    err = np.abs(iv[valid] - want)
    inside = (iv_star[valid] >= bsm.VOL_LO) & (iv_star[valid] <= bsm.VOL_HI)
    denom = bar[valid] + 4.0 * np.spacing(np.abs(iv_star[valid])) / A
    ratio = float(np.max(np.where(inside, err / denom, 0.0), initial=0.0))
    bad = np.flatnonzero(valid)[~(err <= tol)]
    return ratio, nan_mismatch, bad

