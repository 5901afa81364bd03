"""High-precision references for the Fourier edge suite (tests/test_fourier_edges_reference.py on the CPU, tests/test_gpu_fourier_edges.py
on the device), each with an error bar derived per point rather than one fixed rtol.

Heston closed form (pricers/heston_pricer.py:199-214, as oracle/mgf.py::heston_mgf_grid and HestonClosedForm in mgf_kernels.cu write it),
(a, b) carried over the maturity increments:
  - evaluated in mpmath at 50 digits from the exact fp64 inputs, as the ~20 named intermediates of the kernel's own operation order;
  - bar = C_CF * eps * sum_k |dy / dv_k| |v_k|: every intermediate v_k is rounded once, with a relative error of at most a few eps, and that
    error reaches the output y through the first-order sensitivity, measured by re-evaluating with v_k -> v_k (1 + 1e-30).  The formula is
    holomorphic in every intermediate, so one real nudge gives |dy / dv_k| |v_k| whatever the direction of the rounding error.
    C_CF = 6: the worst single operation is Smith's complex division, below 5 eps normwise (numerator and denominator each carry one
    fused product, plus the two quotients); a complex product is below sqrt(5) eps; exp, sincos, log, atan2, hypot and sqrt are within
    2 ulp on the device (CUDA's table) and 1 ulp in glibc, and enter through the operation they serve; one eps more covers the sum of the
    first-order terms of a chain of such operations.

Strike sums (fourier_vanilla_kernel, fourier_sum_kernel, fourier_gamma_batch_kernel; utils/mgf_pricer.py:174-384) on caller-supplied fp64
log-MGF and grid:
  - every summand t_j = Re(w_j exp(lm_j + c g_j)) evaluated from the fp64 inputs in mpmath (34 digits) and summed exactly (mp.fsum) when
    the case has at most MP_TERMS summands; larger cases (long grids, J = 70 000, the constructed entries) in np.clongdouble and summed in
    long double, where the summand bar below is ~1e3 times the long-double error;
  - numpy's non-finite semantics summand by summand: a term numpy evaluates to NaN is dropped (np.nansum), a +-inf term is kept, so the
    sum is then +-inf (or NaN when both signs occur);
  - bar = sum_j |t_j| eps (16 + E_j) + (2 + log2 P + ceil(P / 256)) eps sum_j |t_j| + the assembly's rounding, with
    E_j = |Re lm_j| + |Im lm_j| + (1 + 4 |c|)(|Re g_j| + |Im g_j|) the absolute error of the exponent: c = -ln(F / K) carries eps (1 + 2|c|)
    from F / K and the log (absolute, since c -> 0 at the money), the product c g_j one eps per component, the sum one eps of |lm_j + c g_j|.
    16 covers the weight (h / 3, the quadrature factor, 1 / pi, the division by the weight's denominator), exp and sincos, and the product
    with the weight; the second term is the fixed-order reduction: ceil(P / 256) strided adds per thread, then log2(256) tree levels.
"""
from __future__ import annotations

import functools
import math

import numpy as np

import mpmath as mp

EPS = float(np.finfo(np.float64).eps)
C_CF = 6.0
NUDGE = mp.mpf("1e-30")
DPS_CF = 50
DPS_SUM = 34
MP_TERMS = 2000
TYPE_CODE = {"C": 0, "P": 1, "IC": 2, "IP": 3}


# ----------------------------------------------------------------------------------------------------------------------------------------
# Heston closed form
# ----------------------------------------------------------------------------------------------------------------------------------------
def _mpc(z):
    z = complex(z)
    return mp.mpc(z.real, z.imag)


def _heston_chain_mp(par, ph, ps, taus, a0, b0, nudge=None, carry_b=True, swap_psi=False):
    """the closed form over the increments ``taus`` from (a0, b0) -> [(a, b, log_mgf)] per maturity, in the operation order of
    HestonClosedForm; ``nudge`` names the one intermediate multiplied by (1 + NUDGE).  Returns (outputs, names of the intermediates)."""
    names = []

    def r(name, v):
        names.append(name)
        return v * (1 + NUDGE) if name == nudge else v

    v0, th, ka, rho, vv = (x if isinstance(x, mp.mpf) else mp.mpf(float(x)) for x in par)     # mpf: mp.diff's shifted parameters
    ph, ps = _mpc(ph), _mpc(ps)
    vv2 = r("vv2", vv * vv)
    b1 = r("b1", ka + r("rvph", r("rv", rho * vv) * ph))
    b0_ = r("b0", r("hph", (ph / 2) * r("ph1", ph + 1)) - ps)
    zeta = r("zeta", mp.sqrt(r("disc", r("b1b1", b1 * b1) - r("b0v", (2 * b0_) * vv2))))
    psi_p, psi_m = r("psi_p", zeta - b1), r("psi_m", b1 + zeta)
    if swap_psi:
        psi_p, psi_m = psi_m, psi_p
    tkv = r("tkv", -(r("tk", th * ka) / vv2))
    a, b = _mpc(a0), _mpc(b0)
    out = []
    for m, tau in enumerate(taus):
        s = f"{m}:"
        tau = mp.mpf(float(tau))
        ez = r(s + "ez", mp.exp(-r(s + "tz", tau * zeta)))
        vb = r(s + "vb", vv2 * b)
        c_p = r(s + "c_p", r(s + "cpn", psi_p + vb) / (2 * zeta))
        c_m = r(s + "c_m", r(s + "cmn", psi_m - vb) / (2 * zeta))
        den = r(s + "den", r(s + "cpez", c_p * ez) + c_m)
        num = r(s + "num", r(s + "pmcpez", -r(s + "pmcp", psi_m * c_p) * ez) + r(s + "ppcm", psi_p * c_m))
        b_new = r(s + "b", -(num / r(s + "vden", vv2 * den)))
        targ = r(s + "targ", r(s + "tpp", tau * psi_p) + 2 * r(s + "logden", mp.log(den)))
        a_new = r(s + "a", r(s + "atk", tkv * targ) + a)
        a = a_new
        if carry_b:
            b = b_new
        out.append((a_new, b_new, r(s + "lm", a_new + r(s + "bv", b_new * v0))))
        if not carry_b:
            b = _mpc(b0)
    return out, names


def heston_cf_point(par, ph, ps, taus, a0=0j, b0=0j, **variant):
    """(exact [M, 3] complex: a, b, log_mgf per maturity; bar [M, 3]) at one transform point; NaN where the exact formula is singular"""
    M = len(taus)
    with mp.workdps(DPS_CF):
        try:
            base, names = _heston_chain_mp(par, ph, ps, taus, a0, b0, **variant)
        except (ZeroDivisionError, ValueError):
            return np.full((M, 3), np.nan + 0j), np.full((M, 3), np.nan)
        bar = [[mp.mpf(0)] * 3 for _ in range(M)]
        for name in dict.fromkeys(names):
            pert, _ = _heston_chain_mp(par, ph, ps, taus, a0, b0, nudge=name, **variant)
            for m in range(M):
                for k in range(3):
                    bar[m][k] += abs(pert[m][k] - base[m][k])
        exact = np.array([[complex(v) for v in row] for row in base])
        bars = np.array([[float(C_CF * EPS * v / NUDGE) for v in row] for row in bar])
    return exact, bars


# the parameter extremes: a base set and one axis at a time, plus a set that violates Feller's condition 2 kappa theta > volvol^2 badly
HESTON_BASE = (0.04, 0.04, 2.0, -0.7, 0.3)        # v0, theta, kappa, rho, volvol
HESTON_SETS = {
    "base": HESTON_BASE,
    "rho=-0.999": (0.04, 0.04, 2.0, -0.999, 0.3),
    "rho=0": (0.04, 0.04, 2.0, 0.0, 0.3),
    "rho=0.95": (0.04, 0.04, 2.0, 0.95, 0.3),
    "volvol=0.01": (0.04, 0.04, 2.0, -0.7, 0.01),
    "volvol=5": (0.04, 0.04, 2.0, -0.7, 5.0),
    "kappa=0.01": (0.04, 0.04, 0.01, -0.7, 0.3),
    "kappa=50": (0.04, 0.04, 50.0, -0.7, 0.3),
    "feller-violated": (0.5, 0.01, 0.01, -0.5, 5.0),
}
TAUS = (1e-4, 1.0, 30.0)
PHI_RE = (-0.5, 0.5, -0.2, 0.7)
PHI_IM = (0.0, 5e-324, 1e-8, 1.0, 10.0, 1e2, 1e3, 1e4)
CHAIN_SETS = ("base", "feller-violated")


def heston_phi_points():
    return np.array([re + 1j * im for re in PHI_RE for im in PHI_IM])


def heston_psi_points():
    """the Q_VAR transform: phi = 0 and psi = -1/2 + i y (get_psi_grid)"""
    return np.array([-0.5 + 1j * y for y in (0.0, 1e-8, 0.3, 4.0, 60.0, 4000.0)])


@functools.lru_cache(maxsize=None)
def heston_cases():
    """every closed-form case: dict of arrays over the points of one (parameter set, maturity increments, transform) each.
    Single maturities at every tau, a three-maturity chain (1e-4, 1, 30 carried) for CHAIN_SETS, and the psi != 0 transform."""
    cases = []
    phis, psis = heston_phi_points(), heston_psi_points()
    for name, par in HESTON_SETS.items():
        for taus in [(t,) for t in TAUS] + ([TAUS] if name in CHAIN_SETS else []):
            cases.append(dict(name=f"{name} taus={taus}", par=par, taus=taus, phi=phis, psi=np.zeros_like(phis)))
        cases.append(dict(name=f"{name} psi taus=(1.0,)", par=par, taus=(1.0,), phi=np.zeros_like(psis), psi=psis))
    for c in cases:
        res = [heston_cf_point(c["par"], ph, ps, c["taus"]) for ph, ps in zip(c["phi"], c["psi"])]
        c["exact"] = np.stack([r[0] for r in res], axis=1)         # [M, n, 3]
        c["bar"] = np.stack([r[1] for r in res], axis=1)
    return cases


def heston_numpy(par, taus, phi, psi, carry_b=True, swap_psi=False):
    """oracle/mgf.py::heston_mgf_grid chained over ``taus`` -> [M, n, 3] (a, b, log_mgf); the keyword arguments plant the defects the bars
    must reject"""
    from oracle import mgf
    v0, theta, kappa, rho, volvol = par
    a, b = np.zeros_like(phi), np.zeros_like(phi)
    out = []
    with np.errstate(all="ignore"):
        for tau in taus:
            if swap_psi:
                lm, a, b_new = _heston_swapped(v0, theta, kappa, volvol, rho, tau, phi, psi, a, b)
            else:
                lm, a, b_new = mgf.heston_mgf_grid(v0, theta, kappa, volvol, rho, tau, phi, psi, a, b)
            out.append(np.stack([a, b_new, lm], axis=-1))
            if carry_b:
                b = b_new
    return np.stack(out)


def _heston_swapped(v0, theta, kappa, volvol, rho, dtau, phi, psi, a_t0, b_t0):
    vv2 = volvol * volvol
    b1 = kappa + rho * volvol * phi
    zeta = np.sqrt(b1 * b1 - 2.0 * (0.5 * phi * (phi + 1.0) - psi) * vv2)
    ez = np.exp(-zeta * dtau)
    psi_m, psi_p = -b1 + zeta, b1 + zeta
    c_p, c_m = (psi_p + vv2 * b_t0) / (2.0 * zeta), (psi_m - vv2 * b_t0) / (2.0 * zeta)
    b_t1 = -(-psi_m * c_p * ez + psi_p * c_m) / (vv2 * (c_p * ez + c_m))
    a_t1 = -(theta * kappa / vv2) * (psi_p * dtau + 2.0 * np.log(c_p * ez + c_m)) + a_t0
    return a_t1 + b_t1 * v0, a_t1, b_t1


def bar_ratio(got, exact, bar):
    """|got - exact| / bar where the exact value is finite (0 where both agree exactly), and the points where got is not finite there"""
    fin = np.isfinite(exact) & np.isfinite(bar)
    with np.errstate(all="ignore"):
        r = np.where(fin, np.abs(got - exact) / np.where(bar > 0, bar, np.finfo(float).tiny), 0.0)
    r = np.where(fin & (got == exact), 0.0, r)
    return np.where(fin & ~np.isfinite(got), np.inf, r)


# ----------------------------------------------------------------------------------------------------------------------------------------
# strike sums
# ----------------------------------------------------------------------------------------------------------------------------------------
def legacy_weights(g):
    """the legacy Simpson factors 1, 4, 2, 4, ... with first and last 1 and THEN every odd index 4 (utils/mgf_pricer.py:163-170)"""
    w = np.full(g.shape[0], 2.0)
    w[0] = w[-1] = 1.0
    w[1::2] = 4.0
    return w


def _weights_mp(kind, g, wq, gamma, spot):
    """the exact weights w_j of one grid (mpmath), as the kernels and utils/mgf_pricer.py form them"""
    h3 = (mp.mpf(float(g[1].imag)) - mp.mpf(float(g[0].imag))) / 3
    out = []
    for gj, q in zip(g, wq):
        dp = h3 * mp.mpf(float(q)) / mp.pi
        z = _mpc(gj)
        if kind == "vanilla_half" or kind == "gamma_fast":
            w = dp / (z.imag * z.imag + mp.mpf(0.25))
        elif kind == "vanilla_general":
            w = -dp / ((z + 1) * z if spot else (z - 1) * z)
        elif kind == "gamma_general":
            zg = z + mp.mpf(float(gamma))
            w = -dp / ((zg + 1) * zg)
        elif kind == "qvar":
            w = dp / (z * z)
        elif kind == "pdf":
            w = dp
        elif kind == "digital":
            w = -dp / z if spot else dp / z
        else:
            raise ValueError(kind)
        out.append(w)
    return out


def _weights_np(kind, g, wq, gamma, spot, dtype):
    """the same weights in ``dtype`` (complex128 is numpy's evaluation, clongdouble the reference for long grids)"""
    rdt = np.float64 if dtype == np.complex128 else np.longdouble
    gi = g.imag.astype(rdt)
    z = g.astype(dtype)
    pi = rdt(np.pi) if rdt is np.float64 else np.arccos(rdt(-1))
    dp = ((gi[1] - gi[0]) / rdt(3)) * wq.astype(rdt) / pi
    if kind in ("vanilla_half", "gamma_fast"):
        return (dp / (gi * gi + rdt(0.25))).astype(dtype)
    if kind == "vanilla_general":
        return -dp / ((z + 1) * z if spot else (z - 1) * z)
    if kind == "gamma_general":
        zg = z + rdt(gamma)
        return -dp / ((zg + 1) * zg)
    if kind == "qvar":
        return dp / (z * z)
    if kind == "pdf":
        return dp.astype(dtype)
    if kind == "digital":
        return -dp / z if spot else dp / z
    raise ValueError(kind)


def numpy_terms(kind, lm, g, cs, gamma=0.0, spot=True, nansum_inf=False, wq=None):
    """numpy's summands Re(w_j exp(c g_j + lm_j)) [J, P] in fp64, as utils/mgf_pricer.py evaluates them"""
    wq = legacy_weights(g) if wq is None else wq
    w = _weights_np(kind, g, wq, gamma, spot, np.complex128)
    with np.errstate(all="ignore"):
        t = np.real(w[None, :] * np.exp(np.asarray(cs)[:, None] * g[None, :] + lm[None, :]))
    return t


def numpy_sums(kind, lm, g, cs, gamma=0.0, spot=True, nansum_inf=False, wq=None, scale=None):
    """np.nansum of numpy_terms; ``nansum_inf`` also drops +-inf terms and ``scale`` = (j, factor) scales one summand (planted defects)"""
    t = numpy_terms(kind, lm, g, cs, gamma, spot, wq=wq)
    if scale is not None:
        t[:, scale[0]] *= scale[1]
    if nansum_inf:
        t = np.where(np.isinf(t), np.nan, t)
    return np.nansum(t, axis=1)


def exact_sums(kind, lm, g, cs, gamma=0.0, spot=True, cs_mp=None):
    """(S [J]: the exact sum of the summands numpy keeps, +-inf / NaN where numpy's kept summands are not finite; sbar [J]: the summand
    and reduction bar; asum [J] = sum |t_j|).  ``cs_mp``: the exact coefficients (mpmath) where the fp64 ``cs`` are rounded ones."""
    P, J = g.shape[0], len(cs)
    wq = legacy_weights(g)
    t_np = numpy_terms(kind, lm, g, cs, gamma, spot)
    E = np.abs(lm.real) + np.abs(lm.imag)
    g1 = np.abs(g.real) + np.abs(g.imag)
    red = (2.0 + math.log2(P) + math.ceil(P / 256)) * EPS
    S, sbar, asum = np.empty(J), np.empty(J), np.empty(J)
    long_grid = P * J > MP_TERMS
    if long_grid:
        w = _weights_np(kind, g, wq, gamma, spot, np.clongdouble)
        lml, gl = lm.astype(np.clongdouble), g.astype(np.clongdouble)
    else:
        with mp.workdps(DPS_SUM):
            w = _weights_mp(kind, g, wq, gamma, spot)
            lmm, gm = [_mpc(v) for v in lm], [_mpc(v) for v in g]
    for k in range(J):
        c = float(cs[k])
        keep = ~np.isnan(t_np[k])
        inf = np.isinf(t_np[k]) & keep
        fin = keep & ~inf
        if long_grid:
            cl = np.longdouble(c) if cs_mp is None else np.longdouble(mp.nstr(cs_mp[k], 25))
            with np.errstate(all="ignore"):
                t = np.real(w * np.exp(cl * gl + lml))
            tf = t[fin]
            s = float(np.sum(tf, dtype=np.longdouble))
            at = np.abs(t.astype(np.float64))
        else:
            with mp.workdps(DPS_SUM):
                cm = mp.mpf(c) if cs_mp is None else cs_mp[k]
                tm = [None] * P
                for j in np.nonzero(fin)[0]:
                    tm[j] = mp.re(w[j] * mp.exp(cm * gm[j] + lmm[j]))
                s = float(mp.fsum(tm[j] for j in np.nonzero(fin)[0]))
                at = np.array([abs(float(v)) if v is not None else 0.0 for v in tm])
        at = np.where(fin, at, 0.0)
        if inf.any():
            pos, neg = np.any(t_np[k][inf] > 0), np.any(t_np[k][inf] < 0)
            s = np.nan if (pos and neg) else (np.inf if pos else -np.inf)
        S[k] = s
        asum[k] = at.sum()
        with np.errstate(invalid="ignore"):       # E_j is +-inf / NaN at the constructed entries, whose terms are 0 or not kept
            sbar[k] = EPS * np.sum(np.where(fin & (at > 0), at * (16.0 + E + (1.0 + 4.0 * abs(c)) * g1), 0.0)) + red * asum[k]
    return S, sbar, asum


def _log_ratio_mp(F, Ks):
    with mp.workdps(DPS_SUM):
        return [mp.log(mp.mpf(float(F)) / mp.mpf(float(k))) for k in Ks]


def vanilla_reference(lm, phi, F, Ks, types, df=1.0, spot=True, general=False):
    """exact prices [J] and bars [J] of fourier_vanilla (b200sv_fourier_vanilla) on one slice"""
    kind = "vanilla_general" if general else "vanilla_half"
    xs = _log_ratio_mp(F, Ks)
    with np.errstate(all="ignore"):
        S, sbar, asum = exact_sums(kind, lm, phi, -np.log(F / Ks), spot=spot, cs_mp=[-x for x in xs])
        price, bar = np.empty(len(Ks)), np.empty(len(Ks))
        for k, (K, ty) in enumerate(zip(Ks, types)):
            if spot:
                base = F if ty == "C" else K
                price[k] = df * (base - K * S[k])
                bar[k] = df * K * sbar[k] + 3 * EPS * (abs(F * df) + abs(K * S[k] * df))
            else:
                ex = math.exp(-float(xs[k]))
                base = 1.0 if ty in ("C", "IC") else ex
                price[k] = F * df * (base - S[k])
                bar[k] = F * df * sbar[k] + 3 * EPS * (abs(F * df) + abs(F * df * S[k])) + F * df * ex * EPS * (2 + 2 * abs(float(xs[k])))
    return price, bar


def gamma_reference(lm, phi, gamma, F, normalizer, gamma_forward, Ks, types, fast=False):
    """exact prices and bars of fourier_gamma: (gamma_forward | K) - n K^(1 + gamma) S, no discount factor"""
    xs = _log_ratio_mp(F, Ks)
    S, sbar, _ = exact_sums("gamma_fast" if fast else "gamma_general", lm, phi, -np.log(F / Ks), gamma=gamma, cs_mp=[-x for x in xs])
    price, bar = np.empty(len(Ks)), np.empty(len(Ks))
    with np.errstate(all="ignore"):
        for k, (K, ty) in enumerate(zip(Ks, types)):
            gk = K ** (1.0 + gamma)
            base = gamma_forward if ty == "C" else K
            price[k] = base - normalizer * gk * S[k]
            bar[k] = normalizer * gk * sbar[k] + 4 * EPS * (abs(base) + abs(normalizer * gk * S[k])) * (1 + abs(math.log(gk)))
    return price, bar


def qvar_reference(lm, psi, ttm, Ks, df=1.0):
    """exact prices and bars of fourier_qvar: max(df S / ttm, 1e-10) with coefficient K ttm"""
    with mp.workdps(DPS_SUM):
        cm = [mp.mpf(float(k)) * mp.mpf(float(ttm)) for k in Ks]
    S, sbar, _ = exact_sums("qvar", lm, psi, np.asarray(Ks) * ttm, cs_mp=cm)
    with np.errstate(all="ignore"):
        raw = df * S / ttm
        price = np.where(np.isnan(raw), np.nan, np.maximum(raw, 1e-10))
        bar = np.where(np.isfinite(raw), df * sbar / ttm + 3 * EPS * np.abs(raw), 0.0)     # -inf clamps to exactly 1e-10
    return price, bar


def pdf_reference(lm, grid, z):
    S, sbar, _ = exact_sums("pdf", lm, grid, np.asarray(z, dtype=float))
    return S, sbar


def digital_reference(lm, phi, F, Ks, types, df=1.0):
    """exact prices and bars of fourier_digital (calls and puts; all_calls when every Re phi < 0)"""
    all_calls = bool(np.all(phi.real < 0.0))
    xs = _log_ratio_mp(F, Ks)
    S, sbar, _ = exact_sums("digital", lm, phi, -np.log(F / Ks), spot=all_calls, cs_mp=[-x for x in xs])
    price = np.empty(len(Ks))
    with np.errstate(all="ignore"):
        for k, ty in enumerate(types):
            price[k] = df * (S[k] if (ty == "C") == all_calls else 1.0 - S[k])
    bar = df * sbar + 3 * EPS * df * (1.0 + np.abs(S))
    return price, bar


# ----------------------------------------------------------------------------------------------------------------------------------------
# sum cases: grids, log-MGFs and strikes
# ----------------------------------------------------------------------------------------------------------------------------------------
SUM_PS = (3, 4, 5, 255, 256, 257, 511, 512, 513, 1000, 1001, 40000, 2 ** 20 + 1)
XS = (0.0, 1e-12, -1e-12, 5.0, -5.0, 30.0, -30.0)         # x = ln(F / K): at the money, one rounding either side, deep either side
SUM_PAR = (0.04, 0.04, 2.0, -0.7, 0.3)
F0 = 1.0


def strikes_for(xs=XS, F=F0):
    return F * np.exp(-np.asarray(xs, dtype=float))


def grid(re, stop, P):
    """re + 1j linspace(0, stop, P), as build_phi / build_grid form it"""
    return re + 1j * np.linspace(0.0, stop, P)


def heston_lm(phi, psi=None, tau=0.25, par=SUM_PAR):
    from oracle import mgf
    v0, theta, kappa, rho, volvol = par
    psi = np.zeros_like(phi) if psi is None else psi
    with np.errstate(all="ignore"):
        return mgf.heston_mgf_grid(v0, theta, kappa, volvol, rho, tau, phi, psi)[0]


def constructed(lm, what, j):
    """log-MGF with one constructed entry at j: NaN, +inf, -inf or 700 + i Im(lm_j) (exp overflows once |x| Re phi adds 10)"""
    lm = lm.copy()
    lm[j] = {"nan": complex(np.nan, np.nan), "+inf": complex(np.inf, 0.0), "-inf": complex(-np.inf, 0.0),
             "700": complex(700.0, lm[j].imag)}[what]
    return lm


def vanilla_types(Ks, F=F0, spot=True):
    """out-of-the-money side of each strike: calls above the forward, puts below (deep-OTM quotes are small differences)"""
    if spot:
        return np.where(Ks >= F, "C", "P")
    return np.where(Ks >= F, "IC", "IP")


GAMMA = 0.3
STOP = 5.6 / 0.3


def _types_any(Ks, spot=True):
    return vanilla_types(Ks, spot=spot)


def _sum_case(kind, P, lm=None, g=None, xs=XS, tag=""):
    """one sum case: engine call arguments, the exact outputs and bars, numpy's outputs (oracle/mgf.py, oracle/hawkes.py)"""
    from oracle import hawkes, mgf
    Ks = strikes_for(xs)
    F, df = F0, 0.97
    c = dict(kind=kind, P=P, J=len(Ks), tag=tag)
    with np.errstate(all="ignore"):
        if kind in ("vanilla_spot", "vanilla_inv", "vanilla_general"):
            spot = kind != "vanilla_inv"
            g = grid({"vanilla_spot": -0.5, "vanilla_inv": 0.5, "vanilla_general": -0.7}[kind], STOP, P) if g is None else g
            lm = heston_lm(g) if lm is None else lm
            types = vanilla_types(Ks, spot=spot)
            c["exact"], c["bar"] = vanilla_reference(lm, g, F, Ks, types, df, spot, general=kind == "vanilla_general")
            c["numpy"] = mgf.vanilla_slice_prices(lm, g, F, Ks, types, df, spot)
            c["call"] = ("fourier_vanilla", (lm, g, F, Ks, types, df, spot))
        elif kind in ("gamma_general", "gamma_fast"):
            fast = kind == "gamma_fast"
            g = grid(0.5 + GAMMA if fast else -0.5 - GAMMA, STOP, P) if g is None else g
            lm = heston_lm(g) if lm is None else lm
            types = np.where(Ks >= F, "C", "P")
            norm, gfw = 0.93, 1.02
            c["exact"], c["bar"] = gamma_reference(lm, g, GAMMA, F, norm, gfw, Ks, types, fast)
            c["numpy"] = hawkes.gamma_slice_prices(lm, g, GAMMA, F, norm, gfw, Ks, types)
            c["call"] = ("fourier_gamma", (lm, g, GAMMA, F, norm, gfw, Ks, types))
        elif kind == "qvar":
            g = grid(-0.5, 4000.0 * (P - 1) / 39999.0 if P < 40000 else 4000.0, P) if g is None else g
            lm = heston_lm(np.zeros_like(g), g) if lm is None else lm
            Kq, ttm = 0.04 * np.exp(np.asarray(xs) / 10.0), 0.5
            c["exact"], c["bar"] = qvar_reference(lm, g, ttm, Kq, df)
            c["numpy"] = mgf.qvar_slice_prices(lm, g, ttm, Kq, ["C"] * len(Kq), df)
            c["call"] = ("fourier_qvar", (lm, g, ttm, Kq, ["C"] * len(Kq), df))
        elif kind == "pdf":
            g = grid(0.0, 600.0, P) if g is None else g
            lm = heston_lm(g) if lm is None else lm
            z = np.asarray(xs) / 10.0
            c["exact"], c["bar"] = pdf_reference(lm, g, z)
            c["numpy"] = np.array([np.nansum(np.real((legacy_weights(g) * ((g[1].imag - g[0].imag) / 3.0) / np.pi)
                                                    * np.exp(x * g + lm))) for x in z])
            c["call"] = ("fourier_pdf_sums", (lm, g, z))
        elif kind in ("digital_calls", "digital_puts"):
            g = grid(-0.5 if kind == "digital_calls" else 0.5, STOP, P) if g is None else g
            lm = heston_lm(g) if lm is None else lm
            types = np.where(Ks >= F, "C", "P")
            c["exact"], c["bar"] = digital_reference(lm, g, F, Ks, types, df)
            c["numpy"] = mgf.digital_slice_prices(lm, g, F, Ks, types, df)
            c["call"] = ("fourier_digital", (lm, g, F, Ks, types, df))
        else:
            raise ValueError(kind)
    c["lm"], c["g"] = lm, g
    return c


SUM_KINDS = ("vanilla_spot", "vanilla_inv", "vanilla_general", "gamma_general", "gamma_fast", "qvar", "pdf", "digital_calls", "digital_puts")
CONSTRUCTED = ("nan", "+inf", "-inf", "700")
CONSTRUCTED_P = 513


@functools.lru_cache(maxsize=None)
def sum_cases():
    """every kind at every P up to 1001, the vanilla and Q_VAR sums at 40 000 and 2^20 + 1 points; J = 1 and a J = 70 000 chain (a CTA
    count past 65 535) on the vanilla sum; and the constructed non-finite entries at j = 0, 255, 256 and P - 1 of a 513-point grid.

    Cost cuts, deliberate: the log-MGF of every case is the Heston one of SUM_PAR at tau = 1/4 (the sums are checked for whatever fp64
    log-MGF they are given; the closed form's own extremes are checked by heston_cases); only the vanilla and Q_VAR sums run the two long
    grids, and only the vanilla sum the 70 000-strike launch -- all five entry points share strike_sum / block_sum and the launch shape,
    and the long-double reference of a 2^20 + 1-point sum costs seconds per kind."""
    cases = []
    for P in SUM_PS:
        for kind in (SUM_KINDS if P <= 1001 else ("vanilla_spot", "qvar")):
            cases.append(_sum_case(kind, P))
    cases.append(_sum_case("vanilla_spot", 513, xs=(0.0,), tag="J=1"))
    cases.append(_sum_case("vanilla_spot", 257, xs=tuple(np.linspace(-30.0, 30.0, 70000)), tag="J=70000"))
    for kind in ("vanilla_spot", "vanilla_general", "qvar", "digital_calls", "gamma_general"):
        base = _sum_case(kind, CONSTRUCTED_P)
        for what in CONSTRUCTED:
            for j in (0, 255, 256, CONSTRUCTED_P - 1):
                cases.append(_sum_case(kind, CONSTRUCTED_P, lm=constructed(base["lm"], what, j), g=base["g"], tag=f"lm[{j}]={what}"))
    return cases


def case_name(c):
    return f"{c['kind']} P={c['P']} J={c['J']} {c['tag']}".strip()


def nonfinite_mismatch(got, want):
    """indices where got and want differ in being NaN, +inf or -inf (complex: either part)"""
    got, want = np.ravel(got), np.ravel(want)
    if np.iscomplexobj(got) or np.iscomplexobj(want):
        got, want = np.asarray(got, dtype=complex), np.asarray(want, dtype=complex)
        n = got.size
        return np.unique(nonfinite_mismatch(np.concatenate([got.real, got.imag]), np.concatenate([want.real, want.imag])) % n)

    def cls(v):
        return np.where(np.isnan(v), 3, np.where(np.isposinf(v), 1, np.where(np.isneginf(v), 2, 0)))
    return np.nonzero(cls(got) != cls(want))[0]


def heston_ratio(got, case):
    """bar_ratio of [M, n, 3] closed-form outputs.  Where phi and psi are both real the formula can sit on the log's branch cut: den is a
    negative real, and the sign of Im a (and of Im log-MGF) is the sign of a zero, which fp64 carries and mpmath does not -- there the
    conjugate of the exact value is an equally exact evaluation.  An imaginary part of one denormal ulp (5e-324) is real for fp64 too:
    the first product that touches it rounds it to a signed zero, so the exact side of the cut is out of reach of any fp64 evaluation."""
    r = bar_ratio(got, case["exact"], case["bar"])
    cut = (np.abs(case["phi"].imag) < 1e-300) & (np.abs(case["psi"].imag) < 1e-300)
    rc = bar_ratio(got, case["exact"].real - 1j * case["exact"].imag, case["bar"])
    return np.where(cut[None, :, None], np.minimum(r, rc), r)


# ----------------------------------------------------------------------------------------------------------------------------------------
# Heston sensitivities: d log-MGF / d(v0, theta, kappa, rho, volvol) and the 15 second derivatives on a chain pricer's own grid
# ----------------------------------------------------------------------------------------------------------------------------------------
# The tangent (HestonClosedForm<dcd, dcd>) and Hessian (<hcd, hcd>) kernels behind heston_price_chain_greeks / _hessian.  The reference is
# mp.diff of the 50-digit chained closed form (every maturity at once: the function returns one mp.matrix), at every point of the grid
# phi = -1/2 + i linspace(0, 5.6 / vol_scaler, max_phi).  Bar per point: DERIV_K max(|numpy forward mode - exact| over grid points
# j - 1 .. j + 1) + 32 eps |exact|: the fp64 forward mode through the same closed form (oracle/mgf_greeks.py::heston_chain_greeks, its
# hyper-dual twin tests/mgf_hessian_oracle.py::heston_d2_log_mgf) is a measured sample of how ill-conditioned the derivative is there, and
# the device evaluates the same operations in another order.  DERIV_K = 8, not 4: a sample is not a bound.  At volvol = 0.01 (1 / volvol^2
# = 1e4 amplifies every rounding of the second derivatives) numpy's error is a flat ~1e-12 over the grid, and one device value of 4680 sat
# at 4.02 times it, its neighbours below 0.4; every planted defect still lands 1e9 times and more outside.
DERIV_K = 8.0
PAIRS5 = [(p, q) for p in range(5) for q in range(p, 5)]          # the Hessian rows: upper triangle, row-major
DERIV_SETS = ("base", "rho=-0.999", "volvol=0.01", "volvol=5", "kappa=50", "feller-violated")
DERIV_TTMS = (0.25, 1.0)
DERIV_GRIDS = ((5.6 / 1e4, 13), (0.3, 13))                         # (vol_scaler, max_phi): Im phi up to 1e4, and up to 18.7; odd P


def deriv_grid(vol_scaler, max_phi):
    return -0.5 + 1j * np.linspace(0.0, 5.6 / vol_scaler, max_phi)


def heston_derivs_mp(par, ph, ttms):
    """(d1 [5, M], d2 [15, M]) of the log-MGF at one transform point, mp.diff at 50 digits"""
    taus = np.diff(np.concatenate([[0.0], ttms]))
    with mp.workdps(DPS_CF):
        x = [mp.mpf(float(v)) for v in par]

        def f(*xs):
            return mp.matrix([o[2] for o in _heston_chain_mp(xs, ph, 0j, taus, 0j, 0j)[0]])

        def d(orders):
            v = mp.diff(f, x, orders)
            return [complex(v[m]) for m in range(len(ttms))]

        d1 = [d(tuple(1 if k == p else 0 for k in range(5))) for p in range(5)]
        d2 = [d(tuple((k == p) + (k == q) for k in range(5))) for p, q in PAIRS5]
    return np.array(d1), np.array(d2)


def heston_dlog_mgf_numpy(par, ttms, phi, with_b_tangent=True):
    """the forward mode of oracle/mgf_greeks.py::heston_chain_greeks on any grid -> dlog_mgf [5, M, P] (v0 row = b).
    ``with_b_tangent=False`` drops the b' v0 term of the parameter rows (a planted defect)."""
    from oracle.mgf_greeks import _Dual
    v0 = par[0]
    M, P = len(ttms), phi.shape[0]
    dlm = np.empty((5, M, P), dtype=np.complex128)
    with np.errstate(all="ignore"):
        for d in range(4):
            theta, kappa, rho, volvol = (_Dual(par[1 + k], 1.0 if k == d else 0.0) for k in range(4))
            vv2 = volvol * volvol
            b1 = kappa + rho * volvol * phi
            zeta = (b1 * b1 - 2.0 * (0.5 * phi * (phi + 1.0)) * vv2).sqrt()
            psi_p, psi_m = -b1 + zeta, b1 + zeta
            a, b = _Dual(np.zeros(P)), _Dual(np.zeros(P))
            t0 = 0.0
            for m, ttm in enumerate(ttms):
                dtau = ttm - t0
                ez = (-zeta * dtau).exp()
                c_p, c_m = (psi_p + vv2 * b) / (2.0 * zeta), (psi_m - vv2 * b) / (2.0 * zeta)
                b = -(-psi_m * c_p * ez + psi_p * c_m) / (vv2 * (c_p * ez + c_m))
                a = -(theta * kappa / vv2) * (psi_p * dtau + 2.0 * (c_p * ez + c_m).log()) + a
                dlm[1 + d, m] = a.d + (b.d * v0 if with_b_tangent else 0.0)
                if d == 0:
                    dlm[0, m] = b.v
                t0 = ttm
    return dlm


def heston_d2log_mgf_numpy(par, ttms, phi, pairs=None):
    """the hyper-dual forward mode (tests/mgf_hessian_oracle.py) -> d2log_mgf [15, M, P] in the row order ``pairs`` (default PAIRS5)"""
    import mgf_hessian_oracle as H
    with np.errstate(all="ignore"):
        return np.array([H.heston_d2_log_mgf(par, list(ttms), phi, p, q) for p, q in (pairs or PAIRS5)])


def neighbour_max(e):
    """max over grid points j - 1 .. j + 1 along the last axis"""
    pad = np.concatenate([e[..., :1], e, e[..., -1:]], axis=-1)
    return np.maximum(np.maximum(pad[..., :-2], pad[..., 1:-1]), pad[..., 2:])


def deriv_bar(numpy_fm, exact):
    err = np.where(np.isfinite(numpy_fm), np.abs(numpy_fm - exact), np.inf)
    return DERIV_K * neighbour_max(err) + 32.0 * EPS * np.abs(exact)


@functools.lru_cache(maxsize=None)
def heston_deriv_cases():
    """per (parameter set, grid): the exact d1 [5, M, P] / d2 [15, M, P], the numpy forward modes and the bars"""
    cases = []
    for name in DERIV_SETS:
        par = HESTON_SETS[name]
        for vs, P in DERIV_GRIDS:
            phi = deriv_grid(vs, P)
            ex = [heston_derivs_mp(par, ph, DERIV_TTMS) for ph in phi]
            d1, d2 = np.stack([e[0] for e in ex], axis=-1), np.stack([e[1] for e in ex], axis=-1)
            n1, n2 = heston_dlog_mgf_numpy(par, DERIV_TTMS, phi), heston_d2log_mgf_numpy(par, DERIV_TTMS, phi)
            cases.append(dict(name=f"{name} vol_scaler={vs:.3g} max_phi={P}", par=par, vol_scaler=vs, max_phi=P, phi=phi, d1=d1, d2=d2,
                              numpy_d1=n1, numpy_d2=n2, bar1=deriv_bar(n1, d1), bar2=deriv_bar(n2, d2)))
    return cases
