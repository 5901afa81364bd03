"""oracle.mc -- numpy restatement of the Monte Carlo hot path.  TEST INFRASTRUCTURE ONLY
(see ``oracle/__init__.py``); pinned against ``tests/golden/logsv_mc_fixed_*.npz``,
``heston_mc_fixed_*.npz``, ``payoffs.npz``, ``time_grid.npz``.

``file:line`` citations are relative to ``/root/reference/src/stochvolmodels``.

The last section restates the DEVICE random-number stream (Philox4x32-10 + Box-Muller, defined by
this repo in ``stochvolmodels_b200/csrc/philox.cuh``; the reference pins no stream, SURVEY.md §8c) so
that the fused CUDA kernel can be checked path by path, not only statistically.
"""
from __future__ import annotations

import numpy as np

LOG_RETURN, Q_VAR, SIGMA = 1, 2, 3           # utils/config.py:17-24  VariableType values


# --------------------------------------------------------------------------------------------
# time grid
# --------------------------------------------------------------------------------------------
def set_time_grid(ttm: float, nb_steps_per_year: int = 360):
    """``set_time_grid`` (utils/funcs.py:24-47): S = int(ttm*n)+1; dt = linspace(0, ttm, S+1)[1]-[0]."""
    nb_steps = int(ttm * nb_steps_per_year) + 1
    grid = np.linspace(0.0, ttm, nb_steps + 1)
    return nb_steps, float(grid[1] - grid[0])


# --------------------------------------------------------------------------------------------
# steppers with caller-supplied unit normals Z0, Z1 of shape (S, N)
# --------------------------------------------------------------------------------------------
# the fp64 kernels' log-vol guard (fastmath64.cuh, state in table units Ls = L 256/ln2): a value trips it when the high word of |Ls| exceeds
# that of 258530, i.e. |Ls| >= 258530.125, and is then set to +-258530 (699.997 in log units)
LOG_VOL_CLAMP = 258530.0 * np.log(2.0) / 256.0
LOG_VOL_TRIP = 258530.125 * np.log(2.0) / 256.0


def _clamp_log_vol(L):
    return np.where(np.abs(L) < LOG_VOL_TRIP, L, np.copysign(LOG_VOL_CLAMP, L))


def logsv_step_fixed(x, sigma, qvar, Z0, Z1, dt, theta, kappa1, kappa2, beta, volvol, eta=1.0, is_spot_measure=True, clamp=False):
    """``simulate_logsv_x_vol_terminal`` with W0/W1/dt supplied (pricers/logsv_pricer.py:1027-1047).

    Evaluation order follows the reference expression by expression (it is ``fastmath=False``).
    clamp=True restates the fp64 kernels' guarded re-run of a path whose log-vol leaves the representable range: the initial and
    every updated log-vol that trips the guard are set to +-LOG_VOL_CLAMP.  The reference has no clamp; the default keeps its recursion."""
    x = np.array(x, dtype=np.float64, copy=True)
    sigma = np.array(sigma, dtype=np.float64, copy=True)
    qvar = np.array(qvar, dtype=np.float64, copy=True)
    sdt = np.sqrt(dt)
    if is_spot_measure:
        alpha, adj = -1.0, 0.0
    else:
        alpha, adj = 1.0, beta * eta
    vartheta2 = beta * beta + volvol * volvol
    eta2 = eta * eta
    L = np.log(sigma)
    if clamp:
        L = _clamp_log_vol(L)
    for z0, z1 in zip(Z0, Z1):
        w0 = sdt * z0
        w1 = sdt * z1
        s2dt = eta2 * sigma * sigma * dt
        x = x + alpha * 0.5 * s2dt + eta * sigma * w0
        L = L + ((kappa1 * theta / sigma - kappa1) + kappa2 * (theta - sigma) + adj * sigma - 0.5 * vartheta2) * dt + beta * w0 + volvol * w1
        if clamp:
            L = _clamp_log_vol(L)
        sigma = np.exp(L)
        qvar = qvar + 0.5 * (s2dt + eta2 * sigma * sigma * dt)
    return x, sigma, qvar


def heston_step_fixed(x, var, qvar, Z0, Z1, dt, theta, kappa, rho, volvol):
    """``simulate_heston_x_vol_terminal`` loop (pricers/heston_pricer.py:368-381) with the normals supplied."""
    x = np.array(x, dtype=np.float64, copy=True)
    var = np.array(var, dtype=np.float64, copy=True)
    qvar = np.array(qvar, dtype=np.float64, copy=True)
    sdt = np.sqrt(dt)
    rho_1 = np.sqrt(1.0 - rho * rho)
    for z0, z1 in zip(Z0, Z1):
        w0 = sdt * z0
        w1 = sdt * z1
        sig = np.sqrt(var)
        vdt = var * dt
        x = x - 0.5 * vdt + sig * w0
        qvar = qvar + vdt
        var = var + kappa * (theta - var) * dt + sig * volvol * (rho * w0 + rho_1 * w1)
        var = np.maximum(var, 1e-4)
    return x, var, qvar


# --------------------------------------------------------------------------------------------
# payoffs
# --------------------------------------------------------------------------------------------
def mc_payoffs(x, qvar, ttm, forward, strikes, types, discfactor=1.0, variable_type=LOG_RETURN):
    """``compute_mc_vars_payoff`` (utils/mc_payoffs.py:10-88).

    Spots re-centred on the forward with the nan-mean over ALL paths; nanmean / population nanstd per
    strike; standard error divides by sqrt(len(x)) including NaN paths."""
    spots = forward * np.exp(x)
    spots = spots - (np.nanmean(spots) - forward)
    if variable_type == LOG_RETURN:
        under = spots
    elif variable_type == Q_VAR:
        under = qvar / ttm
    else:
        raise NotImplementedError
    prices = np.zeros(len(strikes))
    stds = np.zeros(len(strikes))
    for j, (k, ty) in enumerate(zip(strikes, types)):
        ty = str(ty)
        if ty == "C":
            pay = np.where(under > k, under - k, 0.0)
        elif ty == "IC":
            pay = np.where(under > k, under - k, 0.0) / spots
        elif ty == "P":
            pay = np.where(under < k, k - under, 0.0)
        elif ty == "IP":
            pay = np.where(under < k, k - under, 0.0) / spots
        else:
            raise ValueError("unknown option payoff code")
        prices[j] = discfactor * np.nanmean(pay)
        stds[j] = discfactor * np.nanstd(pay)
    return prices, stds / np.sqrt(len(x))


# --------------------------------------------------------------------------------------------
# chain loops
# --------------------------------------------------------------------------------------------
def logsv_mc_chain_fixed(params6, ttms, forwards, discfactors, strikes_ttms, types_ttms, etas, Z0s, Z1s, dts,
                         is_spot_measure=True, variable_type=LOG_RETURN, return_states=False):
    """``logsv_mc_chain_pricer_fixed_randoms`` (pricers/logsv_pricer.py:1100-1162): the terminal state of slice m
    seeds slice m+1; unit normals are scaled by sqrt(dt) inside the stepper."""
    sigma0, theta, kappa1, kappa2, beta, volvol = params6
    n = Z0s[0].shape[1]
    x, q, s = np.zeros(n), np.zeros(n), sigma0 * np.ones(n)
    prices, stds, states = [], [], []
    for m, ttm in enumerate(ttms):
        x, s, q = logsv_step_fixed(x, s, q, Z0s[m], Z1s[m], dts[m], theta, kappa1, kappa2, beta, volvol, etas[m], is_spot_measure)
        p, e = mc_payoffs(x, q, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
        prices.append(p)
        stds.append(e)
        states.append((x.copy(), s.copy(), q.copy()))
    return (prices, stds, states) if return_states else (prices, stds)


def heston_mc_chain_fixed(params5, ttms, forwards, discfactors, strikes_ttms, types_ttms, Z0s, Z1s, dts,
                          variable_type=LOG_RETURN, return_states=False):
    """``heston_mc_chain_pricer`` (pricers/heston_pricer.py:285-331) with the normals supplied; params5 = (v0, theta, kappa, rho, volvol)."""
    v0, theta, kappa, rho, volvol = params5
    n = Z0s[0].shape[1]
    x, q, v = np.zeros(n), np.zeros(n), v0 * np.ones(n)
    prices, stds, states = [], [], []
    for m, ttm in enumerate(ttms):
        x, v, q = heston_step_fixed(x, v, q, Z0s[m], Z1s[m], dts[m], theta, kappa, rho, volvol)
        p, e = mc_payoffs(x, q, ttm, forwards[m], strikes_ttms[m], types_ttms[m], discfactors[m], variable_type)
        prices.append(p)
        stds.append(e)
        states.append((x.copy(), v.copy(), q.copy()))
    return (prices, stds, states) if return_states else (prices, stds)


def chain_steps(ttms, nb_steps_per_year):
    """(S_m, dt_m) per slice from maturity differences, as in the chain loops (logsv_pricer.py:840-856, :1064-1073)."""
    out, t0 = [], 0.0
    for ttm in ttms:
        out.append(set_time_grid(ttm - t0, nb_steps_per_year))
        t0 = ttm
    return out


# --------------------------------------------------------------------------------------------
# device RNG restatement: Philox4x32-10 (Salmon et al., SC'11) + Box-Muller
# --------------------------------------------------------------------------------------------
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32 with 10 rounds on arrays of uint32 counters; returns 4 uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _MASK for c in np.broadcast_arrays(c0, c1, c2, c3))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for r in range(10):
        p0 = _M0 * c0
        p1 = _M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0 = (k0 + _W0) & 0xFFFFFFFF
        k1 = (k1 + _W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def _u52(hi, lo):
    """double in [1, 2) whose 52 mantissa bits are (hi >> 12) : lo  -- same bit trick as the device."""
    bits = (np.uint64(0x3FF) << np.uint64(52)) | ((hi.astype(np.uint64) >> np.uint64(12)) << np.uint64(32)) | lo.astype(np.uint64)
    return bits.view(np.float64)


def device_normals(seed: int, path_ids, slice_idx: int, nb_steps: int, gauss: str = "f64"):
    """Unit normals (Z0, Z1), shape (nb_steps, len(path_ids)), that the fused kernels draw for the given
    global path ids in chain slice ``slice_idx``.

    Counter layout (``philox.cuh``): key = (seed_lo, seed_hi); counter = (path_lo, path_hi, call, slice).

    gauss="f64": one call per step s (call = s); u1 = 2 - d(r0,r1|1) in (0,1) (the lowest mantissa bit is forced to 1 so that
                 u1 < 1 and R > 0, gauss64.cuh), u2 = d(r2,r3) - 1 in [0,1);
                 Z0 = R cos(2 pi u2), Z1 = R sin(2 pi u2), R = sqrt(-2 ln u1).
    gauss="f64_paired": the f32 stream's words and layout evaluated in float64: u1 = (ra + 1/2) 2^-32, angle = 2 pi rb 2^-32
                 (the device's check mode B200SV_GAUSS_F64_PAIRED).
    gauss="f32": one call per TWO steps (call = s // 2); even step uses (r0, r1), odd step (r2, r3);
                 u1 = fma(float(ra), 2^-32, 2^-33), angle = float(int32(rb)) * pi * 2^-31, float32 Box-Muller:
                 Z0 = R cos(angle), Z1 = R sin(angle).  The device uses MUFU approximations (lg2/sin/cos), so this variant
                 agrees with the device only to ~1e-6 absolute; bit-level checks of that mode use the normals
                 exported by ``b200sv_device_normals`` instead.
    """
    path_ids = np.asarray(path_ids, dtype=np.uint64)
    plo = (path_ids & _MASK)
    phi = (path_ids >> np.uint64(32))
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    Z0 = np.empty((nb_steps, path_ids.shape[0]))
    Z1 = np.empty((nb_steps, path_ids.shape[0]))
    if gauss == "f64":
        for s in range(nb_steps):
            r0, r1, r2, r3 = philox4x32_10(plo, phi, np.uint64(s), np.uint64(slice_idx), k0, k1)
            u1 = 2.0 - _u52(r0, r1 | np.uint64(1))
            u2 = _u52(r2, r3) - 1.0
            rad = np.sqrt(-2.0 * np.log(u1))
            Z0[s] = rad * np.cos(2.0 * np.pi * u2)
            Z1[s] = rad * np.sin(2.0 * np.pi * u2)
    elif gauss == "f32":
        f32 = np.float32
        for c in range((nb_steps + 1) // 2):
            r = philox4x32_10(plo, phi, np.uint64(c), np.uint64(slice_idx), k0, k1)
            for half in range(2):
                s = 2 * c + half
                if s >= nb_steps:
                    break
                ra, rb = r[2 * half], r[2 * half + 1]
                u1 = ra.astype(f32) * f32(2.0 ** -32) + f32(2.0 ** -33)
                rad = np.sqrt(f32(-2.0) * np.log(u1))
                ang = rb.view(np.int32).astype(f32) * f32(np.pi * 2.0 ** -31)      # [-pi, pi]
                Z0[s] = (rad * np.cos(ang)).astype(np.float64)
                Z1[s] = (rad * np.sin(ang)).astype(np.float64)
    elif gauss == "f64_paired":
        for c in range((nb_steps + 1) // 2):
            r = philox4x32_10(plo, phi, np.uint64(c), np.uint64(slice_idx), k0, k1)
            for half in range(2):
                s = 2 * c + half
                if s >= nb_steps:
                    break
                ra, rb = r[2 * half].astype(np.float64), r[2 * half + 1].astype(np.float64)
                rad = np.sqrt(-2.0 * np.log((ra + 0.5) * 2.0 ** -32))
                ang = 2.0 * np.pi * (rb * 2.0 ** -32)
                Z0[s] = rad * np.cos(ang)
                Z1[s] = rad * np.sin(ang)
    else:
        raise ValueError(gauss)
    return Z0, Z1


def logsv_vol_paths(v0, theta, kappa1, kappa2, beta, volvol, W, dt, is_spot_measure=True):
    """``simulate_vol_paths`` (pricers/logsv_pricer.py:925-947) with the scaled increments W[S, N] supplied:
    sigma_t[(S+1), N], row 0 = v0; single normal per step with loading vartheta; adj = beta (no eta) under the inverse measure."""
    n = W.shape[1]
    sigma = v0 * np.ones(n)
    adj = 0.0 if is_spot_measure else beta
    vartheta2 = beta * beta + volvol * volvol
    vartheta = np.sqrt(vartheta2)
    L = np.log(sigma)
    out = np.zeros((W.shape[0] + 1, n))
    out[0] = sigma
    for t, w1 in enumerate(W):
        L = L + ((kappa1 * theta / sigma - kappa1) + kappa2 * (theta - sigma) + adj * sigma - 0.5 * vartheta2) * dt + vartheta * w1
        sigma = np.exp(L)
        out[t + 1] = sigma
    return out


def heston_qe_step_fixed(x, var, qvar, Z0, Z1, dt, theta, kappa, rho, volvol, psi_c=1.5):
    """Andersen (2008) quadratic-exponential Heston step with central discretisation (gamma1 = gamma2 = 1/2), the opt-in
    ``scheme="qe"`` of this repo (NOT in the reference; restated here as the checker of ``HestonPath::step_qe``).
    Z0 drives the spot, Z1 the variance (U = Phi(Z1) in the exponential branch); qvar by the trapezoid rule."""
    from scipy.special import ndtr
    x = np.array(x, dtype=np.float64, copy=True)
    v = np.array(var, dtype=np.float64, copy=True)
    q = np.array(qvar, dtype=np.float64, copy=True)
    e = np.exp(-kappa * dt)
    m0 = theta * (1.0 - e)
    s1 = volvol * volvol * e * (1.0 - e) / kappa
    s0 = theta * volvol * volvol * (1.0 - e) * (1.0 - e) / (2.0 * kappa)
    kre = kappa * rho / volvol
    K0 = -rho * kappa * theta * dt / volvol
    K1 = 0.5 * dt * (kre - 0.5) - rho / volvol
    K2 = 0.5 * dt * (kre - 0.5) + rho / volvol
    K3 = 0.5 * dt * (1.0 - rho * rho)
    K4 = K3
    for zx, zv in zip(Z0, Z1):
        m = v * e + m0
        s2 = v * s1 + s0
        psi = s2 / (m * m)
        with np.errstate(divide="ignore", invalid="ignore"):
            ip = 2.0 / psi
            b2 = ip - 1.0 + np.sqrt(ip) * np.sqrt(np.maximum(ip - 1.0, 0.0))
            a = m / (1.0 + b2)
            vq = a * (np.sqrt(b2) + zv) ** 2
            p = (psi - 1.0) / (psi + 1.0)
            beta = (1.0 - p) / m
            u = ndtr(zv)
            ve = np.where(u <= p, 0.0, np.log((1.0 - p) / (1.0 - u)) / beta)
        vn = np.where(psi <= psi_c, vq, ve)
        x = x + (K0 + K1 * v + K2 * vn + np.sqrt(K3 * v + K4 * vn) * zx)
        q = q + 0.5 * dt * (v + vn)
        v = vn
    return x, v, q
