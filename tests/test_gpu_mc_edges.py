"""GPU: the Monte Carlo kernels at the edges random samples do not reach, against high-precision references.

  - the fp64 Box-Muller (gauss64.cuh) on constructed Philox words: every log-table seam, u1 = 2^-52 (R = 8.49), u1 -> 1, every
    sin/cos-table interval at both ends and the centre; the paired check mode on its 32-bit uniforms; mpmath at 40 digits;
  - the default float draws (philox.cuh::box_muller_f32) near u1 -> 1 and u1 -> 0, with an error bound derived per point from the
    PTX-documented errors of the SFU instructions;
  - the fp64 helpers fast_div / fast_sqrt / fast_sqrt_pos / neg2_log / exp_table in ulps, at their seams and over their domains;
  - the log-vol range guard of LogsvPath<double> and its clamped re-run, against a clamped restatement in oracle/mc.py;
  - the fp32 state mode, path by path against the oracle fed with the same (float-rounded) normals.
Every input is a valid one: these tests exercise numerics only.
"""
import numpy as np
import pytest

from oracle import mc

pytestmark = pytest.mark.gpu

mpmath = pytest.importorskip("mpmath")
mp = mpmath.mp

EPS = 2.0 ** -52
BTC = (0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458)


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


# ---- word construction (the bit layout of philox.cuh) ----------------------------------------------------------------------------
def _words_f64(k1, m2, junk=0):
    """Philox words whose fp64 draw has u1 = k1 2^-52 (k1 odd, 1 <= k1 < 2^52) and u2 = m2 2^-52 (0 <= m2 < 2^52).
    u1 = 2 - d(r0, r1 | 1): mantissa M1 = 2^52 - k1;  u2 = d(r2, r3) - 1: mantissa m2.  `junk` fills the 12 low bits of r0 / r2 that the
    draw ignores."""
    k1 = np.asarray(k1, dtype=np.uint64)
    m2 = np.asarray(m2, dtype=np.uint64)
    M1 = np.uint64(1 << 52) - k1
    w = np.empty(np.broadcast(k1, m2).shape + (4,), dtype=np.uint32)
    w[..., 0] = (((M1 >> np.uint64(32)) << np.uint64(12)) | np.uint64(junk & 0xFFF)).astype(np.uint32)
    w[..., 1] = (M1 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    w[..., 2] = (((m2 >> np.uint64(32)) << np.uint64(12)) | np.uint64(junk & 0xFFF)).astype(np.uint32)
    w[..., 3] = (m2 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return w.reshape(-1, 4)


def _reachable_k1(u):
    """nearest u1 the fp64 draw can produce: an odd multiple of 2^-52 in (0, 1)"""
    k = int(round(u * 2.0 ** 52))
    k |= 1
    return min(max(k, 1), (1 << 52) - 1)


def _exact_normals(u1, u2, turns=True):
    """(R cos 2 pi u2, R sin 2 pi u2), R = sqrt(-2 ln u1), at 40 digits; u1 / u2 exact binary fractions given as mpf"""
    with mp.workdps(40):
        R = mp.sqrt(-2 * mp.log(u1))
        a = 2 * mp.pi * u2 if turns else u2
        return R, R * mp.cos(a), R * mp.sin(a)


def _log_seams(binades):
    """every g_log_tab interval boundary (hx low 13 bits zero, lo word zero), -2..+2 ulp, in the given binades e (u = 2^e m, m in
    [sqrt(1/2), sqrt(2))), restricted to 0 < u <= 1"""
    OFF = 0x3FF00000 - 0x3FE6A09E
    out = []
    for e in binades:
        for i in range(128):
            hx = ((e + 0x3FF) << 20) | (i << 13)
            hi = hx - OFF
            u = np.array([hi << 32], dtype=np.uint64).view(np.float64)[0]
            for d in (-2, -1, 0, 1, 2):
                v = u
                for _ in range(abs(d)):
                    v = np.nextafter(v, np.inf if d > 0 else -np.inf)
                if 0.0 < v <= 1.0:
                    out.append(v)
    return np.unique(np.array(out))


# ---- fp64 Box-Muller -----------------------------------------------------------------------------------------------------------------
def test_f64_box_muller_edges_vs_mpmath(cuda_lib):
    """box_muller_f64_fast on constructed words: u1 at 2^-52 (R = 8.49), 1 - 2^-52, next to powers of two, next to sqrt(1/2) 2^e and next to
    every log-table seam in several binades; u2 at 0, 1/4, 1/2, 3/4, 1 - 2^-52 and at every sin/cos-table interval's start, centre and last
    ulp.  Error against 40-digit mpmath, in units of 2^-52 max(1, R)."""
    from stochvolmodels_b200 import _capi as C, engine
    u1s = {1, (1 << 52) - 1}
    for e in range(1, 52):
        for k in (_reachable_k1(2.0 ** -e) - 2, _reachable_k1(2.0 ** -e), _reachable_k1(2.0 ** -e) + 2,
                  _reachable_k1(np.sqrt(0.5) * 2.0 ** -e)):
            u1s.add(k)
    for u in _log_seams([0, -1, -2, -7, -20, -40]):
        k = _reachable_k1(u)
        u1s.update({k - 2, k, k + 2})
    k1 = np.array(sorted(k for k in u1s if 1 <= k < (1 << 52)), dtype=np.uint64)
    u2_quarters = np.array([0, 1 << 50, 1 << 51, 3 << 50, (1 << 52) - 1], dtype=np.uint64)
    j = np.arange(256, dtype=np.uint64)
    u2_seams = np.concatenate([j << np.uint64(44), (j << np.uint64(44)) + np.uint64(1 << 43), ((j + np.uint64(1)) << np.uint64(44)) - np.uint64(1)])
    k_few = np.array([1, _reachable_k1(0.5), _reachable_k1(0.9), (1 << 52) - 1], dtype=np.uint64)
    words = np.concatenate([_words_f64(k1[:, None], u2_quarters[None, :], junk=0xABC), _words_f64(k_few[:, None], u2_seams[None, :])])
    z = engine.debug_box_muller(words, C.GAUSS_F64)
    assert np.all(np.isnan(z[:, 2:]))
    worst, worst_at = 0.0, None
    for w, (z0, z1) in zip(words, z[:, :2]):
        M1 = ((int(w[0]) >> 12) << 32) | (int(w[1]) | 1)
        m2 = ((int(w[2]) >> 12) << 32) | int(w[3])
        R, e0, e1 = _exact_normals(mp.mpf((1 << 52) - M1) / 2 ** 52, mp.mpf(m2) / 2 ** 52)
        scale = EPS * max(1.0, float(R))
        err = max(abs(float(mp.mpf(z0) - e0)), abs(float(mp.mpf(z1) - e1))) / scale
        if err > worst:
            worst, worst_at = err, (float(R), m2)
    print(f"fp64 Box-Muller edges: {len(words)} points, max |z - z_exact| = {worst:.3f} x 2^-52 max(1, R) at (R, u2 bits) = {worst_at}")
    assert worst <= 2.5, (worst, worst_at)                   # measured on an H100: 1.89
    # u1 = 2^-52 is the largest radius the fp64 stream can draw
    r_max = np.hypot(*engine.debug_box_muller(_words_f64([1], [0]), C.GAUSS_F64)[0, :2])
    assert abs(r_max - float(mp.sqrt(104 * mp.log(2)))) <= 4 * EPS * 8.5


def test_f64_paired_box_muller_edges_vs_mpmath(cuda_lib):
    """box_muller_f64_u32 (check mode B200SV_GAUSS_F64_PAIRED): ra in {0, 1, 2^31, 2^32 - 1} against every rb >> 24 interval at both ends,
    on both word pairs.  u1 = (ra + 1/2) 2^-32, angle = rb 2^-32 turns."""
    from stochvolmodels_b200 import _capi as C, engine
    ras = np.array([0, 1, 1 << 31, 0xFFFFFFFF], dtype=np.uint64)
    j = np.arange(256, dtype=np.uint64) << np.uint64(24)
    rbs = np.concatenate([j, j | np.uint64(0xFFFFFF), j | np.uint64(0x800000)])
    ra, rb = np.broadcast_arrays(ras[:, None], rbs[None, :])
    ra, rb = ra.ravel().astype(np.uint32), rb.ravel().astype(np.uint32)
    words = np.stack([ra, rb, ra[::-1], rb[::-1]], axis=1)
    z = engine.debug_box_muller(words, C.GAUSS_F64_PAIRED)
    worst = 0.0
    for w, zz in zip(words, z):
        for p in range(2):
            R, e0, e1 = _exact_normals((mp.mpf(int(w[2 * p])) + mp.mpf(0.5)) / 2 ** 32, mp.mpf(int(w[2 * p + 1])) / 2 ** 32)
            scale = EPS * max(1.0, float(R))
            worst = max(worst, abs(float(mp.mpf(zz[2 * p]) - e0)) / scale, abs(float(mp.mpf(zz[2 * p + 1]) - e1)) / scale)
    print(f"fp64 paired Box-Muller edges: {2 * len(words)} pairs, max |z - z_exact| = {worst:.3f} x 2^-52 max(1, R)")
    assert worst <= 2.0, worst                               # measured on an H100: 1.42


# ---- float SFU draws -----------------------------------------------------------------------------------------------------------------
LG2_ABS = 2.0 ** -22       # PTX ISA, lg2.approx.f32: max absolute error 2^-22.6 (mantissa part; the exponent part is exact)
SQRT_REL = 2.0 ** -22      # sqrt.approx.f32: max relative error 2^-23 (taken as 2^-22)
SINCOS_ABS = 2.0 ** -20    # sin / cos.approx.f32: max absolute error 2^-20.5 on [-pi, pi] (taken as 2^-20)
F32_EPS = 2.0 ** -24       # one float rounding


def _f32_uniforms(ra, rb):
    """the float u1 and angle box_muller_f32 computes from (ra, rb), reproduced bit for bit: fmaf(float(ra), 2^-32, 2^-33) is exact
    before its single rounding; the angle is one float product"""
    fra = ra.astype(np.float32).astype(np.float64)
    u1 = (fra * 2.0 ** -32 + 2.0 ** -33).astype(np.float32)
    ang = rb.view(np.int32).astype(np.float32) * np.float32(1.4629180792671596e-09)
    return u1, ang


def _f32_bound(u1):
    """per-point bound of |z_f32 - R cos| for the SAME float u1 / angle, from the SFU error figures:
    R^2 = -2 ln2 lg2(u1) is off by <= 2 ln2 LG2_ABS absolute plus two float roundings (constant, product); sqrt.approx adds SQRT_REL;
    cos / sin add SINCOS_ABS times R; the final product one rounding.  dR <= min(sqrt(dR2), dR2 / R) + (R + ...) SQRT_REL."""
    ld = np.longdouble
    R2 = -2.0 * np.log(u1.astype(ld))
    R = np.sqrt(R2)
    dR2 = 2.0 * np.log(ld(2)) * LG2_ABS + R2 * 3 * F32_EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        dR = np.minimum(np.sqrt(dR2), np.where(R > 0, dR2 / R, np.inf)) + (R + np.sqrt(dR2)) * SQRT_REL
    Rt = R + dR
    return R, (dR + Rt * SINCOS_ABS + Rt * F32_EPS).astype(np.float64)


def _check_f32_draws(ra, rb, what):
    from stochvolmodels_b200 import _capi as C, engine
    words = np.stack([ra, rb, ra[::-1], rb[::-1]], axis=1)
    z = engine.debug_box_muller(words, C.GAUSS_F32)
    zz = np.concatenate([z[:, 0:2], z[:, 2:4]])
    ra_all, rb_all = np.concatenate([ra, ra[::-1]]), np.concatenate([rb, rb[::-1]])
    assert np.all(np.isfinite(zz)), (what, "non-finite draw", ra_all[~np.all(np.isfinite(zz), axis=1)][:8])
    assert np.abs(zz).max() <= 6.764, (what, np.abs(zz).max())
    u1, ang = _f32_uniforms(ra_all, rb_all)
    R, bound = _f32_bound(u1)
    a = ang.astype(np.longdouble)
    err = np.maximum(np.abs(zz[:, 0] - (R * np.cos(a))).astype(np.float64), np.abs(zz[:, 1] - (R * np.sin(a))).astype(np.float64))
    ratio = err / bound
    k = int(np.argmax(ratio))
    near1 = u1 > np.float32(1 - 2.0 ** -10)
    print(f"float draws, {what}: {zz.shape[0]} pairs, max |z - z_exact| = {err.max():.3e} (u1 > 1 - 2^-10: {err[near1].max() if near1.any() else 0:.3e}), "
          f"max err / bound = {ratio[k]:.3f} at u1 = {float(u1[k])!r}")
    assert np.all(err <= bound), (what, float(err[k]), float(bound[k]), float(u1[k]))
    return err, u1


def test_f32_box_muller_near_u1_one_and_zero(cuda_lib):
    """default float draws for every ra in the top 2^20 (u1 -> 1: R down to 3.45e-4, where the lg2.approx error is as large as the value)
    and the bottom 2^16 (u1 -> 2^-33: R up to 6.76), crossed with a handful of rb: finite, |z| <= sqrt(-2 ln 2^-33) = 6.7636, and within
    the SFU error bound derived for the same float u1 and angle"""
    ra_top = np.arange((1 << 32) - (1 << 20), 1 << 32, dtype=np.uint64).astype(np.uint32)
    ra_bot = np.arange(0, 1 << 16, dtype=np.uint32)
    ra = np.concatenate([ra_top, ra_bot])
    rbs = np.array([0, 1 << 30, 0x80000000, 0xC0000000, 0x12345678, 0xFFFFFFFF], dtype=np.uint32)
    for rb in rbs:
        _check_f32_draws(ra, np.full_like(ra, rb), f"rb = {rb:#x}")
    # the largest radius the float stream can draw: ra = 0, u1 = 2^-33
    err, u1 = _check_f32_draws(np.zeros(1, np.uint32), np.zeros(1, np.uint32), "ra = 0")
    assert float(u1[0]) == 2.0 ** -33


def test_f32_box_muller_random_words(cuda_lib):
    rs = np.random.RandomState(20261015)
    ra = rs.randint(0, 1 << 32, size=1 << 20, dtype=np.uint64).astype(np.uint32)
    rb = rs.randint(0, 1 << 32, size=1 << 20, dtype=np.uint64).astype(np.uint32)
    _check_f32_draws(ra, rb, "random words")


# ---- fp64 helpers ----------------------------------------------------------------------------------------------------------------------
def _ulp_err(got, exact_ld):
    """|got - exact| in ulps of the exact value rounded to double"""
    return (np.abs(got.astype(np.longdouble) - exact_ld) / _ulp(exact_ld.astype(np.float64)).astype(np.longdouble)).astype(np.float64)


def _pow2_operands(lo, hi, rs, n_random):
    e = np.arange(lo, hi + 1, dtype=np.float64)
    grid = np.concatenate([np.ldexp(1.0, e.astype(int)), np.ldexp(2.0 - EPS, e.astype(int))])
    rnd = np.ldexp(rs.uniform(1.0, 2.0, n_random), rs.randint(lo, hi + 1, n_random))
    return grid, rnd


def test_fast_div_and_fast_sqrt_within_2_ulp(cuda_lib):
    """fast_div / fast_sqrt (MUFU seed + Newton steps, fastmath64.cuh; documented <= 2 ulp, asserted <= 1 ulp) on operands with exponents -1000..1000 and mantissas 1 and
    2 - ulp, on random operands over that range and over the ranges of the Heston QE step (1e-8..1e8)"""
    from stochvolmodels_b200 import _capi as C, engine
    rs = np.random.RandomState(5)
    grid, rnd = _pow2_operands(-1000, 1000, rs, 400000)
    ga, gb = np.meshgrid(grid[::7], grid[::7])
    a = np.concatenate([ga.ravel(), rnd, 10.0 ** rs.uniform(-8, 8, 200000)])
    b = np.concatenate([gb.ravel(), rnd[::-1], 10.0 ** rs.uniform(-8, 8, 200000)])
    ea, eb = np.frexp(a)[1], np.frexp(b)[1]
    keep = np.abs(ea - eb) <= 1000
    a, b = a[keep], b[keep]
    q = engine.debug_fastmath(C.DEBUG_FAST_DIV, a, b)
    ld = np.longdouble
    e_div = _ulp_err(q, a.astype(ld) / b.astype(ld))
    x = np.concatenate([grid, rnd, 10.0 ** rs.uniform(-8, 8, 200000)])
    s = engine.debug_fastmath(C.DEBUG_FAST_SQRT, x)
    e_sqrt = _ulp_err(s, np.sqrt(x.astype(ld)))
    print(f"fast_div: {a.size} points, max {e_div.max():.3f} ulp;  fast_sqrt: {x.size} points, max {e_sqrt.max():.3f} ulp")
    assert e_div.max() <= 1.0, (e_div.max(), a[np.argmax(e_div)], b[np.argmax(e_div)])
    assert e_sqrt.max() <= 1.0, (e_sqrt.max(), x[np.argmax(e_sqrt)])


def test_fast_sqrt_pos_and_neg2_log_over_their_domains(cuda_lib):
    """the two halves of the fp64 radius: fast_sqrt_pos on its documented domain [2^-60, 2^10] (<= 2 ulp); neg2_log = -2 ln(u) on positive
    normal u <= 1 -- every log-table seam +-2 ulp in several binades against mpmath, u -> 1, and random u over the whole normal range"""
    from stochvolmodels_b200 import _capi as C, engine
    ld = np.longdouble
    rs = np.random.RandomState(6)
    grid, rnd = _pow2_operands(-60, 9, rs, 300000)
    x = np.concatenate([grid, rnd, [2.0 ** -60, 2.0 ** 10]])
    e_sp = _ulp_err(engine.debug_fastmath(C.DEBUG_FAST_SQRT_POS, x), np.sqrt(x.astype(ld)))
    seams = np.append(_log_seams([0, -1, -2, -3, -10, -52, -100, -500, -1000, -1021]), 1.0)
    got = engine.debug_fastmath(C.DEBUG_NEG2_LOG, seams)
    with mp.workdps(40):
        exact = np.array([-2 * mp.log(mp.mpf(float(u))) for u in seams])
    rel_seam = np.array([abs(float((mp.mpf(float(g)) - e) / e)) if e != 0 else abs(float(g)) for g, e in zip(got, exact)])
    near1 = 1.0 - EPS / 2 * np.arange(1, 4097)
    bulk = np.concatenate([near1, np.ldexp(rs.uniform(0.5, 1.0, 500000), -rs.randint(0, 1022, 500000)), rs.uniform(0.0, 1.0, 200000)])
    bulk = bulk[bulk >= 2.0 ** -1022]
    got_b = engine.debug_fastmath(C.DEBUG_NEG2_LOG, bulk)
    ex_b = -2 * np.log(bulk.astype(ld))
    rel_b = (np.abs(got_b.astype(ld) - ex_b) / ex_b).astype(np.float64)
    print(f"fast_sqrt_pos: max {e_sp.max():.3f} ulp;  neg2_log: seams max rel {rel_seam.max() / EPS:.3f} x 2^-52 ({seams.size} points), "
          f"bulk + u -> 1 max rel {rel_b.max() / EPS:.3f} x 2^-52")
    assert e_sp.max() <= 1.0, e_sp.max()
    assert np.all(got[seams == 1.0] == 0.0)
    # measured on an H100: 2.21 / 2.41 x 2^-52
    assert rel_seam.max() <= 3 * EPS and rel_b.max() <= 3 * EPS, (rel_seam.max() / EPS, rel_b.max() / EPS)


def test_exp_table_within_2_ulp(cuda_lib):
    """exp_table (rough-vol kernel): < 3 ulp on [-700, 700] (measured on an H100: 2.97 ulp near x = -474.13), including every table node (256 k + j) ln2/256 and its neighbours +-1 ulp"""
    from stochvolmodels_b200 import _capi as C, engine
    ld = np.longdouble
    n = np.arange(-258530, 258531, dtype=np.float64)
    nodes = (n.astype(ld) * (np.log(ld(2)) / 256)).astype(np.float64)
    nodes = nodes[np.abs(nodes) <= 700.0]
    x = np.concatenate([nodes, np.nextafter(nodes, np.inf), np.nextafter(nodes, -np.inf), [-700.0, 700.0, 0.0, -0.0, 1e-300],
                        np.random.RandomState(7).uniform(-700, 700, 1000000)])
    x = x[np.abs(x) <= 700.0]
    e = _ulp_err(engine.debug_fastmath(C.DEBUG_EXP_TABLE, x), np.exp(x.astype(ld)))
    print(f"exp_table: {x.size} points, max {e.max():.3f} ulp")
    assert e.max() < 3.0, (e.max(), x[np.argmax(e)])


# ---- log-vol range guard ---------------------------------------------------------------------------------------------------------------
def test_logvol_range_guard_rerun_matches_clamped_oracle(cuda_lib):
    """BTC parameters, 252 steps/yr: a path started at sigma0 = 1e-6 sees a1/sigma ~ 1.3e4 on its first step, leaves |log sigma| <= 699.997,
    and is re-run by the kernel with the per-step clamp (one such path per warp).  Every other path must be bit-identical to a run without
    them (the divergent re-run does not disturb its lanes); every tripped path must match the clamped oracle -- sigma_T at exp(+-699.997),
    x and q non-finite -- and the payoffs must follow the NaN convention of compute_mc_vars_payoff."""
    from stochvolmodels_b200 import _capi as C, engine
    N, npy, seed, ttm = 4096, 252, 99, 0.25
    s0 = np.full(N, 0.8)
    tripped = np.arange(N) % 32 == 7
    s0[tripped] = 1e-6
    pc = engine.logsv_params_c(*BTC)
    flags = engine.mc_flags("fp64", "fp64")
    for is_spot in (True, False):
        x, s, q = engine.logsv_terminal_from_state(pc, np.zeros(N), s0, np.zeros(N), ttm, npy, is_spot, 1.0, seed, flags)
        xr, sr, qr = engine.logsv_terminal_from_state(pc, np.zeros(N), np.full(N, 0.8), np.zeros(N), ttm, npy, is_spot, 1.0, seed, flags)
        for a, b in ((x, xr), (s, sr), (q, qr)):
            np.testing.assert_array_equal(a[~tripped], b[~tripped])
        S, dt = mc.set_time_grid(ttm, npy)
        Z0, Z1 = engine.device_normals(seed, 0, N, 0, S, C.GAUSS_F64)
        with np.errstate(over="ignore", invalid="ignore"):
            xo, so, qo = mc.logsv_step_fixed(np.zeros(N), s0, np.zeros(N), Z0, Z1, dt, *BTC[1:], 1.0, is_spot, clamp=True)
            xu, su, _ = mc.logsv_step_fixed(np.zeros(N), s0, np.zeros(N), Z0, Z1, dt, *BTC[1:], 1.0, is_spot)
        assert not np.all(np.isfinite(su[tripped]))        # unclamped, the recursion breaks down: the guard is what keeps sigma finite
        np.testing.assert_allclose(s[tripped], so[tripped], rtol=1e-12)
        with mp.workdps(40):
            edge = {sign: float(mp.exp(sign * mp.mpf(258530) * mp.log(2) / 256)) for sign in (1, -1)}
        at_edge = np.where(s[tripped] > 1, edge[1], edge[-1])
        np.testing.assert_allclose(s[tripped], at_edge, rtol=4 * EPS)
        assert not np.any(np.isfinite(x[tripped])) and not np.any(np.isfinite(xo[tripped]))
        assert not np.any(np.isfinite(q[tripped])) and not np.any(np.isfinite(qo[tripped]))
        np.testing.assert_allclose(x[~tripped], xo[~tripped], rtol=0, atol=1e-11)
        np.testing.assert_allclose(s[~tripped], so[~tripped], rtol=1e-11)
        # payoffs on those states: a NaN path counts in C / P and pays 0, IC / IP skip it (utils/mc_payoffs.py's np.where + nanmean)
        xn = np.where(np.isfinite(x), x, np.nan)
        K, T = np.array([0.8, 1.0, 1.2, 0.9, 1.1]), np.array(["C", "P", "C", "IC", "IP"])
        pg, eg = engine.mc_payoffs(xn, q, ttm, 1.0, K, T, 0.99)
        po, eo = mc.mc_payoffs(xn, q, ttm, 1.0, K, T, 0.99)
        np.testing.assert_allclose(pg, po, rtol=1e-11)                    # re-centring sums in a different order
        np.testing.assert_allclose(eg, eo, rtol=1e-10)
        spots = np.exp(xn[~tripped])
        spots = spots - (spots.mean() - 1.0)
        np.testing.assert_allclose(pg[0], 0.99 * np.sum(np.maximum(spots - 0.8, 0)) / N, rtol=1e-11)
        np.testing.assert_allclose(pg[3], 0.99 * np.mean(np.maximum(spots - 0.9, 0) / spots), rtol=1e-11)


def test_logvol_range_guard_recovering_paths(cuda_lib):
    """kappa1 = kappa2 = 0: the log-vol is a random walk with drift and no 1/sigma or sigma feedback.  Started at 699.8, most paths cross the
    guard and are re-run with the clamp, and many come back into range: their sigma_T is finite and path-specific, so the re-run must restart
    from the loaded state to match the clamped oracle"""
    from stochvolmodels_b200 import _capi as C, engine
    N, npy, seed, ttm = 4096, 252, 5, 0.25
    params = (float(np.exp(699.8)), 1.0, 0.0, 0.0, 0.2, 1.0)
    S, dt = mc.set_time_grid(ttm, npy)
    Z0, Z1 = engine.device_normals(seed, 0, N, 0, S, C.GAUSS_F64)
    x, s, q = engine.logsv_terminal_from_state(engine.logsv_params_c(*params), np.zeros(N), np.full(N, params[0]), np.zeros(N), ttm, npy, True,
                                               1.0, seed, engine.mc_flags("fp64", "fp64"))
    with np.errstate(over="ignore", invalid="ignore"):
        xo, so, qo = mc.logsv_step_fixed(np.zeros(N), np.full(N, params[0]), np.zeros(N), Z0, Z1, dt, *params[1:], 1.0, True, clamp=True)
        _, su, _ = mc.logsv_step_fixed(np.zeros(N), np.full(N, params[0]), np.zeros(N), Z0, Z1, dt, *params[1:], 1.0, True)
    clipped = ~(so == su)
    print(f"recovering guard paths: {clipped.sum()} of {N} clamped, {np.sum(np.log(s[clipped]) < mc.LOG_VOL_CLAMP - 0.1)} back below 699.9")
    assert 0.3 * N < clipped.sum() < 0.95 * N and np.all(np.isfinite(s))
    assert np.mean(np.log(s[clipped]) < mc.LOG_VOL_CLAMP - 0.1) > 0.2          # re-run paths that came back inside the range
    np.testing.assert_allclose(s, so, rtol=1e-10)


# ---- fp32 state --------------------------------------------------------------------------------------------------------------------------
def _dev_slices(model, params, ttms, etas, fws, N, npy, is_spot, seed, flags):
    """chain of device-level slices on float32 torch state; returns the (x, v, q) state after every slice as float64 numpy arrays"""
    import torch
    from ctypes import byref, c_void_p
    from stochvolmodels_b200 import _capi as C, engine
    st = torch.zeros((3, N), dtype=torch.float32, device="cuda")
    mom = torch.zeros(2, dtype=torch.float64, device="cuda")
    stream = c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: c_void_p(t.data_ptr())
    out = []
    for m, (S, dt) in enumerate(mc.chain_steps(ttms, npy)):
        if model == "logsv":
            pc = engine.logsv_params_c(*params)
            C.call("b200sv_dev_logsv_slice", ptr(st[0]), ptr(st[1]), ptr(st[2]), N, 0, int(m == 0), byref(pc), float(etas[m]), int(is_spot), S, dt, m,
                   float(fws[m]), seed, flags, ptr(mom), None, stream)
        else:
            pc = engine.heston_params_c(*params)
            C.call("b200sv_dev_heston_slice", ptr(st[0]), ptr(st[1]), ptr(st[2]), N, 0, int(m == 0), byref(pc), S, dt, m, float(fws[m]), seed, flags,
                   C.HESTON_EULER_FLOOR, ptr(mom), None, stream)
        torch.cuda.synchronize()
        out.append(st.double().cpu().numpy())
    return out


def _f32_normals(seed, N, ttms, npy):
    from stochvolmodels_b200 import _capi as C, engine
    Z = [engine.device_normals(seed, 0, N, m, S, C.GAUSS_F64) for m, (S, _) in enumerate(mc.chain_steps(ttms, npy))]
    return [z[0].astype(np.float32).astype(np.float64) for z in Z], [z[1].astype(np.float32).astype(np.float64) for z in Z]


# Tolerances (fp32 state, fp64 oracle on the same float-rounded normals): each step rounds the log-vol update (3 FMAs), the SFU exponential
# (__expf: ~2 ulp) and reciprocal, and the running sums once each -- up to ~8 float eps of relative error per step if every rounding went
# the same way, which the sums carry to the end of the chain (8 * 2^-24 * 60 steps = 2.9e-5).  Roundings do not all go the same way: on an
# H100 the largest deviations over 20000 paths were 1.5e-6 in x and 6.2e-7 in sigma after 65 steps, ~0.4 float eps per step.  Asserted:
# 2 float eps per step so far, relative on sigma / variance, and on x, q per unit of their scale (7.8e-6 after 65 steps).
F32_STEP_TOL = 2 * 2.0 ** -24


@pytest.mark.parametrize("is_spot,variable_type", [(True, mc.LOG_RETURN), (False, mc.Q_VAR)])
def test_fp32_state_logsv_chain_vs_oracle(cuda_lib, is_spot, variable_type):
    """LogSV with B200SV_STATE_F32 | B200SV_GAUSS_F64: three maturities (float state carried across slices), eta != 1, both measures, Q_VAR
    payoffs: terminal states path by path and chain prices against the oracle fed with the same normals rounded to float"""
    from stochvolmodels_b200 import _capi as C, engine
    N, npy, seed = 20000, 252, 2718
    ttms, fws, dfs, etas = np.array([0.1, 0.2, 0.25]), np.array([1.0, 1.01, 1.02]), np.array([0.999, 0.99, 0.985]), np.array([0.9, 1.1, 0.8])
    K = np.array([0.8, 0.95, 1.0, 1.05, 1.2]) if variable_type == mc.LOG_RETURN else np.array([0.3, 0.5, 0.7, 0.9, 1.2])
    # vanilla codes only: an inverse payoff divides by the re-centred spot, which amplifies the float state's error without bound on
    # paths whose spot is near zero, so no tolerance derived from the state error applies to it
    T = np.array(["P", "P", "C", "C", "C"])
    flags = C.STATE_F32 | C.GAUSS_F64
    states = _dev_slices("logsv", BTC, ttms, etas, fws, N, npy, is_spot, seed, flags)
    Z0, Z1 = _f32_normals(seed, N, ttms, npy)
    steps = mc.chain_steps(ttms, npy)
    po, eo, so = mc.logsv_mc_chain_fixed(BTC, ttms, fws, dfs, [K] * 3, [T] * 3, etas, Z0, Z1, [d for _, d in steps], is_spot, variable_type, True)
    S_cum = np.cumsum([S for S, _ in steps])
    for m in range(3):
        tol = F32_STEP_TOL * S_cum[m]
        (xg, sg, qg), (xo, sig_o, qo) = states[m], so[m]
        ex, es, eq = np.abs(xg - xo).max(), np.abs(sg / sig_o - 1).max(), np.abs(qg - qo).max() / np.abs(qo).max()
        print(f"fp32 LogSV state, slice {m} ({S_cum[m]} steps): max |dx| = {ex:.2e}, max |dsigma/sigma| = {es:.2e}, max |dq|/max q = {eq:.2e}, tol {tol:.2e}")
        assert ex <= tol and es <= tol and eq <= tol, (m, ex, es, eq, tol)
    pg, eg = engine.logsv_mc_chain(engine.logsv_params_c(*BTC), ttms, fws, dfs, etas, [K] * 3, [T] * 3, N, npy, is_spot, variable_type, seed, flags)
    for m in range(3):
        tol = F32_STEP_TOL * S_cum[m]
        scale = fws[m] if variable_type == mc.LOG_RETURN else so[m][2].max() / ttms[m]       # size of the underlying
        np.testing.assert_allclose(pg[m], po[m], rtol=0, atol=3 * tol * scale)
        np.testing.assert_allclose(eg[m], eo[m], rtol=0, atol=3 * tol * scale / np.sqrt(N))


def test_fp32_state_heston_floor_vs_oracle(cuda_lib):
    """Heston with B200SV_STATE_F32 | B200SV_GAUSS_F64 in the floor regime (Feller violated, v = max(v, 1e-4) binds): terminal states path by
    path over two slices and the chain prices against the oracle on the float-rounded normals"""
    from stochvolmodels_b200 import _capi as C, engine
    N, npy, seed = 20000, 360, 1618
    params = (0.01, 0.02, 1.0, -0.7, 1.0)
    ttms, fws, dfs = np.array([0.1, 0.2]), np.array([1.0, 1.01]), np.array([0.995, 0.99])
    flags = C.STATE_F32 | C.GAUSS_F64
    states = _dev_slices("heston", params, ttms, None, fws, N, npy, True, seed, flags)
    Z0, Z1 = _f32_normals(seed, N, ttms, npy)
    steps = mc.chain_steps(ttms, npy)
    K = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
    T = np.array(["P", "P", "C", "C", "C"])
    po, eo, so = mc.heston_mc_chain_fixed(params, ttms, fws, dfs, [K] * 2, [T] * 2, Z0, Z1, [d for _, d in steps], mc.LOG_RETURN, True)
    S_cum = np.cumsum([S for S, _ in steps])
    for m in range(2):
        tol = F32_STEP_TOL * S_cum[m]
        (xg, vg, qg), (xo, vo, qo) = states[m], so[m]
        ex, ev, eq = np.abs(xg - xo).max(), np.abs(vg - vo).max() / vo.max(), np.abs(qg - qo).max() / qo.max()
        print(f"fp32 Heston state, slice {m} ({S_cum[m]} steps): max |dx| = {ex:.2e}, max |dv|/max v = {ev:.2e}, max |dq|/max q = {eq:.2e}, tol {tol:.2e}")
        assert ex <= tol and ev <= tol and eq <= tol, (m, ex, ev, eq, tol)
        assert vg.min() >= np.float32(1e-4) and (m == 0 or np.any(vo == 1e-4))
    pg, eg = engine.heston_mc_chain(engine.heston_params_c(*params), ttms, fws, dfs, [K] * 2, [T] * 2, N, npy, 1, seed, flags)
    for m in range(2):
        tol = F32_STEP_TOL * S_cum[m]
        np.testing.assert_allclose(pg[m], po[m], rtol=0, atol=3 * tol * fws[m])
        np.testing.assert_allclose(eg[m], eo[m], rtol=0, atol=3 * tol * fws[m] / np.sqrt(N))
