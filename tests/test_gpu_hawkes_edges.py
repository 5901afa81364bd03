"""GPU: the Hawkes jump-diffusion Monte Carlo kernels at the edges random samples do not reach.

hawkes_path_steps (hawkes_kernels.cuh) decides a jump in three stages: a candidate filter on the raw 32-bit Philox word that relies on
saturating float-to-unsigned conversion, a logarithm-free accept e + e^2 < lambda dt (1 - 1e-9), and the exact comparison
lambda > -ln(u)/dt of the reference.  Random paths at the reference's parameters (lambda dt ~ 0.5 %) reach the saturating branches, the band
between the stages, the word endpoints and negative intensities rarely or never.  Here:
  - the clock and jump-size draws at the word endpoints against mpmath (b200sv_debug_hawkes_clocks);
  - the stepper's firing decision == the strict decision lambda > clock on constructed (word, intensity) pairs in every regime of lambda dt,
    with every branch of the three stages taken;
  - the four-step grouping of the stepper at S = 1..9 steps, in both Gaussian modes, path by path against the oracle;
  - the pricing and tangent kernels at saturated, zero-crossing and tiny intensities, path by path against the oracle;
  - paths beyond the second grid-stride iteration of both kernels.
Every input is a valid one: these tests exercise numerics and control flow only.
"""
from fractions import Fraction
import math

import numpy as np
import pytest

from oracle import hawkes
from oracle import hawkes_mc_greeks as hg

pytestmark = pytest.mark.gpu

mpmath = pytest.importorskip("mpmath")
mp = mpmath.mp

EPS = 2.0 ** -52
TWO32 = 1 << 32
STEPS_PER_YEAR = hawkes.STEPS_PER_YEAR


def _dt_of(ttm):
    from stochvolmodels_b200.utils.funcs import set_time_grid
    return set_time_grid(ttm, STEPS_PER_YEAR)[:2]


DT_1800 = 1.0 / 1800.0
DT_S1 = _dt_of(0.5 / 1800.0)[1]             # a one-step slice: dt = ttm
assert _dt_of(0.5 / 1800.0)[0] == 1


def _params(**kw):
    from stochvolmodels_b200 import HawkesJDParams
    return {k: v for k, v in HawkesJDParams(**kw).to_dict().items() if k in hawkes.KEYS}


def _pc(d):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    return _params_c(**d)


def _clocks(words, lam, dt, d):
    from stochvolmodels_b200 import engine
    return engine.debug_hawkes_clocks(np.asarray(words, dtype=np.uint32), lam, dt, _pc(d))


# ---- the filter of hawkes_candidate / hawkes_fires, restated in exact arithmetic ------------------------------------------------------------
def _thr(dt):
    return dt * (1.0 + 1e-9) * 4294967296.0          # HawkesFast::thr, same operations


def _tp(lam, dt):
    """__double2uint_rd(fma(-lam, thr, 2^32)): the product and sum exact, one rounding to double, floor, saturated to [0, 2^32 - 1]"""
    v = float(Fraction(TWO32) - Fraction(lam) * Fraction(_thr(dt)))       # Fraction -> float rounds to nearest even
    if v != v or v <= 0.0:
        return 0
    return min(int(math.floor(v)), TWO32 - 1)


def _candidate(r, lam, dt):
    return r >= max(_tp(lam, dt), 1) - 1


def _log_free(r, lam, dt):
    """the logarithm-free accept of hawkes_fires: e <= 1/2 and fma(e, e, e) < lam * dt (1 - 1e-9)"""
    e = Fraction(TWO32 - r) / TWO32 - Fraction(1, 1 << 33)                 # 1 - u, exact
    return e <= Fraction(1, 2) and float(e * e + e) < lam * (dt * (1.0 - 1e-9))


# ---- a. clock and size draws at the word endpoints --------------------------------------------------------------------------------------------
def _size_bound(mean, exact):
    """|size - exact| for size = shift + mean * l (sizes_m: shift - (-mean) l, the same roundings), l = -log(u) within 1 ulp of L = -ln(u):
    l = L (1 + d1), |d1| <= 2^-52; the product rounds once (d2) and the sum once (d3), |d2|, |d3| <= 2^-53.  So
    size - exact = (p - mean L) + d3 (shift + p) with |p - mean L| <= |mean L| (2^-52 + 2^-53 + 2^-105) =: a, and |shift + p| <= |exact| + a:
    the bound a + 2^-53 (|exact| + a) stays absolute where shift + mean L cancels towards 0."""
    a = abs(mean) * exact[1] * (3 * 2.0 ** -53 + 2.0 ** -105)
    return 1.0001 * (a + 2.0 ** -53 * (abs(exact[0]) + a))


@pytest.mark.parametrize("dt", [DT_1800, DT_S1, 1e-6], ids=["dt=1/1800", "dt=S1", "dt=1e-6"])
def test_clock_and_sizes_at_word_endpoints_vs_mpmath(cuda_lib, dt):
    """u = (r + 1/2) 2^-32 exactly; the clock -ln(u)/dt within 2 ulp and both jump sizes within the bound of _size_bound, at 40 digits.
    Two parameter sets: the reference's defaults and one whose sizes cross 0 at u = e^-2 (shift_p + mean_p L = 0.1 (L - 2) / 2, the
    minus size its mirror), with the words around that point included"""
    rs = np.random.RandomState(20261017)
    edge = [0, 1, 2, 3, (1 << 31) - 1, 1 << 31, TWO32 - 3, TWO32 - 2, TWO32 - 1]
    r0 = int(math.exp(-2.0) * TWO32)
    words = np.array(edge + list(range(r0 - 3, r0 + 4)) + list(rs.randint(0, TWO32, 2000, dtype=np.uint64)), dtype=np.uint64)
    worst = {"clock": 0.0, "size_p": 0.0, "size_m": 0.0}
    for d in (_params(), _params(shift_p=-0.1, mean_p=0.05, shift_m=0.1, mean_m=-0.05)):
        out = _clocks(words, 1.0, dt, d)
        u_exact = (words.astype(np.float64) + 0.5) * 2.0 ** -32                 # exact: 33 significant bits
        np.testing.assert_array_equal(out[:, 0], u_exact)
        for w, (u, clock, sp, sm, _, _) in zip(words, out):
            with mp.workdps(40):
                L = -mp.log((mp.mpf(int(w)) + mp.mpf(0.5)) / TWO32)
                c_ex = L / mp.mpf(dt)
                sp_ex = mp.mpf(d["shift_p"]) + mp.mpf(d["mean_p"]) * L
                sm_ex = mp.mpf(d["shift_m"]) + mp.mpf(d["mean_m"]) * L
                e_clock = float(abs(mp.mpf(clock) - c_ex)) / np.spacing(float(c_ex))
                e_sp = float(abs(mp.mpf(sp) - sp_ex)) / _size_bound(d["mean_p"], (float(sp_ex), float(L)))
                e_sm = float(abs(mp.mpf(sm) - sm_ex)) / _size_bound(d["mean_m"], (float(sm_ex), float(L)))
            assert e_clock <= 2.0, ("clock", int(w), dt, e_clock)
            assert e_sp <= 1.0 and e_sm <= 1.0, ("sizes", int(w), d, e_sp, e_sm)
            worst = {"clock": max(worst["clock"], e_clock), "size_p": max(worst["size_p"], e_sp), "size_m": max(worst["size_m"], e_sm)}
    print(f"Hawkes draws, dt = {dt:.3e}: clock max {worst['clock']:.3f} ulp; sizes max {worst['size_p']:.3f} / {worst['size_m']:.3f} of the bound")


# ---- b. the fused decision on constructed pairs ---------------------------------------------------------------------------------------------
LAM_DT = [-10.0, -1e-300, 0.0, 1e-12, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 0.49, 0.5, 0.51, 0.99, 1.0, 1.01, 1.71, 2.3, 50.0]


def _pairs(dt, rs):
    """(words, intensities): per intensity the candidate edge tp - 3 .. tp + 2, the edge of the logarithm-free accept, the word where
    -ln(u)/dt crosses lambda, both endpoints and a few random words"""
    lams = [x / dt for x in LAM_DT]
    lams += [1.0 / (dt * 2.0 ** 32) * (1.0 - 1e-6), 1.0 / (dt * 2.0 ** 32) * (1.0 + 1e-6)]     # lam thr crosses 1
    W, Lm = [], []
    for lam in lams:
        ws = {0, TWO32 - 1}
        tp = _tp(lam, dt)
        ws.update(range(tp - 3, tp + 3))
        a = lam * dt * (1.0 - 1e-9)
        if a > 0.0:
            e = (math.sqrt(1.0 + 4.0 * a) - 1.0) / 2.0                              # e + e^2 = a
            r = int(round(TWO32 * (1.0 - e) - 0.5))
            ws.update(range(r - 2, r + 3))
        r = int(round(math.exp(-min(lam * dt, 700.0)) * TWO32 - 0.5)) if lam > 0.0 else TWO32 - 1
        ws.update(range(r - 2, r + 3))
        ws.update(int(v) for v in rs.randint(0, TWO32, 32, dtype=np.uint64))
        ws = sorted(w for w in ws if 0 <= w < TWO32)
        W += ws
        Lm += [lam] * len(ws)
    return np.array(W, dtype=np.uint64), np.array(Lm)


@pytest.mark.parametrize("dt", [DT_1800, DT_S1], ids=["dt=1/1800", "dt=S1"])
def test_fused_decision_is_the_strict_decision_on_constructed_pairs(cuda_lib, dt):
    """fused == (lambda > clock) with the hook's own clock (what hawkes_step_fixed_kernel compares), candidate == its exact restatement
    and candidate >= fired, on pairs at every regime of lambda dt and on ties lambda = clock, +-1 and +-2 ulp (a tie does not fire);
    every branch -- not a candidate, accepted without a logarithm, exact test true, exact test false -- is taken"""
    rs = np.random.RandomState(int(1 / dt))
    d = _params()
    words, lams = _pairs(dt, rs)
    # ties: lambda at the clock itself and at its neighbours, for endpoint, edge and random words
    tw = np.array([0, 1, 2, (1 << 31), TWO32 - 2, TWO32 - 1] + list(rs.randint(0, TWO32, 200, dtype=np.uint64)), dtype=np.uint64)
    clock = _clocks(tw, 1.0, dt, d)[:, 1]
    near = [clock, np.nextafter(clock, np.inf), np.nextafter(np.nextafter(clock, np.inf), np.inf), np.nextafter(clock, -np.inf),
            np.nextafter(np.nextafter(clock, -np.inf), -np.inf)]
    words = np.concatenate([words] + [tw] * len(near))
    lams = np.concatenate([lams] + near)
    out = _clocks(words, lams, dt, d)
    clock, cand, fired = out[:, 1], out[:, 4] == 1.0, out[:, 5] == 1.0
    strict = lams > clock
    bad = np.flatnonzero(fired != strict)
    assert bad.size == 0, [(int(words[i]), lams[i] * dt, clock[i] * dt, bool(fired[i])) for i in bad[:8]]
    assert not np.any(fired & ~cand)
    cand_ref = np.array([_candidate(int(w), l, dt) for w, l in zip(words, lams)])
    bad = np.flatnonzero(cand != cand_ref)
    assert bad.size == 0, [(int(words[i]), lams[i] * dt, bool(cand[i])) for i in bad[:8]]
    assert not np.any(fired[len(words) - 5 * len(tw):len(words) - 4 * len(tw)]), "lambda == clock must not fire"
    free = np.array([c and _log_free(int(w), l, dt) for w, l, c in zip(words, lams, cand)])
    counts = {"not a candidate": int(np.sum(~cand)), "log-free accept": int(np.sum(free)),
              "exact true": int(np.sum(cand & ~free & fired)), "exact false": int(np.sum(cand & ~free & ~fired))}
    print(f"Hawkes firing decision, dt = {dt:.3e}: {len(words)} pairs, {counts}")
    assert np.all(fired[free]), "the logarithm-free accept must agree with the strict decision"
    assert min(counts.values()) >= 1, counts


# ---- c. the four-step grouping tails ----------------------------------------------------------------------------------------------------------
def _draws(seed, path0, n, m, ttm, gauss, d):
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import hawkesjd_device_draws
    return hawkesjd_device_draws(seed, path0, n, m, ttm, gauss=gauss, **d)


def _fixed_kw(d):
    return {k: v for k, v in d.items() if k not in ("lambda_p", "lambda_m")}


TOL_FUSED = dict(rtol=1e-12, atol=1e-14)       # tests/test_gpu_hawkes.py: contracted arithmetic, same draws and decisions as the strict kernel


@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
def test_four_step_grouping_tails_path_by_path(cuda_lib, gauss):
    """ttm = (S - 1/2)/1800 for S = 1..9 (S mod 4 = 0, 1, 2, 3; S = 1 with dt = ttm): two chained slices of the fused kernel against the
    oracle on the kernel's own draws, and the strict kernel bit for bit against the oracle, at intensities ~0.3/dt where jumps fire"""
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import simulate_hawkesjd_terminal
    N, seed = 4096, 4242
    for S in range(1, 10):
        ttm = (S - 0.5) / STEPS_PER_YEAR
        assert _dt_of(ttm)[0] == S
        lam = 0.3 / _dt_of(ttm)[1]
        d = _params(mu=0.01, sigma=0.5, lambda_p=lam, theta_p=lam, lambda_m=0.8 * lam, theta_m=0.8 * lam, kappa_p=30.0, kappa_m=40.0,
                    beta1_p=50.0, beta2_p=-40.0, beta1_m=60.0, beta2_m=-70.0)
        kw = _fixed_kw(d)
        x, lp, lm = np.zeros(1), np.array([d["lambda_p"]]), np.array([d["lambda_m"]])
        xo, lpo, lmo = np.zeros(N), np.full(N, d["lambda_p"]), np.full(N, d["lambda_m"])
        jumps = 0
        for m in range(2):
            blk = _draws(seed, 0, N, m, ttm, gauss, d)
            x1, lp1, lm1 = simulate_hawkesjd_terminal(ttm=ttm, x0=x, lambda_p0=lp, lambda_m0=lm, nb_path=N, seed=seed, gauss=gauss, slice_index=m,
                                                      **kw)
            xs, lps, lms = simulate_hawkesjd_terminal(ttm=ttm, x0=xo, lambda_p0=lpo, lambda_m0=lmo, nb_path=N, inputs=blk[:5], **kw)
            x2, lp2, lm2, *_, fires = hg.tangent_step_fixed(xo, lpo, lmo, *hg.initial_tangents(N), *blk, return_fires=True, **kw)
            xo, lpo, lmo = hawkes.step_fixed(xo, lpo, lmo, *blk, **d)
            for a, b in ((x2, xo), (lp2, lpo), (lm2, lmo)):
                np.testing.assert_array_equal(a, b)
            for a, b, what in ((x1, xo, "x"), (lp1, lpo, "lambda_p"), (lm1, lmo, "lambda_m")):
                np.testing.assert_allclose(a, b, **TOL_FUSED, err_msg=f"fused, S = {S}, slice {m}, {what}")
            for a, b, what in ((xs, xo, "x"), (lps, lpo, "lambda_p"), (lms, lmo, "lambda_m")):
                np.testing.assert_array_equal(a, b, err_msg=f"strict, S = {S}, slice {m}, {what}")
            jumps += int(fires[-1].sum())
            x, lp, lm = x1.copy(), lp1.copy(), lm1.copy()
        assert jumps > N // 10, ("jumps on the last step of each slice", S, jumps)


# ---- d. regimes the reference parameters never reach --------------------------------------------------------------------------------------
TTMS = np.array([0.01, 0.02])                  # 19 + 19 steps of dt = 1/1900
DT_D = _dt_of(0.01)[1]


def _regime(name):
    """(params, per-path initial intensities for the pricing kernel as a function of N)"""
    if name == "saturated":
        lam = 1.2 / DT_D
        # mixed signs: the mean load per firing step is ~ +4.5 on either intensity (J_p ~ +0.09, J_m ~ -0.09), kappa dt = 5 %
        d = _params(mu=0.0, sigma=0.3, lambda_p=lam, theta_p=lam, lambda_m=lam, theta_m=lam, kappa_p=100.0, kappa_m=100.0, beta1_p=200.0,
                    beta2_p=150.0, beta1_m=-100.0, beta2_m=-150.0)
        return d, lambda n: (np.linspace(0.9, 1.5, n) / DT_D, np.linspace(1.5, 0.9, n) / DT_D)
    if name == "crossing_zero":
        d = _params(mu=0.0, sigma=0.3, lambda_p=200.0, theta_p=200.0, lambda_m=200.0, theta_m=200.0, kappa_p=50.0, kappa_m=50.0, beta1_p=1000.0,
                    beta2_p=5000.0, beta1_m=-5000.0, beta2_m=-1000.0)
        return d, lambda n: (np.linspace(-300.0, 400.0, n), np.linspace(400.0, -300.0, n))
    # tiny: lambda_p below 1/(dt 2^32) for good; the minus clock fires now and then
    d = _params(mu=0.0, sigma=0.3, lambda_p=1e-8, theta_p=1e-8, lambda_m=300.0, theta_m=300.0, kappa_p=20.0, kappa_m=20.0, beta1_p=0.0,
                beta2_p=0.0, beta1_m=100.0, beta2_m=-100.0)
    spread = np.concatenate([[-5.0, -1.0, -1e-300, 0.0, 1e-300, 1e-12, 1e-9], np.geomspace(1e-8, 2.0 / DT_D, 57)])
    return d, lambda n: (np.resize(spread, n), np.resize(spread[::-1], n))


def _oracle_steps(x, lp, lm, tan, blk, kw):
    """hg.tangent_step_fixed one step at a time (the same operations): the state, tangents and the step-start intensities and decisions"""
    lps, lms, fires = [], [], []
    W0, U_P, U_M, J_P, J_M, dt = blk
    for s in range(W0.shape[0]):
        lps.append(lp)
        lms.append(lm)
        x, lp, lm, *tan, f = hg.tangent_step_fixed(x, lp, lm, *tan, W0[s:s + 1], U_P[s:s + 1], U_M[s:s + 1], J_P[s:s + 1], J_M[s:s + 1], dt,
                                                   return_fires=True, **kw)
        fires.append(f[0])
    return x, lp, lm, tan, np.array(lps), np.array(lms), np.array(fires)


def _check_paths(states, tangents, ref_state, ref_tan, what):
    """the per-path comparison of tests/test_gpu_hawkes_mc_greeks.py (relative to each row's scale)"""
    for a, b, name in zip(states, ref_state, ("x", "lambda_p", "lambda_m")):
        np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-10 * np.max(np.abs(b)), err_msg=f"{what} {name}")
    for c, ref, name in zip(tangents, ref_tan, ("dx", "dlambda_p", "dlambda_m", "score")):
        for q, p in enumerate(hg.PARAMS):
            scale = max(float(np.max(np.abs(ref[q]))), 1e-300)
            err = float(np.max(np.abs(c[q] - ref[q])))
            assert err <= 1e-10 * scale, (what, name, p, err / scale)


CHAIN_K, CHAIN_T = np.array([0.9, 1.0, 1.1]), np.array(["P", "C", "IC"])


@pytest.mark.parametrize("gauss", ["fp32", "fp64"])
@pytest.mark.parametrize("regime", ["saturated", "crossing_zero", "tiny"])
def test_pricing_and_tangent_kernels_in_regimes_the_reference_never_reaches(cuda_lib, regime, gauss):
    """two-maturity chain through b200sv_hawkesjd_mc_chain_greeks: the first paths' state, tangents and score per path against the oracle on
    the exported draws, prices bit-identical to the pricing route; the pricing kernel from per-path initial intensities against the oracle.
    Each regime asserts it was reached (share of steps with lambda dt >= 1 and two-clock steps; silent steps at lambda <= 0; lambda dt below
    2^-32 for good)"""
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import simulate_hawkesjd_terminal
    d, init = _regime(regime)
    kw = _fixed_kw(d)
    N, n_out, seed = 5000, 3000, 606
    fw, df = np.array([1.0, 1.0]), np.array([0.999, 0.998])
    flags = engine.mc_flags("fp64", gauss)
    res = engine.hawkesjd_mc_chain_greeks(_pc(d), TTMS, fw, df, [CHAIN_K] * 2, [CHAIN_T] * 2, N, 1, seed, flags, n_out)
    p_ref, e_ref = engine.hawkesjd_mc_chain(_pc(d), TTMS, fw, df, [CHAIN_K] * 2, [CHAIN_T] * 2, N, 1, seed, flags)
    for m in range(2):
        np.testing.assert_array_equal(res[0][m], p_ref[m])
        np.testing.assert_array_equal(res[1][m], e_ref[m])
    states, tangents = res[5], res[6]
    x, lp, lm, tan = np.zeros(n_out), np.full(n_out, d["lambda_p"]), np.full(n_out, d["lambda_m"]), list(hg.initial_tangents(n_out))
    lam_p, lam_m, fires, t0 = [], [], [], 0.0
    for m, ttm in enumerate(TTMS):
        blk = _draws(seed, 0, n_out, m, ttm - t0, gauss, d)
        t0 = ttm
        x, lp, lm, tan, lps, lms, f = _oracle_steps(x, lp, lm, tan, blk, kw)
        _check_paths(states[m], tangents[m], (x, lp, lm), tan, f"{regime} {gauss} tangent kernel, maturity {m}")
        lam_p.append(lps)
        lam_m.append(lms)
        fires.append(f)
    lam_p, lam_m, fires = np.concatenate(lam_p), np.concatenate(lam_m), np.concatenate(fires)
    silent_nonpos = int(np.sum((lam_p <= 0) & ~fires[:, 0]) + np.sum((lam_m <= 0) & ~fires[:, 1]))
    stats = {"lambda dt >= 1": float(np.mean(np.concatenate([lam_p, lam_m]) * DT_D >= 1.0)), "two clocks": int(np.sum(fires[:, 0] & fires[:, 1])),
             "silent at lambda <= 0": silent_nonpos, "fires": int(fires.sum())}
    print(f"Hawkes regime {regime} ({gauss}): {stats}")
    if regime == "saturated":
        assert stats["lambda dt >= 1"] > 0.5 and stats["two clocks"] > 0.3 * fires.shape[0] * n_out, stats
    elif regime == "crossing_zero":
        # a silent step at lambda <= 0 adds nothing to the score (the kernel's weight dt cancels its running -dt): checked in the rows above
        assert silent_nonpos > 1000 and np.any(lam_p < 0) and np.any(lam_m < 0), stats
    else:
        assert np.all(lam_p * DT_D < 2.0 ** -32) and np.all(lam_p > 0) and stats["fires"] > 100, stats
    # the pricing kernel from per-path initial intensities (b200sv_hawkesjd_terminal with use_initial_arrays)
    lp0, lm0 = init(N)
    x1, lp1, lm1 = simulate_hawkesjd_terminal(ttm=TTMS[0], x0=np.zeros(N), lambda_p0=lp0, lambda_m0=lm0, nb_path=N, seed=seed, gauss=gauss, **kw)
    blk = _draws(seed, 0, N, 0, TTMS[0], gauss, d)
    xo, lpo, lmo = hawkes.step_fixed(np.zeros(N), lp0, lm0, *blk, **d)
    for a, b, name in ((x1, xo, "x"), (lp1, lpo, "lambda_p"), (lm1, lmo, "lambda_m")):
        np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-10 * np.max(np.abs(b)), err_msg=f"{regime} {gauss} pricing kernel {name}")


# ---- e. paths beyond the first grid stride --------------------------------------------------------------------------------------------------
def test_paths_beyond_two_grid_strides(cuda_lib):
    """N > 2 x SMs x 2048 + 77 (2048: the most resident threads per H100 SM, so above two strides whatever occupancy persistent_grid picks):
    the first and the last 2048 paths of the pricing kernel and of the tangent kernel (one maturity, every path copied out) against the
    oracle on the draws of those paths"""
    import torch
    from stochvolmodels_b200 import engine
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import simulate_hawkesjd_terminal
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N, B, seed, gauss = 2 * sms * 2048 + 77 + 1000, 2048, 515, "fp32"
    ttm = 4.5 / STEPS_PER_YEAR                                        # 5 steps
    lam = 0.3 / _dt_of(ttm)[1]
    d = _params(sigma=0.4, lambda_p=lam, theta_p=lam, lambda_m=lam, theta_m=lam, kappa_p=30.0, kappa_m=30.0, beta1_p=40.0, beta2_p=-30.0,
                beta1_m=50.0, beta2_m=-60.0)
    kw = _fixed_kw(d)
    x, lp, lm = simulate_hawkesjd_terminal(ttm=ttm, x0=0.0, lambda_p0=d["lambda_p"], lambda_m0=d["lambda_m"], nb_path=N, seed=seed, gauss=gauss,
                                           **kw)
    res = engine.hawkesjd_mc_chain_greeks(_pc(d), [ttm], [1.0], [1.0], [CHAIN_K], [CHAIN_T], N, 1, seed, engine.mc_flags("fp64", gauss), N)
    states, tangents = res[5][0], res[6][0]
    for a, b in ((states[0], x), (states[1], lp), (states[2], lm)):
        np.testing.assert_array_equal(a, b)                           # the tangent kernel's primal is the pricing kernel's, bit for bit
    for path0 in (0, N - B):
        sl = slice(path0, path0 + B)
        blk = _draws(seed, path0, B, 0, ttm, gauss, d)
        xo, lpo, lmo, *tan, fires = hg.tangent_step_fixed(np.zeros(B), np.full(B, lam), np.full(B, lam), *hg.initial_tangents(B), *blk,
                                                          return_fires=True, **kw)
        assert fires.sum() > B // 4, ("jumps in the block", path0, int(fires.sum()))
        for a, b, name in ((x[sl], xo, "x"), (lp[sl], lpo, "lambda_p"), (lm[sl], lmo, "lambda_m")):
            np.testing.assert_allclose(a, b, **TOL_FUSED, err_msg=f"pricing kernel, paths from {path0}, {name}")
        _check_paths(states[:, sl], tangents[:, :, sl], (xo, lpo, lmo), tan, f"tangent kernel, paths from {path0}")
