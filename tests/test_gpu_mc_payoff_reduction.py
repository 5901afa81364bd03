"""GPU: the Monte Carlo payoff reduction on hand-built terminal states -- spot_moments_kernel, payoff_vanilla_kernel<Real>,
payoff_kernel<Real>, reduce_partials_kernel and payoff_finalize_kernel -- through the host entry (engine.mc_payoffs) and the device entries
b200sv_dev_spot_moments / b200sv_dev_payoff_sums / b200sv_dev_payoff_finalize (the only way to the float-state kernels and to choose the
kernel: payoff_kinds_hint 1 = vanilla, 0 = general).

  A. dyadic Q_VAR states (tests/payoff_reduction_reference.py): sums exact in any order, so the device sums, the re-centring moments and the
     prices equal integer-arithmetic references bit for bit, at every strike-chunk count, across the persistent grid's stride / wave /
     unroll boundaries, in fp64 and fp32 state;
  B. LOG_RETURN states with NaN and -inf entries against math.fsum references within explicit bounds, and +inf against oracle/mc.py;
  C. the one-pass std error on low-spread payoffs, against the exact two-pass value, within its stated bound (DESIGN.md 3.5);
  D. one float state of more than 2^31 paths.
"""
import math

import numpy as np
import pytest

import payoff_reduction_reference as R
from oracle import mc

pytestmark = pytest.mark.gpu

F_DYADIC, DF_DYADIC = 2.0, 0.5
J_CHUNKS = [1, 7, 8, 9, 16, 17, 64, 201]
N_EDGES = [1, 2, 31, 33, 255, 257]


class Dev:
    """device buffers and the three device entries on torch's current stream"""

    def __init__(self):
        import torch
        from stochvolmodels_b200 import _capi as C
        self.torch, self.C = torch, C
        self.st = __import__("ctypes").c_void_p(torch.cuda.current_stream().cuda_stream)
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count

    def t(self, a, dtype=None):
        return self.torch.as_tensor(np.ascontiguousarray(a), device="cuda") if dtype is None else \
            self.torch.as_tensor(np.ascontiguousarray(a), device="cuda").to(dtype)

    @staticmethod
    def p(t):
        from ctypes import c_void_p
        return c_void_p(t.data_ptr())

    def moments(self, x64, n, forward):
        mom = self.torch.zeros(2, dtype=self.torch.float64, device="cuda")
        self.C.call("b200sv_dev_spot_moments", self.p(x64), int(n), float(forward), self.p(mom), self.st)
        return mom

    def sums(self, x, q, n, f32, ttm, forward, strikes, types, vt, hint, mom):
        J = strikes.shape[0]
        out = self.torch.full((3 * J,), np.nan, dtype=self.torch.float64, device="cuda")
        self.C.call("b200sv_dev_payoff_sums", self.p(x), self.p(q) if q is not None else None, int(n), int(self.C.STATE_F32 if f32 else 0),
                    float(ttm), float(forward), self.p(strikes), self.p(types), J, int(vt), int(hint), self.p(mom), self.p(out), None, self.st)
        return out

    def finalize(self, sums, df, n):
        J = sums.shape[0] // 3
        out = self.torch.full((2, J), np.nan, dtype=self.torch.float64, device="cuda")
        self.C.call("b200sv_dev_payoff_finalize", self.p(sums), J, float(df), int(n), self.p(out[0]), self.p(out[1]), None, self.st)
        self.torch.cuda.synchronize()
        return out[0].cpu().numpy(), out[1].cpu().numpy()


@pytest.fixture(scope="module")
def dev(cuda_lib):
    return Dev()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _assert_bits(got, ref, what):
    bad = np.nonzero(_bits(got) != _bits(ref))[0]
    assert bad.size == 0, (what, bad[:8], np.asarray(got)[bad[:8]], np.asarray(ref)[bad[:8]])


def _check_dyadic_final(prices, se, sums_ref, n, what):
    p_ref, se_ref, tol = R.finalize_reference(sums_ref, DF_DYADIC, n)
    _assert_bits(prices, p_ref, what + " prices")
    assert np.all(np.abs(se - se_ref) <= tol), (what, np.max(np.abs(se - se_ref) / tol))


def _interleave_inverse(types):
    """every other C/P code turned into its inverse: C -> IC, P -> IP"""
    t = types.copy()
    t[1::2] += 2
    return t


# ---- A. dyadic states -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("J", J_CHUNKS)
def test_dyadic_strike_chunks_bitwise(dev, J):
    """J strikes in ceil(J/8) chunks on gridDim.y, three forms of one slice: all C/P through the vanilla kernel, the same through the
    general kernel, and every other strike inverse (general kernel).  The device sums, moments and prices equal the integer reference bit for
    bit, so the three forms also agree with each other; the host entry engine.mc_payoffs agrees with them; two calls give the same bits."""
    from stochvolmodels_b200 import engine
    n = 40_000 + 3 * J
    m, x, q = R.dyadic_states(n, seed=J)
    k, types = R.dyadic_strikes(J, seed=100 + J)
    strikes = k.astype(np.float64) * R.UNIT
    xd, qd, kd = dev.t(x), dev.t(q), dev.t(strikes)
    mom = dev.moments(xd, n, F_DYADIC)
    cnt_ok = float(np.count_nonzero(~np.isnan(x)))
    _assert_bits(mom.cpu().numpy(), np.array([F_DYADIC * cnt_ok, cnt_ok]), "moments")
    cp_ref = None
    for form, (tys, hint) in {"vanilla": (types, 1), "general": (types, 0), "inverse": (_interleave_inverse(types), 0)}.items():
        ref = R.dyadic_sums(m, x, k, tys, F_DYADIC)
        td = dev.t(tys)
        s = dev.sums(xd, qd, n, False, R.TTM, F_DYADIC, kd, td, R.Q_VAR, hint, mom)
        s_host = s.cpu().numpy()
        _assert_bits(s_host, ref, f"J={J} {form} sums")
        _assert_bits(dev.sums(xd, qd, n, False, R.TTM, F_DYADIC, kd, td, R.Q_VAR, hint, mom).cpu().numpy(), s_host, "determinism")
        prices, se = dev.finalize(s, DF_DYADIC, n)
        _check_dyadic_final(prices, se, ref, n, f"J={J} {form}")
        cp = ~(tys >= 2).repeat(3)
        if cp_ref is None:
            cp_ref = s_host
        _assert_bits(s_host[cp], cp_ref[cp], "C/P strikes across forms")
        hp, hs = engine.mc_payoffs(x, q, R.TTM, F_DYADIC, strikes, np.array(["C", "P", "IC", "IP"])[tys], DF_DYADIC, R.Q_VAR)
        _assert_bits(hp, prices, f"J={J} {form} host prices")
        _assert_bits(hs, se, f"J={J} {form} host std errors")


def _sweep_ns(sms):
    ns = set(N_EDGES)
    for b in range(1, 9):
        for u in (1, 4):
            for d in (-1, 0, 1):
                ns.add(sms * b * 256 * u + d)
    return sorted(ns)


@pytest.mark.parametrize("f32", [False, True], ids=["f64", "f32"])
@pytest.mark.parametrize("J", [9, 17])
def test_dyadic_path_count_sweep(dev, J, f32):
    """N on both sides of sms b 256 u (b = 1..8 resident CTAs per SM, u = 1 or the vanilla kernel's 4-deep unroll) and tiny N: every
    one-wave cap, grid stride and unroll boundary the occupancy could pick.  Prefixes of one dyadic state, both kernels, fp64 and fp32
    state (m < 2^12: exact in float): sums, counts and prices bit for bit.  fp32 runs take the moments from the fp64 copy of x."""
    torch = dev.torch
    ns = _sweep_ns(dev.sms)
    n_max = ns[-1]
    m, x, q = R.dyadic_states(n_max, seed=7 + J)
    k, types = R.dyadic_strikes(J, seed=11 + J)
    kd, td = dev.t(k.astype(np.float64) * R.UNIT), dev.t(types)
    x64 = dev.t(x)
    xs, qs = (dev.t(x, torch.float32), dev.t(q, torch.float32)) if f32 else (x64, dev.t(q))
    for n in ns:
        mom = dev.moments(x64, n, F_DYADIC)
        cnt_ok = float(np.count_nonzero(~np.isnan(x[:n])))
        _assert_bits(mom.cpu().numpy(), np.array([F_DYADIC * cnt_ok, cnt_ok]), f"moments N={n}")
        ref = R.dyadic_sums(m[:n], x[:n], k, types, F_DYADIC)
        for hint in (1, 0):
            s = dev.sums(xs, qs, n, f32, R.TTM, F_DYADIC, kd, td, R.Q_VAR, hint, mom)
            _assert_bits(s.cpu().numpy(), ref, f"N={n} hint={hint} f32={f32} sums")
            prices, se = dev.finalize(s, DF_DYADIC, n)
            _check_dyadic_final(prices, se, ref, n, f"N={n} hint={hint}")


# ---- B. LOG_RETURN states ---------------------------------------------------------------------------------------------------------------
def _log_states(n, seed, sd):
    """x = -sd^2/2 + sd z (seeded z), with NaN on every 11th path and -inf on every 13th (never path 0)"""
    rng = np.random.default_rng(seed)
    x = -0.5 * sd * sd + sd * rng.standard_normal(n)
    i = np.arange(n)
    x[(i % 11 == 5)] = np.nan
    x[(i % 13 == 7)] = -np.inf
    return x


def _ulp(a):
    return np.spacing(np.abs(a))


def _log_reference(x, forward, strikes, types, depth_pay, depth_mom):
    """(sums [3J], d1 [J], d2 [J]) by math.fsum over the numpy spots and payoffs, and the bounds on |kernel sum - reference sum|:
      per path, |F exp(x)| is off by <= 3 ulp (CUDA's and numpy's exp each within 1 ulp, the product by F rounded once each);
      the re-centring corr = S/c - F by dS/c + ulp(S/c) + ulp(corr), dS = gamma_km sum F e^x + sum 3 ulp(F e^x) (km = depth_mom);
      the spot F e^x - corr by ds_i = 3 ulp(F e^x_i) + dcorr + ulp(spot_i);
      a C/P payoff is 1-Lipschitz in the spot: dpay_i = ds_i + ulp(pay_i); IC/IP h/s: (dh + |h/s| ds) / (|s| - ds) + ulp(h/s);
      d1 = sum dpay_i + gamma_k sum |pay_i| + ulp(s1), d2 = sum (2|pay_i| + dpay_i) dpay_i + ulp(pay_i^2) + gamma_k sum pay_i^2 + ulp(s2),
    k = depth_pay, the depth of the kernel's summation tree (payoff_reduction_reference.sum_error_depth)."""
    fe = forward * np.exp(x)
    ok = ~np.isnan(fe)
    S, c = math.fsum(fe[ok]), int(ok.sum())
    corr = S / c - forward
    spot = fe - corr
    dS = R.gamma(depth_mom) * math.fsum(np.abs(fe[ok])) + math.fsum(3 * _ulp(fe[ok]))
    dcorr = dS / c + _ulp(S / c) + _ulp(corr)
    with np.errstate(invalid="ignore"):
        ds = np.where(ok, 3 * _ulp(fe) + dcorr + _ulp(spot), 0.0)       # a NaN-x path pays exactly 0 (C/P) or does not count (IC/IP)
    J = len(strikes)
    sums, d1, d2 = np.empty(3 * J), np.empty(J), np.empty(J)
    g = R.gamma(depth_pay)
    for j in range(J):
        kk, ty = strikes[j], types[j]
        with np.errstate(invalid="ignore", divide="ignore"):
            h = np.where(spot > kk, spot - kk, 0.0) if ty % 2 == 0 else np.where(spot < kk, kk - spot, 0.0)
            dh = ds + _ulp(h)
            if ty >= 2:
                pay = h / spot
                room = np.abs(spot) - ds
                dp = np.where(room > 0, (dh + np.abs(pay) * ds) / room, np.inf) + _ulp(pay)
            else:
                pay, dp = h, dh
        use = ~np.isnan(pay)
        p, e = pay[use], dp[use]
        sums[3 * j: 3 * j + 3] = math.fsum(p), math.fsum(p * p), float(use.sum())
        d1[j] = math.fsum(e) + g * math.fsum(np.abs(p)) + _ulp(sums[3 * j])
        d2[j] = math.fsum((2 * np.abs(p) + e) * e + _ulp(p * p)) + g * math.fsum(p * p) + _ulp(sums[3 * j + 1])
    return sums, d1, d2


def _log_strikes(x, forward, J, seed):
    """deep ITM to deep OTM around the forward, a third of them equal to some path's spot F e^x (the `>` / `<` ties), codes C P IC IP"""
    rng = np.random.default_rng(seed)
    fe = forward * np.exp(x[np.isfinite(x)])
    ks = forward * np.exp(rng.uniform(-3.0, 3.0, J))
    ks[::3] = fe[rng.integers(0, fe.size, ks[::3].size)]
    ks[: min(J, 2)] = [forward * 1e-3, forward * 1e3][: min(J, 2)]
    return ks, np.arange(J, dtype=np.int8) % 4


@pytest.mark.parametrize("sd", [0.01, 0.3, 2.0])
@pytest.mark.parametrize("J", [1, 9, 17, 64])
def test_log_return_against_fsum(dev, J, sd):
    """LOG_RETURN slices with NaN and -inf log-spots (a -inf path has spot F e^x = 0, re-centred to -corr; a NaN one pays 0 for C/P and
    does not count for IC/IP nor for the moments), strikes deep ITM to deep OTM and on path spots, codes C P IC IP.  Each N runs the host
    entry, the general kernel and, on the C/P-only slice, the vanilla kernel; counts must be exact, sums / prices / std errors within the
    bounds of _log_reference and payoff_reduction_reference.finalize_reference.  Two calls give the same bits."""
    from stochvolmodels_b200 import engine
    forward, df = 1.3, 0.97
    sms = dev.sms
    ns = [1, 33, 257, sms * 256 - 1, sms * 256 * 4 + 1] + ([sms * 8 * 256 * 4 + 1] if J <= 9 else [])     # the fsum reference costs J N
    x_all = _log_states(ns[-1], seed=int(1000 * sd) + J, sd=sd)
    x_all[0] = 0.0
    ks, types = _log_strikes(x_all, forward, J, seed=J)
    cp_types = types % 2
    kd = dev.t(ks)
    names = np.array(["C", "P", "IC", "IP"])
    for n in ns:
        x = x_all[:n]
        xd = dev.t(x)
        mom = dev.moments(xd, n, forward)
        depth_mom = R.sum_error_depth(n, sms, 1)
        for tys, hints in ((types, (0,)), (cp_types, (0, 1))):
            chunks = -(-J // 8)
            sums_ref, d1, d2 = _log_reference(x, forward, ks, tys, R.sum_error_depth(n, sms, chunks), depth_mom)
            td = dev.t(tys)
            runs = {}
            for hint in hints:
                s = dev.sums(xd, None, n, False, 1.0, forward, kd, td, R.LOG_RETURN, hint, mom)
                s2 = dev.sums(xd, None, n, False, 1.0, forward, kd, td, R.LOG_RETURN, hint, mom)
                _assert_bits(s2.cpu().numpy(), s.cpu().numpy(), "determinism")
                runs[f"hint {hint}"] = (s.cpu().numpy(), *dev.finalize(s, df, n))
            hp, hs = engine.mc_payoffs(x, None, 1.0, forward, ks, names[tys], df, R.LOG_RETURN)
            runs["host"] = (None, hp, hs)
            p_ref, se_ref, se_tol = R.finalize_reference(sums_ref, df, n, d1, d2)
            cnt = sums_ref[2::3]
            for what, (s, prices, se) in runs.items():
                tag = f"N={n} J={J} sd={sd} {what}"
                if s is not None:
                    _assert_bits(s[2::3], cnt, tag + " counts")
                    assert np.all(np.abs(s[0::3] - sums_ref[0::3]) <= d1), (tag, np.max(np.abs(s[0::3] - sums_ref[0::3]) / d1))
                    assert np.all(np.abs(s[1::3] - sums_ref[1::3]) <= d2), (tag, np.max(np.abs(s[1::3] - sums_ref[1::3]) / d2))
                p_tol = df * d1 / cnt + 2 * R.U * np.abs(p_ref)
                assert np.all(np.abs(prices - p_ref) <= p_tol), (tag, np.max(np.abs(prices - p_ref) / p_tol))
                assert np.all(np.abs(se - se_ref) <= se_tol), (tag, np.max(np.abs(se - se_ref) / se_tol))
            o_p, o_s = mc.mc_payoffs(x, None, 1.0, forward, ks, names[tys], df)
            scale = np.max(np.abs(o_p))
            assert np.allclose(hp, o_p, rtol=1e-9, atol=1e-12 * scale) and np.allclose(hs, o_s, rtol=1e-6, atol=1e-12 * scale), (n, J, sd)


@pytest.mark.parametrize("n", [2, 33, 257, 70_001])
def test_positive_infinite_log_spot_matches_oracle(dev, n):
    """one x = +inf makes the nan-mean infinite: every finite path's re-centred spot is -inf, the +inf path's inf - inf = NaN.  Calls pay 0,
    puts +inf (std error NaN, as np.nanstd), inverse calls -0, inverse puts inf / -inf = NaN on every path (price and std error NaN).  The
    host entry and both device kernels reproduce oracle/mc.py::mc_payoffs NaN for NaN and inf for inf."""
    from stochvolmodels_b200 import engine
    x = _log_states(n, seed=n, sd=0.2)
    x[n // 2] = np.inf
    ks = np.array([0.5, 1.0, 2.0, 0.5, 1.0, 2.0, 0.5, 1.0, 2.0, 0.5, 1.0, 2.0])
    types = np.repeat(np.arange(4, dtype=np.int8), 3)
    names = np.array(["C", "P", "IC", "IP"])[types]
    with np.errstate(invalid="ignore", divide="ignore"), pytest.warns(RuntimeWarning):
        o_p, o_s = mc.mc_payoffs(x, None, 1.0, 1.0, ks, names, 1.0)
    assert np.isposinf(o_p[3:6]).all() and np.isnan(o_s[3:6]).all() and np.isnan(o_p[9:]).all()
    hp, hs = engine.mc_payoffs(x, None, 1.0, 1.0, ks, names, 1.0, R.LOG_RETURN)
    np.testing.assert_array_equal(hp, o_p)
    np.testing.assert_array_equal(hs, o_s)
    xd = dev.t(x)
    mom = dev.moments(xd, n, 1.0)
    for sel, hint in ((slice(0, 6), 1), (slice(0, 6), 0), (slice(0, 12), 0)):
        s = dev.sums(xd, None, n, False, 1.0, 1.0, dev.t(ks[sel]), dev.t(types[sel]), R.LOG_RETURN, hint, mom)
        p, e = dev.finalize(s, 1.0, n)
        np.testing.assert_array_equal(p, o_p[sel])
        np.testing.assert_array_equal(e, o_s[sel])


# ---- C. the std-error floor ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1e-4, 1e-6, 1e-8])
def test_low_spread_std_error_within_one_pass_bound(dev, r):
    """Q_VAR states at 0.04 ttm (1 + r z), a deep-ITM call (K = 0.01), N = sms 8 1024 + 1, both kernels.  The kernel's std error is the
    one-pass df sqrt(s2/cnt - mean^2) / sqrt(N).  Its sums carry a relative error <= gamma_k (pay > 0, k = sum_error_depth), its variance
    E <= (g + u) A + (2g + 3u) B + u V with A = s2/cnt, B = mean^2 <= A, V = A - B (payoff_reduction_reference.finalize_reference), so
        E <= (3 gamma_k + 4u) A = c eps A,   c = 2 + 3 gamma_k / eps  (~ 1.5 k + 2),
    and |se - se_two_pass| <= df sqrt(c eps s2/cnt) / sqrt(N) + 6u se: when the spread is below sqrt(c eps) of the level the one-pass
    value carries no digit of the two-pass one.  The exact two-pass value comes from the payoffs' exact binary values (Fraction)."""
    torch = dev.torch
    ttm, K, df = R.TTM, 0.01, 0.9
    n = dev.sms * 8 * 1024 + 1
    rng = np.random.default_rng(int(-math.log10(r)))
    q = 0.04 * ttm * (1.0 + r * rng.standard_normal(n))
    pay = q / ttm - K                                       # both kernels form exactly this: q / 0.25 and q * 4 are exact
    mean, var = R.exact_two_pass(pay)
    se_exact = df * math.sqrt(var) / math.sqrt(n)
    qd, kd, td = dev.t(q), dev.t(np.array([K])), dev.t(np.array([R.CALL], dtype=np.int8))
    mom = torch.tensor([1.0, 1.0], dtype=torch.float64, device="cuda")
    for hint in (1, 0):
        k = R.sum_error_depth(n, dev.sms, 1, unroll=4 if hint == 1 else 1)
        c = 2.0 + 3.0 * R.gamma(k) / R.EPS
        s = dev.sums(qd, qd, n, False, ttm, 1.0, kd, td, R.Q_VAR, hint, mom)
        p, se = dev.finalize(s, df, n)
        A = float(s[1].item()) / n
        bound = df * math.sqrt(c * R.EPS * A) / math.sqrt(n) + 6 * R.U * se_exact
        print(f"r={r:g} hint={hint}: se={se[0]:.6e} exact two-pass={se_exact:.6e} |diff|={abs(se[0] - se_exact):.2e} bound={bound:.2e} (c={c:.1f})")
        assert abs(se[0] - se_exact) <= bound
        assert abs(p[0] - df * float(mean)) <= df * R.gamma(k) * float(mean) + 2 * R.U * abs(p[0])


@pytest.mark.parametrize("hint", [1, 0])
def test_negative_one_pass_variance_clamped(dev, hint):
    """three paths paying one constant p for which fl(fl(s2/3) - fl(fl(s1/3)^2)) < 0 (checked on the host, with and without fma
    contraction; three equal terms sum the same in every order): the clamp at zero gives a std error of exactly 0, not NaN."""
    p = R.negative_one_pass_constant()
    q = np.full(3, p * R.TTM)
    assert q[0] / R.TTM == p
    qd = dev.t(q)
    mom = dev.torch.tensor([1.0, 1.0], dtype=dev.torch.float64, device="cuda")
    s = dev.sums(qd, qd, 3, False, R.TTM, 1.0, dev.t(np.array([0.0])), dev.t(np.array([R.CALL], dtype=np.int8)), R.Q_VAR, hint, mom)
    _assert_bits(s.cpu().numpy(), np.array([3.0 * p, 3.0 * (p * p), 3.0]), "constant sums")
    prices, se = dev.finalize(s, 1.0, 3)
    assert prices[0] == (3.0 * p) / 3.0 and se[0] == 0.0, (prices, se)


# ---- D. beyond 2^31 paths -----------------------------------------------------------------------------------------------------------
def test_float_state_beyond_2_pow_31_paths(dev):
    """N = 2^31 + 2^20 + 1 float paths (8.6 GB), a period-256 dyadic pattern q = m 2^-8 (m < 2^8) passed as both x and qvar, hand-made
    moments (1, 1), ttm = 1/4: payoffs are multiples of 2^-8 below 4, their squares of 2^-16 below 16, so every sum is below 2^53 units
    and exact in any order.  Both kernels equal the closed-form sums (full periods plus the remainder) bit for bit, and the vanilla kernel's
    arithmetic count is exactly N."""
    torch = dev.torch
    free, _ = torch.cuda.mem_get_info()
    if free < 12e9:
        pytest.skip(f"needs 12 GB of free device memory, {free / 1e9:.1f} GB free")
    n = 2 ** 31 + 2 ** 20 + 1
    m = (np.arange(256, dtype=np.int64) * 167 + 13) % 256
    k = np.array([0, 1024, 17, 300, 512, 513, 768, 999, 5], dtype=np.int64)        # strikes k 2^-8 in [0, 4]
    types = np.array([0, 1, 0, 1, 0, 1, 1, 0, 1], dtype=np.int8)
    under = 4 * m                                                                      # q / ttm in units of 2^-8
    pay = np.where(types[None, :] == 1, np.maximum(k[None, :] - under[:, None], 0), np.maximum(under[:, None] - k[None, :], 0))
    full, rem = divmod(n, 256)
    ref = np.empty(3 * len(k))
    for j in range(len(k)):
        col = [int(v) for v in pay[:, j]]
        s1 = full * sum(col) + sum(col[:rem])
        s2 = full * sum(v * v for v in col) + sum(v * v for v in col[:rem])
        assert s2 < 2 ** 53
        ref[3 * j: 3 * j + 3] = s1 * 2.0 ** -8, s2 * 2.0 ** -16, float(n)
    state = torch.tensor(m.astype(np.float32) * np.float32(2.0 ** -8), device="cuda").repeat(full + 1)[:n]
    try:
        mom = torch.tensor([1.0, 1.0], dtype=torch.float64, device="cuda")
        kd, td = dev.t(k.astype(np.float64) * 2.0 ** -8), dev.t(types)
        for hint in (1, 0):
            s = dev.sums(state, state, n, True, R.TTM, 1.0, kd, td, R.Q_VAR, hint, mom).cpu().numpy()
            _assert_bits(s, ref, f"N = 2^31 + 2^20 + 1, hint {hint}")
    finally:
        del state
        torch.cuda.empty_cache()
