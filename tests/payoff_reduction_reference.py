"""Plain-numpy references for the Monte Carlo payoff reduction (csrc/mc_kernels.cu: spot_moments_kernel, payoff_vanilla_kernel,
payoff_kernel, reduce_partials_kernel, payoff_finalize_kernel) on hand-built terminal states.

Dyadic Q_VAR states (exact in any summation order)
  q = m 2^-12 (integer m in [0, 2^12)), ttm = 1/4, strikes k 2^-12 (integer k in [0, 2^14]), forward F a power of two.
  The underlying q / ttm = 4m 2^-12, so every C/P payoff is an integer multiple of 2^-12 below 4 and its square a multiple of 2^-24
  below 16; an IC/IP payoff is that divided by F.  For N <= 2^25 paths every partial sum of pay and pay^2 is an integer multiple of the
  unit below 2^53 units, hence exact in fp64 whatever the order: the device sums must equal the integer sums below bit for bit.
  Paths whose x is NaN do not count for IC/IP (pay / NaN) nor for the re-centring moments; every other x is 0, so the re-centred spot is
  F exp(0) - (F cnt / cnt - F) = F exactly.

Non-dyadic states: `sum_error_depth` bounds the depth of the kernels' summation trees, for gamma_k = k u / (1 - k u) error bounds.
"""
from fractions import Fraction
import math

import numpy as np

EPS = 2.0 ** -52
U = EPS / 2                     # unit round-off of fp64
UNIT = 2.0 ** -12               # grid of q and of the strikes
M_MAX = 1 << 12                 # q = m UNIT, m < M_MAX
K_MAX = 1 << 14                 # strike k UNIT <= 4
TTM = 0.25
CALL, PUT, INV_CALL, INV_PUT = 0, 1, 2, 3
LOG_RETURN, Q_VAR = 1, 2                # include/b200sv.h


def dyadic_states(n: int, seed: int, nan_every: int = 7, nan_phase: int = 3, m_max: int = M_MAX):
    """(m, x, q): m integer [n] in [0, m_max), x = 0 except NaN on paths i with i % nan_every == nan_phase (never path 0), q = m 2^-12.
    The first paths take m = 0 and m = m_max - 1 so the extremes of the range are always present."""
    rng = np.random.default_rng(seed)
    m = rng.integers(0, m_max, n, dtype=np.int64)
    m[: min(n, 2)] = [0, m_max - 1][: min(n, 2)]
    x = np.zeros(n)
    i = np.arange(n)
    x[(i % nan_every == nan_phase) & (i > 0)] = np.nan
    return m, x, m.astype(np.float64) * UNIT


def dyadic_strikes(J: int, seed: int):
    """(k integer [J] in [0, 2^14], types int8 [J] in {C, P}): k = 0 and k = 2^14 (an underlying of 0 / of 4 is never above / below it),
    multiples of 4 (ties with some path's underlying 4m) and random k in between."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, K_MAX + 1, J, dtype=np.int64)
    k[1::3] &= ~np.int64(3)                                     # k = 4m: the `>` / `<` ties
    k[: min(J, 2)] = [0, K_MAX][: min(J, 2)]
    types = rng.integers(0, 2, J).astype(np.int8)
    return k, types


def payoff_units(under_units: np.ndarray, k: np.ndarray, types: np.ndarray) -> np.ndarray:
    """[len(under_units), J] C/P payoffs in units of 2^-12 (IC/IP: before the division by the spot)"""
    u = under_units[:, None]
    put = (types[None, :] & 1).astype(bool)
    return np.where(put, np.maximum(k[None, :] - u, 0), np.maximum(u - k[None, :], 0))


def dyadic_sums(m: np.ndarray, x: np.ndarray, k: np.ndarray, types: np.ndarray, forward: float):
    """the exact per-strike (sum pay, sum pay^2, count) [3J] of the dyadic states, from integer arithmetic over the histogram of m"""
    assert math.frexp(forward)[0] == 0.5, "forward must be a power of two"
    valid = ~np.isnan(x)
    h_all = np.bincount(m, minlength=M_MAX).astype(np.int64)
    h_ok = np.bincount(m[valid], minlength=M_MAX).astype(np.int64)
    pay = payoff_units(4 * np.arange(M_MAX, dtype=np.int64), k, types)          # [M_MAX, J], < 2^14
    inv = types >= 2
    h = np.where(inv[None, :], h_ok[:, None], h_all[:, None])                   # IC/IP count only the non-NaN-x paths
    s1 = (h * pay).sum(axis=0)
    s2 = (h * pay * pay).sum(axis=0)
    cnt = h.sum(axis=0)
    assert s2.max(initial=0) < 2 ** 53
    out = np.empty(3 * len(k))
    scale = np.where(inv, 1.0 / forward, 1.0)
    out[0::3] = s1.astype(np.float64) * UNIT * scale
    out[1::3] = s2.astype(np.float64) * (UNIT * UNIT) * scale * scale
    out[2::3] = cnt.astype(np.float64)
    return out


def dyadic_pay_floats(m: np.ndarray, x: np.ndarray, k: np.ndarray, types: np.ndarray, forward: float):
    """[n, J] the per-path payoffs as floats, NaN where a path does not count (IC/IP on a NaN x), the way the general kernel forms them"""
    under = m.astype(np.float64) * UNIT / TTM
    spot = forward * np.exp(x)
    kk = k.astype(np.float64) * UNIT
    put = (types & 1).astype(bool)
    pay = np.where(put[None, :], np.where(under[:, None] < kk, kk - under[:, None], 0.0),
                   np.where(under[:, None] > kk, under[:, None] - kk, 0.0))
    return np.where((types >= 2)[None, :], pay / spot[:, None], pay)


def finalize_reference(sums: np.ndarray, discfactor: float, total_paths: int, d1=0.0, d2=0.0):
    """(prices, se, tol) for per-strike sums (s1, s2, cnt) [3J].

    prices = df (s1 / cnt) with the kernel's two IEEE operations.  se = df sqrt(V) / sqrt(N), V = max(s2/cnt - (s1/cnt)^2, 0) evaluated
    exactly (Fraction; V, its square root and the final quotient each rounded once: within 2u se).  tol bounds |se_kernel - se| when the
    kernel's s1, s2 are off by at most d1, d2 (per strike; 0 for exact sums) and it forms var = fl(fl(s2/cnt) - fl(fl(s1/cnt)^2)).  With
    A = s2/cnt, mean = s1/cnt, B = mean^2 and e1 = d1/cnt, the computed var is off by at most
        E = d2/cnt + u A + 2 |mean| e1 + e1^2 + 3u B + u V
    (to first order in u; contracting the subtraction into an fma only removes a rounding).  The clamp at 0 does not increase the error,
    |sqrt(v') - sqrt(V)| <= min(sqrt(E), E / sqrt(V)), and sqrt, the product with df and the quotient by sqrt(N) add 4u se, the reference's
    own rounding 2u se.  E is scaled by 1.01 for the second-order terms."""
    s1, s2, cnt = sums[0::3], sums[1::3], sums[2::3]
    with np.errstate(invalid="ignore", divide="ignore"):
        prices = np.float64(discfactor) * (s1 / cnt)
    se, tol = np.full(len(s1), np.nan), np.full(len(s1), np.nan)
    d1, d2 = np.broadcast_to(d1, s1.shape), np.broadcast_to(d2, s1.shape)
    for j in range(len(s1)):
        if not (np.isfinite(s1[j]) and np.isfinite(s2[j]) and cnt[j] > 0):
            continue
        mean = Fraction(s1[j]) / Fraction(cnt[j])
        A, B = Fraction(s2[j]) / Fraction(cnt[j]), mean * mean
        V = max(A - B, Fraction(0))
        se[j] = float(Fraction(discfactor) * Fraction(math.sqrt(V))) / math.sqrt(total_paths)
        e1 = d1[j] / cnt[j]
        E = 1.01 * (d2[j] / cnt[j] + U * float(A) + 2 * abs(float(mean)) * e1 + e1 * e1 + 3 * U * float(B) + U * float(V))
        d = math.sqrt(E) if V == 0 else min(math.sqrt(E), E / math.sqrt(V))
        tol[j] = abs(discfactor) * d / math.sqrt(total_paths) + 6 * U * se[j]
    return prices, se, tol


def sum_error_depth(n: int, sms: int, chunks: int, unroll: int = 1, threads: int = 256) -> int:
    """an upper bound on the number of additions any one payoff passes through in the kernels' fp64 sums: the per-thread grid-stride loop,
    the CTA's warp and cross-warp shuffle trees (5 + 3 levels), the lane loop of reduce_partials_kernel over the CTAs, and its warp tree.
    launch_payoff_t runs max(1, blocks / chunks) CTAs per chunk, blocks = min(ceil(n / (threads unroll)), sms x resident CTAs per SM), with
    1 <= resident <= 2048 / threads on an SM; so at least max(1, min(ceil(n / (threads unroll)), sms) // chunks) CTAs, at most 8 sms."""
    need = -(-n // (threads * unroll))
    min_blocks = max(1, min(need, sms) // chunks)
    max_blocks = max(1, min(need, sms * (2048 // threads)))
    loop = -(-n // (threads * min_blocks))
    return loop + 5 + 3 + -(-max_blocks // 32) + 5


def gamma(k: int) -> float:
    """gamma_k = k u / (1 - k u): the relative error bound of a sum of k additions of non-negative terms (Higham, Accuracy and Stability, 3.1)"""
    return k * U / (1.0 - k * U)


def exact_two_pass(pay: np.ndarray):
    """(mean, population variance) of the float payoffs, exactly, as Fractions: every fp64 value is an integer times 2^e"""
    mant, ex = np.frexp(pay)
    e0 = int(ex[pay != 0].min()) - 53
    ints = [int(v) for v in np.ldexp(mant, ex - e0)]       # pay = ints 2^e0 exactly: every mantissa has 53 bits, the scale makes it integral
    assert all(math.ldexp(a, e0) == p for a, p in zip(ints, pay.tolist()))
    n = len(ints)
    s1, s2 = sum(ints), sum(a * a for a in ints)
    scale = Fraction(2) ** e0
    mean = Fraction(s1, n) * scale
    var = (Fraction(s2, n) - Fraction(s1, n) ** 2) * scale * scale
    return mean, var


def negative_one_pass_constant(start: float = 0.03):
    """a payoff p >= start paid on each of three paths whose one-pass variance rounds below zero, contracted into an fma or not.
    Three equal terms (and exact zeros) sum to fl(3p) and fl(3 fl(p^2)) in every order, so the kernel's sums are known exactly:
    mean = fl(fl(3p)/3), A = fl(fl(3 fl(p^2))/3), and the exact variance is 0.  Returns the first such p on the grid start (1 + i 2^-20)."""
    for i in range(1 << 16):
        p = start * (1.0 + i * 2.0 ** -20)
        s1, s2 = 3.0 * p, 3.0 * (p * p)
        mean, A = s1 / 3.0, s2 / 3.0
        if A - mean * mean < 0.0 and Fraction(A) - Fraction(mean) ** 2 < 0:
            return p
    raise AssertionError("no such payoff")
