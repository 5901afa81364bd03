"""GPU: the Fourier kernels against the high-precision references of tests/fourier_edges_reference.py, at the parameters, grid lengths and
non-finite inputs the reference goldens never reach.

  - heston_mgf_kernel (HestonClosedForm) through engine.heston_mgf_grid, (a, b) carried over one and three maturities: every a, b and
    log-MGF within its per-point bar of the 50-digit evaluation, at rho in {-0.999, 0, 0.95}, volvol in {0.01, 0.3, 5}, kappa in
    {0.01, 2, 50}, Feller badly violated, tau in {1e-4, 1, 30}, phi from Im 0 (and one denormal ulp) to 1e4, and psi != 0;
  - the strike sums (fourier_vanilla_kernel, fourier_gamma_batch_kernel, fourier_sum_kernel) through engine.fourier_vanilla / _gamma /
    _qvar / _pdf_sums / _digital at P from 3 to 2^20 + 1 (both sides of every 256-thread stride), J = 1, 7 and 70 000 strikes, x = ln F/K
    in {0, +-1e-12, +-5, +-30}, and log-MGF entries NaN, +inf, -inf, 700 + iy at j = 0, 255, 256, P - 1: NaN / +-inf exactly where numpy
    has them, finite outputs within the bar of the exact sum;
  - the launch-size paths of the ODE kernels against the numpy RK45 clones: the LogSV lane kernel (P = 8192) and thread kernel
    (P = 8193), both orders, and the Hawkes and Heston grids at every block size mgf_block_threads can pick, with a ragged tail;
  - the tangent and Hessian kernels (HestonClosedForm over dcd / hcd) through engine.heston_price_chain_greeks / _hessian: dlog_mgf and
    d2log_mgf against mp.diff of the 50-digit closed form at six parameter extremes, on grids reaching Im phi = 1e4 with odd max_phi.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

pytest.importorskip("mpmath")

import fourier_edges_reference as R  # noqa: E402


def _heston_device(par, taus, phi, psi):
    from stochvolmodels_b200 import engine
    hp = engine.heston_params_c(*par)
    a, b = np.zeros_like(phi), np.zeros_like(phi)
    out = []
    for tau in taus:
        lm, a, b = engine.heston_mgf_grid(phi, psi, tau, a, b, hp)
        out.append(np.stack([a, b, lm], axis=-1))
    return np.stack(out)


def test_heston_closed_form_against_mpmath(cuda_lib):
    worst = {}
    for c in R.heston_cases():
        got = _heston_device(c["par"], c["taus"], c["phi"], c["psi"])
        want = R.heston_numpy(c["par"], c["taus"], c["phi"], c["psi"])
        nf = ~np.isfinite(want)
        mm = R.nonfinite_mismatch(got[nf], want[nf])
        assert mm.size == 0, (c["name"], got[nf][mm], want[nf][mm])
        r = np.where(nf, 0.0, R.heston_ratio(got, c))
        key = "psi" if "psi" in c["name"] else f"M={len(c['taus'])}"
        worst[key] = max(worst.get(key, 0.0), float(r.max()))
        i = np.unravel_index(np.argmax(r), r.shape)
        assert r.max() <= 1.0, (c["name"], i, c["phi"][i[1]], c["psi"][i[1]], got[i], c["exact"][i], c["bar"][i])
    print("closed form, max err / bar: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


def _sums_device(c):
    from stochvolmodels_b200 import engine
    name, args = c["call"]
    return getattr(engine, name)(*args)


def test_strike_sums_against_the_exact_sums(cuda_lib):
    worst = {}
    for c in R.sum_cases():
        got = _sums_device(c)
        mm = R.nonfinite_mismatch(got, c["numpy"])
        assert mm.size == 0, (R.case_name(c), mm[:5], got[mm[:5]], c["numpy"][mm[:5]])
        r = R.bar_ratio(got, c["exact"], c["bar"])
        worst[c["kind"]] = max(worst.get(c["kind"], 0.0), float(r.max()))
        assert r.max() <= 1.0, (R.case_name(c), int(np.argmax(r)), r.max())
    print("strike sums, max err / bar: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


def test_overflowing_term_at_grid_point_zero_is_kept(cuda_lib):
    """Im phi_0 = 0: exp(700 + 30 / 2) = +inf times a real weight is +inf (C99 cexp, numpy), which np.nansum keeps -- the call priced on it
    is -inf, not a finite price that silently lacks the term"""
    from stochvolmodels_b200 import engine
    P = 513
    phi = R.grid(-0.5, R.STOP, P)
    lm = R.constructed(R.heston_lm(phi), "700", 0)
    Ks = R.strikes_for((30.0, 0.0))
    got = engine.fourier_vanilla(lm, phi, 1.0, Ks, ["C", "C"], 1.0, True)
    want = R.vanilla_reference(lm, phi, 1.0, Ks, ["C", "C"], 1.0, True)[0]
    assert np.isneginf(want[0]) and np.isneginf(got[0]), got
    assert np.isfinite(got[1]) and abs(got[1] - want[1]) <= 1e-12 * abs(want[1])


# ---- launch-size paths of the ODE kernels -------------------------------------------------------------------------------------------
LOGSV = (1.0, 1.0, 5.0, 5.0, 0.2, 2.0)       # sigma0, theta, kappa1, kappa2, beta, volvol (the quickstart set)
HAWKES = [0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5]
HAWKES_KEYS = ("mu", "sigma", "shift_p", "mean_p", "shift_m", "mean_m", "lambda_p", "theta_p", "kappa_p", "beta1_p", "beta2_p",
               "lambda_m", "theta_m", "kappa_m", "beta1_m", "beta2_m")


def _parity(name, got, want):
    d = float(np.max(np.abs(got - want) / (1.0 + np.abs(want))))
    print(f"{name}: max |gpu - numpy| / (1 + |numpy|) = {d:.3g}")
    assert d <= 1e-12, (name, d)
    return d


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("order", [2, 1])
def test_logsv_lane_and_thread_kernels_against_numpy(cuda_lib, order):
    """P = 8192 runs the lane-parallel kernel, P = 8193 the thread-per-point one; both against the RK45 clone, and against each other on
    the shared first 8192 points"""
    from oracle import mgf
    from stochvolmodels_b200 import engine
    n = 3 if order == 1 else 5
    phi = R.grid(-0.5, 5.6 / 0.2, 8193)
    res = {}
    for P in (8192, 8193):
        ph = phi[:P]
        a, lm = engine.logsv_mgf_grid(ph, None, 0.25, np.zeros((P, n), complex), engine.logsv_params_c(*LOGSV), 1.0, True, order)
        a_np, lm_np = mgf.logsv_a_mgf_grid(0.25, ph, np.zeros_like(ph), np.zeros((P, n), complex), *LOGSV, True, order)
        _parity(f"logsv order {order} P={P} a", a, a_np)
        _parity(f"logsv order {order} P={P} log_mgf", lm, lm_np)
        res[P] = lm
    _parity(f"logsv order {order} lane vs thread", res[8192], res[8193][:8192])


def test_hawkes_and_heston_grids_at_every_block_size(cuda_lib):
    """P = 4S, 4S + 1, 8S + 1, 16S + 1, 32S + 1, 64S + 7 (S = SM count) reach every block size 4 .. 64 of mgf_block_threads, with a
    ragged last block"""
    from oracle import hawkes, mgf
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200 import engine
    S = _sm_count()
    kp, pd = C.HawkesParamsC(*HAWKES), dict(zip(HAWKES_KEYS, HAWKES))
    v0, theta, kappa, rho, volvol = R.SUM_PAR
    for P in (4 * S, 4 * S + 1, 8 * S + 1, 16 * S + 1, 32 * S + 1, 64 * S + 7):
        phi = R.grid(-0.5, 5.6 / 0.1, P)
        a = np.zeros((P, 3), complex)
        lm = engine.hawkesjd_mgf_grid(phi, np.zeros_like(phi), 0.25, a, kp)
        a_np, lm_np = hawkes.a_mgf_grid(0.25, phi, pd)
        _parity(f"hawkes P={P} a", a, a_np)
        _parity(f"hawkes P={P} log_mgf", lm, lm_np)
        lm, ah, bh = engine.heston_mgf_grid(phi, None, 0.5, None, None, engine.heston_params_c(*R.SUM_PAR))
        lm_np, a_np, b_np = mgf.heston_mgf_grid(v0, theta, kappa, volvol, rho, 0.5, phi, np.zeros_like(phi))
        _parity(f"heston P={P} log_mgf", lm, lm_np)
        _parity(f"heston P={P} b", bh, b_np)


# ---- tangent and Hessian kernels of the Heston chain pricer ---------------------------------------------------------------------------
def test_heston_tangent_and_hessian_kernels_against_mp_diff(cuda_lib):
    """dlog_mgf of heston_price_chain_greeks and dlog_mgf / d2log_mgf of heston_price_chain_hessian (HestonClosedForm over dcd / hcd)
    against mp.diff of the 50-digit closed form, on the pricers' own grids: Im phi up to 1e4 through a small vol_scaler, odd max_phi"""
    from stochvolmodels_b200 import engine
    K, T = np.array([0.9, 1.0, 1.1]), np.array(["P", "C", "C"])
    ttms = np.array(R.DERIV_TTMS)
    fw, df = np.ones(len(ttms)), np.ones(len(ttms))
    worst = {"greeks d1": 0.0, "hessian d1": 0.0, "hessian d2": 0.0}
    for c in R.heston_deriv_cases():
        hp = engine.heston_params_c(*c["par"])
        args = (hp, ttms, fw, df, [K] * len(ttms), [T] * len(ttms), c["vol_scaler"], c["max_phi"], True)
        dlm_g = engine.heston_price_chain_greeks(*args)[3]
        dlm_h, d2lm_h = engine.heston_price_chain_hessian(*args)[5:7]
        for key, got, want, bar in (("greeks d1", dlm_g, c["d1"], c["bar1"]), ("hessian d1", dlm_h, c["d1"], c["bar1"]),
                                    ("hessian d2", d2lm_h, c["d2"], c["bar2"])):
            r = R.bar_ratio(got, want, bar)
            worst[key] = max(worst[key], float(r.max()))
            i = np.unravel_index(np.argmax(r), r.shape)
            assert r.max() <= 1.0, (c["name"], key, i, got[i], want[i], bar[i])
    print("tangent / Hessian kernels, max err / bar: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
