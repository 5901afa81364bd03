"""CPU: the numpy restatement of the Hawkes Monte Carlo sensitivities (oracle/hawkes_mc_greeks.py) against central differences of the
oracle's own scheme on fixed draws -- pathwise tangents on paths whose firing decisions do not flip, and the full estimator (score
included) against CRN differences of the expected price -- and the argument checks of HawkesJDPricer.model_mc_chain_greeks (they raise
before any library call)."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import hawkes
from oracle import hawkes_mc_greeks as hg

K5 = np.array([0.9, 0.97, 1.0, 1.03, 1.1])
T5 = np.array(["P", "IP", "C", "IC", "C"])


def _golden_params(name):
    return dict(zip(hawkes.KEYS, load_golden("hawkes_mc.npz")[f"{name}_params"]))


def _draws(params, ttm, n, seed):
    return hawkes.draw_inputs(np.random.RandomState(seed), ttm, n, params["shift_p"], params["mean_p"], params["shift_m"], params["mean_m"])


def _bumped(params, name, eps):
    p = dict(params)
    p[name] += eps
    return p


def _run(params, blk, n, return_fires=False):
    kw = {k: v for k, v in params.items() if k not in ("lambda_p", "lambda_m")}
    x0, lp0, lm0 = np.zeros(n), params["lambda_p"] * np.ones(n), params["lambda_m"] * np.ones(n)
    return hg.tangent_step_fixed(x0, lp0, lm0, *hg.initial_tangents(n), *blk, return_fires=return_fires, **kw)


@pytest.mark.parametrize("name", ["dflt", "drift"])
def test_pathwise_tangents_match_central_differences_where_no_decision_flips(name):
    """fixed draws: d(x, lambda_p, lambda_m) / d p of the oracle's scheme by central differences == the frozen-decision tangents, on the
    paths whose firing decisions are the same at p - eps, p and p + eps, for all 15 directions"""
    params = _golden_params(name)
    n = 3000
    blk = _draws(params, 0.05, n, 11)
    x, lp, lm, dx, dlp, dlm, score, fires = _run(params, blk, n, return_fires=True)
    xs, lps, lms = hawkes.step_fixed(np.zeros(n), params["lambda_p"] * np.ones(n), params["lambda_m"] * np.ones(n), *blk, **params)
    for a, b in zip((x, lp, lm), (xs, lps, lms)):
        np.testing.assert_array_equal(a, b)            # the tangent restatement leaves the state to oracle.hawkes.step_fixed
    assert fires[:, 0].any(axis=0).sum() > 100 and fires[:, 1].any(axis=0).sum() > 100
    for q, p in enumerate(hg.PARAMS):
        eps = 1e-6 * max(abs(params[p]), 1e-2)
        bu, bd = _bumped(params, p, eps), _bumped(params, p, -eps)
        up, dn = _run(bu, _draws(bu, 0.05, n, 11), n, True), _run(bd, _draws(bd, 0.05, n, 11), n, True)   # the sizes follow shift / mean
        keep = np.all(up[7] == fires, axis=(0, 1)) & np.all(dn[7] == fires, axis=(0, 1))
        assert keep.sum() > 0.95 * n, (p, keep.sum())
        for t, a, b, what in zip((dx, dlp, dlm), up[:3], dn[:3], ("x", "lambda_p", "lambda_m")):
            fd = (a - b)[keep] / (2 * eps)
            scale = max(float(np.max(np.abs(fd))), float(np.max(np.abs(t[q][keep]))), 1e-300)
            assert np.max(np.abs(t[q][keep] - fd)) <= 1e-7 * scale, (p, what, np.max(np.abs(t[q][keep] - fd)) / scale)


def _fd_step(params, p):
    return 0.02 * max(abs(params[p]), 0.05)


@pytest.mark.parametrize("name", ["dflt", "drift"])
def test_estimator_matches_crn_differences_of_the_expected_price(name):
    """pathwise + score estimator vs CRN central differences of the oracle's price (same draws at p +- h, decisions free to flip): within
    4 combined standard errors, the difference's SE from its per-path values; delta by bumping the forward"""
    params = _golden_params(name)
    n, ttm, fwd, df = 200_000, 0.02, 1.0, 0.999
    blk = _draws(params, ttm, n, 5)
    p_, e_, g, gse, paths = hg.chain_greeks_fixed(params, [ttm], [fwd], [df], [K5], [T5], [blk], return_paths=True)
    po, eo = hawkes.chain_prices(params, [ttm], [fwd], [df], [K5], [T5], n, inputs=[blk])
    np.testing.assert_allclose(p_[0], po[0], rtol=1e-13)
    np.testing.assert_allclose(e_[0], eo[0], rtol=1e-12)
    x = paths[0][0]

    def per_path(xv, f):
        fe = f * np.exp(xv)
        s = fe - (np.mean(fe) - f)
        cols = []
        for k, ty in zip(K5, T5):
            h = np.maximum(k - s, 0.0) if ty in ("P", "IP") else np.maximum(s - k, 0.0)
            cols.append(df * (h / s if ty in ("IC", "IP") else h))
        return np.array(cols)

    def check(row, fd_paths, what):
        fd, fd_se = fd_paths.mean(axis=1), fd_paths.std(axis=1) / np.sqrt(n)
        z = np.abs(g[0][row] - fd) / np.sqrt(gse[0][row] ** 2 + fd_se ** 2)
        assert np.all(z < 4.0), (what, g[0][row], fd, gse[0][row], fd_se)

    hf = 1e-4
    check(0, (per_path(x, fwd * (1 + hf)) - per_path(x, fwd * (1 - hf))) / (2 * hf * fwd), "delta")
    for q, p in enumerate(hg.PARAMS):
        h = _fd_step(params, p)
        xs = []
        for s in (1.0, -1.0):
            b = _bumped(params, p, s * h)
            blk_b = _draws(b, ttm, n, 5)            # same uniforms / normals: the jump sizes follow shift and mean
            xs.append(hawkes.step_fixed(np.zeros(n), b["lambda_p"] * np.ones(n), b["lambda_m"] * np.ones(n), *blk_b, **b)[0])
        check(1 + q, (per_path(xs[0], fwd) - per_path(xs[1], fwd)) / (2 * h), p)


# ---- argument checks: nothing reaches the library ------------------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from stochvolmodels_b200 import _capi

    def forbidden(*a, **k):
        raise AssertionError("library called")
    monkeypatch.setattr(_capi, "call", forbidden)
    monkeypatch.setattr(_capi, "load_library", forbidden)


@pytest.mark.parametrize("kwargs", [dict(precision="fp32"), dict(exchange="p2p"), dict(exchange="nccl"), dict(gauss="fp64_paired"),
                                    dict(gauss="fp16"), dict(variable_type="Q_VAR"), dict(risk_premia_gamma=0.5)])
def test_hawkes_mc_greeks_rejections_raise_before_the_library(no_library, kwargs):
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain
    from stochvolmodels_b200.utils.config import VariableType
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[T5])
    kwargs = dict(kwargs)
    params = HawkesJDParams(risk_premia_gamma=kwargs.pop("risk_premia_gamma", None))
    if "variable_type" in kwargs:
        kwargs["variable_type"] = VariableType.Q_VAR
    with pytest.raises(NotImplementedError):
        HawkesJDPricer().model_mc_chain_greeks(chain, params, nb_path=1000, seed=1, **kwargs)


@pytest.mark.parametrize("field", ["mean_p", "mean_m"])
def test_degenerate_jump_size_raises_before_the_library(no_library, field):
    """dJ/dmean is the jump's unit exponential (J - shift) / mean: undefined at mean = 0, so that is refused rather than returning NaN rows"""
    from stochvolmodels_b200 import HawkesJDParams, HawkesJDPricer, OptionChain
    chain = OptionChain(ttms=np.array([0.25]), forwards=np.ones(1), strikes_ttms=[K5], optiontypes_ttms=[T5])
    with pytest.raises(ValueError, match="mean_p != 0 and mean_m != 0"):
        HawkesJDPricer().model_mc_chain_greeks(chain, HawkesJDParams(**{field: 0.0}), nb_path=1000, seed=1)


@pytest.mark.parametrize("field", ["mean_p", "mean_m"])
def test_library_refuses_a_degenerate_jump_size_before_any_stream_work(field):
    """the C entry point returns its own error for mean = 0 (needs the library, no GPU: the check runs before the first stream operation)"""
    import ctypes
    from stochvolmodels_b200 import HawkesJDParams
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200.pricers.hawkes_jd_pricer import _params_c
    d = {k: v for k, v in HawkesJDParams(**{field: 0.0}).to_dict().items() if k in hawkes.KEYS}
    lib = C.load_library()
    out = np.zeros(64)
    keep = [C.f64([0.25]), C.f64([1.0]), C.f64(K5)]
    rc = lib.b200sv_hawkesjd_mc_chain_greeks(ctypes.byref(_params_c(**d)), 1, C.dptr(keep[0]), C.dptr(keep[1]), C.dptr(keep[1]),
                                             C.iptr(np.array([0, 5], dtype=np.int32)), C.dptr(keep[2]), C.i8ptr(np.array([1, 1, 0, 0, 0], dtype=np.int8)),
                                             16, C.LOG_RETURN, 0, 0, C.dptr(out), C.dptr(out), C.dptr(out), C.dptr(out), 0, None, None)
    assert (rc, lib.b200sv_last_error().decode()) == (-1, "invalid argument: the Hawkes sensitivities need mean_p != 0 and mean_m != 0")
