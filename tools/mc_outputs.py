"""Every output array of the Monte Carlo entry points on fixed seeded inputs, for bit-for-bit comparisons of two builds.

usage: B200SV_LIB=... [B200SV_CHAIN_COOP=0|1] python tools/mc_outputs.py OUT.npz [--paths N]
       python tools/mc_outputs.py --compare A.npz B.npz
       python tools/mc_outputs.py --dry-run            (builds the inputs and lists the cases; runs without a GPU)

The library is the one named by $B200SV_LIB (default: the in-tree build).  The chain driver (cooperative or multi-launch) is chosen once
per process from B200SV_CHAIN_COOP, so run one process per setting.  The chains mix C / P / IC / IP and include a maturity without
strikes.  --compare reports every array that is not bitwise equal (NaNs must sit in the same places) and exits 1 if there is one.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

SEED = 20261017
TTMS = np.array([0.05, 0.12, 0.25])
FORWARDS = np.array([100.0, 100.5, 101.0])
DISCFACTORS = np.array([0.999, 0.997, 0.994])
ETAS = np.array([1.0, 1.1, 0.9])


def chain():
    """three maturities, the second without strikes, every payoff code"""
    strikes = [np.array([90.0, 95.0, 100.0, 105.0, 110.0, 100.0, 120.0, 80.0, 99.0]), np.array([]), np.array([85.0, 100.0, 115.0, 101.0])]
    types = [np.array(["P", "P", "C", "C", "C", "IC", "IC", "IP", "IP"]), np.array([], dtype=str), np.array(["IP", "C", "IC", "P"])]
    return TTMS, FORWARDS, DISCFACTORS, strikes, types


def cases(n: int):
    """(name, thunk) per entry point call; every thunk returns a tuple of arrays (None entries are skipped)"""
    from stochvolmodels_b200 import _capi as C
    from stochvolmodels_b200 import engine as E

    ttms, fwd, df, ks, ts = chain()
    lp = E.logsv_params_c(0.4, 0.4, 2.21, 2.18, 0.15, 2.0)
    hp = E.heston_params_c(0.04, 0.05, 2.0, -0.5, 0.6)
    kp = C.HawkesParamsC(0.0, 0.3, 0.05, 0.1, -0.05, 0.1, 1.0, 1.0, 2.0, 0.5, 0.5, 1.0, 1.0, 2.0, 0.5, 0.5)
    ch = (ttms, fwd, df, ks, ts)
    out = []
    for prec, gauss in (("fp64", "fp32"), ("fp64", "fp64"), ("fp64", "fp64_paired"), ("fp32", "fp32")):
        f = E.mc_flags(prec, gauss)
        for vt in (1, 2):
            out.append((f"logsv_chain_{prec}_{gauss}_v{vt}", lambda f=f, vt=vt: E.logsv_mc_chain(lp, *ch[:3], ETAS, *ch[3:], n, 360, False, vt, SEED, f)))
            out.append((f"heston_chain_{prec}_{gauss}_v{vt}", lambda f=f, vt=vt: E.heston_mc_chain(hp, *ch, n, 360, vt, SEED, f)))
        out.append((f"heston_qe_chain_{prec}_{gauss}", lambda f=f: E.heston_mc_chain(hp, *ch, n, 360, 1, SEED, f, scheme=C.HESTON_QE)))
    f64, f32 = E.mc_flags("fp64", "fp64"), E.mc_flags("fp64", "fp32")
    lps = [lp, E.logsv_params_c(0.3, 0.35, 2.0, 2.5, -0.2, 1.5)]
    hps = [hp, E.heston_params_c(0.06, 0.04, 1.5, -0.7, 0.8)]
    for name, f in (("f32", f32), ("f64", f64)):
        out.append((f"logsv_batch_{name}", lambda f=f: E.logsv_mc_chain_batch(lps, *ch[:3], np.tile(ETAS, (2, 1)), *ch[3:], n, 360, True, SEED, f)))
        out.append((f"heston_batch_{name}", lambda f=f: E.heston_mc_chain_batch(hps, *ch, n, 360, SEED, f)))
        for vt in (1, 2):
            out.append((f"logsv_greeks_{name}_v{vt}", lambda f=f, vt=vt: E.logsv_mc_chain_greeks(lp, *ch[:3], ETAS, *ch[3:], n, 360, False, vt, SEED, f)))
            out.append((f"heston_greeks_{name}_v{vt}", lambda f=f, vt=vt: E.heston_mc_chain_greeks(hp, *ch, n, 360, vt, SEED, f)))
            out.append((f"logsv_gamma_{name}_v{vt}", lambda f=f, vt=vt: E.logsv_mc_chain_greeks_gamma(lp, *ch[:3], ETAS, *ch[3:], n, 360, False, vt, SEED, f,
                                                                                                    n_paths_out=min(n, 64))))
            out.append((f"heston_gamma_{name}_v{vt}", lambda f=f, vt=vt: E.heston_mc_chain_greeks_gamma(hp, *ch, n, 360, vt, SEED, f, n_paths_out=min(n, 64))))
        out.append((f"logsv_terminal_{name}", lambda f=f: E.logsv_terminal(lp, 0.1, n, 360, True, 1.0, SEED, f)))
        out.append((f"heston_terminal_{name}", lambda f=f: E.heston_terminal(hp, 0.1, n, 360, SEED, f)))
        out.append((f"logsv_terminal_from_state_{name}", lambda f=f: E.logsv_terminal_from_state(
            lp, np.linspace(-0.1, 0.1, n), np.linspace(0.2, 0.6, n), np.zeros(n), 0.1, 360, False, 1.0, SEED, f, slice_index=2)))
        out.append((f"logsv_tangent_terminal_{name}", lambda f=f: E.logsv_tangent_terminal(lp, 0.1, n, 360, False, 1.0, SEED, f, 1, 7)))
        out.append((f"heston_tangent_terminal_{name}", lambda f=f: E.heston_tangent_terminal(hp, 0.1, n, 360, SEED, f, 1, 7)))
        out.append((f"hawkes_chain_{name}", lambda f=f: E.hawkesjd_mc_chain(kp, *ch, n, 1, SEED, f)))
        out.append((f"hawkes_greeks_{name}", lambda f=f: E.hawkesjd_mc_chain_greeks(kp, *ch, n, 1, SEED, f, n_paths_out=min(n, 64))))
        out.append((f"hawkes_terminal_{name}", lambda f=f: E.hawkesjd_terminal(kp, 0.1, np.zeros(n), np.full(n, 1.0), np.full(n, 1.0), SEED, f, 1, True)))
    rng = np.random.default_rng(SEED)
    x, q = rng.normal(0.0, 0.1, n), rng.uniform(0.0, 0.02, n)
    x[::97] = np.nan
    out.append(("mc_payoffs_v1", lambda: E.mc_payoffs(x, q, 0.25, 100.0, ks[0], ts[0], 0.99, 1)))
    out.append(("mc_payoffs_v2", lambda: E.mc_payoffs(x, q, 0.25, 100.0, ks[0], ts[0], 0.99, 2)))
    hs = ttms / np.array([6, 14, 30])
    steps = np.array([6, 14, 30])
    Z = rng.standard_normal((2, 30, n))
    for nf in (1, 3, 8):
        w, nodes = np.linspace(0.5, 1.5, nf) / nf, np.geomspace(0.1, 50.0, nf)
        for name, f in (("f32", f32), ("f64", f64)):
            out.append((f"rough_chain_n{nf}_{name}", lambda w=w, nodes=nodes, f=f: E.rough_logsv_mc_chain(
                lps, w, nodes, *ch, n, steps, hs, variable_type=1, seed=SEED, flags=f, with_ivols=True)[:3]))
            out.append((f"rough_greeks_n{nf}_{name}", lambda w=w, nodes=nodes, f=f: E.rough_logsv_mc_chain_greeks(
                lp, w, nodes, *ch, n, steps, hs, seed=SEED, flags=f, return_states=True, return_tangents=True)))
        out.append((f"rough_greeks_n{nf}_given", lambda w=w, nodes=nodes: E.rough_logsv_mc_chain_greeks(
            lp, w, nodes, *ch, n, steps, hs, Z[0], Z[1], seed=SEED, flags=f32, return_states=True)))
        out.append((f"rough_chain_n{nf}_given", lambda w=w, nodes=nodes: E.rough_logsv_mc_chain(
            lps, w, nodes, *ch, n, steps, hs, Z[0], Z[1], variable_type=2, seed=SEED, flags=f32, with_ivols=True, return_states=False)[:3]))
    for p2p in (False, True):
        out.append((f"dev_chain_p2p{int(p2p)}", lambda p2p=p2p: dev_chain(n, lp, hp, kp, p2p)))
    return out


def dev_chain(n: int, lp, hp, kp, p2p: bool):
    """the device-level entry points on one GPU, each model's slices then dev_payoff_sums / dev_payoff_finalize per maturity; with ``p2p``
    through a one-rank mailbox, so that the exchange fused into the slice, payoff and finalise kernels runs as well"""
    import ctypes
    from ctypes import byref, c_void_p
    import torch
    from stochvolmodels_b200 import _capi as C

    ttms, fwd, df, ks, ts = chain()
    ctx = None
    if p2p:
        ctx, handle = c_void_p(), (ctypes.c_ubyte * 64)()
        C.call("b200sv_p2p_create", 1, 0, 64, byref(ctx), handle)
        C.call("b200sv_p2p_connect", ctx, (ctypes.c_ubyte * 64).from_buffer_copy(bytes(handle)))
    st = c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: c_void_p(t.data_ptr())
    w = np.array([0.6, 0.4])
    nodes = np.array([0.5, 20.0])
    results = []
    for model in ("logsv", "heston", "hawkes", "rough"):
        state = torch.zeros((4, n), dtype=torch.float64, device="cuda")
        mom = torch.zeros(2, dtype=torch.float64, device="cuda")
        out = torch.zeros((len(ttms), 2, 16), dtype=torch.float64, device="cuda")
        t0 = 0.0
        for m, ttm in enumerate(ttms):
            S = int((ttm - t0) * 360) + 1
            dt = (ttm - t0) / S
            t0 = ttm
            if model == "logsv":
                C.call("b200sv_dev_logsv_slice", ptr(state[0]), ptr(state[1]), ptr(state[2]), n, 3, int(m == 0), byref(lp), 1.0, 0, S, dt, m,
                       float(fwd[m]), SEED, 0, ptr(mom), ctx, st)
            elif model == "heston":
                C.call("b200sv_dev_heston_slice", ptr(state[0]), ptr(state[1]), ptr(state[2]), n, 3, int(m == 0), byref(hp), S, dt, m,
                       float(fwd[m]), SEED, 0, 0, ptr(mom), ctx, st)
            elif model == "hawkes":
                C.call("b200sv_dev_hawkesjd_slice", ptr(state[0]), ptr(state[1]), ptr(state[2]), n, 3, int(m == 0), byref(kp), S, dt, m,
                       float(fwd[m]), SEED, 0, ptr(mom), ctx, st)
            else:
                C.call("b200sv_dev_rough_logsv_slice", ptr(state[0]), ptr(state[1]), ptr(state[3]), n, 3, byref(lp), 2, C.dptr(w), C.dptr(nodes),
                       S, ttm / S, float(fwd[m]), SEED, 0, ptr(mom), ctx, st)
            J = len(ks[m])
            if J:
                strikes = torch.as_tensor(ks[m], dtype=torch.float64, device="cuda")
                codes = torch.as_tensor(C.encode_types(ts[m]), device="cuda")
                sums = torch.zeros(3 * J, dtype=torch.float64, device="cuda")
                qrow = state[3] if model == "rough" else state[2]
                C.call("b200sv_dev_payoff_sums", ptr(state[0]), ptr(qrow), n, 0, float(ttm), float(fwd[m]), ptr(strikes), ptr(codes), J, 1, 0,
                       ptr(mom), ptr(sums), ctx, st)
                C.call("b200sv_dev_payoff_finalize", ptr(sums), J, float(df[m]), n, ptr(out[m, 0]), ptr(out[m, 1]), ctx, st)
        spot_mom = torch.zeros(2, dtype=torch.float64, device="cuda")
        C.call("b200sv_dev_spot_moments", ptr(state[0]), n, float(fwd[-1]), ptr(spot_mom), st)
        torch.cuda.synchronize()
        results += [state.cpu().numpy(), mom.cpu().numpy(), out.cpu().numpy(), spot_mom.cpu().numpy()]
    if ctx is not None:
        C.call("b200sv_p2p_destroy", ctx)
    return tuple(results)


def flatten(name, res):
    arrays = {}
    def walk(key, v):
        if v is None:
            return
        if isinstance(v, (list, tuple)):
            for i, e in enumerate(v):
                walk(f"{key}.{i}", e)
        else:
            arrays[key] = np.asarray(v)
    walk(name, res)
    return arrays


def compare(a_path, b_path) -> int:
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        if x.shape != y.shape or x.dtype != y.dtype or x.tobytes() != y.tobytes():
            bad.append(k)
    for k in bad:
        print("DIFFERS", k)
    print(f"{len(set(a.files) & set(b.files))} arrays compared, {len(bad)} differ")
    return 1 if bad else 0


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("out", nargs="?")
    ap.add_argument("--paths", type=int, default=20000)
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    ap.add_argument("--dry-run", action="store_true")
    args = ap.parse_args()
    if args.compare:
        return compare(*args.compare)
    if args.dry_run:
        ttms, fwd, df, ks, ts = chain()
        names = [name for name, _ in cases(args.paths)]
        print(f"chain: {len(ttms)} maturities, strikes per maturity {[len(k) for k in ks]}, codes {sorted(set(np.concatenate(ts)))}")
        print(f"{len(names)} cases: {', '.join(names)}")
        return 0
    if not args.out:
        ap.error("OUT.npz is required")
    arrays = {}
    for name, thunk in cases(args.paths):
        arrays.update(flatten(name, thunk()))
    np.savez(args.out, **arrays)
    print(f"{len(arrays)} arrays -> {args.out} (B200SV_CHAIN_COOP={os.environ.get('B200SV_CHAIN_COOP', 'unset')})")
    return 0


if __name__ == "__main__":
    sys.exit(main())
