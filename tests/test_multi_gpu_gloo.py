"""CPU: the N>1 path with torch.distributed (gloo, world_size 2): sharded chain MC == unsharded, on every rank."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import mc

K5 = np.array([0.8, 0.9, 1.0, 1.1, 1.2])
CASES = {
    "logsv": dict(params=(0.8376, 1.0413, 3.1844, 3.058, 0.1514, 1.8458), ttms=np.array([0.1, 0.3]), fw=np.array([1.0, 1.02]),
                  df=np.array([0.999, 0.99]), etas=np.array([0.9, 1.1]), spot=False,
                  types=[np.array(["IP", "IP", "IC", "IC", "IC"]), np.array(["IP", "P", "C", "IC", "IC"])]),
    "heston": dict(params=(0.04, 0.04, 4.0, -0.5, 0.4), ttms=np.array([0.1, 0.3]), fw=np.array([1.0, 1.02]), df=np.array([0.999, 0.99]),
                   etas=None, spot=True, types=[np.array(["P", "P", "C", "C", "C"])] * 2),
}
N, NPY, SEED = 2001, 252, 77       # odd path count: ranks get 1001 / 1000


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _expected(model):
    c = CASES[model]
    steps = mc.chain_steps(c["ttms"], NPY)
    Z = [mc.device_normals(SEED, np.arange(N), m, steps[m][0], "f64") for m in range(2)]
    dts = [d for _, d in steps]
    if model == "logsv":
        return mc.logsv_mc_chain_fixed(c["params"], c["ttms"], c["fw"], c["df"], [K5, K5], c["types"], c["etas"], [z[0] for z in Z],
                                       [z[1] for z in Z], dts, c["spot"], 1)
    return mc.heston_mc_chain_fixed(c["params"], c["ttms"], c["fw"], c["df"], [K5, K5], c["types"], [z[0] for z in Z], [z[1] for z in Z], dts, 1)


def _worker(rank, world, port, model, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_engine import OracleEngine
        from stochvolmodels_b200 import _capi as C, engine
        from stochvolmodels_b200.multi_gpu import mc_chain_distributed
        c = CASES[model]
        pc = engine.logsv_params_c(*c["params"]) if model == "logsv" else engine.heston_params_c(*c["params"])
        p, e = mc_chain_distributed(model, pc, c["ttms"], c["fw"], c["df"], c["etas"], [K5, K5], c["types"], N, NPY, c["spot"], C.LOG_RETURN,
                                    SEED, C.GAUSS_F64, engine_factory=OracleEngine)
        # an engine without a peer-memory mailbox takes the collective by default, accepts it explicitly, refuses exchange="p2p"
        p2, _ = mc_chain_distributed(model, pc, c["ttms"], c["fw"], c["df"], c["etas"], [K5, K5], c["types"], N, NPY, c["spot"], C.LOG_RETURN,
                                     SEED, C.GAUSS_F64, engine_factory=OracleEngine, exchange="collective")
        assert all(np.array_equal(a, b) for a, b in zip(p, p2))
        for bad, exc in (("p2p", ValueError), ("ring", ValueError)):
            try:
                mc_chain_distributed(model, pc, c["ttms"], c["fw"], c["df"], c["etas"], [K5, K5], c["types"], N, NPY, c["spot"], C.LOG_RETURN,
                                     SEED, C.GAUSS_F64, engine_factory=OracleEngine, exchange=bad)
                raise AssertionError(f"exchange={bad!r} was accepted")
            except exc:
                pass
        out[rank] = (p, e)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("model", ["logsv", "heston"])
def test_sharded_chain_equals_unsharded_under_gloo(model):
    world, port = 2, _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, model, out), nprocs=world, join=True)
    pe, ee = _expected(model)
    assert sorted(out.keys()) == [0, 1]
    for rank in range(world):
        p, e = out[rank]
        for m in range(2):
            np.testing.assert_allclose(p[m], pe[m], rtol=1e-11, atol=1e-14)     # only the fp64 summation order differs
            np.testing.assert_allclose(e[m], ee[m], rtol=1e-9, atol=1e-14)
    for m in range(2):                                                            # every rank returns the same numbers
        np.testing.assert_array_equal(out[0][0][m], out[1][0][m])


def test_unsharded_path_through_the_same_driver():
    """world size 1 (no process group): the driver degenerates to the plain chain loop."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from fake_engine import OracleEngine
    from stochvolmodels_b200 import _capi as C, engine
    from stochvolmodels_b200.multi_gpu import mc_chain_distributed
    c = CASES["logsv"]
    p, e = mc_chain_distributed("logsv", engine.logsv_params_c(*c["params"]), c["ttms"], c["fw"], c["df"], c["etas"], [K5, K5], c["types"], N,
                                NPY, c["spot"], C.LOG_RETURN, SEED, C.GAUSS_F64, engine_factory=OracleEngine)
    pe, ee = _expected("logsv")
    for m in range(2):
        np.testing.assert_allclose(p[m], pe[m], rtol=1e-11, atol=1e-14)
        np.testing.assert_allclose(e[m], ee[m], rtol=1e-9, atol=1e-14)


ROUGH = dict(params=(0.8, 1.0, 2.2, 2.2, 0.2, 1.6), weights=np.array([0.7, 0.5, 0.3]), nodes=np.array([0.05, 1.5, 20.0]),
             ttms=np.array([0.05, 0.15]), types=[np.array(["P", "P", "C", "C", "C"])] * 2)
N_ROUGH, NPY_ROUGH = 801, 120


def _rough_grid():
    from oracle.mc import set_time_grid
    grids = []
    for t in ROUGH["ttms"]:
        S, _ = set_time_grid(t, NPY_ROUGH)
        grids.append(np.linspace(0.0, t, S + 1))
    return grids


def _rough_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import sys
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from fake_engine import OracleEngine
        from stochvolmodels_b200 import _capi as C, engine
        from stochvolmodels_b200.multi_gpu import mc_chain_distributed
        grid = [(g.size - 1, float(g[1] - g[0])) for g in _rough_grid()]
        factory = lambda *a, **k: OracleEngine(*a, factors=(ROUGH["weights"], ROUGH["nodes"]), **k)
        out[rank] = mc_chain_distributed("rough", engine.logsv_params_c(*ROUGH["params"]), ROUGH["ttms"], np.ones(2), np.ones(2), None, [K5, K5],
                                         ROUGH["types"], N_ROUGH, 0, True, C.LOG_RETURN, SEED, C.GAUSS_F64, engine_factory=factory, grid=grid,
                                         se_paths=1)
    finally:
        dist.destroy_process_group()


def test_sharded_rough_chain_equals_unsharded_under_gloo():
    """the rough-vol route through the same driver: per-maturity grids from t = 0 (`grid=`), slice-0 draws, un-normalised standard errors
    (`se_paths=1`), two ranks == the oracle's unsharded chain on the same Philox normals"""
    from oracle import rough
    world, port = 2, _free_port()
    out = mp.Manager().dict()
    mp.spawn(_rough_worker, args=(world, port, out), nprocs=world, join=True)
    grids = _rough_grid()
    Z0, Z1 = mc.device_normals(SEED, np.arange(N_ROUGH), 0, grids[-1].size - 1, "f64")
    pe, ee = rough.rough_chain_fixed(ROUGH["ttms"], np.ones(2), np.ones(2), [K5, K5], ROUGH["types"], Z0, Z1, *ROUGH["params"], ROUGH["weights"],
                                     ROUGH["nodes"], grids)
    for rank in range(world):
        p, e = out[rank]
        for m in range(2):
            np.testing.assert_allclose(p[m], pe[m], rtol=1e-11, atol=1e-14)
            np.testing.assert_allclose(e[m], ee[m], rtol=1e-9, atol=1e-14)


def _bad_code_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from stochvolmodels_b200 import _capi as C, engine
        from stochvolmodels_b200.multi_gpu import mc_chain_distributed
        c, built = CASES["logsv"], []
        try:
            mc_chain_distributed("logsv", engine.logsv_params_c(*c["params"]), c["ttms"], c["fw"], c["df"], c["etas"], [K5, K5],
                                 [c["types"][0], np.array(["P", "P", "X", "C", "C"])], N, NPY, c["spot"], C.LOG_RETURN, SEED, C.GAUSS_F64,
                                 engine_factory=lambda *a, **k: built.append(a))
            out[rank] = "accepted"
        except ValueError as e:
            out[rank] = (str(e), len(built))
    finally:
        dist.destroy_process_group()


def test_unknown_payoff_code_raises_on_every_rank_before_any_engine():
    """the sharded route validates the option types before it builds an engine (the pricers rely on it and do not check them first)"""
    world, port = 2, _free_port()
    out = mp.Manager().dict()
    mp.spawn(_bad_code_worker, args=(world, port, out), nprocs=world, join=True)
    assert dict(out) == {r: ("unknown option payoff code", 0) for r in range(world)}


def _policy_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from stochvolmodels_b200.multi_gpu import SHARD_MIN_PATHS, _shared_seed, _use_distributed
        out[rank] = dict(seed=_shared_seed(None), given=_shared_seed(42),
                         small=_use_distributed({"nb_path": SHARD_MIN_PATHS - 1}), large=_use_distributed({"nb_path": SHARD_MIN_PATHS}),
                         forced=_use_distributed({"nb_path": 10, "exchange": "collective"}), off=_use_distributed({"distributed": False, "nb_path": 10 ** 9}),
                         unknown=_use_distributed({}))
    finally:
        dist.destroy_process_group()


def test_shard_or_replicate_policy_and_shared_seed_under_gloo():
    """small Monte Carlo calls are replicated instead of sharded (launch-bound: one GPU is faster), a named exchange forces sharding, and a
    seedless call uses ONE seed on all ranks (rank 0's, broadcast)"""
    world, port = 2, _free_port()
    out = mp.Manager().dict()
    mp.spawn(_policy_worker, args=(world, port, out), nprocs=world, join=True)
    assert out[0]["seed"] == out[1]["seed"] and out[0]["given"] == out[1]["given"] == 42
    for r in range(world):
        assert out[r]["small"] is False and out[r]["large"] is True and out[r]["forced"] is True and out[r]["off"] is False and out[r]["unknown"] is True
    from stochvolmodels_b200.multi_gpu import _use_distributed
    assert _use_distributed({"nb_path": 10 ** 9}) is False          # no process group: never sharded
