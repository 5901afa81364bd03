"""Multi-GPU Monte Carlo: one process per GPU (torchrun), paths sharded by contiguous GLOBAL path-id ranges.

The path shards naturally (SURVEY.md §8e): state never leaves its GPU; per maturity there are exactly two exchange steps,
both tiny all-reduces of fp64 moments:
    (1) [sum F*exp(x), count]               -> forward re-centring  (utils/mc_payoffs.py:61-63)
    (2) [sum pay, sum pay^2, count] x J     -> prices / standard errors (:85-88)
Default exchange on GPUs (``exchange="p2p"``): the two messages travel through NVLink peer memory INSIDE the kernels that produce and
consume them (csrc/p2p.cuh: mailbox stores from the partial-reduction kernel, acquire-spin + rank-ordered sum in the payoff / finalize
kernel prologues) -- no collective launch, no host synchronisation.  ``exchange="collective"`` uses ``torch.distributed.all_reduce``
(NCCL; gloo in the CPU tests).
torch is plumbing only: device memory (``torch.empty``), the current CUDA stream, and ``torch.distributed`` (NCCL over
NVLink on GPUs, gloo in the CPU tests).  All arithmetic is in libb200sv kernels, called through the device-level C ABI
(``b200sv_dev_*``) with raw pointers.  Because the Philox counter is the global path id, prices do not depend on the number of
GPUs beyond fp64 summation order.
"""
from __future__ import annotations

import os
from ctypes import byref, c_uint, c_void_p
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import _capi as C
from . import engine
from .utils.funcs import set_time_grid


def shard_paths(nb_path: int, world_size: int, rank: int) -> Tuple[int, int]:
    """(n_local, path_offset) of ``rank``: contiguous ranges, remainder spread over the first ranks."""
    base, rem = divmod(int(nb_path), int(world_size))
    n_local = base + (1 if rank < rem else 0)
    offset = rank * base + min(rank, rem)
    return n_local, offset


def _shared_seed(seed) -> int:
    """the Philox key of an MC call: the caller's ``seed``, or a fresh one -- which under a torch.distributed world must be the SAME on every rank
    (sharded: one stream over all paths; replicated: identical prices everywhere), so rank 0 draws it and broadcasts"""
    if seed is not None:
        return int(seed)
    value = engine.fresh_seed()
    try:
        import torch
        import torch.distributed as dist
    except Exception:
        return value
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        device = "cuda" if dist.get_backend() == "nccl" else "cpu"
        box = torch.tensor([value & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=device)
        dist.broadcast(box, src=0)
        value = int(box.item())
    return value


SHARD_MIN_PATHS = 500_000      # below this a chain call is launch-bound: one GPU prices it faster than N GPUs exchanging moments (r02 profile)


def _use_distributed(kwargs) -> bool:
    """shard this Monte Carlo call over the ranks of the initialised torch.distributed world?  Small calls (``nb_path`` < SHARD_MIN_PATHS, env
    B200SV_SHARD_MIN_PATHS) are priced REPLICATED instead -- every rank runs all the paths on its own GPU through the single-launch chain
    kernel and gets bit-identical prices (the Philox counter is the global path id), 0.17 ms against 0.53 ms sharded at 1e4 paths on 2 GPUs
    (`profiles/r02_multi_gpu_latency.txt`).  Naming an ``exchange`` forces the sharded route."""
    if not kwargs.get("distributed", True):
        return False
    try:
        import torch.distributed as dist
    except Exception:       # torch absent: single-process only
        return False
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return False
    nb_path = kwargs.get("nb_path")
    if nb_path is not None and kwargs.get("exchange") is None:
        return int(nb_path) >= int(os.environ.get("B200SV_SHARD_MIN_PATHS", SHARD_MIN_PATHS))
    return True


def payoff_kinds(types: np.ndarray) -> int:
    """the payoff-kind mask of one slice's int8 type codes that b200sv_dev_payoff_sums takes: 1 = a call or put, 2 = an inverse option"""
    return int(np.bitwise_or.reduce(np.where(types >= 2, 2, 1)))


# (group id, device index) -> (ctx, capacity): mailboxes are created once per process group and reused by every chain call, so that the
# per-call cost of the P2P exchange is zero host work (cudaMalloc + IPC mapping happen on first use only)
_P2P_CACHE = {}
_P2P_MIN_VALUES = 3 * 512


def p2p_context(torch, device, group=None, min_values: int = 0):
    """this rank's libb200sv mailbox context for ``group`` (created, IPC-exchanged and mapped on first use; COLLECTIVE on first use and
    whenever ``min_values`` outgrows the cached capacity -- every rank of the group must call it with the same arguments)."""
    import ctypes
    import torch.distributed as dist
    key = (id(group) if group is not None else 0, torch.device(device).index)
    hit = _P2P_CACHE.get(key)
    if hit is not None and hit[1] >= min_values:
        return hit[0]
    if hit is not None:
        torch.cuda.synchronize(device)
        dist.barrier(group)               # nobody is still spinning on the mailbox that is about to go
        C.call("b200sv_p2p_destroy", hit[0])
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    cap = max(int(min_values), _P2P_MIN_VALUES)
    ctx = c_void_p()
    handle = (ctypes.c_ubyte * 64)()
    error = None
    with torch.cuda.device(device):
        try:
            C.call("b200sv_p2p_create", world, rank, cap, ctypes.byref(ctx), handle)
        except C.B200svError as e:       # keep taking part in the collectives below so that every rank reaches the same verdict
            error = e
        handles = [None] * world
        dist.all_gather_object(handles, None if error else bytes(handle), group=group)
        if error is None and all(h is not None for h in handles):
            try:
                C.call("b200sv_p2p_connect", ctx, (ctypes.c_ubyte * (64 * world)).from_buffer_copy(b"".join(handles)))
            except C.B200svError as e:   # e.g. no peer access / IPC not permitted between these devices
                error = e
        elif error is None:
            error = C.B200svError(-2, "a peer could not create its mailbox")
    verdicts = [None] * world
    dist.all_gather_object(verdicts, None if error is None else str(error), group=group)   # also: nobody publishes before all are mapped
    failed = [v for v in verdicts if v is not None]
    if failed:
        if ctx:
            C.call("b200sv_p2p_destroy", ctx)
        raise P2pUnavailable(failed[0])
    if os.environ.get("B200SV_P2P_SPIN_LIMIT"):          # polls of ~200 ns each; default 2^24 (~3 s)
        C.call("b200sv_p2p_set_spin_limit", ctx, int(os.environ["B200SV_P2P_SPIN_LIMIT"]))
    _P2P_CACHE[key] = (ctx, cap)
    return ctx


class P2pUnavailable(RuntimeError):
    """peer-memory mailboxes cannot be set up between the ranks of this group (raised on EVERY rank of the group)."""


class P2pTimeout(C.B200svError):
    """a peer did not publish its values within the mailbox's spin limit (csrc/p2p.cuh): the chain's prices on this rank are poisoned
    with NaN and must not be used.  ``peers`` lists the ranks that never arrived."""

    def __init__(self, status: int):
        self.peers = [r for r in range(32) if status >> r & 1]
        super().__init__(-5, f"peer-memory exchange timed out waiting for rank(s) {self.peers}; re-run with exchange='collective' "
                             "or raise the limit (B200SV_P2P_SPIN_LIMIT)")


# Engines (device-resident path state 3 x n_local x 8 B, strike / result buffers, a pinned host landing buffer) are cached per
# (model, shard, flags, device) and reused by the next API call with the same shard: the N>1 e2e arm of bench.py paid 6-13 ms per call
# for engine construction (VERDICT r1 weak #5).  The state stays allocated between calls (2.4 GB at 1e8 paths) -- release_engines()
# frees it; B200SV_ENGINE_CACHE=0 disables the cache.
_ENGINE_CACHE = {}
TRACE_LOG = []          # filled when B200SV_TRACE is set (one dict per sharded chain call on this rank)


def release_engines():
    """drop every cached CudaMcEngine (frees their path state)."""
    _ENGINE_CACHE.clear()


def _cached_engine(model, params_c, n_local, offset, flags, Jmax, scheme, factors=None):
    import torch
    if os.environ.get("B200SV_ENGINE_CACHE", "1") == "0":
        return CudaMcEngine(model, params_c, n_local, offset, flags, Jmax, scheme=scheme, factors=factors)
    rows = 0 if factors is None else len(factors[0])
    key = (model, int(n_local), int(offset), int(flags), int(scheme), rows, torch.cuda.current_device())
    eng = _ENGINE_CACHE.get(key)
    if eng is None or eng.cap < max(Jmax, 1):
        for k in [k for k in _ENGINE_CACHE if k[0] == model and k[-1] == key[-1]]:    # one resident shard per model and device
            del _ENGINE_CACHE[k]
        eng = CudaMcEngine(model, params_c, n_local, offset, flags, Jmax, scheme=scheme, factors=factors)
        _ENGINE_CACHE[key] = eng
    eng.params_c = params_c
    eng.set_factors(factors)
    return eng


def release_p2p():
    """unmap and free every cached mailbox (call on all ranks before destroy_process_group; optional -- process exit frees them)."""
    import torch
    for ctx, _ in _P2P_CACHE.values():
        torch.cuda.synchronize()
        C.call("b200sv_p2p_destroy", ctx)
    _P2P_CACHE.clear()


class CudaMcEngine:
    """Device-resident MC state + kernel launches on the current CUDA device (used for N>=1 ranks and by bench.py)."""

    MODELS = ("logsv", "heston", "hawkes", "hawkes_exact", "rough")

    def __init__(self, model: str, params_c, n_local: int, path_offset: int, flags: int, max_strikes: int, device=None, scheme: int = 0,
                 factors=None):
        """``model``: 'logsv' / 'heston' (state x, vol or var, qvar), 'hawkes' (state x, lambda_p, lambda_m; x stands in for qvar in the
        payoff, hawkes_jd_pricer.py:703), 'hawkes_exact' (the same state on the exact event-driven route, DESIGN.md §3.13: ``simulate_slice``
        reads ``dt`` as the interval's length and ``nsteps`` not at all) or 'rough' (state log_spot, n vol factors, qvar; ``factors`` =
        (weights, nodes) of the kernel)."""
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("CudaMcEngine needs a CUDA device; stochvolmodels_b200 has no CPU fallback")
        if model not in self.MODELS:
            raise ValueError(f"unknown model {model!r}")
        C.load_library()
        self.torch = torch
        self.model = model
        self.scheme = int(scheme)
        self.params_c = params_c
        self.n_local, self.path_offset, self.flags = int(n_local), int(path_offset), int(flags)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        if model in ("hawkes", "hawkes_exact", "rough") and (flags & C.STATE_F32):
            raise ValueError("the Hawkes and rough-vol routes are float64 only")
        sdtype = torch.float32 if (flags & C.STATE_F32) else torch.float64
        self.factors = None
        self.set_factors(factors)
        rows = 3 if model != "rough" else len(self.factors[0]) + 2
        self.qrow = {"hawkes": 0, "hawkes_exact": 0, "rough": rows - 1}.get(model, 2)          # the state row the Q_VAR payoff reads
        self.state = torch.empty((rows, max(self.n_local, 1)), dtype=sdtype, device=self.device)
        self.moments = torch.zeros(2, dtype=torch.float64, device=self.device)
        self.sums = torch.zeros(3 * max(max_strikes, 1), dtype=torch.float64, device=self.device)
        self.out = torch.zeros(2 * max(max_strikes, 1), dtype=torch.float64, device=self.device)
        self.cap = max(max_strikes, 1)
        self.p2p = None          # libb200sv P2P mailbox context (void*), see enable_p2p
        self._chain_dev = None   # per-chain buffers reused across calls (see chain_buffers)
        self._chain_host = None
        # exact Hawkes route: candidates per path and interval, and the device flag its kernel raises when a path runs out of them
        self.max_candidates = engine.HAWKES_EXACT_DEFAULT_BUDGET
        self.overflow = torch.zeros(1, dtype=torch.int32, device=self.device) if model == "hawkes_exact" else None

    def set_factors(self, factors):
        """(weights, nodes) of the rough kernel's Markovian lift (host float64 arrays of equal length <= 8); None for the other models."""
        if self.model != "rough":
            return
        if factors is None:
            raise ValueError("the rough-vol engine needs factors=(weights, nodes)")
        w, x = (np.ascontiguousarray(a, dtype=np.float64).ravel() for a in factors)
        if w.shape != x.shape or not 1 <= w.shape[0] <= 8:
            raise ValueError("weights and nodes must have the same length, 1..8")
        if self.factors is not None and self.factors[0].shape != w.shape:
            raise ValueError("the number of factors of a cached engine cannot change")
        self.factors = (w, x)

    def chain_buffers(self, Jtot: int):
        """(strikes f64[J], types i8[J], out f64[2, J]) on the device + a pinned host mirror of `out`, grown on demand and reused."""
        torch, J = self.torch, max(int(Jtot), 1)
        if self._chain_dev is None or self._chain_dev[0].shape[0] < J:
            self._chain_dev = (torch.empty(J, dtype=torch.float64, device=self.device), torch.empty(J, dtype=torch.int8, device=self.device),
                               torch.zeros((2, J), dtype=torch.float64, device=self.device))
            self._chain_host = (torch.empty(J, dtype=torch.float64).pin_memory(), torch.empty(J, dtype=torch.int8).pin_memory(),
                                torch.empty((2, J), dtype=torch.float64).pin_memory())
        return self._chain_dev, self._chain_host

    def check_p2p(self):
        """raise P2pTimeout if an exchange of the chain just run timed out on this rank (synchronises the stream)."""
        if self.p2p is None:
            return
        status = c_uint(0)
        C.call("b200sv_p2p_status", self.p2p, byref(status), self._stream())
        if status.value:
            raise P2pTimeout(status.value)

    def enable_p2p(self, group=None):
        """attach this rank's (cached) peer-memory mailbox for ``group``; collective call."""
        self.p2p = p2p_context(self.torch, self.device, group, 3 * self.cap)

    def _stream(self):
        return c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def to_device(self, array: np.ndarray, dtype):
        return self.torch.as_tensor(np.ascontiguousarray(array), dtype=dtype).to(self.device, non_blocking=False)

    def simulate_slice(self, m: int, init: bool, nsteps: int, dt: float, eta: float, is_spot: bool, forward: float, seed: int):
        """advance local paths through maturity slice m; leaves the LOCAL (sum F e^x, count) in ``self.moments``."""
        x, v, q = (c_void_p(self.state[i].data_ptr()) for i in range(3))
        if self.n_local == 0:
            self.moments.zero_()
            if self.p2p is not None:      # a rank without paths still takes part in the exchange
                C.call("b200sv_dev_p2p_publish", self.p2p, c_void_p(self.moments.data_ptr()), 2, self._stream())
            return self.moments
        seed = C.seed64(seed)
        if self.model == "logsv":
            C.call("b200sv_dev_logsv_slice", x, v, q, self.n_local, self.path_offset, int(init), byref(self.params_c), float(eta),
                   int(bool(is_spot)), int(nsteps), float(dt), int(m), float(forward), seed, self.flags,
                   c_void_p(self.moments.data_ptr()), self.p2p, self._stream())
        elif self.model == "hawkes":
            C.call("b200sv_dev_hawkesjd_slice", x, v, q, self.n_local, self.path_offset, int(init), byref(self.params_c), int(nsteps), float(dt),
                   int(m), float(forward), seed, self.flags, c_void_p(self.moments.data_ptr()), self.p2p, self._stream())
        elif self.model == "hawkes_exact":
            C.call("b200sv_dev_hawkesjd_exact_slice", x, v, q, self.n_local, self.path_offset, int(init), byref(self.params_c), float(dt), int(m),
                   float(forward), seed, int(self.max_candidates), c_void_p(self.overflow.data_ptr()), c_void_p(self.moments.data_ptr()),
                   self.p2p, self._stream())
        elif self.model == "rough":       # every maturity restarts at t = 0 on its own grid: `init` and `m` do not enter
            w, nodes = self.factors
            C.call("b200sv_dev_rough_logsv_slice", x, c_void_p(self.state[1].data_ptr()), c_void_p(self.state[self.qrow].data_ptr()), self.n_local,
                   self.path_offset, byref(self.params_c), int(w.shape[0]), C.dptr(w), C.dptr(nodes), int(nsteps), float(dt), float(forward),
                   seed, self.flags, c_void_p(self.moments.data_ptr()), self.p2p, self._stream())
        else:
            C.call("b200sv_dev_heston_slice", x, v, q, self.n_local, self.path_offset, int(init), byref(self.params_c), int(nsteps),
                   float(dt), int(m), float(forward), seed, self.flags, self.scheme,
                   c_void_p(self.moments.data_ptr()), self.p2p, self._stream())
        return self.moments

    def check_overflow(self, group=None, world: int = 1):
        """raise B200svError(-6) if a path of the exact Hawkes route ran out of candidates since the flag was last cleared, on this rank or
        (``world`` > 1: one all-reduce over ``group``) on any rank, then clear the flag.  Synchronises the stream."""
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(self.overflow, op=dist.ReduceOp.MAX, group=group)
        hit = int(self.overflow.item())
        self.overflow.zero_()
        if hit:
            raise C.B200svError(-6, f"candidate budget exhausted: a path of the exact Hawkes route drew more than {self.max_candidates} "
                                    "candidates in one maturity interval")

    def payoff_sums(self, ttm: float, forward: float, strikes_dev, types_dev, J: int, variable_type: int, kinds: int = 0):
        """LOCAL per-strike (sum, sum^2, count) given the GLOBAL moments in ``self.moments``; returns a view of 3*J doubles."""
        sums = self.sums[: 3 * J]
        if self.n_local == 0:
            sums.zero_()
            if self.p2p is not None:
                C.call("b200sv_dev_p2p_publish", self.p2p, c_void_p(sums.data_ptr()), 3 * J, self._stream())
            return sums
        C.call("b200sv_dev_payoff_sums", c_void_p(self.state[0].data_ptr()), c_void_p(self.state[self.qrow].data_ptr()), self.n_local,
               self.flags, float(ttm), float(forward), c_void_p(strikes_dev.data_ptr()), c_void_p(types_dev.data_ptr()), int(J),
               int(variable_type), int(kinds), c_void_p(self.moments.data_ptr()), c_void_p(sums.data_ptr()), self.p2p, self._stream())
        return sums

    def finalize(self, sums, J: int, discfactor: float, total_paths: int, prices=None, stds=None):
        """GLOBAL sums -> (prices, std errors) device views of J doubles each (written into ``prices`` / ``stds`` when given)."""
        if prices is None:
            prices, stds = self.out[:J], self.out[self.cap: self.cap + J]
        C.call("b200sv_dev_payoff_finalize", c_void_p(sums.data_ptr()), int(J), float(discfactor), int(total_paths),
               c_void_p(prices.data_ptr()), c_void_p(stds.data_ptr()), self.p2p, self._stream())
        return prices, stds


def mc_chain_distributed(model: str, params_c, ttms, forwards, discfactors, etas, strikes_ttms, optiontypes_ttms, nb_path: int,
                         nb_steps_per_year: int, is_spot_measure: bool, variable_type: int, seed: int, flags: int,
                         group=None, engine_factory: Optional[Callable] = None, return_engine: bool = False, scheme: int = 0,
                         exchange: Optional[str] = None, grid: Optional[Sequence[Tuple[int, float]]] = None, factors=None,
                         se_paths: Optional[int] = None, max_candidates: Optional[int] = None):
    """Chain MC with ``nb_path`` TOTAL paths split over the ranks of ``group`` (default: the world; works unsharded when
    torch.distributed is not initialised).  Every rank returns the same (prices, std errors) lists.

    Mirrors the slice loop of logsv_mc_chain_pricer / heston_mc_chain_pricer (pricers/logsv_pricer.py:840-865,
    pricers/heston_pricer.py:304-329): the terminal state of slice m seeds slice m+1.  ``model`` 'hawkes' (hawkes_jd_pricer.py:687-715,
    ``nb_steps_per_year`` = 1800 there) and 'rough' (logsv_pricer.py:1199-1216: ``grid`` = the (nb_steps, h) of every maturity's OWN grid
    from t = 0, ``factors`` = (weights, nodes), ``se_paths`` = 1 for that route's un-normalised standard errors) shard the same way, and so
    does 'hawkes_exact' (DESIGN.md §3.13: ``grid`` = (1, interval length) per maturity, ``max_candidates`` its candidate budget; a path
    that runs out of candidates on any rank raises B200svError(-6) on every rank).
    """
    import torch
    import torch.distributed as dist
    distributed = dist.is_available() and dist.is_initialized()
    world = dist.get_world_size(group) if distributed else 1
    rank = dist.get_rank(group) if distributed else 0
    n_local, offset = shard_paths(nb_path, world, rank)
    ttms = np.asarray(ttms, dtype=np.float64)
    M = ttms.shape[0]
    offsets, strikes, types = C.flatten_chain(strikes_ttms, optiontypes_ttms)
    sizes = np.diff(offsets)
    Jmax = int(sizes.max()) if M else 0
    if engine_factory is None:
        eng = _cached_engine(model, params_c, n_local, offset, flags, Jmax, scheme, factors)
    else:
        eng = engine_factory(model, params_c, n_local, offset, flags, Jmax, scheme=scheme) if scheme else engine_factory(model, params_c, n_local, offset, flags, Jmax)
    # exchange mode: P2P mailbox on CUDA engines of a multi-rank group unless the caller asks for the collective
    explicit_p2p = exchange == "p2p"
    if exchange is None:
        exchange = "p2p" if (world > 1 and hasattr(eng, "enable_p2p") and world <= 8) else "collective"
    if exchange not in ("p2p", "collective"):
        raise ValueError("exchange must be 'p2p' or 'collective'")
    use_p2p = exchange == "p2p" and world > 1
    if use_p2p and not hasattr(eng, "enable_p2p"):
        raise ValueError("exchange='p2p' needs an engine with a peer-memory mailbox (CudaMcEngine); use exchange='collective'")
    if use_p2p:
        try:
            eng.enable_p2p(group)
        except P2pUnavailable:            # every rank gets this together: all switch to the collective, or all re-raise
            if explicit_p2p:
                raise
            use_p2p = False
    if not use_p2p and getattr(eng, "p2p", None) is not None:
        eng.p2p = None            # a cached engine may carry the mailbox of an earlier p2p call
    exact = getattr(eng, "overflow", None) is not None
    if exact:
        eng.overflow.zero_()
        eng.max_candidates = engine.HAWKES_EXACT_DEFAULT_BUDGET if max_candidates is None else int(max_candidates)
    etas = np.ones(M) if etas is None else np.asarray(etas, dtype=np.float64)
    Jtot = int(offsets[-1])
    chain_out = hasattr(eng, "chain_buffers")   # CUDA engine: results stay on the device until ONE copy at the end of the chain
    if chain_out:                               # reused device buffers, inputs staged through pinned memory (no allocation per call)
        (strikes_dev, types_dev, out_dev), (strikes_pin, types_pin, out_pin) = eng.chain_buffers(Jtot)
        strikes_pin[:Jtot].numpy()[:] = strikes
        types_pin[:Jtot].numpy()[:] = types
        strikes_dev[:Jtot].copy_(strikes_pin[:Jtot], non_blocking=True)
        types_dev[:Jtot].copy_(types_pin[:Jtot], non_blocking=True)
    else:
        strikes_dev = eng.to_device(strikes, torch.float64)
        types_dev = eng.to_device(types, torch.int8)
        out_dev = None
    trace = chain_out and bool(os.environ.get("B200SV_TRACE"))     # tools/trace_multi_gpu.py: where does a sharded API call spend its time?
    if trace:
        import time as _time
        ev = [eng.torch.cuda.Event(enable_timing=True) for _ in range(2)]
        t_host = [_time.time()]
        ev[0].record()
    results = []
    t0 = 0.0
    for m in range(M):
        if grid is None:
            nsteps, dt, _ = set_time_grid(ttms[m] - t0, nb_steps_per_year)
        else:
            nsteps, dt = int(grid[m][0]), float(grid[m][1])
        t0 = ttms[m]
        moments = eng.simulate_slice(m, m == 0, nsteps, dt, float(etas[m]), is_spot_measure, float(forwards[m]), seed)
        if world > 1 and not use_p2p:
            dist.all_reduce(moments, op=dist.ReduceOp.SUM, group=group)              # exchange (1): 16 bytes
        J = int(sizes[m])
        if J == 0:
            results.append((None, None))
            continue
        jo = int(offsets[m])
        sums = eng.payoff_sums(float(ttms[m]), float(forwards[m]), strikes_dev[jo: jo + J], types_dev[jo: jo + J], J, variable_type,
                               payoff_kinds(types[jo: jo + J]))
        if world > 1 and not use_p2p:
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=group)                 # exchange (2): 24*J bytes
        if chain_out:
            eng.finalize(sums, J, float(discfactors[m]), int(nb_path if se_paths is None else se_paths), out_dev[0, jo: jo + J], out_dev[1, jo: jo + J])
            results.append((jo, J))
        else:
            prices, stds = eng.finalize(sums, J, float(discfactors[m]), int(nb_path if se_paths is None else se_paths))
            results.append((prices.clone(), stds.clone()))
    if exact:
        eng.check_overflow(group, world)          # before any price leaves the device: a stopped path biases every shard's moments
    prices_out: List[np.ndarray] = []
    stds_out: List[np.ndarray] = []
    if chain_out:
        out_pin[:, :max(Jtot, 1)].copy_(out_dev[:, :max(Jtot, 1)], non_blocking=True)     # one async D2H into pinned memory ...
        if trace:
            ev[1].record()
            t_host.append(_time.time())
        eng.torch.cuda.current_stream(eng.device).synchronize()                            # ... and the chain's only host wait
        if trace:
            t_host.append(_time.time())
            TRACE_LOG.append({"rank": rank, "t_enter": t_host[0], "t_launched": t_host[1], "t_synced": t_host[2], "gpu_ms": ev[0].elapsed_time(ev[1])})
        if use_p2p:
            eng.check_p2p()          # a timed-out exchange is an error, never a silent NaN price (ADVICE r1)
        host = out_pin.numpy()
        for r in results:
            jo, J = r if r[0] is not None else (0, 0)
            prices_out.append(host[0, jo: jo + J].copy())
            stds_out.append(host[1, jo: jo + J].copy())
    else:
        for p, s in results:
            prices_out.append(p.cpu().numpy() if p is not None else np.zeros(0))
            stds_out.append(s.cpu().numpy() if s is not None else np.zeros(0))
    if return_engine:
        return prices_out, stds_out, eng
    return prices_out, stds_out


def _fixed_randoms_chain_device(rnd, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, params_c, etas,
                                is_spot_measure, variable_type, fast=True):
    """chain MC on the fixed unit normals of ``rnd`` (a logsv_pricer.DeviceRandoms, resident in HBM): strict stepper reading W from HBM,
    re-centring moments, payoff sums, finalisation -- one stream, no host round trip until the prices are copied back."""
    import torch
    dev = rnd.device
    n = rnd.nb_path
    vt = engine.variable_code(variable_type)
    offsets, strikes, types = C.flatten_chain(strikes_ttms, optiontypes_ttms)
    with torch.cuda.device(dev):
        state = torch.zeros((3, n), dtype=torch.float64, device=dev)
        state[1].fill_(params_c.sigma0)
        mom = torch.zeros(2, dtype=torch.float64, device=dev)
        J_tot = int(offsets[-1])
        sums = torch.zeros(3 * max(J_tot, 1), dtype=torch.float64, device=dev)
        out = torch.zeros((2, max(J_tot, 1)), dtype=torch.float64, device=dev)
        strikes_dev = torch.as_tensor(strikes).to(dev)
        types_dev = torch.as_tensor(types).to(dev)
        stream = c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        ptr = lambda t: c_void_p(t.data_ptr())
        for m, ttm in enumerate(ttms):
            W0, W1 = rnd.W0s[m], rnd.W1s[m]
            C.call("b200sv_dev_logsv_step_fixed", ptr(state[0]), ptr(state[1]), ptr(state[2]), ptr(W0), ptr(W1), int(W0.shape[0]), n,
                   rnd.dts[m], byref(params_c), float(etas[m]), int(bool(is_spot_measure)), int(bool(fast)), stream)
            J, jo = int(offsets[m + 1] - offsets[m]), int(offsets[m])
            if J == 0:
                continue
            C.call("b200sv_dev_spot_moments", ptr(state[0]), n, float(forwards[m]), ptr(mom), stream)
            C.call("b200sv_dev_payoff_sums", ptr(state[0]), ptr(state[2]), n, 0, float(ttm), float(forwards[m]), ptr(strikes_dev[jo:]),
                   ptr(types_dev[jo:]), J, vt, payoff_kinds(types[jo: jo + J]), ptr(mom), ptr(sums[3 * jo:]), None, stream)
            C.call("b200sv_dev_payoff_finalize", ptr(sums[3 * jo:]), J, float(discfactors[m]), n, ptr(out[0, jo:]), ptr(out[1, jo:]), None, stream)
        host = out.cpu().numpy()
    return C.split_chain(host[0], offsets), C.split_chain(host[1], offsets)


def _fixed_randoms_chain_greeks_device(rnd, ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms, params_c, etas, is_spot_measure,
                                       variable_type):
    """_fixed_randoms_chain_device(rnd, ..., fast=True) plus the pathwise sensitivities in one call on the same stream
    (b200sv_dev_logsv_mc_chain_greeks_fixed): (prices, std errors, greeks [1+6, J], greeks_se [1+6, J], offsets), prices and std errors
    bit-identical to _fixed_randoms_chain_device's, greeks row 0 the forward delta, then engine.LOGSV_GREEK_PARAMS."""
    import torch
    dev = rnd.device
    ch = engine._chain_arrays(ttms, forwards, discfactors, strikes_ttms, optiontypes_ttms)
    if len(rnd.W0s) != ch.M:
        raise ValueError("the DeviceRandoms must hold one block of normals per maturity")
    etas = C.f64(etas)
    J, P = ch.strikes.shape[0], len(engine.LOGSV_GREEK_PARAMS)
    ptrs = lambda ws: (c_void_p * ch.M)(*(w.data_ptr() for w in ws))
    nsteps = np.array([w.shape[0] for w in rnd.W0s], dtype=np.int32)
    with torch.cuda.device(dev):
        out = torch.empty((2 * (2 + P), max(J, 1)), dtype=torch.float64, device=dev)     # [prices | std errors | greeks | greeks_se]
        ptr = lambda r: c_void_p(out[r].data_ptr())
        C.call("b200sv_dev_logsv_mc_chain_greeks_fixed", byref(params_c), *C.chain_ptrs(ch, etas), ptrs(rnd.W0s), ptrs(rnd.W1s), C.iptr(nsteps),
               C.dptr(C.f64(rnd.dts)), rnd.nb_path, int(bool(is_spot_measure)), engine.variable_code(variable_type), ptr(0), ptr(1), ptr(2),
               ptr(3 + P), c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        host = out[:, :J].cpu().numpy()
    return C.split_chain(host[0], ch.offsets), C.split_chain(host[1], ch.offsets), host[2: 3 + P].copy(), host[3 + P:].copy(), ch.offsets
