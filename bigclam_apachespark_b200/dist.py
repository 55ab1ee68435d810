"""Node-partitioned hot path across the GPUs of one box (one process per GPU, torch.distributed).

The reference's only parallelism is Spark data-parallel `map` over nodes with the whole F matrix
broadcast to every executor each call (codes/bigclam4-7.scala:154) and driver-side reduces
(:191-192, :219).  The H100 equivalent (DESIGN.md (e)):

  * every rank keeps the CSR and a replica of F (n x ld fp64, double-buffered) in its own HBM;
    rank r owns the contiguous node range [bounds[r], bounds[r+1]) (balanced by neighbour-list
    entries) and runs the step kernel on those rows only (Jacobi: it reads the old replica);
  * one all-reduce (sum) of the partial reductions [sum(old-new) rows (ld) | - | llh | n_updated]
    replaces the driver-side reduce of :191-192 and :219;
  * the owners' new rows are exchanged so that every replica holds the new F (replaces the
    re-broadcast of F at the next call, :154).  `exchange="p2p"` (GPUs): the step kernel itself
    stores every changed row into the peers' replicas (CUDA IPC peer memory over NVLink) — the exchange
    is fused into the compute kernel; `"delta"` all-gathers only the accepted rows with NCCL; `"full"`
    broadcasts every owner's row range.

The collectives go through torch.distributed (NCCL over NVLink on GPUs; gloo in the CPU tests, where
a test-side engine stands in for the C-ABI context).  The engine interface is the multi-GPU part of
include/bigclam_b200.h: set_owned_range / step_local / finish_local / llh_local / device_state.
"""
from __future__ import annotations

import ctypes as C
import os
import time

import numpy as np


def partition_by_nnz(rowptr: np.ndarray, world: int) -> np.ndarray:
    """Contiguous node ranges with ~equal neighbour-list entries (+1 per node so that empty rows
    still count).  Returns bounds[world + 1]."""
    n = len(rowptr) - 1
    w = rowptr.astype(np.int64) + np.arange(n + 1, dtype=np.int64)      # cumulative (deg + 1)
    targets = w[-1] * np.arange(1, world, dtype=np.float64) / world
    cuts = np.searchsorted(w, targets, side="left")
    bounds = np.concatenate([[0], cuts, [n]]).astype(np.int64)
    return np.maximum.accumulate(bounds)


class _DevMem:
    """Wraps a raw device pointer so torch can view it (CUDA array interface v3)."""

    def __init__(self, ptr: int, n_doubles: int):
        self.__cuda_array_interface__ = {"shape": (int(n_doubles),), "typestr": "<f8",
                                         "data": (int(ptr), False), "version": 3}


class _DevMemI8:
    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "|i1", "data": (int(ptr), False), "version": 3}


def deal_all_by_degree(rowptr: np.ndarray, world: int):
    """Owned node sets of all ranks: the degree-sorted node list dealt to the least loaded rank (load = neighbour-list
    entries + 1 per node, ties to the lowest rank) — the same rule as bigclam_multi_create.  The few thousand largest
    nodes go one by one (a hub can hold a sizeable part of a rank's edges); the long tail of similar degrees is dealt
    in snake order, which keeps the loads level.  Every rank gets the same mix of hubs and leaves."""
    deg = np.diff(rowptr).astype(np.int64)
    order = np.argsort(-deg, kind="stable")
    n = len(order)
    head = min(n, 4096 * world)
    owner = np.empty(n, dtype=np.int32)
    load = np.zeros(world, dtype=np.int64)
    for q in range(head):
        r = int(np.argmin(load))
        owner[q] = r
        load[r] += deg[order[q]] + 1
    if head < n:
        # snake deal of the tail, starting with the currently least loaded ranks
        ranks = np.argsort(load, kind="stable").astype(np.int32)
        k = np.arange(n - head)
        pos = k % (2 * world)
        pos = np.where(pos < world, pos, 2 * world - 1 - pos)
        owner[head:] = ranks[pos]
    return [np.sort(order[owner == r]).astype(np.int32) for r in range(world)]


def deal_by_degree(rowptr: np.ndarray, rank: int, world: int) -> np.ndarray:
    """Owned node set of `rank` (see deal_all_by_degree)."""
    return deal_all_by_degree(rowptr, world)[rank]


class CudaEngine:
    """The C-ABI context of one rank (libbigclam_b200.so) behind the engine interface."""

    def __init__(self, solver, lo: int, hi: int, nodes=None, owned_counts=None, rank: int = 0, pool_words=None):
        """owned_counts (sparse rows only): the number of owned nodes of every rank, so that each rank can place
        its part of the output pool behind the parts of the lower ranks (bigclam_set_pool_region)."""
        import torch
        from . import _lib
        self.torch = torch
        self.lib = _lib.load()
        self.check = _lib.check
        self.s = solver
        self.ctx = solver._need()
        self.sparse = bool(solver.flags & _lib.F_SPARSE_ROWS)
        if nodes is None:
            self.check(self.lib.bigclam_set_owned_range(self.ctx, lo, hi), self.ctx)
        else:
            nodes = np.ascontiguousarray(nodes, dtype=np.int32)
            self.check(self.lib.bigclam_set_owned_nodes(self.ctx, nodes.ctypes.data, len(nodes)), self.ctx)
        if self.sparse and owned_counts is not None:
            ld = (solver.K + 3) & ~3
            row_words = _lib.sparse_node_words(ld)        # a full row block + a full delta block per owned node
            cap = C.c_int64()
            self.check(self.lib.bigclam_get_pool_capacity(self.ctx, C.byref(cap)), self.ctx)
            cap_words = cap.value
            if pool_words is not None:
                cap_words = min(cap_words, int(pool_words))       # the smallest pool of all ranks (caller's all-reduce)
            total = int(sum(owned_counts))
            if total * row_words <= cap_words:                    # worst case fits: a region can never overflow
                base = int(sum(owned_counts[:rank])) * row_words
                size = int(owned_counts[rank]) * row_words
            else:                                                 # shares in proportion to the owned nodes (overflow is reported)
                starts = [(cap_words * int(sum(owned_counts[:r])) // total) & ~1 for r in range(len(owned_counts) + 1)]
                base, size = starts[rank], starts[rank + 1] - starts[rank]
            self.check(self.lib.bigclam_set_pool_region(self.ctx, base, size), self.ctx)
        self.lo, self.hi = int(lo), int(hi)
        self._views = {}
        self.n, self.k = solver.n, solver.K
        self.ld = (solver.K + 3) & ~3            # row pitch of the dense layout == length of the partial-sum vectors' D part

    def _view(self, ptr, count):
        return self.torch.as_tensor(_DevMem(ptr, count), device="cuda")

    def _cached(self, ptr, count):
        v = self._views.get((ptr, count))
        if v is None:
            v = self._views[(ptr, count)] = self._view(ptr, count)
        return v

    def state(self):
        f, fn, sf, ld = self.s.device_state()
        return (self._cached(f, self.n * ld).view(self.n, ld), self._cached(fn, self.n * ld).view(self.n, ld),
                self._cached(sf, ld))

    def step_local(self):
        p = C.c_void_p()
        self.check(self.lib.bigclam_step_local(self.ctx, C.byref(p)), self.ctx)
        return self._cached(p.value, 2 * self.ld + 2)

    def llh_local(self):
        p = C.c_void_p()
        self.check(self.lib.bigclam_llh_local(self.ctx, C.byref(p)), self.ctx)
        return self._view(p.value, 2 * self.ld + 2)

    def finish_local(self, sync: bool = True):
        if not sync:
            self.check(self.lib.bigclam_finish_local(self.ctx, None, None), self.ctx)
            return None, None
        llh = C.c_double()
        nupd = C.c_int64()
        self.check(self.lib.bigclam_finish_local(self.ctx, C.byref(llh), C.byref(nupd)), self.ctx)
        return llh.value, nupd.value

    def collect_timing(self):
        self.check(self.lib.bigclam_collect_timing(self.ctx), self.ctx)
        return self.s.kernel_time()

    def rollback(self):
        self.check(self.lib.bigclam_rollback(self.ctx), self.ctx)

    def open_peers(self, dist, rank: int, world: int):
        """Exchange the CUDA IPC handles of the F double buffers and map every peer's replica, so that
        the step kernel can push changed rows straight into them over NVLink (exchange="p2p")."""
        torch = self.torch
        nbytes = 64 * int(self.lib.bigclam_ipc_handle_count(self.ctx))        # 2 handles (dense F) or 4 (sparse rows)
        mine = (C.c_ubyte * nbytes)()
        self.check(self.lib.bigclam_ipc_export(self.ctx, mine), self.ctx)
        t = torch.frombuffer(bytearray(mine), dtype=torch.uint8).cuda()
        allh = torch.empty(world * nbytes, dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(allh, t)
        buf = (C.c_ubyte * (world * nbytes)).from_buffer_copy(allh.cpu().numpy().tobytes())
        self.check(self.lib.bigclam_ipc_open_peers(self.ctx, world, rank, buf), self.ctx)

    def open_xchg(self, dist, rank: int, world: int):
        """Fused collective (sparse rows): exchange buffers of every rank mapped through CUDA IPC; afterwards
        step_local publishes this rank's sums to all ranks and finish_local / llh_finish add them up on the device
        (rank order: the same bits everywhere) — no all-reduce by the host framework on the data path."""
        torch = self.torch
        mine = (C.c_ubyte * 128)()
        self.check(self.lib.bigclam_xchg_export(self.ctx, world, rank, mine), self.ctx)
        t = torch.frombuffer(bytearray(mine), dtype=torch.uint8).cuda()
        allh = torch.empty(world * 128, dtype=torch.uint8, device="cuda")
        dist.all_gather_into_tensor(allh, t)
        buf = (C.c_ubyte * (world * 128)).from_buffer_copy(allh.cpu().numpy().tobytes())
        self.check(self.lib.bigclam_xchg_open_peers(self.ctx, buf), self.ctx)
        self.fused = True

    def llh_finish(self) -> float:
        v = C.c_double()
        self.check(self.lib.bigclam_llh_finish_local(self.ctx, C.byref(v)), self.ctx)
        return v.value

    def set_uset(self, mask_ptr):
        self.check(self.lib.bigclam_set_uset(self.ctx, mask_ptr), self.ctx)

    def mark_all_changed(self):
        self.check(self.lib.bigclam_mark_all_changed(self.ctx), self.ctx)

    def changed_owned(self):
        """Global ids (int64, device) of the owned rows whose step was accepted by the last step_local
        (context created with record_accepted=True)."""
        p = C.c_void_p()
        self.check(self.lib.bigclam_device_accepted(self.ctx, C.byref(p)), self.ctx)
        acc = self.torch.as_tensor(_DevMemI8(p.value, self.n), device="cuda")
        return self.torch.nonzero(acc[self.lo:self.hi] >= 0).flatten() + self.lo


class DistBigClam:
    """backtrackingLineSearchs over node partitions; every rank calls every method collectively."""

    def __init__(self, engine, rowptr: np.ndarray, rank: int, world: int, bounds=None, exchange: str = "full"):
        import torch.distributed as dist
        self.dist = dist
        self.e = engine
        self.rank, self.world = rank, world
        self.bounds = partition_by_nnz(rowptr, world) if bounds is None else np.asarray(bounds)
        self.exchange = exchange
        self.last_n_updated = 0
        self.last_delta_rows = 0
        self._prev_changed = None
        self._need_sync = True          # first delta step: bring the non-owned rows of F_next up to date
        if exchange == "delta":
            import torch
            self.torch = torch
        if getattr(engine, "sparse", False) and exchange != "p2p":
            raise ValueError("sparse rows travel through the fused peer stores only (exchange='p2p')")
        if exchange == "p2p":
            engine.open_peers(self.dist, rank, world)
            if getattr(engine, "sparse", False) and world > 1 and os.environ.get("BIGCLAM_NCCL_ALLREDUCE", "0") != "1":
                engine.open_xchg(self.dist, rank, world)          # fused collective instead of the NCCL all-reduce
        self.fused = bool(getattr(engine, "fused", False))

    @property
    def owned(self):
        return int(self.bounds[self.rank]), int(self.bounds[self.rank + 1])

    def _exchange_rows(self, F_cur, F_next):
        """Afterwards every replica of F_next holds the new F."""
        if self.exchange == "p2p":
            return      # the step kernel already pushed the changed rows into the peers' replicas
        if self.exchange == "full":
            # owners publish their whole row range
            for r in range(self.world):
                lo, hi = int(self.bounds[r]), int(self.bounds[r + 1])
                if hi > lo:
                    self.dist.broadcast(F_next[lo:hi], src=r)
            return
        # delta: only rows whose step was accepted travel.  F_next is the buffer that held the state
        # before the previous step, so the rows the PREVIOUS step changed are stale in it: refresh the
        # non-owned ones from the current state, then apply this step's accepted rows.
        torch = self.torch
        lo, hi = self.owned
        if self._need_sync:
            mask = torch.ones(F_next.shape[0], dtype=torch.bool, device=F_next.device)
            mask[lo:hi] = False
            F_next[mask] = F_cur[mask]
            self._need_sync = False
        elif self._prev_changed is not None and self._prev_changed.numel():
            pc = self._prev_changed
            stale = pc[(pc < lo) | (pc >= hi)]
            if stale.numel():
                F_next[stale] = F_cur[stale]
        idx = self.e.changed_owned()                                   # global ids, int64, on the device
        cnt = torch.tensor([idx.numel()], dtype=torch.int64, device=F_next.device)
        counts = torch.empty(self.world, dtype=torch.int64, device=F_next.device)
        self.dist.all_gather_into_tensor(counts, cnt)
        maxc = int(counts.max().item())
        self.last_delta_rows = int(counts.sum().item())
        if maxc == 0:
            self._prev_changed = idx
            return
        ld = F_next.shape[1]
        send_idx = torch.full((maxc,), -1, dtype=torch.int64, device=F_next.device)
        send_rows = torch.zeros((maxc, ld), dtype=F_next.dtype, device=F_next.device)
        send_idx[: idx.numel()] = idx
        send_rows[: idx.numel()] = F_next[idx]
        all_idx = torch.empty(self.world * maxc, dtype=torch.int64, device=F_next.device)
        all_rows = torch.empty((self.world * maxc, ld), dtype=F_next.dtype, device=F_next.device)
        self.dist.all_gather_into_tensor(all_idx, send_idx)
        self.dist.all_gather_into_tensor(all_rows, send_rows)
        valid = all_idx >= 0
        gidx = all_idx[valid]
        F_next[gidx] = all_rows[valid]
        self._prev_changed = gidx

    def step_nollh(self, sync: bool = True):
        """PRE + line search + row swap + sumF update.  Returns the LLH of the state BEFORE this
        call (== the LLH the previous call returns, the fused identity) and n_updated; with
        sync=False nothing is read back and the host does not wait (None, None)."""
        part = self.e.step_local()
        if not self.fused:
            self.dist.all_reduce(part)                  # sum over ranks (:191-192, :219); fused: done by finish_local
        if self.exchange != "p2p":
            F_cur, F_next, _ = self.e.state()
            self._exchange_rows(F_cur, F_next)
        llh_pre, nupd = self.e.finish_local(sync)       # sumF -= sum(old - new) on every rank
        self.last_n_updated = nupd
        return llh_pre, nupd

    def loglikelihood(self) -> float:
        part = self.e.llh_local()
        if self.fused:
            return self.e.llh_finish()
        self.dist.all_reduce(part)
        return float(part[2 * self.e.ld].item())

    def backtrackingLineSearchs(self) -> float:
        """One full call: returns the LLH after the update (:196-219)."""
        self.step_nollh()
        return self.loglikelihood()

    def run(self, variant: int = 4, rel_tol: float = 1e-4, max_outer: int = 0):
        """SGDFindC / MBSGD with the LLH of call t taken from call t+1's PRE pass.  Returns
        (returned LLH, calls, trace).  Like bigclam_run, a converged loop has executed one
        speculative extra step; it is rolled back by the engine flip (state after `calls` calls)."""
        trace = []
        LLHold = None
        calls = 0
        while True:
            if max_outer and calls >= max_outer:
                L = self.loglikelihood()                 # LLH of the last call (tail pass)
                trace.append(L)
                return L, calls, trace
            llh_pre, _ = self.step_nollh()
            calls += 1
            if calls == 1:
                if variant == 2:
                    LLHold = llh_pre                     # LLHold = loglikelihood()   (Bigclamv2.scala:204)
                continue
            L, c = llh_pre, calls - 1                    # LLH returned by call c
            trace.append(L)
            test = True
            if variant == 4 and c == 1:
                LLHold, test = L, False                  # bigclam4-7.scala:228
            if variant == 3 and c == 1:
                LLHold = 0.0                             # bigclamv3-7.scala:207
            if test:
                with np.errstate(divide="ignore", invalid="ignore"):
                    conv = bool(np.abs(1.0 - np.float64(L) / np.float64(LLHold)) < rel_tol)   # :237
                if conv:
                    self.e.rollback()                    # drop the speculative call just made
                    return (LLHold if variant == 4 else L), c, trace
                LLHold = L


# ------------------------------------------------------------------------------------------------
SETTLE_STEPS = 6         # untimed steps after the W warm-up steps in both arms of bench.py (N = 1: 3 x (retile + 2 steps))


def bench_main(args, load_workload, alg_bytes, hbm_peak, ClockSampler, base_config):
    """bench.py for N > 1: launched by torchrun, one rank per GPU; torch.distributed (NCCL) is the plumbing (rendezvous,
    IPC-handle all-gather, timing reductions), the data path is the step kernel's NVLink row stores plus the fused
    collective (bigclam_xchg_*)."""
    import json

    import torch
    import torch.distributed as dist

    from . import BigClam

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    K = args.k
    rp, col, F0 = load_workload(args.graph, K)
    n, nnz = len(rp) - 1, len(col)
    sparse = args.layout == "sparse"
    b = BigClam(device=local, time_kernels=True, record_accepted=True, sparse_rows=sparse)
    b.set_graph(rp, col).set_K(K)
    stream = torch.cuda.current_stream()
    b.set_stream(stream.cuda_stream)
    b.set_F(F0)
    bounds = partition_by_nnz(rp, world)
    exchange = os.environ.get("BIGCLAM_EXCHANGE", "p2p")
    deal = deal_all_by_degree(rp, world) if exchange == "p2p" else None
    nodes = deal[rank] if deal is not None else None
    counts = [len(x) for x in deal] if deal is not None else None
    pool_words = None
    if sparse:
        from . import _lib
        cap = C.c_int64()
        _lib.check(_lib.load().bigclam_get_pool_capacity(b._need(), C.byref(cap)), b._ctx)
        t_cap = torch.tensor([cap.value], dtype=torch.int64, device="cuda")
        dist.all_reduce(t_cap, op=dist.ReduceOp.MIN)
        pool_words = int(t_cap.item())
    eng = CudaEngine(b, int(bounds[rank]), int(bounds[rank + 1]), nodes=nodes, owned_counts=counts, rank=rank, pool_words=pool_words)
    d = DistBigClam(eng, rp, rank, world, bounds, exchange=exchange)

    for _ in range(args.warmup):
        d.step_nollh()
    settle = SETTLE_STEPS if sparse else 0
    for _ in range(settle):                  # (untimed) the same window of the trajectory as the single-GPU arm of bench.py,
        d.step_nollh()                       # which lets its tile cut settle over this many steps after the warm-up
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    launches = 0
    sync = d.exchange != "p2p"       # the NCCL delta exchange sizes its buffers on the host
    per_step = 4 if d.fused else 3   # step kernel, reduction, (combine,) finish
    for _ in range(args.steps):
        d.step_nollh(sync=sync)
        launches += per_step
    llh_end = d.loglikelihood()              # the LLH of the last call (tail pass, inside the timed region)
    launches += 3
    e1.record(stream)
    dist.barrier()
    torch.cuda.synchronize()
    clocks = sampler.stop() if rank == 0 else None
    t = torch.tensor([e0.elapsed_time(e1)], device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    total_ms = float(t.item())
    kms, nk, _ = eng.collect_timing()        # step-kernel events of the timed (asynchronous) region
    # e2e: the reference-facing call with host buffers (uset mask H2D from pinned memory, one full
    # backtrackingLineSearchs per step, LLH and n_updated read back by the host)
    n_e2e = min(args.steps, 20)
    mask = torch.ones(n, dtype=torch.uint8).pin_memory()
    dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_e2e):
        eng.set_uset(mask.data_ptr())
        d.backtrackingLineSearchs()
    torch.cuda.synchronize()
    te = torch.tensor([(time.perf_counter() - t0) * 1e3 / n_e2e], device="cuda", dtype=torch.float64)
    dist.all_reduce(te, op=dist.ReduceOp.MAX)
    e2e_ms = float(te.item())
    eng.set_uset(None)
    per_rank = torch.zeros(world, device="cuda", dtype=torch.float64)
    per_rank[rank] = kms / max(nk, 1)
    dist.all_reduce(per_rank)
    own0 = deal[0] if deal is not None else np.arange(bounds[0], bounds[1])
    own_nnz = int(np.diff(rp)[own0].sum())
    own_n = len(own0)
    ms_per_step = total_ms / args.steps
    if rank == 0:
        peak, peak_src = hbm_peak()
        value = nnz / (ms_per_step * 1e-3)
        print(json.dumps({
            "metric": "edges/sec in F-gradient step", "value": value, "unit": "edges/s",
            "unit_note": "directed neighbour-list entries per second (2 per undirected edge)", "value_undirected_edges_per_s": value / 2,
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step,
            "untimed_steps_before_timing": args.warmup + settle,
            "iters_per_sec": 1e3 / ms_per_step, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "SNAP topology (package data) or generated R-MAT + synthetic F0",
            "config": base_config(args.graph, K, n, nnz, args.layout),
            "parallelism": f"node-partitioned x{world} ({'degree-sorted nodes dealt to the least loaded rank' if exchange == 'p2p' else 'nnz-balanced contiguous ranges'}), "
                           f"F replicated, rows pushed into the peers' replicas by the step kernel (NVLink), sums [sum(old-new), llh, n_updated] by "
                           f"{'the fused device-side collective (peer stores + flags)' if d.fused else 'an NCCL all-reduce'}",
            "l2": "sparse rows: working set L2-resident by design, no flush" if sparse else "inputs larger than L2, no flush",
            "llh_end": llh_end, "clocks": clocks, "gpu_launches": launches,
            "rank_step_kernel_ms": [round(float(x), 4) for x in per_rank.tolist()],
            "roofline": {"bound": "hbm", "achieved": alg_bytes(own_n, own_nnz, K) / (float(per_rank[0]) * 1e-3) / 1e9,
                         "peak": peak, "unit": "GB/s", "frac": alg_bytes(own_n, own_nnz, K) / (float(per_rank[0]) * 1e-3) / 1e9 / peak,
                         "traffic": None, "kernel": "step kernel of rank 0 (owned rows only, incl. NVLink pushes)", "peak_source": peak_src,
                         "f_layout": args.layout},
            "e2e": {"value": nnz / (e2e_ms * 1e-3), "unit": "edges/s", "h2d_bytes_per_step": int(n) * world, "d2h_bytes_per_step": 16 * world,
                    "ms_per_step": e2e_ms, "note": "per step and rank: bigclam_set_uset (mask H2D from pinned memory) + DistBigClam.backtrackingLineSearchs(): "
                                                   "step kernel + reduction + collective + sumF + separate LLH pass + collective; LLH and n_updated read back "
                                                   "by every rank each step; F replicas stay resident"},
            "cpu_baseline": None,
        }))
    dist.destroy_process_group()
