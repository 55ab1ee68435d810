"""Host-side mirror of the reference's spark-shell surface for the hot path.

The reference is three flat spark-shell scripts; the names below are the script-level
variables and functions a user of codes/bigclam4-7.scala (and the older v2/v3 scripts) edits
and calls.  Every method that computes goes through the C ABI (libbigclam_b200.so); nothing
here does arithmetic on F.

    script variable / function                     here
    numCore            bigclam4-7.scala:14         BigClam(numCore=...)  (Spark partitions -> unused on one GPU)
    minCom/maxCom/divCom :16-20                    BigClam(minCom, maxCom, divCom), Kset()
    alpha, beta, MaxInter :22-26                   BigClam(alpha, beta, MaxInter)
    GraphLoader.edgeListFile + collectNeighborIds :45,:50   BigClam.load_edge_list / read_edge_list
    conductanceLocalMin() / Sbc :58-75             BigClam.conductanceLocalMin()
    K = sc.broadcast(i); initNeighborComF(K) :249-250       BigClam.initNeighborComF(K)  (or set_K(K); set_F(F0))
    backtrackingLineSearchs(uset) :152             BigClam.backtrackingLineSearchs(uset=None)
    loglikelihood()    bigclamv3-7.scala:106       BigClam.loglikelihood()
    SGDFindC()         bigclam4-7.scala:225        BigClam.SGDFindC()
    MBSGD()            bigclamv3-7.scala:206 / Bigclamv2.scala:203   BigClam.MBSGD(version=3|2)
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import Graph, Params, check


def Kset(minCom: int, maxCom: int, divCom: int, int_division: bool = True) -> list[int]:
    """Geometric grid of K values, bigclam4-7.scala:116-133.

    `maxCom/minCom` is an Int division in the Scala (both are Int vars, :16-18); the pasted REPL
    value at :268 (minCom=50, maxCom=200, divCom=15) is only reproduced with that quirk, so it is
    the default.  int_division=False gives the real-valued ratio the thesis describes.
    """
    ratio = (maxCom // minCom) if int_division else (maxCom / minCom)
    conGap = math.exp(math.log(ratio) / divCom)
    ks = [int(minCom)]
    x = int(minCom)
    while True:
        xtemp = int(x * conGap)
        if xtemp == x:
            xtemp += 1
        x = xtemp
        if x >= maxCom:
            break
        ks.append(x)
    ks.append(int(maxCom))
    return ks


def read_edge_list(path: str, multiplicity: str = "dedup"):
    """GraphLoader.edgeListFile + collectNeighborIds(Either) (bigclam4-7.scala:45,50) via the C++ reader.

    Returns (rowptr int64[n+1], col int32[nnz], ids int64[n]).  multiplicity: "keep" = literal
    GraphX (one neighbour entry per edge line and endpoint), "dedup" = simple undirected graph.
    """
    lib = _lib.load()
    g = Graph()
    err = C.create_string_buffer(512)
    mult = {"keep": 0, "dedup": 1}[multiplicity]
    rc = lib.bigclam_graph_read_edgelist(path.encode(), mult, C.byref(g), err, len(err))
    if rc != _lib.OK:
        raise _lib.BigclamError(rc, err.value.decode())
    try:
        n, nnz = g.n, g.nnz
        rowptr = np.ctypeslib.as_array(g.rowptr, shape=(n + 1,)).copy()
        col = np.ctypeslib.as_array(g.col, shape=(max(nnz, 1),))[:nnz].copy()
        ids = np.ctypeslib.as_array(g.ids, shape=(max(n, 1),))[:n].copy()
    finally:
        lib.bigclam_graph_free(C.byref(g))
    return rowptr, col, ids


class BigClam:
    """One solver instance == the global state of one spark-shell session of the reference."""

    def __init__(self, numCore: int = 36, minCom: int = 1000, maxCom: int = 9000, divCom: int = 100,
                 alpha: float = 0.05, beta: float = 0.1, MaxInter: int = 15, device: int = -1,
                 time_kernels: bool = False, record_accepted: bool = False, verbose: bool = False,
                 sparse_rows: bool = False, numGPUs: int = 1, devices=None, exhaustive_linesearch: bool = False):
        self.numCore, self.minCom, self.maxCom, self.divCom = numCore, minCom, maxCom, divCom
        self.alpha, self.beta, self.MaxInter = alpha, beta, MaxInter
        self.MIN_P_, self.MAX_P_, self.MIN_F_, self.MAX_F_ = 0.0001, 0.9999, 0.0, 1000.0   # :40-43
        self.device = device
        self.flags = (_lib.F_TIME_KERNELS if time_kernels else 0) | (_lib.F_RECORD_ACCEPTED if record_accepted else 0)
        if sparse_rows:       # F as sparse rows on the device (the reference's BSV[Double]); K <= 16384
            self.flags |= _lib.F_SPARSE_ROWS
        if exhaustive_linesearch:     # evaluate every candidate of every node (no bounds), like the reference's cartesian (:172-181)
            self.flags |= _lib.F_LS_EXHAUSTIVE
        self.verbose = verbose
        self.K = None
        self.rowptr = self.col = self.ids = None
        self._ctx = None
        self._F0 = None
        # numGPUs > 1: all GPUs of the box behind one handle (bigclam_multi_*, sparse rows, fused NVLink collective) —
        # the role `numCore` plays in the script (:14); devices: CUDA ordinals, default 0 .. numGPUs-1
        self.numGPUs = int(numGPUs)
        self.devices = None if devices is None else [int(d) for d in devices]
        self._multi = None
        if self.numGPUs > 1:
            self.flags |= _lib.F_SPARSE_ROWS

    # ---- graph (collectNeighbor / Neightborbc, :50-51) ----
    def load_edge_list(self, path: str, multiplicity: str = "dedup"):
        self.set_graph(*read_edge_list(path, multiplicity))
        return self

    def set_graph(self, rowptr, col, ids=None):
        self._free()
        self.rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
        self.col = np.ascontiguousarray(col, dtype=np.int32)
        self.ids = ids
        self.Sbc = None
        return self

    @property
    def n(self) -> int:
        return len(self.rowptr) - 1

    # ---- K / F (K = sc.broadcast(i); initNeighborComF(K), :249-250) ----
    def set_K(self, K: int):
        if self.rowptr is None:
            raise ValueError("load a graph first")
        self._free()
        self.K = int(K)
        lib = _lib.load()
        p = Params()
        check(lib.bigclam_default_params(C.byref(p), self.K))
        p.max_inter, p.alpha, p.beta = self.MaxInter, self.alpha, self.beta
        p.min_p, p.max_p, p.min_f, p.max_f = self.MIN_P_, self.MAX_P_, self.MIN_F_, self.MAX_F_
        # above K = 1024 only sparse rows hold F (the dense engine stops there): a K sweep crosses 1024 on its own
        p.device, p.flags = self.device, self.flags | (_lib.F_SPARSE_ROWS if self.K > 1024 else 0)
        ctx = C.c_void_p()
        if self.numGPUs > 1:
            devs = None
            if self.devices is not None:
                devs = (C.c_int32 * self.numGPUs)(*self.devices[:self.numGPUs])
            rc = lib.bigclam_multi_create(C.byref(ctx), self.n, self.rowptr.ctypes.data, self.col.ctypes.data, C.byref(p),
                                          self.numGPUs, devs)
            if rc != _lib.OK:
                raise _lib.BigclamError(rc, (lib.bigclam_multi_last_error(None) or b"").decode())
            self._multi = ctx
            return self
        check(lib.bigclam_create(C.byref(ctx), self.n, self.rowptr.ctypes.data, self.col.ctypes.data, C.byref(p)))
        self._ctx = ctx
        return self

    def _mcheck(self, rc):
        if rc != _lib.OK:
            raise _lib.BigclamError(rc, (_lib.load().bigclam_multi_last_error(self._multi) or b"").decode())

    def _call(self, name, *args):
        """bigclam_multi_<name>(multi handle, *args) on a multi handle, else bigclam_<name>(context, *args)."""
        lib = _lib.load()
        if self._multi is not None:
            self._mcheck(getattr(lib, "bigclam_multi_" + name)(self._multi, *args))
        else:
            check(getattr(lib, "bigclam_" + name)(self._need(), *args), self._ctx)

    def _set_sumF(self, sumF):
        if sumF is not None:
            sumF = np.ascontiguousarray(sumF, dtype=np.float64)
            self._call("set_sumF", sumF.ctypes.data)
        return self

    def set_F_csr(self, indptr, indices, values, K=None, sumF=None):
        """F <- CSR rows (the reference's RDD[(Long, BSV[Double])], :97-104); sumF <- column sums unless given.
        With sparse_rows=True no dense n x K image is built anywhere."""
        indptr = np.ascontiguousarray(indptr, dtype=np.int64)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        values = np.ascontiguousarray(values, dtype=np.float64)
        if K is not None and (self._ctx is None or int(K) != self.K):
            self.set_K(int(K))
        if len(indptr) != self.n + 1 or len(indices) != indptr[-1] or len(values) != indptr[-1]:
            raise ValueError("CSR arrays do not describe n rows")
        self._call("set_F_csr", indptr.ctypes.data, indices.ctypes.data, values.ctypes.data)
        return self._set_sumF(sumF)

    def F_csr(self):
        """Current F as (indptr, indices, values): ascending indices inside a row, no stored zeros."""
        nnz = C.c_int64()
        self._call("get_F_nnz", C.byref(nnz))
        indptr = np.empty(self.n + 1, dtype=np.int64)
        indices = np.empty(max(nnz.value, 1), dtype=np.int32)
        values = np.empty(max(nnz.value, 1), dtype=np.float64)
        self._call("get_F_csr", indptr.ctypes.data, indices.ctypes.data, values.ctypes.data)
        return indptr, indices[:nnz.value], values[:nnz.value]

    def set_F(self, F, sumF=None):
        """F <- n x K (the result of initNeighborComF); sumF <- column sums unless given."""
        if hasattr(F, "tocsr"):                 # scipy.sparse matrix
            m = F.tocsr()
            return self.set_F_csr(m.indptr, m.indices, m.data, K=m.shape[1], sumF=sumF)
        F = np.ascontiguousarray(F, dtype=np.float64)
        if (self._ctx is None and self._multi is None) or F.shape[1] != self.K:
            self.set_K(F.shape[1])
        if F.shape != (self.n, self.K):
            raise ValueError(f"F must be {self.n} x {self.K}")
        self._call("set_F", F.ctypes.data)
        return self._set_sumF(sumF)

    def replica_F(self, rank: int = 0) -> np.ndarray:
        """numGPUs > 1: the F replica of one rank (all replicas are identical after every call)."""
        out = np.empty((self.n, self.K), dtype=np.float64)
        self._mcheck(_lib.load().bigclam_multi_get_F(self._multi, int(rank), out.ctypes.data))
        return out

    def replica_sumF(self, rank: int = 0) -> np.ndarray:
        out = np.empty(self.K, dtype=np.float64)
        self._mcheck(_lib.load().bigclam_multi_get_sumF(self._multi, int(rank), out.ctypes.data))
        return out

    @property
    def F(self) -> np.ndarray:
        if self._multi is not None:
            return self.replica_F(0)
        out = np.empty((self.n, self.K), dtype=np.float64)
        check(_lib.load().bigclam_get_F(self._need(), out.ctypes.data), self._ctx)
        return out

    @property
    def sumF(self) -> np.ndarray:
        if self._multi is not None:
            return self.replica_sumF(0)
        out = np.empty(self.K, dtype=np.float64)
        check(_lib.load().bigclam_get_sumF(self._need(), out.ctypes.data), self._ctx)
        return out

    # ---- init of F (conductanceLocalMin + initNeighborComF, bigclam4-7.scala:58-108) ----
    def conductanceLocalMin(self, on_gpu=None):
        """Ranked seed candidates (dense vertex indices) and the conductance of every vertex.  on_gpu: True = the
        CUDA kernel (csrc/initf_gpu.cu), False = the host path, None = the GPU when there is one."""
        lib = _lib.load()
        cond = np.empty(self.n, dtype=np.float64)
        seeds = np.empty(self.n, dtype=np.int32)
        cnt = C.c_int64()
        if on_gpu is None:
            on_gpu = lib.bigclam_device_count() > 0
        if on_gpu:
            rc = lib.bigclam_conductance_seeds_gpu(self.n, self.rowptr.ctypes.data, self.col.ctypes.data, self.device,
                                                   cond.ctypes.data, seeds.ctypes.data, C.byref(cnt))
        else:
            rc = lib.bigclam_conductance_seeds(self.n, self.rowptr.ctypes.data, self.col.ctypes.data, cond.ctypes.data,
                                               seeds.ctypes.data, C.byref(cnt))
        if rc != _lib.OK:
            raise _lib.BigclamError(rc, "bigclam_conductance_seeds failed")
        self.Sbc = seeds[:cnt.value].copy()             # `Sbc` of the script (:75), reused for every K
        self.conductance = cond
        return self.Sbc

    def init_F(self, K: int, include_self: bool = False, pad_seed: int = 1234):
        """initNeighborComF(K) (:81-108) built on the GPU, straight into the context: the F and sumF bits that loading
        the host's n x K F0 gives (:105-107), with nothing n x K allocated on either side.  (Re)creates the context when
        K changes and ranks the seeds (conductanceLocalMin) when that has not been done."""
        if getattr(self, "Sbc", None) is None:
            self.conductanceLocalMin()
        if (self._ctx is None and self._multi is None) or int(K) != self.K:
            self.set_K(int(K))
        seeds = np.ascontiguousarray(self.Sbc, dtype=np.int32)
        self._call("init_F", seeds.ctypes.data, len(seeds), 1 if include_self else 0, C.c_uint64(pad_seed))
        return self

    def initNeighborComF(self, K: int, include_self: bool = False, pad_seed: int = 1234):
        """Builds F0 from the ranked seeds and loads it (sets F and sumF like the script, :105-107); returns F0 (n x K)."""
        return self.init_F(K, include_self, pad_seed).F

    # ---- the hot path ----
    def backtrackingLineSearchs(self, uset=None) -> float:
        """bigclam4-7.scala:152-223.  uset: None = all vertices (as the reference always passes),
        else an iterable of dense vertex indices."""
        mask_ptr = None
        if uset is not None:
            mask = np.zeros(self.n, dtype=np.uint8)
            mask[np.asarray(list(uset), dtype=np.int64)] = 1
            mask_ptr = mask.ctypes.data
        llh = C.c_double()
        nupd = C.c_int64()
        self._call("step", mask_ptr, C.byref(llh), C.byref(nupd))
        self.last_n_updated = nupd.value
        return llh.value

    def loglikelihood(self) -> float:
        """bigclamv3-7.scala:106-120 / Bigclamv2.scala:187-200."""
        llh = C.c_double()
        self._call("loglikelihood", C.byref(llh))
        return llh.value

    def _run(self, variant: int, rel_tol: float, max_outer: int, trace_cap: int = 65536):
        trace = np.full(trace_cap, np.nan)
        llh = C.c_double()
        calls = C.c_int64()
        self._call("run", variant, rel_tol, max_outer, C.byref(llh), C.byref(calls), trace.ctypes.data, trace_cap)
        self.last_calls = calls.value
        self.last_trace = trace[:min(calls.value, trace_cap)]
        return llh.value

    def SGDFindC(self, rel_tol: float = 0.0001, max_outer: int = 0) -> float:
        """bigclam4-7.scala:225-243: one call for LLHold, then loop until |1 - new/old| < 1e-4;
        returns LLHold.  max_outer=0: no iteration cap, like the reference."""
        ret = self._run(4, rel_tol, max_outer)
        if self.verbose:
            for i, v in enumerate(self.last_trace[1:], start=1):
                print("-------Inter: " + str(i) + " LLH: " + repr(float(v)))          # :236
        return ret

    def MBSGD(self, version: int = 3, rel_tol: float = 0.0001, max_outer: int = 0) -> None:
        """bigclamv3-7.scala:206-222 (LLHold = 0.0) or Bigclamv2.scala:203-219 (LLHold = loglikelihood())."""
        if version not in (2, 3):
            raise ValueError("version must be 2 or 3")
        if self.verbose:
            print("LLH: " + repr(0.0 if version == 3 else self.loglikelihood()))       # v3 :208 / v2 :205
        self._run(version, rel_tol, max_outer)
        if self.verbose:
            for i, v in enumerate(self.last_trace, start=1):
                print(" Inter: " + str(i * self.n) + " LLH: " + repr(float(v)))         # v3 :216 (i += uset.size)

    def Kset(self) -> list[int]:
        return Kset(self.minCom, self.maxCom, self.divCom)

    def sweep_K(self, rel_gain: float = 0.001, max_outer: int = 0):
        """The K sweep at the bottom of the script (bigclam4-7.scala:244-266): for K in Kset, initNeighborComF(K) (init_F),
        SGDFindC(); stop at the first K whose LLH gain over the previous K is below 0.1 % (`1 - new/old < 0.001`).
        As coded, LLHKold starts at 0.0 (the `== null` test is never true for a Double), so the first K never
        stops the sweep.  Returns (KforC, [(K, LLH), ...]); KforC is 0 when the sweep ran out of K values (:245)."""
        LLHKold, KforC, hist = 0.0, 0, []
        for i in self.Kset():
            self.init_F(i)
            LLHKnew = self.SGDFindC(max_outer=max_outer)
            if self.verbose:
                print(str(i) + " LLH: " + repr(LLHKnew))                                   # :258
            hist.append((i, LLHKnew))
            with np.errstate(divide="ignore", invalid="ignore"):
                gain = 1.0 - np.float64(LLHKnew) / np.float64(LLHKold)
            if gain < rel_gain:                                                          # :259
                KforC = i
                break
            LLHKold = LLHKnew
        return KforC, hist

    # ---- the fitted model as a model of edges: P(u,v) = 1 - exp(-F_u.F_v), clamped like :166 ----
    def edge_probability(self, u, v):
        """Affinity x = F_u.F_v and edge probability p = 1 - clamp(exp(-x), MIN_P_, MAX_P_) of the pairs (u[i], v[i]),
        computed on the GPU from the current F.  Returns (x, p) float64 arrays."""
        u = np.ascontiguousarray(u, dtype=np.int32).ravel()
        v = np.ascontiguousarray(v, dtype=np.int32).ravel()
        if len(u) != len(v):
            raise ValueError("u and v must have the same length")
        x = np.empty(len(u), dtype=np.float64)
        p = np.empty(len(u), dtype=np.float64)
        self._call("pair_affinity", u.ctypes.data, v.ctypes.data, len(u), x.ctypes.data, p.ctypes.data)
        return x, p

    def recommend(self, nodes=None, m: int = 10):
        """For each query node u (None = all nodes), the m not-yet-linked nodes at distance 2 with the largest affinity
        x > 0, by x descending then id ascending.  Returns (v, x) arrays of shape len(nodes) x m, padded with -1 and 0."""
        cnt = self.n if nodes is None else None
        ptr = None
        if nodes is not None:
            nodes = np.ascontiguousarray(nodes, dtype=np.int32).ravel()
            cnt, ptr = len(nodes), nodes.ctypes.data
        m = int(m)
        vo = np.empty((cnt, max(m, 0)), dtype=np.int32)
        xo = np.empty((cnt, max(m, 0)), dtype=np.float64)
        self._call("recommend", ptr, cnt, m, vo.ctypes.data, xo.ctypes.data, None)
        return vo, xo

    def sample_graph(self, seed, eps=0.0):
        """A graph drawn from the model on the GPU: a pair that shares a component is an edge with probability p_uv (the
        p of edge_probability), any other pair with probability eps (0 <= eps < 1; 1 - MAX_P_ is the model as coded).
        The same (F, seed, eps) gives the same graph.  Returns (rowptr int64[n + 1], col int32[nnz]): symmetric, rows
        ascending, no self loops, the shape set_graph takes."""
        seed, eps = int(seed) & 0xFFFFFFFFFFFFFFFF, float(eps)
        nnz = C.c_int64()
        self._call("sample_graph_nnz", seed, eps, C.byref(nnz))
        rowptr = np.empty(self.n + 1, dtype=np.int64)
        col = np.empty(max(nnz.value, 1), dtype=np.int32)
        self._call("sample_graph", seed, eps, rowptr.ctypes.data, col.ctypes.data)
        return rowptr, col[:nnz.value]

    def fold_in(self, rowptr, col, max_iter: int = 100, rel_tol: float = 1e-4):
        """Rows for NEW nodes with the fitted F and sumF held fixed (the `transform` of the fit), on the GPU.  Query node i
        has the neighbour list col[rowptr[i]:rowptr[i + 1]] among the fitted nodes; from a zero row, up to max_iter of the
        reference's line searches on its own objective, stopping when none passes or the LLH gains less than rel_tol
        (relative).  Nodes never see each other.  Returns (indptr int64[q + 1], indices int32[nnz], values float64[nnz],
        llh float64[q], iters int32[q]): rows ascending without zeros, the shape set_F_csr takes."""
        rowptr = np.ascontiguousarray(rowptr, dtype=np.int64).ravel()
        col = np.ascontiguousarray(col, dtype=np.int32).ravel()
        if len(rowptr) < 1:
            raise ValueError("rowptr needs q + 1 >= 1 entries")
        q = len(rowptr) - 1
        if rowptr[-1] > len(col):
            raise ValueError("rowptr[-1] is beyond col")
        max_iter, rel_tol = int(max_iter), float(rel_tol)
        nnz = C.c_int64()
        args = (q, rowptr.ctypes.data, col.ctypes.data, max_iter, rel_tol)
        self._call("fold_in_nnz", *args, C.byref(nnz))
        indptr = np.zeros(q + 1, dtype=np.int64)
        indices = np.empty(max(nnz.value, 1), dtype=np.int32)
        values = np.empty(max(nnz.value, 1), dtype=np.float64)
        llh = np.zeros(q, dtype=np.float64)
        iters = np.zeros(q, dtype=np.int32)
        self._call("fold_in", *args, indptr.ctypes.data, indices.ctypes.data, values.ctypes.data, llh.ctypes.data, iters.ctypes.data)
        return indptr, indices[:nnz.value], values[:nnz.value], llh, iters

    def extract_communities(self, delta):
        """The communities of Bigclamv2.scala:223-230 grouped by community, on the GPU, with no n x K image anywhere.
        delta > 0 (not NaN; inf allowed) and F >= 0.  Returns (comptr int64[K + 1], members int32[nnz], zero_rows
        int32[z]): community c is members[comptr[c]:comptr[c + 1]] ascending; an all-zero row is, as coded, a member of
        every community and is listed once in zero_rows (ascending) instead.  communities.group() turns this into
        communities.extract()'s lists."""
        delta = float(delta)
        nnz, z = C.c_int64(), C.c_int64()
        self._call("extract_nnz", delta, C.byref(nnz), C.byref(z))
        comptr = np.zeros(self.K + 1, dtype=np.int64)
        members = np.empty(max(nnz.value, 1), dtype=np.int32)
        zero_rows = np.empty(max(z.value, 1), dtype=np.int32)
        self._call("extract_grouped", delta, comptr.ctypes.data, members.ctypes.data, zero_rows.ctypes.data)
        return comptr, members[:nnz.value], zero_rows[:z.value]

    def community_stats(self, delta, zero_rows_everywhere=True):
        """A label-free score of every community of extract_communities(delta), on the GPU.  Returns dict(size, volume,
        internal, conductance), arrays of length K: |S_c|; the sum of deg(u) over u in S_c; the neighbour-list entries
        u -> v with u and v in S_c (entries counted with multiplicity, self loops included); and conductanceLocalMin's
        formula (bigclam4-7.scala:64-67) with cut = volume - internal, vol_S = internal and sigma = the number of list
        entries of the graph (an empty community scores 0).  zero_rows_everywhere: all-zero rows are in every community
        (as coded) or in none, the two choices of communities.group()."""
        K = self.K
        size, volume, internal = (np.zeros(K, dtype=np.int64) for _ in range(3))
        cond = np.zeros(K, dtype=np.float64)
        self._call("community_stats", float(delta), 1 if zero_rows_everywhere else 0, size.ctypes.data, volume.ctypes.data,
                   internal.ctypes.data, cond.ctypes.data)
        return dict(size=size, volume=volume, internal=internal, conductance=cond)

    def score_against(self, truth, delta, zero_rows_everywhere=True):
        """The communities of extract_communities(delta) scored against a known cover, on the GPU (bigclam_cover_scores,
        whose header comment defines every output).  truth: a list of int arrays of node ids, the form
        communities.load_ground_truth() and communities.group() return (any order; a repeated id counts once).
        zero_rows_everywhere: all-zero rows are in every detected community (as coded) or in none.  Returns dict(avg_f1,
        nmi_lfk, nmi_max, f1_detected, match_detected, f1_truth, match_truth, hcond_detected, hcond_truth): the scores
        as floats; per detected community c (length K) and per truth community t (length len(truth)) the best F1, the
        smallest id attaining it (-1: none) and H*(X_c | Y) / H*(Y_t | X) (NaN outside the NMI)."""
        K, q = self.K, len(truth)
        ptr = np.zeros(q + 1, dtype=np.int64)
        np.cumsum([len(t) for t in truth], out=ptr[1:])
        members = np.concatenate(truth).astype(np.int64) if q else np.zeros(0, dtype=np.int64)
        members[(members < 0) | (members > np.iinfo(np.int32).max)] = -1     # rejected by the call, naming the community
        members = np.ascontiguousarray(members, dtype=np.int32)
        f1_det, hc_det = np.zeros(K), np.zeros(K)
        match_det = np.zeros(K, dtype=np.int32)
        f1_truth, hc_truth = np.zeros(max(q, 1)), np.zeros(max(q, 1))
        match_truth = np.zeros(max(q, 1), dtype=np.int32)
        scores = np.zeros(3)
        self._call("cover_scores", float(delta), 1 if zero_rows_everywhere else 0, q, ptr.ctypes.data,
                   members.ctypes.data if len(members) else None, f1_det.ctypes.data, match_det.ctypes.data, f1_truth.ctypes.data,
                   match_truth.ctypes.data, hc_det.ctypes.data, hc_truth.ctypes.data, scores.ctypes.data)
        return dict(avg_f1=float(scores[0]), nmi_lfk=float(scores[1]), nmi_max=float(scores[2]), f1_detected=f1_det,
                    match_detected=match_det, f1_truth=f1_truth[:q], match_truth=match_truth[:q], hcond_detected=hc_det,
                    hcond_truth=hc_truth[:q])

    def community_overlaps(self, delta, min_shared=1, zero_rows_everywhere=True):
        """How the communities of extract_communities(delta) overlap each other, on the GPU (bigclam_community_overlaps,
        whose header comment defines the counts).  Lists, for every community c, the communities d != c that share at
        least min_shared non-zero rows with it.  Returns dict(ptr int64[K + 1], other int32[nnz], shared int32[nnz],
        size int64[K], jaccard float64[nnz], zero_rows=z): row c is other[ptr[c]:ptr[c + 1]] (ascending) with the shared
        members and the Jaccard index shared / (size_c + size_d - shared) of each pair; the output is symmetric.
        zero_rows_everywhere: the z all-zero rows are in every community (as coded) or in none.  As coded, shared and
        size include z, and a pair that is not listed still shares the z zero rows; min_shared always applies to the
        non-zero rows alone."""
        delta, min_shared = float(delta), int(min_shared)
        nnz, z = C.c_int64(), C.c_int64()
        self._call("community_overlaps_nnz", delta, min_shared, C.byref(nnz), C.byref(z))
        K = self.K
        ptr, size = np.zeros(K + 1, dtype=np.int64), np.zeros(K, dtype=np.int64)
        other, shared = np.empty(max(nnz.value, 1), dtype=np.int32), np.empty(max(nnz.value, 1), dtype=np.int32)
        self._call("community_overlaps", delta, min_shared, ptr.ctypes.data, other.ctypes.data, shared.ctypes.data, size.ctypes.data)
        other, shared = other[:nnz.value], shared[:nnz.value]
        if zero_rows_everywhere and z.value:
            shared = shared + np.int32(z.value)                 # shared + z <= n < 2^31
            size = size + z.value
        rows = np.repeat(np.arange(K), np.diff(ptr))
        jaccard = shared / (size[rows] + size[other] - shared)
        return dict(ptr=ptr, other=other, shared=shared, size=size, jaccard=jaccard, zero_rows=int(z.value))

    # ---- diagnostics ----
    def accepted(self) -> np.ndarray:
        out = np.empty(self.n, dtype=np.int8)
        check(_lib.load().bigclam_get_accepted(self._need(), out.ctypes.data), self._ctx)
        return out

    def kernel_time(self):
        ms = C.c_double()
        nstep = C.c_int64()
        nall = C.c_int64()
        if self._multi is not None:          # slowest rank's sum of step-kernel times
            self._mcheck(_lib.load().bigclam_multi_get_kernel_time(self._multi, C.byref(ms), C.byref(nstep)))
            return ms.value, nstep.value, nstep.value
        check(_lib.load().bigclam_get_kernel_time(self._need(), C.byref(ms), C.byref(nstep), C.byref(nall)), self._ctx)
        return ms.value, nstep.value, nall.value

    def retile(self):
        """Sparse rows: re-cut the tiles of small nodes for the rows' current size / the observed fallback rate
        (bigclam_run does this between its batches of 8 calls)."""
        if self._multi is None:
            check(_lib.load().bigclam_retile(self._need()), self._ctx)

    def tile_stats(self):
        """Sparse rows + time_kernels: dict(tiles_done, tiles_fallback, n_tiles, n_general_nodes, n_split_hubs)."""
        if self._multi is not None:
            raise RuntimeError("tile_stats() reads one context; with numGPUs > 1 use ls_stats() (summed over the ranks)")
        v = [C.c_int64() for _ in range(5)]
        check(_lib.load().bigclam_get_tile_stats(self._need(), *[C.byref(x) for x in v]), self._ctx)
        return dict(zip(("tiles_done", "tiles_fallback", "n_tiles", "n_general_nodes", "n_split_hubs"), (x.value for x in v)))

    def ls_stats(self):
        """Sparse rows: dict(nodes_asked, nodes_searched) of the tile path since the previous read — how many of the
        nodes that asked for a line search had a candidate the bounds could not exclude."""
        a, b = C.c_int64(), C.c_int64()
        self._call("get_ls_stats", C.byref(a), C.byref(b))          # multi handle: summed over the ranks
        return {"nodes_asked": a.value, "nodes_searched": b.value}

    def set_stream(self, cuda_stream: int):
        check(_lib.load().bigclam_set_stream(self._need(), C.c_void_p(cuda_stream)), self._ctx)

    def device_state(self):
        f, fn, sf = C.c_void_p(), C.c_void_p(), C.c_void_p()
        ld = C.c_int64()
        check(_lib.load().bigclam_device_state(self._need(), C.byref(f), C.byref(fn), C.byref(sf), C.byref(ld)), self._ctx)
        return f.value, fn.value, sf.value, ld.value

    def _need(self):
        if self._ctx is None:
            raise RuntimeError("no context: call set_K()/set_F() after loading a graph")
        return self._ctx

    def _free(self):
        if self._ctx is not None:
            _lib.load().bigclam_destroy(self._ctx)
            self._ctx = None
        if getattr(self, "_multi", None) is not None:
            _lib.load().bigclam_multi_destroy(self._multi)
            self._multi = None

    def close(self):
        self._free()

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass
