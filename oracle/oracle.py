"""ctypes front-end of the CPU oracle (oracle/bigclam_oracle.c).

TEST INFRASTRUCTURE ONLY — see the header of bigclam_oracle.c.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this
module.  The product package never does.

PARITY UNPINNED: the reference has no golden vectors and cannot run here (no JVM/Spark); the C
restatement is pinned only against the independent NumPy twin (numpy_twin.py) and the
self-consistency properties in tests/.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")


class OracleParams(C.Structure):
    """Mirror of `oracle_params` (bigclam_oracle.c); defaults = bigclam4-7.scala:22-26,39-43."""

    _fields_ = [
        ("k", C.c_int32),
        ("max_inter", C.c_int32),
        ("alpha", C.c_double),
        ("beta", C.c_double),
        ("min_p", C.c_double),
        ("max_p", C.c_double),
        ("min_f", C.c_double),
        ("max_f", C.c_double),
    ]


def make_params(k, alpha=0.05, beta=0.1, max_inter=15, min_p=0.0001, max_p=0.9999,
                min_f=0.0, max_f=1000.0) -> OracleParams:
    return OracleParams(int(k), int(max_inter), alpha, beta, min_p, max_p, min_f, max_f)


def _cpu_tag() -> str:
    try:
        with open("/proc/cpuinfo") as fh:
            for line in fh:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return "unknown"


def build(force: bool = False, out_dir: str | None = None) -> str:
    """Compile liboracle.so from the C restatement (gcc + OpenMP, -O3 -march=native); returns its path.  The
    library is rebuilt when the source is newer or when it was built for another CPU model (a copied tree may
    land on a host whose CPU differs).  out_dir: where a rebuild goes instead of oracle/ (callers that must not
    write into the tree); the library found current is used from wherever it is."""
    global _LIB_PATH
    src = os.path.join(_HERE, "bigclam_oracle.c")
    tag = _cpu_tag()
    try:
        with open(os.path.join(os.path.dirname(_LIB_PATH), "liboracle.host")) as fh:
            same_cpu = fh.read().strip() == tag
    except OSError:
        same_cpu = False
    if force or not same_cpu or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        d = out_dir or _HERE
        os.makedirs(d, exist_ok=True)
        out = os.path.join(d, "liboracle.so")
        subprocess.run(["make", "-C", _HERE, "-B", f"OUT={out}"], check=True, stdout=subprocess.DEVNULL)
        with open(os.path.join(d, "liboracle.host"), "w") as fh:
            fh.write(tag + "\n")
        _LIB_PATH = out
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        dp = C.POINTER(C.c_double)
        L.oracle_step_sizes.argtypes = [C.c_double, C.c_int32, dp]
        L.oracle_step_sizes.restype = None
        L.oracle_llh.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(OracleParams),
                                 C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_llh.restype = C.c_double
        L.oracle_step.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(OracleParams),
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_void_p, C.c_void_p]
        L.oracle_step.restype = C.c_double
        L.oracle_colsum.argtypes = [C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
        L.oracle_colsum.restype = None
        L.oracle_run.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(OracleParams),
                                 C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_int64,
                                 dp, C.c_void_p, C.c_int64]
        L.oracle_run.restype = C.c_int64
        L.oracle_armijo_margins.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(OracleParams), C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.oracle_armijo_margins.restype = None
        L.oracle_num_threads.restype = C.c_int32
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _chk(rowptr, col, F, k):
    assert rowptr.dtype == np.int64 and col.dtype == np.int32
    assert rowptr.flags.c_contiguous and col.flags.c_contiguous
    n = rowptr.shape[0] - 1
    if F is not None:
        assert F.dtype == np.float64 and F.flags.c_contiguous and F.shape == (n, k), (F.shape, n, k)
    return n


def step_sizes(beta=0.1, max_inter=15) -> np.ndarray:
    out = np.empty(max_inter + 1, dtype=np.float64)
    lib().oracle_step_sizes(beta, max_inter, out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def colsum(F: np.ndarray) -> np.ndarray:
    n, k = F.shape
    out = np.empty(k, dtype=np.float64)
    lib().oracle_colsum(n, k, _p(F), _p(out))
    return out


def llh(rowptr, col, F, sumF, params: OracleParams, per_node: bool = False):
    n = _chk(rowptr, col, F, params.k)
    pn = np.empty(n, dtype=np.float64) if per_node else None
    v = lib().oracle_llh(n, _p(rowptr), _p(col), C.byref(params), _p(F), _p(sumF), _p(pn))
    return (v, pn) if per_node else v


@dataclass
class StepResult:
    F: np.ndarray
    sumF: np.ndarray
    llh: float
    n_updated: int
    accepted: np.ndarray      # int8 n: index of accepted step size, -1 = row unchanged
    trials: np.ndarray        # int8 n: candidates evaluated
    grad: np.ndarray | None   # PRE block outputs (optional)
    llh_u: np.ndarray | None


def step(rowptr, col, F, sumF, params: OracleParams, node_mask=None, early_exit=True,
         want_pre=False) -> StepResult:
    """One backtrackingLineSearchs call on (F, sumF); inputs are not modified."""
    n = _chk(rowptr, col, F, params.k)
    k = params.k
    sumF2 = np.array(sumF, dtype=np.float64, copy=True)
    Fo = np.empty_like(F)
    acc = np.empty(n, dtype=np.int8)
    tr = np.empty(n, dtype=np.int8)
    grad = np.empty((n, k), dtype=np.float64) if want_pre else None
    llh_u = np.empty(n, dtype=np.float64) if want_pre else None
    if node_mask is not None:
        node_mask = np.ascontiguousarray(node_mask, dtype=np.uint8)
    nupd = C.c_int64(0)
    v = lib().oracle_step(n, _p(rowptr), _p(col), C.byref(params), _p(F), _p(sumF2), _p(node_mask),
                          _p(Fo), C.byref(nupd), _p(acc), _p(tr), 1 if early_exit else 0,
                          _p(grad), _p(llh_u))
    return StepResult(Fo, sumF2, v, nupd.value, acc, tr, grad, llh_u)


def run(rowptr, col, F, sumF, params: OracleParams, variant=4, rel_tol=1e-4, max_outer=0,
        trace_cap=4096):
    """Outer loop (SGDFindC / MBSGD).  Returns (F, sumF, llh, calls, trace)."""
    n = _chk(rowptr, col, F, params.k)
    F2 = np.array(F, copy=True)
    s2 = np.array(sumF, dtype=np.float64, copy=True)
    trace = np.full(trace_cap, np.nan)
    out = C.c_double(0.0)
    calls = lib().oracle_run(n, _p(rowptr), _p(col), C.byref(params), _p(F2), _p(s2), variant,
                             rel_tol, max_outer, C.byref(out), _p(trace), trace_cap)
    return F2, s2, out.value, calls, trace[:min(calls, trace_cap)]


def armijo_margins(rowptr, col, F, sumF, params: OracleParams, nodes):
    """Margins llh'(s_j) - (llh_u + alpha s_j |g|^2) of every candidate for the given nodes, and their llh_u."""
    n = _chk(rowptr, col, F, params.k)
    nodes = np.ascontiguousarray(nodes, dtype=np.int64)
    m = np.empty((len(nodes), params.max_inter + 1), dtype=np.float64)
    lu = np.empty(len(nodes), dtype=np.float64)
    sumF = np.ascontiguousarray(sumF, dtype=np.float64)
    lib().oracle_armijo_margins(n, _p(rowptr), _p(col), C.byref(params), _p(F), _p(sumF), _p(nodes), len(nodes), _p(m), _p(lu))
    return m, lu


def num_threads() -> int:
    return int(lib().oracle_num_threads())


# --------------------------------------------------------------------------------------------
# Independent (pure NumPy) edge-list reader used to check the product's C++ reader.
# Semantics restated from the reference's call sites: GraphLoader.edgeListFile
# (bigclam4-7.scala:45) + collectNeighborIds(EdgeDirection.Either) (bigclam4-7.scala:50):
#   * lines starting with '#' and blank lines are skipped, fields split on whitespace (CRLF safe)
#   * every edge LINE (src, dst) contributes dst to src's list and src to dst's list
#     (multiplicity kept: Email-Enron lists both directions => every neighbour twice)
#   * vertex ids are arbitrary longs; the hot path only uses them as keys (SURVEY T10), so
#     they are relabelled to 0..n-1 in ascending id order.
# multiplicity="dedup" collapses repeated neighbours and drops self loops (simple graph).
# --------------------------------------------------------------------------------------------
def read_edge_list(path: str, multiplicity: str = "dedup"):
    src, dst = [], []
    with open(path, "rb") as fh:
        for line in fh:
            line = line.strip()
            if not line or line.startswith(b"#"):
                continue
            parts = line.split()
            if len(parts) < 2:
                raise ValueError(f"Invalid line: {line!r}")
            src.append(int(parts[0]))
            dst.append(int(parts[1]))
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    ids = np.unique(np.concatenate([src, dst]))
    s = np.searchsorted(ids, src)
    d = np.searchsorted(ids, dst)
    return csr_from_pairs(len(ids), s, d, multiplicity), ids


def csr_from_pairs(n, s, d, multiplicity="dedup"):
    s = np.asarray(s, dtype=np.int64)
    d = np.asarray(d, dtype=np.int64)
    a = np.concatenate([s, d])
    b = np.concatenate([d, s])
    if multiplicity == "dedup":
        keep = a != b
        a, b = a[keep], b[keep]
        key = np.unique(a * n + b)
        a, b = key // n, key % n
    elif multiplicity == "keep":
        order = np.lexsort((b, a))
        a, b = a[order], b[order]
    else:
        raise ValueError(multiplicity)
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(rowptr, a + 1, 1)
    rowptr = np.cumsum(rowptr)
    return rowptr.astype(np.int64), b.astype(np.int32)
