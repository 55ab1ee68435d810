"""The caller behind the hot path (SURVEY.md §8f-3): community extraction as coded in
codes/Bigclamv2.scala:223-230, and an Avg-F1 scorer against ground-truth communities (the reference has
no evaluator; its thesis names Avg-F1 as the metric, p.21)."""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

from . import _lib
from .graphs import FIXTURE_DIR


def delta_threshold(n_vertices: int, count: int) -> float:
    """`e = 2.0*count/(N*(N-1)); e = sqrt(-log(1-e))` (Bigclamv2.scala:223-224).  In the script `count` is
    `G.collectEdges(EdgeDirection.Either).count`, i.e. the number of vertices that have edges; the thesis
    (def. 9, p.19) uses |E|.  Pass whichever you mean."""
    e = 2.0 * count / (n_vertices * (n_vertices - 1.0))
    return math.sqrt(-math.log(1.0 - e))


def extract(solver, delta: float):
    """Returns (communities: list of int32 arrays of vertex indices, one per non-empty community id;
    community ids; member matrix n x K uint8).  `Com.flatMap{(x,y) => y.map(c => (c,x))}.groupByKey()` (:229-230)."""
    n, k = solver.n, solver.K
    member = np.empty((n, k), dtype=np.uint8)
    fmax = np.empty(n, dtype=np.float64)
    _lib.check(_lib.load().bigclam_extract(solver._need(), C.c_double(delta), member.ctypes.data, fmax.ctypes.data), solver._ctx)
    comms, cids = [], []
    for c in range(k):
        idx = np.flatnonzero(member[:, c]).astype(np.int32)
        if len(idx):
            comms.append(idx)
            cids.append(c)
    return comms, np.array(cids), member


def group(comptr, members, zero_rows, zero_rows_everywhere: bool = True):
    """BigClam.extract_communities()'s CSR as (communities: list of int32 arrays, community ids), the form extract()
    returns: non-empty communities only, each ascending.  zero_rows_everywhere=True merges the all-zero rows into every
    community, as coded; False leaves them out."""
    comptr = np.asarray(comptr, dtype=np.int64)
    members = np.asarray(members, dtype=np.int32)
    zero_rows = np.asarray(zero_rows, dtype=np.int32)
    merge = zero_rows_everywhere and len(zero_rows) > 0
    comms, cids = [], []
    for c in range(len(comptr) - 1):
        idx = members[comptr[c]:comptr[c + 1]]
        if merge:
            idx = np.union1d(idx, zero_rows).astype(np.int32)
        if len(idx):
            comms.append(idx)
            cids.append(c)
    return comms, np.array(cids)


def load_ground_truth(name: str = "com-amazon.cmty"):
    """Ground-truth communities fixture (dense vertex indices), written by tests/golden/make_fixtures.py."""
    z = np.load(os.path.join(FIXTURE_DIR, name + ".npz"))
    sizes, deltas = z["sizes"], z["deltas"]
    out, p = [], 0
    for s in sizes:
        out.append(np.cumsum(deltas[p:p + s]).astype(np.int32))
        p += s
    return out


def avg_f1(detected, truth, n: int) -> float:
    """Average F1 (Yang & Leskovec): 0.5 * (mean over truth of best F1 against detected + mean over detected of
    best F1 against truth), through one sparse incidence product."""
    import scipy.sparse as sp

    def inc(cs):
        rows = np.concatenate([np.full(len(c), i, dtype=np.int64) for i, c in enumerate(cs)]) if cs else np.zeros(0, dtype=np.int64)
        cols = np.concatenate(cs).astype(np.int64) if cs else np.zeros(0, dtype=np.int64)
        return sp.csr_matrix((np.ones(len(rows), dtype=np.float64), (rows, cols)), shape=(len(cs), n))

    if not detected or not truth:
        return 0.0
    A, B = inc(detected), inc(truth)
    inter = (A @ B.T).tocsr()                       # |C_i ∩ G_j|, only overlapping pairs are stored
    sa = np.asarray(A.sum(axis=1)).ravel()
    sb = np.asarray(B.sum(axis=1)).ravel()
    coo = inter.tocoo()
    f1 = 2.0 * coo.data / (sa[coo.row] + sb[coo.col])
    best_a = np.zeros(len(detected))
    best_b = np.zeros(len(truth))
    np.maximum.at(best_a, coo.row, f1)
    np.maximum.at(best_b, coo.col, f1)
    return 0.5 * (best_a.mean() + best_b.mean())
