"""NumPy/SciPy restatement of the community scores (bigclam_community_stats, csrc/bigclam_sparse.cuh
community_stats_kernel) from F as CSR rows (BigClam.F_csr()), delta, the graph and the zero-row mode.  M is the n x K
membership matrix of the extraction rule (tests/extract_twin.py), the all-zero rows in every column (zero_rows = True)
or in none; A counts neighbour-list entries (A[u, v] = how often v is in u's list):
    size = M.sum(0),   volume = M^T deg,   internal = ((A @ M) * M).sum(0),
    conductance = conductanceLocalMin's formula (bigclam4-7.scala:64-67) with cut_S = volume - internal,
                  vol_S = internal, sigma = the number of list entries."""
import numpy as np
import scipy.sparse as sp

from extract_twin import extract_grouped


def membership(indptr, indices, values, K, delta, zero_rows):
    """The n x K membership matrix M (CSR, int64 ones) of extract_grouped's communities."""
    n = len(indptr) - 1
    comptr, members, zr = extract_grouped(indptr, indices, values, K, delta)
    rows = [members.astype(np.int64)]
    cols = [np.repeat(np.arange(K, dtype=np.int64), np.diff(comptr))]
    if zero_rows and len(zr):
        rows.append(np.repeat(zr.astype(np.int64), K))
        cols.append(np.tile(np.arange(K, dtype=np.int64), len(zr)))
    r, c = np.concatenate(rows), np.concatenate(cols)
    return sp.csr_matrix((np.ones(len(r), dtype=np.int64), (r, c)), shape=(n, K))


def conductance(volume, internal, sigma):
    """bigclam4-7.scala:64-67 on integer counts, element by element, as the GPU computes it."""
    cut_S = (np.asarray(volume) - np.asarray(internal)).astype(np.float64)
    vol_S = np.asarray(internal).astype(np.float64)
    vol_T = float(sigma) - vol_S - cut_S * 2
    with np.errstate(divide="ignore", invalid="ignore"):
        q = cut_S / np.fmin(vol_S, vol_T)
    return np.where(vol_S == 0, 0.0, np.where(vol_T == 0, 1.0, q))


def community_stats(indptr, indices, values, K, delta, rowptr, col, zero_rows=True):
    """dict(size, volume, internal: int64[K], conductance: float64[K])."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    n = len(rowptr) - 1
    M = membership(indptr, indices, values, K, delta, zero_rows)
    deg = np.diff(rowptr)
    A = sp.csr_matrix((np.ones(len(col), dtype=np.int64), col, rowptr), shape=(n, n))   # duplicates add up
    size = np.asarray(M.sum(axis=0)).ravel().astype(np.int64)
    volume = (M.T @ deg).astype(np.int64)
    internal = np.asarray((A @ M).multiply(M).sum(axis=0)).ravel().astype(np.int64)
    return dict(size=size, volume=volume, internal=internal, conductance=conductance(volume, internal, rowptr[-1]))
