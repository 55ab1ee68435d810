"""NumPy/SciPy restatement of the community overlaps (bigclam_community_overlaps, csrc/bigclam_sparse.cuh
community_overlaps_kernel) from F as CSR rows (BigClam.F_csr()), delta and min_shared.  M is the membership matrix of
the extraction rule (tests/community_stats_twin.py) over the non-zero rows only; shared = M^T M off the diagonal, the
entries >= min_shared kept; the zero rows are counted once and, in the as-coded mode, added to every shared count and
every size.  Returns what BigClam.community_overlaps returns."""
import numpy as np

from community_stats_twin import membership
from extract_twin import extract_grouped


def community_overlaps(indptr, indices, values, K, delta, min_shared=1, zero_rows_everywhere=True):
    """dict(ptr int64[K + 1], other int32[nnz], shared int32[nnz], size int64[K], jaccard float64[nnz], zero_rows)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    M = membership(indptr, indices, values, K, delta, zero_rows=False).tocsc()
    z = len(extract_grouped(indptr, indices, values, K, delta)[2])
    size = np.asarray(M.sum(axis=0)).ravel().astype(np.int64)
    S = (M.T @ M).tocoo()                                        # K x K, |M_c ∩ M_d|
    keep = (S.row != S.col) & (S.data >= min_shared)
    r, d, a = S.row[keep].astype(np.int64), S.col[keep].astype(np.int64), S.data[keep]
    o = np.lexsort((d, r))                                       # by row, then d ascending
    ptr = np.zeros(K + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=K), out=ptr[1:])
    other = d[o].astype(np.int32)
    shared = a[o].astype(np.int32)
    if zero_rows_everywhere and z:
        shared = shared + np.int32(z)
        size = size + z
    rows = np.repeat(np.arange(K), np.diff(ptr))
    jaccard = shared / (size[rows] + size[other] - shared)
    return dict(ptr=ptr, other=other, shared=shared, size=size, jaccard=jaccard, zero_rows=z)
