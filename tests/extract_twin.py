"""NumPy restatement of the grouped communities (bigclam_extract_grouped, csrc/bigclam_sparse.cuh MemberPred) from F as
CSR rows (BigClam.F_csr(): ascending indices, no stored zeros).  With fmax_u the maximum of row u over all K components
(the zeros not stored included), u is a member of c iff F_uc == fmax_u when fmax_u < delta, else F_uc >= delta.  An
all-zero row is listed once in zero_rows; any other row's memberships are among its non-zeros (F >= 0, delta > 0)."""
import numpy as np


def extract_grouped(indptr, indices, values, K, delta):
    """(comptr int64[K + 1], members int32[nnz], zero_rows int32[z]), each list ascending."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    values = np.asarray(values, dtype=np.float64)
    n = len(indptr) - 1
    assert delta > 0 and (values >= 0).all()
    cnt = np.diff(indptr)
    row = np.repeat(np.arange(n, dtype=np.int64), cnt)
    fmax = np.zeros(n)
    if len(values):
        np.maximum.at(fmax, row, values)                    # implicit zeros: F >= 0, so the maximum starts at 0
    fm = fmax[row]
    take = np.where(fm < delta, values == fm, values >= delta) & (values != 0)
    c, u = indices[take], row[take]
    o = np.lexsort((u, c))
    comptr = np.zeros(int(K) + 1, dtype=np.int64)
    np.cumsum(np.bincount(c, minlength=int(K)), out=comptr[1:])
    zero_rows = np.flatnonzero(fmax == 0).astype(np.int32)
    return comptr, u[o].astype(np.int32), zero_rows


def dense_member(F, delta):
    """The as-coded rule on a dense n x K F (the form the existing extraction tests write)."""
    F = np.asarray(F, dtype=np.float64)
    fmax = F.max(axis=1, keepdims=True)
    return np.where(fmax < delta, F == fmax, F >= delta)
