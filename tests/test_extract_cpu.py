"""The NumPy twin of the grouped communities (tests/extract_twin.py) against the dense rule as coded
(np.where(fmax < delta, F == fmax, F >= delta), Bigclamv2.scala:225-228) on random F with the rows the rule has to get
right, and communities.group() against communities.extract()'s form."""
import numpy as np
import pytest
import scipy.sparse as sp

from extract_twin import dense_member, extract_grouped


def edge_rows_F(n, K, seed, delta):
    """Random F (about 6 non-zeros a row) with: all-zero rows, a tie at a maximum below delta, an entry exactly delta,
    a row maximum exactly delta, 1e-300 entries, rows at MAX_F_ (1000) and a full row (no implicit zeros)."""
    rng = np.random.default_rng(seed)
    F = rng.random((n, K)) * (rng.random((n, K)) < min(1.0, 6.0 / K))
    F[0] = 0.0
    F[5] = 0.0
    F[1] = 0.0
    F[1, 0] = F[1, K - 1] = delta / 2                       # tie below delta
    F[2] = 0.0
    F[2, K // 2] = delta                                     # the maximum is delta
    F[3, 0] = delta                                          # an entry exactly delta
    F[3, K - 1] = 2 * delta
    F[4] = 0.0
    F[4, K - 1] = 1e-300
    F[6] = np.where(rng.random(K) < 0.5, 1000.0, 0.0)
    F[6, 0] = 1000.0
    F[7] = rng.random(K) * 0.5 * delta + 1e-3                # full row, all below delta
    return F


def _regroup_dense(M):
    return [np.flatnonzero(M[:, c]).astype(np.int32) for c in range(M.shape[1])]


@pytest.mark.parametrize("K", [1, 2, 37, 200, 1025])
@pytest.mark.parametrize("delta", [0.3, 0.9, float("inf")])
def test_twin_matches_dense_rule(K, delta):
    n = 300
    d = delta if np.isfinite(delta) else 0.4
    F = edge_rows_F(n, K, seed=K, delta=d)
    m = sp.csr_matrix(F)
    m.eliminate_zeros()
    comptr, members, zero_rows = extract_grouped(m.indptr, m.indices, m.data, K, delta)
    assert comptr[0] == 0 and comptr[-1] == len(members)
    M = dense_member(F, delta)
    zero = ~F.any(axis=1)
    assert np.array_equal(zero_rows, np.flatnonzero(zero))
    assert M[zero].all()                                     # as coded, a zero row is in every community
    for c, want in enumerate(_regroup_dense(M & ~zero[:, None])):
        got = members[comptr[c]:comptr[c + 1]]
        assert np.array_equal(got, want), c
        assert (np.diff(got) > 0).all()


def test_group_matches_extract_form():
    from bigclam_apachespark_b200 import communities as Cm
    K, delta = 37, 0.5
    F = edge_rows_F(200, K, seed=3, delta=delta)
    m = sp.csr_matrix(F)
    m.eliminate_zeros()
    M = dense_member(F, delta)
    comms, cids = Cm.group(*extract_grouped(m.indptr, m.indices, m.data, K, delta))
    want = [(c, idx) for c, idx in enumerate(_regroup_dense(M)) if len(idx)]
    assert list(cids) == [c for c, _ in want]
    assert all(np.array_equal(a, b) and a.dtype == np.int32 for a, (_, b) in zip(comms, want))
    comms0, cids0 = Cm.group(*extract_grouped(m.indptr, m.indices, m.data, K, delta), zero_rows_everywhere=False)
    zero = ~F.any(axis=1)
    want0 = [(c, idx) for c, idx in enumerate(_regroup_dense(M & ~zero[:, None])) if len(idx)]
    assert list(cids0) == [c for c, _ in want0]
    assert all(np.array_equal(a, b) for a, (_, b) in zip(comms0, want0))
