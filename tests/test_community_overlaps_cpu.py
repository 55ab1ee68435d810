"""The NumPy twin of the community overlaps (tests/community_overlaps_twin.py) on the CPU: hand-worked covers, random F
against intersections of Python sets built straight from the membership rule, ties at the row maximum, zero rows, the
Jaccard index of both zero-row modes, min_shared and symmetry."""
import numpy as np
import pytest

from community_overlaps_twin import community_overlaps


def _csr(F):
    F = np.asarray(F, dtype=np.float64)
    nz = F != 0.0
    indptr = np.zeros(len(F) + 1, dtype=np.int64)
    np.cumsum(nz.sum(axis=1), out=indptr[1:])
    rows, cols = np.nonzero(nz)
    return indptr, cols.astype(np.int32), F[rows, cols]


def _sets(F, delta):
    """Per community, the set of non-zero rows in it (the rule of include/bigclam_b200.h), and the zero rows."""
    F = np.asarray(F, dtype=np.float64)
    K = F.shape[1]
    comm = [set() for _ in range(K)]
    zero = []
    for u, row in enumerate(F):
        mx = row.max()
        if mx == 0.0:
            zero.append(u)
            continue
        for c in range(K):
            if (row[c] == mx) if mx < delta else (row[c] >= delta):
                comm[c].add(u)
    return comm, zero


def _by_sets(F, delta, min_shared, everywhere):
    comm, zero = _sets(F, delta)
    K, z = len(comm), len(zero) if everywhere else 0
    ptr, other, shared, jac = [0], [], [], []
    size = np.array([len(s) + z for s in comm], dtype=np.int64)
    for c in range(K):
        for d in range(K):
            a = len(comm[c] & comm[d])
            if d != c and a >= min_shared:
                other.append(d)
                shared.append(a + z)
                jac.append((a + z) / (size[c] + size[d] - (a + z)))
        ptr.append(len(other))
    return dict(ptr=np.array(ptr, dtype=np.int64), other=np.array(other, dtype=np.int32), shared=np.array(shared, dtype=np.int32),
                size=size, jaccard=np.array(jac, dtype=np.float64), zero_rows=len(zero))


def _same(g, h):
    for key in ("ptr", "other", "shared", "size", "jaccard"):
        x, y = np.asarray(g[key]), np.asarray(h[key])
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), key
    assert g["zero_rows"] == h["zero_rows"]


# rows: {0, 1}; {0, 2}; fmax 0.3 < delta, ties {1, 2}; a zero row; {3}; {0, 1, 2}
HAND = [[0.9, 0.8, 0.0, 0.0],
        [0.6, 0.0, 0.7, 0.0],
        [0.2, 0.3, 0.3, 0.0],
        [0.0, 0.0, 0.0, 0.0],
        [0.0, 0.0, 0.0, 0.9],
        [0.5, 0.5, 0.5, 0.1]]


def test_hand_cover():
    g = community_overlaps(*_csr(HAND), 4, 0.5, zero_rows_everywhere=False)
    # M_0 = {0, 1, 5}, M_1 = {0, 2, 5}, M_2 = {1, 2, 5}, M_3 = {4}: every pair of 0, 1, 2 shares two rows
    assert g["ptr"].tolist() == [0, 2, 4, 6, 6]
    assert g["other"].tolist() == [1, 2, 0, 2, 0, 1]
    assert g["shared"].tolist() == [2] * 6
    assert g["size"].tolist() == [3, 3, 3, 1]
    assert g["zero_rows"] == 1
    assert g["jaccard"].tolist() == [0.5] * 6                    # 2 / (3 + 3 - 2)
    _same(g, _by_sets(HAND, 0.5, 1, False))


def test_hand_cover_as_coded():
    """The zero row is in every community: 3 shared of 4 + 4 - 3; community 3 still lists no pair (min_shared applies
    to the non-zero rows), although it shares the zero row with every other."""
    g = community_overlaps(*_csr(HAND), 4, 0.5)
    assert g["shared"].tolist() == [3] * 6 and g["size"].tolist() == [4, 4, 4, 2]
    assert g["jaccard"].tolist() == [0.6] * 6
    assert g["ptr"][4] == g["ptr"][3]
    _same(g, _by_sets(HAND, 0.5, 1, True))


def test_ties_at_the_row_maximum():
    """fmax < delta: every entry equal to the maximum is a membership; above delta only entries >= delta are."""
    F = [[0.1, 0.1, 0.1], [0.1, 0.1, 0.05], [2.0, 0.1, 1.0]]
    g = community_overlaps(*_csr(F), 3, 0.5, zero_rows_everywhere=False)
    # M_0 = {0, 1, 2}, M_1 = {0, 1}, M_2 = {0, 2}
    assert g["other"].tolist() == [1, 2, 0, 2, 0, 1]
    assert g["shared"].tolist() == [2, 2, 2, 1, 2, 1]
    g = community_overlaps(*_csr(F), 3, float("inf"), zero_rows_everywhere=False)
    # delta = inf: every row goes to its maximum entries: M_0 = {0, 1, 2}, M_1 = {0, 1}, M_2 = {0}
    assert g["other"].tolist() == [1, 2, 0, 2, 0, 1] and g["shared"].tolist() == [2, 1, 2, 1, 1, 1]


def test_min_shared():
    g = community_overlaps(*_csr(HAND), 4, 0.5, min_shared=3, zero_rows_everywhere=False)
    assert len(g["other"]) == 0 and (g["ptr"] == 0).all() and g["size"].tolist() == [3, 3, 3, 1]
    g = community_overlaps(*_csr(HAND), 4, 0.5, min_shared=2, zero_rows_everywhere=True)
    assert g["shared"].tolist() == [3] * 6


@pytest.mark.parametrize("seed", range(6))
def test_random_against_sets(seed):
    rng = np.random.default_rng(seed)
    n, K = int(rng.integers(1, 60)), int(rng.integers(1, 12))
    F = rng.random((n, K)) * (rng.random((n, K)) < 0.4)
    F[rng.random(n) < 0.2] = 0.0
    F[rng.random(n) < 0.2, :] = 0.25                              # ties below delta
    for delta in (0.5, 0.1, float("inf")):
        for min_shared in (1, 2, n + 1):
            for everywhere in (True, False):
                g = community_overlaps(*_csr(F), K, delta, min_shared, everywhere)
                _same(g, _by_sets(F, delta, min_shared, everywhere))
                # symmetric: (c, d, a) listed iff (d, c, a) is
                rows = np.repeat(np.arange(K), np.diff(g["ptr"]))
                fwd = set(zip(rows.tolist(), g["other"].tolist(), g["shared"].tolist()))
                assert fwd == {(d, c, a) for c, d, a in fwd}
