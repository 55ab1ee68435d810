"""The NumPy twin of the edge probabilities and link recommendations (tests/links_twin.py) against plain Python loops on
small hand-checked rows: the left fold in ascending component order, rows without a common component, ties in the
ranking, repeated neighbour entries and a node without two-hop candidates.  No device needed."""
import numpy as np

from links_twin import Twin


def _csr(rows, K):
    indptr, idx, val = [0], [], []
    for r in rows:
        for c in sorted(r):
            idx.append(c)
            val.append(r[c])
        indptr.append(len(idx))
    return np.array(indptr), np.array(idx, dtype=np.int64), np.array(val), K


def _loop_x(rows, u, v):
    x = 0.0
    for c in sorted(set(rows[u]) & set(rows[v])):
        x = x + rows[u][c] * rows[v][c]
    return x


ROWS = [
    {0: 0.1, 3: 0.7, 5: 1e-3},      # 0
    {3: 0.2, 5: 3.0, 6: 0.25},      # 1
    {1: 0.9},                       # 2: no component in common with 0 or 1
    {},                             # 3: all zero
    {0: 1.0, 3: 0.35},              # 4
    {0: 0.5, 3: 0.7, 5: 1e-3},      # 5
]


def test_fold_matches_the_python_loop_and_is_symmetric():
    tw = Twin(*_csr(ROWS, 8))
    n = len(ROWS)
    u, v = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    x = tw.x(u.ravel(), v.ravel())
    want = np.array([_loop_x(ROWS, a, b) for a, b in zip(u.ravel(), v.ravel())])
    assert np.array_equal(x.view(np.int64), want.view(np.int64))
    assert np.array_equal(x.reshape(n, n), x.reshape(n, n).T)
    assert x.reshape(n, n)[0, 2] == 0.0 and x.reshape(n, n)[3, 3] == 0.0
    assert x.reshape(n, n)[0, 1] == (0.7 * 0.2) + 1e-3 * 3.0          # ascending c: (0 + F_03 F_13) + F_05 F_15
    assert x.reshape(n, n)[4, 4] == 1.0 + 0.35 * 0.35


def test_fold_order_changes_the_bits():
    """The order is part of the definition: a fold in another order can give other bits."""
    rows = [{0: 0.1, 1: 0.2, 2: 0.3}, {0: 0.7, 1: 0.11, 2: 0.13}]
    tw = Twin(*_csr(rows, 3))
    x = tw.x([0], [1])[0]
    assert x == (0.1 * 0.7 + 0.2 * 0.11) + 0.3 * 0.13
    assert x == _loop_x(rows, 0, 1)


def test_probability_clamp():
    tw = Twin(*_csr(ROWS, 8))
    x = np.array([0.0, 1e-5, 0.5, 9.3, 50.0])
    p = tw.p(x)
    assert p[0] == 1.0 - 0.9999 and p[1] == 1.0 - 0.9999
    assert abs(p[2] - (1.0 - np.exp(-0.5))) <= 1e-16
    assert p[3] == 1.0 - 0.0001 and p[4] == 1.0 - 0.0001


def _loop_recommend(rowptr, col, rows, u, m):
    nb = set(col[rowptr[u]:rowptr[u + 1]].tolist())
    cand = set()
    for w in col[rowptr[u]:rowptr[u + 1]]:
        cand |= set(col[rowptr[w]:rowptr[w + 1]].tolist())
    cand -= nb | {u}
    scored = [(_loop_x(rows, u, v), v) for v in cand]
    scored = sorted([s for s in scored if s[0] > 0], key=lambda s: (-s[0], s[1]))[:m]
    return [v for _, v in scored], [x for x, _ in scored]


def test_two_hop_ranking_with_ties_and_repeated_neighbours():
    # a path 0-1-2, a star 1-{3,4,5}, repeated entries (1 appears twice in 0's list and 0 twice in 1's), an unsorted
    # list, and node 6 linked only to 2 (2's other neighbour 1 is its only two-hop candidate)
    nbrs = {0: [1, 1], 1: [5, 0, 2, 3, 4, 0], 2: [1, 6], 3: [1], 4: [1], 5: [1], 6: [2]}
    rowptr = np.cumsum([0] + [len(nbrs[u]) for u in range(7)])
    col = np.array([w for u in range(7) for w in nbrs[u]], dtype=np.int32)
    rows = [{0: 1.0, 1: 0.5}, {1: 0.2}, {0: 2.0}, {0: 1.0, 1: 0.5}, {0: 1.0, 1: 0.5}, {}, {0: 0.5}]
    tw = Twin(*_csr(rows, 2))
    for m in (1, 2, 5):
        vo, xo, found = tw.recommend(rowptr, col, None, m)
        for u in range(7):
            v_l, x_l = _loop_recommend(rowptr, col, rows, u, m)
            assert found[u] == len(v_l), (u, m)
            assert vo[u, :found[u]].tolist() == v_l and xo[u, :found[u]].tolist() == x_l, (u, m)
            assert (vo[u, found[u]:] == -1).all() and (xo[u, found[u]:] == 0).all()
    vo, xo, found = tw.recommend(rowptr, col, [0, 5], 5)
    # 0: candidates 2..5 (two hops through 1); 3 and 4 tie with x = 1.25 and come in id order, 5 has x = 0
    assert vo[0].tolist() == [2, 3, 4, -1, -1] and xo[0, :3].tolist() == [2.0, 1.25, 1.25]
    assert found[1] == 0 and (vo[1] == -1).all()          # 5 holds an all-zero row: nothing with x > 0
