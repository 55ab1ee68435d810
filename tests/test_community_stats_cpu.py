"""The NumPy twin of the community scores (tests/community_stats_twin.py) on hand-checked graphs, against a loop over
the definition, and against the reference's own conductance on ego nets.

Ego nets: plant F_uc = 1 for u in {x_c} + N(x_c) with delta = 0.5 and the zero rows in no community; then community c is
the ego net of x_c and its conductance is conductanceLocalMin's score of x_c (bigclam4-7.scala:58-67), bit for bit,
whenever x_c's own list has no repeated entry and no self loop.  Otherwise the two differ on purpose: the reference's
ego net y = [x] ++ neighbours(x) (:55) is a list, so :63 walks a repeated neighbour's list once per repetition, while a
community is a set and walks that list once.  Neither side is wrong; test_repeated_neighbour_differs pins it."""
import numpy as np
import pytest

from community_stats_twin import community_stats, conductance
from conftest import random_graph


def _csr(rows, K):
    """F as CSR rows from a list of {component: value} dicts."""
    indptr = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
    indices = np.array([c for r in rows for c in sorted(r)], dtype=np.int32)
    values = np.array([r[c] for r in rows for c in sorted(r)], dtype=np.float64)
    return indptr, indices, values


def _graph(lists):
    rp = np.cumsum([0] + [len(x) for x in lists]).astype(np.int64)
    col = np.array([v for x in lists for v in x], dtype=np.int32)
    return rp, col


def _check(got, size, volume, internal, cond):
    assert got["size"].tolist() == size
    assert got["volume"].tolist() == volume
    assert got["internal"].tolist() == internal
    assert got["conductance"].tolist() == cond


def test_triangle_pendant_empty_community_and_zero_rows():
    # triangle 0-1-2, path 2-3-4; community 0 = the triangle, 1 = {2, 3}, 2 = nobody; node 4 is an all-zero row
    rp, col = _graph([[1, 2], [0, 2], [0, 1, 3], [2, 4], [3]])
    F = _csr([{0: 1.0}, {0: 1.0}, {0: 1.0, 1: 1.0}, {1: 1.0}, {}], 3)
    # sigma = 10.  c0: cut 1, vol_T = 10 - 6 - 2 = 2 -> 1/2.  c1: cut 3, vol_T = 10 - 2 - 6 = 2 -> 3/2.  c2: empty -> 0.
    _check(community_stats(*F, 3, 0.5, rp, col, zero_rows=False), [3, 2, 0], [7, 5, 0], [6, 2, 0], [0.5, 1.5, 0.0])
    # node 4 in every community.  c0 + 4: cut 2, vol_T = 10 - 6 - 4 = 0 -> 1.  c1 + 4: cut 2, vol_T = 2 -> 1.
    # c2 = {4}: no internal entry -> 0.
    _check(community_stats(*F, 3, 0.5, rp, col, zero_rows=True), [4, 3, 1], [8, 6, 1], [6, 4, 0], [1.0, 1.0, 0.0])


def test_self_loop_entry_counts():
    rp, col = _graph([[0, 1], [0], [1]])                                              # 0 -> 0 is an entry of 0's list
    F = _csr([{0: 2.0}, {0: 1.0}, {}], 1)
    # internal: 0 -> 0, 0 -> 1, 1 -> 0.  sigma = 4, cut 0, vol_T = 4 - 3 = 1 -> 0 / 1 = 0
    _check(community_stats(*F, 1, 0.5, rp, col, zero_rows=False), [2], [3], [3], [0.0])
    # with the zero row 2: 2 -> 1 joins; cut 0, vol_T = 0 -> 1
    _check(community_stats(*F, 1, 0.5, rp, col, zero_rows=True), [3], [4], [4], [1.0])


def test_non_symmetric_lists():
    rp, col = _graph([[1], [], [0, 1, 1]])                                            # 2 -> 1 twice; nothing points at 2
    F = _csr([{0: 1.0}, {0: 1.0, 1: 1.0}, {1: 1.0}], 2)
    # sigma = 4.  c0 = {0, 1}: 0 -> 1 only; cut 0, vol_T = 3 -> 0.  c1 = {1, 2}: 2 -> 1 twice; cut 1, vol_T = 0 -> 1
    _check(community_stats(*F, 2, 0.5, rp, col), [2, 2], [1, 3], [1, 2], [0.0, 1.0])


def _by_loops(F, delta, rp, col, zero_rows):
    """The definition written out: membership by the rule on a dense F, then one pass over every list entry."""
    fmax = F.max(axis=1, keepdims=True)
    M = np.where(fmax < delta, F == fmax, F >= delta)
    if not zero_rows:
        M &= F.any(axis=1)[:, None]
    n, K = F.shape
    size, volume, internal = M.sum(0), np.zeros(K, dtype=np.int64), np.zeros(K, dtype=np.int64)
    for u in range(n):
        volume += M[u] * (rp[u + 1] - rp[u])
        for v in col[rp[u]:rp[u + 1]]:
            internal += M[u] & M[v]
    return size, volume, internal


@pytest.mark.parametrize("zero_rows", [False, True])
@pytest.mark.parametrize("delta", [0.1, 0.5, float("inf")])
def test_twin_matches_loops(zero_rows, delta):
    import scipy.sparse as sp
    rng = np.random.default_rng(7)
    n, K = 60, 9
    rp, col = random_graph(n, 5, seed=7)
    col = col.copy()
    col[::7] = rng.integers(0, n, len(col[::7]))                                        # repeats, self loops, asymmetry
    F = rng.random((n, K)) * (rng.random((n, K)) < 0.3)
    F[::5] = 0.0
    F[3, :3] = 0.25                                                                    # a tie below delta
    m = sp.csr_matrix(F)
    got = community_stats(m.indptr, m.indices, m.data, K, delta, rp, col, zero_rows=zero_rows)
    size, volume, internal = _by_loops(F, delta, rp, col, zero_rows)
    assert got["size"].tolist() == size.tolist()
    assert got["volume"].tolist() == volume.tolist() and got["internal"].tolist() == internal.tolist()
    assert np.array_equal(got["conductance"], conductance(volume, internal, len(col)))


def _ego_F(rp, col, centres):
    """F_uc = 1 for u in {x_c} + N(x_c)."""
    n = len(rp) - 1
    rows = [dict() for _ in range(n)]
    for c, x in enumerate(centres):
        for u in [x, *col[rp[x]:rp[x + 1]].tolist()]:
            rows[u][c] = 1.0
    return _csr(rows, len(centres))


def clean_centres(rp, col, count, seed):
    """Up to count centres whose own list has no repeated entry and no self loop."""
    n = len(rp) - 1
    ok = [x for x in range(n) if len(set(col[rp[x]:rp[x + 1]].tolist()) - {x}) == rp[x + 1] - rp[x]]
    rng = np.random.default_rng(seed)
    return np.sort(rng.choice(ok, size=min(count, len(ok)), replace=False)).astype(np.int64)


def keep_graph(tmp_path, seed=5, n=400):
    """A GraphX `keep` graph: repeated edge lines, reciprocal lines and self loops give repeated list entries."""
    from bigclam_apachespark_b200 import read_edge_list
    rng = np.random.default_rng(seed)
    u, v = rng.integers(0, n, 3 * n), rng.integers(0, n, 3 * n)
    lines = [f"{a} {b}" for a, b in zip(u, v)]
    lines += lines[:n // 8] + [f"{b} {a}" for a, b in zip(u[n // 8:n // 4], v[n // 8:n // 4])] + [f"{a} {a}" for a in range(0, n, 37)]
    path = tmp_path / "keep.txt"
    path.write_text("\n".join(lines) + "\n")
    rp, col, _ = read_edge_list(str(path), "keep")
    return rp, col


def _host_conductance(rp, col):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam()
    b.set_graph(rp, col)
    b.conductanceLocalMin(on_gpu=False)
    return b.conductance


def _ego_graphs(tmp_path):
    from bigclam_apachespark_b200 import graphs as G
    rp, col, _ = G.load_npz_graph("facebook_combined")
    yield "facebook", rp, col
    yield "keep", *keep_graph(tmp_path)


def test_ego_nets_equal_conductance_local_min(tmp_path):
    for name, rp, col in _ego_graphs(tmp_path):
        centres = clean_centres(rp, col, 300, seed=1)
        assert len(centres) >= 100, name
        host = _host_conductance(rp, col)
        got = community_stats(*_ego_F(rp, col, centres), len(centres), 0.5, rp, col, zero_rows=False)
        assert got["size"].tolist() == (np.diff(rp)[centres] + 1).tolist(), name
        assert np.array_equal(got["conductance"].view(np.int64), host[centres].view(np.int64)), name


def test_repeated_neighbour_differs(tmp_path):
    """A centre with a repeated neighbour y: conductanceLocalMin walks y's list once per repetition, the community once."""
    rp, col = keep_graph(tmp_path)
    n = len(rp) - 1
    x = next(x for x in range(n) if len(set(col[rp[x]:rp[x + 1]].tolist())) < rp[x + 1] - rp[x] and x not in col[rp[x]:rp[x + 1]])
    nb = col[rp[x]:rp[x + 1]]
    host = _host_conductance(rp, col)[x]
    got = community_stats(*_ego_F(rp, col, [x]), 1, 0.5, rp, col, zero_rows=False)
    ego = set(nb.tolist()) | {x}
    extra_entries = extra_inside = 0                                                  # the lists walked again by :63
    for y, times in zip(*np.unique(nb, return_counts=True)):
        ly = col[rp[y]:rp[y + 1]]
        extra_entries += (times - 1) * len(ly)
        extra_inside += (times - 1) * int(np.isin(ly, list(ego)).sum())
    vol, inside = int(got["volume"][0]) + extra_entries, int(got["internal"][0]) + extra_inside
    assert host == conductance([vol], [inside], len(col))[0]
    assert extra_entries > 0 and host != got["conductance"][0]
