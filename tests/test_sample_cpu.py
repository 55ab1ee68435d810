"""The NumPy twin of the sampled graph (tests/sample_twin.py) against plain Python: the hash against Python integers mod
2^64, the whole graph against a loop over all pairs on small hand-made rows, and edge frequencies over many seeds against
p_uv.  No device needed."""
import math

import numpy as np

from sample_twin import SampleTwin, sample_r, splitmix64

M64 = (1 << 64) - 1


def _mix(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _r(seed, u, v):
    lo, hi = min(u, v), max(u, v)
    return (_mix((seed & M64) ^ _mix((lo << 32) | hi)) >> 11) * 2.0 ** -53


def test_hash_matches_python_integers():
    rng = np.random.default_rng(1)
    z = np.concatenate([np.array([0, 1, M64, 0x9E3779B97F4A7C15, M64 - 0x9E3779B97F4A7C15], dtype=np.uint64),
                        rng.integers(0, M64, 200, dtype=np.uint64, endpoint=True)])
    assert [int(x) for x in splitmix64(z)] == [_mix(int(x)) for x in z]
    assert int(splitmix64(np.uint64(0))) == 0xE220A8397B1DCDAF            # the first output of splitmix64 seeded with 0
    for seed in (0, 7, M64, 0x123456789ABCDEF0):
        u = rng.integers(0, 1 << 31, 100)
        v = rng.integers(0, 1 << 31, 100)
        r = sample_r(seed, u, v)
        assert [float(x) for x in r] == [_r(seed, int(a), int(b)) for a, b in zip(u, v)]
        assert np.array_equal(r, sample_r(seed, v, u))                     # symmetric in (u, v)
        assert (r >= 0).all() and (r < 1).all()


def _csr(rows, K):
    indptr, idx, val = [0], [], []
    for r in rows:
        for c in sorted(r):
            idx.append(c)
            val.append(r[c])
        indptr.append(len(idx))
    return np.array(indptr), np.array(idx, dtype=np.int64), np.array(val), K


def _loop_graph(rows, seed, eps, min_p=0.0001, max_p=0.9999):
    n = len(rows)
    adj = [[] for _ in range(n)]
    for u in range(n):
        for v in range(u + 1, n):
            common = sorted(set(rows[u]) & set(rows[v]))
            if common:
                x = 0.0
                for c in common:
                    x = x + rows[u][c] * rows[v][c]
                p = 1.0 - min(max(math.exp(-x), min_p), max_p)
            else:
                p = eps
            if _r(seed, u, v) < p:
                adj[u].append(v)
                adj[v].append(u)
    rowptr = np.cumsum([0] + [len(a) for a in adj])
    return rowptr, np.array([v for a in adj for v in sorted(a)], dtype=np.int32)


ROWS = [
    {0: 0.9, 3: 0.7},               # 0
    {3: 1.2, 5: 3.0},               # 1
    {1: 0.9},                       # 2: shares nothing with 0, 1, 4
    {},                             # 3: all zero: background only
    {0: 1.0, 5: 0.35},              # 4
    {0: 0.5, 3: 0.7, 5: 1e-3},      # 5
    {1: 1e-200},                    # 6: shares component 1 with 2, x underflows to 0: the floor, not eps
    {5: 2.0},                       # 7
]


def test_twin_matches_the_loop_over_all_pairs():
    tw = SampleTwin(*_csr(ROWS, 8))
    for seed in range(40):
        for eps in (0.0, 1e-3, 0.3, 0.9999):
            rp, col = tw.sample(seed, eps)
            lrp, lcol = _loop_graph(ROWS, seed, eps)
            assert np.array_equal(rp, lrp) and np.array_equal(col, lcol), (seed, eps)


def test_shared_follows_nonzero_components():
    tw = SampleTwin(*_csr(ROWS, 8))
    p, shared = tw.pair_p([0, 0, 2, 3, 2, 1], [1, 2, 6, 5, 0, 7], 0.25)
    assert shared.tolist() == [True, False, True, False, False, True]
    assert p[1] == 0.25 and p[3] == 0.25 and p[4] == 0.25
    assert p[2] == 1.0 - 0.9999                                            # x = 0 but shared: the clamp floor
    assert abs(p[0] - (1.0 - math.exp(-0.7 * 1.2))) <= 1e-16


def test_edge_frequencies_follow_the_model():
    """Over 400 seeds each pair of a 40-node model is an edge with frequency within 6 sigma of p_uv."""
    rng = np.random.default_rng(5)
    n, K = 40, 6
    F = rng.random((n, K)) * (rng.random((n, K)) < 0.3) * 1.5
    F[:4] = 0.0                                                            # background-only rows
    rows = [{c: F[u, c] for c in range(K) if F[u, c] != 0.0} for u in range(n)]
    tw = SampleTwin(*_csr(rows, K))
    eps = 0.05
    iu, iv = np.triu_indices(n, 1)
    p, _ = tw.pair_p(iu, iv, eps)
    seeds = 400
    hits = np.zeros(len(iu))
    for seed in range(seeds):
        rp, col = tw.sample(seed, eps)
        A = np.zeros((n, n), dtype=bool)
        A[np.repeat(np.arange(n), np.diff(rp)), col] = True
        assert (A == A.T).all() and not A.diagonal().any()
        hits += A[iu, iv]
    sigma = np.sqrt(p * (1 - p) / seeds)
    assert (np.abs(hits / seeds - p) <= 6 * sigma + 1e-12).all()
