"""NumPy restatement of the edge probabilities and link recommendations (bigclam_pair_affinity / bigclam_recommend,
csrc/bigclam_sparse.cuh pair_x): x_uv = sum of F_uc F_vc over the components non-zero in both rows, folded left in
ascending c with every product and every sum rounded on its own, so it gives the device's bits.  F comes as CSR rows
(BigClam.F_csr(): ascending indices, no stored zeros)."""
import numpy as np
import scipy.sparse as sp


class Twin:
    def __init__(self, indptr, indices, values, K, min_p=0.0001, max_p=0.9999):
        self.indptr = np.asarray(indptr, dtype=np.int64)
        self.indices = np.asarray(indices, dtype=np.int64)
        self.values = np.asarray(values, dtype=np.float64)
        self.K, self.min_p, self.max_p = int(K), min_p, max_p
        n = len(self.indptr) - 1
        self.keys = np.repeat(np.arange(n, dtype=np.int64), np.diff(self.indptr)) * self.K + self.indices   # ascending

    def x(self, u, v):
        u = np.asarray(u, dtype=np.int64).ravel()
        v = np.asarray(v, dtype=np.int64).ravel()
        lens = self.indptr[u + 1] - self.indptr[u]
        tot = int(lens.sum())
        pair = np.repeat(np.arange(len(u)), lens)
        first = np.repeat(np.cumsum(lens) - lens, lens)
        pos = np.repeat(self.indptr[u], lens) + (np.arange(tot) - first)
        c, a = self.indices[pos], self.values[pos]
        q = v[pair] * self.K + c
        j = np.minimum(np.searchsorted(self.keys, q), max(len(self.keys) - 1, 0))
        hit = (self.keys[j] == q) if len(self.keys) else np.zeros(tot, dtype=bool)
        pair = pair[hit]
        prod = a[hit] * self.values[j[hit]]
        # rank of each common component inside its pair (entries are in pair order, ascending c inside a pair)
        start = np.searchsorted(pair, pair, side="left")
        rank = np.arange(len(pair)) - start
        x = np.zeros(len(u))
        order = np.argsort(rank, kind="stable")
        bounds = np.searchsorted(rank[order], np.arange(rank.max() + 2 if len(rank) else 1))
        for r in range(len(bounds) - 1):
            sel = order[bounds[r]:bounds[r + 1]]
            x[pair[sel]] = x[pair[sel]] + prod[sel]                # one entry per pair and rank: a left fold in c
        return x

    def p(self, x):
        return 1.0 - np.clip(np.exp(-np.asarray(x)), self.min_p, self.max_p)

    def recommend(self, rowptr, col, nodes, m):
        """Brute force: every v with a path u - w - v, v != u, v not in N(u), x_uv > 0; the m best by (x desc, v asc).
        Returns (v, x, found) like bigclam_recommend."""
        n = len(rowptr) - 1
        nodes = np.arange(n) if nodes is None else np.asarray(nodes, dtype=np.int64)
        A = sp.csr_matrix((np.ones(len(col)), np.array(col, dtype=np.int64), np.array(rowptr, dtype=np.int64)), shape=(n, n))
        A.sum_duplicates()                                            # (in place: hence the copies above)
        uq = np.unique(nodes)
        two = (A[uq] @ A).tocoo()                                     # two-hop paths of the query nodes only
        r, c = uq[two.row].astype(np.int64), two.col.astype(np.int64)
        a = A.tocoo()
        ok = (r != c) & ~np.isin(r * n + c, a.row.astype(np.int64) * n + a.col)
        r, c = r[ok], c[ok]
        x = self.x(r, c)
        pos = x > 0
        r, c, x = r[pos], c[pos], x[pos]
        o = np.lexsort((c, -x, r))
        r, c, x = r[o], c[o], x[o]
        lo = np.searchsorted(r, np.arange(n), side="left")
        hi = np.searchsorted(r, np.arange(n), side="right")
        vo = np.full((len(nodes), m), -1, dtype=np.int32)
        xo = np.zeros((len(nodes), m))
        found = np.zeros(len(nodes), dtype=np.int32)
        for i, u in enumerate(nodes):
            k = min(m, hi[u] - lo[u])
            vo[i, :k] = c[lo[u]:lo[u] + k]
            xo[i, :k] = x[lo[u]:lo[u] + k]
            found[i] = k
        return vo, xo, found
