"""NumPy restatement of the sampled graph (bigclam_sample_graph, csrc/bigclam_sparse.cuh sample_rows_kernel).  For every
unordered pair u < v: p_uv = the p of bigclam_pair_affinity (links_twin.Twin) when rows u and v have a component that is
non-zero in both, else eps; the pair is an edge iff r(seed, u, v) < p_uv with
    key = u << 32 | v,   h = mix(seed ^ mix(key)),   r = (h >> 11) * 2^-53,
mix = the splitmix64 step, all mod 2^64.  F comes as CSR rows (BigClam.F_csr(): ascending indices, no stored zeros)."""
import numpy as np
import scipy.sparse as sp

from links_twin import Twin


def splitmix64(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def sample_r(seed, u, v):
    """r(seed, u, v) for arrays of pairs (either order)."""
    u = np.asarray(u, dtype=np.int64)
    v = np.asarray(v, dtype=np.int64)
    lo, hi = np.minimum(u, v).astype(np.uint64), np.maximum(u, v).astype(np.uint64)
    h = splitmix64(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF) ^ splitmix64((lo << np.uint64(32)) | hi))
    return (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


class SampleTwin:
    def __init__(self, indptr, indices, values, K, min_p=0.0001, max_p=0.9999):
        self.links = Twin(indptr, indices, values, K, min_p, max_p)
        self.n = len(indptr) - 1
        ind = np.asarray(indices, dtype=np.int64)
        self.B = sp.csr_matrix((np.ones(len(ind)), ind, np.asarray(indptr, dtype=np.int64)), shape=(self.n, int(K)))

    def pair_p(self, u, v, eps):
        """p_uv of the pairs (u[i], v[i]) and whether they share a component."""
        u = np.asarray(u, dtype=np.int64)
        v = np.asarray(v, dtype=np.int64)
        shared = np.asarray(self.B[u].multiply(self.B[v]).sum(axis=1)).ravel() > 0
        p = np.full(len(u), float(eps))
        if shared.any():
            p[shared] = self.links.p(self.links.x(u[shared], v[shared]))
        return p, shared

    def sample(self, seed, eps, chunk=1 << 20):
        """The whole graph as a symmetric CSR (rowptr int64, col int32), rows ascending."""
        n = self.n
        iu, iv = np.triu_indices(n, 1)
        keep_u, keep_v = [], []
        for a in range(0, len(iu), chunk):
            u, v = iu[a:a + chunk], iv[a:a + chunk]
            p, _ = self.pair_p(u, v, eps)
            take = sample_r(seed, u, v) < p
            keep_u.append(u[take])
            keep_v.append(v[take])
        u = np.concatenate(keep_u + [np.zeros(0, np.int64)])
        v = np.concatenate(keep_v + [np.zeros(0, np.int64)])
        r = np.concatenate([u, v])
        c = np.concatenate([v, u])
        o = np.lexsort((c, r))
        rowptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(r, minlength=n), out=rowptr[1:])
        return rowptr, c[o].astype(np.int32)

    def row(self, u, seed, eps):
        """Row u of the sampled graph, ascending (one row at a time: for graphs too large for sample())."""
        v = np.arange(self.n, dtype=np.int64)
        v = v[v != u]
        p, _ = self.pair_p(np.full(len(v), u), v, eps)
        return v[sample_r(seed, np.full(len(v), u), v) < p].astype(np.int32)
