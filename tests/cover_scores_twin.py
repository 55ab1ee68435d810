"""NumPy/SciPy restatement of the cover scores (bigclam_cover_scores, csrc/bigclam_sparse.cuh cover_scores_kernel) from F
as CSR rows (BigClam.F_csr()), delta, the zero-row mode and a truth cover (a list of id arrays).  M is the n x K
membership matrix of the extraction rule (tests/community_stats_twin.py), T the n x q incidence of the truth sets
(repeats collapsed); the contingency a = M^T T is one sparse product, and every pair (c, t) of non-empty communities is
then evaluated densely, q in chunks, with the formulas of include/bigclam_b200.h."""
import numpy as np
import scipy.sparse as sp

from community_stats_twin import membership

KEYS = ("f1_detected", "match_detected", "f1_truth", "match_truth", "hcond_detected", "hcond_truth")


def truth_incidence(truth, n):
    """The n x q incidence (CSR, int64 ones) of the truth sets: member order and repeats do not matter."""
    q = len(truth)
    rows = np.concatenate([np.asarray(t, dtype=np.int64) for t in truth]) if q else np.zeros(0, dtype=np.int64)
    cols = np.repeat(np.arange(q, dtype=np.int64), [len(t) for t in truth])
    T = sp.csr_matrix((np.ones(len(rows), dtype=np.int64), (rows, cols)), shape=(n, q))
    T.data[:] = 1                                                   # (duplicates were summed)
    return T


def h_table(n):
    """h[m] = -(p log p), p = m / n, h[0] = 0."""
    h = np.zeros(n + 1)
    p = np.arange(1, n + 1, dtype=np.float64) / float(n)
    h[1:] = -(p * np.log(p))
    return h


def _fold(v):
    """A left fold in ascending index (np.cumsum adds one term at a time)."""
    v = np.asarray(v, dtype=np.float64)
    return float(np.cumsum(v)[-1]) if len(v) else 0.0


def cover_scores(indptr, indices, values, K, delta, truth, zero_rows=True, chunk_pairs=1 << 22):
    """dict(avg_f1, nmi_lfk, nmi_max, f1_detected, match_detected, f1_truth, match_truth, hcond_detected, hcond_truth,
    margin): margin is the smallest non-zero |h(a) + h(n - x - y + a) - h(x - a) - h(y - a)| over the evaluated pairs
    (exact ties, equal sums of the same h values, decide alike anywhere)."""
    n = len(indptr) - 1
    M = membership(indptr, indices, values, K, delta, zero_rows).tocsc()
    T = truth_incidence(truth, n).tocsc()
    q = T.shape[1]
    x = np.asarray(M.sum(axis=0)).ravel().astype(np.int64)
    y = np.asarray(T.sum(axis=0)).ravel().astype(np.int64)
    A = (M.T @ T).tocsc()                                            # K x q, |X_c ∩ Y_t|
    h = h_table(n)
    Hx, Hy = h[x] + h[n - x], h[y] + h[n - y]
    live_c = x > 0
    f1_det, match_det = np.zeros(K), np.full(K, -1, dtype=np.int32)
    hc_det = np.full(K, np.inf)
    f1_t, match_t = np.zeros(q), np.full(q, -1, dtype=np.int32)
    hc_t = np.full(q, np.inf)
    margin = np.inf
    step = max(1, chunk_pairs // max(K, 1))
    for t0 in range(0, q, step):
        t1 = min(q, t0 + step)
        yc = y[t0:t1]
        a = A[:, t0:t1].toarray().astype(np.int64)
        valid = live_c[:, None] & (yc > 0)[None, :]
        X, Y = x[:, None], yc[None, :]
        with np.errstate(invalid="ignore"):                          # 0 / 0 where both are empty
            f1 = np.where(valid, (2.0 * a) / (X + Y).astype(np.float64), 0.0)
        # detected side: a later chunk takes over only where it is strictly better (smallest t on ties)
        jb = np.argmax(f1, axis=1)
        fb = f1[np.arange(K), jb]
        better = fb > f1_det
        f1_det[better] = fb[better]
        match_det[better] = (t0 + jb[better]).astype(np.int32)
        # truth side: argmax gives the smallest c on ties
        cb = np.argmax(f1, axis=0)
        f1_t[t0:t1] = f1[cb, np.arange(t1 - t0)]
        match_t[t0:t1] = np.where(f1_t[t0:t1] > 0, cb, -1)
        ha, hxa, hya, hd = h[a], h[np.where(valid, X - a, 0)], h[np.where(valid, Y - a, 0)], h[np.where(valid, n - X - Y + a, 0)]
        lhs, rhs = ha + hd, hxa + hya
        adm = valid & (lhs > rhs)
        gap = np.abs(lhs - rhs)[valid]
        gap = gap[gap > 0]
        if len(gap):
            margin = min(margin, float(gap.min()))
        hcx = np.where(adm, np.maximum(0.0, ((ha + hxa) + hya) + hd - (h[Y] + h[n - Y])), np.inf)
        hcy = np.where(adm, np.maximum(0.0, ((ha + hya) + hxa) + hd - (h[X] + h[n - X])), np.inf)
        hc_det = np.minimum(hc_det, hcx.min(axis=1))
        hc_t[t0:t1] = hcy.min(axis=0)
    in_x = (x > 0) & (x < n)
    in_y = (y > 0) & (y < n)
    hc_det = np.where(in_x, np.where(np.isinf(hc_det), Hx, hc_det), np.nan)
    hc_t = np.where(in_y, np.where(np.isinf(hc_t), Hy, hc_t), np.nan)
    nx = int(live_c.sum())
    avg = 0.0 if nx == 0 or q == 0 else 0.5 * (_fold(f1_det[live_c]) / nx + _fold(f1_t) / q)
    if in_x.any() and in_y.any():
        lfk = 1.0 - 0.5 * (_fold(hc_det[in_x] / Hx[in_x]) / int(in_x.sum()) + _fold(hc_t[in_y] / Hy[in_y]) / int(in_y.sum()))
        sx, sy = _fold(Hx[in_x]), _fold(Hy[in_y])
        mx = 0.5 * ((sx - _fold(hc_det[in_x])) + (sy - _fold(hc_t[in_y]))) / max(sx, sy)
    else:
        lfk = mx = float("nan")
    return dict(avg_f1=avg, nmi_lfk=lfk, nmi_max=mx, f1_detected=f1_det, match_detected=match_det, f1_truth=f1_t,
                match_truth=match_t, hcond_detected=hc_det, hcond_truth=hc_t, margin=margin)


def nmi_by_sets(X, Y, n):
    """(nmi_lfk, nmi_max) written out over Python sets and math.log, for small covers (lists of node collections)."""
    import math

    def h(m):
        if m == 0:
            return 0.0
        p = m / n
        return -(p * math.log(p))

    X = [set(map(int, c)) for c in X if len(set(c))]
    Y = [set(map(int, c)) for c in Y if len(set(c))]

    def hstar(A, B):
        out = []
        for S in A:
            x = len(S)
            if not 0 < x < n:
                continue
            best = None
            for R in B:
                y, a = len(R), len(S & R)
                if h(a) + h(n - x - y + a) > h(x - a) + h(y - a):
                    v = max(0.0, ((h(a) + h(x - a)) + h(y - a)) + h(n - x - y + a) - (h(y) + h(n - y)))
                    best = v if best is None else min(best, v)
            H = h(x) + h(n - x)
            out.append((H if best is None else best, H))
        return out

    hx, hy = hstar(X, Y), hstar(Y, X)
    if not hx or not hy:
        return float("nan"), float("nan")
    lfk = 1.0 - 0.5 * (sum(c / H for c, H in hx) / len(hx) + sum(c / H for c, H in hy) / len(hy))
    sx, sy = sum(H for _, H in hx), sum(H for _, H in hy)
    mx = 0.5 * ((sx - sum(c for c, _ in hx)) + (sy - sum(c for c, _ in hy))) / max(sx, sy)
    return lfk, mx
