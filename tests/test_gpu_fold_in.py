"""Fold-in on the GPU (bigclam_fold_in / bigclam_fold_in_nnz and their multi-GPU twins, BigClam.fold_in, the C++ mirror):
rows for new nodes with the fitted F and sumF held fixed, against a loop of oracle steps on the graph with the node
appended, against one bigclam_step over the extended graph, independence of the batch, untouched state and the argument
checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import REPO, random_graph

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"
TIE_TOL = 1e-9          # a differing Armijo decision must be a tie: |margin| <= TIE_TOL * max(|llh_u|, 1)


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _fitted(rp, col, K, seed, sparse=True, steps=3, per_row=6.0):
    """A context after a few steps from a random F0 with about per_row non-zeros per row."""
    from bigclam_apachespark_b200 import BigClam
    n = len(rp) - 1
    rng = np.random.default_rng(seed)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < min(1.0, per_row / K))
    b = BigClam(sparse_rows=sparse, record_accepted=True)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    for _ in range(steps):
        b.backtrackingLineSearchs()
    return b


def _queries(n, F, seed, count):
    """count random lists plus the special ones: empty, repeated neighbours, a neighbour with a zero row, a neighbour
    at MAX_F_ (the caller plants it in row 1), a single neighbour."""
    rng = np.random.default_rng(seed)
    lists = [rng.choice(n, size=int(rng.integers(1, 12)), replace=False) for _ in range(count)]
    zero = np.nonzero(F.max(axis=1) == 0)[0]
    lists += [np.array([], dtype=np.int64), np.array([2, 2, 5, 2, 7]), np.array([1, 3, 4]), np.array([9])]
    if len(zero):
        lists.append(np.array([zero[0], 6, 8]))
    rp = np.zeros(len(lists) + 1, dtype=np.int64)
    rp[1:] = np.cumsum([len(x) for x in lists])
    return rp, np.concatenate(lists).astype(np.int32)


def _oracle_fold(O, rp, col, F, sumF, params, lst, max_iter, rel_tol):
    """The definition as a loop of oracle steps on G + u (u = node n with list lst, sumF' = sumF + f, mask {u}).
    Returns (f, llh, iters, tie): tie = some decision was within rounding of its threshold."""
    n, K = F.shape
    f = np.zeros(K)
    if len(lst) == 0:
        return f, 0.0, 0, False
    rp2 = np.concatenate([rp, [rp[-1] + len(lst)]]).astype(np.int64)
    col2 = np.concatenate([col, lst]).astype(np.int32)
    mask = np.zeros(n + 1, dtype=np.uint8)
    mask[n] = 1
    Fx = np.vstack([F, f[None, :]])
    it, lprev, tie = 0, None, False
    while True:
        Fx[n] = f
        sF = sumF + f
        r = O.step(rp2, col2, Fx, sF, params, node_mask=mask, want_pre=True)
        l = float(r.llh_u[n])
        if it > 0:
            gain = abs(1.0 - l / lprev)
            tie |= abs(gain - rel_tol) <= 1e-9 * max(rel_tol, 1e-300) + 1e-12
            if gain < rel_tol:
                break
        if it == max_iter:
            break
        m, lu = O.armijo_margins(rp2, col2, Fx, sF, params, [n])
        near = np.abs(m[0]) <= TIE_TOL * max(abs(lu[0]), 1.0)
        a = int(r.accepted[n])                                       # the decision: a passes, a - 1 fails
        tie |= bool(near.any() if a < 0 else (near[a] or (a > 0 and near[a - 1])))
        if r.accepted[n] < 0:
            break
        f = r.F[n].copy()
        lprev = l
        it += 1
    return f, l, it, tie


def _check_against_oracle(b, rp, col, qrp, qcol, max_iter, rel_tol, params=None):
    """Every node agrees with the oracle loop (iters equal, same support, rows to 1e-12, llh to 1e-10) or its run went
    through a rounding-level Armijo tie; a node that has converged meets one at every further line search, so ties are
    bounded only loosely.  params: the oracle's parameters, those of the context (default: the script's)."""
    from oracle import oracle as O
    F, sumF = b.F, b.sumF
    if params is None:
        params = O.make_params(b.K)
    ip, ix, vl, llh, iters = b.fold_in(qrp, qcol, max_iter=max_iter, rel_tol=rel_tol)
    q = len(qrp) - 1
    assert ip.shape == (q + 1,) and ip[0] == 0 and (np.diff(ip) >= 0).all()
    ties = 0
    for i in range(q):
        lst = qcol[qrp[i]:qrp[i + 1]]
        f, l, it, tie = _oracle_fold(O, rp, col, F, sumF, params, lst, max_iter, rel_tol)
        gi, gv = ix[ip[i]:ip[i + 1]], vl[ip[i]:ip[i + 1]]
        assert (np.diff(gi) > 0).all() and (gv != 0).all(), i
        row = np.zeros(b.K)
        row[gi] = gv
        same = (it == iters[i] and np.array_equal(np.nonzero(f)[0], gi)
                and np.abs(row - f).max() <= 1e-12 * max(np.abs(f).max(), 1e-300)
                and abs(llh[i] - l) <= 1e-10 * max(abs(l), 1e-300))
        if not same:
            assert tie, f"node {i}: iters {iters[i]} vs {it}, llh {llh[i]!r} vs {l!r}, max row err {np.abs(row - f).max():.3e}"
            ties += 1
        if len(lst) == 0:
            assert len(gi) == 0 and llh[i] == 0.0 and iters[i] == 0
    assert ties <= max(2, q // 3), ties
    return ip, ix, vl, llh, iters


KS = [1, 37, 200, 1024, 1025, 9000]


@pytest.mark.parametrize("K", KS)
def test_oracle_parity_random_graph(K):
    n = 120 if (EMU or K > 1024) else 300
    rp, col = random_graph(n, 6, seed=K)
    layouts = [True, False] if K <= 1024 else [True]
    from bigclam_apachespark_b200 import BigClam
    got = {}
    fit = _fitted(rp, col, K, seed=K)
    ip, ix, vl = fit.F_csr()
    vl = vl.copy()
    vl[ip[1]:ip[2]] = 1000.0                                         # row 1 at MAX_F_ on its components
    sumF = fit.sumF
    fit.close()
    for sparse in layouts:                                           # the same F and sumF in both layouts
        b = BigClam(sparse_rows=sparse)
        b.set_graph(rp, col).set_K(K).set_F_csr(ip, ix, vl, K=K, sumF=sumF)
        qrp, qcol = _queries(n, b.F, seed=K, count=8 if (EMU or K > 1024) else 30)
        got[sparse] = _check_against_oracle(b, rp, col, qrp, qcol, max_iter=12 if K > 1024 else 40, rel_tol=1e-4)
        b.close()
    if len(layouts) == 2:                                           # the same F in both layouts: within rounding
        a, d = got[True], got[False]
        assert np.array_equal(a[0], d[0]) and np.array_equal(a[1], d[1]) and np.array_equal(a[4], d[4])
        assert np.allclose(a[2], d[2], rtol=1e-13, atol=0) and np.allclose(a[3], d[3], rtol=1e-13, atol=0)


def test_oracle_parity_facebook_held_out():
    from bigclam_apachespark_b200 import BigClam, graphs as G
    if EMU:
        pytest.skip("facebook is too large for the host emulation")
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n = len(rp) - 1
    rng = np.random.default_rng(7)
    held = np.sort(rng.choice(n, 40, replace=False))
    keep = np.ones(n, dtype=bool)
    keep[held] = False
    new_id = np.cumsum(keep) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    e = keep[u] & keep[col]
    rpk = np.zeros(keep.sum() + 1, dtype=np.int64)
    rpk[1:] = np.cumsum(np.bincount(new_id[u[e]], minlength=keep.sum()))
    colk = new_id[col[e]].astype(np.int32)
    qlists = [new_id[col[rp[h]:rp[h + 1]][keep[col[rp[h]:rp[h + 1]]]]] for h in held]
    qrp = np.zeros(len(held) + 1, dtype=np.int64)
    qrp[1:] = np.cumsum([len(x) for x in qlists])
    qcol = np.concatenate(qlists).astype(np.int32)
    K = 10
    b = BigClam(sparse_rows=True)
    b.set_graph(rpk, colk).set_K(K).set_F(G.synthetic_F0(len(rpk) - 1, K, seed=1234, density=0.3))
    for _ in range(3):
        b.backtrackingLineSearchs()
    _check_against_oracle(b, rpk, colk, qrp, qcol, max_iter=100, rel_tol=1e-4)
    b.close()


def _extended(rp, col, qrp, qcol):
    """G plus the q query nodes as nodes n .. n+q-1, linked to their lists (both ways), not to each other."""
    from bigclam_apachespark_b200 import graphs as G
    n, q = len(rp) - 1, len(qrp) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    keep = u < col
    qu = n + np.repeat(np.arange(q), np.diff(qrp))
    su = np.concatenate([u[keep], qu])
    sv = np.concatenate([col[keep], qcol])
    key = np.unique(np.minimum(su, sv) * (n + q) + np.maximum(su, sv))
    return G.csr_from_undirected(n + q, key // (n + q), key % (n + q))


@pytest.mark.parametrize("K", [37, 1025])
def test_first_iteration_equals_step(K):
    from bigclam_apachespark_b200 import BigClam
    n = 120 if (EMU or K > 1024) else 300
    rp, col = random_graph(n, 6, seed=11 + K)
    b = _fitted(rp, col, K, seed=11)
    rng = np.random.default_rng(5)
    lists = [np.unique(rng.choice(n, size=int(rng.integers(1, 10)))) for _ in range(12)]
    qrp = np.zeros(len(lists) + 1, dtype=np.int64)
    qrp[1:] = np.cumsum([len(x) for x in lists])
    qcol = np.concatenate(lists).astype(np.int32)
    q = len(lists)
    ip, ix, vl, llh, iters = b.fold_in(qrp, qcol, max_iter=1, rel_tol=1e-4)
    erp, ecol = _extended(rp, col, qrp, qcol)
    Fi, Fx, Fv = b.F_csr()
    Fi2 = np.concatenate([Fi, np.full(q, Fi[-1])])
    e = BigClam(sparse_rows=True, record_accepted=True)
    e.set_graph(erp, ecol).set_K(K).set_F_csr(Fi2, Fx, Fv, K=K, sumF=b.sumF)
    e.backtrackingLineSearchs(uset=range(n, n + q))
    acc = e.accepted()[n:]
    assert np.array_equal(acc >= 0, iters == 1)
    Fe = e.F[n:]
    for i in range(q):
        row = np.zeros(K)
        row[ix[ip[i]:ip[i + 1]]] = vl[ip[i]:ip[i + 1]]
        assert np.abs(row - Fe[i]).max() <= 1e-13 * max(np.abs(Fe[i]).max(), 1e-300), i
    e.close()
    # q = 1: T masked steps against max_iter = T, rel_tol = 0
    T = 5
    one_rp, one_col = qrp[:2], qcol[:qrp[1]]
    ip, ix, vl, llh, iters = b.fold_in(one_rp, one_col, max_iter=T, rel_tol=0.0)
    erp, ecol = _extended(rp, col, one_rp, one_col)
    e = BigClam(sparse_rows=True, record_accepted=True)
    e.set_graph(erp, ecol).set_K(K).set_F_csr(np.concatenate([Fi, [Fi[-1]]]), Fx, Fv, K=K, sumF=b.sumF)
    steps = 0
    for _ in range(T):
        e.backtrackingLineSearchs(uset=[n])
        if e.accepted()[n] < 0:
            break
        steps += 1
    assert steps == iters[0]
    row = np.zeros(K)
    row[ix] = vl
    assert np.abs(row - e.F[n]).max() <= 1e-12 * max(np.abs(row).max(), 1e-300)
    e.close()
    b.close()


@pytest.mark.parametrize("K", [37, 200, 1025])
def test_independent_of_the_batch(K):
    n = 120 if (EMU or K > 1024) else 400
    rp, col = random_graph(n, 6, seed=21 + K)
    b = _fitted(rp, col, K, seed=21)
    qrp, qcol = _queries(n, b.F, seed=21, count=10 if EMU else 40)
    q = len(qrp) - 1
    lists = [qcol[qrp[i]:qrp[i + 1]] for i in range(q)]
    ref = b.fold_in(qrp, qcol)

    def rows(res):
        ip, ix, vl, llh, it = res
        return [(ix[ip[i]:ip[i + 1]].tobytes(), _bits(vl[ip[i]:ip[i + 1]]).tobytes(), _bits([llh[i]]).tobytes(), int(it[i]))
                for i in range(len(ip) - 1)]

    r0 = rows(ref)
    assert rows(b.fold_in(qrp, qcol)) == r0                          # rerun
    for i in range(q):                                               # every node alone
        assert rows(b.fold_in(np.array([0, len(lists[i])]), lists[i])) == [r0[i]], i
    rev = lists[::-1]
    rrp = np.zeros(q + 1, dtype=np.int64)
    rrp[1:] = np.cumsum([len(x) for x in rev])
    assert rows(b.fold_in(rrp, np.concatenate(rev).astype(np.int32))) == r0[::-1]
    os.environ["BIGCLAM_FOLD_IN_BUDGET"] = str(40 * 12 * min(K, 60))   # a few nodes per batch
    try:
        assert rows(b.fold_in(qrp, qcol)) == r0
    finally:
        del os.environ["BIGCLAM_FOLD_IN_BUDGET"]
    nnz = C.c_int64()
    assert _lib().bigclam_fold_in_nnz(b._ctx, q, qrp.ctypes.data, qcol.ctypes.data, 100, 1e-4, C.byref(nnz)) == 0
    assert nnz.value == ref[0][-1]
    b.close()


def test_state_untouched():
    from bigclam_apachespark_b200 import BigClam
    rp, col = random_graph(150 if EMU else 600, 6, seed=31)
    n, K = len(rp) - 1, 24
    rng = np.random.default_rng(31)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < 0.3)
    a = BigClam(sparse_rows=True, record_accepted=True, time_kernels=True)
    c = BigClam(sparse_rows=True, record_accepted=True, time_kernels=True)
    for x in (a, c):
        x.set_graph(rp, col).set_K(K).set_F(F0)
    qrp, qcol = _queries(n, F0, seed=31, count=20)
    for it in range(4):
        la, lc = a.backtrackingLineSearchs(), c.backtrackingLineSearchs()
        assert _bits([la]) == _bits([lc]), it
        assert a.kernel_time()[1:] == c.kernel_time()[1:], it       # from the 2nd step on, both commit the speculation
        if it > 0:
            assert a.kernel_time()[1] == 1
        a.fold_in(qrp, qcol)
    for x, y in zip(a.F_csr(), c.F_csr()):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert np.array_equal(_bits(a.sumF), _bits(c.sumF))
    assert np.array_equal(a.accepted(), c.accepted())
    assert _bits([a.loglikelihood()]) == _bits([c.loglikelihood()])
    a.close()
    c.close()


def test_argument_checks():
    from bigclam_apachespark_b200 import BigClam, _lib as L
    rp, col = random_graph(100, 4, seed=3)
    n, K = len(rp) - 1, 8
    b = _fitted(rp, col, K, seed=3, steps=1)
    lib = L.load()
    ctx = b._ctx
    qrp = np.array([0, 2, 3], dtype=np.int64)
    good = np.array([0, 1, 5], dtype=np.int32)
    nnz = C.c_int64()
    ip = np.zeros(3, dtype=np.int64)
    ix = np.zeros(3 * K, dtype=np.int32)
    vl = np.zeros(3 * K)

    def call(q=2, rp_=qrp, c=good, mi=10, rt=1e-4, out=True):
        a = lib.bigclam_fold_in_nnz(ctx, q, None if rp_ is None else rp_.ctypes.data, None if c is None else c.ctypes.data, mi, rt,
                                    C.byref(nnz) if out else None)
        f = lib.bigclam_fold_in(ctx, q, None if rp_ is None else rp_.ctypes.data, None if c is None else c.ctypes.data, mi, rt,
                                ip.ctypes.data, ix.ctypes.data if out else None, vl.ctypes.data, None, None)
        return a, f

    assert call() == (L.OK, L.OK)
    assert call(c=np.array([0, n, 1], dtype=np.int32)) == (L.EINVAL, L.EINVAL)
    assert b"outside" in lib.bigclam_last_error(ctx)
    assert call(c=np.array([0, -1, 1], dtype=np.int32)) == (L.EINVAL, L.EINVAL)
    assert call(rp_=np.array([1, 2, 3], dtype=np.int64)) == (L.EINVAL, L.EINVAL)
    assert call(rp_=np.array([0, 2, 1], dtype=np.int64)) == (L.EINVAL, L.EINVAL)
    assert call(q=-1) == (L.EINVAL, L.EINVAL)
    assert call(mi=0) == (L.EINVAL, L.EINVAL)
    assert call(rt=-1e-3) == (L.EINVAL, L.EINVAL)
    assert call(rt=float("nan")) == (L.EINVAL, L.EINVAL)
    assert call(rp_=None) == (L.EINVAL, L.EINVAL)
    assert call(c=None) == (L.EINVAL, L.EINVAL)
    assert call(out=False) == (L.EINVAL, L.EINVAL)
    nnz.value = 7
    assert call(q=0, rp_=None, c=None) == (L.OK, L.OK) and nnz.value == 0
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    b.close()
    # min_f != 0 (dense rows only): unsupported
    p = L.Params()
    lib.bigclam_default_params(C.byref(p), K)
    p.min_f = 0.001
    ctx2 = C.c_void_p()
    rc = lib.bigclam_create(C.byref(ctx2), n, rp.ctypes.data, col.ctypes.data, C.byref(p))
    assert rc == L.OK, lib.bigclam_last_error(None)
    try:
        assert lib.bigclam_fold_in_nnz(ctx2, 2, qrp.ctypes.data, good.ctypes.data, 10, 1e-4, C.byref(nnz)) == L.EUNSUPPORTED
    finally:
        lib.bigclam_destroy(ctx2)


def test_multi_gpu_handle_matches_one_context():
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    rp, col = random_graph(150 if EMU else 500, 6, seed=41)
    n, K = len(rp) - 1, 37
    rng = np.random.default_rng(41)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < 0.2)
    one = BigClam(sparse_rows=True)
    one.set_graph(rp, col).set_K(K).set_F(F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    qrp, qcol = _queries(n, F0, seed=41, count=20)
    r1, r2 = one.fold_in(qrp, qcol), two.fold_in(qrp, qcol)
    for x, y in zip(r1, r2):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    lib = _lib()
    bad = np.array([0, n], dtype=np.int32)
    brp = np.array([0, 2], dtype=np.int64)
    nnz = C.c_int64()
    assert lib.bigclam_multi_fold_in_nnz(two._multi, 1, brp.ctypes.data, bad.ctypes.data, 10, 1e-4, C.byref(nnz)) == -1
    assert b"outside" in lib.bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


CPP = os.path.join(REPO, "tests", "cpp_host", "fold_in.cpp")


def test_cpp_mirror_agrees_with_python(tmp_path):
    from test_c_host import product_lib
    from bigclam_apachespark_b200 import BigClam
    libdir, libname = product_lib()
    src = CPP
    exe = str(tmp_path / "fold_in")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"), str(src),
                        "-o", exe, "-L", libdir, f"-l:{libname}", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rp, col = random_graph(120, 6, seed=5)
    n, K = len(rp) - 1, 37
    rng = np.random.default_rng(5)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < 0.2)
    qrp, qcol = _queries(n, F0, seed=5, count=10)
    q = len(qrp) - 1
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, q, len(qcol)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes())
        f.write(qrp.astype(np.int64).tobytes() + qcol.astype(np.int32).tobytes())
    r = subprocess.run([exe, str(inp), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                 # max_iter = 0: bigclam::Error with BIGCLAM_EINVAL
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    ip, ix, vl, llh, it = b.fold_in(qrp, qcol)
    raw = open(tmp_path / "out.bin", "rb").read()
    nz = int(ip[-1])
    o = 0
    cip = np.frombuffer(raw, np.int64, q + 1, o); o += 8 * (q + 1)
    cix = np.frombuffer(raw, np.int32, nz, o); o += 4 * nz
    cvl = np.frombuffer(raw, np.float64, nz, o); o += 8 * nz
    cllh = np.frombuffer(raw, np.float64, q, o); o += 8 * q
    cit = np.frombuffer(raw, np.int32, q, o)
    assert np.array_equal(cip, ip) and np.array_equal(cix, ix) and np.array_equal(_bits(cvl), _bits(vl))
    assert np.array_equal(_bits(cllh), _bits(llh)) and np.array_equal(cit, it)
    b.close()
