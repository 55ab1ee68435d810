"""Communities grouped by community on the GPU (bigclam_extract_nnz / bigclam_extract_grouped and their multi-GPU twins,
BigClam.extract_communities, communities.group, the C++ mirror): exact output against the NumPy twin
(tests/extract_twin.py) for sparse and dense rows at every kind of K, against bigclam_extract's member matrix regrouped,
the rows the rule has to get right, fitted models, a planted model, a forced cut into several ranges, the state an
extraction must leave untouched, and the argument checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import REPO, random_graph
from extract_twin import extract_grouped

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def _solver(rp, col, K, F0, sparse=True, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse, record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    return b


def _twin(b, delta):
    return extract_grouped(*b.F_csr(), b.K, delta)


def _same(g, h):
    return all(np.array_equal(x, y) and np.asarray(x).dtype == np.asarray(y).dtype for x, y in zip(g, h))


def _check_shape(g, n, K):
    comptr, members, zero_rows = g
    assert comptr.dtype == np.int64 and members.dtype == np.int32 and zero_rows.dtype == np.int32
    assert len(comptr) == K + 1 and comptr[0] == 0 and comptr[-1] == len(members) and (np.diff(comptr) >= 0).all()
    assert ((members >= 0) & (members < n)).all() and (np.diff(zero_rows) > 0).all()
    assert not np.isin(members, zero_rows).any()
    for c in range(K):
        assert (np.diff(members[comptr[c]:comptr[c + 1]]) > 0).all(), c


def _matches_dense_route(b, delta):
    """communities.group() of the grouped call equals communities.extract()'s lists and ids (bigclam_extract)."""
    from bigclam_apachespark_b200 import communities as Cm
    comms, cids, _ = Cm.extract(b, delta)
    gc, gi = Cm.group(*b.extract_communities(delta))
    return np.array_equal(cids, gi) and all(np.array_equal(x, y) for x, y in zip(comms, gc)) and len(comms) == len(gc)


def _F0(n, K, seed, delta, per_row=6.0):
    """About per_row non-zeros a row, F up to 2 delta, with the rows the rule has to get right: all-zero rows (0 and 5),
    a tie at a maximum below delta (1), a row maximum exactly delta (2), an entry exactly delta (3), 1e-300 entries (4),
    rows at MAX_F_ (6 and 7) and a row whose non-zeros all tie below delta (8)."""
    rng = np.random.default_rng(seed)
    F0 = 2 * delta * rng.random((n, K)) * (rng.random((n, K)) < min(1.0, per_row / K))
    F0[[0, 1, 2, 4, 5, 8]] = 0.0
    F0[1, 0] = F0[1, K - 1] = delta / 2
    F0[2, K // 2] = delta
    F0[3, 0] = delta
    F0[4, 0] = F0[4, K - 1] = 1e-300
    F0[6] = np.where(rng.random(K) < min(1.0, per_row / K), 1000.0, 0.0)
    F0[6, K - 1] = 1000.0
    F0[7] = F0[6]
    F0[8, ::3] = 0.25 * delta
    return F0


KS = [1, 37, 200, 1024, 1025, 9000]
DELTA = 0.5


@pytest.mark.parametrize("K", KS)
def test_extract_matches_twin(K):
    n = 100 if EMU else (600 if K == 9000 else 300)
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K, delta=DELTA)
    layouts = [True, False] if K <= 1024 else [True]
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        for delta in (DELTA, 0.1, float("inf")):
            g = b.extract_communities(delta)
            assert _same(g, _twin(b, delta)), (K, sparse, delta)
            _check_shape(g, n, K)
            assert {0, 5} <= set(g[2].tolist())
            assert _matches_dense_route(b, delta), (K, sparse, delta)
            got[(sparse, delta)] = g
        b.close()
    if len(layouts) == 2:                                                           # the same F in both layouts: the same arrays
        for delta in (DELTA, 0.1, float("inf")):
            assert _same(got[(True, delta)], got[(False, delta)])


@pytest.mark.parametrize("sparse", [True, False])
def test_edge_rows(sparse):
    """Rows the rule has to get right, checked one by one against the rule written out."""
    n, K = 40, 16
    rp, col = random_graph(n, 4, seed=2)
    F0 = _F0(n, K, seed=2, delta=DELTA)
    F0[9] = 0.0
    F0[9, 3] = DELTA
    F0[9, 7] = DELTA * (1 - 2 ** -52)                                               # just below delta: not a member
    b = _solver(rp, col, K, F0, sparse=sparse)
    comptr, members, zero_rows = b.extract_communities(DELTA)

    def comms_of(u):
        return [c for c in range(K) if u in members[comptr[c]:comptr[c + 1]]]

    assert list(zero_rows) == [0, 5]
    assert comms_of(1) == [0, K - 1]                                                # tie below delta: both
    assert comms_of(2) == [K // 2]                                                  # maximum == delta: F >= delta
    assert 0 in comms_of(3)                                                         # entry == delta
    assert comms_of(4) == [0, K - 1]                                                # 1e-300 ties below delta
    assert comms_of(6) == list(np.flatnonzero(F0[6]))                               # MAX_F_
    assert comms_of(8) == list(range(0, K, 3))
    assert comms_of(9) == [3]
    g = b.extract_communities(float("inf"))                                         # every row to its maximum entries
    assert _same(g, _twin(b, float("inf")))
    ip, ix, vl = b.F_csr()
    for u in range(n):
        row = vl[ip[u]:ip[u + 1]]
        want = [] if len(row) == 0 else list(ix[ip[u]:ip[u + 1]][row == row.max()])
        assert [c for c in range(K) if u in g[1][g[0][c]:g[0][c + 1]]] == want, u
    assert list(g[2]) == [0, 5]
    b.close()


def test_facebook_after_steps():
    from bigclam_apachespark_b200 import communities as Cm, graphs as G
    if EMU:
        pytest.skip("facebook is too large for the host emulation")
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(3):
        b.backtrackingLineSearchs()
    for delta in (Cm.delta_threshold(n, int((np.diff(rp) > 0).sum())), Cm.delta_threshold(n, len(col) // 2), 0.5):
        g = b.extract_communities(delta)
        assert _same(g, _twin(b, delta)), delta
        _check_shape(g, n, K)
        assert _matches_dense_route(b, delta), delta
    b.close()


def test_amazon_after_fit():
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G
    if EMU:
        pytest.skip("com-amazon is GPU only")
    rp, col, _ = G.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 200
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    b.initNeighborComF(K)
    for _ in range(3):
        b.backtrackingLineSearchs()
    delta = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))
    g = b.extract_communities(delta)
    assert _same(g, _twin(b, delta))
    _check_shape(g, n, K)
    assert _matches_dense_route(b, delta)
    b.close()


def _planted(n, K, fval, seed):
    """Node u in community u K // n and, for about 30 % of the nodes, in one more; every entry fval."""
    rng = np.random.default_rng(seed)
    rows = []
    for u in range(n):
        r = {(u * K) // n}
        if rng.random() < 0.3:
            r.add(int(rng.integers(0, K)))
        rows.append(sorted(r))
    indptr = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
    indices = np.array([c for r in rows for c in r], dtype=np.int32)
    return indptr, indices, np.full(len(indices), float(fval))


def test_planted_model_on_isolated_nodes():
    from bigclam_apachespark_b200 import BigClam
    n, K = (120 if EMU else 5000), (4 if EMU else 60)
    for fval in (0.9, 0.2):                                                        # above delta, then below it (the tie rule)
        ip, ix, vl = _planted(n, K, fval, seed=6)
        b = BigClam(sparse_rows=True)
        b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
        comptr, members, zero_rows = b.extract_communities(DELTA)
        owner = np.repeat(np.arange(n, dtype=np.int32), np.diff(ip))
        assert len(zero_rows) == 0
        for c in range(K):
            assert np.array_equal(members[comptr[c]:comptr[c + 1]], owner[ix == c]), (fval, c)
        b.close()


def test_several_ranges(monkeypatch):
    """A budget of a few hundred bytes cuts the communities into many ranges (and bigclam_extract's rows into many
    batches); a community longer than the budget gets a range of its own.  The same bits as one range."""
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=9)
    F0 = _F0(n, K, seed=9, delta=DELTA)
    F0[10:60, 4] = 2 * DELTA                                                        # a community of >= 50 members: 200+ bytes
    F0[60:70] = 0.0                                                                 # zero rows: the last range
    for sparse in (True, False):
        b = _solver(rp, col, K, F0, sparse=sparse)
        one = b.extract_communities(DELTA)
        from bigclam_apachespark_b200 import communities as Cm
        ref = Cm.extract(b, DELTA)
        for budget in ("160", "1"):
            monkeypatch.setenv("BIGCLAM_EXTRACT_BUDGET", budget)
            assert _same(b.extract_communities(DELTA), one), (sparse, budget)
            r = Cm.extract(b, DELTA)
            assert np.array_equal(r[2], ref[2]) and np.array_equal(r[1], ref[1])
            monkeypatch.delenv("BIGCLAM_EXTRACT_BUDGET")
        assert _same(one, _twin(b, DELTA))
        b.close()


def test_state_untouched_by_extraction():
    rp, col = random_graph(120 if EMU else 600, 6, seed=31)
    n, K = len(rp) - 1, 24
    F0 = _F0(n, K, seed=31, delta=DELTA)
    a = _solver(rp, col, K, F0, time_kernels=True)
    c = _solver(rp, col, K, F0, time_kernels=True)
    for it in range(4):
        la, lc = a.backtrackingLineSearchs(), c.backtrackingLineSearchs()
        assert np.float64(la).view(np.int64) == np.float64(lc).view(np.int64), it
        assert a.kernel_time()[1:] == c.kernel_time()[1:], it                       # from the 2nd step on, both commit the speculation
        if it > 0:
            assert a.kernel_time()[1] == 1
        a.extract_communities(DELTA)
        a.extract_communities(float("inf"))
    for x, y in zip(a.F_csr(), c.F_csr()):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert np.array_equal(a.sumF.view(np.int64), c.sumF.view(np.int64))
    assert np.array_equal(a.accepted(), c.accepted())
    assert np.float64(a.loglikelihood()).view(np.int64) == np.float64(c.loglikelihood()).view(np.int64)
    a.close()
    c.close()


def test_argument_checks():
    from bigclam_apachespark_b200 import _lib as L
    rp, col = random_graph(100, 4, seed=3)
    n, K = len(rp) - 1, 8
    F0 = _F0(n, K, seed=3, delta=DELTA)
    b = _solver(rp, col, K, F0, time_kernels=True)
    b.backtrackingLineSearchs()
    lib = L.load()
    ctx = b._ctx
    nnz, z = C.c_int64(-5), C.c_int64(-6)
    cp = np.zeros(K + 1, dtype=np.int64)
    mo = np.zeros(K * n, dtype=np.int32)
    zo = np.zeros(n, dtype=np.int32)
    for delta in (float("nan"), 0.0, -0.0, -1e-9, -float("inf")):
        assert lib.bigclam_extract_nnz(ctx, delta, C.byref(nnz), C.byref(z)) == L.EINVAL, delta
        assert b"delta" in lib.bigclam_last_error(ctx)
        assert lib.bigclam_extract_grouped(ctx, delta, cp.ctypes.data, mo.ctypes.data, zo.ctypes.data) == L.EINVAL, delta
    assert nnz.value == -5 and z.value == -6 and not cp.any()
    assert lib.bigclam_extract_nnz(ctx, DELTA, None, C.byref(z)) == L.EINVAL
    assert lib.bigclam_extract_nnz(ctx, DELTA, C.byref(nnz), None) == L.EINVAL
    assert lib.bigclam_extract_grouped(ctx, DELTA, None, mo.ctypes.data, zo.ctypes.data) == L.EINVAL
    assert lib.bigclam_extract_grouped(ctx, DELTA, cp.ctypes.data, None, zo.ctypes.data) == L.EINVAL
    assert lib.bigclam_extract_grouped(ctx, DELTA, cp.ctypes.data, mo.ctypes.data, None) == L.EINVAL
    assert b"NULL" in lib.bigclam_last_error(ctx)
    with pytest.raises(L.BigclamError):
        b.extract_communities(0.0)
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    assert lib.bigclam_extract_nnz(ctx, DELTA, C.byref(nnz), C.byref(z)) == L.OK
    g = b.extract_communities(DELTA)
    assert nnz.value == len(g[1]) and z.value == len(g[2])
    b.close()
    # a negative entry (set_F can leave one): BIGCLAM_EUNSUPPORTED naming the smallest such row
    F1 = F0.copy()
    F1[37, 2] = -1e-3
    F1[71, 0] = -2.0
    for sparse in (True, False):
        b = _solver(rp, col, K, F1, sparse=sparse)
        assert lib.bigclam_extract_nnz(b._ctx, DELTA, C.byref(nnz), C.byref(z)) == L.EUNSUPPORTED
        assert b"row 37 " in lib.bigclam_last_error(b._ctx)
        assert lib.bigclam_extract_grouped(b._ctx, DELTA, cp.ctypes.data, mo.ctypes.data, zo.ctypes.data) == L.EUNSUPPORTED
        b.close()


def test_multi_gpu_handle_matches_one_context():
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=41)
    F0 = _F0(n, K, seed=41, delta=DELTA)
    one = _solver(rp, col, K, F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    for it in range(2):
        for delta in (DELTA, float("inf")):
            assert _same(one.extract_communities(delta), two.extract_communities(delta)), (it, delta)
        if it == 0:                                                                 # one step: the same rows on both
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    assert _same(two.extract_communities(DELTA), _twin(one, DELTA))
    assert _lib().bigclam_multi_extract_nnz(two._multi, 0.0, C.byref(C.c_int64()), C.byref(C.c_int64())) == -1
    assert b"delta" in _lib().bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


def _build_cpp(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    exe = str(tmp_path / "extract")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"),
                        os.path.join(REPO, "tests", "cpp_host", "extract.cpp"), "-o", exe, "-L", libdir, f"-l:{libname}",
                        f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.mark.parametrize("world", [1, 2])
def test_cpp_mirror_agrees_with_python(tmp_path, world):
    from bigclam_apachespark_b200 import communities as Cm
    if world > 1 and int(_lib().bigclam_device_count()) < world:
        pytest.skip(f"needs {world} GPUs")
    exe = _build_cpp(tmp_path)
    n, K = (100 if EMU else 300), 37
    rp, col = random_graph(n, 5, seed=12)
    F0 = _F0(n, K, seed=12, delta=DELTA)
    deltas = [DELTA, 0.1, float("inf")]
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, len(deltas)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes() + np.array(deltas).tobytes())
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, str(inp), str(out), str(world)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                                 # delta = 0: bigclam::Error with BIGCLAM_EINVAL
    raw = open(out, "rb").read()
    b = _solver(rp, col, K, F0)
    o = 0
    for delta in deltas:
        comptr = np.frombuffer(raw, np.int64, K + 1, o)
        z = int(np.frombuffer(raw, np.int64, 1, o + 8 * (K + 1))[0])
        o += 8 * (K + 2)
        members = np.frombuffer(raw, np.int32, int(comptr[-1]), o)
        o += 4 * len(members)
        zero_rows = np.frombuffer(raw, np.int32, z, o)
        o += 4 * z
        assert _same((comptr, members, zero_rows), b.extract_communities(delta)), delta
        lists = []
        for _ in range(K):
            ln = int(np.frombuffer(raw, np.int64, 1, o)[0])
            lists.append(np.frombuffer(raw, np.int32, ln, o + 8))
            o += 8 + 4 * ln
        merged, _ = Cm.group(comptr, members, zero_rows)
        assert [x.tolist() for x in lists if len(x)] == [x.tolist() for x in merged], delta
        if world == 1:                                                              # the single-context extract: bigclam_extract's matrix
            member = Cm.extract(b, delta)[2]
            assert all(np.array_equal(lists[c], np.flatnonzero(member[:, c])) for c in range(K)), delta
    assert o == len(raw)
    b.close()
