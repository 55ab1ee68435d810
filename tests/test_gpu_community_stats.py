"""Community scores on the GPU (bigclam_community_stats and its multi-GPU twin, BigClam.community_stats, the C++
mirror): exact arrays against the NumPy twin (tests/community_stats_twin.py) for sparse and dense rows at every kind of K,
both zero-row modes and several deltas; agreement with extraction; ego nets scored exactly as conductanceLocalMin's GPU
kernel scores their centres; com-amazon's ground-truth communities against counts taken from the lists themselves;
fitted models; the state a query must leave untouched; and the argument checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from community_stats_twin import community_stats as twin_stats
from conftest import REPO, random_graph
from test_community_stats_cpu import _ego_F, clean_centres, keep_graph
from test_gpu_extract import _F0

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"
KEYS = ("size", "volume", "internal", "conductance")


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def _solver(rp, col, K, F0, sparse=True, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse, record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    return b


def _twin(b, delta, everywhere=True):
    return twin_stats(*b.F_csr(), b.K, delta, b.rowptr, b.col, zero_rows=everywhere)


def _same(g, h):
    """Equal arrays, dtypes and bits (conductance compared as bits)."""
    for key in KEYS:
        x, y = np.asarray(g[key]), np.asarray(h[key])
        if x.dtype != y.dtype or x.shape != y.shape or not np.array_equal(x.view(np.int64), y.view(np.int64)):
            return False
    return True


def _agrees_with_extraction(b, delta, g, everywhere):
    comptr, _, zero_rows = b.extract_communities(delta)
    return np.array_equal(g["size"], np.diff(comptr) + (len(zero_rows) if everywhere else 0))


KS = [1, 37, 200, 1024, 1025, 9000]
DELTA = 0.5


@pytest.mark.parametrize("K", KS)
def test_stats_match_twin(K):
    n = 100 if EMU else (600 if K == 9000 else 300)
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K, delta=DELTA)
    layouts = [True, False] if K <= 1024 else [True]
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        for delta in (DELTA, 0.1, float("inf")):
            for everywhere in (True, False):
                g = b.community_stats(delta, zero_rows_everywhere=everywhere)
                assert _same(g, _twin(b, delta, everywhere)), (K, sparse, delta, everywhere)
                assert _agrees_with_extraction(b, delta, g, everywhere), (K, sparse, delta, everywhere)
                got[(sparse, delta, everywhere)] = g
        b.close()
    if len(layouts) == 2:                                                           # the same F in both layouts: the same arrays
        for key in [k for k in got if k[0]]:
            assert _same(got[key], got[(False,) + key[1:]]), key


@pytest.mark.parametrize("sparse", [True, False])
def test_zero_row_modes(sparse):
    """The zero rows' part is the difference between the modes: z in every size, their degrees in every volume, the
    entries between a zero row and a member (either way) or another zero row in every internal count."""
    n, K = 60, 16
    rp, col = random_graph(n, 4, seed=2)
    F0 = _F0(n, K, seed=2, delta=DELTA)
    F0[10:20] = 0.0
    b = _solver(rp, col, K, F0, sparse=sparse)
    one, zero = b.community_stats(DELTA), b.community_stats(DELTA, zero_rows_everywhere=False)
    z = np.flatnonzero(~F0.any(axis=1))
    assert {0, 5, 10} <= set(z.tolist())
    deg = np.diff(rp)
    assert np.array_equal(one["size"] - zero["size"], np.full(K, len(z)))
    assert np.array_equal(one["volume"] - zero["volume"], np.full(K, deg[z].sum()))
    from extract_twin import dense_member
    M = dense_member(F0, DELTA)
    isz = np.zeros(n, dtype=bool)
    isz[z] = True
    for c in range(K):
        extra = 0
        for u in range(n):
            for v in col[rp[u]:rp[u + 1]]:
                extra += (M[u, c] and isz[v]) or (isz[u] and (M[v, c] or isz[v]))
        assert one["internal"][c] - zero["internal"][c] == extra, c
    assert _same(one, _twin(b, DELTA)) and _same(zero, _twin(b, DELTA, False))
    b.close()


def _ego_graphs(tmp_path):
    from bigclam_apachespark_b200 import graphs as G
    if not EMU:
        rp, col, _ = G.load_npz_graph("facebook_combined")
        yield "facebook", rp, col
    yield "keep", *keep_graph(tmp_path, n=150 if EMU else 400)


def test_ego_nets_equal_conductance_seeds_gpu(tmp_path):
    from bigclam_apachespark_b200 import BigClam
    for name, rp, col in _ego_graphs(tmp_path):
        centres = clean_centres(rp, col, 40 if EMU else 300, seed=1)
        K = len(centres)
        ref = BigClam()
        ref.set_graph(rp, col)
        ref.conductanceLocalMin(on_gpu=True)
        b = BigClam(sparse_rows=True)
        b.set_graph(rp, col).set_K(K).set_F_csr(*_ego_F(rp, col, centres))
        g = b.community_stats(DELTA, zero_rows_everywhere=False)
        assert np.array_equal(g["size"], np.diff(rp)[centres] + 1), name
        assert np.array_equal(g["conductance"].view(np.int64), ref.conductance[centres].view(np.int64)), name
        assert _same(g, _twin(b, DELTA, False)), name
        b.close()
        ref.close()


def test_amazon_ground_truth_communities():
    """F planted from the first 5000 ground-truth communities of com-amazon (wide rows): the scores are counts taken
    from the neighbour lists themselves."""
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G
    if EMU:
        pytest.skip("com-amazon is GPU only")
    rp, col, _ = G.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 5000
    truth = [np.unique(c) for c in Cm.load_ground_truth()[:K]]
    u = np.concatenate(truth).astype(np.int64)
    c = np.repeat(np.arange(K, dtype=np.int64), [len(t) for t in truth])
    o = np.lexsort((c, u))
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(u, minlength=n), out=indptr[1:])
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col).set_K(K).set_F_csr(indptr, c[o].astype(np.int32), np.ones(len(u)))
    g = b.community_stats(DELTA, zero_rows_everywhere=False)
    deg = np.diff(rp)
    for k, S in enumerate(truth):
        inside = sum(int(np.isin(col[rp[x]:rp[x + 1]], S).sum()) for x in S)
        assert (g["size"][k], g["volume"][k], g["internal"][k]) == (len(S), deg[S].sum(), inside), k
    assert _same(g, _twin(b, DELTA, False))
    assert _same(b.community_stats(DELTA), _twin(b, DELTA, True))
    b.close()


def test_fitted_facebook_and_amazon():
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G
    if EMU:
        pytest.skip("facebook and com-amazon are too large for the host emulation")
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(3):
        b.backtrackingLineSearchs()
    for delta in (Cm.delta_threshold(n, int((np.diff(rp) > 0).sum())), 0.5):
        for everywhere in (True, False):
            assert _same(b.community_stats(delta, everywhere), _twin(b, delta, everywhere)), (delta, everywhere)
    b.close()
    rp, col, _ = G.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 200
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    b.initNeighborComF(K)
    for _ in range(3):
        b.backtrackingLineSearchs()
    delta = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))
    for everywhere in (True, False):
        g = b.community_stats(delta, everywhere)
        assert _same(g, _twin(b, delta, everywhere)), everywhere
        assert _agrees_with_extraction(b, delta, g, everywhere)
    b.close()


def test_state_untouched_by_stats():
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
        a.community_stats(DELTA)
        a.community_stats(float("inf"), zero_rows_everywhere=False)
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
    out = [np.full(K, -7, dtype=np.int64) for _ in range(3)]
    cond = np.full(K, -7.0)
    ptrs = [x.ctypes.data for x in out]
    for delta in (float("nan"), 0.0, -0.0, -1e-9, -float("inf")):
        assert lib.bigclam_community_stats(ctx, delta, 1, *ptrs, cond.ctypes.data) == L.EINVAL, delta
        assert b"delta" in lib.bigclam_last_error(ctx)
    for zr in (-1, 2, 255):
        assert lib.bigclam_community_stats(ctx, DELTA, zr, *ptrs, cond.ctypes.data) == L.EINVAL, zr
        assert b"zero_rows" in lib.bigclam_last_error(ctx)
    for i in range(3):
        p = list(ptrs)
        p[i] = None
        assert lib.bigclam_community_stats(ctx, DELTA, 1, *p, cond.ctypes.data) == L.EINVAL, i
        assert b"NULL" in lib.bigclam_last_error(ctx)
    assert all((x == -7).all() for x in out) and (cond == -7.0).all()
    with pytest.raises(L.BigclamError):
        b.community_stats(0.0)
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    assert lib.bigclam_community_stats(ctx, DELTA, 1, *ptrs, None) == L.OK                # conductance is optional
    g = b.community_stats(DELTA)
    assert all(np.array_equal(x, g[k]) for x, k in zip(out, KEYS))
    b.close()
    # a negative entry (set_F can leave one): BIGCLAM_EUNSUPPORTED naming the smallest such row
    F1 = F0.copy()
    F1[37, 2] = -1e-3
    F1[71, 0] = -2.0
    for sparse in (True, False):
        b = _solver(rp, col, K, F1, sparse=sparse)
        assert lib.bigclam_community_stats(b._ctx, DELTA, 0, *ptrs, cond.ctypes.data) == L.EUNSUPPORTED
        assert b"row 37 " in lib.bigclam_last_error(b._ctx)
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
            for everywhere in (True, False):
                assert _same(one.community_stats(delta, everywhere), two.community_stats(delta, everywhere)), (it, delta)
        if it == 0:                                                                 # one step: the same rows on both
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    assert _same(two.community_stats(DELTA), _twin(one, DELTA))
    z = np.zeros(K, dtype=np.int64)
    assert _lib().bigclam_multi_community_stats(two._multi, 0.0, 1, z.ctypes.data, z.ctypes.data, z.ctypes.data, None) == -1
    assert b"delta" in _lib().bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


def _build_cpp(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    exe = str(tmp_path / "community_stats")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"),
                        os.path.join(REPO, "tests", "cpp_host", "community_stats.cpp"), "-o", exe, "-L", libdir, f"-l:{libname}",
                        f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.mark.parametrize("world", [1, 2])
def test_cpp_mirror_agrees_with_python(tmp_path, world):
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
    assert len(raw) == len(deltas) * 2 * 4 * 8 * K
    b = _solver(rp, col, K, F0)
    o = 0
    for delta in deltas:
        for everywhere in (True, False):
            g = {}
            for key in KEYS:
                g[key] = np.frombuffer(raw, np.float64 if key == "conductance" else np.int64, K, o)
                o += 8 * K
            assert _same(g, b.community_stats(delta, everywhere)), (delta, everywhere)
    b.close()
