"""Community overlaps on the GPU (bigclam_community_overlaps and its multi-GPU twin, BigClam.community_overlaps, the C++
mirror): every array bit for bit, dtypes included, against the NumPy twin (tests/community_overlaps_twin.py) for sparse
and dense rows at every kind of K, several deltas and min_shared values and both zero-row modes; the same arrays from
both layouts and under many output ranges; symmetry; sizes and zero rows against extract_communities and the row-sum
identity; com-amazon's ground-truth communities planted as F, against set intersections; a planted model whose overlaps
are known by construction; fitted facebook and com-amazon; the state a query must leave untouched; and the argument
checks."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from community_overlaps_twin import community_overlaps as twin_overlaps
from conftest import REPO, random_graph
from test_gpu_extract import _F0

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"
KEYS = ("ptr", "other", "shared", "size", "jaccard")


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def _solver(rp, col, K, F0, sparse=True, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse, record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    return b


def _same(g, h):
    """Every array bit for bit with the same dtype and shape, and the same zero-row count."""
    for key in KEYS:
        x, y = np.asarray(g[key]), np.asarray(h[key])
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), key
    assert g["zero_rows"] == h["zero_rows"]


def _twin(b, delta, min_shared=1, everywhere=True):
    return twin_overlaps(*b.F_csr(), b.K, delta, min_shared, everywhere)


def _symmetric(g):
    K = len(g["size"])
    rows = np.repeat(np.arange(K), np.diff(g["ptr"]))
    assert (rows != g["other"]).all()
    fwd = sorted(zip(rows.tolist(), g["other"].tolist(), g["shared"].tolist()))
    assert fwd == sorted((d, c, a) for c, d, a in fwd)


KS = [1, 37, 200, 1024, 1025, 9000]
DELTA = 0.5


@pytest.mark.parametrize("K", KS)
def test_overlaps_match_twin(K):
    n = 100 if EMU else (600 if K == 9000 else 300)
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K, delta=DELTA, per_row=6.0 if K < 1000 else 40.0)
    layouts = [True, False] if K <= 1024 else [True]
    slow = EMU and K > 1000                                                         # (k blocks of 256 host threads a launch)
    deltas = (DELTA,) if slow else (DELTA, 0.1, float("inf"))
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        for delta in deltas:
            for min_shared in (1, n + 1) if slow else (1, 2, n + 1):
                for everywhere in (True,) if slow else (True, False):
                    g = b.community_overlaps(delta, min_shared, everywhere)
                    _same(g, _twin(b, delta, min_shared, everywhere))
                    _symmetric(g)
                    got[(sparse, delta, min_shared, everywhere)] = g
                if min_shared == n + 1:
                    assert len(g["other"]) == 0
        b.close()
    if len(layouts) == 2:                                                           # the same F in both layouts: the same outputs
        for key in [k for k in got if k[0]]:
            _same(got[key], got[(False,) + key[1:]])


@pytest.mark.parametrize("sparse", [True, False])
def test_many_output_ranges(sparse, monkeypatch):
    """A scratch bound of a few entries cuts the output into many ranges (down to one row each); a bound below one row
    still gives that row a range of its own.  The arrays do not change."""
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=5)
    b = _solver(rp, col, K, _F0(n, K, seed=5, delta=DELTA, per_row=8.0), sparse=sparse)
    want = b.community_overlaps(DELTA)
    assert len(want["other"]) > 3 * K
    for budget in ("1", "64", "1000"):
        monkeypatch.setenv("BIGCLAM_EXTRACT_BUDGET", budget)
        _same(b.community_overlaps(DELTA), want)
    b.close()


def test_sizes_zero_rows_and_row_sums():
    """size and z equal extract_communities' comptr and zero rows; at min_shared = 1 the shared counts of row c add up to
    the sum over u in M_c of (m_u - 1), m_u the number of communities u is in."""
    n, K = (100 if EMU else 500), 37
    rp, col = random_graph(n, 5, seed=6)
    F0 = _F0(n, K, seed=6, delta=DELTA, per_row=7.0)
    F0[20:40] = 0.0
    b = _solver(rp, col, K, F0)
    for delta in (DELTA, 0.1, float("inf")):
        comptr, members, zero_rows = b.extract_communities(delta)
        g = b.community_overlaps(delta, zero_rows_everywhere=False)
        assert np.array_equal(g["size"], np.diff(comptr)) and g["zero_rows"] == len(zero_rows)
        m = np.bincount(members, minlength=n)
        sums = np.add.reduceat(np.append(g["shared"].astype(np.int64), 0), g["ptr"][:-1]) * (np.diff(g["ptr"]) > 0)
        want = [int((m[members[comptr[c]:comptr[c + 1]]] - 1).sum()) for c in range(K)]
        assert sums.tolist() == want, delta
        h = b.community_overlaps(delta)                                             # as coded: + z everywhere
        assert np.array_equal(h["size"], g["size"] + len(zero_rows))
        assert np.array_equal(h["shared"], g["shared"] + len(zero_rows)) and np.array_equal(h["other"], g["other"])
    b.close()


def test_planted_model_overlaps_by_construction():
    """A planted model (node u in community u K // n, 30 % also in a second one, F = 0.15): at either side of F the
    communities are the planted ones, so shared(c, d) is the number of nodes planted in both c and d."""
    from bigclam_apachespark_b200 import BigClam
    sys.path.insert(0, os.path.join(REPO, "scripts"))
    from bench_sample import _planted
    n, K = (300, 12) if EMU else (200_000, 1000)
    ip, ix, vl = _planted(n, K, 0.15, 0.3, seed=3)
    two = np.diff(ip) == 2
    lo, hi = ix[ip[:-1][two]].astype(np.int64), ix[ip[:-1][two] + 1].astype(np.int64)
    pairs = np.bincount(np.concatenate([lo * K + hi, hi * K + lo]), minlength=K * K).reshape(K, K)
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    for delta in (0.1, 0.5):
        g = b.community_overlaps(delta)
        assert g["zero_rows"] == 0
        assert np.array_equal(g["size"], np.bincount(ix, minlength=K))
        assert np.array_equal(g["ptr"], np.concatenate([[0], np.cumsum((pairs > 0).sum(axis=1))]))
        r, d = np.nonzero(pairs)
        assert np.array_equal(g["other"], d.astype(np.int32)) and np.array_equal(g["shared"], pairs[r, d].astype(np.int32))
    b.close()


def test_amazon_ground_truth_planted():
    """F = 1 on the members of com-amazon's first 5000 ground-truth communities: every community is its ground-truth set,
    and every count is the size of a Python set intersection."""
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G
    if EMU:
        pytest.skip("com-amazon is GPU only")
    rp, col, _ = G.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 5000
    truth = [np.unique(t) for t in Cm.load_ground_truth()[:K]]
    rows = np.concatenate(truth).astype(np.int64)
    cols = np.repeat(np.arange(K), [len(t) for t in truth])
    o = np.lexsort((cols, rows))
    ip = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=ip[1:])
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col).set_K(K).set_F_csr(ip, cols[o].astype(np.int32), np.ones(len(rows)))
    g = b.community_overlaps(0.5, zero_rows_everywhere=False)
    sets = [set(t.tolist()) for t in truth]
    of = {}                                                                         # node -> its communities
    for c, t in enumerate(truth):
        for u in t.tolist():
            of.setdefault(u, []).append(c)
    cand = {}
    for cs in of.values():
        for c in cs:
            cand.setdefault(c, set()).update(cs)
    ptr, other, shared = [0], [], []
    for c in range(K):
        for d in sorted(cand.get(c, set()) - {c}):
            other.append(d)
            shared.append(len(sets[c] & sets[d]))
        ptr.append(len(other))
    assert np.array_equal(g["size"], [len(s) for s in sets])
    assert g["zero_rows"] == n - len(of)
    assert np.array_equal(g["ptr"], ptr) and np.array_equal(g["other"], other) and np.array_equal(g["shared"], shared)
    assert len(other) > 0
    b.close()


def test_fitted_models():
    from bigclam_apachespark_b200 import BigClam, communities as Cm, graphs as G
    if EMU:
        pytest.skip("the fitted graphs are GPU only")
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(5):
        b.backtrackingLineSearchs()
    for delta in (Cm.delta_threshold(n, int((np.diff(rp) > 0).sum())), 0.5):
        for everywhere in (True, False):
            _same(b.community_overlaps(delta, 1, everywhere), _twin(b, delta, 1, everywhere))
    b.close()
    rp, col, _ = G.load_npz_graph("com-amazon")
    n = len(rp) - 1
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col)
    b.initNeighborComF(200)
    for _ in range(3):
        b.backtrackingLineSearchs()
    delta = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))
    for min_shared in (1, 10):
        for everywhere in (True, False):
            g = b.community_overlaps(delta, min_shared, everywhere)
            _same(g, _twin(b, delta, min_shared, everywhere))
    _symmetric(g)
    b.close()


def test_state_untouched_by_overlaps():
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
        a.community_overlaps(DELTA)
        a.community_overlaps(float("inf"), 2, zero_rows_everywhere=False)
    for x, y in zip(a.F_csr(), c.F_csr()):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert np.array_equal(a.sumF.view(np.int64), c.sumF.view(np.int64))
    assert np.array_equal(a.accepted(), c.accepted())
    assert np.float64(a.loglikelihood()).view(np.int64) == np.float64(c.loglikelihood()).view(np.int64)
    a.close()
    c.close()


def test_argument_checks():
    import ctypes as C
    from bigclam_apachespark_b200 import _lib as L
    rp, col = random_graph(100, 4, seed=3)
    n, K = len(rp) - 1, 8
    F0 = _F0(n, K, seed=3, delta=DELTA)
    b = _solver(rp, col, K, F0, time_kernels=True)
    b.backtrackingLineSearchs()
    lib = L.load()
    ctx = b._ctx
    nnz, z = C.c_int64(-7), C.c_int64(-7)
    ptr, size = np.full(K + 1, -7, dtype=np.int64), np.full(K, -7, dtype=np.int64)
    other, shared = np.full(K * K, -7, dtype=np.int32), np.full(K * K, -7, dtype=np.int32)
    outs = [ptr, other, shared, size]

    def call(delta=DELTA, ms=1, o=None):
        o = [x.ctypes.data for x in outs] if o is None else o
        return lib.bigclam_community_overlaps(ctx, delta, ms, *o)

    def rejected(rc, what):
        assert rc == L.EINVAL, what
        assert what in lib.bigclam_last_error(ctx), (what, lib.bigclam_last_error(ctx))

    for delta in (float("nan"), 0.0, -0.0, -1e-9, -float("inf")):
        rejected(call(delta=delta), b"delta")
        rejected(lib.bigclam_community_overlaps_nnz(ctx, delta, 1, C.byref(nnz), C.byref(z)), b"delta")
    for ms in (0, -1, -(1 << 31)):
        rejected(call(ms=ms), b"min_shared")
        rejected(lib.bigclam_community_overlaps_nnz(ctx, DELTA, ms, C.byref(nnz), C.byref(z)), b"min_shared")
    for i in range(3):                                                              # other / shared even when nnz would be 0
        o = [x.ctypes.data for x in outs]
        o[i] = None
        rejected(call(o=o), b"NULL")
        rejected(call(ms=n + 1, o=o), b"NULL")
    rejected(lib.bigclam_community_overlaps_nnz(ctx, DELTA, 1, None, C.byref(z)), b"NULL")
    rejected(lib.bigclam_community_overlaps_nnz(ctx, DELTA, 1, C.byref(nnz), None), b"NULL")
    assert nnz.value == -7 and z.value == -7 and all((x == -7).all() for x in outs)
    with pytest.raises(L.BigclamError):
        b.community_overlaps(0.0)
    with pytest.raises(L.BigclamError):
        b.community_overlaps(DELTA, min_shared=0)
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    o = [x.ctypes.data for x in outs]
    o[3] = None                                                                     # size_out is optional
    assert call(o=o) == L.OK and (size == -7).all()
    g = b.community_overlaps(DELTA, zero_rows_everywhere=False)
    m = int(g["ptr"][-1])
    assert np.array_equal(ptr, g["ptr"]) and np.array_equal(other[:m], g["other"]) and np.array_equal(shared[:m], g["shared"])
    assert (other[m:] == -7).all()
    b.close()
    # a negative entry (set_F can leave one): BIGCLAM_EUNSUPPORTED naming the smallest such row
    F1 = F0.copy()
    F1[37, 2] = -1e-3
    F1[71, 0] = -2.0
    for sparse in (True, False):
        b = _solver(rp, col, K, F1, sparse=sparse)
        assert lib.bigclam_community_overlaps_nnz(b._ctx, DELTA, 1, C.byref(nnz), C.byref(z)) == L.EUNSUPPORTED
        assert b"row 37 " in lib.bigclam_last_error(b._ctx)
        assert lib.bigclam_community_overlaps(b._ctx, DELTA, 1, *[x.ctypes.data for x in outs]) == L.EUNSUPPORTED
        assert b"row 37 " in lib.bigclam_last_error(b._ctx)
        b.close()


def test_multi_gpu_handle_matches_one_context():
    import ctypes as C
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=41)
    F0 = _F0(n, K, seed=41, delta=DELTA, per_row=8.0)
    one = _solver(rp, col, K, F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    for it in range(2):
        for delta in (DELTA,) if EMU else (DELTA, float("inf")):
            for min_shared in (1, 3):
                for everywhere in (True, False):
                    _same(one.community_overlaps(delta, min_shared, everywhere), two.community_overlaps(delta, min_shared, everywhere))
        if it == 0:                                                                 # one step: the same rows on both
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    _same(two.community_overlaps(DELTA), _twin(one, DELTA))
    nnz, z = C.c_int64(), C.c_int64()
    assert _lib().bigclam_multi_community_overlaps_nnz(two._multi, DELTA, 0, C.byref(nnz), C.byref(z)) == -1
    assert b"min_shared" in _lib().bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


def _build_cpp(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    exe = str(tmp_path / "community_overlaps")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"),
                        os.path.join(REPO, "tests", "cpp_host", "community_overlaps.cpp"), "-o", exe, "-L", libdir, f"-l:{libname}",
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
    F0 = _F0(n, K, seed=12, delta=DELTA, per_row=8.0)
    cases = [(DELTA, 1), (0.1, 2), (float("inf"), 1)]
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, len(cases)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes())
        f.write(np.array([d for d, _ in cases]).tobytes() + np.array([m for _, m in cases], dtype=np.int32).tobytes())
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, str(inp), str(out), str(world)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                                 # min_shared = 0: bigclam::Error with BIGCLAM_EINVAL
    raw = open(out, "rb").read()
    b = _solver(rp, col, K, F0)
    o = 0

    def take(dtype, count):
        nonlocal o
        x = np.frombuffer(raw, dtype, count, o)
        o += x.nbytes
        return x

    for delta, min_shared in cases:
        for everywhere in (True, False):
            nnz, z = take(np.int64, 2)
            g = dict(zero_rows=int(z), ptr=take(np.int64, K + 1), size=take(np.int64, K))
            g["other"], g["shared"], g["jaccard"] = take(np.int32, nnz), take(np.int32, nnz), take(np.float64, nnz)
            _same(g, b.community_overlaps(delta, min_shared, everywhere))
    assert o == len(raw)
    b.close()
