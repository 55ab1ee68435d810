"""Graphs sampled from the model on the GPU (bigclam_sample_graph_nnz / bigclam_sample_graph and their multi-GPU twins,
BigClam.sample_graph, the C++ mirror): the CSR against the NumPy twin (tests/sample_twin.py) for sparse and dense rows at
every kind of K, the shape of the output, seeds, a planted model on isolated nodes, a sample cut into several batches,
the state a sample must leave untouched, and the argument checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import REPO, random_graph
from sample_twin import SampleTwin, sample_r

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


def _twin(b):
    return SampleTwin(*b.F_csr(), b.K, b.MIN_P_, b.MAX_P_)


def _F0(n, K, seed, per_row=6.0):
    """About per_row non-zeros per row, with the rows the definition has to get right: row 0 all zero (background pairs
    only), rows 1 and 2 sharing only component 0 at 1e-200 (x underflows to 0: the floor 1 - MAX_P_, not eps), rows 3
    and 4 at MAX_F_ (p = 1 - MIN_P_)."""
    rng = np.random.default_rng(seed)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < min(1.0, per_row / K))
    F0[0:3] = 0.0
    F0[1, 0] = F0[2, 0] = 1e-200
    F0[3] = np.where(rng.random(K) < min(1.0, per_row / K), 1000.0, 0.0)
    F0[3, K - 1] = 1000.0
    F0[4] = F0[3]
    return F0


def _eps(b):
    return (0.0, 1e-3, 1.0 - b.MAX_P_)


def _same(g, h):
    return np.array_equal(g[0], h[0]) and np.array_equal(g[1], h[1])


def _check_shape(rp, col, n):
    assert rp.dtype == np.int64 and col.dtype == np.int32 and len(rp) == n + 1
    assert rp[0] == 0 and rp[-1] == len(col) and (np.diff(rp) >= 0).all()
    u = np.repeat(np.arange(n), np.diff(rp))
    assert (col >= 0).all() and (col < n).all() and (u != col).all()                # no self loops
    step = np.diff(col.astype(np.int64))
    assert (step[u[1:] == u[:-1]] > 0).all()                                        # ascending, no duplicates
    fwd = np.sort(u.astype(np.int64) * n + col)
    bwd = np.sort(col.astype(np.int64) * n + u)
    assert np.array_equal(fwd, bwd)                                                 # symmetric


KS = [1, 37, 200, 1024, 1025, 9000]


@pytest.mark.parametrize("K", KS)
def test_sample_matches_twin(K):
    n = 100 if EMU else 300
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K)
    layouts = [True, False] if K <= 1024 else [True]
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        tw = _twin(b)
        for eps in _eps(b):
            g = b.sample_graph(seed=K + 11, eps=eps)
            assert _same(g, tw.sample(K + 11, eps)), (K, sparse, eps)
            _check_shape(*g, n)
            got[(sparse, eps)] = g
        b.close()
    if len(layouts) == 2:                                                           # the same F in both layouts: the same graph
        for eps in _eps(b):
            assert _same(got[(True, eps)], got[(False, eps)])


def test_facebook_after_steps():
    from bigclam_apachespark_b200 import graphs as G
    if EMU:
        pytest.skip("facebook is too large for the host emulation")
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(3):
        b.backtrackingLineSearchs()
    tw = _twin(b)
    for eps in _eps(b):
        g = b.sample_graph(seed=2024, eps=eps)
        assert _same(g, tw.sample(2024, eps)), eps
        _check_shape(*g, n)
    b.close()


def test_output_is_a_graph_the_library_takes():
    from bigclam_apachespark_b200 import BigClam
    n, K = (100 if EMU else 400), 12
    rp, col = random_graph(n, 5, seed=3)
    b = _solver(rp, col, K, _F0(n, K, seed=3, per_row=3.0))
    srp, scol = b.sample_graph(seed=9, eps=0.01)
    _check_shape(srp, scol, n)
    assert len(scol) > 0
    c = BigClam(sparse_rows=True)
    c.set_graph(srp, scol).set_K(K).set_F(_F0(n, K, seed=4))
    llh0 = c.loglikelihood()
    assert c.backtrackingLineSearchs() > llh0
    b.close()
    c.close()


def test_seeds():
    n, K = (80 if EMU else 300), 20
    rp, col = random_graph(n, 5, seed=5)
    b = _solver(rp, col, K, _F0(n, K, seed=5))
    tw = _twin(b)
    for eps in (0.0, 0.02):
        g1 = b.sample_graph(seed=7, eps=eps)
        assert _same(g1, b.sample_graph(seed=7, eps=eps))                           # same seed: same graph
        g2 = b.sample_graph(seed=8, eps=eps)
        assert not _same(g1, g2)                                                    # another seed: another graph
        top = (1 << 64) - 1                                                         # the whole 64-bit seed range
        assert _same(b.sample_graph(seed=top, eps=eps), tw.sample(top, eps))
    b.close()


def _planted(n, K, seed, size=40):
    """Communities of about `size` consecutive-ish nodes; every node in one or two of them, F = 0.9 or 0.5."""
    rng = np.random.default_rng(seed)
    rows = []
    for u in range(n):
        c0 = (u * K) // n
        r = {c0: 0.9}
        if rng.random() < 0.3:
            r[int(rng.integers(0, K))] = 0.5
        rows.append(r)
    indptr = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
    indices = np.array([c for r in rows for c in sorted(r)], dtype=np.int32)
    values = np.array([r[c] for r in rows for c in sorted(r)])
    return indptr, indices, values


def test_planted_model_on_isolated_nodes():
    from bigclam_apachespark_b200 import BigClam
    n, K = (120 if EMU else 2000), (4 if EMU else 50)
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(*_planted(n, K, seed=6))
    tw = _twin(b)
    for eps in (0.0, 1e-3):
        g = b.sample_graph(seed=31, eps=eps)
        assert _same(g, tw.sample(31, eps)), eps
        _check_shape(*g, n)
    # a component's members are linked with p = 1 - exp(-0.81) ~ 0.56 and almost nothing else is
    rp, col = b.sample_graph(seed=31, eps=0.0)
    assert len(col) > 0.3 * n * (n / K - 1)
    b.close()


def test_several_batches():
    """Pure background at eps = 0.9 on 20000 nodes: about 3.6e8 entries, 1.44 GB of int32, past the 1 GiB bound of a
    batch.  Every row against the twin's definition (all pairs unshared: edge iff r < eps)."""
    from bigclam_apachespark_b200 import BigClam
    if EMU:
        pytest.skip("needs more than 1 GiB of output")
    n, eps, seed = 20000, 0.9, 77
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(1)
    b.set_F_csr(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32), np.zeros(0))
    rp, col = b.sample_graph(seed=seed, eps=eps)
    b.close()
    assert len(col) * 4 > (1 << 30)
    v = np.arange(n, dtype=np.int64)
    for a in range(0, n, 400):
        u = np.arange(a, min(n, a + 400), dtype=np.int64)
        hit = (sample_r(seed, u[:, None], v[None, :]) < eps) & (u[:, None] != v[None, :])
        assert np.array_equal(np.diff(rp)[u], hit.sum(axis=1)), a
        assert np.array_equal(col[rp[u[0]]:rp[u[-1] + 1]], np.nonzero(hit)[1].astype(np.int32)), a


def test_state_untouched_by_samples():
    rp, col = random_graph(120 if EMU else 600, 6, seed=31)
    n, K = len(rp) - 1, 24
    F0 = _F0(n, K, seed=31)
    a = _solver(rp, col, K, F0, time_kernels=True)
    c = _solver(rp, col, K, F0, time_kernels=True)
    for it in range(4):
        la, lc = a.backtrackingLineSearchs(), c.backtrackingLineSearchs()
        assert np.float64(la).view(np.int64) == np.float64(lc).view(np.int64), it
        assert a.kernel_time()[1:] == c.kernel_time()[1:], it                       # from the 2nd step on, both commit the speculation
        if it > 0:
            assert a.kernel_time()[1] == 1
        a.sample_graph(seed=it, eps=0.0)
        a.sample_graph(seed=it, eps=1e-3)
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
    b = _solver(rp, col, K, _F0(n, K, seed=3), time_kernels=True)
    b.backtrackingLineSearchs()
    lib = L.load()
    ctx = b._ctx
    nnz = C.c_int64(-5)
    rpo = np.zeros(n + 1, dtype=np.int64)
    co = np.zeros(10 * n, dtype=np.int32)
    for eps in (float("nan"), -1e-9, 1.0, 2.0, float("inf")):
        assert lib.bigclam_sample_graph_nnz(ctx, 1, eps, C.byref(nnz)) == L.EINVAL, eps
        assert b"eps" in lib.bigclam_last_error(ctx)
        assert lib.bigclam_sample_graph(ctx, 1, eps, rpo.ctypes.data, co.ctypes.data) == L.EINVAL, eps
    assert nnz.value == -5 and not rpo.any()
    assert lib.bigclam_sample_graph_nnz(ctx, 1, 0.0, None) == L.EINVAL
    assert lib.bigclam_sample_graph(ctx, 1, 0.0, None, co.ctypes.data) == L.EINVAL
    assert lib.bigclam_sample_graph(ctx, 1, 0.0, rpo.ctypes.data, None) == L.EINVAL
    assert b"NULL" in lib.bigclam_last_error(ctx)
    with pytest.raises(L.BigclamError):
        b.sample_graph(seed=1, eps=1.0)
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    assert lib.bigclam_sample_graph_nnz(ctx, 1, 0.0, C.byref(nnz)) == L.OK and nnz.value == len(b.sample_graph(1, 0.0)[1])
    b.close()


def test_multi_gpu_handle_matches_one_context():
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=41)
    F0 = _F0(n, K, seed=41)
    one = _solver(rp, col, K, F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    for it in range(2):
        for eps in (0.0, 1e-3):
            assert _same(one.sample_graph(5, eps), two.sample_graph(5, eps)), (it, eps)
        if it == 0:                                                                 # one step: the same rows on both
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    assert _same(two.sample_graph(5, 1e-3), _twin(one).sample(5, 1e-3))
    assert _lib().bigclam_multi_sample_graph_nnz(two._multi, 1, -1.0, C.byref(C.c_int64())) == -1
    assert b"eps" in _lib().bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


def _build_cpp(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    exe = str(tmp_path / "sample_graph")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"),
                        os.path.join(REPO, "tests", "cpp_host", "sample_graph.cpp"), "-o", exe, "-L", libdir, f"-l:{libname}",
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
    F0 = _F0(n, K, seed=12)
    cases = [(3, 0.0), (3, 1e-3), ((1 << 64) - 2, 1.0 - 0.9999)]
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, len(cases)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes())
        for s, e in cases:
            f.write(np.array([s], dtype=np.uint64).tobytes() + np.array([e]).tobytes())
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, str(inp), str(out), str(world)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                                 # eps = 1: bigclam::Error with BIGCLAM_EINVAL
    raw = open(out, "rb").read()
    b = _solver(rp, col, K, F0)
    o = 0
    for s, e in cases:
        nnz = int(np.frombuffer(raw, np.int64, 1, o)[0])
        grp = np.frombuffer(raw, np.int64, n + 1, o + 8)
        gcol = np.frombuffer(raw, np.int32, nnz, o + 8 + 8 * (n + 1))
        o += 8 + 8 * (n + 1) + 4 * nnz
        assert _same((grp, gcol), b.sample_graph(s, e)), (s, e)
    assert o == len(raw)
    b.close()
