"""Edge probabilities and link recommendations on the GPU (bigclam_pair_affinity / bigclam_recommend and their multi-GPU
twins, BigClam.edge_probability / recommend, the C++ mirror): the affinity bits against the NumPy twin (tests/links_twin.py)
for sparse and dense rows, the tie to loglikelihood() through the per-edge term, the two-hop ranking against brute force,
the state a query must leave untouched, and the argument checks."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import REPO, random_graph
from links_twin import Twin

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"


def _solver(rp, col, K, F0, sparse=True, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse, record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    return b


def _twin(b):
    return Twin(*b.F_csr(), b.K, b.MIN_P_, b.MAX_P_)


def _F0(n, K, seed, per_row=8.0):
    """About per_row non-zeros per row, with the special rows the definition has to get right: row 0 all zero, rows 1
    and 2 without a common component, row 3 at MAX_F_ on its components (x far above x_hi), row 4 = row 3."""
    rng = np.random.default_rng(seed)
    F0 = rng.random((n, K)) * (rng.random((n, K)) < min(1.0, per_row / K))
    F0[0] = 0.0
    F0[1] = 0.0
    F0[2] = 0.0
    F0[1, 0] = 0.7
    if K > 1:
        F0[2, K - 1] = 0.4
    F0[3] = np.where(rng.random(K) < min(1.0, per_row / K), 1000.0, 0.0)
    F0[3, 0] = 1000.0
    F0[4] = F0[3]
    return F0


def _pairs(n, seed, count=3000):
    rng = np.random.default_rng(seed)
    u = rng.integers(0, n, count)
    v = rng.integers(0, n, count)
    sp = np.array([[0, 1], [1, 2], [2, 1], [3, 4], [3, 3], [0, 0], [1, 1], [5, 5], [3, 1]])
    u = np.concatenate([u, sp[:, 0], np.arange(n)])
    v = np.concatenate([v, sp[:, 1], np.arange(n)])           # self pairs: x_uu = F_u . F_u
    return u, v


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


KS = [1, 37, 200, 1024, 1025, 9000]


@pytest.mark.parametrize("K", KS)
def test_pair_affinity_bits(K):
    n = 120 if EMU else 300
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K)
    u, v = _pairs(n, seed=K, count=600 if EMU else 3000)
    layouts = [True, False] if K <= 1024 else [True]
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        x, p = b.edge_probability(u, v)
        xr, _ = b.edge_probability(v, u)
        tw = _twin(b)
        assert np.array_equal(_bits(x), _bits(tw.x(u, v))), f"K={K} sparse={sparse}"
        assert np.array_equal(_bits(x), _bits(xr))
        assert np.abs(p - tw.p(x)).max() <= 1e-15
        assert x[-n + 0] == 0.0 and x[-n + 3] >= 1e6                 # all-zero row, a row at MAX_F_
        assert p[-n + 3] == 1.0 - b.MIN_P_ and p[-n + 0] == 1.0 - b.MAX_P_
        got[sparse] = (x, p)
        b.close()
    if len(layouts) == 2:                                           # the same F in both layouts: the same bits
        assert np.array_equal(_bits(got[True][0]), _bits(got[False][0]))
        assert np.array_equal(_bits(got[True][1]), _bits(got[False][1]))


def _llh_from_edges(b, rp, col):
    """sum_u [ sum_{v in N(u)} (log p_uv + x_uv) - F_u . sumF + x_uu ]  (bigclam4-7.scala:196-219 through the pair calls)."""
    n = len(rp) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    x, p = b.edge_probability(u, col)
    xs, _ = b.edge_probability(np.arange(n), np.arange(n))
    ip, ix, vl = b.F_csr()
    fsum = np.bincount(np.repeat(np.arange(n), np.diff(ip)), weights=vl * b.sumF[ix], minlength=n)
    return (np.bincount(u, weights=np.log(p) + x, minlength=n) - fsum + xs).sum()


def test_objective_cross_check_facebook():
    from bigclam_apachespark_b200 import graphs as G
    rp, col, _ = G.load_npz_graph("facebook_combined")
    if EMU:
        pytest.skip("facebook is too large for the host emulation")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(3):
        b.backtrackingLineSearchs()
    llh = b.loglikelihood()
    assert abs(_llh_from_edges(b, rp, col) - llh) <= 1e-10 * abs(llh)
    b.close()


def test_objective_cross_check_amazon_k200():
    from bigclam_apachespark_b200 import graphs as G
    if EMU or not G.have_fixture("com-amazon"):
        pytest.skip("com-amazon on the GPU only")
    rp, col, _ = G.load_npz_graph("com-amazon")
    n, K = len(rp) - 1, 200
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col).set_K(K).set_F_csr(*G.synthetic_F0_csr(n, K, seed=1234, density=0.05))
    b.backtrackingLineSearchs()
    b.backtrackingLineSearchs()
    llh = b.loglikelihood()
    assert abs(_llh_from_edges(b, rp, col) - llh) <= 1e-10 * abs(llh)
    b.close()


def _keep_lists(rp, col, seed):
    """multiplicity = keep style lists: some entries repeated, every list shuffled."""
    rng = np.random.default_rng(seed)
    rows = []
    for u in range(len(rp) - 1):
        r = list(col[rp[u]:rp[u + 1]])
        r += [w for w in r if rng.random() < 0.3]
        rng.shuffle(r)
        rows.append(r)
    rp2 = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
    return rp2, np.array([w for r in rows for w in r], dtype=np.int32)


def _graphs():
    from bigclam_apachespark_b200 import graphs as G
    n = 150 if EMU else 500
    rp, col = random_graph(n, 5, seed=7, hub=n // 3)               # a hub with a long two-hop list
    # two extra nodes linked only to each other: no two-hop candidate at all
    u = np.repeat(np.arange(n), np.diff(rp))
    u2 = np.concatenate([u[u < col], [n]])
    v2 = np.concatenate([col[u < col], [n + 1]])
    rp, col = G.csr_from_undirected(n + 2, u2, v2)
    return {"simple": (rp, col), "keep": _keep_lists(rp, col, 8)}


def _check_recommend(b, rp, col, nodes, m):
    lib = _lib()
    cnt = b.n if nodes is None else len(nodes)
    q = None if nodes is None else np.ascontiguousarray(nodes, dtype=np.int32)
    vo = np.empty((cnt, m), dtype=np.int32)
    xo = np.empty((cnt, m))
    found = np.empty(cnt, dtype=np.int32)
    rc = lib.bigclam_recommend(b._ctx, None if q is None else q.ctypes.data, cnt, m, vo.ctypes.data, xo.ctypes.data, found.ctypes.data)
    assert rc == 0, lib.bigclam_last_error(b._ctx)
    tv, tx, tf = _twin(b).recommend(rp, col, nodes, m)
    assert np.array_equal(found, tf) and np.array_equal(vo, tv) and np.array_equal(_bits(xo), _bits(tx))
    v2, x2 = b.recommend(nodes, m)                                  # the Python surface gives the same
    assert np.array_equal(v2, vo) and np.array_equal(_bits(x2), _bits(xo))
    qn = np.arange(b.n) if nodes is None else np.asarray(nodes)
    sel = vo >= 0                                                   # the scores are bigclam_pair_affinity's bits
    xp, _ = b.edge_probability(np.repeat(qn, m).reshape(cnt, m)[sel], vo[sel])
    assert np.array_equal(_bits(xp), _bits(xo[sel]))
    return found


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


@pytest.mark.parametrize("graph", ["simple", "keep"])
@pytest.mark.parametrize("m", [1, 5, 50])
def test_recommend_against_brute_force(graph, m):
    rp, col = _graphs()[graph]
    n, K = len(rp) - 1, 37
    b = _solver(rp, col, K, _F0(n, K, seed=m))
    b.backtrackingLineSearchs()
    found = _check_recommend(b, rp, col, None, m)
    assert found[n - 1] == 0 and found[n - 2] == 0
    rng = np.random.default_rng(m)
    sub = np.concatenate([rng.integers(0, n, 40), [n - 1, 0, 0]])  # a subset with repeats
    _check_recommend(b, rp, col, sub, m)
    b.close()


def test_recommend_dense_rows_and_wide_k():
    rp, col = _graphs()["simple"]
    n = len(rp) - 1
    for K, sparse in ((37, False), (1500, True)):
        b = _solver(rp, col, K, _F0(n, K, seed=K), sparse=sparse)
        _check_recommend(b, rp, col, None, 5)
        b.close()


def test_state_untouched_by_queries():
    rp, col = random_graph(150 if EMU else 600, 6, seed=31)
    n, K = len(rp) - 1, 24
    F0 = _F0(n, K, seed=31)
    a = _solver(rp, col, K, F0, time_kernels=True)
    c = _solver(rp, col, K, F0, time_kernels=True)
    u, v = _pairs(n, seed=31, count=500)
    for it in range(4):
        la, lc = a.backtrackingLineSearchs(), c.backtrackingLineSearchs()
        assert _bits([la]) == _bits([lc]), it
        assert a.kernel_time()[1:] == c.kernel_time()[1:], it     # from the 2nd step on, both commit the speculation
        if it > 0:
            assert a.kernel_time()[1] == 1
        a.edge_probability(u, v)
        a.recommend(None, 5)
        a.recommend(np.arange(10), 3)
    for x, y in zip(a.F_csr(), c.F_csr()):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert np.array_equal(_bits(a.sumF), _bits(c.sumF))
    assert np.array_equal(a.accepted(), c.accepted())
    assert _bits([a.loglikelihood()]) == _bits([c.loglikelihood()])
    a.close()
    c.close()


def test_argument_checks():
    from bigclam_apachespark_b200 import _lib as L
    rp, col = random_graph(100, 4, seed=3)
    n, K = len(rp) - 1, 8
    b = _solver(rp, col, K, _F0(n, K, seed=3), time_kernels=True)
    b.backtrackingLineSearchs()
    lib = L.load()
    good = np.array([0, 1], dtype=np.int32)
    bad = np.array([0, n], dtype=np.int32)
    neg = np.array([-1, 0], dtype=np.int32)
    x = np.zeros(2)
    vo = np.zeros(2 * 3, dtype=np.int32)
    ctx = b._ctx
    assert lib.bigclam_pair_affinity(ctx, bad.ctypes.data, good.ctypes.data, 2, x.ctypes.data, None) == L.EINVAL
    assert b"u[1] = %d is outside" % n in lib.bigclam_last_error(ctx)
    assert lib.bigclam_pair_affinity(ctx, good.ctypes.data, neg.ctypes.data, 2, x.ctypes.data, None) == L.EINVAL
    assert lib.bigclam_pair_affinity(ctx, good.ctypes.data, good.ctypes.data, -1, x.ctypes.data, None) == L.EINVAL
    assert lib.bigclam_pair_affinity(ctx, good.ctypes.data, None, 2, x.ctypes.data, None) == L.EINVAL
    assert lib.bigclam_pair_affinity(ctx, good.ctypes.data, good.ctypes.data, 2, None, None) == L.EINVAL
    assert lib.bigclam_pair_affinity(ctx, None, None, 0, None, None) == L.OK
    assert lib.bigclam_recommend(ctx, good.ctypes.data, 2, 0, vo.ctypes.data, x.ctypes.data, None) == L.EINVAL
    assert b"m = 0" in lib.bigclam_last_error(ctx)
    assert lib.bigclam_recommend(ctx, bad.ctypes.data, 2, 3, vo.ctypes.data, np.zeros(6).ctypes.data, None) == L.EINVAL
    assert lib.bigclam_recommend(ctx, good.ctypes.data, 2, 3, None, np.zeros(6).ctypes.data, None) == L.EINVAL
    assert lib.bigclam_recommend(ctx, None, 2, 3, vo.ctypes.data, np.zeros(6).ctypes.data, None) == L.EINVAL   # NULL = all n
    assert lib.bigclam_recommend(ctx, good.ctypes.data, -1, 3, vo.ctypes.data, np.zeros(6).ctypes.data, None) == L.EINVAL
    with pytest.raises(ValueError):
        b.edge_probability([0, 1], [0])
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    b.close()


def test_multi_gpu_handle_matches_one_context():
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    rp, col = _graphs()["keep"]
    n, K = len(rp) - 1, 37
    F0 = _F0(n, K, seed=41)
    one = _solver(rp, col, K, F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    u, v = _pairs(n, seed=41, count=500)
    for it in range(2):
        x1, p1 = one.edge_probability(u, v)
        x2, p2 = two.edge_probability(u, v)
        assert np.array_equal(_bits(x1), _bits(x2)) and np.array_equal(_bits(p1), _bits(p2)), it
        r1, r2 = one.recommend(None, 5), two.recommend(None, 5)
        assert np.array_equal(r1[0], r2[0]) and np.array_equal(_bits(r1[1]), _bits(r2[1])), it
        if it == 0:                                                 # one step: the same rows on both (sumF may differ in its last bits)
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    lib = _lib()
    bad = np.array([0, n], dtype=np.int32)
    assert lib.bigclam_multi_pair_affinity(two._multi, bad.ctypes.data, bad.ctypes.data, 2, np.zeros(2).ctypes.data, None) == -1
    assert b"outside" in lib.bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


CPP = r"""
#include <cstdio>
#include <vector>
#include "bigclam_b200.hpp"
template <class T> static std::vector<T> rd(FILE *f, size_t n) { std::vector<T> v(n); if (fread(v.data(), sizeof(T), n, f) != n) throw 1; return v; }
int main(int, char **argv) {
    FILE *f = fopen(argv[1], "rb");
    int64_t hd[5];                                   // n, nnz, K, pairs, nodes
    if (fread(hd, 8, 5, f) != 5) return 2;
    auto rp = rd<int64_t>(f, hd[0] + 1);
    auto col = rd<int32_t>(f, hd[1]);
    auto F = rd<double>(f, hd[0] * hd[2]);
    auto u = rd<int32_t>(f, hd[3]), v = rd<int32_t>(f, hd[3]);
    auto q = rd<int32_t>(f, hd[4]);
    fclose(f);
    bigclam::BigClam b(1, 0, true);
    b.set_graph(hd[0], rp.data(), col.data()).set_K((int)hd[2]).set_F(F);
    std::vector<double> x, p, rx, ax;
    std::vector<int32_t> rv, av;
    b.edge_probability(u, v, x, p);
    b.recommend(q, 4, rv, rx);
    b.recommend({}, 4, av, ax);
    FILE *o = fopen(argv[2], "wb");
    fwrite(x.data(), 8, x.size(), o); fwrite(p.data(), 8, p.size(), o);
    fwrite(rv.data(), 4, rv.size(), o); fwrite(rx.data(), 8, rx.size(), o);
    fwrite(av.data(), 4, av.size(), o); fwrite(ax.data(), 8, ax.size(), o);
    fclose(o);
    try { b.recommend(q, 0, rv, rx); } catch (const bigclam::Error &e) { std::printf("%d\n", e.code); }
    return 0;
}
"""


def test_cpp_mirror_agrees_with_python(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    src = tmp_path / "links.cpp"
    src.write_text(CPP)
    exe = str(tmp_path / "links")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"), str(src),
                        "-o", exe, "-L", libdir, f"-l:{libname}", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    rp, col = _graphs()["keep"]
    n, K = len(rp) - 1, 37
    F0 = _F0(n, K, seed=5)
    u, v = _pairs(n, seed=5, count=300)
    q = np.array([0, 3, n - 1, 5], dtype=np.int32)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, len(u), len(q)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes())
        f.write(u.astype(np.int32).tobytes() + v.astype(np.int32).tobytes() + q.tobytes())
    r = subprocess.run([exe, str(inp), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                 # m = 0: bigclam::Error with BIGCLAM_EINVAL
    raw = open(tmp_path / "out.bin", "rb").read()
    np_ = len(u)
    x = np.frombuffer(raw, np.float64, np_, 0)
    p = np.frombuffer(raw, np.float64, np_, 8 * np_)
    o = 16 * np_
    rv = np.frombuffer(raw, np.int32, 4 * len(q), o).reshape(-1, 4)
    rx = np.frombuffer(raw, np.float64, 4 * len(q), o + 16 * len(q)).reshape(-1, 4)
    o += 48 * len(q)
    av = np.frombuffer(raw, np.int32, 4 * n, o).reshape(-1, 4)
    ax = np.frombuffer(raw, np.float64, 4 * n, o + 16 * n).reshape(-1, 4)
    b = _solver(rp, col, K, F0)
    xp, pp = b.edge_probability(u, v)
    assert np.array_equal(_bits(x), _bits(xp)) and np.array_equal(_bits(p), _bits(pp))
    pv, px = b.recommend(q, 4)
    assert np.array_equal(rv, pv) and np.array_equal(_bits(rx), _bits(px))
    pv, px = b.recommend(None, 4)
    assert np.array_equal(av, pv) and np.array_equal(_bits(ax), _bits(px))
    b.close()
