"""Cover scores on the GPU (bigclam_cover_scores and its multi-GPU twin, BigClam.score_against, the C++ mirror):
F1 and matches bit for bit and the conditional entropies and NMIs to 1e-12 against the NumPy twin
(tests/cover_scores_twin.py) for sparse and dense rows at every kind of K, both zero-row modes and several deltas; the
same outputs from both layouts and for any member order or repeats of the truth; the self-score and a planted model at
exactly 1.0; two fits of facebook scored against each other both ways; com-amazon against its ground truth and
communities.avg_f1; the state a query must leave untouched; and the argument checks."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO, random_graph
from cover_scores_twin import KEYS, cover_scores as twin_scores
from test_gpu_extract import _F0

pytestmark = pytest.mark.gpu
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"
EXACT = ("f1_detected", "match_detected", "f1_truth", "match_truth")
SCALARS = ("avg_f1", "nmi_lfk", "nmi_max")


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def _solver(rp, col, K, F0, sparse=True, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse, record_accepted=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0)
    return b


def _truth(n, q, seed):
    """q random truth communities of assorted sizes, unsorted, some with repeats; one empty, one of all n nodes and
    one of n - 1 nodes."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(q):
        s = int(rng.integers(1, max(2, n // 4)))
        c = rng.choice(n, size=s, replace=False)
        if t % 3 == 0:
            c = np.concatenate([c, c[: s // 2 + 1]])
        out.append(rng.permutation(c).astype(np.int32))
    out[1] = np.zeros(0, dtype=np.int32)
    out[2] = rng.permutation(n).astype(np.int32)
    out[3] = np.arange(1, n, dtype=np.int32)
    return out


def _twin(b, truth, delta, everywhere=True):
    return twin_scores(*b.F_csr(), b.K, delta, truth, zero_rows=everywhere)


def _bits(x):
    return np.asarray(x).view(np.uint8)


def _same(g, h):
    """Every output, arrays and scalars, bit for bit (NaN included)."""
    for key in KEYS:
        x, y = np.asarray(g[key]), np.asarray(h[key])
        if x.dtype != y.dtype or x.shape != y.shape or not np.array_equal(_bits(x), _bits(y)):
            return False
    return all(np.float64(g[k]).view(np.int64) == np.float64(h[k]).view(np.int64) for k in SCALARS)


def _close(g, t):
    """F1 and matches bit for bit, hcond and the NMIs to 1e-12, against the twin t; no admissibility margin below 1e-9."""
    assert t["margin"] >= 1e-9, t["margin"]
    for key in EXACT:
        x, y = np.asarray(g[key]), np.asarray(t[key])
        assert x.dtype == y.dtype and np.array_equal(_bits(x), _bits(y)), key
    for key in ("hcond_detected", "hcond_truth"):
        x, y = np.asarray(g[key]), np.asarray(t[key])
        assert np.array_equal(np.isnan(x), np.isnan(y)), key
        assert np.allclose(x, y, rtol=1e-12, atol=1e-12, equal_nan=True), (key, np.nanmax(np.abs(x - y)))
    assert g["avg_f1"] == pytest.approx(t["avg_f1"], rel=1e-15, abs=0)             # the same folds of the same bits
    for key in ("nmi_lfk", "nmi_max"):
        assert g[key] == pytest.approx(t[key], rel=1e-12, abs=1e-12, nan_ok=True), key


KS = [1, 37, 200, 1024, 1025, 9000]
DELTA = 0.5


@pytest.mark.parametrize("K", KS)
def test_scores_match_twin(K):
    n = 100 if EMU else (600 if K == 9000 else 300)
    rp, col = random_graph(n, 6, seed=K)
    F0 = _F0(n, K, seed=K, delta=DELTA, per_row=6.0 if K < 1000 else 40.0)
    truth = _truth(n, 12 if EMU else 40, seed=K)
    layouts = [True, False] if K <= 1024 else [True]
    got = {}
    for sparse in layouts:
        b = _solver(rp, col, K, F0, sparse=sparse)
        for delta in (DELTA, 0.1, float("inf")):
            for everywhere in (True, False):
                g = b.score_against(truth, delta, zero_rows_everywhere=everywhere)
                _close(g, _twin(b, truth, delta, everywhere))
                got[(sparse, delta, everywhere)] = g
        b.close()
    if len(layouts) == 2:                                                           # the same F in both layouts: the same outputs
        for key in [k for k in got if k[0]]:
            assert _same(got[key], got[(False,) + key[1:]]), key


@pytest.mark.parametrize("sparse", [True, False])
def test_zero_row_modes(sparse):
    """Many zero rows: in every community they add z_t to every a and z to every x; in none they are simply absent."""
    n, K = 80, 16
    rp, col = random_graph(n, 4, seed=2)
    F0 = _F0(n, K, seed=2, delta=DELTA)
    F0[10:30] = 0.0
    truth = _truth(n, 15, seed=2) + [np.arange(10, 30, dtype=np.int32), np.arange(5, 15, dtype=np.int32)]
    b = _solver(rp, col, K, F0, sparse=sparse)
    for everywhere in (True, False):
        g = b.score_against(truth, DELTA, everywhere)
        _close(g, _twin(b, truth, DELTA, everywhere))
    # with the zero rows nowhere, the community of exactly the zero rows matches nothing
    assert b.score_against(truth, DELTA, False)["match_truth"][-2] == -1
    b.close()


def test_truth_order_and_repeats():
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=8)
    F0 = _F0(n, K, seed=8, delta=DELTA)
    truth = [np.unique(t) for t in _truth(n, 30, seed=8)]
    rng = np.random.default_rng(8)
    messy = [np.concatenate([rng.permutation(t), t[::2], t[:1]]) if len(t) else t for t in truth]
    b = _solver(rp, col, K, F0)
    for everywhere in (True, False):
        assert _same(b.score_against(truth, DELTA, everywhere), b.score_against(messy, DELTA, everywhere))
    b.close()


def _self_one(b, delta, everywhere):
    from bigclam_apachespark_b200 import communities as Cm
    det, cids = Cm.group(*b.extract_communities(delta), zero_rows_everywhere=everywhere)
    g = b.score_against(det, delta, everywhere)
    assert (g["avg_f1"], g["nmi_lfk"], g["nmi_max"]) == (1.0, 1.0, 1.0), (delta, everywhere)
    # each community matches the first one with the same member set (communities can coincide, e.g. on the zero rows)
    first = {}
    for i, c in enumerate(det):
        first.setdefault(c.tobytes(), i)
    want = np.array([first[c.tobytes()] for c in det], dtype=np.int32)
    assert (g["f1_truth"] == 1.0).all() and (g["f1_detected"][cids] == 1.0).all()
    assert np.array_equal(g["match_truth"], cids[want]) and np.array_equal(g["match_detected"][cids], want)


def test_self_score_is_one():
    from bigclam_apachespark_b200 import graphs as G
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=4)
    b = _solver(rp, col, K, _F0(n, K, seed=4, delta=DELTA))
    for delta in (DELTA, 0.1, float("inf")):
        for everywhere in (True, False):
            _self_one(b, delta, everywhere)
    b.close()
    if EMU:
        return
    rp, col, _ = G.load_npz_graph("facebook_combined")
    n, K = len(rp) - 1, 10
    b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234, density=0.3))
    for _ in range(5):
        b.backtrackingLineSearchs()
    from bigclam_apachespark_b200 import communities as Cm
    for delta in (Cm.delta_threshold(n, int((np.diff(rp) > 0).sum())), 0.5):
        for everywhere in (True, False):
            _self_one(b, delta, everywhere)
    b.close()


def test_planted_model_scores_one():
    """A planted model (every node in one community, 30 % in a second, F = 0.15): extraction recovers the planted
    communities exactly at either side of F, so the scores against them are exactly 1."""
    from bigclam_apachespark_b200 import BigClam
    sys.path.insert(0, os.path.join(REPO, "scripts"))
    from bench_sample import _planted
    n, K = (300, 12) if EMU else (20_000, 200)
    ip, ix, vl = _planted(n, K, 0.15, 0.3, seed=3)
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(ip))
    o = np.argsort(ix, kind="stable")
    truth = np.split(rows[o], np.cumsum(np.bincount(ix, minlength=K))[:-1])
    b = BigClam(sparse_rows=True)
    b.set_graph(np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)).set_K(K).set_F_csr(ip, ix, vl)
    for delta in (0.1, 0.5):
        g = b.score_against(truth, delta)
        assert (g["avg_f1"], g["nmi_lfk"], g["nmi_max"]) == (1.0, 1.0, 1.0), delta
        assert np.array_equal(g["match_detected"], np.arange(K, dtype=np.int32))
    b.close()


def test_two_fits_against_each_other():
    """Fits A and B of facebook at different K: A scored against B's cover and B against A's give the same pairs from
    both sides, so each direction's detected-side outputs are the other's truth-side outputs, ids mapped through
    group()'s community ids, and the NMIs are equal."""
    from bigclam_apachespark_b200 import communities as Cm, graphs as G
    if EMU:
        rp, col = random_graph(120, 6, seed=9)
        fits = [(8, 0.3), (13, 0.2)]
    else:
        rp, col, _ = G.load_npz_graph("facebook_combined")
        fits = [(10, 0.3), (25, 0.2)]
    n = len(rp) - 1
    delta = Cm.delta_threshold(n, int((np.diff(rp) > 0).sum()))
    bs = []
    for K, dens in fits:
        b = _solver(rp, col, K, G.synthetic_F0(n, K, seed=1234 + K, density=dens))
        for _ in range(3):
            b.backtrackingLineSearchs()
        bs.append(b)
    for everywhere in (True, False):
        (ca, ia), (cb, ib) = (Cm.group(*b.extract_communities(delta), zero_rows_everywhere=everywhere) for b in bs)
        ab = bs[0].score_against(cb, delta, everywhere)                                # A detected, B as truth
        ba = bs[1].score_against(ca, delta, everywhere)
        for (d, ids_d), (t, ids_t) in (((ab, ia), (ba, ib)), ((ba, ib), (ab, ia))):
            m = d["match_detected"][ids_d]
            assert np.array_equal(_bits(d["f1_detected"][ids_d]), _bits(t["f1_truth"]))
            assert np.array_equal(np.where(m >= 0, ids_t[np.maximum(m, 0)], -1), t["match_truth"])
            assert np.array_equal(_bits(d["hcond_detected"][ids_d]), _bits(t["hcond_truth"]))
        for key in SCALARS:
            assert np.float64(ab[key]).view(np.int64) == np.float64(ba[key]).view(np.int64), key
        _close(ab, _twin(bs[0], cb, delta, everywhere))
    for b in bs:
        b.close()


@pytest.mark.parametrize("everywhere", [True, False])
def test_amazon_fit_against_ground_truth(everywhere):
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
    truth = Cm.load_ground_truth()
    g = b.score_against(truth, delta, everywhere)
    det, _ = Cm.group(*b.extract_communities(delta), zero_rows_everywhere=everywhere)
    assert g["avg_f1"] == pytest.approx(Cm.avg_f1(det, truth, n), rel=1e-12, abs=0)
    _close(g, _twin(b, truth, delta, everywhere))
    b.close()


def test_state_untouched_by_scores():
    rp, col = random_graph(120 if EMU else 600, 6, seed=31)
    n, K = len(rp) - 1, 24
    F0 = _F0(n, K, seed=31, delta=DELTA)
    truth = _truth(n, 20, seed=31)
    a = _solver(rp, col, K, F0, time_kernels=True)
    c = _solver(rp, col, K, F0, time_kernels=True)
    for it in range(4):
        la, lc = a.backtrackingLineSearchs(), c.backtrackingLineSearchs()
        assert np.float64(la).view(np.int64) == np.float64(lc).view(np.int64), it
        assert a.kernel_time()[1:] == c.kernel_time()[1:], it                       # from the 2nd step on, both commit the speculation
        if it > 0:
            assert a.kernel_time()[1] == 1
        a.score_against(truth, DELTA)
        a.score_against(truth, float("inf"), zero_rows_everywhere=False)
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
    ptr = np.array([0, 3, 3, 5], dtype=np.int64)
    mem = np.array([4, 1, 9, 0, 2], dtype=np.int32)
    q = len(ptr) - 1
    f1d, hcd = np.full(K, -7.0), np.full(K, -7.0)
    md = np.full(K, -7, dtype=np.int32)
    f1t, hct = np.full(q, -7.0), np.full(q, -7.0)
    mt = np.full(q, -7, dtype=np.int32)
    sc = np.full(3, -7.0)
    outs = [f1d, md, f1t, mt, hcd, hct, sc]

    def call(delta=DELTA, zr=1, qq=q, p=ptr, m=mem, o=None):
        o = [x.ctypes.data for x in outs] if o is None else o
        return lib.bigclam_cover_scores(ctx, delta, zr, qq, None if p is None else p.ctypes.data,
                                        None if m is None else m.ctypes.data, *o)

    def rejected(what, **kw):
        assert call(**kw) == L.EINVAL, kw
        assert what in lib.bigclam_last_error(ctx), (kw, lib.bigclam_last_error(ctx))

    for delta in (float("nan"), 0.0, -0.0, -1e-9, -float("inf")):
        rejected(b"delta", delta=delta)
    for zr in (-1, 2, 255):
        rejected(b"zero_rows", zr=zr)
    rejected(b"q = -1", qq=-1)
    rejected(b"q = ", qq=1 << 31)
    rejected(b"truth_ptr[0]", p=np.array([1, 3, 3, 5], dtype=np.int64))
    rejected(b"decreases at truth community 1", p=np.array([0, 3, 2, 5], dtype=np.int64))
    rejected(b"truth community 2 has id 100", m=np.array([4, 1, 9, 0, 100], dtype=np.int32))
    rejected(b"truth community 0 has id -1", m=np.array([4, -1, 9, 0, 2], dtype=np.int32))
    rejected(b"NULL", p=None)
    rejected(b"NULL", m=None)
    for i in (0, 1, 2, 3, 6):
        o = [x.ctypes.data for x in outs]
        o[i] = None
        rejected(b"NULL", o=o)
    assert all((x == -7).all() for x in outs)
    with pytest.raises(L.BigclamError):
        b.score_against([[0, 1]], 0.0)
    with pytest.raises(L.BigclamError):
        b.score_against([[0, 1], [n]], DELTA)
    # nothing ran: the next step still commits the speculative one
    b.backtrackingLineSearchs()
    assert b.kernel_time()[1] == 1
    o = [x.ctypes.data for x in outs]
    o[4] = o[5] = None                                                              # hcond_* are optional
    assert call(o=o) == L.OK
    g = b.score_against([mem[0:3], [], mem[3:5]], DELTA)
    assert np.array_equal(f1d, g["f1_detected"]) and np.array_equal(md, g["match_detected"])
    assert np.array_equal(f1t, g["f1_truth"]) and np.array_equal(mt, g["match_truth"])
    assert np.array_equal(_bits(sc), _bits(np.array([g[k] for k in SCALARS])))
    assert (hcd == -7.0).all() and (hct == -7.0).all()
    # no truth at all: q = 0, nothing matched, the NMIs undefined
    g = b.score_against([], DELTA)
    assert g["avg_f1"] == 0.0 and np.isnan(g["nmi_lfk"]) and np.isnan(g["nmi_max"])
    assert (g["match_detected"] == -1).all() and len(g["f1_truth"]) == 0
    b.close()
    # a negative entry (set_F can leave one): BIGCLAM_EUNSUPPORTED naming the smallest such row
    F1 = F0.copy()
    F1[37, 2] = -1e-3
    F1[71, 0] = -2.0
    for sparse in (True, False):
        b = _solver(rp, col, K, F1, sparse=sparse)
        assert lib.bigclam_cover_scores(b._ctx, DELTA, 0, q, ptr.ctypes.data, mem.ctypes.data, *[x.ctypes.data for x in outs]) == L.EUNSUPPORTED
        assert b"row 37 " in lib.bigclam_last_error(b._ctx)
        b.close()


def test_multi_gpu_handle_matches_one_context():
    from bigclam_apachespark_b200 import BigClam
    if int(_lib().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    n, K = (100 if EMU else 400), 37
    rp, col = random_graph(n, 5, seed=41)
    F0 = _F0(n, K, seed=41, delta=DELTA)
    truth = _truth(n, 20, seed=41)
    one = _solver(rp, col, K, F0)
    two = BigClam(numGPUs=2)
    two.set_graph(rp, col).set_K(K).set_F(F0)
    for it in range(2):
        for delta in (DELTA, float("inf")):
            for everywhere in (True, False):
                assert _same(one.score_against(truth, delta, everywhere), two.score_against(truth, delta, everywhere)), (it, delta)
        if it == 0:                                                                 # one step: the same rows on both
            one.backtrackingLineSearchs()
            two.backtrackingLineSearchs()
    _close(two.score_against(truth, DELTA), _twin(one, truth, DELTA))
    z = np.zeros(max(K, 3))
    zi = np.zeros(K, dtype=np.int32)
    p = np.zeros(1, dtype=np.int64)
    assert _lib().bigclam_multi_cover_scores(two._multi, 0.0, 1, 0, p.ctypes.data, None, z.ctypes.data, zi.ctypes.data,
                                             None, None, None, None, z.ctypes.data) == -1
    assert b"delta" in _lib().bigclam_multi_last_error(two._multi)
    one.close()
    two.close()


def _build_cpp(tmp_path):
    from test_c_host import product_lib
    libdir, libname = product_lib()
    exe = str(tmp_path / "cover_scores")
    cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else shutil.which("g++")
    r = subprocess.run([cxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"),
                        os.path.join(REPO, "tests", "cpp_host", "cover_scores.cpp"), "-o", exe, "-L", libdir, f"-l:{libname}",
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
    truth = _truth(n, 15, seed=12)
    deltas = [DELTA, 0.1, float("inf")]
    tptr = np.zeros(len(truth) + 1, dtype=np.int64)
    np.cumsum([len(t) for t in truth], out=tptr[1:])
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([n, len(col), K, len(deltas), len(truth)], dtype=np.int64).tobytes())
        f.write(rp.astype(np.int64).tobytes() + col.astype(np.int32).tobytes() + F0.tobytes() + np.array(deltas).tobytes())
        f.write(tptr.tobytes() + np.concatenate(truth).astype(np.int32).tobytes())
    out = tmp_path / "out.bin"
    r = subprocess.run([exe, str(inp), str(out), str(world)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "-1"                                                 # delta = 0: bigclam::Error with BIGCLAM_EINVAL
    raw = open(out, "rb").read()
    q = len(truth)
    per = 8 * 3 + 8 * K * 2 + 4 * K + 8 * q * 2 + 4 * q
    assert len(raw) == len(deltas) * 2 * per
    b = _solver(rp, col, K, F0)
    o = 0

    def take(dtype, count):
        nonlocal o
        x = np.frombuffer(raw, dtype, count, o)
        o += x.nbytes
        return x

    for delta in deltas:
        for everywhere in (True, False):
            s = take(np.float64, 3)
            g = dict(zip(SCALARS, s.tolist()))
            g["f1_detected"], g["match_detected"], g["hcond_detected"] = take(np.float64, K), take(np.int32, K), take(np.float64, K)
            g["f1_truth"], g["match_truth"], g["hcond_truth"] = take(np.float64, q), take(np.int32, q), take(np.float64, q)
            assert _same(g, b.score_against(truth, delta, everywhere)), (delta, everywhere)
    b.close()
