"""Sparse rows above K = 1024: the wide variant of the step kernel (csrc/bigclam_sparse.cuh, bigclam_tile.cuh wide_step) —
no tiles, the K-sized per-warp vectors in a global scratch, per-node passes over the touched components only — against
the oracle, with F0 non-zeros above component 1024 so that the high component ids are exercised.  The script's default
sweep (Kset(1000, 9000, 100)) and bigclamv3-7.scala's K = 8385 live in this range."""
import ctypes as C

import numpy as np
import pytest

from conftest import random_graph
from test_gpu_parity import _check_step

pytestmark = pytest.mark.gpu


def _solver(rp, col, K, F0, sumF=None, **kw):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(record_accepted=True, sparse_rows=True, **kw)
    b.set_graph(rp, col).set_K(K).set_F(F0, sumF=sumF)
    return b


def _wide_F0(n, k, seed, per_row=10.0):
    """About `per_row` non-zeros per row spread over all k components, and every 4th row non-zero in component k - 1."""
    rng = np.random.default_rng(seed)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < per_row / k)
    F0[::4, k - 1] = 0.1 + rng.random(len(F0[::4]))
    assert (F0[:, 1024:] != 0).any()
    return F0


def _steps(oracle, b, rp, col, F0, sumF, k, nsteps, max_flips=2, where=""):
    P = oracle.make_params(k)
    F, s = F0, sumF
    for it in range(nsteps):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        _check_step(b, r, llh, max_flips=max_flips, where=f"{where} it{it}", inputs=(rp, col, F, s, P))
        F, s = b.F, b.sumF


@pytest.mark.parametrize("k", [1025, 1028, 2000, 4096, 8385, 9000, 16384])
def test_wide_single_step(oracle, k):
    n = 400
    rp, col = random_graph(n, 6, seed=k, hub=60)
    F0 = _wide_F0(n, k, seed=k)
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    assert np.array_equal(b.F, F0)                      # dense -> sparse -> dense round trip
    assert b.tile_stats()["n_tiles"] == 0
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k))
    _check_step(b, r, llh, where=f"wide k={k}", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    b.close()


def test_wide_full_rows_and_a_hub(oracle):
    """Every component non-zero (the entry buffer holds one row per chunk) and a 300-edge hub."""
    n, k = 400, 2048
    rp, col = random_graph(n, 8, seed=3, hub=300)
    rng = np.random.default_rng(3)
    F0 = rng.random((n, k)) * 0.01
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    _steps(oracle, b, rp, col, F0, sumF, k, 3, where="wide full rows")
    b.close()


def test_wide_split_hubs(oracle, monkeypatch):
    monkeypatch.setenv("BIGCLAM_SPARSE_HUB_DEG", "200")
    n, k = 4000, 3000
    rp, col = random_graph(n, 6, seed=17, hub=1500)
    F0 = _wide_F0(n, k, seed=17)
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    assert b.tile_stats()["n_split_hubs"] > 0
    _steps(oracle, b, rp, col, F0, sumF, k, 3, where="wide hubs")
    b.close()


def test_wide_uset_mask_and_loglikelihood(oracle):
    n, k = 500, 2000
    rp, col = random_graph(n, 5, seed=11)
    F0 = _wide_F0(n, k, seed=11)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = _solver(rp, col, k, F0, sumF)
    assert abs(b.loglikelihood() - oracle.llh(rp, col, F0, sumF, P)) <= 1e-10 * abs(b.loglikelihood())
    mask = (np.random.default_rng(11).random(n) < 0.5).astype(np.uint8)
    llh = b.backtrackingLineSearchs(np.nonzero(mask)[0])
    r = oracle.step(rp, col, F0, sumF, P, node_mask=mask)
    _check_step(b, r, llh, where="wide uset", inputs=(rp, col, F0, sumF, P))
    assert np.array_equal(b.F[mask == 0], F0[mask == 0])
    b.close()


@pytest.mark.parametrize("variant", [2, 3, 4])
def test_wide_run_loop(oracle, variant):
    n, k = 800, 1500
    rp, col = random_graph(n, 6, seed=5)
    F0 = _wide_F0(n, k, seed=5)
    sumF = oracle.colsum(F0)
    b = _solver(rp, col, k, F0, sumF)
    llh = b._run(variant, 1e-4, 24)
    Fo, so, llh_o, calls_o, _ = oracle.run(rp, col, F0, sumF, oracle.make_params(k), variant=variant, rel_tol=1e-4, max_outer=24)
    assert b.last_calls == calls_o
    assert abs(llh - llh_o) <= 1e-9 * abs(llh_o)
    assert np.abs(b.F - Fo).max() <= 1e-7 * max(np.abs(Fo).max(), 1e-300)
    b.close()


def test_wide_reruns_are_bit_identical(oracle):
    n, k = 1000, 5000
    rp, col = random_graph(n, 7, seed=17, hub=300)
    F0 = _wide_F0(n, k, seed=17)
    sumF = oracle.colsum(F0)
    out = []
    for _ in range(2):
        b = _solver(rp, col, k, F0, sumF)
        llh = b._run(4, 0.0, 7)
        out.append((llh, b.last_trace.tobytes(), b.F.tobytes(), b.sumF.tobytes()))
        b.close()
    assert out[0] == out[1]


def test_wide_csr_entry_points_and_extraction(oracle):
    """K = 9000: set_F_csr / get_F_csr round trip, one step, and communities.extract against a NumPy restatement of
    Bigclamv2.scala:223-230."""
    import scipy.sparse as sps
    from bigclam_apachespark_b200 import BigClam
    from bigclam_apachespark_b200.communities import delta_threshold, extract
    n, k = 600, 9000
    rp, col = random_graph(n, 6, seed=8)
    F0 = _wide_F0(n, k, seed=8)
    b = BigClam(record_accepted=True, sparse_rows=True)
    b.set_graph(rp, col).set_K(k)
    b.set_F(sps.csr_matrix(F0))
    assert np.array_equal(b.F, F0)
    assert np.allclose(b.sumF, F0.sum(axis=0), rtol=1e-13)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, oracle.colsum(F0), oracle.make_params(k))
    _check_step(b, r, llh, where="wide csr", inputs=(rp, col, F0, oracle.colsum(F0), oracle.make_params(k)))
    ip, ix, vl = b.F_csr()
    F1 = b.F
    assert ip[-1] == (F1 != 0).sum()
    G = np.zeros_like(F1)
    for u in range(n):
        G[u, ix[ip[u]:ip[u + 1]]] = vl[ip[u]:ip[u + 1]]
    assert np.array_equal(G, F1)
    delta = delta_threshold(n, n)
    comms, cids, member = extract(b, delta)
    fmax = F1.max(axis=1, keepdims=True)
    expect = np.where(fmax < delta, F1 == fmax, F1 >= delta)     # :225-228
    assert np.array_equal(member.astype(bool), expect)
    for c, idx in zip(cids, comms):
        assert np.array_equal(idx, np.flatnonzero(expect[:, c]))
    b.close()


def test_wide_pool_exhaustion_is_reported(monkeypatch):
    from bigclam_apachespark_b200 import BigClam, _lib
    monkeypatch.setenv("BIGCLAM_SPARSE_POOL_WORDS", "2000")
    n, k = 600, 2000
    rp, col = random_graph(n, 6, seed=2)
    b = BigClam(sparse_rows=True)
    b.set_graph(rp, col).set_K(k)
    with pytest.raises(_lib.BigclamError):
        b.set_F(_wide_F0(n, k, seed=2))                  # 600 rows of ~10 entries do not fit 2000 words
    b.close()


def test_driver_picks_sparse_rows_above_1024(oracle):
    from bigclam_apachespark_b200 import BigClam
    n, k = 400, 2000
    rp, col = random_graph(n, 6, seed=21, hub=40)
    F0 = _wide_F0(n, k, seed=21)
    sumF = oracle.colsum(F0)
    b = BigClam(record_accepted=True, sparse_rows=False)
    b.set_graph(rp, col).set_K(k).set_F(F0, sumF=sumF)       # (a dense context would be refused above k = 1024)
    llh = b.backtrackingLineSearchs()
    r = oracle.step(rp, col, F0, sumF, oracle.make_params(k))
    _check_step(b, r, llh, where="driver k=2000", inputs=(rp, col, F0, sumF, oracle.make_params(k)))
    b.close()


def _lib_init_F0(rp, col, K, ranked, pad_seed=1234):
    """initNeighborComF(K) by the library's host implementation (the random padding columns included)."""
    from bigclam_apachespark_b200 import _lib
    n = len(rp) - 1
    ranked = np.ascontiguousarray(ranked, dtype=np.int32)
    F0 = np.empty((n, K), dtype=np.float64)
    rc = _lib.load().bigclam_init_neighbor_com_F(n, rp.ctypes.data, col.ctypes.data, int(K), ranked.ctypes.data, len(ranked), 0,
                                                 C.c_uint64(pad_seed), F0.ctypes.data)
    assert rc == _lib.OK
    return F0


def _oracle_sweep(oracle, rp, col, ks, max_outer):
    """The script's sweep (:244-266) driven by the oracle: the same F0 per K, SGDFindC, the same stop rule."""
    from oracle import numpy_twin as T
    ranked, _ = T.conductance_local_min(rp, col)
    old, kfor, hist = 0.0, 0, []
    for K in ks:
        F0 = _lib_init_F0(np.ascontiguousarray(rp, dtype=np.int64), np.ascontiguousarray(col, dtype=np.int32), K, ranked)
        llh = oracle.run(rp, col, F0, oracle.colsum(F0), oracle.make_params(K), variant=4, rel_tol=1e-4, max_outer=max_outer)[2]
        hist.append((K, llh))
        with np.errstate(divide="ignore", invalid="ignore"):
            gain = 1.0 - np.float64(llh) / np.float64(old)
        if gain < 0.001:
            kfor = K
            break
        old = llh
    return kfor, hist


def test_driver_sweep_crosses_1024(oracle):
    from bigclam_apachespark_b200 import BigClam
    rp, col = random_graph(400, 6, seed=3, hub=30)
    b = BigClam(minCom=1000, maxCom=4000, divCom=4)      # sparse_rows=False: the contexts above 1024 are sparse anyway
    b.set_graph(rp, col)
    assert b.Kset() == [1000, 1414, 1999, 2827, 3997, 4000]
    KforC, hist = b.sweep_K(max_outer=8)
    k_o, hist_o = _oracle_sweep(oracle, rp, col, b.Kset(), 8)
    assert KforC == k_o and [k for k, _ in hist] == [k for k, _ in hist_o], (KforC, k_o, hist, hist_o)
    for (_, l1), (_, l2) in zip(hist, hist_o):
        assert abs(l1 - l2) <= 1e-8 * abs(l2), (l1, l2)
    b.close()


def test_cpp_mirror_sweep_crosses_1024(oracle, tmp_path):
    import subprocess
    from bigclam_apachespark_b200.driver import Kset
    from test_c_host import _case, _write_edgelist
    from test_gpu_zy_c_host import _mirror
    rp, col = _case(tmp_path, n=400, deg=6, k=4, seed=95)[:2]
    edges = str(tmp_path / "sweep.txt")
    _write_edgelist(edges, rp, col)
    lo, hi, div, cap = 1000, 2000, 2, 5
    ks = Kset(lo, hi, div)
    assert ks[0] <= 1024 < ks[-1]
    r = subprocess.run([_mirror(tmp_path), "sweep", edges, str(lo), str(hi), str(div), str(cap)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.strip().splitlines()
    hist = [(int(l.split()[0]), float(l.split()[2])) for l in lines if " LLH: " in l]
    kfor = int(lines[-1].split()[1])
    k_o, hist_o = _oracle_sweep(oracle, rp, col, ks, cap)
    assert kfor == k_o and [k for k, _ in hist] == [k for k, _ in hist_o], (kfor, k_o, hist, hist_o)
    for (_, l1), (_, l2) in zip(hist, hist_o):
        assert abs(l1 - l2) <= 1e-8 * abs(l2), (l1, l2)


def test_wide_multi_gpu_matches_oracle_and_replicas_agree(oracle, monkeypatch):
    from bigclam_apachespark_b200 import BigClam, _lib
    world = 2
    if int(_lib.load().bigclam_device_count()) < world:
        pytest.skip(f"needs {world} GPUs")
    monkeypatch.setenv("BIGCLAM_SPARSE_HUB_DEG", "100")
    n, k = 240, 1100
    rp, col = random_graph(n, 5, seed=9, hub=150)
    F0 = _wide_F0(n, k, seed=3)
    sumF = oracle.colsum(F0)
    P = oracle.make_params(k)
    b = BigClam(record_accepted=False, numGPUs=world)
    b.set_graph(rp, col).set_K(k).set_F(F0, sumF=sumF)
    assert abs(b.loglikelihood() - oracle.llh(rp, col, F0, sumF, P)) <= 1e-10 * abs(oracle.llh(rp, col, F0, sumF, P))
    F, s = F0, sumF
    for it in range(3):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        assert abs(llh - r.llh) <= 1e-10 * abs(r.llh)
        assert b.last_n_updated == r.n_updated
        reps = [b.replica_F(q) for q in range(world)]
        for q in range(1, world):
            assert np.array_equal(reps[0], reps[q]), f"replica {q} differs from replica 0 after step {it}"
            assert np.array_equal(b.replica_sumF(0), b.replica_sumF(q))
        assert np.abs(reps[0] - r.F).max() <= 1e-9 * max(np.abs(r.F).max(), 1e-300)
        assert np.allclose(b.sumF, r.sumF, rtol=1e-11, atol=1e-9)
        F, s = r.F, r.sumF
    b.close()
