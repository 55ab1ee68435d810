"""initNeighborComF's F0 built on the GPU straight into the context (bigclam_init_F / bigclam_multi_init_F, BigClam.init_F)
against the host route it replaces: bigclam_init_neighbor_com_F (csrc/initf.cpp) + bigclam_set_F.  The F rows and sumF
bits are compared exactly, and so is everything that runs after them on sparse and wide rows (the dense-row engine is
reproducible to rounding only, run to run)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import random_graph

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.environ.get("BIGCLAM_HOSTEMU") == "1"
PAD_SEEDS = [0, 1, 1234, 2**64 - 1]


def _lib():
    from bigclam_apachespark_b200 import _lib as L
    return L.load()


def host_F0(rp, col, K, seeds, include_self=False, pad_seed=1234):
    n = len(rp) - 1
    seeds = np.ascontiguousarray(seeds, dtype=np.int32)
    F0 = np.empty((n, K), dtype=np.float64)
    rc = _lib().bigclam_init_neighbor_com_F(n, rp.ctypes.data, col.ctypes.data, K, seeds.ctypes.data, len(seeds),
                                            1 if include_self else 0, C.c_uint64(pad_seed), F0.ctypes.data)
    assert rc == 0
    return F0


def csr_of(F0):
    rows, cols = np.nonzero(F0)
    indptr = np.zeros(F0.shape[0] + 1, dtype=np.int64)
    np.add.at(indptr, rows + 1, 1)
    return np.cumsum(indptr), cols.astype(np.int32), F0[rows, cols]


def solver(rp, col, K, kind, seeds=None):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=(kind != "dense"))
    b.set_graph(np.ascontiguousarray(rp, dtype=np.int64), np.ascontiguousarray(col, dtype=np.int32)).set_K(K)
    if seeds is not None:
        b.Sbc = np.ascontiguousarray(seeds, dtype=np.int32)
    return b


def assert_same_state(a, b):
    for x, y in zip(a.F_csr(), b.F_csr()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.sumF, b.sumF)


def check_against_host(rp, col, K, kind, seeds, include_self=False, pad_seed=1234):
    """init_F == F_csr of the host F0 and sumF of a context loaded with set_F(host F0)."""
    F0 = host_F0(rp, col, K, seeds, include_self, pad_seed)
    g = solver(rp, col, K, kind, seeds).init_F(K, include_self=include_self, pad_seed=pad_seed)
    for x, y in zip(g.F_csr(), csr_of(F0)):
        assert np.array_equal(x, y)
    h = solver(rp, col, K, kind).set_F(F0)
    assert np.array_equal(g.sumF, h.sumF)
    g.close()
    h.close()


def seeds_of(rp, col):
    from bigclam_apachespark_b200 import BigClam
    b = BigClam().set_graph(rp, col)
    return b.conductanceLocalMin(on_gpu=False)


def kinds(K):
    return ["sparse", "dense"] if K <= 1024 else ["wide"]


HUB = random_graph(300, 6, seed=11, hub=60)


@pytest.mark.parametrize("K", [1, 37, 200, 1024, 1025, 9000])
@pytest.mark.parametrize("include_self", [False, True])
def test_random_graph_same_F0(K, include_self):
    rp, col = HUB
    seeds = seeds_of(rp, col)
    for kind in kinds(K):
        for pad_seed in PAD_SEEDS:
            check_against_host(rp, col, K, kind, seeds, include_self, pad_seed)


@pytest.mark.parametrize("name,K", [("facebook_combined", 37), ("facebook_combined", 1025), ("facebook_combined", 9000),
                                    ("email-enron", 200), ("email-enron", 9000)])
def test_fixture_graph_same_F0(graphs, name, K):
    rp, col, _ = graphs.load_npz_graph(name)
    seeds = seeds_of(rp, col)
    for kind in kinds(K):
        check_against_host(rp, col, K, kind, seeds, include_self=(K == 37), pad_seed=1234)


def awkward_graph():
    """Unsorted lists, repeated entries, an asymmetric CSR, a self-loop and nodes without a list."""
    lists = [[5, 3, 3, 9], [], [0, 7, 0, 1], [2], [11, 4, 10, 4, 4], [], [6, 1], [3, 2, 8], [0], [], [5, 5], [1, 0]]
    rp = np.zeros(len(lists) + 1, dtype=np.int64)
    rp[1:] = np.cumsum([len(x) for x in lists])
    col = np.array([v for x in lists for v in x], dtype=np.int32)
    return rp, col


@pytest.mark.parametrize("K", [37, 1025])
@pytest.mark.parametrize("seeds", [[7, 2, 4, 0], [1, 5, 9, 4, 6], [4, 4, 10, 7, 7], [], list(range(12)) * 4],
                         ids=["unsorted", "empty_lists", "duplicates", "none", "more_than_K"])
def test_awkward_inputs(K, seeds):
    rp, col = awkward_graph()
    for kind in kinds(K):
        for include_self in (False, True):
            check_against_host(rp, col, K, kind, seeds, include_self, pad_seed=7)


def _downstream(rp, col, K, kind, seeds, steps):
    F0 = host_F0(rp, col, K, seeds)
    h = solver(rp, col, K, kind).set_F(F0)
    g = solver(rp, col, K, kind, seeds).init_F(K)
    assert_same_state(h, g)
    lh, lg = h.SGDFindC(max_outer=steps), g.SGDFindC(max_outer=steps)
    assert len(g.last_trace) > 1
    if kind == "dense":
        # the dense-row engine adds its partial sums with atomics, so two runs from one F0 agree to rounding only
        assert np.allclose(h.last_trace, g.last_trace, rtol=1e-12, atol=0) and abs(lh - lg) <= 1e-12 * abs(lh)
        assert np.allclose(h.F, g.F, rtol=1e-9, atol=1e-12)
    else:
        assert lh == lg and np.array_equal(h.last_trace, g.last_trace)
        assert_same_state(h, g)
    h.close()
    g.close()


def test_same_bits_downstream_tile_path(graphs):
    rp, col, _ = graphs.load_npz_graph("facebook_combined")
    _downstream(rp, col, 200, "sparse", seeds_of(rp, col), 4)


def test_same_bits_downstream_wide():
    rp, col = HUB
    _downstream(rp, col, 1025, "wide", seeds_of(rp, col), 4)


def test_same_bits_downstream_dense_rows():
    rp, col = HUB
    _downstream(rp, col, 37, "dense", seeds_of(rp, col), 6)


def _host_sweep(rp, col, ks, cap, seeds, sparse_rows):
    """The sweep of bigclam4-7.scala:244-266 driven through bigclam_init_neighbor_com_F + set_F + SGDFindC."""
    from bigclam_apachespark_b200 import BigClam
    b = BigClam(sparse_rows=sparse_rows).set_graph(rp, col)
    LLHKold, hist = 0.0, []
    for K in ks:
        b.set_F(host_F0(b.rowptr, b.col, K, seeds))
        LLHKnew = b.SGDFindC(max_outer=cap)
        hist.append((K, LLHKnew))
        with np.errstate(divide="ignore", invalid="ignore"):
            if 1.0 - np.float64(LLHKnew) / np.float64(LLHKold) < 0.001:
                b.close()
                return K, hist
        LLHKold = LLHKnew
    b.close()
    return 0, hist


# Sparse rows at every K of the sweeps below: the dense-row engine (K <= 1024 without sparse_rows) is reproducible to
# rounding only (see _downstream), sparse and wide rows bit for bit.
def test_driver_sweep_same_bits():
    from bigclam_apachespark_b200 import BigClam
    rp, col = random_graph(400, 6, seed=3, hub=30)
    b = BigClam(minCom=1000, maxCom=4000, divCom=4, sparse_rows=True).set_graph(rp, col)
    KforC, hist = b.sweep_K(max_outer=8)
    assert (KforC, hist) == _host_sweep(rp, col, b.Kset(), 8, b.Sbc, True)
    b.close()


def test_cpp_mirror_sweep_same_bits(tmp_path):
    from bigclam_apachespark_b200 import BigClam
    from bigclam_apachespark_b200.driver import Kset
    from test_c_host import _case, _write_edgelist
    from test_gpu_zy_c_host import _mirror
    rp, col = _case(tmp_path, n=400, deg=6, k=4, seed=95)[:2]
    edges = str(tmp_path / "sweep.txt")
    _write_edgelist(edges, rp, col)
    lo, hi, div, cap = 1100, 2000, 2, 5              # (the mirror's contexts above K = 1024 have sparse rows)
    r = subprocess.run([_mirror(tmp_path), "sweep", edges, str(lo), str(hi), str(div), str(cap)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.strip().splitlines()
    hist = [(int(l.split()[0]), float(l.split()[2])) for l in lines if " LLH: " in l]
    b = BigClam().load_edge_list(edges)
    seeds = b.conductanceLocalMin()
    assert (int(lines[-1].split()[1]), hist) == _host_sweep(b.rowptr, b.col, Kset(lo, hi, div), cap, seeds, True)
    b.close()


_AMAZON_CHILD = r"""
import json, resource, sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from bigclam_apachespark_b200 import BigClam, graphs as G
rp, col, _ = G.load_npz_graph("com-amazon")
K = 9000
b = BigClam(sparse_rows=True).set_graph(rp, col)
b.conductanceLocalMin()
b.set_K(K)
torch.cuda.init()
free0 = torch.cuda.mem_get_info(0)[0]
rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
b.init_F(K)
free1 = torch.cuda.mem_get_info(0)[0]
rss1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
indptr, indices, values = b.F_csr()
sumF = b.sumF
# the rows bigclam_set_F_csr gets from a host CSR built from the seeds' lists
S = np.sort(b.Sbc[:K])
rows = np.concatenate([col[rp[s]:rp[s + 1]] for s in S]).astype(np.int64)
cols = np.repeat(np.arange(len(S)), [rp[s + 1] - rp[s] for s in S])
key = np.unique(rows * K + cols)
r_ptr = np.zeros(len(rp), dtype=np.int64)
np.add.at(r_ptr, key // K + 1, 1)
r_ptr = np.cumsum(r_ptr)
r_idx = (key % K).astype(np.int32)
b.set_F_csr(r_ptr, r_idx, np.ones(len(key)))
same = bool(np.array_equal(indptr, r_ptr) and np.array_equal(indices, r_idx) and np.all(values == 1.0)
            and np.array_equal(sumF, b.sumF))
print(json.dumps({"device_bytes": int(free0 - free1), "rss_growth_kb": int(rss1 - rss0), "nnz": int(len(key)), "same": same}))
"""


@pytest.mark.skipif(EMU, reason="com-amazon at K = 9000 on the device")
def test_amazon_9000_no_n_by_K(tmp_path):
    script = tmp_path / "amazon_child.py"
    script.write_text(_AMAZON_CHILD)
    r = subprocess.run([sys.executable, str(script), REPO], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["same"], res
    assert res["nnz"] > 0
    assert res["device_bytes"] < (1 << 30), res
    assert res["rss_growth_kb"] * 1024 < (1 << 30), res


def test_argument_checks_leave_state():
    from bigclam_apachespark_b200 import _lib as L
    lib = _lib()
    rp, col = HUB
    n, K = len(rp) - 1, 37
    seeds = np.ascontiguousarray(seeds_of(rp, col), dtype=np.int32)
    assert lib.bigclam_init_F(None, seeds.ctypes.data, len(seeds), 0, C.c_uint64(1)) == L.EINVAL
    for kind in ("sparse", "dense"):
        b = solver(rp, col, K, kind)
        b.set_F(host_F0(rp, col, K, seeds[::-1][:K], pad_seed=99))
        before = b.F_csr(), b.sumF
        for bad in (-1, n):
            s = seeds.copy()
            s[min(3, len(s) - 1)] = bad
            assert lib.bigclam_init_F(b._ctx, s.ctypes.data, len(s), 0, C.c_uint64(1)) == L.EINVAL
            assert b"outside" in lib.bigclam_last_error(b._ctx)
            for x, y in zip(before[0], b.F_csr()):
                assert np.array_equal(x, y)
            assert np.array_equal(before[1], b.sumF)
        b.close()
    os.environ["BIGCLAM_SPARSE_POOL_WORDS"] = "64"
    try:
        b = solver(rp, col, K, "sparse")
    finally:
        del os.environ["BIGCLAM_SPARSE_POOL_WORDS"]
    b.set_F_csr(np.r_[0, np.ones(n, dtype=np.int64)], np.array([5], dtype=np.int32), np.array([0.5]))
    before = b.F_csr(), b.sumF
    assert lib.bigclam_init_F(b._ctx, seeds.ctypes.data, len(seeds), 0, C.c_uint64(1)) == L.ENOMEM
    for x, y in zip(before[0], b.F_csr()):
        assert np.array_equal(x, y)
    assert np.array_equal(before[1], b.sumF)
    b.close()


@pytest.mark.parametrize("K", [37, 1025])
def test_multi_gpu_replicas(K):
    from bigclam_apachespark_b200 import BigClam
    if _lib().bigclam_device_count() < 2:
        pytest.skip("needs 2 or more devices")
    rp, col = HUB
    seeds = seeds_of(rp, col)
    m = BigClam(numGPUs=2).set_graph(rp, col)
    m.Sbc = seeds
    m.init_F(K, pad_seed=5)
    one = solver(rp, col, K, "sparse", seeds).init_F(K, pad_seed=5)
    for rank in range(2):
        assert np.array_equal(m.replica_F(rank), one.F)
        assert np.array_equal(m.replica_sumF(rank), one.sumF)
    for x, y in zip(m.F_csr(), one.F_csr()):
        assert np.array_equal(x, y)
    m.close()
    one.close()
