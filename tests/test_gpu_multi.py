"""All the GPUs of one box through the C ABI only (bigclam_multi_*: no torch.distributed, no NCCL): one context per
device, fused NVLink row pushes and the fused collective, against the oracle and against the single-GPU path.
Needs >= 2 GPUs (skipped on a 1-GPU machine: `python -m pytest tests/test_gpu_multi.py -m gpu` on a box with 2/4/8).  Under the host-emulation build (BIGCLAM_HOSTEMU=1) the "devices" are emulated and the
test runs on the CPU (tests/test_hostemu_sparse.py drives it)."""
import os

import numpy as np
import pytest

from conftest import random_graph
from test_gpu_parity import _check_step

pytestmark = pytest.mark.gpu


def _ngpus():
    from bigclam_apachespark_b200 import _lib
    return int(_lib.load().bigclam_device_count())


def _worlds():
    return [2, 3] if os.environ.get("BIGCLAM_HOSTEMU") == "1" else [2, 4, 8]


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("hub", [30, 150])
def test_multi_steps_match_oracle_and_replicas_agree(oracle, world, hub, monkeypatch):
    if world not in _worlds() or _ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    monkeypatch.setenv("BIGCLAM_SPARSE_HUB_DEG", "100")
    from bigclam_apachespark_b200 import BigClam
    n, k = 240, 24
    rp, col = random_graph(n, 5, seed=7 + world, hub=hub)
    rng = np.random.default_rng(3)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.25)
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


@pytest.mark.parametrize("world", [2, 3, 8])
def test_multi_steps_in_the_large_graph_regime(oracle, world):
    """sumF as if the graph were 900 times larger (the hot path takes sumF as given, :38,:192): most components of a node's
    gradient are -sumF_c, fewer and fewer nodes move, and the line search by bounds excludes most candidates — on every rank
    the same way: rows, LLH and the number of updated nodes against the oracle, replicas bit-identical."""
    if world not in _worlds() or _ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    from bigclam_apachespark_b200 import BigClam
    n, k = 400, 64
    rp, col = random_graph(n, 4, seed=164)
    rng = np.random.default_rng(64)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.1)
    sumF = oracle.colsum(F0) * 900
    P = oracle.make_params(k)
    b = BigClam(record_accepted=False, numGPUs=world)
    b.set_graph(rp, col).set_K(k).set_F(F0, sumF=sumF)
    F, s = F0, sumF
    moved = []
    b.ls_stats()
    for it in range(5):
        llh = b.backtrackingLineSearchs()
        r = oracle.step(rp, col, F, s, P)
        assert abs(llh - r.llh) <= 1e-10 * abs(r.llh) and b.last_n_updated == r.n_updated, f"step {it}"
        reps = [b.replica_F(q) for q in range(world)]
        for q in range(1, world):
            assert np.array_equal(reps[0], reps[q]), f"replica {q} differs from replica 0 after step {it}"
        assert np.abs(reps[0] - r.F).max() <= 1e-9 * max(np.abs(r.F).max(), 1e-300)
        moved.append(r.n_updated)
        F, s = r.F, r.sumF
    assert moved[-1] < 0.5 * moved[0], moved            # the regime the test is about
    st = b.ls_stats()                                   # (summed over the ranks: bigclam_multi_get_ls_stats)
    assert 0 < st["nodes_searched"] < st["nodes_asked"], st
    b.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("variant", [4, 2])
def test_multi_run_loop_matches_single_gpu(oracle, world, variant):
    if world not in _worlds() or _ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    from bigclam_apachespark_b200 import BigClam
    n, k = 200, 10
    rp, col = random_graph(n, 6, seed=21)
    rng = np.random.default_rng(21)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < 0.4)
    sumF = oracle.colsum(F0)
    Fo, so, llh_o, calls_o, trace_o = oracle.run(rp, col, F0, sumF, oracle.make_params(k), variant=variant, rel_tol=1e-3, max_outer=12)
    b = BigClam(numGPUs=world)
    b.set_graph(rp, col).set_K(k).set_F(F0, sumF=sumF)
    llh = b._run(variant, 1e-3, 12)
    assert b.last_calls == calls_o
    assert abs(llh - llh_o) <= 1e-9 * abs(llh_o)
    assert np.abs(b.F - Fo).max() <= 1e-8 * max(np.abs(Fo).max(), 1e-300)
    for q in range(1, world):
        assert np.array_equal(b.replica_F(0), b.replica_F(q))
    b.close()
