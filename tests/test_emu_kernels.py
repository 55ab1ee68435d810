"""Kernel LOGIC on the CPU: the source of the DENSE kernels (csrc/bigclam_kernels.cuh) compiled for the host against the SIMT
emulation in tests/emu (one OS thread per CUDA thread, warp collectives as barrier rounds) and checked against
the oracle.  Test infrastructure only — nothing here is reachable from the package, which has no CPU path; the
`-m gpu` tests remain the parity tests of the compiled sm_90a code.  (The sparse-row engine runs under the same
emulation through the host build of the whole C API: tests/test_hostemu_sparse.py.)"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import random_graph, tiny_graph

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(request):
    out = "libemu.so"
    subprocess.run([os.path.join(HERE, "emu", "build.sh")], check=True, env=dict(os.environ, EMU_OUT=out))
    lib = C.CDLL(os.path.join(HERE, "emu", out))
    step_args = [C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                 C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emu_dense_step.restype = C.c_int
    lib.emu_dense_step.argtypes = step_args
    lib.emu_dense_step_hubs.restype = C.c_int
    lib.emu_dense_step_hubs.argtypes = step_args
    return lib


def dense_step(lib, rp, col, F, sumF, mask=None, linesearch=True, grid=1):
    n, k = F.shape
    ld = (k + 3) & ~3
    rp = np.ascontiguousarray(rp, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int32)
    F = np.ascontiguousarray(F, dtype=np.float64)
    sumF = np.ascontiguousarray(sumF, dtype=np.float64)
    Fo = np.empty_like(F)
    partials = np.zeros(2 * ld + 2)
    acc = np.empty(n, dtype=np.int8)
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    rc = lib.emu_dense_step(n, rp.ctypes.data, col.ctypes.data, k, F.ctypes.data, sumF.ctypes.data,
                            None if m is None else m.ctypes.data, 1 if linesearch else 0, 15, 0.05, 0.1, grid,
                            Fo.ctypes.data, partials.ctypes.data, acc.ctypes.data)
    assert rc == 0
    D, llh_pre, nupd = partials[:k], partials[2 * ld], int(round(partials[2 * ld + 1]))
    return Fo, sumF - D if nupd else sumF.copy(), llh_pre, nupd, acc


def check(F, s, llh_pre, nupd, acc, r, oracle_llh_pre, max_flips=0):
    scale = max(np.abs(r.F).max(), 1e-300)
    row_err = np.abs(F - r.F).max(axis=1)
    flipped = row_err > 1e-9 * scale
    assert int(flipped.sum()) <= max_flips, (int(flipped.sum()), row_err.max())
    d = (acc != r.accepted) & ~flipped
    assert (((acc[d] < 0) | (acc[d] >= 12)) & ((r.accepted[d] < 0) | (r.accepted[d] >= 12))).all()
    assert abs(llh_pre - oracle_llh_pre) <= 1e-10 * abs(oracle_llh_pre)
    if not flipped.any():
        assert np.allclose(s, r.sumF, rtol=1e-11, atol=1e-9)
        if not d.any():
            assert nupd == r.n_updated


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k,grid", [(5, 1), (40, 2), (100, 1), (200, 1), (300, 1), (600, 1)])
def test_dense_kernel_source_against_oracle(emu, oracle, k, grid):
    """The GPU-validated dense kernels through the same emulation: pins the emulation itself (shuffle, ballot and
    barrier semantics) as much as the kernel logic (C2 = 1, 1, 2, 4, 8, 16 chunk shapes; dense and pair-list paths)."""
    n = 80
    rp, col = random_graph(n, 5, seed=100 + k, hub=40)
    rng = np.random.default_rng(k)
    F = rng.random((n, k)) * (rng.random((n, k)) < min(1.0, 6.0 / k + 0.05))
    sumF = oracle.colsum(F)
    P = oracle.make_params(k)
    r = oracle.step(rp, col, F, sumF, P)
    Fo, so, llh_pre, nupd, acc = dense_step(emu, rp, col, F, sumF, grid=grid)
    check(Fo, so, llh_pre, nupd, acc, r, oracle.llh(rp, col, F, sumF, P))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k", [12, 200])
def test_dense_kernel_source_hub_phase(emu, oracle, k):
    """step_kernel<C2,R,true,false>: a 700-edge hub as a multi-phase "mega" hub (two 384-edge slices through the
    global scratch), a 300-edge hub done by the whole block (phase 0), the other nodes one warp each."""
    from bigclam_apachespark_b200 import graphs as G
    n = 900
    rng = np.random.default_rng(44)
    u = np.concatenate([rng.integers(0, n, 1500), np.zeros(700, dtype=np.int64), np.ones(300, dtype=np.int64)])
    v = np.concatenate([rng.integers(0, n, 1500), rng.choice(np.arange(2, n), 700, replace=False),
                        rng.choice(np.arange(2, n), 300, replace=False)])
    keep = u != v
    lo, hi = np.minimum(u[keep], v[keep]), np.maximum(u[keep], v[keep])
    key = np.unique(lo * n + hi)
    rp, col = G.csr_from_undirected(n, key // n, key % n)
    F = rng.random((n, k)) * (rng.random((n, k)) < min(1.0, 4.0 / k + 0.05))
    sumF = oracle.colsum(F)
    P = oracle.make_params(k)
    ld = (k + 3) & ~3
    Fo = np.empty_like(F)
    partials = np.zeros(2 * ld + 2)
    acc = np.empty(n, dtype=np.int8)
    rp64, col32 = np.ascontiguousarray(rp, dtype=np.int64), np.ascontiguousarray(col, dtype=np.int32)
    rc = emu.emu_dense_step_hubs(n, rp64.ctypes.data, col32.ctypes.data, k, F.ctypes.data, sumF.ctypes.data, None, 1, 15,
                                 0.05, 0.1, 280, Fo.ctypes.data, partials.ctypes.data, acc.ctypes.data)
    assert rc == 1002
    r = oracle.step(rp, col, F, sumF, P)
    nupd = int(round(partials[2 * ld + 1]))
    check(Fo, sumF - partials[:k] if nupd else sumF, partials[2 * ld], nupd, acc, r, oracle.llh(rp, col, F, sumF, P), max_flips=1)
