"""`-m gpu` part of tests/test_c_host.py: the plain-C caller (tests/c_host/sgd_find_c.c) on the H100 against the product
library — edge list -> SGDFindC to the reference's stop rule (bigclam4-7.scala:225-243) -> F, sumF, LLH trace against the
oracle's outer loop from the same F0; two GPUs behind one handle; the `init` mode against the Python driver."""
import os
import subprocess

import numpy as np
import pytest

from test_c_host import _build, _case, _check_against_oracle, _read_out, _write_edgelist, product_lib

pytestmark = pytest.mark.gpu


def test_c_caller_matches_oracle_on_gpu(oracle, tmp_path):
    rp, col, F0, edges, f0 = _case(tmp_path, n=600, deg=6, k=12, seed=77, dens=0.3)
    exe = _build(str(tmp_path / "sgd_find_c"), *product_lib())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, "12", "0", f0, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    _check_against_oracle(oracle, rp, col, F0, 12, out, 0)


def test_c_caller_two_gpus_behind_one_handle(oracle, tmp_path):
    from bigclam_apachespark_b200 import _lib
    if int(_lib.load().bigclam_device_count()) < 2:
        pytest.skip("needs 2 GPUs")
    rp, col, F0, edges, f0 = _case(tmp_path, n=600, deg=6, k=12, seed=78, dens=0.3)
    exe = _build(str(tmp_path / "sgd_find_c"), *product_lib())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, "12", "0", f0, out, "2"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    _check_against_oracle(oracle, rp, col, F0, 12, out, 0)


def test_c_caller_init_mode_equals_the_driver(graphs, tmp_path):
    """`init`: GPU conductance seeds + initNeighborComF + SGDFindC from C, against the Python driver on the same graph
    (same library, same entry points: the two callers must agree bit for bit)."""
    from bigclam_apachespark_b200 import BigClam
    if os.environ.get("BIGCLAM_HOSTEMU") == "1":           # development run on a CPU box: a graph the emulation finishes
        rp, col = _case(tmp_path, n=150, deg=5, k=10, seed=3)[:2]
    else:
        rp, col, _ = graphs.load_npz_graph("facebook_combined")
    edges = str(tmp_path / "fb.txt")
    _write_edgelist(edges, rp, col)
    exe = _build(str(tmp_path / "sgd_find_c"), *product_lib())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, "10", "5", "init", out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    calls, llh, trace, sumF, F = _read_out(out)
    b = BigClam(device=0, sparse_rows=True)
    b.set_graph(rp, col).set_K(10)
    b.conductanceLocalMin(on_gpu=True)
    b.initNeighborComF(10, pad_seed=1)
    ret = b.SGDFindC(max_outer=5)
    assert b.last_calls == calls and ret == llh
    assert np.array_equal(np.asarray(b.last_trace), trace)
    assert b.F.tobytes() == F.tobytes() and b.sumF.tobytes() == sumF.tobytes()
    b.close()


@pytest.mark.parametrize("world,mode", [(1, "run"), (1, "csr"), (2, "run"), (2, "csr")])
def test_jni_shim_through_the_fake_jvm(oracle, tmp_path, world, mode):
    """integration/jni/bigclam_b200_jni.c driven by tests/jni_stub/fake_jvm.c (see tests/test_jni_shim.py) against the product
    library: create(Multi) -> setF -> run(SGDFindC) -> getF / getSumF (mode csr: setFCsr, getFNnz + getFCsr — F as rows of
    (index, data) like the reference's BSV rows), against the oracle's outer loop."""
    from bigclam_apachespark_b200 import _lib
    from test_jni_shim import build_fake_jvm
    if int(_lib.load().bigclam_device_count()) < world:
        pytest.skip(f"needs {world} GPUs")
    small = os.environ.get("BIGCLAM_HOSTEMU") == "1"
    n, k = (150, 6) if small else (600, 12)
    rp, col, F0, edges, f0 = _case(tmp_path, n=n, deg=5, k=k, seed=80 + world, dens=0.3)
    exe = build_fake_jvm(str(tmp_path / "fake_jvm"), *product_lib())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, str(k), "6", f0, out, str(world), mode], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    calls, llh, trace, sumF, F = _read_out(out)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, oracle.colsum(F0), oracle.make_params(k), variant=4, max_outer=6)
    assert calls == callso and abs(llh - llho) <= 1e-9 * abs(llho)
    assert np.abs(F - Fo).max() <= 1e-9 * np.abs(Fo).max() and np.allclose(sumF, so, rtol=1e-8)


# ---- include/bigclam_b200.hpp: the C++ mirror of the script surface (tests/test_cpp_host.py), against the product library
def _mirror(tmp_path):
    from test_cpp_host import build_mirror
    return build_mirror(str(tmp_path / "script_mirror"), *product_lib())


def _sizes():
    return (150, 6) if os.environ.get("BIGCLAM_HOSTEMU") == "1" else (600, 12)


@pytest.mark.parametrize("mode,version", [("sgd", 4), ("mbsgd", 3), ("mbsgd", 2)])
def test_cpp_mirror_outer_loops(oracle, tmp_path, mode, version):
    """SGDFindC (bigclam4-7.scala:225-243) and MBSGD (bigclamv3-7.scala:206-222, Bigclamv2.scala:203-219) from C++."""
    n, k = _sizes()
    rp, col, F0, edges, f0 = _case(tmp_path, n=n, deg=6, k=k, seed=90 + version, dens=0.3)
    out = str(tmp_path / "out.bin")
    r = subprocess.run([_mirror(tmp_path), mode, edges, str(k), "8", f0, out, "1", str(version)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    calls, llh, trace, sumF, F = _read_out(out)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, oracle.colsum(F0), oracle.make_params(k), variant=version, max_outer=8)
    assert calls == callso and np.allclose(trace, tro, rtol=1e-9)
    assert np.abs(F - Fo).max() <= 1e-9 * np.abs(Fo).max() and np.allclose(sumF, so, rtol=1e-8)


def test_cpp_mirror_k_sweep(oracle, tmp_path):
    """conductanceLocalMin (GPU kernel) + for K in Kset: initNeighborComF, SGDFindC, stop rule (:244-266) from C++ against the
    oracle-driven sweep."""
    from bigclam_apachespark_b200.driver import Kset
    from test_cpp_host import check_sweep_output
    small = os.environ.get("BIGCLAM_HOSTEMU") == "1"
    rp, col = _case(tmp_path, n=150 if small else 400, deg=6, k=4, seed=95)[:2]
    edges = str(tmp_path / "sweep.txt")
    _write_edgelist(edges, rp, col)
    lo, hi, div, cap = (4, 8, 2, 5) if small else (4, 16, 4, 30)
    r = subprocess.run([_mirror(tmp_path), "sweep", edges, str(lo), str(hi), str(div), str(cap)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    check_sweep_output(oracle, r.stdout, rp, col, Kset(lo, hi, div), cap)
