"""The C ABI from a compiled, non-Python caller (tests/c_host/sgd_find_c.c: plain C99, no torch, no ctypes).

The drop-in boundary of this repo is `include/bigclam_b200.h` and the caller it is meant for is a JNI shim under the
reference's Scala driver (INTEGRATION.md) — compiled code that only sees the header and the shared library.  These
tests build such a caller with the C compiler of the image and

* (CPU) check that the header is valid strict C99 and that every entry point the program uses links against the
  product library; that the program then FAILS LOUDLY on a box without a CUDA device (no CPU path behind the ABI);
  and that its own logic — reader, F0 file, bigclam_run / bigclam_multi_run, getters, output file — is right by
  running it against the host-emulation build of the same C API (tests/emu/build_hostemu.sh) and the oracle;
* (`-m gpu`, tests/test_gpu_zy_c_host.py — collected next to last so that a problem here cannot hide the parity
  results of the suite under `-x`) run it on the H100 against the product library: edge list -> SGDFindC to the reference's stop rule ->
  F, sumF, LLH trace, compared with the oracle's outer loop (bigclam4-7.scala:225-243) from the same F0; and the
  `init` mode (GPU ego-net conductance + initNeighborComF, :58-108) against the driver's own path.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import REPO, random_graph

SRC = os.path.join(REPO, "tests", "c_host", "sgd_find_c.c")
PRODUCT_DIR = os.path.join(REPO, "bigclam_apachespark_b200")
EMU_DIR = os.path.join(REPO, "tests", "emu")
RTOL_F = 1e-9


def product_lib():
    """(directory, file) of the library the `-m gpu` tests link the C caller with: the product library — or, in a
    BIGCLAM_HOSTEMU=1 development run on a CPU box (tests/conftest.py), the host-emulation build of the same C API."""
    if os.environ.get("BIGCLAM_HOSTEMU") == "1":
        return EMU_DIR, "libbigclam_hostemu.so"
    return PRODUCT_DIR, "libbigclam_b200.so"


def _cc():
    return "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else (shutil.which("gcc") or shutil.which("cc"))


_BUILT = {}


def cached_build(key, out, build):
    """One compilation per (program, library) and pytest process: later requests copy the first binary."""
    if key not in _BUILT:
        _BUILT[key] = build(out)
        return out
    shutil.copy2(_BUILT[key], out)
    return out


def _build(out, libdir, libname):
    return cached_build(("c", libdir), out, lambda o: _build_now(o, libdir, libname))


def _build_now(out, libdir, libname):
    cmd = [_cc(), "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(REPO, "include"), SRC,
           "-o", out, "-L", libdir, f"-l:{libname}", f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _write_edgelist(path, rp, col, ids=None):
    """One line per undirected edge (u < v), SNAP style with a comment header; `ids` maps dense index -> vertex id."""
    n = len(rp) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    keep = u < col
    a, b = u[keep], col[keep]
    if ids is not None:
        a, b = ids[a], ids[b]
    with open(path, "w") as fh:
        fh.write("# test graph\n# FromNodeId\tToNodeId\n")
        for x, y in zip(a.tolist(), b.tolist()):
            fh.write(f"{x}\t{y}\n")


def _read_out(path):
    raw = open(path, "rb").read()
    n, k, calls, ntrace = np.frombuffer(raw, dtype=np.int64, count=4)
    body = np.frombuffer(raw, dtype=np.float64, offset=32)
    llh, trace, sumF, F = body[0], body[1:1 + ntrace], body[1 + ntrace:1 + ntrace + k], body[1 + ntrace + k:]
    assert F.size == n * k
    return int(calls), float(llh), trace.copy(), sumF.copy(), F.reshape(n, k).copy()


def _case(tmp_path, n=260, deg=5, k=8, seed=5, dens=0.4):
    """Graph without isolated nodes (the reader only sees vertices that have an edge), F0 file, edge-list file."""
    rp, col = random_graph(n, deg, seed=seed)
    has = np.diff(rp) > 0
    new = np.cumsum(has) - 1
    sel = np.nonzero(has)[0]
    from bigclam_apachespark_b200 import graphs as G
    u = np.repeat(np.arange(n), np.diff(rp))
    keep = u < col
    rp, col = G.csr_from_undirected(len(sel), new[u[keep]], new[col[keep]])
    n = len(sel)
    rng = np.random.default_rng(seed)
    F0 = rng.random((n, k)) * (rng.random((n, k)) < dens)
    ids = np.arange(n) * 3 + 7                      # sparse, ascending vertex ids: the reader relabels them 0..n-1
    edges = str(tmp_path / "edges.txt")
    _write_edgelist(edges, rp, col, ids)
    f0 = str(tmp_path / "F0.f64")
    F0.tofile(f0)
    return rp, col, F0, edges, f0


def _check_against_oracle(oracle, rp, col, F0, k, out, max_outer):
    calls, llh, trace, sumF, F = _read_out(out)
    Fo, so, llho, callso, tro = oracle.run(rp, col, F0, oracle.colsum(F0), oracle.make_params(k), variant=4, max_outer=max_outer)
    assert calls == callso, (calls, callso)
    assert np.allclose(trace, tro, rtol=1e-9)
    assert abs(llh - llho) <= 1e-9 * abs(llho)
    assert np.abs(F - Fo).max() <= RTOL_F * np.abs(Fo).max()
    assert np.allclose(sumF, so, rtol=1e-8)
    # north_star: identical top-community assignment (argmax_c F_uc; a row whose two largest entries agree to rounding may
    # name either)
    top = Fo.argmax(axis=1)
    rows = np.arange(len(top))
    assert (F[rows, top] >= F.max(axis=1) - 1e-9 * max(np.abs(Fo).max(), 1e-300)).all()


# ------------------------------------------------------------------------------------------------ CPU
def test_header_is_strict_c99_and_the_c_caller_links(tmp_path):
    exe = _build(str(tmp_path / "sgd_find_c"), PRODUCT_DIR, "libbigclam_b200.so")
    assert os.access(exe, os.X_OK)


def test_c_caller_fails_loudly_without_a_device(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    rp, col, F0, edges, f0 = _case(tmp_path)
    exe = _build(str(tmp_path / "sgd_find_c"), PRODUCT_DIR, "libbigclam_b200.so")
    r = subprocess.run([exe, edges, "8", "3", f0, str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "bigclam_create failed (-2)" in r.stderr, (r.returncode, r.stderr)
    assert not os.path.exists(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, "8", "3", "init", str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "bigclam_conductance_seeds_gpu failed (-2)" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("world", [1, 2])
def test_c_caller_logic_under_host_emulation(oracle, tmp_path, world):
    """The program itself (not the kernels' sm_90a code) against the oracle: linked with the host-emulation build of the
    C API, which runs the same sources on OS threads.  Test infrastructure only."""
    emu = os.path.join(EMU_DIR, "libbigclam_hostemu.so")
    if not os.path.exists(emu):
        subprocess.run([os.path.join(EMU_DIR, "build_hostemu.sh")], check=True)
    rp, col, F0, edges, f0 = _case(tmp_path, n=120, deg=4, k=6, seed=9)
    exe = _build(str(tmp_path / "sgd_find_c_emu"), EMU_DIR, "libbigclam_hostemu.so")
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, edges, "6", "3", f0, out, str(world)], capture_output=True, text=True, timeout=800)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.startswith("SGDFindC: n=%d K=6 world=%d calls=" % (len(rp) - 1, world))
    _check_against_oracle(oracle, rp, col, F0, 6, out, 3)
