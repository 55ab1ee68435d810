"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol the header
declares, refuses to compute without a GPU, and its edge-list reader has GraphX semantics."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import REPO


def _lib():
    from bigclam_apachespark_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib


def test_library_exports_every_declared_symbol():
    L = _lib()
    lib = L.load()
    header = open(os.path.join(REPO, "include", "bigclam_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(bigclam_[a-z_A-Z0-9]+)\s*\(", header))
    assert len(declared) >= 20
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/bigclam_b200.h but not exported"
    assert declared == set(L.SIGNATURES), declared ^ set(L.SIGNATURES)
    assert b"sm_90a" in lib.bigclam_version()


def test_params_struct_layout_and_defaults():
    L = _lib()
    p = L.Params()
    assert C.sizeof(L.Params) == 64
    assert L.load().bigclam_default_params(C.byref(p), 200) == 0
    # bigclam4-7.scala:22-26,39-43
    assert (p.k, p.max_inter, p.alpha, p.beta) == (200, 15, 0.05, 0.1)
    assert (p.min_p, p.max_p, p.min_f, p.max_f) == (0.0001, 0.9999, 0.0, 1000.0)
    out = np.empty(16)
    assert L.load().bigclam_step_sizes(0.1, 15, out.ctypes.data) == 0
    assert out[2] == 0.010000000000000002 and out[6] == 1.0000000000000004e-06


def test_reader_graphx_semantics(tmp_path, oracle):
    from bigclam_apachespark_b200 import read_edge_list, BigclamError
    text = ("# comment line\r\n"
            "#another\n"
            "\n"
            "10\t20\r\n"
            "20\t10\r\n"          # reciprocal line (Email-Enron style)
            "10 30   \n"
            "  30\t 40\n"
            "40 40\n"             # self loop
            "7 10 extra-field\n"
            "10\t20\n")           # exact duplicate line
    path = tmp_path / "g.txt"
    path.write_bytes(text.encode())
    for mult in ("keep", "dedup"):
        rp, col, ids = read_edge_list(str(path), mult)
        (rp2, col2), ids2 = oracle.read_edge_list(str(path), mult)
        assert np.array_equal(ids, [7, 10, 20, 30, 40]) and np.array_equal(ids, ids2)
        assert np.array_equal(rp, rp2) and np.array_equal(col, col2), mult
    rp, col, _ = read_edge_list(str(path), "keep")
    # collectNeighborIds(Either): one entry per edge line per endpoint; the self loop counts twice
    assert rp[-1] == 2 * 7
    assert list(col[rp[1]:rp[2]]) == [0, 2, 2, 2, 3]      # node "10": 7, 20 x3, 30
    assert list(col[rp[4]:rp[5]]) == [3, 4, 4]            # node "40": 30, self, self
    rp, col, _ = read_edge_list(str(path), "dedup")
    assert list(col[rp[1]:rp[2]]) == [0, 2, 3] and list(col[rp[4]:rp[5]]) == [3]
    bad = tmp_path / "bad.txt"
    bad.write_text("1 2\n3\n")
    with pytest.raises(BigclamError, match="Invalid line 2"):
        read_edge_list(str(bad))
    with pytest.raises(BigclamError):
        read_edge_list(str(tmp_path / "missing.txt"))
    empty = tmp_path / "empty.txt"
    empty.write_text("# nothing\n")
    rp, col, ids = read_edge_list(str(empty))
    assert len(rp) == 1 and len(col) == 0 and len(ids) == 0


def test_reader_matches_fixture_graph(tmp_path, graphs):
    # write facebook back out as an edge list with the SNAP header conventions and re-read it
    from bigclam_apachespark_b200 import read_edge_list
    rp, col, ids = graphs.load_npz_graph("facebook_combined")
    n = len(rp) - 1
    u = np.repeat(np.arange(n), np.diff(rp))
    m = u < col
    lines = ["# Undirected graph", "# Nodes: %d Edges: %d" % (n, m.sum())]
    lines += ["%d\t%d" % (ids[a], ids[b]) for a, b in zip(u[m], col[m])]
    p = tmp_path / "fb.txt"
    p.write_text("\r\n".join(lines) + "\r\n")
    rp2, col2, ids2 = read_edge_list(str(p), "keep")
    assert np.array_equal(rp, rp2) and np.array_equal(col, col2) and np.array_equal(ids, ids2)
    assert n == 4039 and len(col) == 176468 and np.diff(rp).max() == 1045     # SURVEY.md §8 table


def test_no_cpu_fallback():
    """Without a CUDA device the product must fail loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the -m gpu tests")
    L = _lib()
    lib = L.load()
    assert lib.bigclam_device_count() <= 0
    from bigclam_apachespark_b200 import BigClam, BigclamError
    b = BigClam()
    b.set_graph(np.array([0, 1, 2], dtype=np.int64), np.array([1, 0], dtype=np.int32))
    with pytest.raises(BigclamError, match="no CUDA device"):
        b.set_K(4)
    with pytest.raises(RuntimeError):
        b.backtrackingLineSearchs()


def test_create_argument_validation():
    L = _lib()
    lib = L.load()
    p = L.Params()
    lib.bigclam_default_params(C.byref(p), 8)
    ctx = C.c_void_p()
    rp = np.array([0, 2, 1], dtype=np.int64)       # not monotone
    col = np.array([1, 0], dtype=np.int32)
    assert lib.bigclam_create(C.byref(ctx), 2, rp.ctypes.data, col.ctypes.data, C.byref(p)) == L.EINVAL
    assert b"monotone" in lib.bigclam_last_error(None)
    rp = np.array([0, 1, 2], dtype=np.int64)
    col = np.array([1, 5], dtype=np.int32)         # out of range
    assert lib.bigclam_create(C.byref(ctx), 2, rp.ctypes.data, col.ctypes.data, C.byref(p)) == L.EINVAL
    p.k = 0
    assert lib.bigclam_create(C.byref(ctx), 2, rp.ctypes.data, col.ctypes.data, C.byref(p)) == L.EINVAL
    p.k = 5000
    col = np.array([1, 0], dtype=np.int32)
    assert lib.bigclam_create(C.byref(ctx), 2, rp.ctypes.data, col.ctypes.data, C.byref(p)) == L.EUNSUPPORTED
