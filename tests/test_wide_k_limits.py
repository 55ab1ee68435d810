"""The limits on K that bigclam_create checks before it touches a device: 1024 for dense rows, 16384 with sparse rows."""
import ctypes as C
import os

import numpy as np

RP = np.array([0, 1, 2], dtype=np.int64)
COL = np.array([1, 0], dtype=np.int32)


def _lib():
    from bigclam_apachespark_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib


def _create(k, flags):
    L = _lib()
    lib = L.load()
    p = L.Params()
    assert lib.bigclam_default_params(C.byref(p), k) == L.OK
    p.flags = flags
    ctx = C.c_void_p()
    rc = lib.bigclam_create(C.byref(ctx), 2, RP.ctypes.data, COL.ctypes.data, C.byref(p))
    if rc == L.OK:
        lib.bigclam_destroy(ctx)
    return rc, lib.bigclam_last_error(None)


def test_sparse_rows_above_16384_are_refused_with_the_limit_named():
    L = _lib()
    rc, msg = _create(16385, L.F_SPARSE_ROWS)
    assert rc == L.EUNSUPPORTED and b"16384" in msg, msg


def test_sparse_rows_at_16384_pass_validation():
    L = _lib()
    rc, msg = _create(16384, L.F_SPARSE_ROWS)
    if int(L.load().bigclam_device_count()) > 0:
        assert rc == L.OK, msg
    else:
        assert rc == L.ECUDA and b"no CUDA device" in msg, msg


def test_dense_rows_above_1024_are_still_refused():
    L = _lib()
    rc, msg = _create(1025, 0)
    assert rc == L.EUNSUPPORTED and b"1024" in msg, msg
