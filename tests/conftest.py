import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


if os.environ.get("BIGCLAM_HOSTEMU") == "1":
    # development aid (tests/emu/build_hostemu.sh): drive the HOST LOGIC of the C API with the `-m gpu` tests on a
    # machine without a GPU — the ctypes binding is pointed at the host-emulation build for this pytest run only
    import subprocess

    if os.environ.get("BIGCLAM_HOSTEMU_NOBUILD") != "1":
        subprocess.run([os.path.join(REPO, "tests", "emu", "build_hostemu.sh")], check=True)
    from bigclam_apachespark_b200 import _lib as _L

    _L.LIB_PATH = os.path.join(REPO, "tests", "emu", "libbigclam_hostemu.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def golden():
    return np.load(os.path.join(REPO, "tests", "golden", "oracle_steps.npz"))


@pytest.fixture(scope="session")
def graphs():
    from bigclam_apachespark_b200 import graphs as G
    return G


def tiny_graph(G):
    edges = [(0, 1), (0, 2), (0, 3), (0, 4), (0, 5), (1, 2), (2, 3), (6, 7), (7, 8), (8, 9), (9, 6), (5, 6)]
    u, v = np.array(edges).T
    return G.csr_from_undirected(12, u, v)


def random_graph(n, avg_deg, seed, hub=0):
    """Simple undirected random graph with an optional hub of degree `hub` and isolated nodes possible."""
    from bigclam_apachespark_b200 import graphs as G
    rng = np.random.default_rng(seed)
    m = n * avg_deg // 2
    u = rng.integers(0, n, m)
    v = rng.integers(0, n, m)
    if hub:
        u = np.concatenate([u, np.zeros(hub, dtype=np.int64)])
        v = np.concatenate([v, rng.choice(np.arange(1, n), size=min(hub, n - 1), replace=False)])
    keep = u != v
    lo, hi = np.minimum(u[keep], v[keep]), np.maximum(u[keep], v[keep])
    key = np.unique(lo * n + hi)
    return G.csr_from_undirected(n, key // n, key % n)
