"""Neighbour lists as GraphX gives them (repeated entries, self loops, shuffled and one-sided lists) on the CPU.

First the oracle itself: on such lists it must still restate bigclam4-7.scala:157-184, so oracle.step is held against the
independent NumPy twin (oracle/numpy_twin.py) on small GraphX graphs.  Then the `-m gpu` tests of
tests/test_gpu_graphx_lists.py, in a child pytest against the host-emulation build of the C API (tests/emu/build_hostemu.sh,
as tests/test_hostemu_params.py does): every engine case, the LLH identity, uset masks, list order and the sparse-row
device loop.  Email-Enron is left to the GPU run (too large for the emulation), and so is the device loop on dense rows
(a minute of emulation for a path the sparse-row loop shares).  The `-m gpu` run on an H100 remains the test of the
compiled sm_90a code."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import random_graph
from test_gpu_graphx_lists import _F0, DEFAULTS, _graph, graphx
from test_gpu_parity import TIE_TOL

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = "not enron and not (run_loop and dense_rows)"
EXPECTED = 39                 # 43 tests in the file, less Email-Enron and the three dense-row device loops


def _twin_graphs():
    """A 200-node graph with the special nodes, a one-sided one, and a 60-node graph with many repeats and self loops."""
    yield "graphx", _graph("graphx")
    yield "one_sided", _graph("one_sided")
    rp, col = random_graph(60, 5, seed=4)
    yield "dense_repeats", graphx(rp, col, seed=4, self_loop_frac=0.3, repeat_frac=0.4)


@pytest.mark.parametrize("K", [5, 13])
def test_oracle_step_matches_numpy_twin_on_graphx_lists(oracle, K):
    """oracle.step against numpy_twin.backtracking_line_searchs, three steps on the oracle's state: the same accepted
    step (the twin returns its value, NaN for none; the oracle its index), rows within 1e-12 and the LLH within 1e-12
    relative.  A decision that differs must be a tie by the oracle's own Armijo margins."""
    from oracle import numpy_twin as T
    P = oracle.make_params(K)
    steps = oracle.step_sizes(P.beta, P.max_inter)
    for name, (rp, col) in _twin_graphs():
        n = len(rp) - 1
        F = _F0(n, K, DEFAULTS, seed=K)
        s = oracle.colsum(F)
        for it in range(3):
            where = f"{name} K={K} step {it}"
            r = oracle.step(rp, col, F, s, P)
            Ft, st, llh_t, acc_t = T.backtracking_line_searchs(rp, col, F, s)
            acc_o = np.where(r.accepted >= 0, steps[np.maximum(r.accepted, 0)], np.nan)
            same = (acc_o == acc_t) | (np.isnan(acc_o) & np.isnan(acc_t))
            scale = max(np.abs(r.F).max(), 1.0)
            if not same.all():
                nodes = np.flatnonzero(~same)
                margins, llh_u = oracle.armijo_margins(rp, col, F, s, P, nodes)
                for i, u in enumerate(nodes):
                    jt = P.max_inter + 1 if np.isnan(acc_t[u]) else int(np.flatnonzero(steps == acc_t[u])[0])
                    jo = P.max_inter + 1 if r.accepted[u] < 0 else int(r.accepted[u])
                    assert abs(margins[i, min(jt, jo)]) <= TIE_TOL * max(abs(llh_u[i]), 1.0), (where, u, jt, jo)
            assert np.abs(Ft[same] - r.F[same]).max() <= 1e-12 * scale, where
            assert same.mean() >= 0.98, where
            if same.all():
                assert np.abs(st - r.sumF).max() <= 1e-12 * max(np.abs(r.sumF).max(), 1.0), where
                assert abs(llh_t - r.llh) <= 1e-12 * abs(r.llh), where
            assert r.n_updated > 0, where
            F, s = r.F, r.sumF


@pytest.mark.timeout(1500)
def test_graphx_lists_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_graphx_lists.py"), "-m", "gpu", "-q",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"\b(\d+) passed", r.stdout)
    assert m and int(m.group(1)) == EXPECTED and "failed" not in r.stdout and "skipped" not in r.stdout, tail
