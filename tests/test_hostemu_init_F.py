"""Kernel LOGIC of bigclam_init_F on the CPU: a selection of the `-m gpu` tests of tests/test_gpu_init_F.py in a child pytest
against the host-emulation build of the C API (tests/emu/build_hostemu.sh, as tests/test_hostemu_fold_in.py does): the host
F0 bit for bit on a small graph at K = 37 (dense and sparse rows) and K = 1025 (wide rows, padding), the awkward inputs,
the same bits through SGDFindC on wide rows, the argument checks with untouched state, and the multi-GPU handle on 2
emulated devices.  The `-m gpu` tests on the H100 remain the tests of the compiled sm_90a code."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = ("random_graph_same_F0[False-37] or random_graph_same_F0[True-1025] or awkward_inputs or "
             "downstream_wide or argument_checks or multi_gpu")


@pytest.mark.timeout(1500)
def test_init_F_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_init_F.py"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert re.search(r"\b16 passed", r.stdout) and "failed" not in r.stdout and "skipped" not in r.stdout, tail
