"""Kernel LOGIC of the fold-in on the CPU: a selection of the `-m gpu` tests of tests/test_gpu_fold_in.py in a child pytest
against the host-emulation build of the C API (tests/emu/build_hostemu.sh, as tests/test_hostemu_links.py does): oracle
parity at K = 37 (sparse and dense rows) and K = 1025 (wide rows), the first iteration against bigclam_step, independence
of the batch, untouched state, the argument checks, the C++ mirror and the multi-GPU handle on 2 emulated devices.
The `-m gpu` tests on the H100 remain the tests of the compiled sm_90a code."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = ("oracle_parity_random_graph[37] or oracle_parity_random_graph[1025] or first_iteration_equals_step[37] or "
             "independent_of_the_batch[37] or state_untouched or argument_checks or cpp_mirror or multi_gpu")


@pytest.mark.timeout(1500)
def test_fold_in_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_fold_in.py"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert re.search(r"\b8 passed", r.stdout) and "failed" not in r.stdout and "skipped" not in r.stdout, tail
