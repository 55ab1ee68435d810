"""Kernel LOGIC of the grouped community extraction on the CPU: a selection of the `-m gpu` tests of
tests/test_gpu_extract.py in a child pytest against the host-emulation build of the C API (tests/emu/build_hostemu.sh, as
tests/test_hostemu_sample.py does for the sampler): the arrays against the NumPy twin at K = 37 (sparse and dense rows)
and 1025, the edge rows, a forced cut into several ranges, untouched state, the argument checks, and the multi-GPU
handle and the C++ mirror on 2 emulated devices.  The `-m gpu` tests on the H100 remain the tests of the compiled sm_90a
code."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = ("extract_matches_twin[37] or extract_matches_twin[1025] or edge_rows or several_ranges or state_untouched "
             "or argument_checks or multi_gpu or cpp_mirror")


@pytest.mark.timeout(1500)
def test_extract_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_extract.py"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert re.search(r"\b10 passed", r.stdout) and "failed" not in r.stdout and "skipped" not in r.stdout, tail
