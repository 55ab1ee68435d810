"""Kernel LOGIC of the edge probabilities and link recommendations on the CPU: a selection of the `-m gpu` tests of
tests/test_gpu_links.py in a child pytest against the host-emulation build of the C API (tests/emu/build_hostemu.sh, as
tests/test_hostemu_wide_k.py does for the wide rows): the affinity bits at K = 37, 1024 and 9000, the two-hop ranking
against brute force for sparse and dense rows, untouched state, the argument checks, the C++ mirror and the multi-GPU handle on 2 emulated devices.
The `-m gpu` tests on the H100 remain the tests of the compiled sm_90a code."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = ("pair_affinity_bits[37] or pair_affinity_bits[1024] or pair_affinity_bits[9000] or "
             "(recommend_against_brute_force and 5-) or dense_rows or state_untouched or argument_checks or cpp_mirror or multi_gpu")


@pytest.mark.timeout(1500)
def test_links_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_links.py"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert re.search(r"\b10 passed", r.stdout) and "failed" not in r.stdout and "skipped" not in r.stdout, tail
