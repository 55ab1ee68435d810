"""Kernel LOGIC of the wide-row variant (K > 1024) on the CPU: a selection of the `-m gpu` tests of tests/test_gpu_wide_k.py
in a child pytest against the host-emulation build of the C API (tests/emu/build_hostemu.sh, as tests/test_hostemu_sparse.py
does for the sparse engine): single steps at K = 1025 and 2000, split hubs, a uset mask with loglikelihood(), bit-identical
reruns and the multi-GPU handle on 2 emulated devices.  The `-m gpu` tests on the H100 remain the parity tests of the
compiled sm_90a code."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = ("(single_step and (1025 or 2000)) or split_hubs or uset_mask or bit_identical or multi_gpu")


@pytest.mark.timeout(1500)
def test_wide_rows_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_wide_k.py"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert re.search(r"\b6 passed", r.stdout) and "failed" not in r.stdout and "skipped" not in r.stdout, tail
