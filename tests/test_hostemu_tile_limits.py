"""The tile path's shared-memory limits (tests/test_gpu_tile_limits.py) on the CPU: every limit at L and L + 1, at K = 32,
161 and 257, with the line-search bounds on and off, plus the degree-32 / degree-33 cut, the uset, device-loop, rerun,
wide-row and re-cut cases, in a child pytest against the host-emulation build of the C API (tests/emu/build_hostemu.sh,
as tests/test_hostemu_sparse.py does).  The logic of every construction and every predicted counter is checked here
before the `-m gpu` run on an H100, which remains the test of the compiled sm_90a code.  Wall time 146 s on an 8-core
x86 host, build included."""
import os
import re
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SELECTION = "(at_and_past and (-32- or -161- or -257-)) or not at_and_past"


@pytest.mark.timeout(1500)
def test_tile_limits_under_host_emulation():
    env = dict(os.environ, BIGCLAM_HOSTEMU="1")
    env.pop("BIGCLAM_HOSTEMU_NOBUILD", None)
    cmd = [sys.executable, "-m", "pytest", os.path.join(REPO, "tests", "test_gpu_tile_limits.py"), "-m", "gpu", "-q",
           "-p", "no:cacheprovider", "-k", SELECTION]
    r = subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=1400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    m = re.search(r"\b(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 46 and "failed" not in r.stdout, tail
