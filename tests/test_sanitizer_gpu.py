"""compute-sanitizer memcheck over one small invocation of every kernel family (tools/san_check.py).  Opt-in
(MONOPORT_B200_RUN_SANITIZER=1): the instrumented run takes minutes, the plain GPU suite seconds.
    MONOPORT_B200_RUN_SANITIZER=1 python -m pytest tests/test_sanitizer_gpu.py -m gpu -q"""
import os
import shutil
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_memcheck_reports_no_errors():
    if os.environ.get("MONOPORT_B200_RUN_SANITIZER", "0") != "1":
        pytest.skip("opt-in: MONOPORT_B200_RUN_SANITIZER=1")
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer not found")
    r = subprocess.run([exe, "--tool", "memcheck", "--error-exitcode", "9", sys.executable, os.path.join(ROOT, "tools", "san_check.py")],
                       capture_output=True, text=True, timeout=1500, cwd=ROOT)
    out = r.stdout + r.stderr
    log = os.environ.get("MONOPORT_B200_SANITIZER_LOG")
    if log:
        open(log, "w").write(out)
    assert "ERROR SUMMARY: 0 errors" in out, out[-3000:]
    assert r.returncode == 0, out[-3000:]
