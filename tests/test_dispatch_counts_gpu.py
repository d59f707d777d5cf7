"""The forward, training and augmentation kernels at SM counts and persistent grid sizes other than this device's, bit for bit:
tests/dispatch_counts_traced.py, run in a pytest process of its own so that its CUDA activity sessions leave this process's tracer
untouched (see that module).  -s prints its report."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_dispatch_counts_in_own_process():
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(py + ["-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", os.path.join(HERE, "dispatch_counts_traced.py")],
                       cwd=os.path.dirname(HERE), capture_output=True, text=True)
    print(r.stdout[-200000:], r.stderr[-20000:])
    failed = [line for line in r.stdout.splitlines() if line.startswith(("FAILED", "ERROR"))]
    assert r.returncode == 0, "\n".join(failed or [r.stdout[-5000:], r.stderr[-5000:]])
