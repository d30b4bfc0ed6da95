"""GPU: every kernel of librtti_b200.so against a plain PyTorch fp32 reference of the same op
(tests/gpu_diag.py holds the cases; each runs in its own process under a timeout so a dead-locked kernel
cannot hang the box)."""
import os
import subprocess
import sys

import pytest

from tests import gpu_diag

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", list(gpu_diag.CASES))
def test_kernel_case(case):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gpu_diag.py"), case], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert "FAIL" not in r.stdout
