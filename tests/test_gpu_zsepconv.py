"""Sepconv on the GPU (SURVEY.md section 8 row a12): tools/sepconv_gpu_check.py in a SUBPROCESS (sorted after the verified
tests; a trap in new code must not poison their CUDA context): every stage, on the CUDA-core checker and on the wgmma
kernel, vs the unmodified reference Network."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_sepconv_gpu_check_subprocess():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sepconv_gpu_check.py")],
                       capture_output=True, text=True, timeout=420, cwd=ROOT)
    tail = (r.stdout[-6000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
