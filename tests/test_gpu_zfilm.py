"""FILM on the GPU (SURVEY.md section 8 row a10): tools/film_gpu_check.py --quick in a SUBPROCESS (a kernel trap in
the newest kernels must not poison the CUDA context of the RIFE tests that share this pytest process; the file name
sorts it after them).  The checker reports, stage by stage: single streamconv layers (wgmma kernel vs the CUDA-core
checker vs torch conv2d with the layer's real weights), the whole network on the checker and on the wgmma kernel vs
the unmodified reference's output (PSNR >= 50 dB), and the node vs the unmodified reference node."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_film_gpu_check_subprocess():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "film_gpu_check.py"), "--quick"],
                       capture_output=True, text=True, timeout=420, cwd=ROOT)
    tail = (r.stdout[-6000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail


@pytest.mark.gpu
def test_film_gpu_check_full_subprocess():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "film_gpu_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    tail = (r.stdout[-8000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
