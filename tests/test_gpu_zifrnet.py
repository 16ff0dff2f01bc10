"""IFRNet on the GPU: tools/ifrnet_gpu_check.py in a SUBPROCESS (a kernel trap in the newest kernels must not poison the
CUDA context of the tests that share this pytest process; the file name sorts it after them).  The checker reports, stage
by stage: every streamconv layer kind IFRNet uses with its epilogue (wgmma kernel vs the CUDA-core checker vs torch
conv2d / conv_transpose2d, fp16 and bf16), one at the 1080p geometry, both variants' model goldens on the checker and on
the wgmma kernel vs the unmodified reference (PSNR >= 50 dB), and the node goldens.  With VFI_PARENT_SRC naming a
checkout of the parent commit it also builds that library in a temp directory and requires FILM, Sepconv and FLAVR
outputs to be bit-identical."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_ifrnet_gpu_check_subprocess():
    cmd = [sys.executable, os.path.join(ROOT, "tools", "ifrnet_gpu_check.py")]
    if os.environ.get("VFI_PARENT_SRC"):
        cmd += ["--parent-src", os.environ["VFI_PARENT_SRC"]]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    tail = (r.stdout[-8000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
