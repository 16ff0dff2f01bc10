"""The WHOLE CAIN path of the library on the CPU: csrc/cain.cu (vfi_cain_load + vfi_cain_forward: weight packing, the
bordered layout and its border fills, buffer sizing, the schedule), csrc/cain_elem.cu and streamconv.cu's packer +
CUDA-core checker kernel, compiled for the host (tests/host_emu) and compared with the output of the unmodified
reference CAIN (tests/golden/cain_*.npz).  The tensor-core kernel is not part of this; tools/cain_gpu_check.py compares
it with the same checker kernel on the GPU."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_cain import cain_cases, cain_inputs, case_state_dict  # noqa: E402
from oracle import cain as OC  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libcainfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "cain_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.vfi_last_error.restype = C.c_char_p
    lib.emu_cain.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return lib


def _run(emu, sd, img0, img1):
    hold = [sd[n].contiguous() for n, _ in OC.state_dict_spec()]
    ptrs = (C.c_void_p * len(hold))(*[x.data_ptr() for x in hold])
    numel = (C.c_int64 * len(hold))(*[x.numel() for x in hold])
    _, h, w = img0.shape
    out = torch.zeros(3, h, w)
    rc = emu.emu_cain(ptrs, numel, len(hold), img0.contiguous().data_ptr(), img1.contiguous().data_ptr(), h, w,
                      out.data_ptr())
    return rc, out


@pytest.mark.parametrize("name", [k for k, v in cain_cases().items() if v["kind"] == "net"])
def test_cain_whole_path_on_host_matches_reference(emu, name):
    cfg = cain_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"])[0]
    x = cain_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    rc, out = _run(emu, case_state_dict(cfg), x[0], x[1])
    assert rc >= 1000, (rc, emu.vfi_last_error())
    mse = float(((out.double() - ref.double()) ** 2).mean())
    p = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"{name}: host emulation of the whole CAIN path, {rc - 1000} launches, PSNR {p:.2f} dB, "
          f"max abs {float((out - ref).abs().max()):.2e}")
    assert rc - 1000 == 376
    assert p >= 50.0, p


def test_refuses_a_wrong_shape_by_name_and_a_frame_too_small(emu):
    sd = OC.synthetic_state_dict(0)
    x = torch.rand(2, 3, 64, 64)
    bad = dict(sd)
    bad["encoder.interpolate.body.2.body.7.body.3.conv_du.0.weight"] = torch.zeros(16, 192, 1, 1)
    rc, _ = _run(emu, bad, x[0], x[1])
    assert rc != 0 and rc < 1000
    assert b"encoder.interpolate.body.2.body.7.body.3.conv_du.0.weight" in emu.vfi_last_error()
    # 40 columns pad to 128 with 44 on one side: ReflectionPad2d raises in the reference
    x = torch.rand(2, 3, 64, 40)
    rc, out = _run(emu, sd, x[0], x[1])
    assert rc != 0 and rc < 1000 and b"cannot be reflection-padded" in emu.vfi_last_error()
    assert OC.geometry(64, 40) is None
    assert not out.any()
