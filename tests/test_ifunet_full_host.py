"""The WHOLE IFUnet path of the library on the CPU: csrc/ifunet.cu (vfi_ifunet_load + vfi_ifunet_forward: BatchNorm
folding, weight packing, the channel layout, workspace sizing, the schedule), csrc/ifunet_elem.cu and streamconv.cu's
packer + CUDA-core checker kernel, compiled for the host (tests/host_emu) and compared with the output of the unmodified
reference IFUNetModel (tests/golden/ifunet_*.npz).  The tensor-core kernel is not part of this; tools/ifunet_gpu_check.py
compares it with the reference on the GPU."""
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
from make_golden_ifunet import case_state_dict, ifunet_cases, ifunet_inputs  # noqa: E402
from oracle import ifunet as OU  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"
# the host path against the reference on the model goldens (fp16 operands, fp32 accumulation): 75.9 - 78.5 dB; the
# figure of each case is in DESIGN.md section 12
PSNR_FLOOR = 70.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libifunetfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "ifunet_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.vfi_last_error.restype = C.c_char_p
    lib.emu_ifunet.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double,
                               C.c_double, C.c_int, C.c_void_p]
    return lib


def _run(emu, sd, img0, img1, t, scale, ensemble):
    hold = [sd[n].float().contiguous() for n, _ in OU.state_dict_spec()]
    ptrs = (C.c_void_p * len(hold))(*[x.data_ptr() for x in hold])
    numel = (C.c_int64 * len(hold))(*[x.numel() for x in hold])
    _, h, w = img0.shape
    out = torch.zeros(3, h, w)
    rc = emu.emu_ifunet(ptrs, numel, len(hold), img0.contiguous().data_ptr(), img1.contiguous().data_ptr(), h, w,
                        float(t), float(scale), int(ensemble), out.data_ptr())
    return rc, out


@pytest.mark.parametrize("name", [k for k, v in ifunet_cases().items() if v["kind"] == "net"])
def test_ifunet_whole_path_on_host_matches_reference(emu, name):
    cfg = ifunet_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"])[0]
    x = ifunet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    rc, out = _run(emu, case_state_dict(cfg), x[0], x[1], cfg["t"], cfg["scale"], cfg["ensemble"])
    assert rc >= 1000, (rc, emu.vfi_last_error())
    mse = float(((out.double() - ref.double()) ** 2).mean())
    p = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"{name}: host emulation of the whole IFUnet path, {rc - 1000} launches, PSNR {p:.2f} dB, "
          f"max abs {float((out - ref).abs().max()):.2e}")
    assert p >= PSNR_FLOOR, p


def test_refuses_a_wrong_shape_by_name_and_a_scale_the_reference_cannot_run(emu):
    sd = OU.synthetic_state_dict(0)
    x = torch.rand(2, 3, 64, 64)
    bad = dict(sd)
    bad["flownet.block1.maskconvx8.bias"] = torch.zeros(575)
    rc, _ = _run(emu, bad, x[0], x[1], 0.5, 1.0, True)
    assert rc != 0 and rc < 1000
    assert b"flownet.block1.maskconvx8.bias" in emu.vfi_last_error()
    for s in (0.25, 0.7, 1.2):
        x = torch.rand(2, 3, 100, 150)
        rc, out = _run(emu, sd, x[0], x[1], 0.5, s, True)
        assert rc != 0 and rc < 1000 and b"the reference raises" in emu.vfi_last_error(), s
        assert OU.geometry(100, 150, s) is None
        assert not out.any()
