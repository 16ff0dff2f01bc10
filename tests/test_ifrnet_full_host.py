"""The WHOLE IFRNet path of the library on the CPU: csrc/ifrnet.cu (vfi_ifrnet_load + vfi_ifrnet_forward: the channel
layout, the packing of the side-channel, space-to-depth and ConvT phase weights, buffer sizing, the schedule),
csrc/ifrnet_elem.cu and streamconv.cu's packer + CUDA-core checker kernel, compiled for the host (tests/host_emu) and
compared with the output of the unmodified reference IRFNet_S / IRFNet_L (tests/golden/ifrnet_*.npz).  The tensor-core
kernel is not part of this; tools/ifrnet_gpu_check.py compares it with the same checker kernel on the GPU."""
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
from make_golden_ifrnet import case_state_dict, ifrnet_cases, ifrnet_inputs  # noqa: E402
from oracle import ifrnet as OI  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libifrnetfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "ifrnet_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.vfi_last_error.restype = C.c_char_p
    lib.emu_ifrnet.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double,
                               C.c_double, C.c_void_p, C.c_void_p]
    return lib


def _run(emu, sd, variant, img0, img1, t, embt):
    hold = [sd[n].contiguous() for n, _ in OI.state_dict_spec(variant)]
    ptrs = (C.c_void_p * len(hold))(*[x.data_ptr() for x in hold])
    numel = (C.c_int64 * len(hold))(*[x.numel() for x in hold])
    _, h, w = img0.shape
    out = torch.zeros(3, h, w)
    v = C.c_int(-1)
    rc = emu.emu_ifrnet(ptrs, numel, len(hold), img0.data_ptr(), img1.data_ptr(), h, w, t, embt, out.data_ptr(),
                        C.byref(v))
    return rc, out, v.value


@pytest.mark.parametrize("name", [k for k, v in ifrnet_cases().items() if v["kind"] == "net"])
def test_ifrnet_whole_path_on_host_matches_reference(emu, name):
    cfg = ifrnet_cases()[name]
    sd = case_state_dict(cfg)
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"])[0]
    x = ifrnet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    rc, out, variant = _run(emu, sd, cfg["variant"], x[0], x[1], cfg["t"], cfg["embt"])
    assert rc >= 1000, (rc, emu.vfi_last_error())
    assert variant == (1 if cfg["variant"] == "L" else 0)
    mse = float(((out.double() - ref.double()) ** 2).mean())
    p = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"{name}: host emulation of the whole IFRNet path, {rc - 1000} launches, PSNR {p:.2f} dB, "
          f"max abs {float((out - ref).abs().max()):.2e}")
    assert p >= 50.0, p


def test_refuses_wrong_shapes_and_bad_resize_factors(emu):
    sd = OI.synthetic_state_dict("S", 0)
    x = torch.rand(2, 3, 40, 40)
    # a ResBlock side conv with L's 64 side channels in an S checkpoint
    bad = dict(sd)
    bad["decoder3.convblock.1.conv2.0.weight"] = torch.zeros(64, 64, 3, 3)
    rc, _, _ = _run(emu, bad, "S", x[0], x[1], 0.5, 1.0)
    assert rc != 0 and rc < 1000
    assert b"decoder3.convblock.1.conv2" in emu.vfi_last_error()
    # multiplier 1000 on a 40 x 40 frame: floor(64 / 1000) = 0 rows
    rc, _, _ = _run(emu, sd, "S", x[0], x[1], 1.0 / 1000, 1.0)
    assert rc != 0 and rc < 1000 and b"empty encoder input" in emu.vfi_last_error()
    assert OI.geometry(40, 40, 1.0 / 1000) is None
