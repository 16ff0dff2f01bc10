"""The WHOLE FLAVR path of the library on the CPU: csrc/flavr.cu (vfi_flavr_load + vfi_flavr_forward: the packing of the
temporal, space-to-depth and transposed-phase weights, buffer sizing, the schedule), csrc/flavr_elem.cu and streamconv.cu's
packer + CUDA-core checker kernel, compiled for the host (tests/host_emu) and compared with the output of the unmodified
reference UNet_3D_3D (tests/golden/flavr_*.npz).  The tensor-core kernel is not part of this; tools/flavr_gpu_check.py
compares it with the same checker kernel on the GPU."""
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
from make_golden_flavr import flavr_cases, flavr_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402  (synthetic_clip)
from oracle import flavr as OV  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libflavrfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "flavr_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.vfi_last_error.restype = C.c_char_p
    return lib


def _run(emu, sd, names, frames, first):
    hold = [sd[n].contiguous() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    n, h, w, c = frames.shape
    fr = frames.contiguous()
    fi = np.ascontiguousarray(np.asarray(first, np.int32))
    out = torch.zeros(len(first), h, w, 3)
    n_out, eb = C.c_int(), C.c_int()
    rc = emu.emu_flavr(ptrs, numel, len(hold), C.c_void_p(fr.data_ptr()), n, h, w, c, C.c_void_p(fi.ctypes.data),
                       len(first), C.c_void_p(out.data_ptr()), C.byref(n_out), C.byref(eb))
    assert rc >= 1000, (rc, emu.vfi_last_error())
    return out, rc - 1000, n_out.value, eb.value


@pytest.mark.parametrize("name", [k for k, v in flavr_cases().items() if v["kind"] == "net"])
def test_flavr_whole_path_on_host_matches_reference(emu, pkg, name):
    from cfi_b200.engine import flavr_state_dict_names
    cfg = flavr_cases()[name]
    n_out, bias = OV.VARIANTS[cfg["variant"]]
    sd = OV.synthetic_state_dict(cfg["seed"], cfg["variant"])
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"])[0].permute(1, 2, 0)
    fr = flavr_inputs(cfg)
    out, launches, got_n, got_b = _run(emu, sd, flavr_state_dict_names(bias), fr, [0])
    mse = float(((out[0].double() - ref.double()) ** 2).mean())
    p = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"host emulation of the whole FLAVR path: {launches} launches, PSNR {p:.2f} dB, "
          f"max abs {float((out[0] - ref).abs().max()):.2e}")
    assert (got_n, got_b) == (n_out, int(bias))
    assert p >= 50.0, p
    mean_only = OV.mean_only(fr[..., :3])
    mse0 = float(((mean_only.double() - ref.double()) ** 2).mean())
    assert 10 * math.log10(1.0 / mse0) < 30.0


def test_eight_output_checkpoint_uses_output_zero_on_host(emu, pkg):
    """FLAVR_8x.pth has 7 outputs (21 outconv channels) and encoder biases; the library reads both from the tensors and
    computes output 0 only, which the oracle (outconv.1 channels 0..2) also gives.  Two windows in one call."""
    from cfi_b200.engine import flavr_state_dict_names
    sd = OV.synthetic_state_dict(11, "8x")
    fr = OF.synthetic_clip(5, 16, 24, seed=57)
    out, _, n_out, eb = _run(emu, sd, flavr_state_dict_names(True), fr, [1, 0])
    assert (n_out, eb) == (7, 1)
    for k, f in enumerate([1, 0]):
        ref = OV.interpolate(sd, fr[f:f + 4])
        mse = float(((out[k].double() - ref.double()) ** 2).mean())
        assert 10 * math.log10(1.0 / mse) >= 50.0
