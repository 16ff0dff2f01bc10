"""The WHOLE Sepconv path of the library on the CPU: csrc/sepconv.cu (vfi_sepconv_load + vfi_sepconv_forward: tensor order,
PReLU slopes, buffer sizing, the schedule with its crop-after-conv decoder path), csrc/sepconv_elem.cu and streamconv.cu's
packer + CUDA-core checker kernel, compiled for the host (tests/host_emu) and compared with the output of the unmodified
reference Network (tests/golden/sepconv_net_*.npz, three sizes).  ops.cu's tiled
separable-convolution kernel runs too; only the tensor-core kernel is replaced (by the checker kernel with the same weights)."""
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
from make_golden_sepconv import sepconv_cases, sepconv_inputs  # noqa: E402
from oracle import sepconv as OS  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libsepfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "sepconv_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src] + os.environ.get("VFI_EMU_CXXFLAGS", "").split(),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.mark.parametrize("name", ["sepconv_net_21x30", "sepconv_net_48x64", "sepconv_net_45x54"])
def test_sepconv_whole_path_on_host_matches_reference(emu, pkg, name):
    """21x30: small and odd; 48x64: every encoder row even (no crop in the decoder); 45x54: odd height only, odd rows at
    different pyramid levels in the two axes."""
    from cfi_b200.engine import sepconv_state_dict_names
    cfg = sepconv_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"]).permute(0, 2, 3, 1)
    sd = OS.synthetic_state_dict(cfg["seed"])
    hold = [sd[n].contiguous() for n in sepconv_state_dict_names()]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    fr = sepconv_inputs(cfg).contiguous()
    h, w = cfg["h"], cfg["w"]
    out = torch.zeros(1, h, w, 3)
    he, we = h + h % 2, w + w % 2
    coef = torch.zeros(4, 51, he, we)
    rc = emu.emu_sepconv(ptrs, numel, len(hold), C.c_void_p(fr.data_ptr()), h, w, 3, C.c_void_p(out.data_ptr()),
                         C.c_void_p(coef.data_ptr()))
    emu.vfi_last_error.restype = C.c_char_p
    assert rc >= 1000, (rc, emu.vfi_last_error())
    launches = rc - 1000
    assert 45 <= launches <= 60     # 2 + 4*2+3 + 4*3 + 3*(3 or 4) + 1 + 4*3 + 5
    mse = float(((out.double() - ref.double()) ** 2).mean())
    psnr = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"host emulation of the whole Sepconv path: {launches} launches, PSNR {psnr:.2f} dB, max abs {float((out - ref).abs().max()):.2e}")
    # the output is a normalised blur whose kernels are dominated by the heads' bias (a broken trunk still gives ~41 dB), so
    # the bars are set at the level of fp16 rounding, and the coefficient planes - the trunk's actual product - are
    # compared with the oracle's one by one
    assert psnr >= 80.0, psnr
    assert float((out - ref).abs().max()) < 1e-3
    dbg = {}
    x = fr.permute(0, 3, 1, 2).contiguous()
    OS.network_forward(sd, x[0:1], x[1:2], debug=dbg)
    for k, key in enumerate(("ver1", "ver2", "hor1", "hor2")):
        want = dbg[key][0]
        bias = sd[("netVerone", "netVertwo", "netHorone", "netHortwo")[k] + ".netMain.3.bias"].view(-1, 1, 1)
        err = float((coef[k] - want).abs().max())
        signal = float((want - bias).abs().max())       # what the trunk contributes on top of the bias
        assert err <= 0.02 * signal + 2e-3, (key, err, signal)


def test_sepconv_three_pairs_in_one_call_on_host(emu, pkg):
    """n_pairs = 3 in one vfi_sepconv_forward (per-pair statistics, batch strides of every buffer, a repeated and a reversed
    pair, 4-channel frames): each output equals the oracle run on that pair alone."""
    from cfi_b200.engine import sepconv_state_dict_names
    sd = OS.synthetic_state_dict(5)
    hold = [sd[n].contiguous() for n in sepconv_state_dict_names()]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    h, w = 19, 26
    g = torch.Generator().manual_seed(77)
    fr = torch.rand(3, h, w, 4, generator=g)
    fr[1] = fr[1] * 0.5 + 0.4            # different mean / std per pair
    fr[2] = fr[2] * 0.2
    f0 = (C.c_int32 * 3)(0, 1, 2)
    f1 = (C.c_int32 * 3)(1, 2, 0)
    out = torch.zeros(3, h, w, 3)
    rc = emu.emu_sepconv_pairs(ptrs, numel, len(hold), C.c_void_p(fr.data_ptr()), 3, h, w, 4, f0, f1, 3, C.c_void_p(out.data_ptr()))
    emu.vfi_last_error.restype = C.c_char_p
    assert rc >= 1000, (rc, emu.vfi_last_error())
    x = fr[..., :3].permute(0, 3, 1, 2).contiguous()
    for i, (a, b) in enumerate(((0, 1), (1, 2), (2, 0))):
        ref = OS.network_forward(sd, x[a:a + 1], x[b:b + 1])[0].permute(1, 2, 0)
        err = float((out[i] - ref).abs().max())
        assert err < 2e-3, (i, err)
