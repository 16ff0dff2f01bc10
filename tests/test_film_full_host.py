"""The WHOLE FILM path of the library on the CPU: csrc/film.cu (vfi_film_load + vfi_film_forward: 82 tensors, channel maps,
buffer sizing, the ~190-launch schedule), csrc/film_elem.cu and streamconv.cu's packer + CUDA-core checker kernel, compiled
for the host (tests/host_emu, one host thread per emulated block) and compared with the output of the unmodified reference
Interpolator (tests/golden/film_net_64x64_rand.npz, white-noise frames outside [0, 1]).  The tensor-core kernel is not part of
this; tools/film_gpu_check.py compares it with the same checker kernel on the GPU."""
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
from make_golden_film import film_cases, film_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libfilmfull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "film_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src] + os.environ.get("VFI_EMU_CXXFLAGS", "").split(),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.mark.parametrize("name", ["film_net_64x64_rand", "film_net_72x104"])   # the second: odd level sizes down the pyramid
def test_film_whole_path_on_host_matches_reference(emu, pkg, name):
    from cfi_b200.engine import film_state_dict_names
    cfg = film_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"]).permute(0, 2, 3, 1)
    sd = OF.synthetic_state_dict(cfg["seed"], cfg["flow_gain"])
    hold = [sd[n].contiguous() for n in film_state_dict_names()]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    fr = film_inputs(cfg).contiguous()
    out = torch.zeros(1, cfg["h"], cfg["w"], 3)
    emu.vfi_last_error.restype = C.c_char_p
    h, w = cfg["h"], cfg["w"]
    nflow = sum((h >> l) * (w >> l) * 2 for l in range(5))
    flows = torch.zeros(2 * nflow)
    rc = emu.emu_film(ptrs, numel, len(hold), C.c_void_p(fr.data_ptr()), h, w, 3, 0, C.c_void_p(out.data_ptr()),
                      C.c_void_p(flows.data_ptr()), 0)
    assert rc >= 1000, (rc, emu.vfi_last_error())
    mse = float(((out.double() - ref.double()) ** 2).mean())
    psnr = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"host emulation of the whole FILM path: {rc - 1000} launches, PSNR {psnr:.2f} dB, "
          f"max abs {float((out - ref).abs().max()):.2e}")
    # the flow pyramids (fp32 recurrence on fp16 features) against the reference's debug_forward output, level by level
    gold = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    off = 0
    worst = 0.0
    for key in ("fwd_flow", "bwd_flow"):
        for l in range(5):
            n = (h >> l) * (w >> l) * 2
            got = flows[off:off + n].view(h >> l, w >> l, 2)
            want = torch.from_numpy(gold[f"{key}{l}"])[0].permute(1, 2, 0)
            worst = max(worst, float((got - want).abs().max()))
            off += n
    print(f"flow pyramids: max abs error {worst:.4f} px")
    assert worst <= 0.05, worst
    assert rc - 1000 == 192
    assert psnr >= 55.0, psnr   # fp16 operands / activations vs the fp32 reference (GPU, same checker: 64.9 dB at 72x104)


def test_film_two_pairs_in_one_call_on_host(emu, pkg):
    """B = 2 (images indexed k * B + pair through every buffer of the schedule) equals the single-pair call, bit for bit; frames have 4 channels (the alpha channel is skipped by gather_rgb)."""
    from cfi_b200.engine import film_state_dict_names
    sd = OF.synthetic_state_dict(5)
    hold = [sd[n].contiguous() for n in film_state_dict_names()]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    fr = torch.cat([OF.synthetic_clip(3, 64, 64, seed=9), torch.ones(3, 64, 64, 1)], -1).contiguous()
    both = torch.zeros(2, 64, 64, 3)
    emu.vfi_last_error.restype = C.c_char_p
    assert emu.emu_film_batch2(ptrs, numel, len(hold), C.c_void_p(fr.data_ptr()), 64, 64, 4, C.c_void_p(both.data_ptr())) == 0, \
        emu.vfi_last_error()
    for i in (1,):   # the second pair is the one whose images sit at the non-trivial indices (1 and B + 1)
        one = torch.zeros(1, 64, 64, 3)
        pair = fr[i:i + 2].contiguous()
        rc = emu.emu_film(ptrs, numel, len(hold), C.c_void_p(pair.data_ptr()), 64, 64, 4, 1, C.c_void_p(one.data_ptr()), None,
                          0)
        assert rc >= 1000, emu.vfi_last_error()
        assert torch.equal(both[i], one[0]), i
