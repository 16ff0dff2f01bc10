"""streamconv's CUDA-core checker kernel, plan and product packer on the CPU: csrc/streamconv.cu compiled for the host
(tests/host_emu/streamconv_emu.cpp) and driven through vfi_streamconv_debug_conv with impl = 1, over the case table of
tests/streamconv_util.py, per element against a float64 operator that shares neither the packed weights nor the plan.
This pins the packer's swizzle, the plan's halo / temporal-tap geometry, the launcher's argument checks and the reference
itself; tests/test_gpu_zstreamconv.py runs the same table on the wgmma kernel."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

import streamconv_util as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libstreamconv.so")
    src = os.path.join(ROOT, "tests", "host_emu", "streamconv_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    yield U.bind(C.CDLL(so))
    for (dtype, ext), w in sorted(WORST.items()):
        print(f"checker {dtype} ext {ext}: worst error / bound {w:.3f}")


WORST = {}    # (dtype, ext) -> worst error / bound over the table


@pytest.mark.parametrize("dtype", list(U.DTYPES))
@pytest.mark.parametrize("c", U.CASES, ids=[c["name"] for c in U.CASES])
def test_checker_meets_the_bound(emu, c, dtype):
    tdt = U.DTYPES[dtype][1]
    r = U.check_case(emu, c, tdt, "cpu", impl=1, seed=len(c["name"]))
    key = (dtype, c["ext"])
    WORST[key] = max(WORST.get(key, 0.0), r["ratio16"], r["ratio32"])
    print(f"{c['name']} {dtype}: worst error / bound {r['ratio16']:.3f} (16-bit), {r['ratio32']:.3f} (fp32)")


@pytest.mark.parametrize("name,change,why", U.REFUSALS, ids=[r[0] for r in U.REFUSALS])
def test_refusals_leave_the_output_untouched(emu, name, change, why):
    """Through the checker (impl 1), the launch path the host emulation has: the refusal must come from the launcher's
    argument checks, with their text."""
    U.check_refusal(emu, U.case(name, **change), torch.float16, "cpu", 1, why)


def test_plan_refuses_what_the_kernel_cannot_run(emu):
    for name, change, why in U.REFUSALS:
        if why != U.SHAPE:
            continue
        assert U.plan(emu, U.case(name, **change)) is None, name
    p = U.plan(emu, U.case("ok"))
    assert p == dict(n_cta=64, nsplit=1, a_slots=p["a_slots"], b_slots=p["b_slots"], smem_bytes=p["smem_bytes"],
                     halo_y0=-1, halo_x0=-1)
    assert p["smem_bytes"] <= 232448


def test_plan_splits_and_halo(emu):
    """n_total -> (n_cta, nsplit): the whole layer up to 128 columns, else the widest multiple of 16 that divides it;
    the halo origin of every padding form the case table runs."""
    want = {16: (16, 1), 80: (80, 1), 128: (128, 1), 144: (48, 3), 192: (96, 2), 256: (128, 2), 512: (128, 4)}
    for n, (n_cta, nsplit) in want.items():
        p = U.plan(emu, U.case("n", n_total=n))
        assert (p["n_cta"], p["nsplit"]) == (n_cta, nsplit), n
    for kw, halo in ((dict(ksize=1), (0, 0)), (dict(ksize=2), (0, 0)), (dict(ksize=3), (-1, -1)),
                     (dict(ksize=2, pad_before=1), (-1, -1)), (dict(ksize=2, pad_before=0, pad_before_x=1), (0, -1)),
                     (dict(ksize=2, pad_before=1, pad_before_x=0), (-1, 0))):
        p = U.plan(emu, U.case("pad", **kw))
        assert (p["halo_y0"], p["halo_x0"]) == halo, kw
