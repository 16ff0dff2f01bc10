"""-m gpu: IFUnet on the H100.

In this process: every streamconv layer kind IFUnet runs (the space-to-depth stride-2 convs, 3x3 convs with per-channel
PReLU up to 512 channels, the ConvTranspose2d phases, UpConv conv1 on two sources, the fp32 flow / mask / decode columns,
the 1x1 mask convs at 2304 and 144 outputs, the RDB convs on the growth tensor with LeakyReLU and the RDB conv5 with its
residual) through the generic hook vfi_streamconv_debug_conv, wgmma kernel and CUDA-core checker, fp16 and bf16, per
element within the float64 bound of tests/streamconv_util.py, one of them on IFBlock 0's 1080p grid (68 x 120); and
the plan of every one of IFUnet's 194 layers (vfi_ifunet_layer_plan) equals the generic hook's plan of the same layer.

In a subprocess (tools/ifunet_gpu_check.py; a kernel trap must not poison the CUDA context of the tests sharing this
pytest process): the element-wise kernels against torch, the model goldens on the checker and on the wgmma kernel
(PSNR >= 50 dB against the unmodified reference), the node goldens, the refusal of the scale factors the reference
cannot run, and with VFI_PARENT_SRC naming a checkout of the parent commit, RIFE, FILM, Sepconv, FLAVR, IFRNet and CAIN
outputs bit-identical to that build's."""
import os
import subprocess
import sys

import pytest
import torch

import streamconv_util as U

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KINDS = {
    "unet1_s2d": dict(ksize=2, c0=128, n_total=64, act=0, ext=2, pad_before=1),
    "prelu_64": dict(c0=64, n_total=64, act=0, ext=2),
    "prelu_512": dict(c0=512, n_total=512, act=0, ext=2),
    "s2d_1024": dict(ksize=2, c0=1024, n_total=512, act=0, ext=2, pad_before=1),
    "convT_phase": dict(ksize=2, c0=512, n_total=256, act=0, ext=2, pad_before=0, pad_before_x=1),
    "upconv_conv1": dict(c0=256, c1=256, n_total=256, act=0, ext=2),
    "flowconv": dict(c0=256, n_total=16, act=0, ext=2, n_f32=4),
    "mask_x16": dict(ksize=1, c0=256, n_total=2304, act=0, ext=0),
    "mask_x4": dict(ksize=1, c0=64, n_total=144, act=0, ext=0),
    "rdb_conv4": dict(c0=64, c1=128, n_total=32, act=1, ext=0),
    "rdb_conv5": dict(c0=64, c1=128, n_total=64, act=0, ext=2, res="sep"),
    "lastconv_phase": dict(ksize=2, c0=256, n_total=16, act=0, ext=2, n_f32=4, pad_before=1, pad_before_x=0),
}
GRIDS = {"ragged": dict(B=2, H=21, W=13)}
BIG = ("prelu_256_1080p", dict(c0=256, n_total=256, act=0, ext=2, B=1, H=68, W=120))


@pytest.fixture(scope="module")
def L(pkg):
    from cfi_b200._lib import lib
    return U.bind(lib())


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("dtype", list(U.DTYPES))
@pytest.mark.parametrize("kind", list(KINDS) + [BIG[0]])
def test_layer_kind_meets_the_bound(L, kind, dtype, impl):
    kw = dict(BIG[1]) if kind == BIG[0] else dict(KINDS[kind], **GRIDS["ragged"])
    c = U.case(f"ifunet_{kind}", **kw)
    r = U.check_case(L, c, U.DTYPES[dtype][1], "cuda", impl, seed=len(kind) + impl,
                     stream=torch.cuda.current_stream().cuda_stream)
    print(f"{c['name']} {dtype} impl {impl}: worst error / bound {r['ratio16']:.3f}")


def test_every_layer_is_planned_as_the_generic_hook_plans_it(L, pkg):
    from cfi_b200.engine import IfunetEngine
    from oracle import ifunet as OU
    eng = IfunetEngine(OU.synthetic_state_dict(0), 0, "float16")
    seen = set()
    for i in range(194):
        p = eng.layer_plan(i)
        c = U.case(f"layer{i}", ksize=p["ksize"], c0=p["c0"], c1=p["c1"], n_total=p["n_total"], act=p["act"],
                   ext=p["ext"], n_f32=p["n_f32"], pad_before=p["pad_before"], pad_before_x=p["pad_before_x"])
        q = U.plan(L, c)
        assert q is not None, (i, p)
        for key in ("n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes"):
            assert p[key] == q[key], (i, key, p[key], q[key])
        seen.add((p["ksize"], p["c0"], p["c1"], p["n_total"], p["ext"], p["act"], p["n_f32"]))
    # the kinds above are among the layers' own shapes
    for k in ("unet1_s2d", "s2d_1024", "upconv_conv1", "flowconv", "mask_x16", "mask_x4", "rdb_conv4", "rdb_conv5",
              "lastconv_phase"):
        c = U.case(k, **KINDS[k])
        assert (c["ksize"], c["c0"], c["c1"], c["n_total"], c["ext"], c["act"], c["n_f32"]) in seen, k
    eng.close()


def test_ifunet_gpu_check_subprocess():
    cmd = [sys.executable, os.path.join(ROOT, "tools", "ifunet_gpu_check.py")]
    if os.environ.get("VFI_PARENT_SRC"):
        cmd += ["--parent-src", os.environ["VFI_PARENT_SRC"]]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
    print(r.stdout[-8000:])
    tail = (r.stdout[-8000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
