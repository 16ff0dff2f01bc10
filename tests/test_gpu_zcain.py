"""-m gpu: CAIN on the H100.

In this process: every streamconv layer kind CAIN runs (headConv on two 192-channel sources of one 384-channel tensor,
RCAB conv1 with LeakyReLU(0.2), conv2 / tailConv without activation, the group tail conv with the group input as ext 1
residual) through the generic hook vfi_streamconv_debug_conv, wgmma kernel and CUDA-core checker, fp16 and bf16, on a
ragged small grid and on the bordered 1080p grid (146 x 242), per element within the float64 bound of
tests/streamconv_util.py; and the plan of every one of CAIN's 127 layers (vfi_cain_layer_plan) equals the generic hook's
plan of its case.

In a subprocess (tools/cain_gpu_check.py; a kernel trap must not poison the CUDA context of the tests sharing this
pytest process): the element-wise kernels against torch, the model goldens on the checker and on the wgmma kernel
(PSNR >= 50 dB against the unmodified reference), the node goldens, the refusal of a frame too small to pad, and with
VFI_PARENT_SRC naming a checkout of the parent commit, FILM, Sepconv, FLAVR and IFRNet outputs bit-identical to that
build's."""
import os
import subprocess
import sys

import pytest
import torch

import streamconv_util as U

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KINDS = {
    "head": dict(c0=192, pitch0=384, c1=192, off1=192, pitch1=384, n_total=192, act=0),
    "rcab_conv1": dict(c0=192, n_total=192, act=1),
    "rcab_conv2": dict(c0=192, n_total=192, act=0),
    "group_tail": dict(c0=192, n_total=192, ext=1, act=0, slope=1.0, res="sep"),
}
# layer ids of each kind (csrc/cain.cu): 0 headConv; 1 + 25 g + 2 r (+ 1) RCAB conv1 (conv2); 1 + 25 g + 24 the group
# tail; 126 tailConv, planned as conv2
IDS = {"head": [0],
       "rcab_conv1": [1 + 25 * g + 2 * r for g in range(5) for r in range(12)],
       "rcab_conv2": [2 + 25 * g + 2 * r for g in range(5) for r in range(12)] + [126],
       "group_tail": [25 * (g + 1) for g in range(5)]}
GRIDS = {"ragged": dict(B=1, H=21, W=13), "1080p": dict(B=1, H=146, W=242)}


@pytest.fixture(scope="module")
def L(pkg):
    from cfi_b200._lib import lib
    return U.bind(lib())


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("dtype", list(U.DTYPES))
@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("kind", list(KINDS))
def test_layer_kind_meets_the_bound(L, kind, grid, dtype, impl):
    c = U.case(f"cain_{kind}_{grid}", **KINDS[kind], **GRIDS[grid])
    r = U.check_case(L, c, U.DTYPES[dtype][1], "cuda", impl, seed=len(kind) + impl,
                     stream=torch.cuda.current_stream().cuda_stream)
    print(f"{c['name']} {dtype} impl {impl}: worst error / bound {r['ratio16']:.3f}")


def test_every_layer_is_planned_as_its_case(L, pkg):
    from cfi_b200.engine import CainEngine
    from oracle import cain as OC
    eng = CainEngine(OC.synthetic_state_dict(0), 0, "float16")
    assert sorted(i for ids in IDS.values() for i in ids) == list(range(127))
    for kind, ids in IDS.items():
        q = U.plan(L, U.case(kind, **KINDS[kind]))
        assert q is not None, kind
        for i in ids:
            p = eng.layer_plan(i)
            k = KINDS[kind]
            assert (p["c0"], p["c1"], p["n_total"], p["ksize"]) == (k["c0"], k.get("c1", 0), 192, 3), (kind, i, p)
            assert (p["act"], p["ext"]) == (k["act"], k.get("ext", 0)), (kind, i, p)
            for key in ("n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes"):
                assert p[key] == q[key], (kind, i, key, p[key], q[key])
    print("CAIN plans:", {kind: eng.layer_plan(ids[0]) for kind, ids in IDS.items()})
    eng.close()


def test_cain_gpu_check_subprocess():
    cmd = [sys.executable, os.path.join(ROOT, "tools", "cain_gpu_check.py")]
    if os.environ.get("VFI_PARENT_SRC"):
        cmd += ["--parent-src", os.environ["VFI_PARENT_SRC"]]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(r.stdout[-8000:])
    tail = (r.stdout[-8000:] + "\n--- stderr ---\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
