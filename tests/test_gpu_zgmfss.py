"""-m gpu: GMFSS Fortuna (union) on the H100 (SURVEY.md section 8 row a11): gmops kernels + fused soft splat + RIFE engine under
the product's schedule against outputs of the UNMODIFIED reference model (tests/golden/gmfss_*.npz), and the node mirror.
The same schedule is pinned on the CPU through a host build of the kernels (tests/test_gmfss_host.py)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import rife46 as R  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(gmfss_cases().keys()))
def test_gmfss_model_matches_reference(pkg, name):
    from cfi_b200.gmfss import build_gpu_model
    cfg = gmfss_cases()[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sds = GW.synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous().cuda()
    m = build_gpu_model(sds, 0)
    h, w = cfg["h"], cfg["w"]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    i0, i1 = m.o.new(1, 3, ph, pw), m.o.new(1, 3, ph, pw)
    m.o.copy_slice(fr[0:1].contiguous(), i0, 3)
    m.o.copy_slice(fr[1:2].contiguous(), i1, 3)
    state = m.reuse(i0, i1)
    e01 = (state[0].cpu() - torch.from_numpy(g["flow01"])).abs().max().item()
    e10 = (state[1].cpu() - torch.from_numpy(g["flow10"])).abs().max().item()
    em = (state[2].cpu() - torch.from_numpy(g["metric0"])).abs().max().item()
    out = m.interpolate(fr[0:1].contiguous(), fr[1:2].contiguous(), cfg["t"]).cpu()
    ref = torch.from_numpy(g["out"])
    p = R.psnr(out, ref)
    print(f"{name}: flows within {max(e01, e10):.2e} px, metric within {em:.2e}, frame PSNR {p:.1f} dB vs the unmodified reference")
    m._engine.close()
    assert out.shape == ref.shape and max(e01, e10) <= 2e-2 and p >= 50.0


def test_gmfss_node(pkg):
    """`GMFSS Fortuna VFI` node, 2 frames, multiplier 2: the middle frame is the golden's (timestep 0.5), the ends pass through"""
    import cfi_b200.gmfss_node as GN
    from cfi_b200.gmfss import build_gpu_model
    name = "gmfss_96x128_t0.5"
    cfg = gmfss_cases()[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    m = build_gpu_model(GW.synthetic_state_dicts(cfg["seed"]), 0)
    (out,) = GN.GMFSS_Fortuna_VFI().vfi("GMFSS_fortuna_union", fr, multiplier=2, _model=m)
    m._engine.close()
    assert out.shape == (3, cfg["h"], cfg["w"], 3) and out.dtype == torch.float32 and not out.is_cuda
    assert torch.equal(out[0], fr[0]) and torch.equal(out[2], fr[1])
    p = R.psnr(out[1].permute(2, 0, 1)[None], torch.from_numpy(g["out"]))
    print(f"GMFSS node: PSNR {p:.1f} dB")
    assert p >= 50.0
