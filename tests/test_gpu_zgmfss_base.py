"""-m gpu: the GMFSS Fortuna base model (the `GMFSS_fortuna` checkpoint: no RIFE sub-model, a 12-channel GridNet head) on the
H100: gmops kernels + fused soft splat under the product's schedule against outputs of the UNMODIFIED reference model
(tests/golden/gmfss_base_*.npz), and the node with that checkpoint selected.  The same schedule is pinned on the CPU through a
host build of the kernels (tests/test_gmfss_base_host.py)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import rife46 as R  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = gmfss_cases("base")


@pytest.fixture(scope="module")
def base_model(pkg):
    """the base model of case seed 0 (the 96x128 goldens), shared by the node tests"""
    from cfi_b200.gmfss import build_gpu_model
    return build_gpu_model(GB.synthetic_state_dicts(CASES["gmfss_base_96x128_t0.5"]["seed"]), 0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_gmfss_base_model_matches_reference(pkg, name):
    from cfi_b200.gmfss import build_gpu_model
    cfg = CASES[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sds = GB.synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous().cuda()
    m = build_gpu_model(sds, 0)
    assert m.variant == "base" and m._engine is None and m.rife is None
    h, w = cfg["h"], cfg["w"]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    i0, i1 = m.o.new(1, 3, ph, pw), m.o.new(1, 3, ph, pw)
    m.o.copy_slice(fr[0:1].contiguous(), i0, 3)
    m.o.copy_slice(fr[1:2].contiguous(), i1, 3)
    state = m.reuse(i0, i1)
    e01 = (state[0].cpu() - torch.from_numpy(g["flow01"])).abs().max().item()
    e10 = (state[1].cpu() - torch.from_numpy(g["flow10"])).abs().max().item()
    em = max((state[k].cpu() - torch.from_numpy(g[n])).abs().max().item() for k, n in ((2, "metric0"), (3, "metric1")))
    out = m.interpolate(fr[0:1].contiguous(), fr[1:2].contiguous(), cfg["t"]).cpu()
    ref = torch.from_numpy(g["out"])
    p = R.psnr(out, ref)
    print(f"{name}: flows within {max(e01, e10):.2e} px, metrics within {em:.2e}, frame PSNR {p:.1f} dB vs the unmodified reference")
    assert out.shape == ref.shape and max(e01, e10) <= 2e-2 and p >= 50.0


def test_gmfss_base_creates_no_rife_engine(pkg, monkeypatch):
    """building the base model never constructs a RIFE engine (so none of its weights or workspace are allocated)"""
    import cfi_b200.engine as E
    from cfi_b200.gmfss import build_gpu_model

    def refuse(*a, **k):
        raise AssertionError("the base model must not build a RIFE engine")

    monkeypatch.setattr(E, "Rife46Engine", refuse)
    m = build_gpu_model(GB.synthetic_state_dicts(0), 0)
    assert m._engine is None and m.rife is None and m.variant == "base"
    with pytest.raises(AssertionError, match="RIFE engine"):     # the union model does build one, through the same name
        build_gpu_model(GW.synthetic_state_dicts(0), 0)


def test_gmfss_base_node(base_model):
    """`GMFSS Fortuna VFI` node with `GMFSS_fortuna`, 2 frames, multiplier 2: the middle frame is the golden's (timestep 0.5),
    the ends pass through bit-exact"""
    import cfi_b200.gmfss_node as GN
    name = "gmfss_base_96x128_t0.5"
    cfg = CASES[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    (out,) = GN.GMFSS_Fortuna_VFI().vfi("GMFSS_fortuna", fr, multiplier=2, _model=base_model)
    assert out.shape == (3, cfg["h"], cfg["w"], 3) and out.dtype == torch.float32 and not out.is_cuda
    assert torch.equal(out[0], fr[0]) and torch.equal(out[2], fr[1])
    p = R.psnr(out[1].permute(2, 0, 1)[None], torch.from_numpy(g["out"]))
    print(f"GMFSS_fortuna node: PSNR {p:.1f} dB")
    assert p >= 50.0


def test_gmfss_base_node_multiplier3_skip(base_model):
    """4 frames, multiplier 3, pair 1 skipped: the node's frames are generic_frame_loop's (frame_loop.py, pinned to the
    reference's loop by tests/test_frame_loop.py) with the CPU oracle of the base model as the middle-frame function - the
    same frame layout, the input frames bit-exact, every middle frame >= 50 dB"""
    import cfi_b200.gmfss_node as GN
    from cfi_b200.frame_loop import generic_frame_loop
    from cfi_b200.node import InterpolationStateList
    cfg = CASES["gmfss_base_96x128_t0.5"]
    sds = GB.synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(4, cfg["h"], cfg["w"], seed=91)
    states = InterpolationStateList([1], True)
    (out,) = GN.GMFSS_Fortuna_VFI().vfi("GMFSS_fortuna", fr, multiplier=3, optional_interpolation_states=states,
                                        _model=base_model)

    def oracle(f0, f1, t):
        with torch.no_grad():
            return GB.interpolate(sds, f0.cpu(), f1.cpu(), float(t))

    ref = generic_frame_loop("GMFSS_Fortuna_VFI", fr.permute(0, 3, 1, 2), 10, 3, oracle, interpolation_states=states,
                             use_timestep=True, dtype=torch.float32).permute(0, 2, 3, 1)
    assert out.shape == ref.shape == (1 + 2 + 1 + 1 + 2 + 1, cfg["h"], cfg["w"], 3)   # f0 m m f1 f2 m m f3
    for i, k in ((0, 0), (3, 1), (4, 2), (7, 3)):
        assert torch.equal(out[i], fr[k]) and torch.equal(ref[i], fr[k])
    ps = [R.psnr(out[i].permute(2, 0, 1)[None], ref[i].permute(2, 0, 1)[None]) for i in (1, 2, 5, 6)]
    print("GMFSS_fortuna node, multiplier 3 with a skip: middle frames vs the oracle " + ", ".join(f"{p:.1f}" for p in ps) + " dB")
    assert min(ps) >= 50.0
