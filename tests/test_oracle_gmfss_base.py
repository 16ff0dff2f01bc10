"""Pin oracle/gmfss_base.py (GMFSS_Fortuna_arch.py, the `GMFSS_fortuna` checkpoint - no
IFNet, a 12-channel GridNet head) to outputs of the unmodified reference model (tests/golden/gmfss_base_*.npz, made by
`tools/make_golden_gmfss.py --variant base`), and keep its seeded weights in step with the reference's state_dict layout
(tests/golden/gmfss_base_spec.json)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmflow as GF  # noqa: E402
from oracle import gmfss as OG  # noqa: E402
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import rife46 as R  # noqa: E402

CASES = gmfss_cases("base")


def _case(name):
    cfg = CASES[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sds = GB.synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous()
    h, w = cfg["h"], cfg["w"]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64      # CommonModelInference.forward, gmfss_fortuna/__init__.py:41-47
    i0, i1 = F.pad(fr[0:1], (0, pw - w, 0, ph - h)), F.pad(fr[1:2], (0, pw - w, 0, ph - h))
    return cfg, g, sds, fr, i0, i1


def _count(sd):
    return sum(v.numel() for v in sd.values() if v.dtype == torch.float32)


def test_base_weights_match_the_reference_layout():
    """names / shapes / dtypes of the seeded base weights are the spec's (written from the reference's four state_dicts); the
    base GridNet is union's with residual_model_head0 (9 -> 64) replaced by residual_model_head (12 -> 64)"""
    spec = GB.load_spec()
    assert tuple(spec) == GB.NETS == ("flownet", "metricnet", "feat_ext", "fusionnet")
    a, b = GB.synthetic_state_dicts(0), GB.synthetic_state_dicts(0)
    assert tuple(a) == GB.NETS
    for net in GB.NETS:
        assert [(k, list(v.shape), str(v.dtype)) for k, v in a[net].items()] == [tuple(e) for e in spec[net]], net
        assert all(torch.equal(a[net][k], b[net][k]) for k in a[net])
    union_spec = GW.load_spec()
    ucount = {net: sum(int(np.prod(s)) for _, s, d in union_spec[net] if d == "torch.float32") for net in union_spec}
    for net in ("flownet", "metricnet", "feat_ext"):
        assert [tuple(e) for e in spec[net]] == [tuple(e) for e in union_spec[net]], net     # same architectures
        assert _count(a[net]) == ucount[net]
    assert _count(a["fusionnet"]) == ucount["fusionnet"] + 3 * 64 * 9
    fus = dict((n, tuple(s)) for n, s, _ in spec["fusionnet"])
    assert fus["residual_model_head.1.weight"] == (64, 12, 3, 3) and "residual_model_head0.1.weight" not in fus
    assert 4.6e6 < _count(a["flownet"]) < 4.8e6 and 7.8e6 < _count(a["fusionnet"]) < 7.9e6
    c = GB.synthetic_state_dicts(1)
    assert not torch.equal(a["fusionnet"]["residual_model_head.1.weight"], c["fusionnet"]["residual_model_head.1.weight"])
    u = GW.synthetic_state_dicts(0)
    assert not torch.equal(a["flownet"]["backbone.conv1.weight"], u["flownet"]["backbone.conv1.weight"])   # own seeds


@pytest.mark.parametrize("name", sorted(CASES))
def test_base_goldens_are_sane(name):
    cfg, g, *_ = _case(name)
    assert g["out"].shape == (1, 3, cfg["h"], cfg["w"]) and np.isfinite(g["out"]).all()
    assert g["out"].min() >= 0.0 and g["out"].max() <= 1.0 and g["out"].std() > 0.05
    ph, pw = ((cfg["h"] - 1) // 64 + 1) * 64, ((cfg["w"] - 1) // 64 + 1) * 64
    for k in ("flow01", "flow10"):
        assert g[k].shape == (1, 2, ph // 2, pw // 2) and np.isfinite(g[k]).all() and np.abs(g[k]).max() > 1.0
    for k in ("metric0", "metric1"):
        assert g[k].shape == (1, 1, ph // 2, pw // 2) and np.isfinite(g[k]).all()


@pytest.mark.parametrize("name", sorted(CASES))
def test_base_downstream_of_gmflow_matches_reference(name):
    cfg, g, sds, fr, i0, i1 = _case(name)
    h, w = cfg["h"], cfg["w"]
    f01, f10 = torch.from_numpy(g["flow01"]), torch.from_numpy(g["flow10"])
    with torch.no_grad():
        m0, m1, f1, f2 = OG.reuse_from_flows(sds, i0, i1, f01, f10)
        assert (m0 - torch.from_numpy(g["metric0"])).abs().max().item() <= 1e-4
        assert (m1 - torch.from_numpy(g["metric1"])).abs().max().item() <= 1e-4
        out = GB.inference(sds, i0, i1, f01, f10, m0, m1, f1, f2, cfg["t"])[:, :, :h, :w]
    ref = torch.from_numpy(g["out"])
    assert (out - ref).abs().max().item() <= 2e-4 and R.psnr(out, ref) >= 50.0


@pytest.mark.parametrize("name", sorted(CASES))
def test_base_gmflow_matches_reference_flows(name):
    cfg, g, sds, fr, i0, i1 = _case(name)
    h0 = F.interpolate(i0, scale_factor=0.5, mode="bilinear", align_corners=False)
    h1 = F.interpolate(i1, scale_factor=0.5, mode="bilinear", align_corners=False)
    with torch.no_grad():
        f01, f10 = GF.gmflow(sds["flownet"], h0, h1), GF.gmflow(sds["flownet"], h1, h0)
    assert f01.shape == g["flow01"].shape
    assert (f01 - torch.from_numpy(g["flow01"])).abs().max().item() <= 1e-3        # pixels
    assert (f10 - torch.from_numpy(g["flow10"])).abs().max().item() <= 1e-3


@pytest.mark.parametrize("name", sorted(CASES))
def test_base_whole_model_matches_reference(name):
    cfg, g, sds, fr, *_ = _case(name)
    with torch.no_grad():
        out = GB.interpolate(sds, fr[0:1], fr[1:2], cfg["t"])
    ref = torch.from_numpy(g["out"])
    p = R.psnr(out, ref)
    print(f"{name}: base oracle PSNR {p:.1f} dB, max abs {(out - ref).abs().max().item():.2e}")
    assert (out - ref).abs().max().item() <= 5e-4 and p >= 50.0

