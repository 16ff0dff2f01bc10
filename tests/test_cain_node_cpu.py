"""The CAIN node on the CPU: CAIN_VFI.vfi with a fake engine that runs the CPU oracle (oracle/cain.py) against the
unmodified reference node's outputs (tests/golden/cain_node_*.npz), which checks the output order, the recursive
midpoint bisection (multiplier 4 keeps the shared midpoint, 5 drops it), the skip list and the list multiplier; the
oracle against the model goldens; the node surface and registration; the engine's state-dict spec against the
oracle's; the MAC count and the geometry, including the frames the reference cannot pad."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_cain import cain_cases, cain_inputs, case_state_dict  # noqa: E402
from oracle import cain as OC  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


class OracleEngine:
    """CainEngine.forward on the CPU; counts the calls."""
    torch_device = torch.device("cpu")

    def __init__(self, sd):
        self.sd = sd
        self.calls = 0

    def forward(self, img0, img1):
        self.calls += 1
        with torch.no_grad():
            return OC.forward(self.sd, img0, img1)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


@pytest.mark.parametrize("name", [k for k, v in cain_cases().items() if v["kind"] == "net"])
def test_oracle_matches_reference_model(name):
    cfg = cain_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    x = cain_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        out = OC.forward(case_state_dict(cfg), x[0:1], x[1:2])
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-4


# model calls of each node case: bisecting n = m - 1 costs c(n) = 1 + 2 c(n // 2), c(1) = 1 (m 4: 3 calls, m 5: 7, of
# which the shared midpoint is dropped); a skipped pair none; [3, 0] on four frames: 3 + 0 + 1 (the list padded with 2)
CALLS = {"cain_node_m2": 2, "cain_node_m4": 3, "cain_node_m5": 7, "cain_node_skip": 2, "cain_node_mlist": 4,
         "cain_node_rgba": 1}


@pytest.mark.parametrize("name", [k for k, v in cain_cases().items() if v["kind"] == "node"])
def test_node_matches_reference_node(pkg, name):
    import cfi_b200.cain_node as CN
    cfg = cain_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = OracleEngine(case_state_dict(cfg))
    st = None if cfg["states"] is None else CN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    (out,) = CN.CAIN_VFI().vfi("pretrained_cain.pth", cain_inputs(cfg), multiplier=cfg["multiplier"],
                               optional_interpolation_states=st, _engine=eng)
    assert out.shape == ref.shape
    assert psnr(out, ref) >= 80.0
    assert eng.calls == CALLS[name]


def test_node_surface_and_registration(pkg):
    import cfi_b200 as P
    import cfi_b200.cain_node as CN
    assert P.NODE_CLASS_MAPPINGS["CAIN VFI"] is CN.CAIN_VFI
    assert P.NODE_DISPLAY_NAME_MAPPINGS["CAIN VFI"] == "CAIN VFI (H100 native)"
    it = CN.CAIN_VFI.INPUT_TYPES()
    req = it["required"]
    assert req["ckpt_name"][0] == OC.CKPT_NAMES
    assert req["clear_cache_after_n_frames"][1] == {"default": 10, "min": 1, "max": 1000}
    assert req["multiplier"][1] == {"default": 2, "min": 2, "max": 1000}
    assert list(it["optional"]) == ["optional_interpolation_states"]
    assert (CN.CAIN_VFI.RETURN_TYPES, CN.CAIN_VFI.FUNCTION) == (("IMAGE",), "vfi")


def test_node_reads_the_released_checkpoint_form(pkg, tmp_path, monkeypatch):
    """{"state_dict": {"module.<name>": tensor}} from <ckpts>/cain/, prefix stripped, handed to the engine."""
    import cfi_b200.cain_node as CN
    sd = OC.synthetic_state_dict(0)
    (tmp_path / "cain").mkdir()
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, tmp_path / "cain" / "pretrained_cain.pth")
    monkeypatch.setenv("VFI_CKPT_DIR", str(tmp_path))
    seen = {}

    class Probe:
        def __init__(self, state_dict, device=0, dtype="float32"):
            seen.update(state_dict)

    monkeypatch.setattr(CN, "CainEngine", Probe)
    monkeypatch.setattr(CN.torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(CN, "_model_cache", {})
    CN._load_engine("pretrained_cain.pth")
    assert list(seen) == [n for n, _ in OC.state_dict_spec()]
    assert all(torch.equal(seen[k], sd[k]) for k in sd)


def test_engine_spec_is_the_reference_state_dict(pkg):
    from cfi_b200.engine import cain_state_dict_spec
    assert cain_state_dict_spec() == OC.state_dict_spec()
    assert len(cain_state_dict_spec()) == 494
    n = sum(math.prod(s) for _, s in OC.state_dict_spec())
    assert round(n / 1e6, 2) == 42.78


def test_mac_count_of_the_issue_figure():
    assert round(OC.cain_macs(1080, 1920) / 1e9, 2) == 1467.67


def test_geometry():
    assert OC.geometry(1080, 1920) == dict(hp=1152, wp=1920, gh=144, gw=240, top=36, left=0)
    assert OC.geometry(130, 135) == dict(hp=256, wp=256, gh=32, gw=32, top=63, left=60)
    assert OC.geometry(64, 40) is None      # 44 columns of padding on the right of a 40-column frame
    assert OC.geometry(44, 200) is not None and OC.geometry(43, 200) is None
