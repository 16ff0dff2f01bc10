"""The IFRNet node on the CPU: IFRNet_VFI.vfi with a fake engine that runs the CPU oracle (oracle/ifrnet.py) against the
unmodified reference node's outputs (tests/golden/ifrnet_node_*.npz), which checks the loop schedule and the reference's
argument swap (the timestep is the resize factor, the node's scale_factor is embt); the oracle against the model goldens;
the node surface and registration; the engine's state-dict spec against the oracle's."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_ifrnet import case_state_dict, ifrnet_cases, ifrnet_inputs  # noqa: E402
from oracle import ifrnet as OI  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


class OracleEngine:
    """IfrnetEngine.forward on the CPU; records (t, embt) of every call."""
    torch_device = torch.device("cpu")

    def __init__(self, sd):
        self.sd = sd
        self.calls = []

    def forward(self, img0, img1, t, embt):
        self.calls.append((t, embt))
        with torch.no_grad():
            return OI.forward(self.sd, img0, img1, t, embt)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


@pytest.mark.parametrize("name", [k for k, v in ifrnet_cases().items() if v["kind"] == "net"])
def test_oracle_matches_reference_model(name):
    cfg = ifrnet_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    x = ifrnet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        out = OI.forward(case_state_dict(cfg), x[0:1], x[1:2], cfg["t"], cfg["embt"])
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-4


@pytest.mark.parametrize("name", [k for k, v in ifrnet_cases().items() if v["kind"] == "node"])
def test_node_matches_reference_node(pkg, name):
    import cfi_b200.ifrnet_node as IN
    cfg = ifrnet_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = OracleEngine(case_state_dict(cfg))
    st = None if cfg["states"] is None else IN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    (out,) = IN.IFRNet_VFI().vfi(cfg["ckpt"], ifrnet_inputs(cfg), multiplier=cfg["multiplier"],
                                 scale_factor=cfg["scale_factor"], optional_interpolation_states=st, _engine=eng)
    assert out.shape == ref.shape
    assert psnr(out, ref) >= 80.0
    assert all(e == cfg["scale_factor"] for _, e in eng.calls)  # embt is always the node's scale_factor
    if cfg["multiplier"] == 3:
        assert [t for t, _ in eng.calls] == [1 / 3, 2 / 3] * (cfg["n"] - 1)


def test_node_surface_and_registration(pkg):
    import cfi_b200 as P
    import cfi_b200.ifrnet_node as IN
    assert P.NODE_CLASS_MAPPINGS["IFRNet VFI"] is IN.IFRNet_VFI
    assert P.NODE_DISPLAY_NAME_MAPPINGS["IFRNet VFI"] == "IFRNet VFI (H100 native)"
    req = IN.IFRNet_VFI.INPUT_TYPES()["required"]
    assert req["ckpt_name"][0] == OI.CKPT_NAMES
    assert req["scale_factor"] == ([0.25, 0.5, 1.0, 2.0, 4.0], {"default": 1.0})
    assert req["multiplier"][1] == {"default": 2, "min": 2, "max": 1000}
    assert (IN.IFRNet_VFI.RETURN_TYPES, IN.IFRNet_VFI.FUNCTION) == (("IMAGE",), "vfi")


@pytest.mark.parametrize("variant", ["S", "L"])
def test_engine_spec_is_the_reference_state_dict(pkg, variant):
    from cfi_b200.engine import ifrnet_state_dict_spec
    assert ifrnet_state_dict_spec(variant) == OI.state_dict_spec(variant)
    assert len(ifrnet_state_dict_spec(variant)) == 104


def test_mac_count_of_the_issue_figures():
    assert round(OI.ifrnet_macs("S", 1080, 1920, 0.5) / 1e9, 2) == 57.36
    assert round(OI.ifrnet_macs("L", 1080, 1920, 0.5) / 1e9, 2) == 400.02
