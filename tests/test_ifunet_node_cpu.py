"""The IFUnet node on the CPU: IFUnet_VFI.vfi with a fake engine that runs the CPU oracle (oracle/ifunet.py) against the
unmodified reference node's outputs (tests/golden/ifunet_node_*.npz), which checks the output order, the timesteps, the
skip list, the list multiplier, 4-channel frames and the arguments each call passes; the oracle against the model
goldens; the node surface, defaults and registration; the engine's state-dict spec against the oracle's and the
reference's; the MAC count; and the scale_factor values at which the reference raises, through the library's own
geometry (vfi_ifunet_geometry) and the node."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_ifunet import case_state_dict, ifunet_cases, ifunet_inputs  # noqa: E402
from oracle import ifunet as OU  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


class OracleEngine:
    """IfunetEngine.forward on the CPU: the oracle, behind the library's geometry check; records every call."""
    torch_device = torch.device("cpu")

    def __init__(self, sd):
        self.sd = sd
        self.calls = []

    def forward(self, img0, img1, timestep=0.5, scale=1.0, ensemble=True):
        from cfi_b200.engine import ifunet_geometry
        self.calls.append((timestep, scale, ensemble))
        ifunet_geometry(img0.shape[2], img0.shape[3], scale)   # raises where the reference raises
        with torch.no_grad():
            return OU.forward(self.sd, img0, img1, timestep, scale, ensemble)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


@pytest.mark.parametrize("name", [k for k, v in ifunet_cases().items() if v["kind"] == "net"])
def test_oracle_matches_reference_model(name):
    cfg = ifunet_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    x = ifunet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        out = OU.forward(case_state_dict(cfg), x[0:1], x[1:2], cfg["t"], cfg["scale"], cfg["ensemble"])
    assert out.shape == ref.shape
    assert float((out - ref).abs().max()) <= 1e-4


# the calls of each node case: (timestep, scale, ensemble) per interpolated frame, in order
def _want_calls(cfg):
    m, n = cfg["multiplier"], cfg["n"]
    skip = set(cfg["states"][0]) if cfg["states"] else set()
    ts = []
    if isinstance(m, list):
        ms = m + [2] * (n - 1 - len(m))
        for k in ms:
            ts += [j / k for j in range(1, k)] if k else []
    else:
        for i in range(n - 1):
            if i not in skip:
                ts += [j / m for j in range(1, m)]
    return [(t, cfg["scale"], cfg["ensemble"]) for t in ts]


@pytest.mark.parametrize("name", [k for k, v in ifunet_cases().items() if v["kind"] == "node"])
def test_node_matches_reference_node(pkg, name):
    import cfi_b200.ifunet_node as UN
    cfg = ifunet_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = OracleEngine(case_state_dict(cfg))
    st = None if cfg["states"] is None else UN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    (out,) = UN.IFUnet_VFI().vfi("IFUNet.pth", ifunet_inputs(cfg), multiplier=cfg["multiplier"],
                                 scale_factor=cfg["scale"], ensemble=cfg["ensemble"], optional_interpolation_states=st,
                                 _engine=eng)
    assert out.shape == ref.shape
    assert psnr(out, ref) >= 80.0
    assert eng.calls == _want_calls(cfg)


def test_node_defaults_reach_the_engine(pkg):
    """Only the required arguments: multiplier 2, scale_factor 1.0, ensemble True, timestep 0.5 as a Python float."""
    import cfi_b200.ifunet_node as UN
    eng = OracleEngine(OU.synthetic_state_dict(0))
    fr = ifunet_inputs(dict(kind="node", n=2, h=40, w=56, clip_seed=3))
    (out,) = UN.IFUnet_VFI().vfi("IFUNet.pth", fr, _engine=eng)
    assert out.shape == (3, 40, 56, 3)
    assert eng.calls == [(0.5, 1.0, True)]
    assert all(type(v) is float for v in eng.calls[0][:2]) and type(eng.calls[0][2]) is bool


@pytest.mark.parametrize("scale", [0.25, 0.7, 1.2])
def test_node_raises_where_the_reference_raises(pkg, scale):
    import cfi_b200.ifunet_node as UN
    from cfi_b200.engine import ifunet_geometry
    eng = OracleEngine(OU.synthetic_state_dict(0))
    fr = ifunet_inputs(dict(kind="node", n=2, h=100, w=150, clip_seed=4))
    with pytest.raises(RuntimeError, match="the reference raises"):
        UN.IFUnet_VFI().vfi("IFUNet.pth", fr, scale_factor=scale, _engine=eng)
    with pytest.raises(RuntimeError):
        ifunet_geometry(100, 150, scale)


def test_library_geometry_is_the_reference_table(pkg):
    """vfi_ifunet_geometry runs / refuses exactly where the unmodified reference ran / raised
    (tests/golden/ifunet_spec.json, recorded by tools/make_golden_ifunet.py), and agrees with the oracle's sizes."""
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import ifunet_geometry
    table = json.load(open(os.path.join(GOLD, "ifunet_spec.json")))["scale_factor_table"]
    for size, row in table.items():
        h, w = map(int, size.split("x"))
        for s, outcome in row.items():
            g = OU.geometry(h, w, float(s))
            if outcome == "runs":
                got = ifunet_geometry(h, w, float(s))
                assert (got["hp"], got["wp"]) == (g["hp"], g["wp"]) and got["levels"] == g["levels"], (size, s)
            else:
                assert g is None
                with pytest.raises(VfiError):
                    ifunet_geometry(h, w, float(s))
    assert ifunet_geometry(1080, 1920, 1.0)["levels"][4] == (68, 120)


def test_node_surface_and_registration(pkg):
    import cfi_b200 as P
    import cfi_b200.ifunet_node as UN
    assert P.NODE_CLASS_MAPPINGS["IFUnet VFI"] is UN.IFUnet_VFI
    assert P.NODE_DISPLAY_NAME_MAPPINGS["IFUnet VFI"] == "IFUnet VFI (H100 native)"
    it = UN.IFUnet_VFI.INPUT_TYPES()
    req = it["required"]
    assert list(req) == ["ckpt_name", "frames", "clear_cache_after_n_frames", "multiplier", "scale_factor", "ensemble"]
    assert req["ckpt_name"][0] == OU.CKPT_NAMES
    assert req["clear_cache_after_n_frames"][1] == {"default": 10, "min": 1, "max": 1000}
    assert req["multiplier"][1] == {"default": 2, "min": 2, "max": 1000}
    assert req["scale_factor"] == ("FLOAT", {"default": 1.0, "min": 0.1, "max": 100, "step": 0.1})
    assert req["ensemble"] == ("BOOLEAN", {"default": True})
    assert list(it["optional"]) == ["optional_interpolation_states"]
    assert (UN.IFUnet_VFI.RETURN_TYPES, UN.IFUnet_VFI.FUNCTION) == (("IMAGE",), "vfi")


def test_node_reads_the_raw_checkpoint(pkg, tmp_path, monkeypatch):
    """A raw state dict from <ckpts>/ifunet/, handed to the engine unchanged."""
    import cfi_b200.ifunet_node as UN
    sd = OU.synthetic_state_dict(0)
    (tmp_path / "ifunet").mkdir()
    torch.save(sd, tmp_path / "ifunet" / "IFUNet.pth")
    monkeypatch.setenv("VFI_CKPT_DIR", str(tmp_path))
    seen = {}

    class Probe:
        def __init__(self, state_dict, device=0, dtype="float32"):
            seen.update(state_dict)

    monkeypatch.setattr(UN, "IfunetEngine", Probe)
    monkeypatch.setattr(UN.torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(UN, "_model_cache", {})
    UN._load_engine("IFUNet.pth")
    assert list(seen) == [n for n, _ in OU.state_dict_spec()]
    assert all(torch.equal(seen[k], sd[k]) for k in sd)


def test_engine_spec_is_the_reference_state_dict(pkg):
    from cfi_b200.engine import ifunet_state_dict_spec
    assert ifunet_state_dict_spec() == OU.state_dict_spec()
    assert len(ifunet_state_dict_spec()) == 608
    n = sum(math.prod(s) for _, s in OU.state_dict_spec())
    assert round(n / 1e6, 1) == 32.3


def test_engine_refuses_missing_and_extra_keys(pkg, monkeypatch):
    from cfi_b200 import engine as E
    monkeypatch.setattr(E.torch.cuda, "is_available", lambda: True)
    sd = OU.synthetic_state_dict(0)
    extra = dict(sd, **{"flownet.block3.flowconv.weight": torch.zeros(1)})
    with pytest.raises(KeyError, match="unexpected key flownet.block3"):
        E.IfunetEngine(extra)
    missing = dict(sd)
    del missing["refinenet.degrad.conv0.0.weight"]
    with pytest.raises(KeyError, match="missing refinenet.degrad.conv0.0.weight"):
        E.IfunetEngine(missing)


def test_mac_count_of_the_issue_figures():
    assert round(OU.ifunet_macs(1080, 1920, 1.0, ensemble=False) / 1e9, 1) == 1438.4
    assert round(OU.ifunet_macs(1080, 1920, 1.0, ensemble=True) / 1e9, 1) == 1755.3
