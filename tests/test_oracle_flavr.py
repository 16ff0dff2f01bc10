"""oracle/flavr.py (the CPU restatement of FLAVR) against the unmodified reference's outputs in tests/golden/flavr_*.npz,
and the state-dict layouts of the three checkpoints."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_flavr import flavr_cases, flavr_inputs  # noqa: E402
from oracle import flavr as OV  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


@pytest.mark.parametrize("name", [k for k, v in flavr_cases().items() if v["kind"] == "net"])
def test_oracle_matches_reference_model(name):
    cfg = flavr_cases()[name]
    sd = OV.synthetic_state_dict(cfg["seed"], cfg["variant"])
    fr = flavr_inputs(cfg)[..., :3]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])[0].permute(1, 2, 0)
    got = OV.interpolate(sd, fr)
    p = psnr(got, ref)
    assert p >= 50.0, p
    # the golden is not trivially close to the window's mean colour (see make_golden_flavr.py: gain)
    assert psnr(OV.mean_only(fr), ref) < 30.0


def test_spec_records_gain_and_activation_range():
    spec = json.load(open(os.path.join(GOLD, "flavr_spec.json")))
    for name, cfg in flavr_cases().items():
        assert name in spec
        if cfg["kind"] == "net":
            assert spec[name]["std_out_minus_mean"] >= 0.05
            assert spec[name]["max_abs_activation"] < 1000.0   # far below fp16's 65504
    assert spec["flavr_node_m3"]["warned"] and not spec["flavr_node_dup"]["warned"]


@pytest.mark.parametrize("variant,n_out,bias,count", [("2x", 1, False, 59), ("4x", 3, True, 76), ("8x", 7, True, 76)])
def test_state_dict_names_for_each_checkpoint(pkg, variant, n_out, bias, count):
    from cfi_b200.engine import flavr_state_dict_names
    sd = OV.synthetic_state_dict(0, variant)
    names = flavr_state_dict_names(enc_bias=bias)
    assert len(names) == count
    assert names == list(sd.keys())
    assert sd["outconv.1.weight"].shape[0] == 3 * n_out
    assert ("encoder.stem.0.bias" in sd) == bias
