"""RIFE node scale_factor 2 / 4 (up-scaled last blocks, archs 4.6 / 4.7 / 4.17 / 4.26) on the GPU against the unmodified reference's outputs.
front_up / fold_down are also checked through the host emulation (tests/test_rife_full_host.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import rife46 as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden import cases, make_inputs  # noqa: E402

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("name", [n for n, c in cases().items() if c["kind"] == "ifnet" and "scale_factor" in c])
def test_ifnet_scale_factor_golden(pkg, name):
    from cfi_b200.engine import Rife46Engine
    cfg = cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"]).clamp(0, 1)
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"], arch=cfg.get("arch", "4.6"))
    eng = Rife46Engine(sd, 0, "float32")
    fr = make_inputs(cfg)
    b = len(cfg["ts"])
    out = eng.forward(fr.cuda().contiguous(), [0] * b, [1] * b, list(cfg["ts"]), scale_factor=cfg["scale_factor"]).cpu()
    eng.close()
    assert O.psnr(out, ref.permute(0, 2, 3, 1)) >= 50.0
