#!/usr/bin/env python
"""Generate tests/golden/ifrnet_*.npz and tests/golden/ifrnet_spec.json by running the UNMODIFIED reference IFRNet code.

    python tools/make_golden_ifrnet.py

``vfi_models.ifrnet.IFRNet_{S,L}_arch.IRFNet_{S,L}`` are imported as they are and loaded with
``oracle.ifrnet.synthetic_state_dict``.  Model cases call ``model(img0, img1, t, embt)`` in the node's argument order
(the resize factor ``t`` first, see ifrnet_node.py).  For the node cases the reference's ``IFRNet_VFI.vfi`` runs
unmodified, with its downloader stubbed to return a temp checkpoint.

Gain: seeded default-style weights give an almost trivial blend, so a check that the output is close to the golden
could pass by doing little.  The decoder weights are scaled by ``oracle.ifrnet.DEFAULT_GAIN``; for every model case this
tool asserts that the final flows move pixels (mean |flow| >= 1 px) and that the residual is not negligible
(std >= 0.02), and records both.  The flows come from the oracle, which this tool also checks against the reference's
output.  Inputs are regenerated from seeds by the tests; only the reference outputs are stored.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden import _install_stub  # noqa: E402
from oracle import film as OF  # noqa: E402  (synthetic_clip)
from oracle import ifrnet as OI  # noqa: E402


def ifrnet_cases():
    """Shared with the tests: name -> kwargs.  Sizes are not multiples of 64."""
    return {
        # t = 1/2 (multiplier 2), both variants, embt 1.0 (the node's default) and 0.25
        "ifrnet_S_70x100_t2": dict(kind="net", variant="S", seed=0, h=70, w=100, t=0.5, embt=1.0, clip_seed=61),
        "ifrnet_L_60x90_t2": dict(kind="net", variant="L", seed=1, h=60, w=90, t=0.5, embt=0.25, clip_seed=62),
        # t = 1/3: the decoder grids (6, 12, 24, 48 rows) differ from the encoder levels they warp (6, 11, 21 rows)
        "ifrnet_S_100x180_t3": dict(kind="net", variant="S", seed=2, h=100, w=180, t=1.0 / 3.0, embt=1.0, clip_seed=63),
        "ifrnet_L_100x120_t3": dict(kind="net", variant="L", seed=3, h=100, w=120, t=1.0 / 3.0, embt=0.25, clip_seed=64),
        # node level
        "ifrnet_node_m3": dict(kind="node", ckpt="IFRNet_S_Vimeo90K.pth", seed=4, n=3, h=40, w=72, c=3, multiplier=3,
                               scale_factor=1.0, states=None, clip_seed=65),
        "ifrnet_node_skip": dict(kind="node", ckpt="IFRNet_L_GoPro.pth", seed=5, n=4, h=36, w=52, c=3, multiplier=2,
                                 scale_factor=0.25, states=([1], True), clip_seed=66),
        "ifrnet_node_mlist": dict(kind="node", ckpt="IFRNet_S_GoPro.pth", seed=6, n=4, h=40, w=56, c=3,
                                  multiplier=[3, 0], scale_factor=2.0, states=None, clip_seed=67),
        "ifrnet_node_rgba": dict(kind="node", ckpt="IFRNet_L_Vimeo90K.pth", seed=7, n=2, h=44, w=60, c=4, multiplier=2,
                                 scale_factor=4.0, states=None, clip_seed=68),
    }


def ifrnet_inputs(cfg):
    n = 2 if cfg["kind"] == "net" else cfg["n"]
    fr = OF.synthetic_clip(n, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    if cfg.get("c", 3) == 4:
        fr = torch.cat([fr, torch.ones_like(fr[..., :1])], -1)
    return fr


def case_state_dict(cfg):
    variant = cfg["variant"] if cfg["kind"] == "net" else OI.variant_of(cfg["ckpt"])
    return OI.synthetic_state_dict(variant, cfg["seed"])


def main():
    _install_stub()
    import vfi_models.ifrnet as FI
    from vfi_models.ifrnet.IFRNet_L_arch import IRFNet_L
    from vfi_models.ifrnet.IFRNet_S_arch import IRFNet_S
    from vfi_utils import InterpolationStateList

    out_dir = os.path.join(ROOT, "tests", "golden")
    spec = {}
    for name, cfg in ifrnet_cases().items():
        sd = case_state_dict(cfg)
        fr = ifrnet_inputs(cfg)
        rec = dict(cfg)
        if cfg["kind"] == "net":
            m = (IRFNet_S() if cfg["variant"] == "S" else IRFNet_L())
            m.load_state_dict(sd)
            m.eval()
            x = fr[..., :3].permute(0, 3, 1, 2).contiguous()
            with torch.no_grad():
                out = m(x[0:1], x[1:2], cfg["t"], cfg["embt"])
                mine, flow, res = OI.forward(sd, x[0:1], x[1:2], cfg["t"], cfg["embt"], return_flows=True)
            assert float((out - mine).abs().max()) <= 1e-5, name
            mflow, sres = float(flow.abs().mean()), float(res.std())
            assert mflow >= 1.0, (name, mflow)
            assert sres >= 0.02, (name, sres)
            rec["mean_abs_flow_px"] = round(mflow, 3)
            rec["std_residual"] = round(sres, 4)
            print(name, tuple(out.shape), "mean |flow|", round(mflow, 3), "std(res)", round(sres, 4))
        else:
            with tempfile.TemporaryDirectory() as td:
                path = os.path.join(td, cfg["ckpt"])
                torch.save(sd, path)
                FI.load_file_from_github_release = lambda model_type, ckpt_name, _p=path: _p
                st = None
                if cfg["states"] is not None:
                    st = InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
                (out,) = FI.IFRNet_VFI().vfi(cfg["ckpt"], fr, multiplier=cfg["multiplier"],
                                             scale_factor=cfg["scale_factor"], optional_interpolation_states=st)
            print(name, tuple(out.shape))
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy())
        spec[name] = rec
    with open(os.path.join(out_dir, "ifrnet_spec.json"), "w") as fh:
        json.dump(spec, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
