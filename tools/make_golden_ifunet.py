#!/usr/bin/env python
"""Generate tests/golden/ifunet_*.npz and tests/golden/ifunet_spec.json by running the UNMODIFIED reference IFUNet code.

    python tools/make_golden_ifunet.py

``vfi_models.ifunet.IFUNet_arch.IFUNetModel`` is imported as it is, loaded strictly with
``oracle.ifunet.synthetic_state_dict`` and run in eval mode; model cases call ``model(img0, img1, timestep=t,
scale=s, ensemble=e)``.  For the node cases the reference's ``IFUnet_VFI.vfi`` runs unmodified, with its downloader
stubbed to return a temp checkpoint holding the raw state dict, as ``IFUNet.pth`` does.

The goldens must be able to fail: mutated oracles (``oracle.ifunet.MUTATIONS``: the ensemble pass reading the flow with
its channels swapped, no convex upsampling, zero-padded warps, BatchNorm skipped, resize coordinates from the size
ratio, ResynNet without the ``deg`` term) are scored against the model goldens taken together; at least four must stay
below 40 dB, and every figure is recorded.  The tool also asserts that the seeded flows move pixels by several pixels
and that the masks and CBAM gates are not saturated, and it records, for every ``scale_factor`` of the table in
DESIGN.md section 12, whether the reference runs or raises at 128 x 192 and 100 x 150 (``oracle.ifunet.geometry``
must agree).  Inputs are regenerated from seeds by the tests; only the reference outputs are stored.
"""
import json
import math
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
from oracle import ifunet as OU  # noqa: E402

SCALE_TABLE = (0.1, 0.2, 0.25, 0.5, 0.7, 0.8, 1.0, 1.2, 1.5, 2.0, 2.5, 3.0, 4.0)
TABLE_SIZES = ((128, 192), (100, 150))


def ifunet_cases():
    """Shared with the tests: name -> kwargs."""
    return {
        # 128 x 192: no padding; 100 x 150 padded to 128 x 192
        "ifunet_128x192_t2": dict(kind="net", seed=0, h=128, w=192, t=0.5, scale=1.0, ensemble=True, clip_seed=81),
        "ifunet_100x150_t3": dict(kind="net", seed=1, h=100, w=150, t=1 / 3, scale=1.0, ensemble=False, clip_seed=82),
        "ifunet_128x192_s05": dict(kind="net", seed=2, h=128, w=192, t=0.5, scale=0.5, ensemble=True, clip_seed=83),
        "ifunet_100x150_s15": dict(kind="net", seed=3, h=100, w=150, t=1 / 3, scale=1.5, ensemble=True, clip_seed=84),
        "ifunet_120x130_s2": dict(kind="net", seed=0, h=120, w=130, t=0.5, scale=2.0, ensemble=False, clip_seed=85),
        # node level: multiplier 3 with a skip list; a list multiplier; 4-channel frames; ensemble off
        "ifunet_node_m3_skip": dict(kind="node", seed=4, n=4, h=48, w=72, c=3, multiplier=3, states=([1], True),
                                    scale=1.0, ensemble=True, clip_seed=86),
        "ifunet_node_mlist": dict(kind="node", seed=5, n=4, h=56, w=64, c=3, multiplier=[3, 0], states=None,
                                  scale=1.0, ensemble=True, clip_seed=87),
        "ifunet_node_rgba": dict(kind="node", seed=6, n=2, h=60, w=50, c=4, multiplier=2, states=None, scale=1.0,
                                 ensemble=True, clip_seed=88),
        "ifunet_node_noens": dict(kind="node", seed=7, n=3, h=64, w=70, c=3, multiplier=2, states=None, scale=0.5,
                                  ensemble=False, clip_seed=89),
    }


def ifunet_inputs(cfg):
    n = 2 if cfg["kind"] == "net" else cfg["n"]
    fr = OF.synthetic_clip(n, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    if cfg.get("c", 3) == 4:
        fr = torch.cat([fr, torch.ones_like(fr[..., :1])], -1)
    return fr


def case_state_dict(cfg):
    return OU.synthetic_state_dict(cfg["seed"])


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


def scale_table(IFUNetModel, sd):
    """{"HxW": {scale: "runs" | "raises"}} from the unmodified reference (ensemble on)."""
    m = IFUNetModel()
    m.load_state_dict(sd)
    m.eval()
    table = {}
    for h, w in TABLE_SIZES:
        x = torch.rand(2, 3, h, w, generator=torch.Generator().manual_seed(5))
        row = {}
        for s in SCALE_TABLE:
            try:
                with torch.no_grad():
                    m(x[0:1], x[1:2], timestep=0.5, scale=s, ensemble=True)
                row[str(s)] = "runs"
            except RuntimeError:
                row[str(s)] = "raises"
            assert (row[str(s)] == "runs") == (OU.geometry(h, w, s) is not None), (h, w, s, row[str(s)])
        table[f"{h}x{w}"] = row
        print("scale_factor table", h, w, row)
    return table


def main():
    _install_stub()
    import vfi_models.ifunet as FU
    from vfi_models.ifunet.IFUNet_arch import IFUNetModel
    from vfi_utils import InterpolationStateList

    out_dir = os.path.join(ROOT, "tests", "golden")
    spec, sq, n_el = {}, {}, 0
    for name, cfg in ifunet_cases().items():
        sd = case_state_dict(cfg)
        fr = ifunet_inputs(cfg)
        rec = dict(cfg)
        if cfg["kind"] == "net":
            m = IFUNetModel()
            m.load_state_dict(sd)
            m.eval()
            x = fr[..., :3].permute(0, 3, 1, 2).contiguous()
            kw = dict(timestep=cfg["t"], scale=cfg["scale"], ensemble=cfg["ensemble"])
            with torch.no_grad():
                out = m(x[0:1].clone(), x[1:2].clone(), **kw)
                mine, st = OU.forward(sd, x[0:1], x[1:2], cfg["t"], cfg["scale"], cfg["ensemble"], return_stats=True)
                assert float((out - mine).abs().max()) <= 1e-4, name
                assert torch.isfinite(out).all(), name
                fl = st["flow_absmax"]
                assert 1.0 <= max(fl) <= 64.0 and max(st["resyn_flow_absmax"]) >= 2.0, (name, fl, st["resyn_flow_absmax"])
                lo, hi = st["fusion_mask_range"]
                assert 2e-4 <= lo and hi <= 1 - 2e-4, (name, lo, hi)
                rm = [v for r in st["resyn_mask_range"] for v in r]
                assert max(abs(v) for v in rm) < 4.0, (name, rm)
                cg = [v for g in st["gates"] for v in g]
                assert 0.02 <= min(cg) and max(cg) <= 0.98, (name, min(cg), max(cg))
                rec["flow_absmax_per_level"] = [round(v, 3) for v in fl]
                rec["resyn_flow_absmax"] = [round(v, 3) for v in st["resyn_flow_absmax"]]
                rec["fusion_mask_range"] = [round(lo, 4), round(hi, 4)]
                rec["resyn_mask_range"] = [round(min(rm), 4), round(max(rm), 4)]
                rec["gate_range"] = [round(min(cg), 4), round(max(cg), 4)]
                rec["mutations_db"] = {}
                for mname in OU.MUTATIONS:
                    mut = OU.forward(sd, x[0:1], x[1:2], cfg["t"], cfg["scale"], cfg["ensemble"], **{mname: True})
                    sq[mname] = sq.get(mname, 0.0) + float(((mut.double() - out.double()) ** 2).sum())
                    rec["mutations_db"][mname] = round(psnr(mut, out), 2)
                n_el += out.numel()
            print(name, tuple(out.shape), "flows", rec["flow_absmax_per_level"], rec["resyn_flow_absmax"], "masks",
                  rec["fusion_mask_range"], rec["resyn_mask_range"], "gates", rec["gate_range"], "mutations",
                  rec["mutations_db"], flush=True)
        else:
            with tempfile.TemporaryDirectory() as td:
                path = os.path.join(td, "IFUNet.pth")
                torch.save(sd, path)
                FU.load_file_from_github_release = lambda model_type, ckpt_name, _p=path: _p
                st = None
                if cfg["states"] is not None:
                    st = InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
                (out,) = FU.IFUnet_VFI().vfi("IFUNet.pth", fr, multiplier=cfg["multiplier"],
                                             scale_factor=cfg["scale"], ensemble=cfg["ensemble"],
                                             optional_interpolation_states=st)
            print(name, tuple(out.shape), flush=True)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy())
        spec[name] = rec
    pooled = {m: round(10 * math.log10(n_el / v), 2) if v > 0 else 99.0 for m, v in sq.items()}
    print("mutations over all model goldens (dB):", pooled)
    assert sum(p < 40.0 for p in pooled.values()) >= 4, pooled
    spec["mutations_pooled_db"] = pooled
    spec["scale_factor_table"] = scale_table(IFUNetModel, OU.synthetic_state_dict(0))
    with open(os.path.join(out_dir, "ifunet_spec.json"), "w") as fh:
        json.dump(spec, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
