#!/usr/bin/env python
"""Target vectors for GMFSS Fortuna, SURVEY.md section 8 row a11: outputs of the UNMODIFIED reference model.

    python tools/make_golden_gmfss.py                   # union: tests/golden/gmfss_spec.json and tests/golden/gmfss_*.npz
    python tools/make_golden_gmfss.py --variant base    # base:  tests/golden/gmfss_base_spec.json and gmfss_base_*.npz

``--variant union`` (the default) runs ``vfi_models/gmfss_fortuna/GMFSS_Fortuna_union_arch.Model`` (GMFlow + IFNet 4.6 +
MetricNet + FeatureNet + GridNet), ``--variant base`` runs ``GMFSS_Fortuna_arch.Model`` (the ``GMFSS_fortuna`` checkpoint: no
IFNet, a 12-channel GridNet head).  Either runs as it is on the CPU; its one custom op, ``softsplat`` (``vfi_models.ops``,
cupy), is replaced by ``oracle.ops_ref.softsplat``, which tests/test_ops_ref_pinned.py pins to the reference's own kernel.
Weights: ``oracle.gmfss_weights`` (union) / ``oracle.gmfss_base`` (base), seeded and regenerated from the spec file
without the reference.  The vectors pin the CPU oracles (oracle/gmfss.py, oracle/gmfss_base.py) and the product schedule
(gmfss.py) on the host build and on the GPU: flows, metrics and the frame of ``CommonModelInference.forward``,
gmfss_fortuna/__init__.py:41-77.  Each variant writes only its own files.
"""
import argparse
import importlib
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden import _install_stub  # noqa: E402
from oracle import film as OF  # noqa: E402  (synthetic_clip)
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import ops_ref  # noqa: E402

ARCH = {"union": "GMFSS_Fortuna_union_arch", "base": "GMFSS_Fortuna_arch"}
WEIGHTS = {"union": GW, "base": GB}   # NETS, SPEC, synthetic_state_dicts(seed) of each variant


def gmfss_cases(variant: str = "union"):
    """name -> case; the base variant uses the same seeds and clips under the prefix gmfss_base_"""
    p = {"union": "gmfss_", "base": "gmfss_base_"}[variant]
    return {
        p + "96x128_t0.5": dict(seed=0, h=96, w=128, t=0.5, clip_seed=71),
        p + "70x100_t0.3": dict(seed=1, h=70, w=100, t=0.3, clip_seed=72),   # padded to 128 x 128 by the wrapper
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", choices=sorted(ARCH), default="union")
    variant = ap.parse_args().variant
    _install_stub()
    import vfi_models
    ops = types.ModuleType("vfi_models.ops")
    ops.softsplat = lambda tenIn, tenFlow, tenMetric, strMode: ops_ref.softsplat(tenIn, tenFlow, tenMetric, strMode)
    sys.modules["vfi_models.ops"] = ops
    vfi_models.ops = ops
    A = importlib.import_module("vfi_models.gmfss_fortuna." + ARCH[variant])
    A.device = torch.device("cpu")
    out_dir = os.path.join(ROOT, "tests", "golden")
    W = WEIGHTS[variant]
    nets = W.NETS
    m = A.Model()
    m.eval()
    spec = {net: [[k, list(v.shape), str(v.dtype)] for k, v in getattr(m, net).state_dict().items()] for net in nets}
    with open(W.SPEC, "w") as fh:
        json.dump(spec, fh)
    for name, cfg in gmfss_cases(variant).items():
        sds = W.synthetic_state_dicts(cfg["seed"])
        for net in nets:
            getattr(m, net).load_state_dict(sds[net])
        fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous()
        h, w = cfg["h"], cfg["w"]
        ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64     # CommonModelInference.forward, scale = 1
        i0, i1 = F.pad(fr[0:1], (0, pw - w, 0, ph - h)), F.pad(fr[1:2], (0, pw - w, 0, ph - h))
        with torch.no_grad():
            r = m.reuse(i0, i1, 1.0)
            out = m.inference(i0, i1, *r, cfg["t"])[:, :, :h, :w]
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy(), flow01=r[0].numpy(), flow10=r[1].numpy(),
                            metric0=r[2].numpy(), metric1=r[3].numpy())
        print(name, tuple(out.shape), float(out.mean()), float(out.std()), "flow absmax", float(r[0].abs().max()),
              "finite", bool(torch.isfinite(out).all()))


if __name__ == "__main__":
    main()
