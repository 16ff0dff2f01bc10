#!/usr/bin/env python
"""Generate tests/golden/cain_*.npz and tests/golden/cain_spec.json by running the UNMODIFIED reference CAIN code.

    python tools/make_golden_cain.py

``vfi_models.cain.cain_arch.CAIN(depth=3)`` is imported as it is and loaded with ``oracle.cain.synthetic_state_dict``;
model cases call ``model(img0, img1)[0]``.  For the node cases the reference's ``CAIN_VFI.vfi`` runs unmodified, with its
downloader stubbed to return a temp checkpoint in the released form ``{"state_dict": {"module.<name>": tensor}}``.

The goldens must be able to fail: four mutated oracles (zero padding in ConvNorm, no channel attention, the mean not
added back, the pixel-shuffle sub-pixel order transposed) are scored against the model goldens taken together and each
must stay below 40 dB; the figure of every case is recorded.  (Zero padding changes only what the border cells feed
into the crop: at 130 x 135, 63 rows and 60 columns of padding lie between them and the output.)  The 3x3 weights carry
``oracle.cain.DEFAULT_GAIN``.  The tool also records that the seeded weights keep the trunk's features finite and the
attention gates away from 0 and 1.  Inputs are regenerated from seeds by the tests; only the reference outputs are stored.
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
from oracle import cain as OC  # noqa: E402
from oracle import film as OF  # noqa: E402  (synthetic_clip)

MUTATIONS = {
    "zero_padding": dict(pad="constant"),
    "no_attention": dict(attention=False),
    "mean_not_added": dict(add_mean=False),
    "shuffle_transposed": dict(transpose_shuffle=True),
}


def cain_cases():
    """Shared with the tests: name -> kwargs."""
    return {
        # 128 rows: no row padding; 200 columns padded to 256 (28 / 28)
        "cain_128x200": dict(kind="net", seed=0, h=128, w=200, clip_seed=71),
        # both axes padded, uneven split: 130 -> 256 (63 / 63), 135 -> 256 (60 / 61)
        "cain_130x135": dict(kind="net", seed=1, h=130, w=135, clip_seed=72),
        # 100 -> 128 (14 / 14), 300 -> 384 (42 / 42)
        "cain_100x300": dict(kind="net", seed=2, h=100, w=300, clip_seed=73),
        # node level: multiplier 2; 4 (three bisections: the shared midpoint kept); 5 (four: dropped); a skip list; a list
        # multiplier; 4-channel frames
        "cain_node_m2": dict(kind="node", seed=3, n=3, h=48, w=72, c=3, multiplier=2, states=None, clip_seed=74),
        "cain_node_m4": dict(kind="node", seed=4, n=2, h=56, w=64, c=3, multiplier=4, states=None, clip_seed=75),
        "cain_node_m5": dict(kind="node", seed=5, n=2, h=50, w=60, c=3, multiplier=5, states=None, clip_seed=76),
        "cain_node_skip": dict(kind="node", seed=6, n=4, h=48, w=52, c=3, multiplier=2, states=([1], True),
                               clip_seed=77),
        "cain_node_mlist": dict(kind="node", seed=7, n=4, h=44, w=68, c=3, multiplier=[3, 0], states=None,
                                clip_seed=78),
        "cain_node_rgba": dict(kind="node", seed=8, n=2, h=60, w=50, c=4, multiplier=2, states=None, clip_seed=79),
    }


def cain_inputs(cfg):
    n = 2 if cfg["kind"] == "net" else cfg["n"]
    fr = OF.synthetic_clip(n, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    if cfg.get("c", 3) == 4:
        fr = torch.cat([fr, torch.ones_like(fr[..., :1])], -1)
    return fr


def case_state_dict(cfg):
    """Model cases carry oracle.cain.DEFAULT_GAIN.  Node cases check the loop (order, bisection, skip, lists) and use
    nn.Conv2d's default ranges: at multiplier 5 the deepest middles are bisected from frames the model produced, and the
    gained trunk amplifies the 16-bit rounding those inputs carry (49.8 dB on the H100 at gain 1.25)."""
    return OC.synthetic_state_dict(cfg["seed"], OC.DEFAULT_GAIN if cfg["kind"] == "net" else 1.0)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


def main():
    _install_stub()
    import vfi_models.cain as FC
    from vfi_models.cain.cain_arch import CAIN
    from vfi_utils import InterpolationStateList

    out_dir = os.path.join(ROOT, "tests", "golden")
    spec, sq, n_el = {}, {}, 0
    for name, cfg in cain_cases().items():
        sd = case_state_dict(cfg)
        fr = cain_inputs(cfg)
        rec = dict(cfg)
        if cfg["kind"] == "net":
            m = CAIN(depth=3)
            m.load_state_dict(sd)
            m.eval()
            x = fr[..., :3].permute(0, 3, 1, 2).contiguous()
            with torch.no_grad():
                out = m(x[0:1].clone(), x[1:2].clone())[0]
                mine, gates, peak = OC.forward(sd, x[0:1], x[1:2], return_gates=True)
                assert float((out - mine).abs().max()) <= 1e-4, name
                assert math.isfinite(peak) and torch.isfinite(out).all(), name
                lo, hi = float(gates.min()), float(gates.max())
                assert 0.02 <= lo and hi <= 0.98, (name, lo, hi)
                rec["max_abs_feature"] = round(peak, 3)
                rec["gate_range"] = [round(lo, 4), round(hi, 4)]
                rec["mutations_db"] = {}
                for mname, kw in MUTATIONS.items():
                    mut = OC.forward(sd, x[0:1], x[1:2], **kw)
                    sq[mname] = sq.get(mname, 0.0) + float(((mut.double() - out.double()) ** 2).sum())
                    rec["mutations_db"][mname] = round(psnr(mut, out), 2)
                n_el += out.numel()
            print(name, tuple(out.shape), "max |feature|", round(peak, 3), "gates", rec["gate_range"],
                  "mutations", rec["mutations_db"])
        else:
            with tempfile.TemporaryDirectory() as td:
                path = os.path.join(td, "pretrained_cain.pth")
                torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
                FC.load_file_from_github_release = lambda model_type, ckpt_name, _p=path: _p
                st = None
                if cfg["states"] is not None:
                    st = InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
                (out,) = FC.CAIN_VFI().vfi("pretrained_cain.pth", fr, multiplier=cfg["multiplier"],
                                           optional_interpolation_states=st)
            print(name, tuple(out.shape))
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy())
        spec[name] = rec
    pooled = {m: round(10 * math.log10(n_el / v), 2) for m, v in sq.items()}
    print("mutations over all model goldens (dB):", pooled)
    assert all(p < 40.0 for p in pooled.values()), pooled
    spec["mutations_pooled_db"] = pooled
    with open(os.path.join(out_dir, "cain_spec.json"), "w") as fh:
        json.dump(spec, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
