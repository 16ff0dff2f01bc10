#!/usr/bin/env python
"""Generate tests/golden/flavr_*.npz and tests/golden/flavr_spec.json by running the UNMODIFIED reference FLAVR code.

    python tools/make_golden_flavr.py

``vfi_models.flavr.flavr_arch.UNet_3D_3D`` is imported as it is and loaded with ``oracle.flavr.synthetic_state_dict``;
``resnet_3D.useBias`` (a module global the reference sets for n_outputs > 1 and never resets) is reset before every
build, so one process can build the 2x and then the 4x model.  For the node cases the reference's ``FLAVR_VFI.vfi``
runs unmodified, with its downloader stubbed to return a temp checkpoint ``{"state_dict": ...}`` whose keys carry the
``module.`` prefix that build_flavr strips.

Gain: seeded default-style weights give a prediction that barely differs from the window mean, so a check that the
output is close to the golden could pass by doing nothing.  The decoder and outconv weights are therefore scaled by
``oracle.flavr.DEFAULT_GAIN``; this tool asserts std(out - mean) >= 0.05 for every model case and prints the largest
|activation| of every reference module (it must stay far below fp16's 65504).
Inputs are regenerated from seeds by the tests; only the reference outputs are stored.
"""
import importlib
import json
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden import _install_stub  # noqa: E402
from oracle import film as OF  # noqa: E402  (synthetic_clip)
from oracle import flavr as OV  # noqa: E402


def flavr_cases():
    """Shared with the tests: name -> kwargs."""
    return {
        # model level (one window); sizes that are not multiples of 16: centred replicate padding, partial tiles
        "flavr_2x_40x56": dict(kind="net", variant="2x", seed=0, h=40, w=56, clip_seed=51),
        "flavr_4x_36x90": dict(kind="net", variant="4x", seed=1, h=36, w=90, clip_seed=52),
        # node level, 7 frames = 4 windows
        "flavr_node_dup": dict(kind="node", variant="2x", ckpt="FLAVR_2x.pth", seed=2, n=7, h=40, w=56, c=4,
                               multiplier=2, dup=True, states=None, clip_seed=53),
        # frames 0 and 1 skipped: the first window is dropped together with the frames it would have appended
        "flavr_node_skip_first": dict(kind="node", variant="2x", ckpt="FLAVR_2x.pth", seed=3, n=7, h=40, w=56, c=3,
                                      multiplier=2, dup=False, states=([0, 1, 4], True), clip_seed=54),
        # multiplier 3: the reference warns and interpolates 2x
        "flavr_node_m3": dict(kind="node", variant="4x", ckpt="FLAVR_4x.pth", seed=4, n=7, h=36, w=52, c=3,
                              multiplier=3, dup=False, states=None, clip_seed=55),
    }


def flavr_inputs(cfg):
    n = 4 if cfg["kind"] == "net" else cfg["n"]
    fr = OF.synthetic_clip(n, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    if cfg.get("c", 3) == 4:
        fr = torch.cat([fr, torch.ones_like(fr[..., :1])], -1)
    return fr


def _build(n_outputs, sd):
    importlib.import_module("vfi_models.flavr.resnet_3D").useBias = False
    from vfi_models.flavr.flavr_arch import UNet_3D_3D
    m = UNet_3D_3D("unet_18", n_inputs=4, n_outputs=n_outputs, joinType="concat", upmode="transpose")
    m.load_state_dict(sd)
    return m.eval()


def main():
    _install_stub()
    import vfi_models.flavr as FV
    from vfi_models.flavr.flavr_arch import InputPadder
    from vfi_utils import InterpolationStateList

    out_dir = os.path.join(ROOT, "tests", "golden")
    spec = {}
    for name, cfg in flavr_cases().items():
        n_out = OV.VARIANTS[cfg["variant"]][0]
        sd = OV.synthetic_state_dict(cfg["seed"], cfg["variant"])
        fr = flavr_inputs(cfg)
        rec = dict(cfg)
        if cfg["kind"] == "net":
            m = _build(n_out, sd)
            peaks = {}
            hooks = [mod.register_forward_hook(lambda mod, i, o, k=k: peaks.__setitem__(
                k, max(peaks.get(k, 0.0), float(max(t.abs().max() for t in (o if isinstance(o, (list, tuple)) else [o]))))))
                for k, mod in m.named_modules() if k and len(list(mod.children())) == 0]
            x = fr[..., :3].permute(0, 3, 1, 2)
            padder = InputPadder(x.shape, 16)
            xp = padder.pad(x)
            with torch.no_grad():
                out = m([xp[i:i + 1] for i in range(4)])[0]
            for h in hooks:
                h.remove()
            out = padder.unpad(out)
            mean = xp.mean(dim=(0, 2, 3)).view(1, 3, 1, 1)
            dev = float((out - mean).std())
            assert dev >= 0.05, (name, dev)
            rec["std_out_minus_mean"] = round(dev, 4)
            rec["max_abs_activation"] = round(max(peaks.values()), 2)
            print(name, tuple(out.shape), "std(out - mean)", round(dev, 4))
            for k, v in peaks.items():
                print(f"  {k:45s} max |a| {v:9.3f}")
            np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy())
        else:
            with tempfile.TemporaryDirectory() as td:
                path = os.path.join(td, cfg["ckpt"])
                torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, path)
                FV.load_file_from_github_release = lambda model_type, ckpt_name, _p=path: _p
                importlib.import_module("vfi_models.flavr.resnet_3D").useBias = False
                st = None
                if cfg["states"] is not None:
                    st = InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
                with warnings.catch_warnings(record=True) as caught:
                    warnings.simplefilter("always")
                    (out,) = FV.FLAVR_VFI().vfi(cfg["ckpt"], fr, multiplier=cfg["multiplier"],
                                                duplicate_first_last_frames=cfg["dup"], optional_interpolation_states=st)
                rec["warned"] = any("FLAVR only supports 2x" in str(w.message) for w in caught)
            np.savez_compressed(os.path.join(out_dir, name + ".npz"), out=out.numpy())
            print(name, tuple(out.shape), "warned", rec["warned"])
        spec[name] = rec
    with open(os.path.join(out_dir, "flavr_spec.json"), "w") as fh:
        json.dump(spec, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
