"""The GMFSS Fortuna base model (the ``GMFSS_fortuna`` checkpoint) - seeded stand-in weights and the CPU restatement (fp32).
TEST INFRASTRUCTURE ONLY: what the product schedule (comfyui-frame-interpolation_b200/gmfss.py) is tested against when it
runs the base model.

Follows ``vfi_models/gmfss_fortuna/GMFSS_Fortuna_arch.py`` of Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc.  It differs
from the union model of oracle/gmfss.py in three places only (a diff of the two architecture files shows nothing else):
``Model`` has no IFNet and loads four sub-networks, not five; GridNet's first head is ``residual_model_head`` with 12 input
channels instead of union's 9-channel ``residual_model_head0`` (:1586, :1594, :1641); and ``Model.inference`` feeds it
``[img0, I1t, I2t, img1]`` of the half-size frames instead of ``[I1t, rife, I2t]`` (:1843-1848).  GMFlow, MetricNet,
FeatureNet, the eight soft splats and GridNet's body and tail are shared, so this file reuses oracle/gmfss.py and
oracle/gmflow.py for them.

Weights: no GMFSS checkpoint ships with the reference and there is no network, so the golden vectors of
``tools/make_golden_gmfss.py --variant base`` (outputs of the UNMODIFIED ``GMFSS_Fortuna_arch.Model``) are made on weights
generated here from ``tests/golden/gmfss_base_spec.json`` (names, shapes and dtypes of the four ``state_dict()``s as the
reference builds them).  The recipe is oracle/gmfss_weights.py's, per tensor, with seeds of its own; it does not import the
reference, so a GPU box can regenerate the same tensors.
"""
from __future__ import annotations

import json
import os
from typing import Dict

import torch
import torch.nn.functional as F

from . import gmfss as OG
from . import ops_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPEC = os.path.join(ROOT, "tests", "golden", "gmfss_base_spec.json")
NETS = ("flownet", "metricnet", "feat_ext", "fusionnet")


def load_spec() -> Dict[str, list]:
    with open(SPEC) as fh:
        return json.load(fh)


def synthetic_state_dicts(seed: int = 0) -> Dict[str, Dict[str, torch.Tensor]]:
    """the four state_dicts of the base model, seeded (oracle/gmfss_weights.py's recipe per tensor)"""
    spec = load_spec()
    out: Dict[str, Dict[str, torch.Tensor]] = {}
    for k, net in enumerate(NETS):
        g = torch.Generator().manual_seed(4000 + 10 * seed + k)
        sd: Dict[str, torch.Tensor] = {}
        for name, shape, dtype in spec[net]:
            shape = tuple(shape)
            if dtype != "torch.float32":                    # e.g. BatchNorm's num_batches_tracked
                sd[name] = torch.zeros(shape, dtype=getattr(torch, dtype.split(".")[1]))
                continue
            n = 1
            for s in shape:
                n *= s
            if len(shape) >= 2:                            # conv / linear / transposed conv weights
                fan_in = n // shape[0]
                v = (torch.rand(shape, generator=g) * 2 - 1) * (3.0 / max(fan_in, 1)) ** 0.5
            elif name.endswith("running_var"):
                v = 1.0 + 0.1 * torch.rand(shape, generator=g)
            elif name.endswith("running_mean"):
                v = 0.05 * (torch.rand(shape, generator=g) * 2 - 1)
            elif name.endswith(".weight") and ("norm" in name or "bn" in name):
                v = 1.0 + 0.1 * (torch.rand(shape, generator=g) * 2 - 1)
            elif name.endswith(".weight") or name.endswith("beta"):  # PReLU slopes (1-D "weight"), ResConv beta
                v = (0.25 + 0.1 * (torch.rand(shape, generator=g) * 2 - 1)) if not name.endswith("beta") else \
                    1.0 + 0.25 * (torch.rand(shape, generator=g) * 2 - 1)
            else:                                          # biases and the like
                v = 0.05 * (torch.rand(shape, generator=g) * 2 - 1)
            sd[name] = v.float()
        out[net] = sd
    return out


def gridnet(sd, x, x1, x2, x3):
    """GridNet.forward :1639-1688 of the base model: union's GridNet (oracle.gmfss.gridnet) with residual_model_head, which
    reads 12 channels, in the place of residual_model_head0"""
    p = "residual_model_head."
    return OG.gridnet({("residual_model_head0." + k[len(p):]) if k.startswith(p) else k: v for k, v in sd.items()},
                      x, x1, x2, x3)


def inference(sds: Dict[str, dict], img0, img1, flow01, flow10, metric0, metric1, f1, f2, timestep: float) -> torch.Tensor:
    """Model.inference :1779-1850."""
    splat = lambda a, fl, z: ops_ref.softsplat(a, fl, z, "soft")   # noqa: E731
    dn = lambda a, s: F.interpolate(a, scale_factor=s, mode="bilinear", align_corners=False)   # noqa: E731
    F1t, F2t = timestep * flow01, (1 - timestep) * flow10
    Z1t, Z2t = timestep * metric0, (1 - timestep) * metric1
    h0, h1 = dn(img0, 0.5), dn(img1, 0.5)
    I1t, I2t = splat(h0, F1t, Z1t), splat(h1, F2t, Z2t)
    a1, b1 = splat(f1[0], F1t, Z1t), splat(f2[0], F2t, Z2t)
    a2, b2 = splat(f1[1], dn(F1t, 0.5) * 0.5, dn(Z1t, 0.5)), splat(f2[1], dn(F2t, 0.5) * 0.5, dn(Z2t, 0.5))
    a3, b3 = splat(f1[2], dn(F1t, 0.25) * 0.25, dn(Z1t, 0.25)), splat(f2[2], dn(F2t, 0.25) * 0.25, dn(Z2t, 0.25))
    out = gridnet(sds["fusionnet"], torch.cat([h0, I1t, I2t, h1], 1), torch.cat([a1, b1], 1), torch.cat([a2, b2], 1),
                  torch.cat([a3, b3], 1))
    return torch.clamp(out, 0, 1)


def interpolate(sds: Dict[str, dict], frame0, frame1, timestep: float) -> torch.Tensor:
    """CommonModelInference.forward, gmfss_fortuna/__init__.py:41-77, scale 1: pad to multiples of 64 at the bottom / right,
    Model.reuse (the same as union's, oracle.gmfss.reuse) + inference, crop."""
    h, w = frame0.shape[2], frame0.shape[3]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    i0, i1 = F.pad(frame0, (0, pw - w, 0, ph - h)), F.pad(frame1, (0, pw - w, 0, ph - h))
    flow01, flow10, m0, m1, f1, f2 = OG.reuse(sds, i0, i1)
    return inference(sds, i0, i1, flow01, flow10, m0, m1, f1, f2, timestep)[:, :, :h, :w]
