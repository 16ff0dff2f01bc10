"""CPU restatement of GMFSS Fortuna (union) around its flow network (oracle/gmflow.py) - SURVEY.md section 8 row a11.
TEST INFRASTRUCTURE ONLY; GMFSS is not built in this repo yet, this file pins most of its target.

Follows ``vfi_models/gmfss_fortuna/GMFSS_Fortuna_union_arch.py`` of Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc:
``MetricNet`` :1420-1467 (with ``backwarp`` :1375-1417 and ``forward_backward_consistency_check`` :994-1013 / ``flow_warp``
:985-991 / ``bilinear_sample`` :955-983), ``FeatureNet`` :1470-1500, ``GridNet`` :1582-1688 with its blocks :1503-1579,
and ``Model.reuse`` / ``Model.inference`` :1726-1857.  The IFNet inside is ``oracle.rife46.ifnet46_forward`` (arch 4.6), the
one custom op ``softsplat`` is ``oracle.ops_ref.softsplat`` (pinned to the reference's own kernel by
tests/test_ops_ref_pinned.py), ``GMFlow`` (:35-1372, the transformer flow network) is ``oracle.gmflow.gmflow``.
``reuse_from_flows`` takes the two flows as inputs: the goldens of tools/make_golden_gmfss.py store the unmodified
reference's flows, so everything downstream of GMFlow is pinned on its own (tests/test_oracle_gmfss.py: metrics and the frame
from the golden flows), GMFlow on its own (the flows), and ``interpolate`` - the whole model as
``CommonModelInference.forward`` (gmfss_fortuna/__init__.py:41-77) runs it at scale 1 - end to end (the frame from the images).
Like oracle/gmflow.py it computes in the dtype and on the device of its inputs (fp32 or float64).
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from . import gmflow as GF
from . import ops_ref
from . import rife46 as R


def backwarp(ten_in: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """:1375-1417: grid_sample(bilinear, zeros, align_corners=True) at pixel + flow."""
    h, w = flow.shape[2], flow.shape[3]
    hor = torch.linspace(-1.0, 1.0, w, dtype=flow.dtype, device=flow.device).view(1, 1, 1, -1).repeat(1, 1, h, 1)
    ver = torch.linspace(-1.0, 1.0, h, dtype=flow.dtype, device=flow.device).view(1, 1, -1, 1).repeat(1, 1, 1, w)
    grid = torch.cat([hor, ver], 1)
    fl = torch.cat([flow[:, 0:1] / ((ten_in.shape[3] - 1.0) / 2.0), flow[:, 1:2] / ((ten_in.shape[2] - 1.0) / 2.0)], 1)
    return F.grid_sample(ten_in, (grid + fl).permute(0, 2, 3, 1), mode="bilinear", padding_mode="zeros", align_corners=True)


def _flow_warp(feature: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """flow_warp :985-991 + bilinear_sample :955-983 (padding 'zeros', align_corners=True) + coords_grid :916-932."""
    b, c, h, w = feature.shape
    y, x = torch.meshgrid(torch.arange(h, device=flow.device), torch.arange(w, device=flow.device), indexing="ij")
    coords = torch.stack([x, y], 0).to(flow.dtype)[None].repeat(b, 1, 1, 1) + flow
    xg = 2 * coords[:, 0] / (w - 1) - 1
    yg = 2 * coords[:, 1] / (h - 1) - 1
    return F.grid_sample(feature, torch.stack([xg, yg], -1), mode="bilinear", padding_mode="zeros", align_corners=True)


def fb_consistency(fwd: torch.Tensor, bwd: torch.Tensor, alpha: float = 0.01, beta: float = 0.5):
    """forward_backward_consistency_check :994-1013."""
    mag = torch.norm(fwd, dim=1) + torch.norm(bwd, dim=1)
    diff_f = torch.norm(fwd + _flow_warp(bwd, fwd), dim=1)
    diff_b = torch.norm(bwd + _flow_warp(fwd, bwd), dim=1)
    thr = alpha * mag + beta
    return (diff_f > thr).to(fwd.dtype), (diff_b > thr).to(fwd.dtype)


def _pconv(sd, prefix: str, x: torch.Tensor, stride: int = 1) -> torch.Tensor:
    """nn.Sequential(PReLU(), Conv2d(3x3, pad 1)): modules .0 (one slope) and .1."""
    return F.conv2d(F.prelu(x, sd[prefix + ".0.weight"]), sd[prefix + ".1.weight"], sd[prefix + ".1.bias"], stride=stride, padding=1)


def metricnet(sd, img0, img1, flow01, flow10) -> Tuple[torch.Tensor, torch.Tensor]:
    """MetricNet.forward :1429-1467 (images at the flows' resolution)."""
    m0 = F.l1_loss(img0, backwarp(img1, flow01), reduction="none").mean([1], True)
    m1 = F.l1_loss(img1, backwarp(img0, flow10), reduction="none").mean([1], True)
    occ_f, occ_b = fb_consistency(flow01, flow10)
    n01 = torch.cat([flow01[:, 0:1] / ((flow01.shape[3] - 1.0) / 2.0), flow01[:, 1:2] / ((flow01.shape[2] - 1.0) / 2.0)], 1)
    n10 = torch.cat([flow10[:, 0:1] / ((flow10.shape[3] - 1.0) / 2.0), flow10[:, 1:2] / ((flow10.shape[2] - 1.0) / 2.0)], 1)
    x = torch.cat([img0, img1, -m0, -m1, n01, n10, occ_f.unsqueeze(1), occ_b.unsqueeze(1)], 1)
    feat = F.conv2d(x, sd["metric_in.weight"], sd["metric_in.bias"], padding=1)
    for k in (1, 2, 3):
        feat = _pconv(sd, f"metric_net{k}", feat) + feat
    metric = torch.tanh(_pconv(sd, "metric_out", feat)) * 10
    return metric[:, :1], metric[:, 1:2]


def featurenet(sd, x):
    """FeatureNet.forward :1494-1500: three blocks of PReLU-conv(s2)-PReLU-conv."""
    outs = []
    for k in (1, 2, 3):
        p = f"block{k}"
        x = F.conv2d(F.prelu(x, sd[p + ".0.weight"]), sd[p + ".1.weight"], sd[p + ".1.bias"], stride=2, padding=1)
        x = F.conv2d(F.prelu(x, sd[p + ".2.weight"]), sd[p + ".3.weight"], sd[p + ".3.bias"], padding=1)
        outs.append(x)
    return outs


def _block(sd, p: str, x, kind: str):
    """ResidualBlock :1503-1524 / DownsampleBlock :1527-1543 / UpsampleBlock :1546-1561 (modules .0 PReLU .1 conv .2 PReLU .3 conv).
    Note ResidualBlock passes `stride` to BOTH convs (it is only ever built with stride 1)."""
    y = F.prelu(x, sd[p + ".0.weight"])
    if kind == "up":
        y = F.conv_transpose2d(y, sd[p + ".1.weight"], sd[p + ".1.bias"], stride=2, padding=1)
    else:
        y = F.conv2d(y, sd[p + ".1.weight"], sd[p + ".1.bias"], stride=2 if kind == "down" else 1, padding=1)
    return F.conv2d(F.prelu(y, sd[p + ".2.weight"]), sd[p + ".3.weight"], sd[p + ".3.bias"], padding=1)


def gridnet(sd, x, x1, x2, x3):
    """GridNet.forward :1639-1688."""
    r = lambda n, t: _block(sd, "residual_model_" + n, t, "res")        # noqa: E731
    d = lambda n, t: _block(sd, "downsample_model_" + n, t, "down")     # noqa: E731
    u = lambda n, t: _block(sd, "upsample_model_" + n, t, "up")         # noqa: E731
    X00 = r("head0", x) + r("head1", x1)
    X01 = r("01", X00) + X00
    X10 = d("10", X00) + r("head2", x2)
    X20 = d("20", X10) + r("head3", x3)
    X11 = (r("11", X10) + X10) + d("11", X01)
    X21 = (r("21", X20) + X20) + d("21", X11)
    X24 = r("24", X21) + X21
    X25 = r("25", X24) + X24
    X14 = u("14", X24) + (r("14", X11) + X11)
    X04 = u("04", X14) + (r("04", X01) + X01)
    X15 = u("15", X25) + (r("15", X14) + X14)
    X05 = u("05", X15) + (r("05", X04) + X04)
    # PixelShuffleBlcok :1564-1579
    t = "residual_model_tail."
    y = F.prelu(F.conv2d(X05, sd[t + "conv_before_upsample.0.weight"], sd[t + "conv_before_upsample.0.bias"], padding=1),
                sd[t + "conv_before_upsample.1.weight"])
    y = F.pixel_shuffle(F.conv2d(y, sd[t + "upsample.0.weight"], sd[t + "upsample.0.bias"], padding=1), 2)
    return F.conv2d(y, sd[t + "conv_last.weight"], sd[t + "conv_last.bias"], padding=1)


def reuse_from_flows(sds: Dict[str, dict], img0, img1, flow01, flow10):
    """Model.reuse :1726-1782 at scale 1.0 with the two GMFlow outputs given: features of the full-size frames, metrics on the
    half-size frames."""
    f1 = featurenet(sds["feat_ext"], img0)
    f2 = featurenet(sds["feat_ext"], img1)
    h0 = F.interpolate(img0, scale_factor=0.5, mode="bilinear", align_corners=False)
    h1 = F.interpolate(img1, scale_factor=0.5, mode="bilinear", align_corners=False)
    m0, m1 = metricnet(sds["metricnet"], h0, h1, flow01, flow10)
    return m0, m1, f1, f2


def inference(sds: Dict[str, dict], img0, img1, flow01, flow10, metric0, metric1, f1, f2, timestep: float, rife=None) -> torch.Tensor:
    """Model.inference :1784-1857.  `rife` (h0, h1, t) -> merged frame stands in for the IFNet 4.6 sub-model when given
    (e.g. another implementation's output, so that the rest of the model can be compared on its own)."""
    splat = lambda a, fl, z: ops_ref.softsplat(a, fl, z, "soft")   # noqa: E731
    dn = lambda a, s: F.interpolate(a, scale_factor=s, mode="bilinear", align_corners=False)   # noqa: E731
    F1t, F2t = timestep * flow01, (1 - timestep) * flow10
    Z1t, Z2t = timestep * metric0, (1 - timestep) * metric1
    h0, h1 = dn(img0, 0.5), dn(img1, 0.5)
    I1t, I2t = splat(h0, F1t, Z1t), splat(h1, F2t, Z2t)
    if rife is None:
        ts = torch.full((img0.shape[0], 1, 1, 1), float(timestep))
        rife = R.ifnet46_forward(sds["ifnet"], h0, h1, ts, (8, 4, 2, 1))
    else:
        rife = rife(h0, h1, timestep)
    a1, b1 = splat(f1[0], F1t, Z1t), splat(f2[0], F2t, Z2t)
    a2, b2 = splat(f1[1], dn(F1t, 0.5) * 0.5, dn(Z1t, 0.5)), splat(f2[1], dn(F2t, 0.5) * 0.5, dn(Z2t, 0.5))
    a3, b3 = splat(f1[2], dn(F1t, 0.25) * 0.25, dn(Z1t, 0.25)), splat(f2[2], dn(F2t, 0.25) * 0.25, dn(Z2t, 0.25))
    out = gridnet(sds["fusionnet"], torch.cat([I1t, rife, I2t], 1), torch.cat([a1, b1], 1), torch.cat([a2, b2], 1),
                  torch.cat([a3, b3], 1))
    return torch.clamp(out, 0, 1)


def reuse(sds: Dict[str, dict], img0, img1):
    """Model.reuse :1726-1782 at scale 1.0: both GMFlow directions on the half-size frames, then reuse_from_flows."""
    h0 = F.interpolate(img0, scale_factor=0.5, mode="bilinear", align_corners=False)
    h1 = F.interpolate(img1, scale_factor=0.5, mode="bilinear", align_corners=False)
    flow01, flow10 = GF.gmflow(sds["flownet"], h0, h1), GF.gmflow(sds["flownet"], h1, h0)
    return (flow01, flow10) + tuple(reuse_from_flows(sds, img0, img1, flow01, flow10))


def interpolate(sds: Dict[str, dict], frame0, frame1, timestep: float, rife=None) -> torch.Tensor:
    """CommonModelInference.forward, gmfss_fortuna/__init__.py:41-77, scale 1: pad to multiples of 64 at the bottom / right,
    reuse + inference (`rife` as there), crop."""
    h, w = frame0.shape[2], frame0.shape[3]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    i0, i1 = F.pad(frame0, (0, pw - w, 0, ph - h)), F.pad(frame1, (0, pw - w, 0, ph - h))
    flow01, flow10, m0, m1, f1, f2 = reuse(sds, i0, i1)
    return inference(sds, i0, i1, flow01, flow10, m0, m1, f1, f2, timestep, rife)[:, :, :h, :w]
