"""CPU restatement of GMFlow as GMFSS Fortuna uses it - SURVEY.md section 8 row a11.  TEST INFRASTRUCTURE ONLY; GMFSS is
not built in this repo yet, this file and oracle/gmfss.py pin its target.

Follows ``vfi_models/gmfss_fortuna/GMFSS_Fortuna_union_arch.py`` of Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc, the
inference configuration ``Model.reuse`` :1726-1782 runs (``GMFlow()`` defaults :1157-1199: two scales, swin attention with
[2, 8] splits, global matching then radius-4 local matching, global then radius-1 flow propagation, convex x4 up-sampling,
``pred_bidir_flow=False``; eval mode):

* ``encoder``          CNNEncoder :218-312 with ResidualBlock_class :165-215 (InstanceNorm2d without affine) and the two-branch
                       MultiScaleTridentConv :68-162 (one shared 3x3 weight, strides 1 and 2; test_branch_idx = -1 keeps both);
* ``add_position``     feature_add_position :1134-1154 + PositionEmbeddingSine :1015-1056 inside the attention windows;
* ``transformer``      FeatureTransformer :592-685, TransformerBlock :526-589, TransformerLayer :439-523 with the
                       single-head full / split-window attention :315-436 and the shifted-window mask :326-364;
* ``global_match`` / ``local_match``   global_correlation_softmax :806-843, local_correlation_softmax :846-913;
* ``propagate``        FeatureFlowAttention :688-803 (note the reference's key = k_proj(q_proj(x)) in the global form);
* ``upsample_convex``  GMFlow.upsample_flow :1220-1260;
* ``gmflow``           GMFlow.forward :1262-1369.

Pinned by tests/test_oracle_gmfss.py against the flows of the unmodified reference (tests/golden/gmfss_*.npz).

Every tensor it creates takes the dtype and device of its inputs: fp32 CPU tensors give the fp32 restatement the goldens pin,
float64 tensors on any device the float64 reference tests/test_gpu_zgmfss_shadow.py compares
the product with.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _inorm(x):
    return F.instance_norm(x, eps=1e-5)


def _resblock(sd, p: str, x, stride: int):
    y = F.relu(_inorm(F.conv2d(x, sd[p + ".conv1.weight"], None, stride=stride, padding=1)))
    y = F.relu(_inorm(F.conv2d(y, sd[p + ".conv2.weight"], None, padding=1)))
    if p + ".downsample.0.weight" in sd:
        x = _inorm(F.conv2d(x, sd[p + ".downsample.0.weight"], sd[p + ".downsample.0.bias"], stride=stride))
    return F.relu(x + y)


def encoder(sd, x):
    """[quarter-resolution, eighth-resolution] 128-channel features of a normalised image batch."""
    p = "backbone."
    x = F.relu(_inorm(F.conv2d(x, sd[p + "conv1.weight"], None, stride=2, padding=3)))
    for layer, stride in (("layer1", 1), ("layer2", 2), ("layer3", 1)):
        x = _resblock(sd, p + layer + ".0", x, stride)
        x = _resblock(sd, p + layer + ".1", x, 1)
    x = F.conv2d(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"])
    w = sd[p + "trident_conv.weight"]
    return [F.conv2d(x, w, None, stride=1, padding=1), F.conv2d(x, w, None, stride=2, padding=1)]


def _windows(x, k: int):
    """[B, C, H, W] -> [B*k*k, C, H/k, W/k] (split_feature :1059-1091)."""
    b, c, h, w = x.shape
    return x.view(b, c, k, h // k, k, w // k).permute(0, 2, 4, 1, 3, 5).reshape(b * k * k, c, h // k, w // k)


def _unwindows(x, k: int):
    bk, c, h, w = x.shape
    b = bk // (k * k)
    return x.view(b, k, k, c, h, w).permute(0, 3, 1, 4, 2, 5).contiguous().view(b, c, k * h, k * w)


def _windows_last(x, k: int):
    b, h, w, c = x.shape
    return x.view(b, k, h // k, k, w // k, c).permute(0, 1, 3, 2, 4, 5).reshape(b * k * k, h // k, w // k, c)


def _unwindows_last(x, k: int):
    bk, h, w, c = x.shape
    b = bk // (k * k)
    return x.view(b, k, k, h, w, c).permute(0, 1, 3, 2, 4, 5).contiguous().view(b, k * h, k * w, c)


def position_sine(b: int, h: int, w: int, feats: int = 64, temperature: float = 10000.0, dtype=torch.float32, device=None):
    ones = torch.ones(b, h, w, dtype=dtype, device=device)
    ye, xe = ones.cumsum(1, dtype=dtype), ones.cumsum(2, dtype=dtype)
    ye = ye / (ye[:, -1:, :] + 1e-6) * (2 * math.pi)
    xe = xe / (xe[:, :, -1:] + 1e-6) * (2 * math.pi)
    dim_t = torch.arange(feats, dtype=dtype, device=device)
    dim_t = temperature ** (2 * (dim_t // 2) / feats)
    px, py = xe[:, :, :, None] / dim_t, ye[:, :, :, None] / dim_t
    px = torch.stack((px[:, :, :, 0::2].sin(), px[:, :, :, 1::2].cos()), dim=4).flatten(3)
    py = torch.stack((py[:, :, :, 0::2].sin(), py[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((py, px), dim=3).permute(0, 3, 1, 2)


def add_position(f0, f1, splits: int):
    a, b = _windows(f0, splits), _windows(f1, splits)
    pos = position_sine(a.shape[0], a.shape[2], a.shape[3], f0.shape[1] // 2, dtype=f0.dtype, device=f0.device)
    return _unwindows(a + pos, splits), _unwindows(b + pos, splits)


def shift_mask(h: int, w: int, splits: int, dtype=torch.float32, device=None):
    wh, ww = h // splits, w // splits
    sh, sw = wh // 2, ww // 2
    img = torch.zeros(1, h, w, 1, dtype=dtype, device=device)
    cnt = 0
    for hs in (slice(0, -wh), slice(-wh, -sh), slice(-sh, None)):
        for ws in (slice(0, -ww), slice(-ww, -sw), slice(-sw, None)):
            img[:, hs, ws, :] = cnt
            cnt += 1
    mw = _windows_last(img, w // ww).view(-1, wh * ww)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def _window_attention(q, k, v, splits: int, shifted: bool, h: int, w: int, mask):
    b, _, c = q.shape
    q, k, v = q.view(b, h, w, c), k.view(b, h, w, c), v.view(b, h, w, c)
    sh, sw = (h // splits) // 2, (w // splits) // 2
    if shifted:
        q, k, v = (torch.roll(t, shifts=(-sh, -sw), dims=(1, 2)) for t in (q, k, v))
    bn = b * splits * splits
    q, k, v = (_windows_last(t, splits).reshape(bn, -1, c) for t in (q, k, v))
    scores = torch.matmul(q, k.permute(0, 2, 1)) / c ** 0.5
    if shifted:
        scores = scores + mask.repeat(b, 1, 1)
    out = torch.matmul(torch.softmax(scores, dim=-1), v)
    out = _unwindows_last(out.view(bn, h // splits, w // splits, c), splits)
    if shifted:
        out = torch.roll(out, shifts=(sh, sw), dims=(1, 2))
    return out.view(b, -1, c)


def _layer(sd, p: str, source, target, h, w, splits, shifted, mask, ffn: bool):
    q = F.linear(source, sd[p + ".q_proj.weight"])
    k = F.linear(target, sd[p + ".k_proj.weight"])
    v = F.linear(target, sd[p + ".v_proj.weight"])
    if splits > 1:
        msg = _window_attention(q, k, v, splits, shifted, h, w, mask)
    else:
        msg = torch.matmul(torch.softmax(torch.matmul(q, k.permute(0, 2, 1)) / q.shape[2] ** 0.5, dim=2), v)
    c = source.shape[-1]
    msg = F.layer_norm(F.linear(msg, sd[p + ".merge.weight"]), (c,), sd[p + ".norm1.weight"], sd[p + ".norm1.bias"])
    if ffn:
        msg = F.linear(F.gelu(F.linear(torch.cat([source, msg], dim=-1), sd[p + ".mlp.0.weight"])), sd[p + ".mlp.2.weight"])
        msg = F.layer_norm(msg, (c,), sd[p + ".norm2.weight"], sd[p + ".norm2.bias"])
    return source + msg


def transformer(sd, f0, f1, splits: int, num_layers: int = 6):
    b, c, h, w = f0.shape
    a = f0.flatten(-2).permute(0, 2, 1)
    bb = f1.flatten(-2).permute(0, 2, 1)
    mask = shift_mask(h, w, splits, f0.dtype, f0.device) if splits > 1 else None
    c0, c1 = torch.cat((a, bb), 0), torch.cat((bb, a), 0)
    for i in range(num_layers):
        p = f"transformer.layers.{i}"
        shifted = i % 2 == 1                       # with_shift is a property of the layer, used only when splits > 1
        c0 = _layer(sd, p + ".self_attn", c0, c0, h, w, splits, shifted, mask, ffn=False)
        c0 = _layer(sd, p + ".cross_attn_ffn", c0, c1, h, w, splits, shifted, mask, ffn=True)
        c1 = torch.cat(c0.chunk(2, 0)[::-1], 0)
    a, bb = c0.chunk(2, 0)
    return (a.view(b, h, w, c).permute(0, 3, 1, 2).contiguous(), bb.view(b, h, w, c).permute(0, 3, 1, 2).contiguous())


def _grid(b: int, h: int, w: int, dtype=torch.float32, device=None):
    y, x = torch.meshgrid(torch.arange(h, device=device), torch.arange(w, device=device), indexing="ij")
    return torch.stack([x, y], 0).to(dtype)[None].repeat(b, 1, 1, 1)


def global_match(f0, f1):
    b, c, h, w = f0.shape
    corr = torch.matmul(f0.view(b, c, -1).permute(0, 2, 1), f1.view(b, c, -1)).view(b, h, w, h, w) / c ** 0.5
    init = _grid(b, h, w, f0.dtype, f0.device)
    prob = F.softmax(corr.view(b, h * w, h * w), dim=-1)
    return torch.matmul(prob, init.view(b, 2, -1).permute(0, 2, 1)).view(b, h, w, 2).permute(0, 3, 1, 2) - init


def local_match(f0, f1, radius: int):
    b, c, h, w = f0.shape
    init = _grid(b, h, w, f0.dtype, f0.device)
    coords = init.view(b, 2, -1).permute(0, 2, 1)
    k = 2 * radius + 1
    lin = torch.linspace(-radius, radius, k, dtype=f0.dtype, device=f0.device)
    gx, gy = torch.meshgrid([lin, lin], indexing="ij")
    window = torch.stack((gx, gy), -1).transpose(0, 1).reshape(-1, 2).repeat(b, 1, 1, 1)
    sample = coords.unsqueeze(-2) + window                                             # [B, H*W, k*k, 2]
    valid = (sample[..., 0] >= 0) & (sample[..., 0] < w) & (sample[..., 1] >= 0) & (sample[..., 1] < h)
    half = torch.tensor([(w - 1) / 2.0, (h - 1) / 2.0], dtype=f0.dtype, device=f0.device)
    feat = F.grid_sample(f1, (sample - half) / half, padding_mode="zeros", align_corners=True).permute(0, 2, 1, 3)
    corr = torch.matmul(f0.permute(0, 2, 3, 1).reshape(b, h * w, 1, c), feat).view(b, h * w, -1) / c ** 0.5
    corr[~valid] = -1e9
    prob = F.softmax(corr, -1)
    return torch.matmul(prob.unsqueeze(-2), sample).squeeze(-2).view(b, h, w, 2).permute(0, 3, 1, 2) - init


def propagate(sd, f0, flow, radius: int):
    p = "feature_flow_attn."
    b, c, h, w = f0.shape
    x = f0.view(b, c, h * w).permute(0, 2, 1)
    q = F.linear(x, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"])
    if radius <= 0:
        k = F.linear(q, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])        # the reference projects the projected query
        prob = torch.softmax(torch.matmul(q, k.permute(0, 2, 1)) / c ** 0.5, dim=-1)
        return torch.matmul(prob, flow.view(b, 2, h * w).permute(0, 2, 1)).view(b, h, w, 2).permute(0, 3, 1, 2)
    ks = 2 * radius + 1
    kp = F.linear(x, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"]).permute(0, 2, 1).reshape(b, c, h, w)
    kw = F.unfold(kp, kernel_size=ks, padding=radius).view(b, c, ks * ks, h, w).permute(0, 3, 4, 1, 2).reshape(b * h * w, c, ks * ks)
    fw = F.unfold(flow, kernel_size=ks, padding=radius).view(b, 2, ks * ks, h, w).permute(0, 3, 4, 2, 1).reshape(b * h * w, ks * ks, 2)
    prob = torch.softmax(torch.matmul(q.reshape(b * h * w, 1, c), kw) / c ** 0.5, dim=-1)
    return torch.matmul(prob, fw).view(b, h, w, 2).permute(0, 3, 1, 2).contiguous()


def upsample_convex(sd, flow, feature, factor: int = 4):
    x = F.conv2d(torch.cat((flow, feature), 1), sd["upsampler.0.weight"], sd["upsampler.0.bias"], padding=1)
    mask = F.conv2d(F.relu(x), sd["upsampler.2.weight"], sd["upsampler.2.bias"])
    b, _, h, w = flow.shape
    mask = torch.softmax(mask.view(b, 1, 9, factor, factor, h, w), dim=2)
    up = F.unfold(factor * flow, [3, 3], padding=1).view(b, 2, 9, 1, 1, h, w)
    return torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(b, 2, factor * h, factor * w)


def _warp(feature, flow):
    b, c, h, w = feature.shape
    co = _grid(b, h, w, flow.dtype, flow.device) + flow
    g = torch.stack([2 * co[:, 0] / (w - 1) - 1, 2 * co[:, 1] / (h - 1) - 1], -1)
    return F.grid_sample(feature, g, mode="bilinear", padding_mode="zeros", align_corners=True)


def gmflow(sd, img0, img1):
    """Flow img0 -> img1 at the images' resolution (images in [0, 1], sides multiples of 32)."""
    mean = torch.tensor([0.485, 0.456, 0.406], dtype=img0.dtype, device=img0.device).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], dtype=img0.dtype, device=img0.device).view(1, 3, 1, 1)
    feats = encoder(sd, torch.cat(((img0 - mean) / std, (img1 - mean) / std), 0))[::-1]     # low to high resolution
    flow = None
    for scale, (splits, corr_radius, prop_radius) in enumerate(((2, -1, -1), (8, 4, 1))):
        f0, f1 = torch.chunk(feats[scale], 2, 0)
        if scale > 0:
            flow = F.interpolate(flow, scale_factor=2, mode="bilinear", align_corners=True) * 2
            f1 = _warp(f1, flow)
        f0, f1 = add_position(f0, f1, splits)
        f0, f1 = transformer(sd, f0, f1, splits)
        pred = global_match(f0, f1) if corr_radius == -1 else local_match(f0, f1, corr_radius)
        flow = pred if flow is None else flow + pred
        flow = propagate(sd, f0, flow, prop_radius)
    return upsample_convex(sd, flow, f0)
