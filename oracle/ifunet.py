"""IFUNetModel restated in PyTorch on the CPU: the checker for the library's IFUnet path.

Written from vfi_models/ifunet/IFUNet_arch.py and ifunet/__init__.py; it does not import them.
``forward(sd, img0, img1, timestep, scale, ensemble)`` is ``IFUNetModel()(img0, img1, timestep=..., scale=...,
ensemble=...)`` in eval mode on [1, 3, H, W] frames; ``synthetic_state_dict`` makes seeded weights with the reference's
tensor names (608 entries, the unused DegCNN included); ``geometry`` gives every grid size of one call, or ``None`` where
the reference raises; ``ifunet_macs`` counts the multiply-accumulates of the convolutions of one call.

The keyword switches of ``forward`` are mutations of the model; tools/make_golden_ifunet.py scores each of them against
the goldens and records the figure.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

CKPT_NAMES = ["IFUNet.pth"]
BN_EPS = 1e-5
FEAT_C = (32, 64, 128, 256, 512)          # FeatureNet UNetConv levels 1..5 (out_planes 256)
BLOCK_C = (256, 128, 64)                  # IFBlock c of levels 0, 1, 2
BLOCK_L = (16, 8, 4)                      # their convex-upsampling factor
MASK_L = (16, 8, 4)                       # every IFBlock holds maskconvx16, x8 and x4
N_RRDB, RDB_GROW, RDB_FEAT = 6, 32, 64
RESYN_SCALES = (4, 2, 1)
# gain of the goldens' weights: see synthetic_state_dict
DEFAULT_GAIN = 1.0


def _conv_prelu(p, co, ci, k):
    return [(p + "0.weight", (co, ci, k, k)), (p + "0.bias", (co,)), (p + "1.weight", (co,))]


def _bn(p, c):
    return [(p + "weight", (c,)), (p + "bias", (c,)), (p + "running_mean", (c,)), (p + "running_var", (c,)),
            (p + "num_batches_tracked", ())]


def _spec_cbam(p, c):
    h = c // 16
    return ([(p + "ChannelGate.mlp.1.weight", (h, c)), (p + "ChannelGate.mlp.1.bias", (h,)),
             (p + "ChannelGate.mlp.3.weight", (c, h)), (p + "ChannelGate.mlp.3.bias", (c,)),
             (p + "SpatialGate.spatial.conv.weight", (1, 2, 7, 7))] + _bn(p + "SpatialGate.spatial.bn.", 1))


def _spec_conv_bn(p, co, ci):
    return [(p + "0.weight", (co, ci, 3, 3))] + _bn(p + "1.", co) + [(p + "2.weight", (co,))]


def state_dict_spec() -> List[Tuple[str, Tuple[int, ...]]]:
    """IFUNetModel().state_dict() names and shapes, in order (608 tensors; num_batches_tracked are int64 scalars)."""
    s = []
    f = "flownet.fmap."
    s += _conv_prelu(f + "conv0.", 17, 7, 1)
    cin = 17
    for i, co in enumerate(FEAT_C):
        p = f"{f}conv{i + 1}."
        s += _conv_prelu(p + "conv1.", co, cin, 3) + _conv_prelu(p + "conv2.", co, co, 3)
        if i > 0:
            s += _spec_cbam(p + "cbam.", co)
        cin = co
    for lvl, (cin, co, att) in zip((5, 4, 3), ((512, 256, True), (256, 128, False), (128, 64, False))):
        p = f"{f}deconv{lvl}."
        s += [(p + "deconv.0.weight", (cin, cin // 2, 4, 4)), (p + "deconv.0.bias", (cin // 2,)),
              (p + "deconv.1.weight", (cin // 2,))]
        s += _conv_prelu(p + "conv1.", cin // 2, cin, 3) + _conv_prelu(p + "conv2.", co, cin // 2, 3)
        if att:
            s += _spec_cbam(p + "cbam.", co)
    for b, c in enumerate(BLOCK_C):
        p = f"flownet.block{b}."
        for j in range(6):
            s += _conv_prelu(f"{p}convblock.{j}.", c, c, 3)
        s += [(p + "flowconv.weight", (4, c, 3, 3)), (p + "flowconv.bias", (4,))]
        for L in MASK_L:
            s += [(f"{p}maskconvx{L}.weight", (L * L * 9, c, 1, 1)), (f"{p}maskconvx{L}.bias", (L * L * 9,))]
    p = "fusionnet."
    s += [(p + "conv_first.weight", (64, 16, 3, 3)), (p + "conv_first.bias", (64,))]
    for r in range(N_RRDB):
        for d in range(1, 4):
            q = f"{p}body.{r}.rdb{d}."
            for k in range(1, 5):
                s += [(f"{q}conv{k}.weight", (32, 64 + 32 * (k - 1), 3, 3)), (f"{q}conv{k}.bias", (32,))]
            s += [(q + "conv5.weight", (64, 192, 3, 3)), (q + "conv5.bias", (64,))]
    for n in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
        s += [(f"{p}{n}.weight", (64, 64, 3, 3)), (f"{p}{n}.bias", (64,))]
    s += [(p + "conv_last.weight", (1, 64, 3, 3)), (p + "conv_last.bias", (1,))]
    for b, cin in enumerate((6, 12, 12)):
        p = f"refinenet.block{b}."
        s += _spec_conv_bn(p + "conv0.0.", 64, cin) + _spec_conv_bn(p + "conv0.1.", 128, 64) + _spec_conv_bn(p + "conv0.2.", 256, 128)
        for j in range(6):
            s += _spec_conv_bn(f"{p}convblock.{j}.", 256, 256)
        s += [(p + "lastconv.weight", (256, 4, 4, 4)), (p + "lastconv.bias", (4,))]
    p = "refinenet.degrad."
    s += _conv_prelu(p + "conv0.", 32, 3, 3)
    for j in (1, 2, 3):
        s += _conv_prelu(f"{p}conv{j}.", 32, 32, 3)
    s += [(p + "deconv.1.weight", (128, 32, 4, 4)), (p + "deconv.1.bias", (32,)), (p + "deconv.2.weight", (32,)),
          (p + "deconv.3.weight", (3, 32, 3, 3)), (p + "deconv.3.bias", (3,))]
    for c in (0, 1):
        s += _conv_prelu(f"refinenet.context{c}.0.", 16, 3, 3) + _conv_prelu(f"refinenet.context{c}.1.", 32, 16, 3)
    s += [("refinenet.decode.0.weight", (64, 32, 4, 4)), ("refinenet.decode.0.bias", (32,)),
          ("refinenet.decode.1.weight", (32, 3, 4, 4)), ("refinenet.decode.1.bias", (3,))]
    return s


def synthetic_state_dict(seed: int = 0, gain: float = DEFAULT_GAIN) -> Dict[str, torch.Tensor]:
    """Seeded weights: He-normal convs (fan-in; a ConvT(4, 2, 1) output sums cin * 2 * 2 taps) times ``gain``, PReLU
    slopes around 0.25, small biases, BatchNorm statistics near identity, CBAM MLPs with nn.Linear's default ranges.
    The heads that decide the motion get their own scales so that the flows move pixels by several pixels and the
    masks stay in the sigmoid's / softmax's working range (tools/make_golden_ifunet.py asserts both)."""
    g = torch.Generator().manual_seed(seed)
    spec = state_dict_spec()
    bn = {n[:-len("running_mean")] for n, _ in spec if n.endswith("running_mean")}
    sd = {}
    for name, shape in spec:
        if name.endswith("num_batches_tracked"):
            sd[name] = torch.tensor(0, dtype=torch.int64)
            continue
        last = name.rsplit(".", 1)[-1]
        if name[:-len(last)] in bn:
            if last == "weight":
                t = 1.0 + 0.1 * torch.randn(shape, generator=g)
            elif last == "bias":
                t = 0.05 * torch.randn(shape, generator=g)
            elif last == "running_mean":
                t = 0.05 * torch.randn(shape, generator=g)
            else:
                t = 0.6 + 0.8 * torch.rand(shape, generator=g)
        elif len(shape) == 1 and last == "weight":      # PReLU slopes
            t = 0.25 + 0.1 * torch.randn(shape, generator=g)
        elif last == "bias":
            t = 0.02 * torch.randn(shape, generator=g)
        elif "ChannelGate" in name:
            t = (torch.rand(shape, generator=g) * 2 - 1) * shape[1] ** -0.5
        else:
            convt = "deconv" in name or "lastconv" in name or "decode" in name
            fan_in = shape[0] * 4 if convt else shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5 * gain
            if "SpatialGate" in name:
                t = t * 0.5
            if name.endswith("flowconv.weight"):
                t = t * 1.0
            if "maskconv" in name:
                t = t * 0.5
            if "lastconv" in name:
                t = t * 0.15
            if "decode.1" in name:
                t = t * 0.5
            if "conv_last" in name:
                t = t * 0.25
            if name == "flownet.fmap.conv1.conv1.0.weight":   # the flow channels of levels 1 and 2: pixels, not [0, 1]
                t[:, 13:] *= 0.05
        sd[name] = t.float()
    return sd


# ---------------------------------------------------------------- geometry
def _down(n):
    return (n + 1) // 2


def geometry(h: int, w: int, scale: float) -> Optional[dict]:
    """Sizes of one call with the reference's arithmetic, or None where it raises: the padded frame; the flow net's input
    floor(n * scale) (n itself at scale 1) and its five stride-2 levels; the IFBlock grids (1/16, 1/8, 1/4 levels) and
    their flows, which must come back to the padded size (else torch.cat / the flow sum raises), and each UpConv's
    ConvT output, which must equal its skip connection (else torch.cat raises)."""
    if h < 1 or w < 1 or not (scale > 0) or not math.isfinite(scale):
        return None
    hp, wp = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    if scale != 1:
        h0, w0 = math.floor(float(hp) * scale), math.floor(float(wp) * scale)
    else:
        h0, w0 = hp, wp
    if h0 < 1 or w0 < 1:
        return None
    lv = [(h0, w0)]
    for _ in range(5):
        lv.append((_down(lv[-1][0]), _down(lv[-1][1])))
    inv = 1.0 / scale
    blocks = []
    for i in range(3):
        for up in range(4 - i, 5):   # deconv5 (level 4 skip), deconv4 (level 3), deconv3 (level 2)
            if 2 * lv[up + 1][0] != lv[up][0] or 2 * lv[up + 1][1] != lv[up][1]:
                return None
        gh, gw = lv[4 - i]
        L = BLOCK_L[i]
        fh, fw = math.floor(float(L * gh) * inv), math.floor(float(L * gw) * inv)
        if (fh, fw) != (hp, wp):
            return None
        blocks.append(dict(grid=(gh, gw), up=(L * gh, L * gw)))
    return dict(hp=hp, wp=wp, levels=lv, blocks=blocks)


def ifunet_macs(h: int, w: int, scale: float = 1.0, ensemble: bool = True) -> int:
    """Multiply-accumulates of every Conv2d / ConvTranspose2d of one call (logical channels), as forward hooks on the
    reference count them: output pixels x cin x cout x k x k (a ConvT(4, 2, 1): input pixels x cin x cout x 16)."""
    g = geometry(h, w, scale)
    hp, wp = g["hp"], g["wp"]
    lv = g["levels"]
    px = lambda t: t[0] * t[1]  # noqa: E731

    def cbam(n, c):
        return n * 2 * 49

    def fmap(level):
        m = 0
        if level == 0:
            m += px(lv[0]) * 7 * 17
        cin = 17
        for i, co in enumerate(FEAT_C):
            n = px(lv[i + 1])
            m += n * 9 * (cin * co + co * co)
            if i > 0:
                m += cbam(n, co)
            cin = co
        ups = ((512, 256, True), (256, 128, False), (128, 64, False))[:level + 1]
        for j, (ci, co, att) in enumerate(ups):
            nin, nout = px(lv[5 - j]), px(lv[4 - j])
            m += nin * ci * (ci // 2) * 16 + nout * 9 * (ci * (ci // 2) + (ci // 2) * co)
            if att:
                m += cbam(nout, co)
        return m

    def block(i):
        c, L = BLOCK_C[i], BLOCK_L[i]
        n = px(g["blocks"][i]["grid"])
        return n * (6 * 9 * c * c + 9 * c * 4 + c * L * L * 9)

    total = 0
    for i in range(3):
        total += (fmap(i) + block(i)) * (2 if ensemble else 1)
    q = (hp // 4) * (wp // 4)
    rdb = sum(9 * (64 + 32 * k) * 32 for k in range(4)) + 9 * 192 * 64
    total += q * 9 * 16 * 64 + q * N_RRDB * 3 * rdb + q * 9 * 64 * 64
    total += 4 * q * 9 * 64 * 64 + 16 * q * 9 * 64 * 64 * 2 + 16 * q * 9 * 64
    resyn = 0
    for b, s in enumerate(RESYN_SCALES):
        cin = 6 if b == 0 else 12
        h1, w1 = hp // s, wp // s
        n1, n2, n3 = px((h1 // 2, w1 // 2)), px((h1 // 4, w1 // 4)), px((h1 // 8, w1 // 8))
        resyn += n1 * 9 * cin * 64 + n2 * 9 * 64 * 128 + n3 * 9 * 128 * 256 + n3 * 6 * 9 * 256 * 256 + n3 * 256 * 4 * 16
    n1, n2 = (hp // 2) * (wp // 2), q
    resyn += 2 * (n1 * 9 * 3 * 16 + n2 * 9 * 16 * 32)
    resyn += n2 * 64 * 32 * 16 + n1 * 32 * 3 * 16
    total += 2 * resyn
    return total


# ---------------------------------------------------------------- building blocks
def resize(x, scale_factor, size_ratio=False):
    """F.interpolate(bilinear, align_corners=False) by a factor; size_ratio: the mutation that takes the source
    coordinates from the ratio of the sizes instead of the factor."""
    if size_ratio:
        h, w = x.shape[2:]
        return F.interpolate(x, size=(math.floor(h * scale_factor), math.floor(w * scale_factor)), mode="bilinear",
                             align_corners=False)
    return F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=False)


def warp(img, flow, padding_mode="border"):
    """grid from the flow's size, samples img (its own size) with align_corners=True, border padding."""
    B, _, H, W = flow.shape
    xx = torch.linspace(-1.0, 1.0, W, device=flow.device).view(1, 1, 1, W).expand(B, -1, H, -1)
    yy = torch.linspace(-1.0, 1.0, H, device=flow.device).view(1, 1, H, 1).expand(B, -1, -1, W)
    grid = torch.cat([xx, yy], 1).to(img)
    fl = torch.cat([flow[:, 0:1] / ((img.shape[3] - 1.0) / 2.0), flow[:, 1:2] / ((img.shape[2] - 1.0) / 2.0)], 1)
    return F.grid_sample(img, (grid + fl).permute(0, 2, 3, 1), mode="bilinear", padding_mode=padding_mode,
                         align_corners=True)


def _cp(sd, p, x, stride=1, padding=1):
    return F.prelu(F.conv2d(x, sd[p + "0.weight"], sd[p + "0.bias"], stride, padding), sd[p + "1.weight"])


def _bnorm(sd, p, x, skip):
    if skip:
        return x
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd[p + "weight"], sd[p + "bias"], False, 0.0,
                        BN_EPS)


def _cbam(sd, p, x, m, stats=None):
    def mlp(v):
        h = F.relu(F.linear(v, sd[p + "ChannelGate.mlp.1.weight"], sd[p + "ChannelGate.mlp.1.bias"]))
        return F.linear(h, sd[p + "ChannelGate.mlp.3.weight"], sd[p + "ChannelGate.mlp.3.bias"])
    att = mlp(x.mean(dim=(2, 3))) + mlp(x.amax(dim=(2, 3)))
    cg = torch.sigmoid(att)
    x = x * cg[:, :, None, None]
    comp = torch.cat([x.amax(1, keepdim=True), x.mean(1, keepdim=True)], 1)
    s = F.conv2d(comp, sd[p + "SpatialGate.spatial.conv.weight"], padding=3)
    s = _bnorm(sd, p + "SpatialGate.spatial.bn.", s, m.get("bn_skipped", False))
    sg = torch.sigmoid(s)
    if stats is not None:
        stats["gates"].append((float(cg.min()), float(cg.max()), float(sg.min()), float(sg.max())))
    return x * sg


def _fmap(sd, x, level, m, stats):
    f = "flownet.fmap."
    if x.shape[1] != 17:
        x = _cp(sd, f + "conv0.", x, 1, 0)
    skips = []
    for i in range(5):
        p = f"{f}conv{i + 1}."
        x = _cp(sd, p + "conv1.", x, 2, 1)
        x = _cp(sd, p + "conv2.", x)
        if i > 0:
            x = _cbam(sd, p + "cbam.", x, m, stats)
        skips.append(x)
    y = x
    for j, lvl in enumerate((5, 4, 3)[:level + 1]):
        p = f"{f}deconv{lvl}."
        up = F.prelu(F.conv_transpose2d(y, sd[p + "deconv.0.weight"], sd[p + "deconv.0.bias"], 2, 1),
                     sd[p + "deconv.1.weight"])
        y = _cp(sd, p + "conv1.", torch.cat([up, skips[3 - j]], 1))
        y = _cp(sd, p + "conv2.", y)
        if lvl == 5:
            y = _cbam(sd, p + "cbam.", y, m, stats)
    return y


def _ifblock(sd, i, x, scale, m):
    p = f"flownet.block{i}."
    L = BLOCK_L[i]
    y = x
    for j in range(6):
        y = _cp(sd, f"{p}convblock.{j}.", y)
    x = y + x
    tmp = F.conv2d(x, sd[p + "flowconv.weight"], sd[p + "flowconv.bias"], padding=1)
    mask = F.conv2d(x, sd[f"{p}maskconvx{L}.weight"], sd[f"{p}maskconvx{L}.bias"])
    N, _, H, W = tmp.shape
    if m.get("no_convex", False):
        up = F.interpolate(L * tmp, scale_factor=L, mode="bilinear", align_corners=False)
    else:
        mk = torch.softmax(mask.view(N, 1, 9, L, L, H, W), dim=2)
        uf = F.unfold(L * tmp, [3, 3], padding=1).view(N, 4, 9, 1, 1, H, W)
        up = torch.sum(mk * uf, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(N, 4, L * H, L * W)
    return resize(up, scale, m.get("resize_size_ratio", False)) * scale


def _flownet(sd, img0, img1, scale, timestep, ensemble, m, stats):
    t = (img0[:, :1].clone() * 0 + 1) * timestep
    pad_mode = "zeros" if m.get("zero_padded_warps", False) else "border"
    rr = m.get("resize_size_ratio", False)
    w0, w1 = img0, img1
    flow = None
    for i in range(3):
        passes = [(img0, img1, t)] + ([(img1, img0, 1 - t)] if ensemble else [])
        first = None
        for k, (a, b, tt) in enumerate(passes):
            base = flow if k == 0 else first
            if flow is None:
                x = torch.cat((a, b, tt), 1)
            else:
                x = torch.cat((a, b, tt, w0, w1), 1)
            if scale != 1:
                x = resize(x, scale, rr)
            if flow is not None:
                ft = base
                if k == 1 and m.get("ensemble_flow_swapped", False):
                    ft = torch.cat([ft[:, 2:4], ft[:, 0:2]], 1)
                if scale != 1:
                    ft = resize(ft, scale, rr) * scale
                x = torch.cat((x, ft), 1)
            d = _ifblock(sd, i, _fmap(sd, x, i, m, stats), 1.0 / scale, m)
            if k == 0:
                first = d if flow is None else flow + d
            else:
                second = d if flow is None else first + d
                first = (first + second) / 2
        flow = first
        w0 = warp(img0, flow[:, :2], pad_mode)
        w1 = warp(img1, flow[:, 2:4], pad_mode)
        if stats is not None:
            stats["flow_absmax"].append(float(flow.abs().max()))
    return flow, w0, w1


def _fusion(sd, img0, img1, w0, w1, flow):
    p = "fusionnet."
    lr = lambda v: F.leaky_relu(v, 0.2)  # noqa: E731
    cv = lambda n, v: F.conv2d(v, sd[p + n + ".weight"], sd[p + n + ".bias"], padding=1)  # noqa: E731
    x = resize(torch.cat((img0, img1, w0, w1), 1), 0.25)
    fl = resize(flow, 0.25) * 0.25
    feat = cv("conv_first", torch.cat((x, fl), 1))
    body = feat
    for r in range(N_RRDB):
        rin = body
        for d in range(1, 4):
            q = f"body.{r}.rdb{d}."
            xs = [body]
            for k in range(1, 5):
                xs.append(lr(cv(q + f"conv{k}", torch.cat(xs, 1))))
            body = cv(q + "conv5", torch.cat(xs, 1)) * 0.2 + body
        body = body * 0.2 + rin
    feat = feat + cv("conv_body", body)
    feat = lr(cv("conv_up1", F.interpolate(feat, scale_factor=2.0, mode="nearest")))
    feat = lr(cv("conv_up2", F.interpolate(feat, scale_factor=2.0, mode="nearest")))
    out = cv("conv_last", lr(cv("conv_hr", feat)))
    return torch.sigmoid(out)


def _conv_bn(sd, p, x, stride, m):
    y = F.conv2d(x, sd[p + "0.weight"], None, stride, 1)
    y = _bnorm(sd, p + "1.", y, m.get("bn_skipped", False))
    return F.prelu(y, sd[p + "2.weight"])


def _flowblock(sd, b, x, flow, scale, m):
    p = f"refinenet.block{b}."
    x = resize(x, 1.0 / scale)
    if flow is not None:
        x = torch.cat((x, resize(flow, 1.0 / scale) * 1.0 / scale), 1)
    feat = x
    for j in range(3):
        feat = _conv_bn(sd, f"{p}conv0.{j}.", feat, 2, m)
    y = feat
    for j in range(6):
        y = _conv_bn(sd, f"{p}convblock.{j}.", y, 1, m)
    feat = y + feat
    tmp = F.conv_transpose2d(feat, sd[p + "lastconv.weight"], sd[p + "lastconv.bias"], 2, 1)
    tmp = resize(tmp, scale * 4)
    return tmp[:, :2] * scale * 4, tmp[:, 2:3]


def _resyn(sd, imgs, deg, m, stats):
    pad_mode = "zeros" if m.get("zero_padded_warps", False) else "border"
    masks, warps = [], []
    for img in (imgs[:, :3], imgs[:, 3:6]):
        flow = mask = wi = None
        for b, s in enumerate(RESYN_SCALES):
            if flow is None:
                flow, mask = _flowblock(sd, b, torch.cat((img, deg), 1), None, s, m)
            else:
                fd, md = _flowblock(sd, b, torch.cat((img, deg, wi, mask), 1), flow, s, m)
                flow, mask = flow + fd, mask + md
            wi = warp(img, flow, pad_mode)
        fdn = resize(flow, 0.25) * 0.25
        c0 = warp(_cp(sd, "refinenet.context0.1.", _cp(sd, "refinenet.context0.0.", img, 2), 2), fdn, pad_mode)
        c1 = _cp(sd, "refinenet.context1.1.", _cp(sd, "refinenet.context1.0.", wi, 2), 2)
        d = F.conv_transpose2d(torch.cat((c0, c1), 1), sd["refinenet.decode.0.weight"], sd["refinenet.decode.0.bias"],
                               2, 1)
        d = torch.tanh(F.conv_transpose2d(d, sd["refinenet.decode.1.weight"], sd["refinenet.decode.1.bias"], 2, 1))
        masks.append(mask)
        warps.append(torch.clamp(wi + d, 0, 1))
        if stats is not None:
            stats["resyn_mask_range"].append((float(mask.min()), float(mask.max())))
            stats["resyn_flow_absmax"].append(float(flow.abs().max()))
    if not m.get("resyn_no_deg", False):
        masks.append(masks[-1] * 0)
        warps.append(deg)
    p = F.softmax(torch.clamp(torch.cat(masks, 1), -4, 4), dim=1)
    out = 0
    for i, wv in enumerate(warps):
        out = out + wv * p[:, i:i + 1]
    return out


MUTATIONS = ("ensemble_flow_swapped", "no_convex", "zero_padded_warps", "bn_skipped", "resize_size_ratio",
             "resyn_no_deg")


def forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, timestep: float = 0.5,
            scale: float = 1.0, ensemble: bool = True, return_stats: bool = False, **mutations):
    """IFUNetModel()(img0, img1, timestep=timestep, scale=scale, ensemble=ensemble) for [1, 3, H, W] frames (fp32).
    return_stats: also a dict of the flows' and masks' ranges and every CBAM gate's range."""
    for k in mutations:
        assert k in MUTATIONS, k
    m = {k: bool(v) for k, v in mutations.items()}
    n, c, h, w = img0.shape
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    img0 = F.pad(img0, (0, pw - w, 0, ph - h))
    img1 = F.pad(img1, (0, pw - w, 0, ph - h))
    stats = dict(gates=[], flow_absmax=[], resyn_mask_range=[], resyn_flow_absmax=[]) if return_stats else None
    flow, w0, w1 = _flownet(sd, img0, img1, scale, timestep, ensemble, m, stats)
    mask = _fusion(sd, img0, img1, w0, w1, flow)
    merged = w0 * mask + w1 * (1 - mask)
    out = _resyn(sd, torch.cat((img0, img1), 1), merged, m, stats)[:, :, :h, :w]
    if return_stats:
        stats["fusion_mask_range"] = (float(mask.min()), float(mask.max()))
        return out, stats
    return out
