"""IFRNet-S / IFRNet-L restated in PyTorch on the CPU: the checker for the library's IFRNet path.

Written from vfi_models/ifrnet/IFRNet_{S,L}_arch.py and ifrnet/__init__.py; it does not import them.
``synthetic_state_dict`` makes seeded weights for either variant; ``forward`` is ``model(img0, img1, t, embt)`` as the
node calls it (the resize factor ``t`` is the loop's timestep and ``embt`` the node's ``scale_factor``, see
ifrnet_node.py), and ``ifrnet_macs`` counts the multiply-accumulates of one call from the shapes.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

# pyramid channels, ResBlock side channels, first conv kernel, decoder4..1 convblock channels, ConvT outputs
ARCH = {
    "S": dict(enc=(24, 36, 54, 72), side=24, k0=3, dc=(144, 162, 108, 72), dout=(58, 40, 28, 8)),
    "L": dict(enc=(64, 96, 144, 192), side=64, k0=7, dc=(384, 432, 288, 192), dout=(148, 100, 68, 8)),
}
CKPT_NAMES = ["IFRNet_S_Vimeo90K.pth", "IFRNet_L_Vimeo90K.pth", "IFRNet_S_GoPro.pth", "IFRNet_L_GoPro.pth"]
# gain of the decoder weights of the goldens: default-style weights give an almost trivial blend (see
# tools/make_golden_ifrnet.py)
DEFAULT_GAIN = 0.8


def variant_of(ckpt_name: str) -> str:
    """The node's rule (ifrnet/__init__.py:44)."""
    return "S" if "S" in ckpt_name else "L"


def _dec_in(a, k):
    if k == 0:
        return 2 * a["enc"][3] + 1
    return a["dout"][k - 1] - 4 + 2 * a["enc"][3 - k] + 4


def state_dict_spec(variant: str) -> List[Tuple[str, Tuple[int, ...]]]:
    """IRFNet_{S,L}.state_dict() names and shapes, in order."""
    a = ARCH[variant]
    spec = []
    cin = 3
    for l, co in enumerate(a["enc"]):
        for j in range(2):
            k = a["k0"] if (l == 0 and j == 0) else 3
            ci = cin if j == 0 else co
            p = f"encoder.pyramid{l + 1}.{j}."
            spec += [(p + "0.weight", (co, ci, k, k)), (p + "0.bias", (co,)), (p + "1.weight", (co,))]
        cin = co
    for k in range(4):
        p = f"decoder{4 - k}.convblock."
        C, s, ci = a["dc"][k], a["side"], _dec_in(a, k)
        spec += [(p + "0.0.weight", (C, ci, 3, 3)), (p + "0.0.bias", (C,)), (p + "0.1.weight", (C,))]
        for j in range(1, 5):
            n = s if j in (2, 4) else C
            q = p + f"1.conv{j}."
            spec += [(q + "0.weight", (n, n, 3, 3)), (q + "0.bias", (n,)), (q + "1.weight", (n,))]
        spec += [(p + "1.conv5.weight", (C, C, 3, 3)), (p + "1.conv5.bias", (C,)), (p + "1.prelu.weight", (C,))]
        spec += [(p + "2.weight", (C, a["dout"][k], 4, 4)), (p + "2.bias", (a["dout"][k],))]
    return spec


def synthetic_state_dict(variant: str = "S", seed: int = 0, gain: float = DEFAULT_GAIN) -> Dict[str, torch.Tensor]:
    """Seeded He-normal conv weights (fan-in; a ConvT(4, 2, 1) output sums cin * 2 * 2 taps), PReLU slopes drawn around
    0.25 (nn.PReLU's default), small random biases; decoder weights scaled by ``gain``."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_spec(variant):
        if len(shape) == 1 and (name.endswith("1.weight") or name.endswith("prelu.weight")):
            t = 0.25 + 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=g)
        else:
            fan_in = shape[0] * 4 if name.endswith("convblock.2.weight") else shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
            if name.startswith("decoder"):
                t = t * gain
        sd[name] = t.float()
    return sd


def resize(x, scale_factor):
    return F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=False)


def warp(img, flow):
    """grid from the flow's size, samples img (its own size) with align_corners=True, border padding."""
    B, _, H, W = flow.shape
    xx = torch.linspace(-1.0, 1.0, W, device=flow.device).view(1, 1, 1, W).expand(B, -1, H, -1)
    yy = torch.linspace(-1.0, 1.0, H, device=flow.device).view(1, 1, H, 1).expand(B, -1, -1, W)
    grid = torch.cat([xx, yy], 1).to(img)
    fl = torch.cat([flow[:, 0:1] / ((W - 1.0) / 2.0), flow[:, 1:2] / ((H - 1.0) / 2.0)], 1)
    return F.grid_sample(img, (grid + fl).permute(0, 2, 3, 1), mode="bilinear", padding_mode="border", align_corners=True)


def _convrelu(sd, p, x, stride=1, padding=1):
    return F.prelu(F.conv2d(x, sd[p + "0.weight"], sd[p + "0.bias"], stride, padding), sd[p + "1.weight"])


def _resblock(sd, p, x, s):
    out = _convrelu(sd, p + "conv1.", x)
    out = torch.cat([out[:, :-s], _convrelu(sd, p + "conv2.", out[:, -s:])], 1)
    out = _convrelu(sd, p + "conv3.", out)
    out = torch.cat([out[:, :-s], _convrelu(sd, p + "conv4.", out[:, -s:])], 1)
    return F.prelu(x + F.conv2d(out, sd[p + "conv5.weight"], sd[p + "conv5.bias"], padding=1), sd[p + "prelu.weight"])


def _decoder(sd, a, k, f_in):
    p = f"decoder{4 - k}.convblock."
    x = _convrelu(sd, p + "0.", f_in)
    x = _resblock(sd, p + "1.", x, a["side"])
    return F.conv_transpose2d(x, sd[p + "2.weight"], sd[p + "2.bias"], stride=2, padding=1)


def forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, t: float, embt: float,
            return_flows: bool = False):
    """img0, img1: [1, 3, H, W] -> [1, 3, H, W]: IRFNet.forward(img0, img1, scale_factor=t, timestep=embt)."""
    variant = "L" if sd["encoder.pyramid1.0.0.weight"].shape[-1] == 7 else "S"
    a = ARCH[variant]
    n, c, h, w = img0.shape
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    img0 = F.pad(img0, (0, pw - w, 0, ph - h))
    img1 = F.pad(img1, (0, pw - w, 0, ph - h))
    mean_ = torch.cat([img0, img1], 2).mean(1, keepdim=True).mean(2, keepdim=True).mean(3, keepdim=True)
    img0, img1 = img0 - mean_, img1 - mean_
    feats = []
    x = torch.cat([resize(img0, t), resize(img1, t)], 0)
    for l in range(4):
        p = f"encoder.pyramid{l + 1}."
        k = a["k0"] if l == 0 else 3
        x = _convrelu(sd, p + "0.", x, 2, k // 2)
        x = _convrelu(sd, p + "1.", x)
        feats.append(x)
    f4 = feats[3]
    e = torch.full((1, 1, f4.shape[2], f4.shape[3]), float(embt), device=f4.device)
    out = _decoder(sd, a, 0, torch.cat([f4[0:1], f4[1:2], e], 1))
    flow, ft = out[:, 0:4], out[:, 4:]
    for k in range(1, 4):
        f = feats[3 - k]
        f_in = torch.cat([ft, warp(f[0:1], flow[:, 0:2]), warp(f[1:2], flow[:, 2:4]), flow[:, 0:2], flow[:, 2:4]], 1)
        out = _decoder(sd, a, k, f_in)
        flow = out[:, 0:4] + 2.0 * resize(flow, 2.0)
        ft = out[:, 4:]
    mask = torch.sigmoid(ft[:, 0:1])
    res = ft[:, 1:]
    flow = resize(flow, 1.0 / t) * (1.0 / t)
    mask = resize(mask, 1.0 / t)
    res = resize(res, 1.0 / t)
    merged = mask * warp(img0, flow[:, 0:2]) + (1 - mask) * warp(img1, flow[:, 2:4]) + mean_
    pred = torch.clamp(merged + res, 0, 1)[:, :, :h, :w]
    if return_flows:
        return pred, flow[:, :, :h, :w], res[:, :, :h, :w]
    return pred


def geometry(h: int, w: int, t: float):
    """Sizes of one call: padded, resized input, pyramid levels 1..4, decoder 1 output, final resize (None: the
    reference would give an empty tensor or an output smaller than the frame)."""
    hp, wp = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    h0, w0 = math.floor(hp * t), math.floor(wp * t)
    if h0 < 1 or w0 < 1:
        return None
    lv = [(h0, w0)]
    for _ in range(4):
        lv.append(((lv[-1][0] + 1) // 2, (lv[-1][1] + 1) // 2))
    hq, wq = 16 * lv[4][0], 16 * lv[4][1]
    hf, wf = math.floor(hq * (1.0 / t)), math.floor(wq * (1.0 / t))
    if hf < h or wf < w:
        return None
    return dict(hp=hp, wp=wp, levels=lv, hq=hq, wq=wq, hf=hf, wf=wf)


def ifrnet_macs(variant: str, h: int, w: int, t: float) -> int:
    """Multiply-accumulates of the model's convolutions for one call (logical channels; no padding channels)."""
    a = ARCH[variant]
    g = geometry(h, w, t)
    lv = g["levels"]
    macs = 0
    cin = 3
    for l, co in enumerate(a["enc"]):
        ho, wo = lv[l + 1]
        k = a["k0"] if l == 0 else 3
        macs += 2 * ho * wo * co * (cin * k * k + co * 9)  # two frames
        cin = co
    gh, gw = lv[4]
    for k in range(4):
        C, s = a["dc"][k], a["side"]
        px = gh * gw
        macs += px * 9 * (C * _dec_in(a, k) + 3 * C * C + 2 * s * s)
        macs += 4 * px * C * a["dout"][k] * 4  # ConvT(4, 2, 1): 4 output pixels per input pixel, 2 x 2 taps each
        gh, gw = 2 * gh, 2 * gw
    return macs
