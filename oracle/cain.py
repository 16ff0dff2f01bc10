"""CAIN (depth 3) restated in PyTorch on the CPU: the checker for the library's CAIN path.

Written from vfi_models/cain/cain_arch.py, common.py and cain/__init__.py; it does not import them.
``forward(sd, img0, img1)`` is ``CAIN(depth=3)(img0, img1)[0]`` on [1, 3, H, W] frames; ``synthetic_state_dict`` makes
seeded weights with the reference's tensor names; ``cain_macs`` counts the multiply-accumulates of one call and
``geometry`` gives the padded size, the 1/8 grid and the crop (``None`` where the reference raises).

The keyword switches of ``forward`` are mutations of the model (zero padding in ConvNorm, no channel attention, the mean
not added back, the pixel-shuffle sub-pixel order transposed); tools/make_golden_cain.py shows that each of them moves
the output far from the goldens.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

CKPT_NAMES = ["pretrained_cain.pth"]
N_GROUPS, N_BLOCKS, N_FEATS, N_HIDDEN = 5, 12, 192, 12   # Interpolation(5, 12, 3 * 4**3), CALayer reduction 16
PREFIX = "encoder.interpolate."
# gain of the 3x3 conv weights of the goldens: with nn.Conv2d's default ranges each residual branch is so small that the
# trunk barely differs from its input, and a wrong border or attention would hardly show (see tools/make_golden_cain.py)
DEFAULT_GAIN = 1.25


def state_dict_spec() -> List[Tuple[str, Tuple[int, ...]]]:
    """CAIN(depth=3).state_dict() names and shapes, in order (494 tensors)."""
    C, R = N_FEATS, N_HIDDEN
    spec = [(PREFIX + "headConv.weight", (C, 2 * C, 3, 3)), (PREFIX + "headConv.bias", (C,))]
    for g in range(N_GROUPS):
        for r in range(N_BLOCKS):
            p = f"{PREFIX}body.{g}.body.{r}.body."
            spec += [(p + "0.conv.weight", (C, C, 3, 3)), (p + "0.conv.bias", (C,)),
                     (p + "2.conv.weight", (C, C, 3, 3)), (p + "2.conv.bias", (C,)),
                     (p + "3.conv_du.0.weight", (R, C, 1, 1)), (p + "3.conv_du.0.bias", (R,)),
                     (p + "3.conv_du.2.weight", (C, R, 1, 1)), (p + "3.conv_du.2.bias", (C,))]
        p = f"{PREFIX}body.{g}.body.{N_BLOCKS}.conv."
        spec += [(p + "weight", (C, C, 3, 3)), (p + "bias", (C,))]
    spec += [(PREFIX + "tailConv.weight", (C, C, 3, 3)), (PREFIX + "tailConv.bias", (C,))]
    return spec


def synthetic_state_dict(seed: int = 0, gain: float = DEFAULT_GAIN) -> Dict[str, torch.Tensor]:
    """Seeded weights with nn.Conv2d's default ranges, U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weights and biases; the
    3x3 conv weights scaled by ``gain``."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_spec():
        fan_in = 1
        for s in (shape[1:] if len(shape) > 1 else ()):
            fan_in *= s
        if len(shape) == 1:   # the bias of the weight just before it
            prev = sd[name[:-len("bias")] + "weight"]
            fan_in = prev[0].numel()
        bound = fan_in ** -0.5
        sd[name] = (torch.rand(shape, generator=g) * 2 - 1) * bound
        if len(shape) == 4 and shape[-1] == 3:
            sd[name] = sd[name] * gain
    return sd


def geometry(h: int, w: int) -> Optional[dict]:
    """InOutPaddings: each axis padded up to a multiple of 128 (p // 2 before, p - p // 2 after) by ReflectionPad2d, which
    needs every side's padding to be smaller than the axis; the trunk runs on the 1/8 grid."""
    def axis(n):
        p = 0 if n % 128 == 0 else (n // 128 + 1) * 128 - n
        return p // 2, p - p // 2
    top, bottom = axis(h)
    left, right = axis(w)
    if h < 1 or w < 1 or max(top, bottom) >= h or max(left, right) >= w:
        return None
    hp, wp = h + top + bottom, w + left + right
    return dict(hp=hp, wp=wp, gh=hp // 8, gw=wp // 8, top=top, left=left)


def cain_macs(h: int, w: int) -> int:
    """Multiply-accumulates of one call: headConv (384 -> 192), 5 x (12 x 2 + 1) body convs and tailConv, all 3x3 on the
    1/8 grid, plus the channel-attention MLPs."""
    g = geometry(h, w)
    cells = g["gh"] * g["gw"]
    C = N_FEATS
    conv = cells * 9 * C * (2 * C + (N_GROUPS * (2 * N_BLOCKS + 1) + 1) * C)
    return conv + N_GROUPS * N_BLOCKS * 2 * C * N_HIDDEN


def space_to_depth(x: torch.Tensor, transpose: bool = False) -> torch.Tensor:
    """pixel_shuffle(x, 1/8): channel c, sub-pixel (sy, sx) -> c * 64 + sy * 8 + sx (transpose: c * 64 + sx * 8 + sy)."""
    b, c, h, w = x.shape
    v = x.reshape(b, c, h // 8, 8, w // 8, 8)
    v = v.permute(0, 1, 5, 3, 2, 4) if transpose else v.permute(0, 1, 3, 5, 2, 4)
    return v.reshape(b, c * 64, h // 8, w // 8)


def depth_to_space(x: torch.Tensor, transpose: bool = False) -> torch.Tensor:
    """pixel_shuffle(x, 8), the inverse of space_to_depth."""
    b, c, h, w = x.shape
    v = x.reshape(b, c // 64, 8, 8, h, w)
    v = v.permute(0, 1, 4, 3, 5, 2) if transpose else v.permute(0, 1, 4, 2, 5, 3)
    return v.reshape(b, c // 64, h * 8, w * 8)


def forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, pad: str = "reflect",
            attention: bool = True, add_mean: bool = True, transpose_shuffle: bool = False,
            return_gates: bool = False):
    """CAIN(depth=3)(img0, img1)[0] for [B, 3, H, W] frames (fp32).  return_gates: also every channel-attention gate
    [60, B, 192] and the largest |feature| of the trunk."""
    _, _, H, W = img0.shape
    geo = geometry(H, W)
    if geo is None:
        raise ValueError(f"CAIN cannot reflection-pad a {H} x {W} frame")
    t, l = geo["top"], geo["left"]
    pads = (l, geo["wp"] - W - l, t, geo["hp"] - H - t)
    m0 = img0.mean(dim=(2, 3), keepdim=True)
    m1 = img1.mean(dim=(2, 3), keepdim=True)
    x0 = space_to_depth(F.pad(img0 - m0, pads, mode="reflect"), transpose_shuffle)
    x1 = space_to_depth(F.pad(img1 - m1, pads, mode="reflect"), transpose_shuffle)

    def conv_norm(name, x):   # ConvNorm: ReflectionPad2d(1) + 3x3 conv
        return F.conv2d(F.pad(x, (1, 1, 1, 1), mode=pad), sd[name + ".weight"], sd[name + ".bias"])

    gates, peak = [], 0.0
    x = F.conv2d(torch.cat([x0, x1], 1), sd[PREFIX + "headConv.weight"], sd[PREFIX + "headConv.bias"], padding=1)
    res = x
    for g in range(N_GROUPS):
        gin = res
        for r in range(N_BLOCKS):
            p = f"{PREFIX}body.{g}.body.{r}.body."
            y = F.leaky_relu(conv_norm(p + "0.conv", res), 0.2)
            y = conv_norm(p + "2.conv", y)
            if attention:
                m = y.mean(dim=(2, 3), keepdim=True)
                a = F.relu(F.conv2d(m, sd[p + "3.conv_du.0.weight"], sd[p + "3.conv_du.0.bias"]))
                gate = torch.sigmoid(F.conv2d(a, sd[p + "3.conv_du.2.weight"], sd[p + "3.conv_du.2.bias"]))
                gates.append(gate.flatten(1))
                y = y * gate
            res = y + res
            peak = max(peak, float(res.abs().max()))
        res = conv_norm(f"{PREFIX}body.{g}.body.{N_BLOCKS}.conv", res) + gin
    res = res + x
    out = F.conv2d(res, sd[PREFIX + "tailConv.weight"], sd[PREFIX + "tailConv.bias"], padding=1)
    out = depth_to_space(out, transpose_shuffle)[:, :, t:t + H, l:l + W]
    if add_mean:
        out = out + (m0 + m1) / 2
    if return_gates:
        return out, torch.stack(gates) if gates else None, peak
    return out
