"""FLAVR (UNet_3D_3D "unet_18", 4 input frames) restated in PyTorch on the CPU: the checker for the library's FLAVR path.

Written from vfi_models/flavr/flavr_arch.py, resnet_3D.py and flavr/__init__.py; it does not import them.
``synthetic_state_dict`` makes seeded weights for the three checkpoints (they differ only in the number of outputs and
in whether the encoder convs carry a bias); ``flavr_forward`` is ``model(frames)[0]`` on already padded frames and
``interpolate`` adds the node's centred replicate padding and the crop.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

VARIANTS = {"2x": (1, False), "4x": (3, True), "8x": (7, True)}  # n_outputs, encoder conv bias (resnet_3D.useBias)
CKPT_VARIANT = {"FLAVR_2x.pth": "2x", "FLAVR_4x.pth": "4x", "FLAVR_8x.pth": "8x"}
ENC_C = (64, 128, 256, 512)
# decoder: (input channels, output channels, transposed)
DEC = ((512, 256, False), (512, 128, True), (256, 64, True), (128, 64, False), (128, 64, True))
# gain applied to the decoder and outconv weights of the goldens: default-initialised weights give an output that
# hardly differs from the mean (see tools/make_golden_flavr.py)
DEFAULT_GAIN = 1.6


def state_dict_spec(n_outputs: int = 1, enc_bias: bool = False) -> List[Tuple[str, Tuple[int, ...]]]:
    """UNet_3D_3D.state_dict() names and shapes, in order."""
    spec = [("encoder.stem.0.weight", (64, 3, 3, 7, 7))]
    if enc_bias:
        spec.append(("encoder.stem.0.bias", (64,)))
    cin = 64
    for l, co in enumerate(ENC_C):
        for b in range(2):
            p = f"encoder.layer{l + 1}.{b}."
            ci = cin if b == 0 else co
            spec.append((p + "conv1.0.weight", (co, ci, 3, 3, 3)))
            if enc_bias:
                spec.append((p + "conv1.0.bias", (co,)))
            spec.append((p + "conv2.0.weight", (co, co, 3, 3, 3)))
            if enc_bias:
                spec.append((p + "conv2.0.bias", (co,)))
            spec += [(p + "fg.attn_layer.0.weight", (co, co, 1, 1, 1)), (p + "fg.attn_layer.0.bias", (co,))]
            if b == 0 and l > 0:
                spec.append((p + "downsample.0.weight", (co, ci, 1, 1, 1)))
        cin = co
    for d, (ci, co, tr) in enumerate(DEC):
        if tr:
            spec += [(f"decoder.{d}.upconv.0.weight", (ci, co, 3, 4, 4)), (f"decoder.{d}.upconv.0.bias", (co,)),
                     (f"decoder.{d}.upconv.1.attn_layer.0.weight", (co, co, 1, 1, 1)),
                     (f"decoder.{d}.upconv.1.attn_layer.0.bias", (co,))]
        else:
            spec += [(f"decoder.{d}.conv.0.weight", (co, ci, 3, 3, 3)), (f"decoder.{d}.conv.0.bias", (co,)),
                     (f"decoder.{d}.conv.1.attn_layer.0.weight", (co, co, 1, 1, 1)),
                     (f"decoder.{d}.conv.1.attn_layer.0.bias", (co,))]
    spec += [("feature_fuse.conv.0.weight", (64, 256, 1, 1)),
             ("outconv.1.weight", (3 * n_outputs, 64, 7, 7)), ("outconv.1.bias", (3 * n_outputs,))]
    return spec


def synthetic_state_dict(seed: int = 0, variant: str = "2x", gain: float = DEFAULT_GAIN) -> Dict[str, torch.Tensor]:
    """Seeded He-normal conv weights (fan-in; a transposed conv's fan-in is cin * 3 * 2 * 2 taps per output), gate
    weights N(0, 1/C), small random biases; decoder and outconv weights scaled by ``gain``."""
    n_out, eb = VARIANTS[variant]
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_spec(n_out, eb):
        if name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=g)
        elif "attn_layer" in name:
            t = torch.randn(shape, generator=g) / shape[0] ** 0.5
        else:
            if ".upconv.0." in name:
                fan_in = shape[0] * 3 * 2 * 2
            else:
                fan_in = 1
                for s in shape[1:]:
                    fan_in *= s
            t = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
            if name.startswith("decoder.") or name.startswith("outconv."):
                t = t * gain
        sd[name] = t.float()
    return sd


def _gate(x, sd, p):
    m = x.mean(dim=(2, 3, 4), keepdim=True)
    return x * torch.sigmoid(F.conv3d(m, sd[p + ".weight"], sd[p + ".bias"]))


def flavr_forward(sd: Dict[str, torch.Tensor], frames: torch.Tensor) -> torch.Tensor:
    """frames: [B, 4, 3, H, W] (H, W multiples of 16, already padded) -> output 0 of the model, [B, 3, H, W]."""
    x = frames.permute(0, 2, 1, 3, 4).float()  # [B, 3, T, H, W]
    mean = x.mean(dim=(2, 3, 4), keepdim=True)
    x = x - mean
    b_ = lambda n: sd.get(n)  # noqa: E731  (absent encoder biases = none)
    x = F.relu(F.conv3d(x, sd["encoder.stem.0.weight"], b_("encoder.stem.0.bias"), stride=(1, 2, 2), padding=(1, 3, 3)))
    skips = [x]
    for l in range(4):
        for b in range(2):
            p = f"encoder.layer{l + 1}.{b}."
            s = (1, 2, 2) if (l in (1, 2) and b == 0) else 1
            y = F.relu(F.conv3d(x, sd[p + "conv1.0.weight"], b_(p + "conv1.0.bias"), stride=s, padding=1))
            y = F.conv3d(y, sd[p + "conv2.0.weight"], b_(p + "conv2.0.bias"), padding=1)
            y = _gate(y, sd, p + "fg.attn_layer.0")
            res = F.conv3d(x, sd[p + "downsample.0.weight"], stride=s) if (p + "downsample.0.weight") in sd else x
            x = F.relu(y + res)
        skips.append(x)
    x0, x1, x2, x3, x4 = skips
    dx = x4
    joins = [x3, x2, x1, x0, None]
    for d, (_, _, tr) in enumerate(DEC):
        if tr:
            p = f"decoder.{d}.upconv."
            y = F.conv_transpose3d(dx, sd[p + "0.weight"], sd[p + "0.bias"], stride=(1, 2, 2), padding=1)
        else:
            p = f"decoder.{d}.conv."
            y = F.conv3d(dx, sd[p + "0.weight"], sd[p + "0.bias"], padding=1)
        y = F.leaky_relu(_gate(y, sd, p + "1.attn_layer.0"), 0.2)
        dx = y if joins[d] is None else torch.cat([y, joins[d]], 1)
    dx = torch.cat(torch.unbind(dx, 2), 1)
    out = F.leaky_relu(F.conv2d(dx, sd["feature_fuse.conv.0.weight"]), 0.2)
    out = F.conv2d(F.pad(out, (3, 3, 3, 3), mode="reflect"), sd["outconv.1.weight"][:3], sd["outconv.1.bias"][:3])
    return out + mean.squeeze(2)


def pad_amounts(h: int, w: int, divisor: int = 16):
    """InputPadder: (left, right, top, bottom), centred."""
    ph = (((h // divisor) + 1) * divisor - h) % divisor
    pw = (((w // divisor) + 1) * divisor - w) % divisor
    return pw // 2, pw - pw // 2, ph // 2, ph - ph // 2


def interpolate(sd: Dict[str, torch.Tensor], frames: torch.Tensor) -> torch.Tensor:
    """frames: [4, H, W, 3] NHWC -> the node's new frame [H, W, 3]: pad (replicate, centred), model()[0], crop."""
    h, w = frames.shape[1:3]
    pl, pr, pt, pb = pad_amounts(h, w)
    x = F.pad(frames.permute(0, 3, 1, 2), (pl, pr, pt, pb), mode="replicate")
    with torch.no_grad():
        y = flavr_forward(sd, x.unsqueeze(0))[0]
    return y[:, pt:pt + h, pl:pl + w].permute(1, 2, 0)


def mean_only(frames: torch.Tensor) -> torch.Tensor:
    """The prediction that outputs the window's mean colour everywhere (what a model that does nothing would give)."""
    h, w = frames.shape[1:3]
    pl, pr, pt, pb = pad_amounts(h, w)
    x = F.pad(frames.permute(0, 3, 1, 2), (pl, pr, pt, pb), mode="replicate")
    return x.mean(dim=(0, 2, 3)).view(1, 1, 3).expand(h, w, 3)
