"""CPU restatement (fp32) of the reference's Sepconv ("revisiting sepconv") path - SURVEY.md section 8 row a12.
TEST INFRASTRUCTURE ONLY.

Follows ``vfi_models/sepconv/sepconv_enhanced.py`` (``Network`` :536-706 with its ``Basic`` / ``Encode`` / ``Decode``
building blocks :47-533) and the node ``vfi_models/sepconv/__init__.py:32-57`` (``generic_frame_loop`` with
``use_timestep=False``) of Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc.  ATen operators are called functionally; the
one custom op, ``sepconv_func`` (``vfi_models/ops/cupy_ops/sepconv.py:86-117``), is ``oracle.ops_ref.sepconv``.

Pinning: ``tools/make_golden_sepconv.py`` runs the UNMODIFIED ``Network`` on seeded weights with ``vfi_models.ops``
pre-seeded by that op restatement (cupy cannot be imported here, SURVEY.md section 8c) and stores the outputs in
``tests/golden/sepconv_*.npz``; ``tests/test_oracle_sepconv.py`` holds this file to them.  So the network around the op
is pinned to the reference; the op itself is pinned only to its published loop (parity of the op: unpinned).

16-bit-faithful mode.  ``network_forward(..., operand="float16" | "bfloat16")`` evaluates the same graph in float64 and
rounds to 16 bits (``oracle.rife46.q16``) exactly where the CUDA library stores a 16-bit value, so that a comparison with
the library measures accumulation order only.  With ``operand=None`` (the default) nothing changes: the fp32 graph above
runs as it always did, bit for bit.  It also runs on CUDA tensors (the weights follow the frames' device).  T is the
operand type; where the library stores each tensor (csrc/sepconv.cu, csrc/sepconv_elem.cu, csrc/streamconv.cu's EXT
epilogue: ``acc + bias``, PReLU, ``+ residual``, then the T store):

| tensor | library | operand mode |
|---|---|---|
| stats of the replicate-padded pair | ``sep_stats``: double sums; mean, ``inv = 1 / (std + 1e-7)`` (unbiased std) in fp32 | float64 sums, mean / std / inv rounded to fp32 the same way |
| normalised input | ``sep_input_conv``: ``(x - mean) * inv`` in fp32 | the same two fp32 roundings |
| netInput + the PReLU of ``netEncode.0.netVer.1.netMain.0`` | ``sep_input_conv``: fp32 weights, fp32 FMAs, stored in T (space-to-depth) | unrounded weights, ``round_T(prelu(y))`` |
| every 3x3 conv (streamconv) | weights packed to T, fp32 bias, PReLU, then the residual, T store | ``round_T(w)``, bias as is, ``round_T(prelu(y) + res)`` |
| PReLU of rows 2..4 before the stride-2 conv | ``prelu_s2d16``: fp32 on T inputs, stored in T | ``round_T(prelu(x))`` |
| PReLU before ``netHor``'s first conv | ``prelu16``, stored in T | ``round_T(prelu(x))`` |
| PReLU + bilinear x2 before ``netVer`` and the heads (slope 1) | ``prelu_up2_16``: PReLU first, fp32 interpolation, T | ``round_T(up(prelu(x)))`` |
| ``netHor``'s residual conv | residual fused: one rounding | ``round_T(conv + x)`` |
| ``netVer``'s last conv, up-sampled size == the row's | residual fused: one rounding | ``round_T(conv + x)`` |
| ``netVer``'s last conv, up-sampled size != the row's | conv stored in T, then ``add_crop16`` adds it and stores in T: two roundings | ``round_T(x + crop(round_T(conv)))`` |
| the 51 coefficients of each head | T (streamconv), widened exactly to fp32 by ``sep_coeff_nchw`` | ``round_T(conv)`` |
| padded frames, the op, normalise and crop | fp32 (``sep_pad_input``, ``sepconv_tile_kernel``, ``sep_finish``) | float64 |

In operand mode ``debug["levels"][0]`` is what the library stores for row 0: netInput's output after that PReLU, in T.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

from . import ops_ref
from .rife46 import _dt, q16

CHANNELS = (32, 64, 128, 256, 512)  # Network.intChannels, sepconv_enhanced.py:541
KSIZE = 51                           # :598-612


def state_dict_spec() -> List[Tuple[str, Tuple[int, ...]]]:
    """Names / shapes of ``Network().state_dict()`` in the reference's order (88 tensors, 13,560,102 values)."""
    spec: List[Tuple[str, Tuple[int, ...]]] = [("netInput.weight", (16, 3, 3, 3)), ("netInput.bias", (16,))]

    def basic(prefix, idx_prelu0, convs):
        # convs: list of (module index, cin, cout); a PReLU (one scalar) precedes each conv except where idx is None
        for (pi, ci, cin, cout) in convs:
            if pi is not None:
                spec.append((f"{prefix}.netMain.{pi}.weight", (1,)))
            spec.append((f"{prefix}.netMain.{ci}.weight", (cout, cin, 3, 3)))
            spec.append((f"{prefix}.netMain.{ci}.bias", (cout,)))

    for r in range(1, 5):   # Encode: prelu-sconv-prelu-conv (:549-556)
        basic(f"netEncode.0.netVer.{r}", 0, [(0, 1, CHANNELS[r - 1], CHANNELS[r]), (2, 3, CHANNELS[r], CHANNELS[r])])
    for k, r in enumerate((4, 3, 2, 1)):   # Decode rows, coarse first: prelu-conv-prelu-conv+skip (:571-580)
        basic(f"netDecode.0.netHor.{k}", 0, [(0, 1, CHANNELS[r], CHANNELS[r]), (2, 3, CHANNELS[r], CHANNELS[r])])
    for k, r in enumerate((3, 2, 1), start=1):   # prelu-up-conv-prelu-conv
        basic(f"netDecode.0.netVer.{k}", 0, [(0, 2, CHANNELS[r + 1], CHANNELS[r]), (3, 4, CHANNELS[r], CHANNELS[r])])
    for head in ("netVerone", "netVertwo", "netHorone", "netHortwo"):   # up-conv-prelu-conv (:583-598)
        basic(head, None, [(None, 1, 64, 64), (2, 3, 64, KSIZE)])
    return spec


def synthetic_state_dict(seed: int = 0, head_gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for ``sepconv.pth``: variance-preserving uniform conv weights, PReLU slopes in [0.1, 0.4], and head
    biases shaped as a positive bump around the kernel centre so the 51x51 kernels are blur-like and their sum (the
    normaliser, :697-699) stays away from zero, like a trained model's.  The 51-channel head weights are scaled by
    0.02 x ``head_gain``: at the default gain of 1 the coefficients are nearly the bias alone; a larger gain makes the
    trunk's share of them visible (gain 1 gives the same tensors as before the argument existed)."""
    g = torch.Generator().manual_seed(2000 + seed)
    sd: Dict[str, torch.Tensor] = {}
    bump = torch.exp(-0.5 * ((torch.arange(KSIZE, dtype=torch.float32) - 25.0) / 3.0) ** 2)
    for name, shape in state_dict_spec():
        if shape == (1,):
            v = 0.1 + 0.3 * torch.rand(1, generator=g)
        elif name.endswith(".bias"):
            v = (torch.rand(shape, generator=g) * 2 - 1) * 0.05
            if shape == (KSIZE,):
                v = v * 0.2 + bump
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            v = (torch.rand(shape, generator=g) * 2 - 1) * (6.0 / (1.1 * fan_in)) ** 0.5
            if shape[0] == KSIZE:
                v = v * 0.02
                if head_gain != 1.0:
                    v = v * head_gain
        sd[name] = v.float()
    return sd


def _basic(sd, prefix: str, x: torch.Tensor, kind: str) -> torch.Tensor:
    """Basic.forward (:295-306) for the four layer strings the network uses."""
    w = lambda i: sd[f"{prefix}.netMain.{i}.weight"]   # noqa: E731
    b = lambda i: sd[f"{prefix}.netMain.{i}.bias"]     # noqa: E731
    if kind == "enc":      # prelu(0.25)-sconv(3)-prelu(0.25)-conv(3)
        y = F.conv2d(F.prelu(x, w(0)), w(1), b(1), stride=2, padding=1)
        return F.conv2d(F.prelu(y, w(2)), w(3), b(3), padding=1)
    if kind == "hor":      # prelu-conv-prelu-conv+skip (identity shortcut: equal channels, stride 1 - :222-223)
        y = F.conv2d(F.prelu(x, w(0)), w(1), b(1), padding=1)
        return F.conv2d(F.prelu(y, w(2)), w(3), b(3), padding=1) + x
    if kind == "dec":      # prelu-up(bilinear)-conv-prelu-conv
        y = F.interpolate(F.prelu(x, w(0)), scale_factor=2.0, mode="bilinear", align_corners=False)
        y = F.conv2d(y, w(2), b(2), padding=1)
        return F.conv2d(F.prelu(y, w(3)), w(4), b(4), padding=1)
    if kind == "head":     # up(bilinear)-conv-prelu-conv
        y = F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=False)
        y = F.conv2d(y, w(1), b(1), padding=1)
        return F.conv2d(F.prelu(y, w(2)), w(3), b(3), padding=1)
    raise ValueError(kind)


def network_forward(sd, x1: torch.Tensor, x2: torch.Tensor, debug: dict = None, operand: str = None) -> torch.Tensor:
    """Network.forward, sepconv_enhanced.py:605-706.  x1, x2: [B,3,H,W] fp32.  ``operand``: see the module docstring."""
    dt = _dt(operand)
    if dt is not None:
        return _forward16(sd, x1, x2, debug, dt)
    with torch.no_grad():
        W_, H_ = x1.shape[3], x1.shape[2]
        padr, padb = (2 - (W_ % 2)) % 2, (2 - (H_ % 2)) % 2
        one = F.pad(x1, [0, padr, 0, padb], mode="replicate")
        two = F.pad(x2, [0, padr, 0, padb], mode="replicate")
        stack = torch.stack([one, two], 1)
        mean = stack.view(stack.shape[0], -1).mean(1, True).view(-1, 1, 1, 1)
        std = stack.view(stack.shape[0], -1).std(1, True).view(-1, 1, 1, 1)
        seq = [(f - mean) / (std + 0.0000001) for f in (one, two)]
        feat = [F.conv2d(s, sd["netInput.weight"], sd["netInput.bias"], padding=1) for s in seq]
        lv = [torch.cat(feat, 1)]
        # Encode (:345-369): rows 1..4 = Ver(previous row); row 0 passes through
        for r in range(1, 5):
            lv.append(_basic(sd, f"netEncode.0.netVer.{r}", lv[r - 1], "enc"))
        # Decode (:447-497): Hor on rows 4..1, then Ver added on rows 3..1 (cropped by one where the coarser row is odd)
        for k, r in enumerate((4, 3, 2, 1)):
            lv[r] = _basic(sd, f"netDecode.0.netHor.{k}", lv[r], "hor")
        for k, r in enumerate((3, 2, 1), start=1):
            v = _basic(sd, f"netDecode.0.netVer.{k}", lv[r + 1], "dec")
            if v.shape[2] == lv[r].shape[2] + 1:
                v = v[:, :, :-1]
            if v.shape[3] == lv[r].shape[3] + 1:
                v = v[:, :, :, :-1]
            lv[r] = lv[r] + v
        out = lv[1]
        p = int(math.floor(0.5 * KSIZE))
        onep = F.pad(one, [p, p, p, p], mode="replicate")
        twop = F.pad(two, [p, p, p, p], mode="replicate")
        onep = torch.cat([onep, onep.new_ones([onep.shape[0], 1, onep.shape[2], onep.shape[3]])], 1)
        twop = torch.cat([twop, twop.new_ones([twop.shape[0], 1, twop.shape[2], twop.shape[3]])], 1)
        ver1 = _basic(sd, "netVerone", out, "head")
        ver2 = _basic(sd, "netVertwo", out, "head")
        hor1 = _basic(sd, "netHorone", out, "head")
        hor2 = _basic(sd, "netHortwo", out, "head")
        if debug is not None:
            debug.update(levels=lv, ver1=ver1, ver2=ver2, hor1=hor1, hor2=hor2, mean=mean, std=std)
        res = ops_ref.sepconv(onep, ver1, hor1) + ops_ref.sepconv(twop, ver2, hor2)
        norm = res[:, -1:, :, :].clone()
        norm[norm.abs() < 0.01] = 1.0
        res = res[:, :-1, :, :] / norm
        return res[:, :, :H_, :W_]


# ------------------------------------------------------------------------------------------------- 16-bit-faithful mode
def op64(ten_in: torch.Tensor, ver: torch.Tensor, hor: torch.Tensor, absolute: bool = False) -> torch.Tensor:
    """The separable convolution of ``ops_ref.sepconv`` in float64 on the inputs' device, without rounding the products:
    out[n,c,y,x] = sum_fy ver[n,fy,y,x] sum_fx hor[n,fx,y,x] in[n,c,y+fy,x+fx].  ``absolute``: the same sum of
    absolute values (the S of an error bound)."""
    n, c, hp, wp = ten_in.shape
    kv, kh = ver.shape[1], hor.shape[1]
    h, w = ver.shape[2], ver.shape[3]
    assert hp == h + kv - 1 and wp == w + kh - 1
    x, v, hz = ten_in.double(), ver.double(), hor.double()
    if absolute:
        x, v, hz = x.abs(), v.abs(), hz.abs()
    out = torch.zeros(n, c, h, w, dtype=torch.float64, device=ten_in.device)
    for fy in range(kv):
        rd = torch.zeros_like(out)
        for fx in range(kh):
            rd.addcmul_(x[:, :, fy:fy + h, fx:fx + w], hz[:, fx:fx + 1])
        out.addcmul_(rd, v[:, fy:fy + 1])
    return out


def pad_frames(x: torch.Tensor) -> torch.Tensor:
    """:611-618 and :644-681: replicate padding to even, then by 25, and a channel of ones (float64)."""
    H_, W_ = x.shape[2], x.shape[3]
    p = KSIZE // 2
    x = F.pad(x.double(), [0, W_ % 2, 0, H_ % 2], mode="replicate")
    x = F.pad(x, [p, p, p, p], mode="replicate")
    return torch.cat([x, x.new_ones([x.shape[0], 1, x.shape[2], x.shape[3]])], 1)


NORM_EPS = float(torch.tensor(0.01, dtype=torch.float32))   # :697-698 compares an fp32 tensor: 0.01 in fp32


def finish(res: torch.Tensor, H_: int, W_: int) -> torch.Tensor:
    """:692-702: divide by the ones channel's result (|n| < 0.01 -> 1) and crop."""
    norm = res[:, -1:].clone()
    norm[norm.abs() < NORM_EPS] = 1.0
    return (res[:, :-1] / norm)[:, :, :H_, :W_]


def _forward16(sd, x1: torch.Tensor, x2: torch.Tensor, debug, dt) -> torch.Tensor:
    dev = x1.device
    with torch.no_grad():
        t = {k: v.to(dev) for k, v in sd.items()}
        slope = lambda name: float(t[name + ".weight"])   # noqa: E731
        prelu = lambda x, s: torch.where(x > 0, x, s * x)   # noqa: E731

        def conv(x, prefix, i, stride=1):
            w, b = t[f"{prefix}.netMain.{i}.weight"], t[f"{prefix}.netMain.{i}.bias"]
            return F.conv2d(x, q16(w, dt), b.double(), stride=stride, padding=1)

        def up(x):
            return F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=False)

        H_, W_ = x1.shape[2], x1.shape[3]
        one = F.pad(x1.float(), [0, W_ % 2, 0, H_ % 2], mode="replicate")
        two = F.pad(x2.float(), [0, W_ % 2, 0, H_ % 2], mode="replicate")
        stack = torch.stack([one, two], 1).reshape(one.shape[0], -1).double()
        cnt = float(stack.shape[1])
        ssum, ssq = stack.sum(1), (stack * stack).sum(1)
        mean_d = ssum / cnt                                          # sep_input_conv_kernel's formula
        var_d = (ssq - cnt * mean_d * mean_d) / (cnt - 1.0)
        mean = mean_d.float().view(-1, 1, 1, 1)
        std = var_d.clamp(min=0).sqrt().float().view(-1, 1, 1, 1)
        inv = 1.0 / (std + torch.tensor(0.0000001, dtype=torch.float32, device=dev))
        w_in, b_in = t["netInput.weight"].double(), t["netInput.bias"].double()
        feat = [F.conv2d(((f - mean) * inv).double(), w_in, b_in, padding=1) for f in (one, two)]
        lv = [q16(prelu(torch.cat(feat, 1), slope("netEncode.0.netVer.1.netMain.0")), dt)]
        for r in range(1, 5):
            p = f"netEncode.0.netVer.{r}"
            a = lv[0] if r == 1 else q16(prelu(lv[r - 1], slope(p + ".netMain.0")), dt)
            y = q16(prelu(conv(a, p, 1, stride=2), slope(p + ".netMain.2")), dt)
            lv.append(q16(conv(y, p, 3), dt))
        for k, r in enumerate((4, 3, 2, 1)):
            p = f"netDecode.0.netHor.{k}"
            a = q16(prelu(lv[r], slope(p + ".netMain.0")), dt)
            y = q16(prelu(conv(a, p, 1), slope(p + ".netMain.2")), dt)
            lv[r] = q16(conv(y, p, 3) + lv[r], dt)
        for k, r in enumerate((3, 2, 1), start=1):
            p = f"netDecode.0.netVer.{k}"
            a = q16(up(prelu(lv[r + 1], slope(p + ".netMain.0"))), dt)
            y = q16(prelu(conv(a, p, 2), slope(p + ".netMain.3")), dt)
            v = conv(y, p, 4)
            h, w = lv[r].shape[2], lv[r].shape[3]
            if v.shape[2:] == lv[r].shape[2:]:
                lv[r] = q16(v + lv[r], dt)
            else:                                                    # stored, then add_crop16
                lv[r] = q16(lv[r] + q16(v, dt)[:, :, :h, :w], dt)
        u = q16(up(lv[1]), dt)
        coef = []
        for head in ("netVerone", "netVertwo", "netHorone", "netHortwo"):
            y = q16(prelu(conv(u, head, 1), slope(head + ".netMain.2")), dt)
            coef.append(q16(conv(y, head, 3), dt))
        if debug is not None:
            debug.update(levels=lv, ver1=coef[0], ver2=coef[1], hor1=coef[2], hor2=coef[3], mean=mean.double(),
                         std=std.double(), stats=torch.stack([ssum, ssq], 1))
        res = op64(pad_frames(x1), coef[0], coef[2]) + op64(pad_frames(x2), coef[1], coef[3])
        return finish(res, H_, W_)
