"""CPU restatement (fp32) of the reference's RIFE-4.6 hot path.  TEST INFRASTRUCTURE ONLY.

Each function cites the reference file:line it follows (paths relative to the reference
checkout, Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc).  The arithmetic of the
reference path lives in a third-party dependency that it calls directly - PyTorch ATen
(``requirements-no-cupy.txt:1`` "torch", unpinned; this image pins torch 2.11.0) - at the
call sites ``rife_arch.py:64-70`` (grid_sample), ``:238-266`` (interpolate), ``:96-107``
(conv2d), ``:215-218`` (conv_transpose2d + pixel_shuffle).  This restatement calls the
same ATen CPU operators functionally (no ``nn.Module`` from the reference, no reference
code), and ``oracle/primitives_np.py`` restates each of those operators' published
algorithm in numpy so the semantics the CUDA kernels implement are written down
independently of ATen.

Pinning: the reference ships no golden vectors or tests for this path (SURVEY.md section 4),
so the oracle is pinned against outputs of the reference itself, imported unmodified in
the build container by ``tools/make_golden.py``; the vectors live in ``tests/golden/``
and ``tests/test_oracle_golden.py`` checks this file against them bit-for-bit-close
(max abs 1e-6) on every CPU run.

16-bit-faithful mode.  ``ifnet*_forward(..., operand="float16" | "bfloat16")`` (and ``ifblock``) evaluate the same
graph in float64 and round to 16 bits exactly where the CUDA library stores or packs a 16-bit value, so that a
comparison with the library measures accumulation order only.  With ``operand=None`` (the default) nothing is
rounded and the fp32 graph above runs unchanged, bit for bit.  T is the operand type; where the library stores or
packs each tensor (csrc/elementwise.cu, csrc/rife46.cu, csrc/tapconv.cu):

| tensor | stored / packed by | type |
|---|---|---|
| frames, clamped to [0,1] and zero-padded (``imgs``) | ``prep_frames_kernel`` | fp32: read by encoders and ``final`` |
| the same frames (``imgs_h``) | ``prep_frames_kernel`` | fp16 for either T: read by the block-input warps |
| 4.7 encode Conv2d output (``e16``) | ``encode_conv_kernel``, fp32 weights | fp32 |
| 4.7 encoded features f0 / f1 | ``encode_deconv_kernel``, fp32 weights | fp16 for either T |
| 4.17 / 4.26 Head cnn0 output | ``head0_kernel``, fp32 weights | T |
| 4.17 / 4.26 Head cnn1, cnn2 outputs | tapconv, weights round_T(w) | T |
| 4.17 / 4.26 Head features f0 / f1 (cnn3) | tapconv, weights round_T(w) | T |
| block input [warps, t, mask, (features), flow/s] after the 1/s resampling | ``front*`` / ``front_up*`` kernels, fp32 arithmetic | T |
| conv0.0, conv0.1 outputs | tapconv, weights round_T(w), bias fp32 | T |
| ResConv outputs | tapconv, weights round_T(w*beta) (product in fp32), shift bias*beta (fp32), residual = the T input | T |
| lastconv flow (4) and mask (1) at the block's resolution | tapconv, weights round_T(w), bias fp32 | fp32 |
| 4.26 lastconv feature channels 5..12 (layer 11) at the block's resolution | tapconv, weights round_T(w), bias fp32 | T |
| accumulated flow / mask, final warps, sigmoid blend | ``flow_at``, ``fold_down``, ``final_kernel`` | fp32 |
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

# (in_planes, c) of the four IFBlocks of arch 4.6 -- rife_arch.py:404-408
BLOCK_SPECS: Tuple[Tuple[int, int], ...] = ((7, 192), (12, 128), (12, 96), (12, 64))
LRELU_SLOPE = 0.2  # rife_arch.py:106 / :26


# arch 4.7 (checkpoints rife47.pth / rife49.pth, rife/__init__.py:10-12): same IFBlocks with 8 (block 0) / 8 more input
# channels for the encoded features of both frames, plus the `encode` head -- rife_arch.py:409-417
BLOCK_SPECS_47: Tuple[Tuple[int, int], ...] = ((7 + 8, 192), (8 + 4 + 8, 128), (8 + 4 + 8, 96), (8 + 4 + 8, 64))
# arch 4.17 (rife417.pth): + Head_417 features, 8 channels per frame -- rife_arch.py:417-421, :356-375
BLOCK_SPECS_417: Tuple[Tuple[int, int], ...] = ((7 + 16, 192), (8 + 4 + 16, 128), (8 + 4 + 16, 96), (8 + 4 + 16, 64))
# arch 4.26 (rife426.pth): five blocks; inputs carry the 4-channel Head features of both frames (block 0) plus, from
# block 1 on, the previous block's 8 feature channels; lastconv has 13 = 4 flow + mask + 8 feature channels
# -- rife_arch.py:453-459, :226-233
BLOCK_SPECS_426: Tuple[Tuple[int, int], ...] = ((7 + 8, 192), (8 + 4 + 8 + 8, 128), (8 + 4 + 8 + 8, 96),
                                                (8 + 4 + 8 + 8, 64), (8 + 4 + 8 + 8, 32))
_BLOCKS = {"4.6": BLOCK_SPECS, "4.7": BLOCK_SPECS_47, "4.17": BLOCK_SPECS_417, "4.26": BLOCK_SPECS_426}
SCALE_LIST = {"4.6": (8, 4, 2, 1), "4.7": (8, 4, 2, 1), "4.17": (8, 4, 2, 1), "4.26": (16, 8, 4, 2, 1)}


def state_dict_spec(arch: str = "4.6") -> List[Tuple[str, Tuple[int, ...]]]:
    """Names and shapes of IFNet(arch).state_dict(), in the reference's order (arch "4.6", "4.7" or "4.17").

    Follows the module construction in rife_arch.py:177-218 (IFBlock.__init__),
    :20-28 (ResConv) and :404-408 (IFNet.__init__ for arch 4.6): 4 blocks x
    (conv0.0, conv0.1, 8 x ResConv{beta, conv}, lastconv) = 120 tensors, 5,306,256 values.
    """
    spec: List[Tuple[str, Tuple[int, ...]]] = []
    for b, (cin, c) in enumerate(_BLOCKS[arch]):
        p = f"block{b}."
        spec += [(p + "conv0.0.0.weight", (c // 2, cin, 3, 3)), (p + "conv0.0.0.bias", (c // 2,))]
        spec += [(p + "conv0.1.0.weight", (c, c // 2, 3, 3)), (p + "conv0.1.0.bias", (c,))]
        for j in range(8):
            q = p + f"convblock.{j}."
            spec += [(q + "beta", (1, c, 1, 1)), (q + "conv.weight", (c, c, 3, 3)), (q + "conv.bias", (c,))]
        nlast = 4 * 13 if arch == "4.26" else 4 * 6  # rife_arch.py:215-218 / :230-233
        spec += [(p + "lastconv.0.weight", (c, nlast, 4, 4)), (p + "lastconv.0.bias", (nlast,))]
    if arch == "4.7":  # encode = Sequential(Conv2d(3,16,3,2,1), ConvTranspose2d(16,4,4,2,1)) -- rife_arch.py:414-416
        spec += [("encode.0.weight", (16, 3, 3, 3)), ("encode.0.bias", (16,)),
                 ("encode.1.weight", (16, 4, 4, 4)), ("encode.1.bias", (4,))]
    if arch == "4.17":  # encode = Head_417: cnn0 3->32 s2, cnn1/cnn2 32->32, cnn3 ConvT 32->8 -- rife_arch.py:356-363
        spec += [("encode.cnn0.weight", (32, 3, 3, 3)), ("encode.cnn0.bias", (32,)),
                 ("encode.cnn1.weight", (32, 32, 3, 3)), ("encode.cnn1.bias", (32,)),
                 ("encode.cnn2.weight", (32, 32, 3, 3)), ("encode.cnn2.bias", (32,)),
                 ("encode.cnn3.weight", (32, 8, 4, 4)), ("encode.cnn3.bias", (8,))]
    if arch == "4.26":  # encode = Head: cnn0 3->16 s2, cnn1/cnn2 16->16, cnn3 ConvT 16->4 -- rife_arch.py:378-385
        spec += [("encode.cnn0.weight", (16, 3, 3, 3)), ("encode.cnn0.bias", (16,)),
                 ("encode.cnn1.weight", (16, 16, 3, 3)), ("encode.cnn1.bias", (16,)),
                 ("encode.cnn2.weight", (16, 16, 3, 3)), ("encode.cnn2.bias", (16,)),
                 ("encode.cnn3.weight", (16, 4, 4, 4)), ("encode.cnn3.bias", (4,))]
    return spec


def synthetic_state_dict(seed: int = 0, flow_gain: float = 1.0, beta_jitter: float = 0.25,
                         arch: str = "4.6") -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights (no checkpoint ships with the reference and there is no network).

    Same family as PyTorch's default init the reference would get from ``IFNet("4.6")``
    (uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)) for conv weight and bias; SURVEY.md section 8c
    found it well conditioned: per-block flow of a few pixels), but drawn from our own
    generator so it does not depend on the reference's module construction order, and with
    ``beta`` jittered around 1 so the per-channel ResConv scale (rife_arch.py:24,28) is
    actually exercised.  ``flow_gain`` scales every ``lastconv`` to sweep flow magnitude.
    """
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in state_dict_spec(arch):
        if name.endswith("beta"):
            sd[name] = 1.0 + beta_jitter * (2 * torch.rand(shape, generator=g) - 1)
            continue
        if name.endswith("weight"):
            if "lastconv" in name:  # ConvTranspose2d weight is [Cin, Cout, kh, kw]; torch's fan_in uses dim 1
                fan_in = shape[1] * shape[2] * shape[3]
            else:
                fan_in = shape[1] * shape[2] * shape[3]
            bound = 1.0 / math.sqrt(fan_in)
            last_fan_in = fan_in
        else:  # bias follows its weight in the spec order
            bound = 1.0 / math.sqrt(last_fan_in)
        t = (2 * torch.rand(shape, generator=g) - 1) * bound
        if "lastconv" in name:
            t = t * flow_gain
        sd[name] = t
    return sd


# --------------------------------------------------------------------------------------
# model pieces
# --------------------------------------------------------------------------------------
_OPERAND = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def _dt(operand: Optional[str]):
    if operand is not None and operand not in _OPERAND:
        raise ValueError(f"operand must be None, 'float16' or 'bfloat16', not {operand!r}")
    return None if operand is None else _OPERAND[operand]


def q16(x: torch.Tensor, dt) -> torch.Tensor:
    """``x`` rounded to the 16-bit type ``dt`` and widened to float64; ``x`` itself when ``dt`` is None."""
    return x if dt is None else x.to(dt).to(torch.float64)


def _wb(sd: Dict[str, torch.Tensor], prefix: str, dt, wdt="same"):
    """(weight, bias) of ``prefix``: as stored when ``dt`` is None, else the weight rounded to ``wdt`` (``dt`` unless
    given; None keeps fp32 - the CUDA-core encoders) and both widened to float64."""
    w, b = sd[prefix + "weight"], sd[prefix + "bias"]
    if dt is None:
        return w, b
    return q16(w, dt if wdt == "same" else wdt).double(), b.double()


def warp(img: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """Backward bilinear warp -- rife_arch.py:31-70.

    ``out[y,x] = bilinear(img, x + flow_x, y + flow_y)``: a [-1,1] linspace grid plus the
    flow divided by ((W-1)/2, (H-1)/2) of ``img`` (:45-52), sampled with
    ``grid_sample(bilinear, padding_mode="border", align_corners=True)`` (:64-70).
    """
    n, _, h, w = flow.shape
    hor = torch.linspace(-1.0, 1.0, w, dtype=flow.dtype, device=flow.device).view(1, 1, 1, w).expand(n, -1, h, -1)
    ver = torch.linspace(-1.0, 1.0, h, dtype=flow.dtype, device=flow.device).view(1, 1, h, 1).expand(n, -1, -1, w)
    grid = torch.cat([hor, ver], 1)
    fl = torch.cat(
        [flow[:, 0:1] / ((img.shape[3] - 1.0) / 2.0), flow[:, 1:2] / ((img.shape[2] - 1.0) / 2.0)], 1
    )
    g = (grid + fl).permute(0, 2, 3, 1)
    return F.grid_sample(img, g, mode="bilinear", padding_mode="border", align_corners=True)


def conv_lrelu(x, w, b, stride):
    """``conv()`` of arch >= 4.2: Conv2d(k3, stride, pad 1, bias) + LeakyReLU(0.2) -- rife_arch.py:96-107."""
    return F.leaky_relu(F.conv2d(x, w, b, stride=stride, padding=1), LRELU_SLOPE)


def resconv(x, w, b, beta):
    """ResConv.forward: ``lrelu(conv3x3(x) * beta + x)`` -- rife_arch.py:20-28."""
    return F.leaky_relu(F.conv2d(x, w, b, stride=1, padding=1) * beta + x, LRELU_SLOPE)


def resconv_packed(sd: Dict[str, torch.Tensor], q: str, dt):
    """The library's ResConv operands (csrc/rife46.cu conv2d with beta): (conv(x)+b)*beta == conv_{w*beta}(x) + b*beta, the
    products w*beta and b*beta formed in fp32, w*beta rounded to ``dt``; returned in float64."""
    beta = sd[q + "beta"].reshape(-1)
    return q16(sd[q + "conv.weight"] * beta.view(-1, 1, 1, 1), dt).double(), (sd[q + "conv.bias"] * beta).double()


def ifblock(sd: Dict[str, torch.Tensor], b: int, x: torch.Tensor, flow: Optional[torch.Tensor], scale: float,
            taps: Optional[dict] = None, operand: Optional[str] = None):
    """IFBlock.forward for arch 4.6 -- rife_arch.py:237-276.

    down-scale x (and flow, also divided by scale) bilinearly with align_corners=False
    (:238-249), conv0 = two stride-2 conv+lrelu (:250), 8 ResConv (:254), lastconv =
    ConvTranspose2d(c,24,4,2,1) + PixelShuffle(2) (:215-218,:256), up-scale by ``scale``,
    flow = ch0-3 * scale, mask = ch4 (:263-266,:275).  ``operand``: see the module docstring.
    """
    dt = _dt(operand)
    p = f"block{b}."
    x = F.interpolate(x, scale_factor=1.0 / scale, mode="bilinear", align_corners=False)
    if flow is not None:
        flow = F.interpolate(flow, scale_factor=1.0 / scale, mode="bilinear", align_corners=False) * 1.0 / scale
        x = torch.cat((x, flow), 1)
    x = q16(x, dt)
    if taps is not None:
        taps[f"b{b}.x"] = x
    feat = q16(conv_lrelu(x, *_wb(sd, p + "conv0.0.0.", dt), 2), dt)
    if taps is not None:
        taps[f"b{b}.c00"] = feat
    feat = q16(conv_lrelu(feat, *_wb(sd, p + "conv0.1.0.", dt), 2), dt)
    if taps is not None:
        taps[f"b{b}.c01"] = feat
    for j in range(8):
        q = p + f"convblock.{j}."
        if dt is None:
            feat = resconv(feat, sd[q + "conv.weight"], sd[q + "conv.bias"], sd[q + "beta"])
        else:
            feat = q16(F.leaky_relu(F.conv2d(feat, *resconv_packed(sd, q, dt), padding=1) + feat, LRELU_SLOPE), dt)
    if taps is not None:
        taps[f"b{b}.feat"] = feat
    tmp = F.conv_transpose2d(feat, *_wb(sd, p + "lastconv.0.", dt), stride=2, padding=1)
    tmp = F.pixel_shuffle(tmp, 2)
    if tmp.shape[1] == 13 and dt is not None:  # arch 4.26: the 8 feature channels are stored in T, flow / mask in fp32
        tmp = torch.cat((tmp[:, :5], q16(tmp[:, 5:], dt)), 1)
    if taps is not None:
        taps[f"b{b}.tmp"] = tmp
    tmp = F.interpolate(tmp, scale_factor=scale, mode="bilinear", align_corners=False)
    if tmp.shape[1] == 13:  # arch 4.26: flow, mask, 8 feature channels for the next block -- rife_arch.py:267-274
        return tmp[:, :4] * scale, tmp[:, 4:5], tmp[:, 5:]
    return tmp[:, :4] * scale, tmp[:, 4:5]


def _prep(img0, img1, timestep, operand):
    """clamp + zero-pad to x64 (rife_arch.py:476-485) and the timestep plane (:491-494).  Returns (img0, img1, t, the
    frames the block inputs sample, dt): with an operand the fp32 frames widened to float64 and their fp16 copies."""
    dt = _dt(operand)
    if dt is not None:
        img0, img1 = img0.double(), img1.double()
    img0 = torch.clamp(img0, 0, 1)
    img1 = torch.clamp(img1, 0, 1)
    n, c, h, w = img0.shape
    ph = ((h - 1) // 64 + 1) * 64
    pw = ((w - 1) // 64 + 1) * 64
    img0 = F.pad(img0, (0, pw - w, 0, ph - h))
    img1 = F.pad(img1, (0, pw - w, 0, ph - h))
    t = timestep.reshape(n, 1, 1, 1).to(img0.device).to(img0.dtype).repeat(1, 1, ph, pw)
    hdt = None if dt is None else torch.float16
    return img0, img1, t, (q16(img0, hdt), q16(img1, hdt)), dt


def _head(sd: Dict[str, torch.Tensor], x: torch.Tensor, dt) -> torch.Tensor:
    """Head (4.26) / Head_417 (4.17) with feat=False -- rife_arch.py:356-395: cnn0 3->c stride 2, cnn1, cnn2 c->c, each +
    LeakyReLU(0.2), cnn3 ConvTranspose c->4|8.  With an operand: cnn0 on the CUDA cores with fp32 weights, cnn1..cnn3 with
    weights rounded to T, every output stored in T."""
    y = q16(F.leaky_relu(F.conv2d(x, *_wb(sd, "encode.cnn0.", dt, None), stride=2, padding=1), 0.2), dt)
    y = q16(F.leaky_relu(F.conv2d(y, *_wb(sd, "encode.cnn1.", dt), padding=1), 0.2), dt)
    y = q16(F.leaky_relu(F.conv2d(y, *_wb(sd, "encode.cnn2.", dt), padding=1), 0.2), dt)
    return q16(F.conv_transpose2d(y, *_wb(sd, "encode.cnn3.", dt), stride=2, padding=1), dt)


def _blend(img0, img1, flow, mask, w0, w1, dt):
    """sigmoid blend of the last warps -- rife_arch.py:703-717.  With an operand the block inputs sampled the fp16 frames
    (w0, w1) but the final warps read the fp32 ones."""
    if dt is not None:
        w0, w1 = warp(img0, flow[:, :2]), warp(img1, flow[:, 2:4])
    m = torch.sigmoid(mask)
    return w0 * m + w1 * (1 - m)


def ifnet46_forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, timestep: torch.Tensor,
                    scale_list: Sequence[float] = (8, 4, 2, 1), taps: Optional[dict] = None,
                    operand: Optional[str] = None) -> torch.Tensor:
    """IFNet.forward restricted to arch 4.6, ensemble=False -- rife_arch.py:465-732.

    clamp + zero-pad right/bottom to x64 (:476-485), timestep plane (:491-494), block0 on
    cat(img0,img1,t) (:527-532), blocks 1-3 on cat(warped0,warped1,t,mask)+flow with
    ``flow += f0; mask += m0`` (:589-596,:694-696), warp after every block (:703-704),
    sigmoid blend of the last pair (:713-717), crop (:732).  ``training``/``fastmode`` do
    not touch the 4.6 result and the node's ``ensemble`` never reaches the model
    (SURVEY.md F7), so they are not parameters here.
    NCHW fp32 in, NCHW fp32 out; ``timestep`` is [B,1,1,1].
    """
    h, w = img0.shape[2], img0.shape[3]
    img0, img1, t, (h0, h1), dt = _prep(img0, img1, timestep, operand)
    w0, w1, flow, mask = h0, h1, None, None
    for i in range(4):
        if flow is None:
            flow, mask = ifblock(sd, i, torch.cat((h0, h1, t), 1), None, scale_list[i], taps, operand)
        else:
            f0, m0 = ifblock(sd, i, torch.cat((w0, w1, t, mask), 1), flow, scale_list[i], taps, operand)
            flow = flow + f0
            mask = mask + m0
        if taps is not None:
            taps[f"flow{i}"] = flow
            taps[f"mask{i}"] = mask
        w0 = warp(h0, flow[:, :2])
        w1 = warp(h1, flow[:, 2:4])
    return _blend(img0, img1, flow, mask, w0, w1, dt)[:, :, :h, :w]


def ifnet47_forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, timestep: torch.Tensor,
                    scale_list: Sequence[float] = (8, 4, 2, 1), taps: Optional[dict] = None,
                    operand: Optional[str] = None) -> torch.Tensor:
    """IFNet.forward restricted to arch 4.7 (rife47.pth / rife49.pth) and 4.17 (rife417.pth, same forward with the
    Head_417 encoder and 8 feature channels per frame), ensemble=False -- rife_arch.py:465-732.

    Differences to 4.6: f0/f1 = encode(img) (Conv2d 3->16 s2, ConvTranspose2d 16->4, no activation; :501-503) are
    concatenated to block 0's input (:543-548) and, warped with the current flow, to the later blocks' inputs
    (:629-645); `flow = flow + fd` but `mask = m0` is REPLACED, not accumulated (:646, :698-699); the final blend
    uses sigmoid of that last mask (:721-723)."""
    h, w = img0.shape[2], img0.shape[3]
    img0, img1, t, (h0, h1), dt = _prep(img0, img1, timestep, operand)

    def encode(x):
        if "encode.cnn0.weight" in sd:  # arch 4.17, Head_417.forward -- rife_arch.py:365-375 (feat=False)
            return _head(sd, x, dt)
        # arch 4.7: both layers on the CUDA cores with fp32 weights, the features stored as fp16 whatever T is
        y = F.conv2d(x, *_wb(sd, "encode.0.", dt, None), stride=2, padding=1)
        y = F.conv_transpose2d(y, *_wb(sd, "encode.1.", dt, None), stride=2, padding=1)
        return q16(y, None if dt is None else torch.float16)

    f0, f1 = encode(img0), encode(img1)
    if taps is not None:
        taps["f0"], taps["f1"] = f0, f1
    w0, w1, flow, mask = h0, h1, None, None
    for i in range(4):
        if flow is None:
            flow, mask = ifblock(sd, i, torch.cat((h0, h1, f0, f1, t), 1), None, scale_list[i], taps, operand)
        else:
            fd, m0 = ifblock(sd, i, torch.cat((w0, w1, warp(f0, flow[:, :2]), warp(f1, flow[:, 2:4]), t, mask), 1),
                             flow, scale_list[i], taps, operand)
            flow = flow + fd
            mask = m0
        if taps is not None:
            taps[f"flow{i}"] = flow
            taps[f"mask{i}"] = mask
        w0 = warp(h0, flow[:, :2])
        w1 = warp(h1, flow[:, 2:4])
    return _blend(img0, img1, flow, mask, w0, w1, dt)[:, :, :h, :w]


def ifnet426_forward(sd: Dict[str, torch.Tensor], img0: torch.Tensor, img1: torch.Tensor, timestep: torch.Tensor,
                     scale_list: Sequence[float] = (16, 8, 4, 2, 1), taps: Optional[dict] = None,
                     operand: Optional[str] = None) -> torch.Tensor:
    """IFNet.forward restricted to arch 4.26 (rife426.pth; the node forces ensemble=False, rife/__init__.py:123-125)
    -- rife_arch.py:465-732.

    Five blocks at scales 16..1 (:508-511; still padded to x64 only, :480-482).  f0/f1 = Head(img) (cnn0 3->16 stride 2,
    cnn1, cnn2 16->16, each + LeakyReLU(0.2), cnn3 ConvTranspose 16->4; :378-395).  Block 0 sees cat(img0, img1, f0, f1, t)
    (:521-526); block i > 0 sees cat(warped0, warped1, warp(f0), warp(f1), t, mask, feat) + flow, where `feat` is the
    previous block's 8 extra lastconv channels up-scaled to full resolution (:563-587); `flow += fd`, `mask = m0`
    REPLACED (:586-587); blend with sigmoid of the last mask (:707-711)."""
    h, w = img0.shape[2], img0.shape[3]
    img0, img1, t, (h0, h1), dt = _prep(img0, img1, timestep, operand)

    f0, f1 = _head(sd, img0, dt), _head(sd, img1, dt)  # Head.forward, feat=False -- rife_arch.py:387-395
    if taps is not None:
        taps["f0"], taps["f1"] = f0, f1
    w0, w1, flow, mask, feat = h0, h1, None, None, None
    for i in range(5):
        if flow is None:
            flow, mask, feat = ifblock(sd, i, torch.cat((h0, h1, f0, f1, t), 1), None, scale_list[i], taps, operand)
        else:
            x = torch.cat((w0, w1, warp(f0, flow[:, :2]), warp(f1, flow[:, 2:4]), t, mask, feat), 1)
            fd, m0, feat = ifblock(sd, i, x, flow, scale_list[i], taps, operand)
            flow = flow + fd
            mask = m0
        if taps is not None:
            taps[f"flow{i}"] = flow
            taps[f"mask{i}"] = mask
        w0 = warp(h0, flow[:, :2])
        w1 = warp(h1, flow[:, 2:4])
    return _blend(img0, img1, flow, mask, w0, w1, dt)[:, :, :h, :w]


def ifnet_forward(arch: str, sd, img0, img1, timestep, scale_list=None, taps=None, operand=None):
    if scale_list is None:
        scale_list = SCALE_LIST[arch]
    fn = ifnet46_forward if arch == "4.6" else ifnet426_forward if arch == "4.26" else ifnet47_forward
    return fn(sd, img0, img1, timestep, scale_list, taps, operand)


# --------------------------------------------------------------------------------------
# node-level loop
# --------------------------------------------------------------------------------------
def is_frame_skipped(frame_indices: Sequence[int], is_skip_list: bool, idx: int) -> bool:
    """InterpolationStateList.is_frame_skipped -- vfi_utils.py:55-57."""
    inside = idx in frame_indices
    return (is_skip_list and inside) or (not is_skip_list and not inside)


def build_tasks(n_frames: int, multiplier, states: Optional[Tuple[Sequence[int], bool]] = None):
    """(pair_idx, timestep) task list and per-pair multipliers -- rife/__init__.py:149-174."""
    n_pairs = n_frames - 1
    if isinstance(multiplier, int):
        mults = [int(multiplier)] * n_pairs
    else:
        mults = list(map(int, multiplier))
        mults += [2] * (n_pairs - len(mults))
    tasks = []
    for p in range(n_pairs):
        if states is not None and is_frame_skipped(states[0], states[1], p):
            continue
        m = mults[p]
        for step in range(1, m):
            tasks.append((p, step / m))
    return tasks, mults


def rife_vfi(sd: Dict[str, torch.Tensor], frames: torch.Tensor, multiplier=2, scale_factor: float = 1.0,
             states: Optional[Tuple[Sequence[int], bool]] = None, batch_size: int = 1,
             arch: str = "4.6") -> torch.Tensor:
    """RIFE_VFI.vfi for ckpt arch 4.6, dtype float32 -- rife/__init__.py:146-239.

    frames: [N,H,W,C>=3] fp32 NHWC in [0,1]; returns [(sum over pairs of mids)+N, H, W, 3] fp32
    NHWC: each original frame followed by its interpolated frames (:225-238); mids are
    ``model(...).clamp(0,1)`` (:200-207); first 3 channels only (vfi_utils.py:139-143).
    """
    fr = frames[..., :3].permute(0, 3, 1, 2)
    tasks, _ = build_tasks(len(fr), multiplier, states)
    scale_list = [s / scale_factor for s in SCALE_LIST[arch]]  # rife/__init__.py:156-160
    results: Dict[int, List[torch.Tensor]] = {i: [] for i in range(len(fr) - 1)}
    with torch.inference_mode():
        pos = 0
        while pos < len(tasks):
            bt = tasks[pos:pos + batch_size]
            f0 = torch.cat([fr[p:p + 1] for p, _ in bt]).float()
            f1 = torch.cat([fr[p + 1:p + 2] for p, _ in bt]).float()
            ts = torch.tensor([t for _, t in bt], dtype=torch.float32).view(-1, 1, 1, 1)
            mid = ifnet_forward(arch, sd, f0, f1, ts, scale_list).clamp(0, 1)
            for k, (p, _) in enumerate(bt):
                results[p].append(mid[k:k + 1])
            pos += len(bt)
    out = []
    for p in range(len(fr) - 1):
        out.append(fr[p:p + 1].float())
        out += results[p]
    out.append(fr[-1:].float())
    return torch.cat(out).permute(0, 2, 3, 1)[..., :3].contiguous()


# --------------------------------------------------------------------------------------
# metrics / synthetic clips (SURVEY.md section 8d config 2)
# --------------------------------------------------------------------------------------
def psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    mse = torch.mean((a.double() - b.double()) ** 2).item()
    return float("inf") if mse == 0 else 10.0 * math.log10(1.0 / mse)


def synthetic_clip(n: int, h: int, w: int, seed: int = 1234, noise: float = 0.02) -> torch.Tensor:
    """Smooth moving content: a low-frequency random image translated by (2,1) px per frame
    plus a little noise, clamped -- NHWC fp32 [n,h,w,3] (SURVEY.md section 8d, config 2)."""
    g = torch.Generator().manual_seed(seed)
    lh, lw = max(h // 16, 4), max(w // 16, 4)
    low = torch.rand(1, 3, lh, lw, generator=g)
    big = F.interpolate(low, size=(h + 2 * n + 8, w + 2 * n + 8), mode="bicubic", align_corners=False).clamp(0, 1)
    out = torch.empty(n, h, w, 3)
    for i in range(n):
        crop = big[0, :, i:i + h, 2 * i:2 * i + w]
        fr = crop + noise * (2 * torch.rand(3, h, w, generator=g) - 1)
        out[i] = fr.clamp(0, 1).permute(1, 2, 0)
    return out
