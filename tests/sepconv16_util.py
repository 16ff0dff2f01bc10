"""The Sepconv path against float64 references: per kernel of csrc/sepconv_elem.cu (vfi_sepconv_debug_elem), the
separable-convolution op of csrc/ops.cu, and the whole path (vfi_sepconv_forward + vfi_sepconv_debug_state) split at the
coefficients: the trunk against the 16-bit-faithful oracle (oracle/sepconv.py, ``operand=``), the tail against float64
arithmetic on the library's own coefficients.

Shared by tests/test_sepconv16_host.py (the library compiled for the host, tests/host_emu/sepconv_full_emu.cpp, every conv
on the CUDA-core checker) and tests/test_gpu_zsepconv16.py (the H100, wgmma convs).

Per kernel.  Inputs are seeded; the reference is the operation in float64 on the kernel's own inputs (16-bit values,
fp32 frames and weights widened exactly).  With n the number of fp32 roundings on the way to one output and S the sum of
the absolute values of its terms, every output satisfies
    16-bit outputs:  |y - y^| <= ulp_T(y^) + n 2^-24 S
    fp32 outputs:    |y - y^| <= n 2^-24 S
(``worst_ratio`` of tests/streamconv_util.py with K = n / 2); n is stated with each kernel.  coeff_nchw (a widening),
pad_input (a copy plus the ones channel) and the zero cells of prelu_s2d16 past an odd edge must be bit-exact; the stats
are double sums, held to n 2^-53 S with n the number of terms.  Every output is NaN-filled with a NaN image before and
after the images the kernel writes; add_crop16 updates its target in place, so the guards sit around that target.

The op.  ``sepconv_tile_kernel<51, PY>`` forms, per output row fy, rd = sum_fx hor[fx] in[.., fx] as a chain of K fp32
FMAs from 0 (K roundings, each at most 2^-24 of a partial sum bounded by S_fy = sum_fx |hor in|), multiplies by ver[fy]
(one rounding) and adds that into a Kahan-compensated sum over the K rows (at most 2 roundings' worth of the sum of the
absolute terms, plus O(K 2^-48)).  To first order the error is (K + 1 + 2) 2^-24 S with S = sum |ver hor in|; the bound
used is (K + 4) 2^-24 S, the 4th unit covering the second-order terms (K 2^-24 < 2^-18).  The generic kernel (any Kv, Kh)
rounds each product twice and Kahan-sums Kv Kh of them: (2 + 2) 2^-24 S + O(Kv Kh 2^-48) S, inside the same (Kh + 4).

Whole path.  (a) The trunk: the four coefficient planes and the four pyramid rows against the faithful oracle.  There is no
a-priori bound (fp32 accumulation order flips a 16-bit store by one ulp now and then and the flip propagates), so each
case's bound is MARGIN x the error the host emulation showed on that case (OBSERVED), over the whole plane and over a
2-pixel border band (tests/rife16_util.py ``compare``).  (b) The tail: the frame against float64
finish(op(pad(frames), library coefficients)), whose inputs are all exact, with the a-priori bound of ``tail_reference``; and
the frame against the faithful oracle under the calibrated bound.
"""
import ctypes as C
import math
import os
import subprocess
import sys
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import sepconv as OS
from rife16_util import compare
from streamconv_util import worst_ratio

DTYPES = {"float16": (0, torch.float16), "bfloat16": (1, torch.bfloat16)}
NAN = float("nan")
U = 2.0 ** -24
K51 = OS.KSIZE
ROWS = (1, 2, 3, 4)
ROW_C = (32, 64, 128, 256, 512)
HEADS = ("netVerone", "netVertwo", "netHorone", "netHortwo")
PLANES = ("ver1", "ver2", "hor1", "hor2")     # debug_state plane index k = heads' order

# kernel ids of vfi_sepconv_debug_elem (include/vfi_b200.h)
STATS, INPUT_CONV, PRELU_S2D, PRELU, PRELU_UP2, ADD_CROP, COEFF_NCHW, PAD_INPUT, FINISH = range(9)


# ----------------------------------------------------------------------------------------------------- per kernel
class Elem:
    """vfi_sepconv_debug_elem on one loaded context: ``L`` the ctypes library (product .so or host emulation), ``ctx``
    its context, tensors on ``dev`` (CPU for the host emulation)."""

    def __init__(self, L, ctx, dev, stream=None):
        vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
        L.vfi_sepconv_debug_elem.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, i32, f32, i32, vp]
        L.vfi_sepconv_debug_elem.restype = i32
        L.vfi_last_error.restype = C.c_char_p
        self.L, self.ctx, self.dev, self.stream = L, ctx, dev, stream

    def __call__(self, kernel, in0, out, C_=0, B=1, H=1, W=1, in1=None, f0=None, f1=None, n_frames=0, h=0, w=0,
                 slope=1.0, which=0):
        p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        a = None if f0 is None else (C.c_int32 * len(f0))(*f0)
        b = None if f1 is None else (C.c_int32 * len(f1))(*f1)
        rc = self.L.vfi_sepconv_debug_elem(self.ctx, kernel, p(in0), p(in1), None if a is None else C.cast(a, C.c_void_p),
                                           None if b is None else C.cast(b, C.c_void_p), n_frames, p(out), C_, B, H, W,
                                           h, w, slope, which, self.stream)
        if self.dev != "cpu":
            torch.cuda.synchronize()
        return rc, self.L.vfi_last_error().decode()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _ratio(name, got, ref, S, n, tdt):
    r, at = worst_ratio(got, ref, S, n / 2.0, tdt)
    assert r <= 1.0, f"{name}: worst error / bound {r:.3f} at {at}"
    return r


def _guarded(shape, dt, dev):
    """NaN-filled [B + 2, ...]: image 0 and B + 1 are the guards."""
    return torch.full((shape[0] + 2, *shape[1:]), NAN, dtype=dt, device=dev)


def _check_guards(name, out):
    assert bool(torch.isnan(out[0].float()).all() and torch.isnan(out[-1].float()).all()), f"{name}: store into a guard image"
    left = int(torch.isnan(out[1:-1].float()).sum())
    assert left == 0, f"{name}: {left} output cells never written (or NaN)"


def _t16(shape, tdt, g, scale=1.0):
    return ((torch.rand(*shape, generator=g) * 2 - 1) * scale).to(tdt)


def _frames(kind, n, H, W, C_, g):
    """[n, H, W, C_] float32 frames: "rand" in [0, 1]; "const" one value everywhere (std 0); "onepx" a constant clip
    but for one pixel of frame 1; "means" frames around very different means (0.02 and 0.9, then -3 and 5)."""
    if kind == "const":
        return torch.full((n, H, W, C_), 0.37)
    if kind == "onepx":
        fr = torch.full((n, H, W, C_), 0.25)
        fr[1, H // 2, W // 2, 1] = 0.75
        return fr
    fr = torch.rand(n, H, W, C_, generator=g)
    if kind == "means":
        for i, (m, s) in enumerate(((0.02, 0.01), (0.9, 0.05), (-3.0, 0.5), (5.0, 2.0))):
            if i < n:
                fr[i] = m + s * (fr[i] * 2 - 1)
    return fr


def _pairs(B, n_frames):
    """B pairs over n_frames frames: (i, i + 1), then a repeated and a reversed pair."""
    f0 = [i % (n_frames - 1) for i in range(B)]
    f1 = [x + 1 for x in f0]
    if B >= 3:
        f0[1], f1[1] = f0[0], f1[0]           # repeated
        f0[2], f1[2] = f1[0], f0[0]           # reversed
    return f0, f1


def _padded_pair(fr, a, b, H, W):
    """[2, 3, He, We] float64: frames a and b replicate-padded to even."""
    x = fr[[a, b]][..., :3].permute(0, 3, 1, 2).double()
    return F.pad(x, [0, W % 2, 0, H % 2], mode="replicate")


def ref_stats(fr, f0, f1, H, W):
    """(sum, sum of squares) per pair in float64 and the sums of absolute values."""
    s = [_padded_pair(fr, a, b, H, W) for a, b in zip(f0, f1)]
    st = torch.stack([torch.stack([x.sum(), (x * x).sum()]) for x in s])
    S = torch.stack([torch.stack([x.abs().sum(), (x * x).sum()]) for x in s])
    return st, S


def mean_inv(stats, cnt):
    """sep_input_conv's fp32 mean and 1 / (std + 1e-7) from double sums (unbiased std, sepconv_enhanced.py:630)."""
    mean_d = stats[:, 0] / cnt
    var_d = (stats[:, 1] - cnt * mean_d * mean_d) / (cnt - 1.0)
    mean = mean_d.float()
    std = var_d.clamp(min=0).sqrt().float()
    return mean, 1.0 / (std + torch.tensor(0.0000001, dtype=torch.float32))


def k_stats(E, tdt, dev, H, W, C_=3, B=1, kind="rand"):
    """n = the number of terms (6 He We): a double sum of exact fp32 values and their exact squares."""
    g = _g(11 + H + W)
    n_frames = max(B, 2) + 1
    fr = _frames(kind, n_frames, H, W, C_, g)
    f0, f1 = _pairs(B, n_frames)
    out = _guarded((B, 2), torch.float64, dev)
    rc, msg = E(STATS, fr.to(dev), out[1], C_=C_, B=B, H=H, W=W, f0=f0, f1=f1, n_frames=n_frames)
    assert rc == 0, msg
    name = f"stats {H}x{W} C{C_} B{B} {kind}"
    _check_guards(name, out)
    ref, S = ref_stats(fr, f0, f1, H, W)
    n = 6 * (H + H % 2) * (W + W % 2)
    r = float(((out[1:-1].cpu() - ref).abs() / (n * 2.0 ** -53 * S + 1e-300)).max())
    assert r <= 1.0, f"{name}: worst error / bound {r:.3f}"
    return r


def k_input_conv(E, tdt, dev, sd, H, W, C_=3, B=1, kind="rand"):
    """Reference: netInput in float64 on ((x - mean) * inv) from the same stats (mean and inv rounded to fp32 as the
    library defines them, std unbiased), PReLU of netEncode.0.netVer.1, space-to-depth.  n = 2 (the normalisation) + 28
    (27 FMAs onto the bias) + 1 (the PReLU product), S = sum |w| |x_n| + |b|."""
    g = _g(21 + H * W)
    n_frames = max(B, 2) + 1
    fr = _frames(kind, n_frames, H, W, C_, g)
    f0, f1 = _pairs(B, n_frames)
    stats, _ = ref_stats(fr, f0, f1, H, W)
    He, We = H + H % 2, W + W % 2
    out = _guarded((B, He // 2, We // 2, 128), tdt, dev)
    rc, msg = E(INPUT_CONV, fr.to(dev), out[1], C_=C_, B=B, H=H, W=W, in1=stats.to(dev).contiguous(), f0=f0, f1=f1,
                n_frames=n_frames)
    assert rc == 0, msg
    name = f"input_conv {H}x{W} C{C_} B{B} {kind}"
    _check_guards(name, out)
    mean, inv = mean_inv(stats, 6.0 * He * We)
    w, b = sd["netInput.weight"].double(), sd["netInput.bias"].double()
    slope = float(sd["netEncode.0.netVer.1.netMain.0.weight"])
    ys, Ss = [], []
    for i, (a, c) in enumerate(zip(f0, f1)):
        xn = (_padded_pair(fr, a, c, H, W) - mean[i].double()) * inv[i].double()
        y = F.conv2d(xn, w, b, padding=1)                           # [2, 16, He, We]
        S = F.conv2d(xn.abs(), w.abs(), padding=1) + b.abs().view(1, -1, 1, 1)
        ys.append(torch.where(y > 0, y, slope * y).reshape(32, He, We))
        Ss.append(S.reshape(32, He, We))

    def s2d(t):   # [B, 32, He, We] -> [B, He/2, We/2, (a, b, 32)]
        return t.view(B, 32, He // 2, 2, We // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, He // 2, We // 2, 128)
    ref, S = s2d(torch.stack(ys)), s2d(torch.stack(Ss))
    return _ratio(name, out[1:-1].cpu().double(), ref, S, 31, tdt)


def _prelu(x, s):
    return torch.where(x > 0, x, s * x)


def k_prelu_s2d16(E, tdt, dev, C_, H, W, B=2, slope=0.3):
    """n = 1 (the PReLU product); the cells past an odd edge must be +0 bit for bit."""
    g = _g(31 + C_ + H)
    x = _t16((B, H, W, C_), tdt, g, 4.0)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = _guarded((B, Ho, Wo, 4 * C_), tdt, dev)
    rc, msg = E(PRELU_S2D, x.to(dev), out[1], C_=C_, B=B, H=H, W=W, slope=slope)
    assert rc == 0, msg
    name = f"prelu_s2d16 C{C_} {H}x{W} B{B}"
    _check_guards(name, out)
    xp = F.pad(_prelu(x.double(), slope).permute(0, 3, 1, 2), [0, 2 * Wo - W, 0, 2 * Ho - H])
    ref = xp.view(B, C_, Ho, 2, Wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, Ho, Wo, 4 * C_)
    inside = F.pad(torch.ones(B, 1, H, W), [0, 2 * Wo - W, 0, 2 * Ho - H]).expand(B, C_, 2 * Ho, 2 * Wo)
    inside = inside.reshape(B, C_, Ho, 2, Wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, Ho, Wo, 4 * C_) > 0
    got = out[1:-1].cpu()
    assert bool((got[~inside].view(torch.int16) == 0).all()), f"{name}: a cell past the edge is not +0"
    return _ratio(name, got.double(), ref, ref.abs(), 1, tdt)


def k_prelu16(E, tdt, dev, C_, H, W, B=2, slope=-0.5):
    """n = 1 (the PReLU product)."""
    g = _g(41 + C_)
    x = _t16((B, H, W, C_), tdt, g, 4.0)
    out = _guarded((B, H, W, C_), tdt, dev)
    rc, msg = E(PRELU, x.to(dev), out[1], C_=C_, B=B, H=H, W=W, slope=slope)
    assert rc == 0, msg
    name = f"prelu16 C{C_} {H}x{W} slope {slope}"
    _check_guards(name, out)
    ref = _prelu(x.double(), slope)
    return _ratio(name, out[1:-1].cpu().double(), ref, ref.abs(), 1, tdt)


def k_prelu_up2_16(E, tdt, dev, C_, h, w, H, W, B=2, slope=0.2):
    """Reference: F.interpolate(scale_factor 2, bilinear) of the PReLU in float64, cropped.  The sample positions and
    weights (quarters) are exact in fp32; n = 1 (PReLU) + 4 (a product and three FMAs), S = the same interpolation of
    |prelu(x)|."""
    g = _g(51 + C_ + h * w)
    x = _t16((B, h, w, C_), tdt, g, 4.0)
    out = _guarded((B, H, W, C_), tdt, dev)
    rc, msg = E(PRELU_UP2, x.to(dev), out[1], C_=C_, B=B, H=H, W=W, h=h, w=w, slope=slope)
    assert rc == 0, msg
    name = f"prelu_up2_16 C{C_} {h}x{w}->{H}x{W} slope {slope}"
    _check_guards(name, out)
    a = _prelu(x.double(), slope).permute(0, 3, 1, 2)
    up = lambda t: F.interpolate(t, scale_factor=2.0, mode="bilinear", align_corners=False)[:, :, :H, :W]   # noqa: E731
    ref, S = up(a).permute(0, 2, 3, 1), up(a.abs()).permute(0, 2, 3, 1)
    return _ratio(name, out[1:-1].cpu().double(), ref, S, 5, tdt)


def k_add_crop16(E, tdt, dev, C_, h, w, H, W, B=2):
    """x[:, :H, :W] += v[:, :H, :W] in place on x; n = 1, S = |x| + |v|."""
    g = _g(61 + C_ + h)
    v = _t16((B, h, w, C_), tdt, g, 3.0)
    x0 = _t16((B, H, W, C_), tdt, g, 3.0)
    xg = _guarded((B, H, W, C_), tdt, "cpu")
    xg[1:-1] = x0
    xg = xg.to(dev)
    rc, msg = E(ADD_CROP, v.to(dev), xg[1], C_=C_, B=B, H=H, W=W, h=h, w=w)
    assert rc == 0, msg
    name = f"add_crop16 C{C_} {h}x{w}->{H}x{W}"
    _check_guards(name, xg)
    vc = v[:, :H, :W].double()
    ref = x0.double() + vc
    return _ratio(name, xg[1:-1].cpu().double(), ref, x0.double().abs() + vc.abs(), 1, tdt)


def k_coeff_nchw(E, tdt, dev, H, W, B=2):
    """A widening: bit-exact.  Channels 51..63 of the head's padded output hold NaN and must not reach the planes."""
    g = _g(71 + H * W)
    x = _t16((B, H, W, 64), tdt, g, 2.0)
    x[..., K51:] = NAN
    out = _guarded((B, K51, H, W), torch.float32, dev)
    rc, msg = E(COEFF_NCHW, x.to(dev), out[1], B=B, H=H, W=W)
    assert rc == 0, msg
    name = f"coeff_nchw {H}x{W} B{B}"
    _check_guards(name, out)
    assert torch.equal(out[1:-1].cpu(), x[..., :K51].float().permute(0, 3, 1, 2)), f"{name}: not an exact widening"
    return 0.0


def k_pad_input(E, tdt, dev, H, W, C_=3, B=1, which=0):
    """A copy with replicate padding (to even, then by 25) plus a channel of ones: bit-exact."""
    g = _g(81 + H + W)
    n_frames = max(B, 2) + 1
    fr = torch.rand(n_frames, H, W, C_, generator=g) * 3 - 1
    f0, f1 = _pairs(B, n_frames)
    He, We = H + H % 2, W + W % 2
    out = _guarded((B, 4, He + K51 - 1, We + K51 - 1), torch.float32, dev)
    rc, msg = E(PAD_INPUT, fr.to(dev), out[1], C_=C_, B=B, H=H, W=W, f0=f0, f1=f1, n_frames=n_frames, which=which)
    assert rc == 0, msg
    name = f"pad_input {H}x{W} C{C_} B{B} which {which}"
    _check_guards(name, out)
    src = f1 if which else f0
    ref = OS.pad_frames(fr[src][..., :3].permute(0, 3, 1, 2)).float()
    assert torch.equal(out[1:-1].cpu(), ref), f"{name}: not a bit-exact copy"
    return 0.0


FINISH_NORMS = (0.0, 0.01, -0.01, 0.0099, -0.0099, 0.0101, -0.0101, -0.5, -3.0, 1e-30, 2.0)   # as fp32 values


def k_finish(E, tdt, dev, H, W, B=2):
    """(o1 + o2)[:3] / (o1 + o2)[3] with |n| < 0.01 -> 1, cropped to H x W; n = 2 (the sum and the division), S =
    (|o1| + |o2|) / |n|.  The normalisers of the first pixels are set to FINISH_NORMS (o2's ones channel 0 there); the
    rule compares with 0.01 in fp32, so a normaliser of exactly 0.01f is kept."""
    g = _g(91 + H * W)
    He, We = H + H % 2, W + W % 2
    o1 = torch.rand(B, 4, He, We, generator=g) * 4 - 2
    o2 = torch.rand(B, 4, He, We, generator=g) * 4 - 2
    o1[:, 3] = o1[:, 3].abs() + 0.5
    cells = [(y, x) for y in range(H) for x in range(W)][:len(FINISH_NORMS)]
    for i, (y, x) in enumerate(cells):
        o1[:, 3, y, x] = FINISH_NORMS[i]
        o2[:, 3, y, x] = 0.0
    out = _guarded((B, H, W, 3), torch.float32, dev)
    rc, msg = E(FINISH, o1.to(dev), out[1], B=B, H=H, W=W, in1=o2.to(dev))
    assert rc == 0, msg
    name = f"finish {H}x{W} B{B}"
    _check_guards(name, out)
    s = o1.double() + o2.double()
    n = s[:, 3:4].clone()
    n[n.abs() < OS.NORM_EPS] = 1.0
    ref = (s[:, :3] / n)[:, :, :H, :W].permute(0, 2, 3, 1)
    S = ((o1.double().abs() + o2.double().abs())[:, :3] / n.abs())[:, :, :H, :W].permute(0, 2, 3, 1)
    return _ratio(name, out[1:-1].cpu().double(), ref, S, 2, None)


def kernel_cases():
    """(id, function name, kwargs) of every per-kernel case; each runs in both operand types."""
    cs = []
    for H, W, C_, B, kind in ((5, 7, 4, 1, "rand"), (1, 1, 3, 1, "rand"), (2, 3, 3, 3, "rand"), (67, 33, 3, 16, "rand"),
                              (9, 13, 4, 1, "const"), (9, 13, 3, 1, "onepx"), (11, 6, 3, 3, "means")):
        cs.append((f"stats_{H}x{W}_C{C_}_B{B}_{kind}", "k_stats", dict(H=H, W=W, C_=C_, B=B, kind=kind)))
    for H, W, C_, B, kind in ((1, 1, 3, 1, "rand"), (3, 1, 4, 1, "rand"), (2, 3, 3, 3, "rand"), (17, 22, 3, 3, "rand"),
                              (9, 13, 3, 16, "rand"), (9, 13, 4, 1, "const"), (9, 13, 3, 1, "onepx"),
                              (11, 6, 3, 3, "means")):
        cs.append((f"input_conv_{H}x{W}_C{C_}_B{B}_{kind}", "k_input_conv", dict(H=H, W=W, C_=C_, B=B, kind=kind)))
    for C_, H, W, B in ((32, 5, 7, 2), (64, 1, 1, 3), (128, 3, 2, 1), (256, 2, 1, 2), (32, 17, 30, 16), (512, 4, 5, 1)):
        cs.append((f"prelu_s2d16_C{C_}_{H}x{W}_B{B}", "k_prelu_s2d16", dict(C_=C_, H=H, W=W, B=B)))
    for C_, H, W, slope in ((64, 5, 7, -0.5), (512, 1, 1, 0.3), (256, 3, 4, 1.0), (32, 9, 1, 2.5)):
        cs.append((f"prelu16_C{C_}_{H}x{W}_s{slope}", "k_prelu16", dict(C_=C_, H=H, W=W, slope=slope)))
    # every target the schedule uses (2h x 2w: rows 4 -> 3 -> 2 -> 1 and the heads), odd rows, 1-pixel rows, and a
    # cropped target (2h - 1), which the kernel accepts
    for C_, h, w, H, W, slope in ((512, 1, 1, 2, 2, 0.2), (256, 3, 5, 6, 10, 0.2), (128, 2, 1, 4, 2, 0.3),
                                  (64, 9, 13, 18, 26, 1.0), (64, 1, 1, 2, 2, 1.0), (512, 5, 3, 9, 5, 0.25),
                                  (256, 4, 7, 7, 13, -0.4), (32, 1, 6, 1, 11, 0.2)):
        cs.append((f"prelu_up2_16_C{C_}_{h}x{w}_{H}x{W}", "k_prelu_up2_16", dict(C_=C_, h=h, w=w, H=H, W=W, slope=slope)))
    cs.append(("prelu_up2_16_C128_B16", "k_prelu_up2_16", dict(C_=128, h=3, w=2, H=6, W=4, B=16)))
    for C_, h, w, H, W in ((32, 6, 10, 5, 9), (64, 2, 2, 1, 1), (128, 4, 6, 4, 5), (256, 8, 2, 7, 2), (32, 3, 3, 3, 3)):
        cs.append((f"add_crop16_C{C_}_{h}x{w}_{H}x{W}", "k_add_crop16", dict(C_=C_, h=h, w=w, H=H, W=W)))
    for H, W, B in ((1, 1, 1), (5, 7, 2), (4, 8, 3), (33, 17, 1), (2, 200, 1)):
        cs.append((f"coeff_nchw_{H}x{W}_B{B}", "k_coeff_nchw", dict(H=H, W=W, B=B)))
    for H, W, C_, B, which in ((5, 7, 3, 1, 0), (5, 7, 4, 3, 1), (1, 1, 3, 1, 1), (6, 2, 4, 16, 0)):
        cs.append((f"pad_input_{H}x{W}_C{C_}_B{B}_w{which}", "k_pad_input", dict(H=H, W=W, C_=C_, B=B, which=which)))
    for H, W, B in ((3, 4, 1), (5, 7, 2), (4, 6, 3)):
        cs.append((f"finish_{H}x{W}_B{B}", "k_finish", dict(H=H, W=W, B=B)))
    return cs


NEEDS_SD = {"k_input_conv"}


def run_kernel_case(E, fn, kw, tdt, dev, sd):
    f = globals()[fn]
    return f(E, tdt, dev, sd, **kw) if fn in NEEDS_SD else f(E, tdt, dev, **kw)


def refusal_cases():
    """(id, call kwargs, text of the refusal)."""
    pair = dict(f0=[0], f1=[1], n_frames=2)
    return [
        ("prelu16_C12", dict(kernel=PRELU, C_=12, H=2, W=2), "C must be a multiple of 8"),
        ("prelu_s2d16_C20", dict(kernel=PRELU_S2D, C_=20, H=2, W=2), "C must be a multiple of 8"),
        ("prelu_up2_16_C4", dict(kernel=PRELU_UP2, C_=4, H=2, W=2, h=1, w=1), "C must be a multiple of 8"),
        ("add_crop16_C0", dict(kernel=ADD_CROP, C_=0, H=1, W=1, h=1, w=1), "C must be a multiple of 8"),
        ("stats_H0", dict(kernel=STATS, C_=3, H=0, W=4, **pair), "empty launch"),
        ("finish_W0", dict(kernel=FINISH, H=3, W=0, in1=True), "empty launch"),
        ("prelu_up2_16_h0", dict(kernel=PRELU_UP2, C_=8, H=2, W=2, h=0, w=1), "empty source"),
        ("prelu16_B0", dict(kernel=PRELU, C_=8, B=0, H=2, W=2), "B must be in [1,16]"),
        ("coeff_nchw_B17", dict(kernel=COEFF_NCHW, B=17, H=2, W=2), "B must be in [1,16]"),
        ("prelu_up2_16_target_3x2_from_1x1", dict(kernel=PRELU_UP2, C_=8, H=3, W=2, h=1, w=1),
         "up-sampling target larger than 2h x 2w"),
        ("prelu_up2_16_target_4x7_from_2x3", dict(kernel=PRELU_UP2, C_=8, H=4, W=7, h=2, w=3),
         "up-sampling target larger than 2h x 2w"),
        ("add_crop16_source_3x4_to_4x4", dict(kernel=ADD_CROP, C_=8, H=4, W=4, h=3, w=4),
         "crop source smaller than its target"),
        ("add_crop16_source_4x3_to_4x4", dict(kernel=ADD_CROP, C_=8, H=4, W=4, h=4, w=3),
         "crop source smaller than its target"),
        ("stats_frame_index", dict(kernel=STATS, C_=3, H=2, W=2, f0=[0], f1=[2], n_frames=2), "frame index"),
        ("input_conv_C2", dict(kernel=INPUT_CONV, C_=2, H=2, W=2, in1=True, **pair), "frames need >= 3 channels"),
        ("pad_input_which_2", dict(kernel=PAD_INPUT, C_=3, H=2, W=2, which=2, **pair), "pad_input pads frame 0 or 1"),
        ("no_such_kernel", dict(kernel=9, H=2, W=2), "no such element-wise kernel"),
    ]


def check_refusal(E, dev, kw, why):
    buf = torch.full((4096,), NAN, dtype=torch.float32, device=dev)
    buf[::3] = 1.5
    before = buf.clone()
    kw = dict(kw)
    kernel = kw.pop("kernel")
    if kw.pop("in1", None):
        kw["in1"] = buf
    rc, msg = E(kernel, buf, buf, **kw)
    assert rc != 0, (kernel, kw)
    assert why in msg, msg
    assert torch.equal(buf.isnan(), before.isnan()) and torch.equal(buf.nan_to_num(), before.nan_to_num()), \
        "refused, yet the buffer changed"


# ----------------------------------------------------------------------------------------------------- the op
def op_ref(x, ver, hor):
    """float64 (out, S = sum |ver hor in|) of the op on the inputs' device (oracle/sepconv.py ``op64``)."""
    return OS.op64(x, ver, hor), OS.op64(x, ver, hor, absolute=True)


def op_bound_n(kh):
    """The op's bound in units of 2^-24 S (module docstring)."""
    return kh + 4


# (id, N, C, H, W, Kv, Kh): K = 51 at the tile edges (32-wide columns, 8 PY-row bands), C > 4 (the pass loop), N up to 16
OP_CASES = [
    ("k51_N1_C4_1x1", 1, 4, 1, 1, 51, 51),
    ("k51_N1_C1_1x95", 1, 1, 1, 95, 51, 51),
    ("k51_N3_C4_49x1", 3, 4, 49, 1, 51, 51),
    ("k51_N1_C3_15x31", 1, 3, 15, 31, 51, 51),
    ("k51_N1_C4_16x32", 1, 4, 16, 32, 51, 51),
    ("k51_N1_C5_17x33", 1, 5, 17, 33, 51, 51),
    ("k51_N3_C8_16x33", 3, 8, 16, 33, 51, 51),
    ("k51_N1_C4_49x95", 1, 4, 49, 95, 51, 51),
    ("k51_N16_C1_17x31", 16, 1, 17, 31, 51, 51),
    ("k51_N16_C5_3x32", 16, 5, 3, 32, 51, 51),
    ("generic_N2_C3_9x13_kv7_kh5", 2, 3, 9, 13, 7, 5),
]


def op_inputs(case):
    _, N, C_, H, W, kv, kh = case
    g = _g(101 + N * 7 + C_ * 3 + H + W)
    x = torch.rand(N, C_, H + kv - 1, W + kh - 1, generator=g) * 3 - 1
    ver = (torch.rand(N, kv, H, W, generator=g) * 2 - 1) / kv * 4      # both signs
    hor = (torch.rand(N, kh, H, W, generator=g) * 2 - 1) / kh * 4
    return x, ver, hor


def check_op(run, case, dev):
    """``run(x, ver, hor, out_ptr)`` launches the op (host or device tensors on ``dev``); the output sits between two NaN
    guards of 1000 floats.  Returns the worst error / bound."""
    x, ver, hor = op_inputs(case)
    _, N, C_, H, W, kv, kh = case
    n = N * C_ * H * W
    buf = torch.full((n + 2000,), NAN, dtype=torch.float32, device=dev)
    xd, vd, hd = x.to(dev).contiguous(), ver.to(dev).contiguous(), hor.to(dev).contiguous()
    rc = run(xd, vd, hd, buf[1000:].data_ptr(), N, C_, H, W, kv, kh)
    assert rc == 0, (case[0], rc)
    b = buf.cpu()
    assert bool(torch.isnan(b[:1000]).all() and torch.isnan(b[1000 + n:]).all()), f"{case[0]}: store outside the output"
    got = b[1000:1000 + n].view(N, C_, H, W).double()
    ref, S = op_ref(x, ver, hor)
    return _ratio(f"op {case[0]}", got, ref, S, op_bound_n(kh), None)


def op_subprocess(py, mode, so=None):
    """Run every K = 51 op case in a fresh process with VFI_SEPCONV_PY = ``py`` (the launcher reads it once per process):
    ``mode`` "host" (the emulation ``so``) or "gpu" (the library).  Returns {case id: ratio}."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, VFI_SEPCONV_PY=str(py))
    code = f"import sys; sys.path.insert(0, {os.path.dirname(here)!r}); import sepconv16_util as U; U._op_child({mode!r}, {so!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=here, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = {}
    for line in r.stdout.splitlines():
        if line.startswith("OP "):
            _, cid, v = line.split()
            res[cid] = float(v)
    assert set(res) == {c[0] for c in OP_CASES if c[5] == 51}, r.stdout[-2000:]
    return res


def _op_child(mode, so):
    if mode == "host":
        L = C.CDLL(so)
        L.emu_sepconv_op.argtypes = [C.c_void_p] * 4 + [C.c_int] * 6
        run = lambda x, v, h, o, *a: L.emu_sepconv_op(x.data_ptr(), v.data_ptr(), h.data_ptr(), o, *a)   # noqa: E731
        dev = "cpu"
    else:
        run, dev = gpu_op_runner(), "cuda"
    for case in OP_CASES:
        if case[5] == 51:
            print(f"OP {case[0]} {check_op(run, case, dev):.4f}", flush=True)


def gpu_op_runner():
    """vfi_sepconv (the C ABI the ops surface calls) on the current stream."""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.ops import _context
    from cfi_b200._lib import lib
    L = lib()

    def run(x, v, h, o, N, C_, H, W, kv, kh):
        rc = L.vfi_sepconv(_context(x.device), x.data_ptr(), v.data_ptr(), h.data_ptr(), o, N, C_, H, W, kv, kh,
                           torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc
    return run


# ----------------------------------------------------------------------------------------------------- whole path
MARGIN = 4.0
TRUNK_GAIN = 4.0          # head gain at which the trunk's share of every coefficient plane is comparable to the bias
TRUNK_SHARE = 0.5         # ... asserted on TRUNK_CASES: max |coef - bias| >= TRUNK_SHARE x max |bias| on every plane
TRUNK_CASES = ("67x130_clip_g4", "45x54_noise_g4_rgba")   # (the 2x2 and 3-pixel-thin trunks are too small to show it)
MIN_NORM = 10.0           # ... and |normaliser| >= MIN_NORM (1000 x the 0.01 threshold) at every pixel
# (id, h, w, weight seed, head gain, frames: "golden:<name>", "clip", "noise" (outside [0, 1]); channels)
PATH_CASES = [
    ("21x30_golden", 21, 30, None, 1.0, "golden:sepconv_net_21x30", 3),
    ("45x54_golden", 45, 54, None, 1.0, "golden:sepconv_net_45x54", 3),
    ("48x64_golden", 48, 64, None, 1.0, "golden:sepconv_net_48x64", 3),
    ("2x2_noise_g4", 2, 2, 21, TRUNK_GAIN, "noise", 3),
    ("3x200_clip_g4", 3, 200, 22, TRUNK_GAIN, "clip", 3),
    ("200x3_noise_g4", 200, 3, 23, TRUNK_GAIN, "noise", 3),
    ("67x130_clip_g4", 67, 130, 24, TRUNK_GAIN, "clip", 3),
    ("45x54_noise_g4_rgba", 45, 54, 25, TRUNK_GAIN, "noise", 4),
]
# max |engine - oracle| of the host emulation
OBSERVED = {  # case: {operand: (coef, row 1, row 2, row 3, row 4, frame)}
    "21x30_golden": {"float16": (9.77e-04, 7.81e-03, 3.91e-03, 3.91e-03, 9.77e-04, 3.09e-05),
                    "bfloat16": (7.81e-03, 3.12e-02, 3.12e-02, 3.12e-02, 7.81e-03, 2.19e-04)},
    "45x54_golden": {"float16": (9.77e-04, 7.81e-03, 7.81e-03, 7.81e-03, 3.91e-03, 5.68e-05),
                    "bfloat16": (7.81e-03, 6.25e-02, 6.25e-02, 6.25e-02, 3.12e-02, 4.07e-04)},
    "48x64_golden": {"float16": (9.77e-04, 7.81e-03, 7.81e-03, 7.81e-03, 3.91e-03, 1.09e-04),
                    "bfloat16": (7.81e-03, 6.25e-02, 6.25e-02, 4.69e-02, 3.12e-02, 5.91e-04)},
    "2x2_noise_g4": {"float16": (1.22e-04, 2.44e-04, 1.22e-04, 6.10e-05, 3.05e-05, 2.49e-06),
                    "bfloat16": (0.00e+00, 0.00e+00, 0.00e+00, 0.00e+00, 0.00e+00, 9.19e-08)},
    "3x200_clip_g4": {"float16": (9.77e-04, 1.95e-03, 1.95e-03, 4.88e-04, 2.44e-04, 6.75e-05),
                     "bfloat16": (7.81e-03, 1.56e-02, 7.81e-03, 3.91e-03, 1.46e-03, 5.12e-04)},
    "200x3_noise_g4": {"float16": (9.77e-04, 3.91e-03, 1.46e-03, 4.88e-04, 1.83e-04, 6.24e-05),
                      "bfloat16": (7.81e-03, 1.56e-02, 7.81e-03, 3.91e-03, 9.77e-04, 4.24e-04)},
    "67x130_clip_g4": {"float16": (1.95e-03, 1.56e-02, 1.56e-02, 1.56e-02, 7.81e-03, 5.38e-04),
                      "bfloat16": (1.56e-02, 1.88e-01, 1.25e-01, 1.25e-01, 4.69e-02, 6.17e-03)},
    "45x54_noise_g4_rgba": {"float16": (9.77e-04, 7.81e-03, 7.81e-03, 7.81e-03, 3.91e-03, 1.96e-04),
                           "bfloat16": (7.81e-03, 6.25e-02, 6.25e-02, 6.25e-02, 3.12e-02, 1.44e-03)},
}


def path_inputs(case):
    """(state dict, frames [2, h, w, ch] float32)."""
    cid, h, w, seed, gain, frames, ch = case
    if frames.startswith("golden:"):
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        sys.path.insert(0, os.path.join(root, "tools"))
        from make_golden_sepconv import sepconv_cases, sepconv_inputs
        cfg = sepconv_cases()[frames[7:]]
        assert (cfg["h"], cfg["w"]) == (h, w)
        return OS.synthetic_state_dict(cfg["seed"]), sepconv_inputs(cfg).contiguous()
    sd = OS.synthetic_state_dict(seed, gain)
    g = _g(300 + h + w)
    if frames == "clip":
        t = torch.linspace(0, 1, w).view(1, 1, w, 1)
        y = torch.linspace(0, 1, h).view(1, h, 1, 1)
        base = 0.5 + 0.4 * torch.sin(7 * t + 3 * y + torch.tensor([0.0, 1.0, 2.0]).view(1, 1, 1, 3))
        fr = torch.cat([base, base.roll(2, dims=2)]) + 0.05 * torch.rand(2, h, w, 3, generator=g)
    else:
        fr = torch.rand(2, h, w, 3, generator=g) * 1.6 - 0.3
    if ch == 4:
        fr = torch.cat([fr, torch.rand(2, h, w, 1, generator=g)], -1)
    return sd, fr.float().contiguous()


def path_oracle(sd, fr, f0, f1, operand, device="cpu"):
    """The faithful oracle for pairs (f0[i], f1[i]): {"frame" [B,h,w,3], "coef" [4][B,He,We,51], "rows" [4][B,h,w,C],
    "stats" [B,2]}."""
    x = fr.to(device)[..., :3].permute(0, 3, 1, 2)
    d: Dict = {}
    out = OS.network_forward(sd, x[list(f0)], x[list(f1)], d, operand=operand)
    return dict(frame=out.permute(0, 2, 3, 1), coef=[d[k].permute(0, 2, 3, 1) for k in PLANES],
                rows=[d["levels"][r].permute(0, 2, 3, 1) for r in ROWS], stats=d["stats"])


def tail_reference(fr, f0, f1, coef):
    """float64 finish(op(pad(frames), coefficients)) on the library's own coefficients coef[k] [B,51,He,We] and its
    a-priori bound: with e = (K + 4) 2^-24 S the op's bound on each of the two op outputs (module docstring), a = o1 + o2
    and n = the ones channel's, the frame a / n is off by at most (e_a + u |a|) / |n| + |a / n| (e_n + u |n|) / |n| +
    u |a / n| (the fp32 sum and division), times 1.01 for the second-order terms.  Returns (frame [B,h,w,3], bound)."""
    H_, W_ = fr.shape[1], fr.shape[2]
    dev = coef[0].device
    x = fr.to(dev)[..., :3].permute(0, 3, 1, 2)
    p1, p2 = OS.pad_frames(x[list(f0)]), OS.pad_frames(x[list(f1)])
    o1, S1 = op_ref(p1, coef[0], coef[2])
    o2, S2 = op_ref(p2, coef[1], coef[3])
    a = o1 + o2
    e = op_bound_n(K51) * U * (S1 + S2)
    n = a[:, 3:4]
    assert bool((n.abs() >= 0.02).all()), "tail: a normaliser near the 0.01 threshold"
    q = a[:, :3] / n
    bound = ((e[:, :3] + U * a[:, :3].abs()) / n.abs() + q.abs() * (e[:, 3:4] + U * n.abs()) / n.abs() + U * q.abs()) * 1.01
    crop = lambda t: t[:, :, :H_, :W_].permute(0, 2, 3, 1)   # noqa: E731
    return crop(q), crop(bound)


def tol(case_id, operand):
    """MARGIN x the host emulation's errors on the case (coef, rows 1..4, frame); a case without calibration (1080p, 4K)
    gets MARGIN x the largest calibrated error of each."""
    if case_id not in OBSERVED:
        return tuple(MARGIN * max(v[operand][k] for v in OBSERVED.values()) for k in range(6))
    # an error the emulation did not show at all (a 1 x 1 row) is bounded by the smallest one its column showed elsewhere
    floor = [min(v[operand][k] for v in OBSERVED.values() if v[operand][k] > 0) for k in range(6)]
    return tuple(MARGIN * max(o, f) for o, f in zip(OBSERVED[case_id][operand], floor))


def path_compare(label, got, want, h, w, t):
    """got: {"frame", "coef" [4][B,51,He,We], "rows"}; want: path_oracle's.  Returns (lines, fails, observed tuple)."""
    lines, fails, obs = [], [], []
    He, We = h + h % 2, w + w % 2
    e = 0.0
    for k in range(4):
        g = got["coef"][k].permute(0, 2, 3, 1)
        ln, fl = compare(label, [g], [want["coef"][k]], h, w, {PLANES[k]: t[0]}, names=(PLANES[k],))
        lines += ln
        fails += fl
        e = max(e, float((g.to(want["coef"][k].device).double() - want["coef"][k]).abs().max()))
    obs.append(e)
    for i, r in enumerate(ROWS):
        hr, wr = He, We
        for _ in range(r):
            hr, wr = (hr + 1) // 2, (wr + 1) // 2
        g, ref = got["rows"][i], want["rows"][i]
        assert tuple(g.shape[1:]) == (hr, wr, ROW_C[r]) == tuple(ref.shape[1:]), (r, tuple(g.shape), tuple(ref.shape))
        ln, fl = compare(label, [g], [ref], hr, wr, {f"row{r}": t[1 + i]}, names=(f"row{r}",))
        lines += ln
        fails += fl
        obs.append(float((g.to(ref.device).double() - ref).abs().max()))
    ln, fl = compare(label, [got["frame"]], [want["frame"]], h, w, {"frame": t[5]}, names=("frame",))
    lines += ln
    fails += fl
    obs.append(float((got["frame"].to(want["frame"].device).double() - want["frame"]).abs().max()))
    return lines, fails, tuple(obs)


def check_stats(got, want, label):
    """The library's double sums against float64 sums of the same values: equal to ~1e-13 relative."""
    err = float(((got.to(want.device).double() - want).abs() / want.abs().clamp(min=1e-30)).max())
    assert err <= 1e-12, f"{label}: stats off by {err:.2e} relative"


def check_tail(label, fr, f0, f1, got):
    """(b): the library's frame against float64 arithmetic on its own coefficients; returns the worst error / bound."""
    q, bound = tail_reference(fr, f0, f1, [c.double() for c in got["coef"]])
    err = (got["frame"].to(q.device).double() - q).abs()
    r = float((err / bound).max())
    assert not math.isnan(r) and r <= 1.0, f"{label}: tail error / bound {r:.3f}"
    return r
