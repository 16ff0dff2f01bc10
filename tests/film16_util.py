"""The FILM path against float64 references: per kernel of csrc/film_elem.cu (vfi_film_debug_elem) and as a whole
(vfi_film_forward + vfi_film_debug_state) against the 16-bit-faithful oracle (oracle/film.py, ``operand=``).

Shared by tests/test_film16_host.py (the library compiled for the host, tests/host_emu/film_full_emu.cpp, every conv on
the CUDA-core checker) and tests/test_gpu_zfilm16.py (the H100, wgmma convs).

Per kernel.  Inputs are seeded; the reference is the operation in float64 on the kernel's own inputs (16-bit values and
fp32 weights widened exactly).  With n the number of fp32 roundings on the way to one output and S the sum of the absolute
values of the terms, every output satisfies
    16-bit outputs:  |y - y^| <= ulp_T(y^) + n 2^-24 S
    fp32 outputs:    |y - y^| <= n 2^-24 S
(``worst_ratio`` of tests/streamconv_util.py with K = n / 2); gather_rgb and nearest16 copy and must be bit-exact.  A
sample position p (bilinear taps, the source index of a resize) is itself rounded in fp32: it moves the output by at most
2^-24 |p| max|v| per rounding (bilinear interpolation is continuous in p, also across a change of the integer tap), so
|p| max|v| counts as a term of S.  Every output tensor is filled with NaN, with a NaN image before and after the images the
kernel writes and NaN in every channel outside the slice it writes; those must still hold NaN afterwards.

Whole path.  There is no a-priori bound: fp32 accumulation order flips a 16-bit store by one ulp now and then and the flip
propagates through the later layers and the warps.  Each case's bound is MARGIN x the error the host emulation showed on
that case (OBSERVED), over the whole plane and over a 2-pixel border band (tests/rife16_util.py ``compare``).
"""
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import film as OF
from rife16_util import compare
from streamconv_util import worst_ratio

DTYPES = {"float16": (0, torch.float16), "bfloat16": (1, torch.bfloat16)}
LEVELS = 7
NAN = float("nan")

# kernel ids of vfi_film_debug_elem (include/vfi_b200.h)
GATHER, POOL_RGB, CONV_RGB, POOL16, FLOW_UP, WARP16, MISC64, NEAREST16, FLOW_HEAD, OUT_RGB = range(10)
HEAD_C = (16, 32, 64, 128)   # nf / 2 of the flow predictors 0..3


# ----------------------------------------------------------------------------------------------------- per kernel
class Elem:
    """vfi_film_debug_elem on one loaded context: ``L`` the ctypes library (product .so or host emulation), ``ctx`` its
    context, tensors on ``dev`` (CPU for the host emulation)."""

    def __init__(self, L, ctx, dev, stream=None):
        import ctypes as C
        vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
        L.vfi_film_debug_elem.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, f32,
                                          i32, i32, vp]
        L.vfi_film_debug_elem.restype = i32
        L.vfi_last_error.restype = C.c_char_p
        self.L, self.ctx, self.dev, self.stream, self.C = L, ctx, dev, stream, C

    def __call__(self, kernel, in0, out, C_=0, B=1, H=1, W=1, in_pitch=0, in1=None, in2=None, in3=None, frame_idx=None,
                 out_pitch=0, h=0, w=0, fscale=1.0, clamp01=0, predictor=0, ptr0=None, optr=None):
        p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        idx = None if frame_idx is None else (self.C.c_int32 * len(frame_idx))(*frame_idx)
        rc = self.L.vfi_film_debug_elem(self.ctx, kernel, ptr0 if ptr0 is not None else p(in0), in_pitch, p(in1), p(in2),
                                        p(in3), None if idx is None else self.C.cast(idx, self.C.c_void_p),
                                        optr if optr is not None else p(out), out_pitch, C_, B, H, W, h, w, fscale,
                                        clamp01, predictor, self.stream)
        if self.dev != "cpu":
            torch.cuda.synchronize()
        return rc, self.L.vfi_last_error().decode()


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _ratio(name, got, ref, S, n, tdt):
    r, at = worst_ratio(got, ref, S, n / 2.0, tdt)
    assert r <= 1.0, f"{name}: worst error / bound {r:.3f} at (b,y,x,c) {at}"
    return r


def _guarded(B, H, W, pitch, dt, dev):
    """NaN-filled [B + 2, H, W, pitch]: image 0 and B + 1 are the guards."""
    return torch.full((B + 2, H, W, pitch), NAN, dtype=dt, device=dev)


def _check_guards(name, out, off, n):
    """Images 0 and -1 and the channels outside [off, off + n) still NaN; no NaN inside."""
    assert bool(torch.isnan(out[0].float()).all() and torch.isnan(out[-1].float()).all()), f"{name}: store into a guard image"
    assert bool(torch.isnan(out[1:-1, ..., :off].float()).all()), f"{name}: store before the slice"
    assert bool(torch.isnan(out[1:-1, ..., off + n:].float()).all()), f"{name}: store after the slice"
    left = int(torch.isnan(out[1:-1, ..., off:off + n].float()).sum())
    assert left == 0, f"{name}: {left} output cells never written (or NaN)"


def _src16(B, H, W, C, off, pitch, tdt, g, scale=1.0):
    """[B, H, W, pitch] 16-bit: NaN outside channels [off, off + C), seeded values (rounded to T) inside."""
    t = torch.full((B, H, W, pitch), NAN, dtype=tdt)
    t[..., off:off + C] = ((torch.rand(B, H, W, C, generator=g) * 2 - 1) * scale).to(tdt)
    return t


def _bilinear(src, fx, fy):
    """float64 [B, H, W, C] sampled at (x + fx, y + fy), coordinates clamped to the image (grid_sample 'border'), and the
    sum of |tap value x weight|."""
    B, H, W, C = src.shape
    ys = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    sx = (xs + fx).clamp(0, W - 1)
    sy = (ys + fy).clamp(0, H - 1)
    x0, y0 = sx.floor(), sy.floor()
    wx, wy = sx - x0, sy - y0
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
    bi = torch.arange(B).view(B, 1, 1)
    out = torch.zeros(B, H, W, C, dtype=torch.float64)
    S = torch.zeros_like(out)
    for yy, xx, wt in ((y0, x0, (1 - wx) * (1 - wy)), (y0, x1, wx * (1 - wy)), (y1, x0, (1 - wx) * wy), (y1, x1, wx * wy)):
        v = src[bi, yy, xx] * wt[..., None]
        out += v
        S += v.abs()
    return out, S


def _pos_term(src, fx, fy):
    """|sample position| x max |value| of each (image, channel): the position rounding's share of S."""
    B, H, W, C = src.shape
    ys = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    p = (xs + fx.abs() + ys + fy.abs() + 2)[..., None]
    return p * src.abs().amax(dim=(1, 2), keepdim=True)


def k_gather(E, tdt, dev, C=3, n_frames=17, pairs=16, H=5, W=7):
    g = _g(1)
    fr = (torch.rand(n_frames, H, W, C, generator=g) * 3 - 1).to(dev)
    idx = list(range(pairs)) + list(range(1, pairs + 1))
    B = len(idx)
    out = _guarded(B, H, W, 3, torch.float32, dev)
    rc, msg = E(GATHER, fr, out[1], C_=C, B=B, H=H, W=W, frame_idx=idx)
    assert rc == 0, msg
    _check_guards("gather_rgb", out, 0, 3)
    assert torch.equal(out[1:-1].cpu(), fr[idx][..., :3].cpu()), "gather_rgb: not a bit-exact copy"
    return 0.0


def k_pool_rgb(E, tdt, dev, H=67, W=33, B=3):
    g = _g(2)
    x = (torch.rand(B, H, W, 3, generator=g) * 3 - 1)
    out = _guarded(B, H // 2, W // 2, 3, torch.float32, dev)
    rc, msg = E(POOL_RGB, x.to(dev), out[1], B=B, H=H, W=W)
    assert rc == 0, msg
    _check_guards("pool_rgb", out, 0, 3)
    xd = x.double()[:, :H // 2 * 2, :W // 2 * 2]
    ref = xd.view(B, H // 2, 2, W // 2, 2, 3).mean(dim=(2, 4))
    S = xd.abs().view(B, H // 2, 2, W // 2, 2, 3).mean(dim=(2, 4))
    return _ratio(f"pool_rgb {H}x{W}", out[1:-1].cpu().double(), ref, S, 4, None)


def k_conv_rgb(E, tdt, dev, sd, H, W, B=2, off=8, pitch=80):
    g = _g(3)
    x = torch.rand(B, H, W, 3, generator=g) * 1.4 - 0.2
    out = _guarded(B, H, W, pitch, tdt, dev)
    rc, msg = E(CONV_RGB, x.to(dev), None, B=B, H=H, W=W, out_pitch=pitch, optr=out[1].data_ptr() + 2 * off)
    assert rc == 0, msg
    _check_guards(f"conv_rgb {H}x{W}", out, off, 64)
    w = sd["extract.extract_sublevels.convs.0.0.0.weight"].double()
    b = sd["extract.extract_sublevels.convs.0.0.0.bias"].double()
    xc = x.double().permute(0, 3, 1, 2)
    ref = F.leaky_relu(F.conv2d(xc, w, b, padding=1), 0.2).permute(0, 2, 3, 1)
    S = (F.conv2d(xc.abs(), w.abs(), padding=1) + b.abs().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    return _ratio(f"conv_rgb {H}x{W}", out[1:-1, ..., off:off + 64].cpu().double(), ref, S, 28, tdt)


def k_pool16(E, tdt, dev, C, H, W, B=2, in_off=64, in_pitch=None, out_off=32, out_pitch=None):
    g = _g(4)
    in_pitch = in_pitch or in_off + C + 16
    out_pitch = out_pitch or out_off + C + 32
    src = _src16(B, H, W, C, in_off, in_pitch, tdt, g, 4.0)
    Ho, Wo = H // 2, W // 2
    out = _guarded(B, Ho, Wo, out_pitch, tdt, dev)
    sd_ = src.to(dev)
    rc, msg = E(POOL16, None, None, C_=C, B=B, H=H, W=W, in_pitch=in_pitch, out_pitch=out_pitch,
                ptr0=sd_.data_ptr() + 2 * in_off, optr=out[1].data_ptr() + 2 * out_off)
    assert rc == 0, msg
    _check_guards(f"pool16 C{C} {H}x{W}", out, out_off, C)
    xd = src[:, :Ho * 2, :Wo * 2, in_off:in_off + C].double()
    ref = xd.reshape(B, Ho, 2, Wo, 2, C).mean(dim=(2, 4))
    S = xd.abs().reshape(B, Ho, 2, Wo, 2, C).mean(dim=(2, 4))
    return _ratio(f"pool16 C{C} {H}x{W}", out[1:-1, ..., out_off:out_off + C].cpu().double(), ref, S, 4, tdt)


def k_flow_up(E, tdt, dev, h, w, H, W, B=2):
    g = _g(5)
    v = (torch.rand(B, h, w, 2, generator=g) * 2 - 1) * 20
    out = _guarded(B, H, W, 2, torch.float32, dev)
    rc, msg = E(FLOW_UP, v.to(dev), out[1], B=B, H=H, W=W, h=h, w=w)
    assert rc == 0, msg
    _check_guards(f"flow_up {h}x{w}->{H}x{W}", out, 0, 2)
    vd = 2 * v.double().permute(0, 3, 1, 2)
    ref = F.interpolate(vd, size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    S = F.interpolate(vd.abs(), size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    # source index max(in / out * (dst + 0.5) - 0.5, 0): three roundings of a position up to the input size per axis
    S = S + (h + w + 2) * vd.abs().amax(dim=(2, 3)).view(B, 1, 1, 2)
    return _ratio(f"flow_up {h}x{w}->{H}x{W}", out[1:-1].cpu().double(), ref, S, 16, None)


def k_warp16(E, tdt, dev, C, H, W, fscale, flow_kind, B=2, src_off=0, src_pitch=None, dst_off=0, dst_pitch=None):
    """flow_kind: "out" (tens of pixels off every side), "int" (positions on integers), "small" (fractions of a pixel)."""
    g = _g(6 + C)
    src_pitch = src_pitch or src_off + C
    dst_pitch = dst_pitch or dst_off + C
    src = _src16(B, H, W, C, src_off, src_pitch, tdt, g, 3.0)
    if flow_kind == "out":
        fl = (torch.rand(B, H, W, 2, generator=g) * 2 - 1) * 3 * max(H, W) / fscale
        fl[:, : H // 4, :, 1] = -30.0 / fscale            # off the top
        fl[:, -(H // 4):, :, 1] = 30.0 / fscale           # off the bottom
        fl[:, :, : W // 4, 0] = -25.5 / fscale            # off the left
        fl[:, :, -(W // 4):, 0] = 41.25 / fscale          # off the right
    elif flow_kind == "int":
        fl = torch.randint(-3, 4, (B, H, W, 2), generator=g).float() / fscale
    else:
        fl = (torch.rand(B, H, W, 2, generator=g) * 2 - 1) * 1.5
    out = _guarded(B, H, W, dst_pitch, tdt, dev)
    sdv = src.to(dev)
    rc, msg = E(WARP16, None, None, C_=C, B=B, H=H, W=W, in_pitch=src_pitch, in1=fl.to(dev), out_pitch=dst_pitch,
                fscale=fscale, ptr0=sdv.data_ptr() + 2 * src_off, optr=out[1].data_ptr() + 2 * dst_off)
    assert rc == 0, msg
    name = f"warp16 C{C} {H}x{W} fscale {fscale} {flow_kind}"
    _check_guards(name, out, dst_off, C)
    a = src[..., src_off:src_off + C].double()
    fx, fy = fl[..., 0].double() * fscale, fl[..., 1].double() * fscale
    ref, S = _bilinear(a, fx, fy)
    S = S + _pos_term(a, fx, fy)
    return _ratio(name, out[1:-1, ..., dst_off:dst_off + C].cpu().double(), ref, S, 12, tdt)


def k_misc64(E, tdt, dev, H, W, B=2, off=128, pitch=256):
    g = _g(7)
    img = [torch.rand(B, H, W, 3, generator=g) * 1.4 - 0.2 for _ in range(2)]
    fl = [(torch.rand(B, H, W, 2, generator=g) * 2 - 1) * 2 * max(H, W) for _ in range(2)]   # bwd, fwd: many leave
    out = _guarded(B, H, W, pitch, tdt, dev)
    rc, msg = E(MISC64, img[0].to(dev), None, B=B, H=H, W=W, in1=img[1].to(dev), in2=fl[0].to(dev), in3=fl[1].to(dev),
                out_pitch=pitch, optr=out[1].data_ptr() + 2 * off)
    assert rc == 0, msg
    name = f"misc64 {H}x{W}"
    _check_guards(name, out, off, 64)
    got = out[1:-1, ..., off:off + 64].cpu()
    assert bool((got[..., 10:] == 0).all()), f"{name}: channels 10-63 are not exactly 0"
    r = 0.0
    for k, (im, f, c0) in enumerate(((img[0], fl[0], 0), (img[1], fl[1], 3))):   # image 0 through bwd, image 1 through fwd
        fx, fy = 0.5 * f[..., 0].double(), 0.5 * f[..., 1].double()
        ref, S = _bilinear(im.double(), fx, fy)
        S = S + _pos_term(im.double(), fx, fy)
        r = max(r, _ratio(f"{name} image {k}", got[..., c0:c0 + 3].double(), ref, S, 12, tdt))
    half = torch.cat([0.5 * fl[0].double(), 0.5 * fl[1].double()], -1)
    r = max(r, _ratio(f"{name} flows", got[..., 6:10].double(), half, torch.zeros_like(half), 1, tdt))
    return r


def k_nearest16(E, tdt, dev, C, h, w, H, W, B=2):
    g = _g(8)
    src = _src16(B, h, w, C, 0, C, tdt, g, 5.0)
    out = _guarded(B, H, W, C, tdt, dev)
    rc, msg = E(NEAREST16, src.to(dev), out[1], C_=C, B=B, H=H, W=W, h=h, w=w)
    assert rc == 0, msg
    name = f"nearest16 C{C} {h}x{w}->{H}x{W}"
    _check_guards(name, out, 0, C)
    ref = F.interpolate(src.double().permute(0, 3, 1, 2), size=(H, W), mode="nearest").permute(0, 2, 3, 1).to(tdt)
    assert torch.equal(out[1:-1].cpu().view(torch.int16), ref.contiguous().view(torch.int16)), f"{name}: not bit-exact"
    return 0.0


def k_flow_head(E, tdt, dev, sd, pr, with_up, H=9, W=13, B=2, off=16):
    g = _g(9 + pr)
    C = HEAD_C[pr]
    pitch = off + C + 8
    x = _src16(B, H, W, C, off, pitch, tdt, g, 2.0)
    up = (torch.rand(B, H, W, 2, generator=g) * 2 - 1) * 30 if with_up else None
    out = _guarded(B, H, W, 2, torch.float32, dev)
    xv = x.to(dev)
    rc, msg = E(FLOW_HEAD, None, out[1], C_=C, B=B, H=H, W=W, in_pitch=pitch, in1=None if up is None else up.to(dev),
                predictor=pr, ptr0=xv.data_ptr() + 2 * off)
    assert rc == 0, msg
    name = f"flow_head C{C}{' + v_up' if with_up else ''}"
    _check_guards(name, out, 0, 2)
    prefix = "predict_flow._predictor" if pr == 3 else f"predict_flow._predictors.{2 - pr}"
    w = sd[f"{prefix}._convs.4.weight"].double().view(2, C)
    b = sd[f"{prefix}._convs.4.bias"].double()
    a = x[..., off:off + C].double()
    ref = a @ w.t() + b
    S = a.abs() @ w.abs().t() + b.abs()
    if up is not None:
        ref = ref + up.double()
        S = S + up.double().abs()
    return _ratio(name, out[1:-1].cpu().double(), ref, S, C + 3, None)


def k_out_rgb(E, tdt, dev, sd, clamp01, H=11, W=6, B=3, off=64, pitch=192):
    g = _g(10)
    x = _src16(B, H, W, 64, off, pitch, tdt, g, 6.0)     # outputs well outside [0, 1]
    out = _guarded(B, H, W, 3, torch.float32, dev)
    xv = x.to(dev)
    rc, msg = E(OUT_RGB, None, out[1], B=B, H=H, W=W, in_pitch=pitch, clamp01=int(clamp01), ptr0=xv.data_ptr() + 2 * off)
    assert rc == 0, msg
    name = f"out_rgb clamp {int(clamp01)}"
    _check_guards(name, out, 0, 3)
    w = sd["fuse.output_conv.weight"].double().view(3, 64)
    b = sd["fuse.output_conv.bias"].double()
    a = x[..., off:off + 64].double()
    ref = a @ w.t() + b
    S = a.abs() @ w.abs().t() + b.abs()
    if clamp01:
        ref = ref.clamp(0, 1)
    else:
        assert float(ref.max()) > 1.5 and float(ref.min()) < -0.5, "out_rgb: inputs do not leave [0, 1]"
    return _ratio(name, out[1:-1].cpu().double(), ref, S, 65, None)


def kernel_cases():
    """(id, function name, kwargs) of every per-kernel case; each runs in both operand types."""
    cs = [("gather_C3", "k_gather", dict(C=3)), ("gather_C4_16pairs", "k_gather", dict(C=4))]
    for H, W in ((67, 33), (3, 2), (2, 3), (9, 130)):           # odd sizes floor; 1-pixel outputs
        cs.append((f"pool_rgb_{H}x{W}", "k_pool_rgb", dict(H=H, W=W)))
    for H, W in ((1, 1), (1, 9), (9, 1), (33, 67), (17, 16)):
        cs.append((f"conv_rgb_{H}x{W}", "k_conv_rgb", dict(H=H, W=W)))
    for C, H, W in ((32, 67, 33), (64, 3, 3), (128, 2, 5), (256, 33, 16), (32, 135, 9)):
        cs.append((f"pool16_C{C}_{H}x{W}", "k_pool16", dict(C=C, H=H, W=W)))
    # every ratio of the schedule: 64 -> 1, 67 -> 33 -> 16, 72 -> 9 -> 4, 1080 -> 135 -> 67 -> 33 -> 16
    for h, w, H, W in ((1, 1, 2, 2), (2, 1, 4, 2), (33, 16, 67, 33), (4, 9, 9, 18), (4, 8, 9, 16), (16, 8, 33, 16),
                       (67, 33, 135, 67), (8, 6, 16, 13), (1, 2, 3, 4)):
        cs.append((f"flow_up_{h}x{w}_{H}x{W}", "k_flow_up", dict(h=h, w=w, H=H, W=W)))
    for C in (64, 192, 448, 960):
        for fs in (1.0, 0.5):
            cs.append((f"warp16_C{C}_fs{fs:g}_out", "k_warp16", dict(C=C, H=17, W=23, fscale=fs, flow_kind="out")))
    cs.append(("warp16_C64_int", "k_warp16", dict(C=64, H=9, W=11, fscale=1.0, flow_kind="int")))
    cs.append(("warp16_C64_int_fs0.5", "k_warp16", dict(C=64, H=9, W=11, fscale=0.5, flow_kind="int")))
    cs.append(("warp16_C128_1x1", "k_warp16", dict(C=128, H=1, W=1, fscale=1.0, flow_kind="small")))
    # a source slice whose pitch is not C; a destination at channel offset C in a pitch of 2C + 64 (the aligned pyramid)
    for C in (64, 192):
        cs.append((f"warp16_C{C}_slices", "k_warp16", dict(C=C, H=13, W=10, fscale=0.5, flow_kind="out", src_off=C,
                                                          src_pitch=3 * C, dst_off=C, dst_pitch=2 * C + 64)))
    for H, W in ((17, 23), (1, 1), (4, 9)):
        cs.append((f"misc64_{H}x{W}", "k_misc64", dict(H=H, W=W)))
    for C, h, w, H, W in ((64, 9, 13, 9, 13), (128, 4, 8, 8, 16), (192, 4, 9, 9, 18), (1984, 4, 6, 9, 13),
                          (512, 16, 33, 33, 67), (64, 33, 67, 67, 135), (256, 1, 1, 2, 3)):
        cs.append((f"nearest16_C{C}_{h}x{w}_{H}x{W}", "k_nearest16", dict(C=C, h=h, w=w, H=H, W=W)))
    for pr in range(4):
        for up in (False, True):
            cs.append((f"flow_head_C{HEAD_C[pr]}{'_up' if up else ''}", "k_flow_head", dict(pr=pr, with_up=up)))
    for cl in (0, 1):
        cs.append((f"out_rgb_clamp{cl}", "k_out_rgb", dict(clamp01=cl)))
    return cs


NEEDS_SD = {"k_conv_rgb", "k_flow_head", "k_out_rgb"}


def run_kernel_case(E, fn, kw, tdt, dev, sd):
    f = globals()[fn]
    return f(E, tdt, dev, sd, **kw) if fn in NEEDS_SD else f(E, tdt, dev, **kw)


def refusal_cases():
    """(id, call kwargs, text of the refusal)."""
    return [
        ("pool16_C12", dict(kernel=POOL16, C_=12, H=8, W=8, in_pitch=12, out_pitch=12), "C must be a multiple of 8"),
        ("warp16_C60", dict(kernel=WARP16, C_=60, H=4, W=4, in_pitch=60, out_pitch=60), "C must be a multiple of 8"),
        ("nearest16_C20", dict(kernel=NEAREST16, C_=20, H=4, W=4, h=2, w=2), "C must be a multiple of 8"),
        ("flow_head_C136", dict(kernel=FLOW_HEAD, C_=136, H=4, W=4, in_pitch=136, predictor=3),
         "flow_head reads at most 128 channels"),
        ("flow_head_C64_on_predictor_3", dict(kernel=FLOW_HEAD, C_=64, H=4, W=4, in_pitch=64, predictor=3),
         "flow_head of predictor 3 reads 128 channels"),
        ("pool16_1_row", dict(kernel=POOL16, C_=64, H=1, W=8, in_pitch=64, out_pitch=64), "level too small to pool"),
        ("pool_rgb_1_col", dict(kernel=POOL_RGB, H=8, W=1), "level too small to pool"),
    ]


def check_refusal(E, dev, kw, why):
    buf = torch.full((4096 * 4,), NAN, dtype=torch.float32, device=dev)
    before = buf.clone()
    kernel = kw.pop("kernel")
    rc, msg = E(kernel, buf, buf, in1=None, **kw)
    assert rc != 0, (kernel, kw)
    assert why in msg, msg
    assert torch.equal(buf.isnan(), before.isnan()), "refused, yet the buffer changed"


# ----------------------------------------------------------------------------------------------------- whole path
MARGIN = 4.0
# (id, h, w, weight seed, flow_gain, frames: clip seed or -1 for white noise outside [0, 1])
PATH_CASES = [
    ("64x64_noise_g1", 64, 64, 2, 1.0, -1),        # level 6 is 1 x 1 (film_net_64x64_rand)
    ("72x104_clip_g2", 72, 104, 1, 2.0, 42),       # film_net_72x104
    ("67x130_clip_g4", 67, 130, 11, 4.0, 7),       # odd at level 0; warps reach the border
    ("200x64_noise_g4", 200, 64, 12, 4.0, -1),
]
# max |engine - oracle| of the host emulation (frame, flow in px over all 7 levels of both directions)
OBSERVED = {  # case: (float16 (frame, flow), bfloat16 (frame, flow))
    "64x64_noise_g1": ((1.82e-03, 5.62e-03), (1.88e-02, 6.80e-02)),
    "72x104_clip_g2": ((1.95e-03, 1.00e-02), (1.78e-02, 8.31e-02)),
    "67x130_clip_g4": ((3.65e-03, 1.66e-02), (2.83e-02, 1.72e-01)),
    "200x64_noise_g4": ((8.34e-03, 5.88e-02), (7.15e-02, 3.85e-01)),
}


def path_inputs(case):
    _, h, w, seed, gain, clip = case
    sd = OF.synthetic_state_dict(seed, gain)
    if clip < 0:
        g = torch.Generator().manual_seed(98 + h + w)
        fr = torch.rand(2, h, w, 3, generator=g) * 1.2 - 0.1
    else:
        fr = OF.synthetic_clip(2, h, w, seed=clip)
    return sd, fr


def path_oracle(sd, fr, f0, f1, operand, device="cpu"):
    """(frame [B,h,w,3] unclamped, flows[dir][level] [B,H_l,W_l,2]) of the faithful oracle for pairs (f0[i], f1[i])."""
    x = fr.to(device).permute(0, 3, 1, 2)
    d: Dict = {}
    sdd = {k: v.to(device) for k, v in sd.items()}
    out = OF.interpolator_forward(sdd, x[list(f0)], x[list(f1)], torch.full((len(f0), 1), 0.5, device=device), d,
                                  operand=operand)
    flows = [[v.permute(0, 2, 3, 1) for v in d[k]] for k in ("forward_flow_levels", "backward_flow_levels")]
    return out.permute(0, 2, 3, 1), flows


def tol(case_id, operand):
    i = 0 if operand == "float16" else 1
    obs = OBSERVED[case_id][i] if case_id in OBSERVED else tuple(max(v[i][k] for v in OBSERVED.values()) for k in range(2))
    return MARGIN * obs[0], MARGIN * obs[1]


def path_compare(label, got, want, h, w, tf, tv):
    """got / want: (frame, flows[dir][level]); returns (report lines, failures, worst frame error, worst flow error)."""
    lines, fails = compare(label, [got[0]], [want[0]], h, w, {"frame": tf}, names=("frame",))
    worst_v = 0.0
    for d, dn in enumerate(("fwd", "bwd")):
        for l in range(LEVELS):
            g, r = got[1][d][l], want[1][d][l]
            nm = f"{dn}{l}"
            ln, fl = compare(label, [g], [r], h >> l, w >> l, {nm: tv}, names=(nm,))
            lines += ln
            fails += fl
            worst_v = max(worst_v, float((g.to(r.device).double() - r.double()).abs().max()))
    worst_f = float((got[0].to(want[0].device).double() - want[0].double()).abs().max())
    return lines, fails, worst_f, worst_v
