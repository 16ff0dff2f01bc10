"""Op-level surface of the reference's `vfi_models.ops` package (vfi_models/ops/__init__.py:19-21), backed by the
ahead-of-time sm_90a kernels in libvfi_b200.so instead of cupy/NVRTC or taichi.  Same names, argument meaning and
tensor contract (CUDA float32 NCHW); inference only - the reference's backward kernels (training) are out of scope.
There is no CPU path: CPU tensors raise.
"""
import ctypes as C

import torch

from ._lib import VfiError, check, lib

_ctx = {}


def _context(device: torch.device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _ctx:
        h = C.c_void_p()
        check(lib().vfi_create(idx, C.byref(h)))
        _ctx[idx] = h
    return _ctx[idx]


def _prep(*ts):
    out = []
    for t in ts:
        if not t.is_cuda:
            raise VfiError("vfi ops need CUDA tensors (no CPU fallback)")
        out.append(t.to(torch.float32).contiguous())  # reference: @custom_fwd(cast_inputs=torch.float32)
    return out


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def init():
    """Reference: cupy_ops.init() warms the NVRTC cache; nothing to compile here."""
    return None


class softsplat_func:
    """cupy_ops/softsplat.py:195-224 (forward only)."""

    @staticmethod
    def apply(tenIn, tenFlow):
        tenIn, tenFlow = _prep(tenIn, tenFlow)
        n, c, h, w = tenIn.shape
        assert tuple(tenFlow.shape) == (n, 2, h, w)
        out = torch.empty_like(tenIn)
        check(lib().vfi_softsplat_sum(_context(tenIn.device), tenIn.data_ptr(), tenFlow.data_ptr(), out.data_ptr(),
                                      n, c, h, w, _stream(tenIn)))
        return out


_SPLAT_MODE = {"avg": 0, "linear": 1, "soft": 2}
_SPLAT_EPS = {"addeps": 0, "zeroeps": 1, "clipeps": 2}


def softsplat(tenIn, tenFlow, tenMetric, strMode: str):
    """Forward splat with the reference's modes - same call contract as cupy_ops/softsplat.py:382-435: strMode is
    "sum" | "avg" | "linear" | "soft", the last three optionally suffixed "-addeps" (default) / "-zeroeps" / "-clipeps";
    tenMetric is required for linear / soft and must be None for sum / avg.

    Not the reference's tensor chain (concatenate a weight channel, splat C + 1 channels, slice, divide): "sum" is one
    launch of the splat kernel; the weighted modes go through vfi_softsplat_weighted, which applies the per-source-pixel
    weight (1, metric or exp(metric)) while splatting, splats the weights into one normalisation plane and divides in a
    second launch - no temporaries and about half the HBM traffic."""
    base, _, variant = strMode.partition("-")
    if base == "sum":
        if tenMetric is not None or variant:
            raise AssertionError("sum mode takes no metric and no eps variant")
        return softsplat_func.apply(tenIn, tenFlow)
    if base not in _SPLAT_MODE or (variant or "addeps") not in _SPLAT_EPS:
        raise AssertionError(f"unknown softsplat mode {strMode!r}")
    needs_metric = base != "avg"
    if needs_metric != (tenMetric is not None):
        raise AssertionError(f"{base} mode {'needs' if needs_metric else 'takes no'} metric")
    if needs_metric:
        tenIn, tenFlow, tenMetric = _prep(tenIn, tenFlow, tenMetric)
    else:
        tenIn, tenFlow = _prep(tenIn, tenFlow)
    n, c, h, w = tenIn.shape
    out = torch.empty_like(tenIn)
    norm = tenIn.new_empty(n, 1, h, w)
    check(lib().vfi_softsplat_weighted(_context(tenIn.device), tenIn.data_ptr(), tenFlow.data_ptr(),
                                       tenMetric.data_ptr() if needs_metric else None, _SPLAT_MODE[base],
                                       _SPLAT_EPS[variant or "addeps"], out.data_ptr(), norm.data_ptr(), n, c, h, w,
                                       _stream(tenIn)))
    return out


def FunctionSoftsplat(tenInput, tenFlow, tenMetric, strType):
    """cupy_ops/softsplat.py:325-358 (older spelling used by EISAI): summation / average / linear / softmax."""
    mode = {"summation": "sum", "average": "avg", "linear": "linear", "softmax": "soft"}[strType]
    return softsplat(tenInput, tenFlow, tenMetric, mode)


class ModuleSoftsplat(torch.nn.Module):
    def __init__(self, strType):
        super().__init__()
        self.strType = strType

    def forward(self, tenInput, tenFlow, tenMetric):
        return FunctionSoftsplat(tenInput, tenFlow, tenMetric, self.strType)


class costvol_func:
    """cupy_ops/costvol.py:135-179 (forward only): [N,C,H,W] x2 -> [N,81,H,W]."""

    @staticmethod
    def apply(tenOne, tenTwo):
        tenOne, tenTwo = _prep(tenOne, tenTwo)
        n, c, h, w = tenOne.shape
        out = tenOne.new_empty([n, 81, h, w])
        check(lib().vfi_costvol_l1(_context(tenOne.device), tenOne.data_ptr(), tenTwo.data_ptr(), out.data_ptr(),
                                   n, c, h, w, _stream(tenOne)))
        return out


class sepconv_func:
    """cupy_ops/sepconv.py:155-190 (forward only): in [N,C,H+Kv-1,W+Kh-1], ver [N,Kv,H,W], hor [N,Kh,H,W]."""

    @staticmethod
    def apply(tenIn, tenVer, tenHor):
        tenIn, tenVer, tenHor = _prep(tenIn, tenVer, tenHor)
        n, c = tenIn.shape[:2]
        kv, kh = tenVer.shape[1], tenHor.shape[1]
        h, w = tenVer.shape[2], tenVer.shape[3]
        assert tenIn.shape[2] == h + kv - 1 and tenIn.shape[3] == w + kh - 1 and tuple(tenHor.shape[2:]) == (h, w)
        out = tenIn.new_empty([n, c, h, w])
        check(lib().vfi_sepconv(_context(tenIn.device), tenIn.data_ptr(), tenVer.data_ptr(), tenHor.data_ptr(),
                                out.data_ptr(), n, c, h, w, kv, kh, _stream(tenIn)))
        return out


class _FunctionCorrelation:
    """cupy_ops/correlation.py:231-296 (forward only)."""

    @staticmethod
    def apply(first, second):
        first, second = _prep(first, second)
        n, c, h, w = first.shape
        out = first.new_empty([n, 81, h, w])
        check(lib().vfi_corr_dot(_context(first.device), first.data_ptr(), second.data_ptr(), out.data_ptr(),
                                 n, c, h, w, _stream(first)))
        return out


def FunctionCorrelation(tenFirst, tenSecond):
    return _FunctionCorrelation.apply(tenFirst, tenSecond)


class ModuleCorrelation(torch.nn.Module):
    def forward(self, tenFirst, tenSecond):
        return _FunctionCorrelation.apply(tenFirst, tenSecond)


def batch_edt(img, block=1024):
    """cupy_ops/batch_edt.py:46-117: Euclidean distance transform of a batch of line drawings (white lines, black
    whitespace), img (bs,h,w) or (bs,1,h,w); `block` is accepted for signature compatibility only."""
    expand = False
    if len(img.shape) == 4:
        assert img.shape[1] == 1
        img = img.squeeze(1)
        expand = True
    if not img.is_cuda:
        raise VfiError("vfi ops need CUDA tensors (no CPU fallback)")  # the reference raises NotImplementedError here (:97)
    bs, h, w = img.shape
    diam2 = h ** 2 + w ** 2
    odtype = img.dtype
    ctx, st = _context(img.device), _stream(img)
    data = ((1 - img.type(torch.float32)) * diam2).contiguous()           # first pass, y-axis (:66-80)
    intermed = torch.empty_like(data)
    check(lib().vfi_edt_pass(ctx, data.data_ptr(), intermed.data_ptr(), bs, h, w, float(diam2), st))
    intermed = intermed.permute(0, 2, 1).contiguous()                     # second pass, x-axis (:82-95)
    out = torch.empty_like(intermed)
    check(lib().vfi_edt_pass(ctx, intermed.data_ptr(), out.data_ptr(), bs, w, h, float(diam2), st))
    ans = out.permute(0, 2, 1).sqrt()
    ans = ans.type(odtype) if odtype != ans.dtype else ans
    if expand:
        ans = ans.unsqueeze(1)
    return ans


class FunctionAdaCoF:
    """cupy_ops/adacof.py:259-330 (forward only): adaptive collaboration of flows."""

    @staticmethod
    def apply(input, weight, offset_i, offset_j, dilation):
        input, weight, offset_i, offset_j = _prep(input, weight, offset_i, offset_j)
        n, c, hin, win = input.shape
        f = int(round(weight.size(1) ** 0.5))
        ho, wo = weight.size(2), weight.size(3)
        assert hin - ((f - 1) * dilation + 1) == ho - 1 and win - ((f - 1) * dilation + 1) == wo - 1
        assert tuple(offset_i.shape) == tuple(weight.shape) == tuple(offset_j.shape)
        out = input.new_empty(n, c, ho, wo)
        check(lib().vfi_adacof(_context(input.device), input.data_ptr(), weight.data_ptr(), offset_i.data_ptr(),
                               offset_j.data_ptr(), out.data_ptr(), n, c, hin, win, f, int(dilation), ho, wo, _stream(input)))
        return out
