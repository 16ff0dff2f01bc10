"""Host-side engine: owns a vfi_ctx, feeds it PyTorch device memory / host buffers through the C ABI.

PyTorch is plumbing here (device memory, streams); all arithmetic of the path runs in libvfi_b200.so.
"""
import ctypes as C
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from ._lib import VfiError, check, lib

OPERAND = {"float32": 0, "float16": 0, "bfloat16": 1}
# names in IFNet("4.6").state_dict() order (reference rife_arch.py:177-218, :404-408)
BLOCK_C = (192, 128, 96, 64)


def state_dict_names(arch: str = "4.6"):
    names = []
    for b in range(5 if arch == "4.26" else 4):  # rife_arch.py:453-459: arch 4.26 has block0..block4
        p = f"block{b}."
        names += [p + "conv0.0.0.weight", p + "conv0.0.0.bias", p + "conv0.1.0.weight", p + "conv0.1.0.bias"]
        for j in range(8):
            q = p + f"convblock.{j}."
            names += [q + "beta", q + "conv.weight", q + "conv.bias"]
        names += [p + "lastconv.0.weight", p + "lastconv.0.bias"]
    if arch == "4.7":
        names += ["encode.0.weight", "encode.0.bias", "encode.1.weight", "encode.1.bias"]
    if arch in ("4.17", "4.26"):  # Head_417 - rife_arch.py:356-363; Head - rife_arch.py:378-385
        names += [f"encode.cnn{i}.{k}" for i in range(4) for k in ("weight", "bias")]
    return names


ARCH_CODE = {"4.6": 46, "4.7": 47, "4.17": 417, "4.26": 426}


def _i32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32))


def host_copy_frames(frames: torch.Tensor, slots, out: torch.Tensor, threads: int = 0):
    """out[slots[i]] = frames[i, ..., :3] for every i with slots[i] >= 0 (CPU float32 tensors), on `threads` copy threads of
    the library (default VFI_COPY_THREADS or 12) - vfi_host_copy_frames."""
    assert not frames.is_cuda and not out.is_cuda and frames.dtype == torch.float32 and out.dtype == torch.float32
    assert frames.is_contiguous() and out.is_contiguous() and frames.dim() == 4 and tuple(out.shape[1:3]) == tuple(frames.shape[1:3])
    n, h, w, c = frames.shape
    sl = _i32(slots)
    assert len(sl) == n and (len(sl) == 0 or int(sl.max()) < out.shape[0]) and out.shape[3] == 3
    if threads <= 0:
        import os
        threads = int(os.environ.get("VFI_COPY_THREADS", "12"))
    check(lib().vfi_host_copy_frames(frames.data_ptr(), n, h, w, c, sl.ctypes.data, out.data_ptr(), int(threads)))


class Rife46Engine:
    """RIFE 4.6 / 4.7 / 4.17 / 4.26 (rife46.pth; rife47.pth, rife49.pth; rife417.pth; rife426.pth) on one H100.  `state_dict` maps the reference's parameter names to tensors (any float dtype)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32", batch: int = 8,
                 arch: str = None):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        if arch is None:  # the 4.7 family (rife47.pth / rife49.pth) has the encode head, rife417.pth the Head_417 one
            arch = ("4.26" if "block4.conv0.0.0.weight" in state_dict else
                    "4.17" if "encode.cnn0.weight" in state_dict else
                    "4.7" if "encode.0.weight" in state_dict else "4.6")
        if arch not in ARCH_CODE:
            raise VfiError(f"RIFE arch {arch} is not built (4.6, 4.7, 4.17 and 4.26 are)")
        self.arch = arch
        names = state_dict_names(arch)
        missing = [n for n in names if n not in state_dict]
        if missing:
            raise KeyError(f"state_dict is not a RIFE {arch} checkpoint; missing {missing[:3]} ...")
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n in names]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_rife_load(self._ctx, ARCH_CODE[arch], ptrs, numel, len(hold), OPERAND[dtype]))
        check(self._L.vfi_set_batch(self._ctx, int(batch)))
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ device-resident path
    def forward(self, frames: torch.Tensor, f0: Sequence[int], f1: Sequence[int], t: Sequence[float],
                scale_factor: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: CUDA float32 [N,H,W,C>=3] NHWC; returns CUDA float32 [len(t),H,W,3] on the current stream."""
        assert frames.is_cuda and frames.dtype == torch.float32 and frames.is_contiguous() and frames.dim() == 4
        n, h, w, c = frames.shape
        f0a, f1a = _i32(f0), _i32(f1)
        ta = np.ascontiguousarray(np.asarray(t, dtype=np.float32))
        nt = len(ta)
        if out is None:
            out = torch.empty((nt, h, w, 3), dtype=torch.float32, device=frames.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (nt, h, w, 3)
        st = torch.cuda.current_stream(frames.device).cuda_stream
        check(self._L.vfi_rife46_forward(self._ctx, frames.data_ptr(), n, h, w, c, f0a.ctypes.data, f1a.ctypes.data,
                                         ta.ctypes.data, nt, float(scale_factor), out.data_ptr(), st))
        return out

    # ------------------------------------------------------------------ host-buffer path (node / e2e)
    def interpolate_host(self, frames: torch.Tensor, f0, f1, t, out: torch.Tensor, out_slots=None,
                         frame_range=None, scale_factor: float = 1.0, frame_slots=None):
        """frames: CPU float32 [N,H,W,C]; out: CPU float32 [M,H,W,3]; task i -> out[out_slots[i]] (default i);
        frame_slots (optional, one per source frame, -1 = none): frame i is also copied unchanged to out[frame_slots[i]]."""
        assert not frames.is_cuda and frames.dtype == torch.float32 and frames.is_contiguous()
        assert not out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()
        n, h, w, c = frames.shape
        assert tuple(out.shape[1:]) == (h, w, 3)
        f0a, f1a = _i32(f0), _i32(f1)
        ta = np.ascontiguousarray(np.asarray(t, dtype=np.float32))
        lo, hi = (0, n) if frame_range is None else frame_range
        slots = None
        if out_slots is not None:
            slots = _i32(out_slots)
            assert len(slots) == len(ta) and (len(slots) == 0 or int(slots.max()) < out.shape[0])
        else:
            assert out.shape[0] >= len(ta)
        fslots = None
        if frame_slots is not None:
            fslots = _i32(frame_slots)
            assert len(fslots) == n and int(fslots.max()) < out.shape[0]
        check(self._L.vfi_rife46_interpolate_host(
            self._ctx, frames.data_ptr(), n, h, w, c, int(lo), int(hi), f0a.ctypes.data, f1a.ctypes.data,
            ta.ctypes.data, None if slots is None else slots.ctypes.data, None if fslots is None else fslots.ctypes.data,
            len(ta), float(scale_factor), out.data_ptr()))
        return out

    # ------------------------------------------------------------------ primitives / hooks
    def warp(self, img: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
        """NHWC float32 CUDA: img [B,H,W,C], flow [B,H,W,2] (pixels) -> [B,H,W,C]  (rife_arch.warp semantics)."""
        assert img.is_cuda and flow.is_cuda and img.is_contiguous() and flow.is_contiguous()
        b, h, w, c = img.shape
        assert tuple(flow.shape) == (b, h, w, 2)
        out = torch.empty_like(img)
        st = torch.cuda.current_stream(img.device).cuda_stream
        check(self._L.vfi_warp_bilinear_border(self._ctx, img.data_ptr(), flow.data_ptr(), out.data_ptr(), b, h, w, c, st))
        return out

    def debug_layer(self, block, layer, x, out, out_mask=None, impl=0):
        b, h, w = x.shape[0], x.shape[1], x.shape[2]
        st = torch.cuda.current_stream(x.device).cuda_stream
        check(self._L.vfi_rife46_debug_layer(self._ctx, block, layer, x.data_ptr(), out.data_ptr(),
                                             None if out_mask is None else out_mask.data_ptr(), b, h, w, impl, st))
        return out

    def layer_plan(self, block, layer):
        st, nc, ns, sm, mc, cm, ws = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int64(), C.c_int(), C.c_int()
        check(self._L.vfi_rife46_layer_plan(self._ctx, block, layer, C.byref(st), C.byref(nc), C.byref(ns),
                                            C.byref(sm), C.byref(mc), C.byref(cm), C.byref(ws)))
        return dict(stages=st.value, n_cta=nc.value, nsplit=ns.value, smem_bytes=sm.value, macs_per_cell=mc.value,
                    cmajor=bool(cm.value), wstream=bool(ws.value))

    def debug_conv0_fused(self, block, x, out):
        """conv0.0 -> conv0.1 of `block` as the one fused launch: x [B,H,W,64] 16-bit -> out [B,H/2,W/2,64] 16-bit."""
        b, h, w = x.shape[0], x.shape[1], x.shape[2]
        st = torch.cuda.current_stream(x.device).cuda_stream
        check(self._L.vfi_rife46_debug_conv0_fused(self._ctx, block, x.data_ptr(), out.data_ptr(), b, h, w, st))
        return out

    def set_unfused_conv0(self, unfused: bool):
        """Test hook: run every block's conv0.0 and conv0.1 as two launches (True) or fused where possible (False)."""
        check(self._L.vfi_rife46_debug_unfused_conv0(self._ctx, 1 if unfused else 0))

    def conv0_plan(self, block):
        v = np.zeros(5, np.int32)
        check(self._L.vfi_rife46_conv0_plan(self._ctx, block, v.ctypes.data, 5))
        return dict(fused=bool(v[0]), stages=int(v[1]), smem_bytes=int(v[2]), regs=int(v[3]), local_bytes=int(v[4]))

    def debug_state(self, batch):
        """(flow [B,Hp,Wp,4], mask [B,Hp,Wp]) of the last internal pass as torch CUDA tensors."""
        hp, wp = C.c_int(), C.c_int()
        check(self._L.vfi_rife46_debug_state(self._ctx, None, None, batch, C.byref(hp), C.byref(wp)))
        flow = torch.empty((batch, hp.value, wp.value, 4), dtype=torch.float32, device=f"cuda:{self.device}")
        mask = torch.empty((batch, hp.value, wp.value), dtype=torch.float32, device=f"cuda:{self.device}")
        check(self._L.vfi_rife46_debug_state(self._ctx, flow.data_ptr(), mask.data_ptr(), batch, C.byref(hp),
                                             C.byref(wp)))
        return flow, mask

    def profile(self, enable: bool):
        """Start / stop per-kernel-group event timing of the forward schedule (vfi_rife_profile)."""
        check(self._L.vfi_rife_profile(self._ctx, 1 if enable else 0))

    def profile_read(self):
        """{group id: (total ms, spans)} since profile(True); ids: 10 * block + {0 front, 1 conv0.0, 2 conv0.1, 3 ResConv x8,
        4 lastconv}, 90 final."""
        ids = np.zeros(64, np.int32)
        ms = np.zeros(64, np.float32)
        cnt = np.zeros(64, np.int32)
        n = C.c_int()
        check(self._L.vfi_rife_profile_read(self._ctx, ids.ctypes.data, ms.ctypes.data, cnt.ctypes.data, 64, C.byref(n)))
        return {int(ids[i]): (float(ms[i]), int(cnt[i])) for i in range(n.value)}

    def set_batch(self, b):
        check(self._L.vfi_set_batch(self._ctx, int(b)))

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# ------------------------------------------------------------------------------------------------- FILM
def film_state_dict_names():
    """film_arch.Interpolator().state_dict() order (film_arch.py:91-100, :515-528, :550-565, :222-256, :391-393)."""
    names = []
    for i in range(4):
        for j in range(2):
            names += [f"extract.extract_sublevels.convs.{i}.{j}.0.weight", f"extract.extract_sublevels.convs.{i}.{j}.0.bias"]
    for prefix in ["predict_flow._predictor"] + [f"predict_flow._predictors.{k}" for k in range(3)]:
        for j in range(4):
            names += [f"{prefix}._convs.{j}.0.weight", f"{prefix}._convs.{j}.0.bias"]
        names += [f"{prefix}._convs.4.weight", f"{prefix}._convs.4.bias"]
    names += ["fuse.output_conv.weight", "fuse.output_conv.bias"]
    for k in range(4):
        names += [f"fuse.convs.{k}.0.weight", f"fuse.convs.{k}.0.bias"]
        for j in (1, 2):
            names += [f"fuse.convs.{k}.{j}.0.weight", f"fuse.convs.{k}.{j}.0.bias"]
    return names


class FilmEngine:
    """FILM (film_net_fp32.pt) on one H100: `state_dict` = the TorchScript module's / Interpolator's state_dict."""

    MAX_PAIRS = 16

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        names = film_state_dict_names()
        missing = [n for n in names if n not in state_dict]
        if missing:
            raise KeyError(f"state_dict is not a FILM checkpoint; missing {missing[:3]} ...")
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n in names]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_film_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, frames: torch.Tensor, f0: Sequence[int], f1: Sequence[int], clamp: bool = False,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: CUDA float32 [N,H,W,C>=3] NHWC -> CUDA float32 [len(f0),H,W,3]: the midpoint frame of every pair
        (Interpolator.forward, film_arch.py:458-459), optionally clamped to [0,1] as the node does (film/__init__.py:38)."""
        assert frames.is_cuda and frames.dtype == torch.float32 and frames.is_contiguous() and frames.dim() == 4
        n, h, w, c = frames.shape
        f0a, f1a = _i32(f0), _i32(f1)
        npairs = len(f0a)
        assert npairs == len(f1a) and 1 <= npairs <= self.MAX_PAIRS
        if out is None:
            out = torch.empty((npairs, h, w, 3), dtype=torch.float32, device=frames.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (npairs, h, w, 3)
        st = torch.cuda.current_stream(frames.device).cuda_stream
        check(self._L.vfi_film_forward(self._ctx, frames.data_ptr(), n, h, w, c, f0a.ctypes.data, f1a.ctypes.data, npairs,
                                       1 if clamp else 0, out.data_ptr(), st))
        return out

    def midpoint(self, x0: torch.Tensor, x1: torch.Tensor) -> torch.Tensor:
        """[H,W,3] x 2 (CUDA float32) -> clamped midpoint [H,W,3]: one `model(x0, x1, dt).clamp(0, 1)` of the node."""
        pair = torch.stack([x0, x1]).contiguous()
        return self.forward(pair, [0], [1], clamp=True)[0]

    # ------------------------------------------------------------------ hooks
    def set_ref(self, use_ref: bool):
        check(self._L.vfi_film_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_conv(self, group, layer, src0, src1, out, B, H, W, impl=0, pitch0=None, pitch1=None, out_pitch=None):
        st = torch.cuda.current_stream(src0.device).cuda_stream
        check(self._L.vfi_film_debug_conv(
            self._ctx, group, layer, src0.data_ptr(), int(pitch0 if pitch0 is not None else src0.shape[-1]),
            None if src1 is None else src1.data_ptr(),
            0 if src1 is None else int(pitch1 if pitch1 is not None else src1.shape[-1]),
            out.data_ptr(), int(out_pitch if out_pitch is not None else out.shape[-1]), B, H, W, impl, st))
        return out

    def debug_state(self, direction, level, batch):
        """Flow v[direction][level] of the last forward (0 forward, 1 backward; level 0..6) as a CUDA float32
        [batch, H_l, W_l, 2] tensor (vfi_film_debug_state)."""
        h, w = C.c_int(), C.c_int()
        check(self._L.vfi_film_debug_state(self._ctx, direction, level, None, batch, C.byref(h), C.byref(w)))
        out = torch.empty((batch, h.value, w.value, 2), dtype=torch.float32, device=f"cuda:{self.device}")
        check(self._L.vfi_film_debug_state(self._ctx, direction, level, out.data_ptr(), batch, C.byref(h), C.byref(w)))
        return out

    def debug_elem(self, kernel, in0, out, C_, B, H, W, in_pitch=0, in1=None, in2=None, in3=None, frame_idx=None,
                   out_pitch=0, h=0, w=0, fscale=1.0, clamp01=False, predictor=0):
        """One film_elem.cu kernel on CUDA tensors (vfi_film_debug_elem; kernel ids in include/vfi_b200.h).  in* and out
        may be tensor views: their data_ptr() is the slice start, the pitches are in elements."""
        p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        idx = None if frame_idx is None else _i32(frame_idx)
        st = torch.cuda.current_stream(in0.device).cuda_stream
        check(self._L.vfi_film_debug_elem(self._ctx, kernel, p(in0), int(in_pitch), p(in1), p(in2), p(in3),
                                          None if idx is None else idx.ctypes.data, p(out), int(out_pitch), int(C_), B, H,
                                          W, h, w, float(fscale), 1 if clamp01 else 0, predictor, st))
        return out

    def layer_plan(self, group, layer):
        v = [C.c_int() for _ in range(10)]
        check(self._L.vfi_film_layer_plan(self._ctx, group, layer, *[C.byref(x) for x in v]))
        keys = ("c0", "c1", "n_total", "ksize", "n_cta", "nsplit", "mt", "a_slots", "b_slots", "smem_bytes")
        return dict(zip(keys, [x.value for x in v]))

    def last_macs(self) -> int:
        return int(self._L.vfi_film_last_macs(self._ctx))

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# ------------------------------------------------------------------------------------------------- Sepconv
def sepconv_state_dict_names():
    """sepconv_enhanced.Network().state_dict() order (sepconv_enhanced.py:536-598)."""
    names = ["netInput.weight", "netInput.bias"]

    def basic(prefix, prelu0, c0, prelu1, c1):
        out = []
        if prelu0 is not None:
            out.append(f"{prefix}.netMain.{prelu0}.weight")
        out += [f"{prefix}.netMain.{c0}.weight", f"{prefix}.netMain.{c0}.bias", f"{prefix}.netMain.{prelu1}.weight",
                f"{prefix}.netMain.{c1}.weight", f"{prefix}.netMain.{c1}.bias"]
        return out

    for r in range(1, 5):
        names += basic(f"netEncode.0.netVer.{r}", 0, 1, 2, 3)
    for k in range(4):
        names += basic(f"netDecode.0.netHor.{k}", 0, 1, 2, 3)
    for k in range(1, 4):
        names += basic(f"netDecode.0.netVer.{k}", 0, 2, 3, 4)
    for head in ("netVerone", "netVertwo", "netHorone", "netHortwo"):
        names += basic(head, None, 1, 2, 3)
    return names


class SepconvEngine:
    """Sepconv (sepconv.pth) on one H100: `state_dict` = sepconv_enhanced.Network's."""

    MAX_PAIRS = 16

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        names = sepconv_state_dict_names()
        missing = [n for n in names if n not in state_dict]
        if missing:
            raise KeyError(f"state_dict is not a Sepconv checkpoint; missing {missing[:3]} ...")
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n in names]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_sepconv_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        self._dt16 = torch.bfloat16 if dtype == "bfloat16" else torch.float16

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, frames: torch.Tensor, f0: Sequence[int], f1: Sequence[int],
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: CUDA float32 [N,H,W,C>=3] NHWC -> CUDA float32 [len(f0),H,W,3] = Network.forward(frame f0, frame f1)."""
        assert frames.is_cuda and frames.dtype == torch.float32 and frames.is_contiguous() and frames.dim() == 4
        n, h, w, c = frames.shape
        f0a, f1a = _i32(f0), _i32(f1)
        npairs = len(f0a)
        assert npairs == len(f1a) and 1 <= npairs <= self.MAX_PAIRS
        if out is None:
            out = torch.empty((npairs, h, w, 3), dtype=torch.float32, device=frames.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (npairs, h, w, 3)
        st = torch.cuda.current_stream(frames.device).cuda_stream
        check(self._L.vfi_sepconv_forward(self._ctx, frames.data_ptr(), n, h, w, c, f0a.ctypes.data, f1a.ctypes.data, npairs,
                                          out.data_ptr(), st))
        return out

    def middle_frame(self, frame_0: torch.Tensor, frame_1: torch.Tensor) -> torch.Tensor:
        """NCHW [1,3,H,W] x 2 -> NCHW [1,3,H,W]: `model(frame_0, frame_1)` as generic_frame_loop calls it
        (sepconv/__init__.py:47-48)."""
        dev = torch.device("cuda", self.device)
        pair = torch.cat([frame_0, frame_1]).to(dev, torch.float32).permute(0, 2, 3, 1).contiguous()
        return self.forward(pair, [0], [1]).permute(0, 3, 1, 2)

    def set_ref(self, use_ref: bool):
        check(self._L.vfi_sepconv_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_state(self, what, index, batch):
        """A tensor of the last forward as a CUDA tensor (vfi_sepconv_debug_state): what 0 = coefficient plane `index`
        (0 Verone, 1 Vertwo, 2 Horone, 3 Hortwo) float32 [batch, 51, He, We]; 1 = pyramid row `index` (1..4) after
        decoding, [batch, h, w, C] in the operand type; 2 = the per-pair (sum, sum of squares) float64 [batch, 2]."""
        shape = (C.c_int * 4)()
        check(self._L.vfi_sepconv_debug_state(self._ctx, what, index, None, batch, shape))
        dt = {0: torch.float32, 1: self._dt16, 2: torch.float64}[what]
        out = torch.empty(tuple(shape) if what != 2 else (batch, 2), dtype=dt, device=f"cuda:{self.device}")
        check(self._L.vfi_sepconv_debug_state(self._ctx, what, index, out.data_ptr(), batch, shape))
        return out

    def debug_elem(self, kernel, in0, out, C_, B, H, W, in1=None, f0=None, f1=None, n_frames=0, h=0, w=0, slope=1.0,
                   which=0):
        """One sepconv_elem.cu kernel on CUDA tensors (vfi_sepconv_debug_elem; kernel ids in include/vfi_b200.h)."""
        p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        a = None if f0 is None else _i32(f0)
        b = None if f1 is None else _i32(f1)
        st = torch.cuda.current_stream(in0.device).cuda_stream
        check(self._L.vfi_sepconv_debug_elem(self._ctx, kernel, p(in0), p(in1), None if a is None else a.ctypes.data,
                                             None if b is None else b.ctypes.data, int(n_frames), p(out), int(C_), B, H, W,
                                             h, w, float(slope), int(which), st))
        return out

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# ------------------------------------------------------------------------------------------------- FLAVR
def flavr_state_dict_names(enc_bias: bool = False):
    """UNet_3D_3D("unet_18", 4, n_outputs).state_dict() order (flavr_arch.py:134-164, resnet_3D.py:118-151); the
    encoder convs carry a bias only in the 4x / 8x checkpoints (resnet_3D.useBias)."""
    names = ["encoder.stem.0.weight"] + (["encoder.stem.0.bias"] if enc_bias else [])
    for l in range(1, 5):
        for b in range(2):
            p = f"encoder.layer{l}.{b}."
            for conv in ("conv1", "conv2"):
                names += [p + conv + ".0.weight"] + ([p + conv + ".0.bias"] if enc_bias else [])
            names += [p + "fg.attn_layer.0.weight", p + "fg.attn_layer.0.bias"]
            if b == 0 and l > 1:
                names.append(p + "downsample.0.weight")
    for d in range(5):
        m = "upconv" if d in (1, 2, 4) else "conv"
        names += [f"decoder.{d}.{m}.0.weight", f"decoder.{d}.{m}.0.bias", f"decoder.{d}.{m}.1.attn_layer.0.weight",
                  f"decoder.{d}.{m}.1.attn_layer.0.bias"]
    return names + ["feature_fuse.conv.0.weight", "outconv.1.weight", "outconv.1.bias"]


class FlavrEngine:
    """FLAVR (FLAVR_2x.pth / FLAVR_4x.pth / FLAVR_8x.pth) on one H100: `state_dict` = UNet_3D_3D's, keys without the
    `module.` prefix.  Whether the encoder convs carry a bias and how many outputs the model has are read from the
    state dict; only output 0 is computed (the node uses no other)."""

    MAX_WINDOWS = 8

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        names = flavr_state_dict_names("encoder.stem.0.bias" in state_dict)
        missing = [n for n in names if n not in state_dict]
        if missing:
            raise KeyError(f"state_dict is not a FLAVR checkpoint; missing {missing[:3]} ...")
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n in names]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_flavr_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        n_out, eb = C.c_int(), C.c_int()
        check(self._L.vfi_flavr_info(self._ctx, C.byref(n_out), C.byref(eb)))
        self.n_outputs, self.enc_bias = n_out.value, bool(eb.value)
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, frames: torch.Tensor, first: Sequence[int], out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: CUDA float32 [N,H,W,C>=3] NHWC -> CUDA float32 [len(first),H,W,3]: for window k (frames first[k] ..
        first[k] + 3) the model's first output on the padded frames, cropped (not clamped)."""
        assert frames.is_cuda and frames.dtype == torch.float32 and frames.is_contiguous() and frames.dim() == 4
        n, h, w, c = frames.shape
        fa = _i32(first)
        nw = len(fa)
        assert 1 <= nw <= self.MAX_WINDOWS
        if out is None:
            out = torch.empty((nw, h, w, 3), dtype=torch.float32, device=frames.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (nw, h, w, 3)
        st = torch.cuda.current_stream(frames.device).cuda_stream
        check(self._L.vfi_flavr_forward(self._ctx, frames.data_ptr(), n, h, w, c, fa.ctypes.data, nw, out.data_ptr(), st))
        return out

    # ------------------------------------------------------------------ hooks
    def set_ref(self, use_ref: bool):
        check(self._L.vfi_flavr_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_conv(self, layer, src0, src1, out, n_windows, H, W, impl=0, pitch0=None, pitch1=None, out_pitch=None):
        st = torch.cuda.current_stream(src0.device).cuda_stream
        check(self._L.vfi_flavr_debug_conv(
            self._ctx, layer, src0.data_ptr(), int(pitch0 if pitch0 is not None else src0.shape[-1]),
            None if src1 is None else src1.data_ptr(), 0 if src1 is None else int(pitch1 if pitch1 is not None else src1.shape[-1]),
            out.data_ptr(), int(out_pitch if out_pitch is not None else out.shape[-1]), n_windows, H, W, impl, st))
        return out

    def layer_plan(self, layer):
        v = np.zeros(16, np.int32)
        check(self._L.vfi_flavr_layer_plan(self._ctx, layer, v.ctypes.data, 16))
        keys = ("c0", "c1", "n_total", "ksize", "kt", "pad_t", "T_in", "T_out", "pad_y", "pad_x", "n_cta", "nsplit",
                "a_slots", "b_slots", "smem_bytes", "ext")
        return dict(zip(keys, [int(x) for x in v]))

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# IRFNet_S / IRFNet_L.state_dict(): pyramid channels, ResBlock side channels, first conv kernel, decoder4..1 convblock
# channels and ConvT outputs (IFRNet_S_arch.py / IFRNet_L_arch.py)
IFRNET_ARCH = {
    "S": dict(enc=(24, 36, 54, 72), side=24, k0=3, dc=(144, 162, 108, 72), dout=(58, 40, 28, 8)),
    "L": dict(enc=(64, 96, 144, 192), side=64, k0=7, dc=(384, 432, 288, 192), dout=(148, 100, 68, 8)),
}


def ifrnet_state_dict_spec(variant: str):
    """IRFNet_{S,L}.state_dict() names and shapes, in order (104 tensors)."""
    a = IFRNET_ARCH[variant]
    spec, cin = [], 3
    for l, co in enumerate(a["enc"]):
        for j in range(2):
            k = a["k0"] if (l == 0 and j == 0) else 3
            p = f"encoder.pyramid{l + 1}.{j}."
            spec += [(p + "0.weight", (co, cin if j == 0 else co, k, k)), (p + "0.bias", (co,)), (p + "1.weight", (co,))]
        cin = co
    for k in range(4):
        p = f"decoder{4 - k}.convblock."
        C, s = a["dc"][k], a["side"]
        ci = 2 * a["enc"][3] + 1 if k == 0 else a["dout"][k - 1] + 2 * a["enc"][3 - k]
        spec += [(p + "0.0.weight", (C, ci, 3, 3)), (p + "0.0.bias", (C,)), (p + "0.1.weight", (C,))]
        for j in range(1, 5):
            n = s if j in (2, 4) else C
            spec += [(p + f"1.conv{j}.0.weight", (n, n, 3, 3)), (p + f"1.conv{j}.0.bias", (n,)), (p + f"1.conv{j}.1.weight", (n,))]
        spec += [(p + "1.conv5.weight", (C, C, 3, 3)), (p + "1.conv5.bias", (C,)), (p + "1.prelu.weight", (C,))]
        spec += [(p + "2.weight", (C, a["dout"][k], 4, 4)), (p + "2.bias", (a["dout"][k],))]
    return spec


def ifrnet_geometry(h: int, w: int, t: float):
    """The sizes vfi_ifrnet_forward uses for an h x w frame at resize factor t (the reference's arithmetic), as a dict;
    raises VfiError for a t the reference cannot run (an empty encoder input, an output smaller than the frame)."""
    v = np.zeros(22, np.int32)
    check(lib().vfi_ifrnet_geometry(int(h), int(w), float(t), v.ctypes.data, 22))
    keys = ("hp", "wp", "h0", "w0", "h1", "w1", "h2", "w2", "h3", "w3", "h4", "w4", "dh3", "dw3", "dh2", "dw2", "dh1", "dw1",
            "hq", "wq", "hf", "wf")
    return dict(zip(keys, [int(x) for x in v]))


class IfrnetEngine:
    """IFRNet-S / IFRNet-L (IFRNet_{S,L}_{Vimeo90K,GoPro}.pth) on one H100: `state_dict` = IRFNet_S's or IRFNet_L's; the
    variant is read from the shapes and every shape is checked.  fp16 operands with fp32 accumulation ("float32", as the
    node runs it); flows, mask, warps and the blend are fp32."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        first = state_dict.get("encoder.pyramid1.0.0.weight")
        if first is None:
            raise KeyError("state_dict is not an IFRNet checkpoint; missing encoder.pyramid1.0.0.weight")
        variant = "L" if tuple(first.shape[-2:]) == (7, 7) else "S"
        spec = ifrnet_state_dict_spec(variant)
        for name, shape in spec:
            if name not in state_dict:
                raise KeyError(f"state_dict is not an IFRNet-{variant} checkpoint; missing {name}")
            if tuple(state_dict[name].shape) != shape:
                raise ValueError(f"IFRNet-{variant}: {name} has shape {tuple(state_dict[name].shape)}, expected {shape}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n, _ in spec]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_ifrnet_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        v = C.c_int()
        check(self._L.vfi_ifrnet_info(self._ctx, C.byref(v)))
        self.variant = "L" if v.value else "S"
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, img0: torch.Tensor, img1: torch.Tensor, t: float, embt: float,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """img0, img1: CUDA float32 [1, 3, H, W] -> [1, 3, H, W] = model(img0, img1, scale_factor=t, timestep=embt)."""
        for x in (img0, img1):
            assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4 and x.shape[:2] == (1, 3)
        assert img0.shape == img1.shape
        _, _, h, w = img0.shape
        if out is None:
            out = torch.empty((1, 3, h, w), dtype=torch.float32, device=img0.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and out.shape == img0.shape
        st = torch.cuda.current_stream(img0.device).cuda_stream
        check(self._L.vfi_ifrnet_forward(self._ctx, img0.data_ptr(), img1.data_ptr(), h, w, float(t), float(embt),
                                         out.data_ptr(), st))
        return out

    # ------------------------------------------------------------------ hooks
    def set_ref(self, use_ref: bool):
        check(self._L.vfi_ifrnet_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_conv(self, layer, src0, pitch0, src1, pitch1, out, out_pitch, n_images, H, W, impl=0, res=None,
                   out_f32=None, f32_pitch=0):
        """One conv layer on raw tensors (pointers with element offsets already applied by the caller's views)."""
        st = torch.cuda.current_stream(src0.device).cuda_stream
        check(self._L.vfi_ifrnet_debug_conv(
            self._ctx, layer, src0.data_ptr(), int(pitch0), None if src1 is None else src1.data_ptr(), int(pitch1),
            out.data_ptr(), int(out_pitch), None if res is None else res.data_ptr(),
            None if out_f32 is None else out_f32.data_ptr(), int(f32_pitch), n_images, H, W, impl, st))
        return out

    def layer_plan(self, layer):
        v = np.zeros(12, np.int32)
        check(self._L.vfi_ifrnet_layer_plan(self._ctx, layer, v.ctypes.data, 12))
        keys = ("c0", "c1", "n_total", "ksize", "pad_y", "pad_x", "n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes",
                "n_f32")
        return dict(zip(keys, [int(x) for x in v]))

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# CAIN(depth=3).state_dict(): Interpolation(5, 12, 192) - headConv, 5 groups of 12 RCABs (conv1, conv2, CALayer
# 192 -> 12 -> 192) and a tail conv, tailConv (cain_arch.py, common.py)
def cain_state_dict_spec():
    """CAIN(depth=3).state_dict() names and shapes, in order (494 tensors)."""
    C_, R, pre = 192, 12, "encoder.interpolate."
    spec = [(pre + "headConv.weight", (C_, 2 * C_, 3, 3)), (pre + "headConv.bias", (C_,))]
    for g in range(5):
        for r in range(12):
            p = f"{pre}body.{g}.body.{r}.body."
            spec += [(p + "0.conv.weight", (C_, C_, 3, 3)), (p + "0.conv.bias", (C_,)),
                     (p + "2.conv.weight", (C_, C_, 3, 3)), (p + "2.conv.bias", (C_,)),
                     (p + "3.conv_du.0.weight", (R, C_, 1, 1)), (p + "3.conv_du.0.bias", (R,)),
                     (p + "3.conv_du.2.weight", (C_, R, 1, 1)), (p + "3.conv_du.2.bias", (C_,))]
        spec += [(f"{pre}body.{g}.body.12.conv.weight", (C_, C_, 3, 3)), (f"{pre}body.{g}.body.12.conv.bias", (C_,))]
    spec += [(pre + "tailConv.weight", (C_, C_, 3, 3)), (pre + "tailConv.bias", (C_,))]
    return spec


def cain_geometry(h: int, w: int):
    """The sizes vfi_cain_forward uses for an h x w frame: padded size, trunk grid, padding before; raises VfiError for
    a frame the reference's ReflectionPad2d cannot pad."""
    v = np.zeros(6, np.int32)
    check(lib().vfi_cain_geometry(int(h), int(w), v.ctypes.data, 6))
    return dict(zip(("hp", "wp", "gh", "gw", "top", "left"), [int(x) for x in v]))


class CainEngine:
    """CAIN (pretrained_cain.pth, CAIN(depth=3)) on one H100: `state_dict` = CAIN's, without the checkpoint's "module."
    prefix; every name and shape is checked.  fp16 operands with fp32 accumulation ("float32", as the node runs it); the
    means, the attention gates and the output are fp32."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        spec = cain_state_dict_spec()
        for name, shape in spec:
            if name not in state_dict:
                raise KeyError(f"state_dict is not a CAIN checkpoint; missing {name}")
            if tuple(state_dict[name].shape) != shape:
                raise ValueError(f"CAIN: {name} has shape {tuple(state_dict[name].shape)}, expected {shape}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        hold = [state_dict[n].detach().to("cpu", torch.float32).contiguous() for n, _ in spec]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_cain_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, img0: torch.Tensor, img1: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """img0, img1: CUDA float32 [1, 3, H, W] -> [1, 3, H, W] = model(img0, img1)[0] (not clamped)."""
        for x in (img0, img1):
            assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4 and x.shape[:2] == (1, 3)
        assert img0.shape == img1.shape
        _, _, h, w = img0.shape
        if out is None:
            out = torch.empty((1, 3, h, w), dtype=torch.float32, device=img0.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and out.shape == img0.shape
        st = torch.cuda.current_stream(img0.device).cuda_stream
        check(self._L.vfi_cain_forward(self._ctx, img0.data_ptr(), img1.data_ptr(), h, w, out.data_ptr(), st))
        return out

    # ------------------------------------------------------------------ hooks
    def set_ref(self, use_ref: bool):
        check(self._L.vfi_cain_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_conv(self, layer, src0, pitch0, src1, pitch1, out, out_pitch, n_images, H, W, impl=0, res=None):
        """One conv layer on raw 16-bit NHWC tensors (pointers with element offsets already applied)."""
        st = torch.cuda.current_stream(src0.device).cuda_stream
        check(self._L.vfi_cain_debug_conv(
            self._ctx, layer, src0.data_ptr(), int(pitch0), None if src1 is None else src1.data_ptr(), int(pitch1),
            out.data_ptr(), int(out_pitch), None if res is None else res.data_ptr(), n_images, H, W, impl, st))
        return out

    def layer_plan(self, layer):
        v = np.zeros(11, np.int32)
        check(self._L.vfi_cain_layer_plan(self._ctx, layer, v.ctypes.data, 11))
        keys = ("c0", "c1", "n_total", "ksize", "act", "ext", "n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes")
        return dict(zip(keys, [int(x) for x in v]))

    def debug_elem(self, kernel, H, W, img0=None, img1=None, x=None, res=None, out=None, rcab=0):
        """One element-wise stage for an H x W frame (vfi_cain_debug_elem): 0 prep, 1 reflected border, 2 zero border
        + res, 3 channel attention of RCAB `rcab`, 4 final."""
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        st = torch.cuda.current_stream(self.device).cuda_stream
        check(self._L.vfi_cain_debug_elem(self._ctx, kernel, p(img0), p(img1), H, W, p(x), p(res), p(out), rcab, st))
        return out

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))


# IFUNetModel().state_dict(): the flow net (FeatureNet UNet with CBAM, three IFBlocks), the RRDBNet fusion net and the
# ResynNet refinement net, the unused DegCNN included (IFUNet_arch.py)
def ifunet_state_dict_spec():
    """IFUNetModel().state_dict() names and shapes, in order (608 tensors; num_batches_tracked are int64 scalars)."""
    def conv_prelu(p, co, ci, k):
        return [(p + "0.weight", (co, ci, k, k)), (p + "0.bias", (co,)), (p + "1.weight", (co,))]

    def bn(p, c):
        return [(p + n, (c,)) for n in ("weight", "bias", "running_mean", "running_var")] + [(p + "num_batches_tracked", ())]

    def cbam(p, c):
        return ([(p + "ChannelGate.mlp.1.weight", (c // 16, c)), (p + "ChannelGate.mlp.1.bias", (c // 16,)),
                 (p + "ChannelGate.mlp.3.weight", (c, c // 16)), (p + "ChannelGate.mlp.3.bias", (c,)),
                 (p + "SpatialGate.spatial.conv.weight", (1, 2, 7, 7))] + bn(p + "SpatialGate.spatial.bn.", 1))

    def conv_bn(p, co, ci):
        return [(p + "0.weight", (co, ci, 3, 3))] + bn(p + "1.", co) + [(p + "2.weight", (co,))]

    f = "flownet.fmap."
    s = conv_prelu(f + "conv0.", 17, 7, 1)
    cin = 17
    for i, co in enumerate((32, 64, 128, 256, 512)):
        s += conv_prelu(f"{f}conv{i + 1}.conv1.", co, cin, 3) + conv_prelu(f"{f}conv{i + 1}.conv2.", co, co, 3)
        s += cbam(f"{f}conv{i + 1}.cbam.", co) if i else []
        cin = co
    for lvl, ci, co in ((5, 512, 256), (4, 256, 128), (3, 128, 64)):
        p = f"{f}deconv{lvl}."
        s += [(p + "deconv.0.weight", (ci, ci // 2, 4, 4)), (p + "deconv.0.bias", (ci // 2,)),
              (p + "deconv.1.weight", (ci // 2,))]
        s += conv_prelu(p + "conv1.", ci // 2, ci, 3) + conv_prelu(p + "conv2.", co, ci // 2, 3)
        s += cbam(p + "cbam.", co) if lvl == 5 else []
    for b, c in enumerate((256, 128, 64)):
        p = f"flownet.block{b}."
        for j in range(6):
            s += conv_prelu(f"{p}convblock.{j}.", c, c, 3)
        s += [(p + "flowconv.weight", (4, c, 3, 3)), (p + "flowconv.bias", (4,))]
        for L in (16, 8, 4):
            s += [(f"{p}maskconvx{L}.weight", (L * L * 9, c, 1, 1)), (f"{p}maskconvx{L}.bias", (L * L * 9,))]
    p = "fusionnet."
    s += [(p + "conv_first.weight", (64, 16, 3, 3)), (p + "conv_first.bias", (64,))]
    for r in range(6):
        for d in range(1, 4):
            q = f"{p}body.{r}.rdb{d}."
            for k in range(1, 5):
                s += [(f"{q}conv{k}.weight", (32, 32 + 32 * k, 3, 3)), (f"{q}conv{k}.bias", (32,))]
            s += [(q + "conv5.weight", (64, 192, 3, 3)), (q + "conv5.bias", (64,))]
    for n in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
        s += [(f"{p}{n}.weight", (64, 64, 3, 3)), (f"{p}{n}.bias", (64,))]
    s += [(p + "conv_last.weight", (1, 64, 3, 3)), (p + "conv_last.bias", (1,))]
    for b, ci in enumerate((6, 12, 12)):
        p = f"refinenet.block{b}."
        s += conv_bn(p + "conv0.0.", 64, ci) + conv_bn(p + "conv0.1.", 128, 64) + conv_bn(p + "conv0.2.", 256, 128)
        for j in range(6):
            s += conv_bn(f"{p}convblock.{j}.", 256, 256)
        s += [(p + "lastconv.weight", (256, 4, 4, 4)), (p + "lastconv.bias", (4,))]
    p = "refinenet.degrad."
    s += conv_prelu(p + "conv0.", 32, 3, 3)
    for j in (1, 2, 3):
        s += conv_prelu(f"{p}conv{j}.", 32, 32, 3)
    s += [(p + "deconv.1.weight", (128, 32, 4, 4)), (p + "deconv.1.bias", (32,)), (p + "deconv.2.weight", (32,)),
          (p + "deconv.3.weight", (3, 32, 3, 3)), (p + "deconv.3.bias", (3,))]
    for c in (0, 1):
        s += conv_prelu(f"refinenet.context{c}.0.", 16, 3, 3) + conv_prelu(f"refinenet.context{c}.1.", 32, 16, 3)
    s += [("refinenet.decode.0.weight", (64, 32, 4, 4)), ("refinenet.decode.0.bias", (32,)),
          ("refinenet.decode.1.weight", (32, 3, 4, 4)), ("refinenet.decode.1.bias", (3,))]
    return s


def ifunet_geometry(h: int, w: int, scale: float):
    """The sizes vfi_ifunet_forward uses for an h x w frame at `scale`: the padded size and the flow net's input and its
    five stride-2 levels; raises VfiError (a RuntimeError) where the reference raises."""
    v = np.zeros(14, np.int32)
    check(lib().vfi_ifunet_geometry(int(h), int(w), float(scale), v.ctypes.data, 14))
    return dict(hp=int(v[0]), wp=int(v[1]), levels=[(int(v[2 + 2 * i]), int(v[3 + 2 * i])) for i in range(6)])


class IfunetEngine:
    """IFUnet (IFUNet.pth, IFUNetModel) on one H100: `state_dict` = the raw checkpoint; a missing or extra key and every
    shape are refused, as the reference's strict load_state_dict refuses them.  fp16 operands with fp32 accumulation
    ("float32", as the node runs it); flows, masks, gates and the output are fp32."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, dtype: str = "float32"):
        if not torch.cuda.is_available():
            raise VfiError("no CUDA device: this path has no CPU fallback")
        if dtype not in OPERAND:
            raise ValueError(f"dtype must be one of {list(OPERAND)}")
        spec = ifunet_state_dict_spec()
        names = {n for n, _ in spec}
        extra = [k for k in state_dict if k not in names]
        if extra:
            raise KeyError(f"state_dict is not an IFUNet checkpoint; unexpected key {extra[0]}")
        for name, shape in spec:
            if name not in state_dict:
                raise KeyError(f"state_dict is not an IFUNet checkpoint; missing {name}")
            if tuple(state_dict[name].shape) != shape:
                raise ValueError(f"IFUNet: {name} has shape {tuple(state_dict[name].shape)}, expected {shape}")
        self._L = lib()
        self.device = int(device)
        self._ctx = C.c_void_p()
        check(self._L.vfi_create(self.device, C.byref(self._ctx)))
        hold = [state_dict[n].detach().to("cpu", torch.float32).reshape(-1).contiguous() for n, _ in spec]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        check(self._L.vfi_ifunet_load(self._ctx, ptrs, numel, len(hold), OPERAND[dtype]))
        self.dtype = dtype

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self._L.vfi_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, img0: torch.Tensor, img1: torch.Tensor, timestep: float = 0.5, scale: float = 1.0,
                ensemble: bool = True, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """img0, img1: CUDA float32 [1, 3, H, W] -> [1, 3, H, W] = model(img0, img1, timestep=timestep, scale=scale,
        ensemble=ensemble).  Raises VfiError (a RuntimeError) before any launch where the reference raises."""
        for x in (img0, img1):
            assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4 and x.shape[:2] == (1, 3)
        assert img0.shape == img1.shape
        _, _, h, w = img0.shape
        if out is None:
            out = torch.empty((1, 3, h, w), dtype=torch.float32, device=img0.device)
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and out.shape == img0.shape
        st = torch.cuda.current_stream(img0.device).cuda_stream
        check(self._L.vfi_ifunet_forward(self._ctx, img0.data_ptr(), img1.data_ptr(), h, w, float(timestep), float(scale),
                                         1 if ensemble else 0, out.data_ptr(), st))
        return out

    # ------------------------------------------------------------------ hooks
    def set_ref(self, use_ref: bool):
        check(self._L.vfi_ifunet_debug_set_ref(self._ctx, 1 if use_ref else 0))

    def debug_conv(self, layer, src0, pitch0, src1, pitch1, out, out_pitch, B, H, W, impl=0, res=None, out_f32=None,
                   f32_pitch=0):
        """One conv layer on raw 16-bit NHWC tensors (pointers with element offsets already applied)."""
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        st = torch.cuda.current_stream(src0.device).cuda_stream
        check(self._L.vfi_ifunet_debug_conv(self._ctx, layer, p(src0), int(pitch0), p(src1), int(pitch1), p(out),
                                            int(out_pitch), p(res), p(out_f32), int(f32_pitch), B, H, W, impl, st))
        return out

    def layer_plan(self, layer):
        v = np.zeros(14, np.int32)
        check(self._L.vfi_ifunet_layer_plan(self._ctx, layer, v.ctypes.data, 14))
        keys = ("c0", "c1", "n_total", "ksize", "act", "ext", "n_f32", "pad_before", "pad_before_x", "n_cta", "nsplit",
                "a_slots", "b_slots", "smem_bytes")
        return dict(zip(keys, [int(x) for x in v]))

    def debug_elem(self, kernel, H, W, img0=None, img1=None, x=None, y=None, out=None, index=0, timestep=0.5,
                   scale=1.0):
        """One element-wise stage (vfi_ifunet_debug_elem): 0 the level-0 input of `index` images, 1 CBAM `index` in
        place on out, 2 the convex upsampling of IFBlock `index`, 3 the warps of a pair."""
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        st = torch.cuda.current_stream(self.device).cuda_stream
        check(self._L.vfi_ifunet_debug_elem(self._ctx, kernel, p(img0), p(img1), H, W, float(timestep), float(scale),
                                            p(x), p(y), p(out), index, st))
        return out

    def launch_count(self) -> int:
        return int(self._L.vfi_launch_count(self._ctx))

    def sync(self):
        check(self._L.vfi_sync(self._ctx))
