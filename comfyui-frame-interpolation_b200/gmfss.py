"""GMFSS Fortuna on H100 - SURVEY.md section 8 row a11 / BASELINE.json configs[3].

Host schedule of `vfi_models/gmfss_fortuna/GMFSS_Fortuna_union_arch.py`: `Model.reuse` :1726-1782 (GMFlow in both directions
on the half-size frames, MetricNet, FeatureNet) and `Model.inference` :1784-1857 (eight soft splats, the RIFE 4.6 sub-model,
GridNet), with the padding wrapper of `CommonModelInference.forward` (gmfss_fortuna/__init__.py:41-77).  Every tensor
operation is a kernel of libvfi_b200.so: the fp32 building blocks of csrc/gmops.cu (vfi_gm_*), the fused soft splat
(vfi_softsplat_weighted) and the RIFE engine (vfi_rife46_forward); PyTorch only owns the device memory and the stream.
There is no PyTorch / CPU fallback on the product path.  (tests/ run this same schedule on CPU tensors against a host build
of gmops.cu - `Ops(lib=<emulation library>)` - with the oracle standing in for the two components that have their own GPU
tests, the splat and the RIFE engine.)

The same class serves the base model, `GMFSS_Fortuna_arch.py` (the `GMFSS_fortuna` checkpoint), chosen by the weights: a set
without `ifnet` is the base model.  It has no RIFE sub-model, and GridNet's first head (`residual_model_head`, 12 input
channels) reads `[h0, splat(h0), splat(h1), h1]` instead of `[splat(h0), rife, splat(h1)]` (base :1843-1848).

Tensors are NCHW float32 like the reference's; weights are the reference's state_dicts, used in place.
"""
import ctypes as C
import math
from typing import Dict, Optional

import torch


class Ops:
    """Thin typed wrappers around the vfi_gm_* entry points on torch tensors (device memory + current stream)."""

    def __init__(self, lib, device: torch.device):
        self.L = lib
        self.dev = device
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float
        sig = {
            "vfi_gm_conv2d": [vp] * 6 + [i32] * 13 + [f32, i32, f32, vp],
            "vfi_gm_conv2d_packed": [vp] * 6 + [i32] * 14 + [f32, i32, f32, vp],
            "vfi_gm_transpose": [vp, vp, i32, i32, i32, vp],
            "vfi_gm_convt4": [vp] * 4 + [i32] * 6 + [f32, vp],
            "vfi_gm_instance_norm": [vp, vp, i32, i32, f32, i32, vp],
            "vfi_gm_layer_norm": [vp] * 5 + [i32, i32, f32, vp],
            "vfi_gm_softmax_rows": [vp, i32, i32, vp],
            "vfi_gm_gemm": [i32] + [vp] * 5 + [i32] * 7 + [i64] * 3 + [f32, i32, i32, vp],
            "vfi_gm_window": [vp, vp] + [i32] * 8 + [vp],
            "vfi_gm_nchw_tokens": [vp, vp, i32, i32, i32, i32, vp],
            "vfi_gm_add_position": [vp] + [i32] * 5 + [vp],
            "vfi_gm_local_match": [vp] * 3 + [i32] * 5 + [vp],
            "vfi_gm_local_prop": [vp] * 4 + [i32] * 4 + [vp],
            "vfi_gm_convex_up": [vp] * 3 + [i32] * 4 + [vp],
            "vfi_gm_warp_zeros": [vp] * 3 + [i32] * 4 + [vp],
            "vfi_gm_resize": [vp, vp] + [i32] * 6 + [f32, vp],
            "vfi_gm_metric_input": [vp] * 5 + [i32] * 3 + [vp],
            "vfi_gm_pixel_shuffle2": [vp, vp] + [i32] * 4 + [vp],
            "vfi_gm_axpby": [vp, vp, vp, i64, f32, f32, f32, i32, vp],
            "vfi_gm_copy_slice": [vp, vp] + [i32] * 12 + [vp, vp, vp],
        }
        for name, args in sig.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = i32
        self._err = getattr(lib, "vfi_last_error", None)
        if self._err is not None:
            self._err.restype = C.c_char_p
        self._packed: Dict[int, torch.Tensor] = {}   # conv weight data_ptr -> [Cin*k*k, CoutP] (output channel fastest)
        self._wt: Dict[int, torch.Tensor] = {}       # linear weight data_ptr -> its transpose [K, N]

    # ------------------------------------------------------------------ load-time weight layouts (host side, once)
    def register_conv(self, w: torch.Tensor):
        """the fast conv kernel reads wt[(ci, ky, kx)][co] with co padded to a multiple of 16"""
        cout, cin, k, _ = w.shape
        coutp = (cout + 15) // 16 * 16
        wt = torch.zeros(cin * k * k, coutp, dtype=torch.float32)
        wt[:, :cout] = w.detach().to("cpu", torch.float32).permute(1, 2, 3, 0).reshape(cin * k * k, cout)
        self._packed[w.data_ptr()] = wt.to(self.dev).contiguous()

    def register_linear(self, w: torch.Tensor):
        if w.shape[0] % 8 == 0 and w.shape[1] % 4 == 0:
            self._wt[w.data_ptr()] = w.detach().t().contiguous().to(self.dev)

    # ------------------------------------------------------------------ plumbing
    def _st(self):
        return torch.cuda.current_stream(self.dev).cuda_stream if self.dev.type == "cuda" else None

    def _ck(self, rc, what):
        if rc != 0:
            msg = self._err().decode() if self._err is not None else ""
            raise RuntimeError(f"{what} failed ({rc}): {msg}")

    def new(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.dev)

    @staticmethod
    def _p(t):
        return None if t is None else t.data_ptr()

    def _chk(self, *ts):
        for t in ts:
            if t is not None:
                assert t.dtype == torch.float32 and t.is_contiguous() and t.device.type == self.dev.type, (t.dtype, t.shape, t.device)

    # ------------------------------------------------------------------ ops
    def conv(self, x, w, b=None, stride=1, pad=None, pre=None, post=0, post_slope=0.0, res1=None, res2=None, out=None, out_coff=0,
             in_coff=0, cin=None):
        """conv2d with the PReLU in front (pre = slope tensor / float) and residual adds behind fused; reads channels
        [in_coff, in_coff + cin) of x, writes channels [out_coff, out_coff + Cout) of out."""
        n, ctot, h, wd = x.shape
        cout, cin_w, k, _ = w.shape
        cin = cin_w if cin is None else cin
        assert cin == cin_w
        pad = k // 2 if pad is None else pad
        ho, wo = (h + 2 * pad - k) // stride + 1, (wd + 2 * pad - k) // stride + 1
        if out is None:
            out = self.new(n, cout, ho, wo)
        assert tuple(out.shape[2:]) == (ho, wo) and out.shape[0] == n
        slope = float(pre) if pre is not None else 0.0
        self._chk(x, w, b, res1, res2, out)
        wt = self._packed.get(w.data_ptr())
        if wt is not None and ((k in (1, 3) and stride in (1, 2)) or (k == 7 and stride == 2)):
            self._ck(self.L.vfi_gm_conv2d_packed(self._p(x), self._p(wt), self._p(b), self._p(res1), self._p(res2), self._p(out), n, cin, h,
                                                 wd, cout, wt.shape[1], k, stride, pad, ctot, in_coff, out.shape[1], out_coff,
                                                 1 if pre is not None else 0, slope, post, float(post_slope), self._st()), "conv2d_packed")
            return out
        self._ck(self.L.vfi_gm_conv2d(self._p(x), self._p(w), self._p(b), self._p(res1), self._p(res2), self._p(out), n, cin, h, wd, cout,
                                      k, stride, pad, ctot, in_coff, out.shape[1], out_coff, 1 if pre is not None else 0, slope, post,
                                      float(post_slope), self._st()), "conv2d")
        return out

    def convt4(self, x, w, b, pre=None):
        n, cin, h, wd = x.shape
        cout = w.shape[1]
        out = self.new(n, cout, 2 * h, 2 * wd)
        self._chk(x, w, b, out)
        self._ck(self.L.vfi_gm_convt4(self._p(x), self._p(w), self._p(b), self._p(out), n, cin, h, wd, cout, 1 if pre is not None else 0,
                                      float(pre) if pre is not None else 0.0, self._st()), "convt4")
        return out

    def inorm(self, x, relu=False):
        n, c, h, w = x.shape
        out = self.new(n, c, h, w)
        self._chk(x)
        self._ck(self.L.vfi_gm_instance_norm(self._p(x), self._p(out), n * c, h * w, 1e-5, 1 if relu else 0, self._st()), "instance_norm")
        return out

    def layer_norm(self, x, g, b, src=None):
        rows, c = x.numel() // x.shape[-1], x.shape[-1]
        out = torch.empty_like(x)
        self._chk(x, g, b, src)
        self._ck(self.L.vfi_gm_layer_norm(self._p(x), self._p(g), self._p(b), self._p(src), self._p(out), rows, c, 1e-5, self._st()), "layer_norm")
        return out

    def softmax_(self, x):
        rows, l = x.numel() // x.shape[-1], x.shape[-1]
        self._chk(x)
        self._ck(self.L.vfi_gm_softmax_rows(self._p(x), rows, l, self._st()), "softmax_rows")
        return x

    def linear(self, x, w, b=None, act=0):
        """x [..., K] @ w[N, K]^T (+ b) -> [..., N]"""
        k = x.shape[-1]
        m = x.numel() // k
        n = w.shape[0]
        out = self.new(*x.shape[:-1], n)
        self._chk(x, w, b)
        wt = self._wt.get(w.data_ptr())
        if wt is not None:   # x @ wt, the 8 x 8-tile kernel
            self._ck(self.L.vfi_gm_gemm(0, self._p(x), self._p(wt), self._p(b), None, self._p(out), 1, m, n, k, k, n, n, 0, 0, 0, 1.0, 1, act,
                                        self._st()), "gemm")
            return out
        self._ck(self.L.vfi_gm_gemm(1, self._p(x), self._p(w), self._p(b), None, self._p(out), 1, m, n, k, k, k, n, 0, 0, 0, 1.0, 1, act,
                                    self._st()), "gemm")
        return out

    def transpose(self, x):
        """[nb, R, C] -> [nb, C, R]"""
        nb, r, c = x.shape
        out = self.new(nb, c, r)
        self._chk(x)
        self._ck(self.L.vfi_gm_transpose(self._p(x), self._p(out), nb, r, c, self._st()), "transpose")
        return out

    def scores(self, q, k, alpha, mask=None):
        """alpha * q k^T (+ mask): [nb, L, C] x [nb, Lk, C] -> [nb, L, Lk]; the keys are transposed once so that the product
        runs in the coalesced 8 x 8-tile form"""
        if k.shape[1] % 8 == 0 and k.shape[2] % 4 == 0:
            return self.bmm(q, self.transpose(k), False, alpha, mask)
        return self.bmm(q, k, True, alpha, mask)

    def bmm(self, a, b, bt, alpha=1.0, mask=None):
        """a [nb, M, K] x (b [nb, N, K] if bt else b [nb, K, N]) * alpha (+ mask[nb % nmask]) -> [nb, M, N]"""
        nb, m, k = a.shape
        n = b.shape[1] if bt else b.shape[2]
        out = self.new(nb, m, n)
        self._chk(a, b, mask)
        self._ck(self.L.vfi_gm_gemm(1 if bt else 0, self._p(a), self._p(b), None, self._p(mask), self._p(out), nb, m, n, k, k,
                                    k if bt else n, n, m * k, b.shape[1] * b.shape[2], m * n, float(alpha),
                                    1 if mask is None else mask.shape[0], 0, self._st()), "gemm")
        return out

    def window(self, x, k, sh, sw, to_windows, b, h, w, c):
        out = self.new(b * k * k, (h // k) * (w // k), c) if to_windows else self.new(b, h * w, c)
        self._chk(x)
        self._ck(self.L.vfi_gm_window(self._p(x), self._p(out), b, h, w, c, k, sh, sw, 1 if to_windows else 0, self._st()), "window")
        return out

    def to_tokens(self, x):
        b, c, h, w = x.shape
        out = self.new(b, h * w, c)
        self._chk(x)
        self._ck(self.L.vfi_gm_nchw_tokens(self._p(x), self._p(out), b, c, h * w, 1, self._st()), "nchw_tokens")
        return out

    def to_nchw(self, t, h, w):
        b, hw, c = t.shape
        out = self.new(b, c, h, w)
        self._chk(t)
        self._ck(self.L.vfi_gm_nchw_tokens(self._p(t), self._p(out), b, c, hw, 0, self._st()), "nchw_tokens")
        return out

    def add_position_(self, x, k):
        b, c, h, w = x.shape
        self._chk(x)
        self._ck(self.L.vfi_gm_add_position(self._p(x), b, c, h, w, k, self._st()), "add_position")
        return x

    def local_match(self, f0, f1, r):
        b, c, h, w = f0.shape
        out = self.new(b, 2, h, w)
        self._chk(f0, f1)
        self._ck(self.L.vfi_gm_local_match(self._p(f0), self._p(f1), self._p(out), b, c, h, w, r, self._st()), "local_match")
        return out

    def local_prop(self, q, k, flow):
        b, _, h, w = flow.shape
        out = self.new(b, 2, h, w)
        self._chk(q, k, flow)
        self._ck(self.L.vfi_gm_local_prop(self._p(q), self._p(k), self._p(flow), self._p(out), b, q.shape[-1], h, w, self._st()), "local_prop")
        return out

    def convex_up(self, mask, flow, f):
        b, _, h, w = flow.shape
        out = self.new(b, 2, h * f, w * f)
        self._chk(mask, flow)
        self._ck(self.L.vfi_gm_convex_up(self._p(mask), self._p(flow), self._p(out), b, h, w, f, self._st()), "convex_up")
        return out

    def warp(self, x, flow):
        b, c, h, w = x.shape
        out = self.new(b, c, h, w)
        self._chk(x, flow)
        self._ck(self.L.vfi_gm_warp_zeros(self._p(x), self._p(flow), self._p(out), b, c, h, w, self._st()), "warp_zeros")
        return out

    def resize(self, x, ho, wo, align=False, mul=1.0):
        b, c, h, w = x.shape
        out = self.new(b, c, ho, wo)
        self._chk(x)
        self._ck(self.L.vfi_gm_resize(self._p(x), self._p(out), b * c, h, w, ho, wo, 1 if align else 0, float(mul), self._st()), "resize")
        return out

    def metric_input(self, i0, i1, f01, f10):
        b, _, h, w = i0.shape
        out = self.new(b, 14, h, w)
        self._chk(i0, i1, f01, f10)
        self._ck(self.L.vfi_gm_metric_input(self._p(i0), self._p(i1), self._p(f01), self._p(f10), self._p(out), b, h, w, self._st()), "metric_input")
        return out

    def pixel_shuffle2(self, x):
        b, c4, h, w = x.shape
        out = self.new(b, c4 // 4, 2 * h, 2 * w)
        self._chk(x)
        self._ck(self.L.vfi_gm_pixel_shuffle2(self._p(x), self._p(out), b, c4 // 4, h, w, self._st()), "pixel_shuffle2")
        return out

    def axpby(self, a, b=None, alpha=1.0, beta=1.0, gamma=0.0, post=0, out=None):
        out = torch.empty_like(a) if out is None else out
        self._chk(a, b, out)
        self._ck(self.L.vfi_gm_axpby(self._p(a), self._p(b), self._p(out), a.numel(), float(alpha), float(beta), float(gamma), post,
                                     self._st()), "axpby")
        return out

    def copy_slice(self, src, dst, c, s_coff=0, d_coff=0, src_nhwc=False, dst_nhwc=False, mean=None, std=None):
        """dst[:, d_coff : d_coff + c] = src[:, s_coff : s_coff + c] (spatially cropped / zero padded to dst's size)"""
        b = src.shape[0]
        hs, ws, sct = (src.shape[1], src.shape[2], src.shape[3]) if src_nhwc else (src.shape[2], src.shape[3], src.shape[1])
        hd, wd, dct = (dst.shape[1], dst.shape[2], dst.shape[3]) if dst_nhwc else (dst.shape[2], dst.shape[3], dst.shape[1])
        self._chk(src, dst, mean, std)
        self._ck(self.L.vfi_gm_copy_slice(self._p(src), self._p(dst), b, c, hs, ws, hd, wd, sct, s_coff, dct, d_coff, 1 if src_nhwc else 0,
                                          1 if dst_nhwc else 0, self._p(mean), self._p(std), self._st()), "copy_slice")
        return dst


def _shift_mask(h: int, w: int, splits: int) -> torch.Tensor:
    """The shifted-window attention mask of generate_shift_window_attn_mask :326-364 ([k*k, L, L] of 0 / -100): a constant of
    the geometry, built once on the host and kept on the device."""
    wh, ww = h // splits, w // splits
    sh, sw = wh // 2, ww // 2
    img = torch.zeros(1, h, w, 1)
    cnt = 0
    for hs in (slice(0, -wh), slice(-wh, -sh), slice(-sh, None)):
        for ws in (slice(0, -ww), slice(-ww, -sw), slice(-sw, None)):
            img[:, hs, ws, :] = cnt
            cnt += 1
    mw = img.view(1, splits, wh, splits, ww, 1).permute(0, 1, 3, 2, 4, 5).reshape(splits * splits, wh * ww)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0).contiguous()


class GMFSS:
    """`sds`: {"flownet", "metricnet", "feat_ext", "fusionnet", "ifnet"} state_dicts of the reference's five sub-networks
    (gmfss_fortuna/__init__.py:27-39 loads them from five checkpoint files) for the union model, the same without "ifnet"
    (four files) for the base model; `self.variant` ("union" / "base") records which.  The base model takes no `rife`."""

    def __init__(self, sds: Dict[str, Dict[str, torch.Tensor]], ops: Ops, splat=None, rife=None):
        self.variant = "union" if "ifnet" in sds else "base"
        self._head = "head0" if self.variant == "union" else "head"
        if f"residual_model_{self._head}.1.weight" not in sds["fusionnet"]:
            raise KeyError(f"GMFSS {self.variant}: fusionnet has no residual_model_{self._head} (GridNet of the other variant?)")
        self.o = ops
        dev = ops.dev
        self.sd = {net: {k: v.detach().to(dev, torch.float32).contiguous() for k, v in sd.items()} for net, sd in sds.items() if net != "ifnet"}
        self.slope = {net: {k: float(v) for k, v in sd.items() if v.numel() == 1 and k.endswith(".weight")} for net, sd in sds.items() if net != "ifnet"}
        for sd in self.sd.values():
            for k_, v_ in sd.items():
                if v_.dim() == 4 and not ("upsample_model" in k_ and k_.endswith(".1.weight")):   # (ConvTranspose weights keep their layout)
                    ops.register_conv(v_)
                elif v_.dim() == 2:
                    ops.register_linear(v_)
        self._mask: Dict = {}
        self.mean = torch.tensor([0.485, 0.456, 0.406], device=dev)
        self.std = torch.tensor([0.229, 0.224, 0.225], device=dev)
        self.splat = splat     # (x, flow, metric) -> soft splat, NCHW fp32
        self.rife = rife       # (half0, half1 NCHW fp32, t) -> merged frame NCHW fp32; union only

    # ------------------------------------------------------------------ GMFlow (:35-1372)
    def _resblock(self, p, x, stride):
        o, sd = self.o, self.sd["flownet"]
        y = o.inorm(o.conv(x, sd[p + ".conv1.weight"], stride=stride), relu=True)
        y = o.inorm(o.conv(y, sd[p + ".conv2.weight"]), relu=True)
        if p + ".downsample.0.weight" in sd:
            x = o.inorm(o.conv(x, sd[p + ".downsample.0.weight"], sd[p + ".downsample.0.bias"], stride=stride, pad=0))
        return o.axpby(x, y, post=1)

    def _encoder(self, x):
        o, sd = self.o, self.sd["flownet"]
        p = "backbone."
        x = o.inorm(o.conv(x, sd[p + "conv1.weight"], stride=2, pad=3), relu=True)
        for layer, stride in (("layer1", 1), ("layer2", 2), ("layer3", 1)):
            x = self._resblock(p + layer + ".0", x, stride)
            x = self._resblock(p + layer + ".1", x, 1)
        x = o.conv(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"], pad=0)
        w = sd[p + "trident_conv.weight"]
        return [o.conv(x, w, stride=2), o.conv(x, w, stride=1)]   # low resolution first

    def _attend(self, q, k, v, h, w, splits, shifted):
        """single-head attention over tokens [B, L, C]; splits > 1: inside (shifted) windows"""
        o = self.o
        b, _, c = q.shape
        scale = 1.0 / math.sqrt(c)
        if splits <= 1:
            return o.bmm(o.softmax_(o.scores(q, k, scale)), v, False)
        sh, sw = ((h // splits) // 2, (w // splits) // 2) if shifted else (0, 0)
        qw, kw, vw = (o.window(t, splits, sh, sw, True, b, h, w, c) for t in (q, k, v))
        mask = None
        if shifted:
            key = (h, w, splits)
            if key not in self._mask:
                self._mask[key] = _shift_mask(h, w, splits).to(o.dev)
            mask = self._mask[key]
        out = o.bmm(o.softmax_(o.scores(qw, kw, scale, mask)), vw, False)
        return o.window(out, splits, sh, sw, False, b, h, w, c)

    def _layer(self, p, source, target, h, w, splits, shifted, ffn):
        o, sd = self.o, self.sd["flownet"]
        q = o.linear(source, sd[p + ".q_proj.weight"])
        k = o.linear(target, sd[p + ".k_proj.weight"])
        v = o.linear(target, sd[p + ".v_proj.weight"])
        msg = self._attend(q, k, v, h, w, splits, shifted)
        msg = o.linear(msg, sd[p + ".merge.weight"])
        if not ffn:
            return o.layer_norm(msg, sd[p + ".norm1.weight"], sd[p + ".norm1.bias"], src=source)
        msg = o.layer_norm(msg, sd[p + ".norm1.weight"], sd[p + ".norm1.bias"])
        cat = torch.empty((*source.shape[:-1], 2 * source.shape[-1]), dtype=torch.float32, device=o.dev)
        # the concatenation [source, msg] as two channel-slice copies (tokens are "NHWC" with H*W = L, 1)
        b, l, c = source.shape
        o.copy_slice(source.view(b, l, 1, c), cat.view(b, l, 1, 2 * c), c, 0, 0, True, True)
        o.copy_slice(msg.view(b, l, 1, c), cat.view(b, l, 1, 2 * c), c, 0, c, True, True)
        hid = o.linear(cat, sd[p + ".mlp.0.weight"], act=1)
        msg = o.linear(hid, sd[p + ".mlp.2.weight"])
        return o.layer_norm(msg, sd[p + ".norm2.weight"], sd[p + ".norm2.bias"], src=source)

    def _transformer(self, f0, f1, splits):
        o = self.o
        b, c, h, w = f0.shape
        both = o.new(2 * b, c, h, w)
        o.copy_slice(f0, both[:b], c)
        o.copy_slice(f1, both[b:], c)
        c0 = o.to_tokens(both)                       # [2b, L, C] = [f0 tokens; f1 tokens]
        swap = o.new(2 * b, c, h, w)
        o.copy_slice(f1, swap[:b], c)
        o.copy_slice(f0, swap[b:], c)
        c1 = o.to_tokens(swap)                       # [f1; f0]
        for i in range(6):
            p = f"transformer.layers.{i}"
            shifted = (i % 2 == 1) and splits > 1
            c0 = self._layer(p + ".self_attn", c0, c0, h, w, splits, shifted, ffn=False)
            c0 = self._layer(p + ".cross_attn_ffn", c0, c1, h, w, splits, shifted, ffn=True)
            c1 = o.new(*c0.shape)                    # the two halves swapped
            l = c0.shape[1]
            o.copy_slice(c0[b:].view(b, l, 1, c), c1[:b].view(b, l, 1, c), c, 0, 0, True, True)
            o.copy_slice(c0[:b].view(b, l, 1, c), c1[b:].view(b, l, 1, c), c, 0, 0, True, True)
        return o.to_nchw(c0[:b].contiguous(), h, w), o.to_nchw(c0[b:].contiguous(), h, w)

    def _grid_tokens(self, b, h, w):
        key = ("grid", b, h, w)
        if key not in self._mask:
            y, x = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            self._mask[key] = torch.stack([x, y], -1).float().view(1, h * w, 2).repeat(b, 1, 1).contiguous().to(self.o.dev)
        return self._mask[key]

    def _global_match(self, f0, f1):
        o = self.o
        b, c, h, w = f0.shape
        grid = self._grid_tokens(b, h, w)                                           # [B, L, 2] (x, y)
        prob = o.softmax_(o.scores(o.to_tokens(f0), o.to_tokens(f1), 1.0 / math.sqrt(c)))
        corr = o.bmm(prob, grid, False)                                             # expected match position
        return o.to_nchw(o.axpby(corr, grid, 1.0, -1.0), h, w)

    def _propagate(self, f0, flow, radius):
        o, sd = self.o, self.sd["flownet"]
        p = "feature_flow_attn."
        b, c, h, w = f0.shape
        x = o.to_tokens(f0)
        q = o.linear(x, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"])
        if radius <= 0:
            k = o.linear(q, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])         # the reference projects the projected query
            prob = o.softmax_(o.scores(q, k, 1.0 / math.sqrt(c)))
            return o.to_nchw(o.bmm(prob, o.to_tokens(flow), False), h, w)
        k = o.linear(x, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])
        return o.local_prop(q, k, flow)

    def gmflow(self, img0, img1):
        """flow img0 -> img1 at the images' resolution (NCHW in [0, 1], sides multiples of 32) - GMFlow.forward :1262-1369"""
        o, sd = self.o, self.sd["flownet"]
        b, _, h, w = img0.shape
        x = o.new(2 * b, 3, h, w)
        o.copy_slice(img0, x[:b], 3, mean=self.mean, std=self.std)
        o.copy_slice(img1, x[b:], 3, mean=self.mean, std=self.std)
        feats = self._encoder(x)
        flow = None
        f0 = None
        for scale, (splits, corr_radius, prop_radius) in enumerate(((2, -1, -1), (8, 4, 1))):
            f0, f1 = feats[scale][:b].contiguous(), feats[scale][b:].contiguous()
            if scale > 0:
                flow = o.resize(flow, 2 * flow.shape[2], 2 * flow.shape[3], align=True, mul=2.0)
                f1 = o.warp(f1, flow)
            o.add_position_(f0, splits)
            o.add_position_(f1, splits)
            f0, f1 = self._transformer(f0, f1, splits)
            pred = self._global_match(f0, f1) if corr_radius == -1 else o.local_match(f0, f1, corr_radius)
            flow = pred if flow is None else o.axpby(flow, pred)
            flow = self._propagate(f0, flow, prop_radius)
        cat = o.new(b, 2 + f0.shape[1], f0.shape[2], f0.shape[3])
        o.copy_slice(flow, cat, 2)
        o.copy_slice(f0, cat, f0.shape[1], 0, 2)
        xm = o.conv(cat, sd["upsampler.0.weight"], sd["upsampler.0.bias"], post=1)
        mask = o.conv(xm, sd["upsampler.2.weight"], sd["upsampler.2.bias"], pad=0)
        return o.convex_up(mask, flow, 4)

    # ------------------------------------------------------------------ MetricNet :1420-1467, FeatureNet :1470-1500
    def metricnet(self, h0, h1, f01, f10):
        o, sd, sl = self.o, self.sd["metricnet"], self.slope["metricnet"]
        feat = o.conv(o.metric_input(h0, h1, f01, f10), sd["metric_in.weight"], sd["metric_in.bias"])
        for k in (1, 2, 3):
            feat = o.conv(feat, sd[f"metric_net{k}.1.weight"], sd[f"metric_net{k}.1.bias"], pre=sl[f"metric_net{k}.0.weight"], res1=feat)
        return o.conv(feat, sd["metric_out.1.weight"], sd["metric_out.1.bias"], pre=sl["metric_out.0.weight"], post=2)   # tanh * 10

    def featurenet(self, x):
        o, sd, sl = self.o, self.sd["feat_ext"], self.slope["feat_ext"]
        outs = []
        for k in (1, 2, 3):
            p = f"block{k}"
            x = o.conv(x, sd[p + ".1.weight"], sd[p + ".1.bias"], stride=2, pre=sl[p + ".0.weight"])
            x = o.conv(x, sd[p + ".3.weight"], sd[p + ".3.bias"], pre=sl[p + ".2.weight"])
            outs.append(x)
        return outs

    # ------------------------------------------------------------------ GridNet :1503-1688
    def _block(self, p, x, kind, res1=None, res2=None):
        """PReLU-conv-PReLU-conv (residual / stride-2 / transposed first conv) + up to two tensors added to the result"""
        o, sd, sl = self.o, self.sd["fusionnet"], self.slope["fusionnet"]
        if kind == "up":
            y = o.convt4(x, sd[p + ".1.weight"], sd[p + ".1.bias"], pre=sl[p + ".0.weight"])
        else:
            y = o.conv(x, sd[p + ".1.weight"], sd[p + ".1.bias"], stride=2 if kind == "down" else 1, pre=sl[p + ".0.weight"])
        return o.conv(y, sd[p + ".3.weight"], sd[p + ".3.bias"], pre=sl[p + ".2.weight"], res1=res1, res2=res2)

    def gridnet(self, x, x1, x2, x3):
        o, sd, sl = self.o, self.sd["fusionnet"], self.slope["fusionnet"]
        r = lambda n, t, a=None, b=None: self._block("residual_model_" + n, t, "res", a, b)        # noqa: E731
        d = lambda n, t, a=None, b=None: self._block("downsample_model_" + n, t, "down", a, b)     # noqa: E731
        u = lambda n, t, a=None, b=None: self._block("upsample_model_" + n, t, "up", a, b)         # noqa: E731
        X00 = r("head1", x1, r(self._head, x))
        X01 = r("01", X00, X00)
        X10 = d("10", X00, r("head2", x2))
        X20 = d("20", X10, r("head3", x3))
        X11 = r("11", X10, X10, d("11", X01))
        X21 = r("21", X20, X20, d("21", X11))
        X24 = r("24", X21, X21)
        X25 = r("25", X24, X24)
        X14 = u("14", X24, r("14", X11, X11))
        X04 = u("04", X14, r("04", X01, X01))
        X15 = u("15", X25, r("15", X14, X14))
        X05 = u("05", X15, r("05", X04, X04))
        t = "residual_model_tail."
        y = o.conv(X05, sd[t + "conv_before_upsample.0.weight"], sd[t + "conv_before_upsample.0.bias"], post=3,
                   post_slope=sl[t + "conv_before_upsample.1.weight"])
        y = o.pixel_shuffle2(o.conv(y, sd[t + "upsample.0.weight"], sd[t + "upsample.0.bias"]))
        return o.conv(y, sd[t + "conv_last.weight"], sd[t + "conv_last.bias"])

    # ------------------------------------------------------------------ Model.reuse / Model.inference
    def reuse(self, img0, img1):
        o = self.o
        b, _, h, w = img0.shape
        h0, h1 = o.resize(img0, h // 2, w // 2), o.resize(img1, h // 2, w // 2)
        f01, f10 = self.gmflow(h0, h1), self.gmflow(h1, h0)
        metric = self.metricnet(h0, h1, f01, f10)
        m0, m1 = o.new(b, 1, h // 2, w // 2), o.new(b, 1, h // 2, w // 2)
        o.copy_slice(metric, m0, 1, 0, 0)
        o.copy_slice(metric, m1, 1, 1, 0)
        return f01, f10, m0, m1, self.featurenet(img0), self.featurenet(img1), h0, h1

    def inference(self, state, timestep: float):
        o = self.o
        f01, f10, m0, m1, fa, fb, h0, h1 = state
        t = float(timestep)
        F1t, F2t = o.axpby(f01, alpha=t), o.axpby(f10, alpha=1.0 - t)
        Z1t, Z2t = o.axpby(m0, alpha=t), o.axpby(m1, alpha=1.0 - t)
        b, _, hh, wh = h0.shape
        if self.variant == "union":   # [I1t, rife, I2t]
            x = o.new(b, 9, hh, wh)
            o.copy_slice(self.splat(h0, F1t, Z1t), x, 3, 0, 0)
            o.copy_slice(self.rife(h0, h1, t), x, 3, 0, 3)
            o.copy_slice(self.splat(h1, F2t, Z2t), x, 3, 0, 6)
        else:                         # base: [img0, I1t, I2t, img1] of the half-size frames
            x = o.new(b, 12, hh, wh)
            o.copy_slice(h0, x, 3, 0, 0)
            o.copy_slice(self.splat(h0, F1t, Z1t), x, 3, 0, 3)
            o.copy_slice(self.splat(h1, F2t, Z2t), x, 3, 0, 6)
            o.copy_slice(h1, x, 3, 0, 9)
        levels = []
        fl1, fl2, z1, z2 = F1t, F2t, Z1t, Z2t
        for lv in range(3):
            if lv > 0:   # flows and metrics of the half / quarter size feature maps: F.interpolate(0.5^lv) * 0.5^lv of the FULL maps
                s = 0.5 ** lv
                hs, ws = int(hh * s), int(wh * s)
                fl1, fl2 = o.resize(F1t, hs, ws, mul=s), o.resize(F2t, hs, ws, mul=s)
                z1, z2 = o.resize(Z1t, hs, ws), o.resize(Z2t, hs, ws)
            c = fa[lv].shape[1]
            cat = o.new(b, 2 * c, fa[lv].shape[2], fa[lv].shape[3])
            o.copy_slice(self.splat(fa[lv], fl1, z1), cat, c, 0, 0)
            o.copy_slice(self.splat(fb[lv], fl2, z2), cat, c, 0, c)
            levels.append(cat)
        out = self.gridnet(x, levels[0], levels[1], levels[2])
        return o.axpby(out, post=2)   # clamp(0, 1)

    def interpolate(self, frame0, frame1, timestep: float):
        """CommonModelInference.forward (gmfss_fortuna/__init__.py:41-77) at scale 1: NCHW frames in [0, 1] of any size ->
        the frame at `timestep`; zero padding to multiples of 64 at the bottom / right, cropped again."""
        o = self.o
        b, _, h, w = frame0.shape
        ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
        i0, i1 = o.new(b, 3, ph, pw), o.new(b, 3, ph, pw)
        o.copy_slice(frame0, i0, 3)
        o.copy_slice(frame1, i1, 3)
        out = self.inference(self.reuse(i0, i1), timestep)
        res = o.new(b, 3, h, w)
        return o.copy_slice(out, res, 3)


def build_gpu_model(sds: Dict[str, Dict[str, torch.Tensor]], device: int = 0) -> GMFSS:
    """The product configuration: gmops + fused soft splat + RIFE engine of libvfi_b200.so on cuda:`device`.  Without
    sds["ifnet"] this is the base model: no RIFE engine (and none of its workspace), `_engine` is None."""
    from . import ops as OPS
    from ._lib import lib
    dev = torch.device("cuda", device)
    o = Ops(lib(), dev)

    def splat(x, flow, metric):
        return OPS.softsplat(x, flow, metric, "soft")

    if "ifnet" not in sds:
        m = GMFSS(sds, o, splat=splat)
        m._engine = None
        return m
    from .engine import Rife46Engine
    eng = Rife46Engine(sds["ifnet"], device=device, dtype="float32", batch=1, arch="4.6")

    def rife(h0, h1, t):
        b, _, h, w = h0.shape
        assert b == 1, "GMFSS runs one pair per call (generic_frame_loop)"
        frames = o.new(2, h, w, 3)
        o.copy_slice(h0, frames[0:1], 3, dst_nhwc=True)
        o.copy_slice(h1, frames[1:2], 3, dst_nhwc=True)
        mid = eng.forward(frames, [0], [1], [float(t)])          # [1, H, W, 3], IFNet 4.6 at scale list [8, 4, 2, 1]
        out = o.new(1, 3, h, w)
        return o.copy_slice(mid, out, 3, src_nhwc=True)

    m = GMFSS(sds, o, splat=splat, rife=rife)
    m._engine = eng
    return m
