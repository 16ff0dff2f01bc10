"""A float64 shadow of the GMFSS schedule: every gmops launch of comfyui-frame-interpolation_b200/gmfss.py checked per element
against the same operation in float64, with an error bound derived beforehand from the kernel's arithmetic.

``ShadowOps`` is ``gmfss.Ops`` with every method wrapped: the inputs are cloned as float64 before the call (the in-place
methods ``softmax_``, ``add_position_`` and ``axpby`` with ``out`` aliasing ``a`` overwrite them), ``super()`` runs unchanged,
and the operation is evaluated again in float64 from the clones with plain torch ops (conv2d, conv_transpose2d, matmul,
grid_sample(align_corners=True), interpolate, softmax) on the inputs' device.  Every call records its method, the kernel
variant the launcher took (``gemm_variant`` / ``conv_variant``, read from the arguments of the C call), the shape and the
worst |got - ref| / bound with its location; a NaN or inf in the output counts as an infinite ratio.  Buffers from
``Ops.new`` start as NaN, so an element a kernel never writes cannot pass.  ``shadow_splat`` does the same for the fused soft
splat (mode "soft", addeps) of ``build_gpu_model``.  Tests: tests/test_gmfss_shadow_host.py (host build of gmops.cu) and
tests/test_gpu_zgmfss_shadow.py (H100).

Bounds.  u = 2^-24.  Scalars the launcher passes as C float (slopes, alpha, mul, axpby coefficients) are rounded to fp32 in
the reference too.  "2 n u S" is ``streamconv_util.worst_ratio``'s form: n roundings each at most u of a partial result
bounded by S, doubled to cover second-order terms.  L is the Lipschitz constant of what follows the rounded value.

    kernel              n, S (and what is added)                                   post
    conv2d / _packed    n = Cin k^2 + 4 (fma chain, PReLU in front, bias, res1,    ReLU L=1; PReLU L=max(1,|a|) + u|y|;
                        res2); S = conv(|pre(x)|, |w|) + |b| + |res1| + |res2|     tanh*10 L=10 + 60 u |y| (tanhf 2 ulp,
                                                                                    the *10)
    convt4              n = 4 Cin + 3; S = convT(|pre(x)|, |w|) + |b|
    gemm (linear, bmm,  n = K + 3 (fma chain, *alpha, bias, mask);                 GELU L=1.2 + u (|v| (4 + |v|) + 2|y|)
    scores)             S = |alpha| sum |a b| + |bias| + |mask|                     (erff 2 ulp, v/sqrt2, products)
    instance_norm,      one block of 128 threads per row of L: m = ceil(L / 128) serial adds per thread + a 7-level tree.
    layer_norm          e_mu = (m + 8) u mean|x|; rho_V = (m + 10) u + e_mu^2 / (V + eps) (relative, variance);
                        |dy| <= 2 [(e_mu + u |x - mu|) r + |y_n| (rho_V / 2 + 4 u)] (r = 1 / sqrt(V + eps), y_n the
                        normalised value); layer_norm: times |gamma|, + 3 u (|y_n gamma| + |beta| + |src|); ReLU L=1
    softmax_rows        |dp_i| <= 2 p_i u (|x_i - max| + m + 12) + 2^-126 (subtraction, expf 2 ulp, the (m + 6)-deep sum,
                        the reciprocal and the product; the constant covers fp32 underflow of tiny terms)
    local_match,        scores: ds_d = (C + 3) u S_d (S_d = |scale| sum |f0 f1|); weights: eps_d = u (|s_d - max| + 4);
    local_prop,         out = sum p_d v_d: |dout| <= 2 [(max ds + max eps) sum p_d |v_d - out| + (T + 3) u sum p_d |v_d|
    convex_up           + u (|x| + |out|)] with T taps and v_d the displaced position (match, x included: the kernel
                        averages absolute positions and subtracts x), the flow (prop) or f * flow (convex_up; ds = 0)
    add_position        |dx| <= 2 u (32 |arg| + 4 + |out|) (fp32 argument: division, powf 4 ulp of 10000^(2j/F) = 9.2 u per
                        unit of exponent rounding, products; sinf / cosf 2 ulp; the add)
    warp_zeros, resize, bilinear at the exact float64 coordinate c; the kernel's fp32 coordinate is within dc (warp: u |c|;
    metric_input        resize: 4 u (|c| + 1)), so |dv| <= 2 [max over the cells of [c - dc, c + dc] of (Dx dc_x + Dy dc_y)
                        + 8 u max|tap|] with Dx, Dy the largest tap differences along x / y of a cell (zero padded for
                        warps, edge-clamped for resize); resize: times |mul|, + u |out|.  metric_input: the photometric
                        channels 2 [(sum_c e_c) / 3 + u sum (|v0| + |s|) + u |out|], the normalised flows 2 u |out|, the
                        images bit-exact; the occlusion flags may differ from float64 only where |d - thr| is within
                        2 (dd + dthr) (dd from the sampled flows' bounds + 3 u d, dthr = 0.01 dmag + 2 u thr); those
                        pixels are counted in ``occ_near``, a flag flipped outside its margin is an infinite ratio
    axpby               n = 3, S = |alpha a| + |beta b| + |gamma|; ReLU / clamp L=1
    copy_slice          with mean / std: 2 u (|v| + |mean|) / |std| x 2; without: bit-exact
    transpose, window, nchw_tokens, pixel_shuffle2: bit-exact
    splat (soft,        per source: w = corner weight at the fp32 coordinate (|dw| <= dc_x + dc_y), e = expf(metric) (4 u),
    addeps)             in e w (8 u in all); per target, n_t contributions summed in any order: (n_t + 1) u sum|terms|;
                        E_N, E_D the numerator / normaliser errors, |dout| <= 2 [(E_N + |out| (E_D + u (D + 1e-7)))
                        / (D + 1e-7) + u |out|]

A kernel that writes outside its output (a channel slice of ``out``) is caught by comparing the rest of ``out`` with its
state before the call, bit for bit.
"""
import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

U = 2.0 ** -24
TINY = 2.0 ** -126
NAN = float("nan")


def f32(v: float) -> float:
    """the value a C float argument carries"""
    return float(torch.tensor(float(v), dtype=torch.float32))


# ----------------------------------------------------------------------------------------------- variant classification
def gemm_variant(bt, a_ptr, b_ptr, nb, M, N, K, lda, ldb, sA, sB) -> str:
    """the kernel gm_gemm (csrc/gmops.cu) launches for these arguments"""
    aligned = ((K | N | lda | ldb) & 3) == 0 and (N & 7) == 0 and ((sA | sB) & 3) == 0 and ((a_ptr | b_ptr) & 15) == 0
    if not bt and aligned:
        cols = nb * (N // 8)
        mt = 8 if cols * ((M + 7) // 8) >= 60000 else (4 if cols * ((M + 3) // 4) >= 60000 else 2)
        return f"nn8<{mt}>"
    return "bt" if bt else "nn"


def conv_variant(name, args) -> str:
    """vfi_gm_conv2d_packed -> packed(k,s); vfi_gm_conv2d -> generic(k,s)"""
    if name == "vfi_gm_conv2d_packed":
        return f"packed({args[12]},{args[13]})"
    return f"generic({args[11]},{args[12]})"


class _Recorder:
    """the library seen through Ops: every vfi_gm_* call is recorded (name, arguments, return code)"""

    def __init__(self, lib, calls):
        self._lib, self._calls = lib, calls

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("vfi_gm_"):
            return fn

        def call(*args):
            rc = fn(*args)
            self._calls.append((name, args, rc))
            return rc
        return call


# ----------------------------------------------------------------------------------------------- ratio bookkeeping
def ratio_of(got, ref, bound):
    """elementwise |got - ref| / bound (0 where both are 0, inf where got is not finite)"""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf)).nan_to_num(nan=math.inf, posinf=math.inf)


def _argmax(r):
    if r.numel() == 0:
        return 0.0, ()
    i = int(torch.argmax(r))
    at = []
    for d in reversed(r.shape):
        at.append(i % d)
        i //= d
    return float(r.flatten()[int(torch.argmax(r))]), tuple(reversed(at))


# ----------------------------------------------------------------------------------------------- float64 building blocks
def _pre(x, slope):
    return x if slope is None else torch.where(x < 0, x * f32(slope), x)


def _cells(img, cx, cy, dcx, dcy, zero):
    """max over the (up to four) bilinear cells the segment [c - dc, c + dc] touches of Dx dc_x + Dy dc_y, and the largest
    |tap|; img [P, H, W], coordinates [P, Ho, Wo] in pixels (float64)"""
    P, H, W = img.shape
    flat = img.reshape(P, H * W)
    lip = torch.zeros_like(cx)
    amax = torch.zeros_like(cx)
    for sx in (-1.0, 1.0):
        for sy in (-1.0, 1.0):
            x0, y0 = torch.floor(cx + sx * dcx), torch.floor(cy + sy * dcy)
            t = []
            for yy, xx in ((y0, x0), (y0, x0 + 1), (y0 + 1, x0), (y0 + 1, x0 + 1)):
                if zero:
                    ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
                else:
                    xx, yy = xx.clamp(0, W - 1), yy.clamp(0, H - 1)
                    ok = None
                idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long().reshape(P, -1)
                v = torch.gather(flat, 1, idx).view_as(cx)
                t.append(v if ok is None else torch.where(ok, v, torch.zeros_like(v)))
            dx = torch.maximum((t[1] - t[0]).abs(), (t[3] - t[2]).abs())
            dy = torch.maximum((t[2] - t[0]).abs(), (t[3] - t[1]).abs())
            lip = torch.maximum(lip, dx * dcx + dy * dcy)
            amax = torch.maximum(amax, torch.stack([v.abs() for v in t]).amax(0))
    return lip, amax


def _grid_sample_px(img, cx, cy):
    """bilinear, zero padding, at pixel coordinates (grid_sample with align_corners=True): img [B, C, H, W], c [B, Ho, Wo]"""
    _, _, H, W = img.shape
    g = torch.stack([2 * cx / (W - 1) - 1, 2 * cy / (H - 1) - 1], -1)
    return F.grid_sample(img, g, mode="bilinear", padding_mode="zeros", align_corners=True)


def _warp_bound(img, cx, cy):
    """per-element bound of a zero-padded bilinear sample at the fp32 coordinate x + f (|dc| <= u |c|): [B, C, Ho, Wo]"""
    B, Cc, H, W = img.shape
    dcx, dcy = U * cx.abs(), U * cy.abs()
    e = lambda t: t[:, None].expand(B, Cc, *t.shape[1:]).reshape(B * Cc, *t.shape[1:])   # noqa: E731
    lip, amax = _cells(img.reshape(B * Cc, H, W), e(cx), e(cy), e(dcx), e(dcy), True)
    return (lip + 8 * U * amax).view(B, Cc, *cx.shape[1:])


def _window_split(t, b, h, w, c, k, sh, sw):
    """tokens [b, h*w, c] -> windows [b*k*k, (h/k)*(w/k), c] of the grid rolled by (-sh, -sw)"""
    g = torch.roll(t.view(b, h, w, c), shifts=(-sh, -sw), dims=(1, 2))
    return g.view(b, k, h // k, k, w // k, c).permute(0, 1, 3, 2, 4, 5).reshape(b * k * k, (h // k) * (w // k), c)


def _window_merge(t, b, h, w, c, k, sh, sw):
    g = t.view(b, k, k, h // k, w // k, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h, w, c)
    return torch.roll(g, shifts=(sh, sw), dims=(1, 2)).reshape(b, h * w, c)


def _softavg_bound(s, ds, v, out, taps, extra):
    """softmax-weighted average over the last dim: scores s [.., T] (float64, -inf for excluded taps), per-tap score error
    ds, values v [.., T]; out [..] the float64 result; extra the absolute terms added"""
    p = torch.softmax(s, -1)
    mx = s.amax(-1, keepdim=True)
    eps = U * ((s - mx).abs().nan_to_num(posinf=0.0) + 4)
    eps = torch.where(p > 0, eps, torch.zeros_like(eps))
    spread = (p * (v - out[..., None]).abs()).sum(-1)
    return 2 * ((ds.amax(-1) + eps.amax(-1)) * spread + (taps + 3) * U * (p * v.abs()).sum(-1) + extra)



def ref_position(shape, k, dev):
    """PositionEmbeddingSine (normalised, temperature 10000) inside each of the k x k windows, float64: (pos [1, C, H, W],
    its sine / cosine argument)"""
    b, c, h, w = shape
    hh, ww, Fh = h // k, w // k, c // 2
    iy = (torch.arange(h, device=dev, dtype=torch.float64) % hh + 1) / (hh + 1e-6) * (2 * math.pi)
    ix = (torch.arange(w, device=dev, dtype=torch.float64) % ww + 1) / (ww + 1e-6) * (2 * math.pi)
    f = torch.arange(Fh, device=dev, dtype=torch.float64)
    dim_t = 10000.0 ** (2 * torch.div(f, 2, rounding_mode="floor") / Fh)
    ay = (iy.view(1, h, 1) / dim_t.view(-1, 1, 1)).expand(Fh, h, w)
    ax = (ix.view(1, 1, w) / dim_t.view(-1, 1, 1)).expand(Fh, h, w)
    odd = (torch.arange(Fh, device=dev) % 2 == 1).view(-1, 1, 1)
    py = torch.where(odd, torch.cos(ay), torch.sin(ay))
    px = torch.where(odd, torch.cos(ax), torch.sin(ax))
    return torch.cat([py, px], 0)[None], torch.cat([ay, ax], 0)[None]


def ref_local_match(A, B_, r):
    """radius-r local correlation softmax in float64 (f0, f1 NCHW): [(flow x, bound), (flow y, bound)]"""
    b, c, h, w = A.shape
    ks = 2 * r + 1
    sc = 1.0 / math.sqrt(c)
    Bp = F.pad(B_, (r, r, r, r))
    okp = F.pad(torch.ones(1, 1, h, w, dtype=torch.float64, device=A.device), (r, r, r, r))
    s, S, ok, px, py = [], [], [], [], []
    xs = torch.arange(w, device=A.device, dtype=torch.float64).view(1, 1, w)
    ys = torch.arange(h, device=A.device, dtype=torch.float64).view(1, h, 1)
    for d in range(ks * ks):                       # x fastest, like the reference's window
        dy, dx = d // ks - r, d % ks - r
        g = Bp[:, :, r + dy:r + dy + h, r + dx:r + dx + w]
        s.append((A * g).sum(1) * sc)
        S.append((A * g).abs().sum(1) * sc)
        ok.append(okp[:, 0, r + dy:r + dy + h, r + dx:r + dx + w].expand(b, h, w) > 0)
        px.append((xs + dx).expand(b, h, w))
        py.append((ys + dy).expand(b, h, w))
    s, S, ok = torch.stack(s, -1), torch.stack(S, -1), torch.stack(ok, -1)
    s = torch.where(ok, s, torch.full_like(s, -math.inf))
    ds = torch.where(ok, (c + 3) * U * S, torch.zeros_like(S))
    p = torch.softmax(s, -1)
    res = []
    for pos, base in ((px, xs.expand(b, h, w)), (py, ys.expand(b, h, w))):
        v = torch.stack(pos, -1)
        o_abs = (p * v).sum(-1)
        res.append((o_abs - base, _softavg_bound(s, ds, v, o_abs, ks * ks, U * (base.abs() + o_abs.abs()))))
    return res


def ref_local_prop(Q, K_, Fl):
    """radius-1 flow propagation in float64: q, k tokens [B, H*W, C], flow NCHW (zero padded keys and flow)"""
    b, _, h, w = Fl.shape
    c = Q.shape[-1]
    sc = 1.0 / math.sqrt(c)
    Qn = Q.view(b, h, w, c)
    Kp = F.pad(K_.view(b, h, w, c).permute(0, 3, 1, 2), (1, 1, 1, 1))
    Fp = F.pad(Fl, (1, 1, 1, 1))
    s, S, v = [], [], []
    for d in range(9):
        dy, dx = d // 3 - 1, d % 3 - 1
        kk = Kp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w].permute(0, 2, 3, 1)
        s.append((Qn * kk).sum(-1) * sc)
        S.append((Qn * kk).abs().sum(-1) * sc)
        v.append(Fp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w])
    s, S, v = torch.stack(s, -1), torch.stack(S, -1), torch.stack(v, -1)   # v [b, 2, h, w, 9]
    ds = (c + 3) * U * S
    p = torch.softmax(s, -1)
    res = []
    for comp in (0, 1):
        o = (p * v[:, comp]).sum(-1)
        res.append((o, _softavg_bound(s, ds, v[:, comp], o, 9, U * o.abs())))
    return res


def ref_convex_up(Mk, Fl, f):
    """convex up-sampling by f in float64: mask [B, 9 f f, H, W] (raw), flow [B, 2, H, W]"""
    b, _, h, w = Fl.shape
    m = Mk.view(b, 9, f, f, h, w).permute(0, 4, 2, 5, 3, 1).reshape(b, h * f, w * f, 9)   # [b, y f + fy, x f + fx, t]
    Fp = F.pad(f * Fl, (1, 1, 1, 1))
    v = torch.stack([Fp[:, :, t // 3:t // 3 + h, t % 3:t % 3 + w] for t in range(9)], -1)
    v = v.repeat_interleave(f, 2).repeat_interleave(f, 3)                                   # [b, 2, h f, w f, 9]
    p = torch.softmax(m, -1)
    res = []
    for comp in (0, 1):
        o = (p * v[:, comp]).sum(-1)
        res.append((o, _softavg_bound(m, torch.zeros_like(m), v[:, comp], o, 9, U * o.abs())))
    return res


def ref_warp(X, Fl):
    """x sampled at pixel + flow, bilinear with zero padding, float64: (value, bound)"""
    b, c, h, w = X.shape
    cx = torch.arange(w, device=X.device, dtype=torch.float64).view(1, 1, w) + Fl[:, 0]
    cy = torch.arange(h, device=X.device, dtype=torch.float64).view(1, h, 1) + Fl[:, 1]
    return _grid_sample_px(X, cx, cy), _warp_bound(X, cx, cy)


def ref_fb_margins(A, Cf):
    """forward-backward consistency in float64: per direction (d - thr, allowed |d - thr| for a flag that differs)"""
    wb, ewb = ref_warp(Cf, A)
    wf, ewf = ref_warp(A, Cf)
    mag = A.norm(dim=1) + Cf.norm(dim=1)
    thr = 0.01 * mag + 0.5
    dthr = 0.01 * 4 * U * mag + 2 * U * thr
    out = []
    for fw, ww_, ew in ((A, wb, ewb), (Cf, wf, ewf)):
        z = fw + ww_
        dval = z.norm(dim=1)
        dd = (ew + U * z.abs()).sum(1) + 3 * U * dval
        out.append((dval - thr, 2 * (dd + dthr)))
    return out


# ----------------------------------------------------------------------------------------------- the shadow
class ShadowStats:
    def __init__(self):
        self.rows: Dict[Tuple[str, str], dict] = {}
        self.occ_near = 0
        self.occ_flips = 0
        self.occ_pixels = 0
        self.seen = set()      # (method, variant, shape) of every call

    def add(self, method, variant, shape, r, at):
        row = self.rows.setdefault((method, variant), dict(calls=0, worst=0.0, shape=None, at=()))
        row["calls"] += 1
        self.seen.add((method, variant, tuple(shape)))
        if r > row["worst"] or row["shape"] is None:
            row.update(worst=r, shape=tuple(shape), at=at)

    def worst(self):
        return max((v["worst"] for v in self.rows.values()), default=0.0)

    def lines(self, tag=""):
        out = []
        for (m, v), row in sorted(self.rows.items()):
            out.append(f"{tag}{m:14s} {v:14s} calls {row['calls']:5d}  worst {row['worst']:.3e}  at {row['at']} of {row['shape']}")
        if self.occ_pixels:
            out.append(f"{tag}metric_input occlusion flags: {self.occ_near} of {self.occ_pixels} pixels within their margin, "
                       f"{self.occ_flips} differ from float64")
        return out

    def failures(self):
        return [f"{m}/{v}: {row['worst']:.3e} at {row['at']} of {row['shape']}" for (m, v), row in sorted(self.rows.items())
                if not row["worst"] <= 1.0]

    def variants(self, method):
        return {v for (m, v) in self.rows if m == method}


def _d(t):
    return None if t is None else t.detach().double().clone()


def make_shadow_class(Ops):
    """ShadowOps: the subclass of the product's Ops (``shadow_class()`` imports it; ``shadow(ops)`` converts an instance)"""
    class Shadow(Ops):
        def _shadow_init(self):
            self.stats = ShadowStats()
            self.calls: List = []
            self.L = _Recorder(self.L, self.calls)

        def __init__(self, lib, device):
            super().__init__(lib, device)
            self._shadow_init()

        # ---------------------------------------------------------------- plumbing
        def new(self, *shape):
            return super().new(*shape).fill_(NAN)

        def _last(self, name):
            n, a, rc = self.calls[-1]
            assert n == name, (n, name)
            return a

        def _rec(self, method, variant, got, ref, bound):
            r = ratio_of(got, ref, bound)
            w, at = _argmax(r)
            self.stats.add(method, variant, got.shape, w, at)
            return w

        def _untouched(self, method, variant, before, after, keep):
            """elements of `after` outside the written region (keep == True) equal `before` bit for bit"""
            same = (before == after) | (torch.isnan(before) & torch.isnan(after))
            bad = keep & ~same
            if bool(bad.any()):
                self.stats.add(method, variant + "/guard", after.shape, math.inf, tuple(int(i) for i in bad.nonzero()[0]))

        # ---------------------------------------------------------------- convolutions
        def conv(self, x, w, b=None, stride=1, pad=None, pre=None, post=0, post_slope=0.0, res1=None, res2=None, out=None,
                 out_coff=0, in_coff=0, cin=None):
            cin_ = w.shape[1] if cin is None else cin
            k = w.shape[2]
            pd = k // 2 if pad is None else pad
            X = _d(x)[:, in_coff:in_coff + cin_]
            W_, B_, R1, R2 = _d(w), _d(b), _d(res1), _d(res2)
            before = None if out is None else out.detach().clone()
            y = super().conv(x, w, b, stride, pad, pre, post, post_slope, res1, res2, out, out_coff, in_coff, cin)
            name, args, _ = self.calls[-1]
            variant = conv_variant(name, args)
            xp = _pre(X, pre)
            ref = F.conv2d(xp, W_, B_, stride=stride, padding=pd)
            S = F.conv2d(xp.abs(), W_.abs(), None, stride=stride, padding=pd)
            if B_ is not None:
                S = S + B_.abs().view(1, -1, 1, 1)
            for r_ in (R1, R2):
                if r_ is not None:
                    ref, S = ref + r_, S + r_.abs()
            n = cin_ * k * k + 4
            L, extra = 1.0, 0.0
            if post == 1:
                ref = ref.clamp(min=0)
            elif post == 2:
                ref = torch.tanh(ref) * 10
                L, extra = 10.0, 60 * U * ref.abs()
            elif post == 3:
                a = f32(post_slope)
                ref = torch.where(ref < 0, ref * a, ref)
                L, extra = max(1.0, abs(a)), U * ref.abs()
            cout = w.shape[0]
            got = y[:, out_coff:out_coff + cout]
            self._rec("conv", variant, got, ref, 2 * n * U * S * L + extra)
            if before is not None:
                keep = torch.ones_like(before, dtype=torch.bool)
                keep[:, out_coff:out_coff + cout] = False
                self._untouched("conv", variant, before, y, keep)
            return y

        def convt4(self, x, w, b, pre=None):
            X, W_, B_ = _d(x), _d(w), _d(b)
            y = super().convt4(x, w, b, pre)
            xp = _pre(X, pre)
            ref = F.conv_transpose2d(xp, W_, B_, stride=2, padding=1)
            S = F.conv_transpose2d(xp.abs(), W_.abs(), B_.abs(), stride=2, padding=1)
            self._rec("convt4", "-", y, ref, 2 * (4 * x.shape[1] + 3) * U * S)
            return y

        # ---------------------------------------------------------------- reductions
        @staticmethod
        def _norm_parts(X, eps):
            Lr = X.shape[-1]
            m = -(-Lr // 128)
            mu = X.mean(-1, keepdim=True)
            d = X - mu
            V = (d * d).mean(-1, keepdim=True)
            r = 1.0 / torch.sqrt(V + eps)
            yn = d * r
            e_mu = (m + 8) * U * X.abs().mean(-1, keepdim=True)
            rho = (m + 10) * U + e_mu ** 2 / (V + eps)
            e = (e_mu + U * d.abs()) * r + yn.abs() * (rho / 2 + 4 * U)
            return yn, e

        def inorm(self, x, relu=False):
            X = _d(x)
            y = super().inorm(x, relu)
            n_, c_, h_, w_ = x.shape
            yn, e = self._norm_parts(X.view(n_ * c_, h_ * w_), f32(1e-5))
            ref = yn.clamp(min=0) if relu else yn
            self._rec("inorm", "-", y, ref.view_as(X), 2 * e.view_as(X))
            return y

        def layer_norm(self, x, g, b, src=None):
            X, G, B_, S_ = _d(x), _d(g), _d(b), _d(src)
            y = super().layer_norm(x, g, b, src)
            c = x.shape[-1]
            yn, e = self._norm_parts(X.reshape(-1, c), f32(1e-5))
            ref = yn * G + B_
            extra = 3 * U * ((yn * G).abs() + B_.abs())
            if S_ is not None:
                ref = ref + S_.reshape(-1, c)
                extra = extra + 3 * U * S_.reshape(-1, c).abs()
            self._rec("layer_norm", "-", y, ref.view_as(X), (2 * (e * G.abs() + extra)).view_as(X))
            return y

        def softmax_(self, x):
            X = _d(x)
            y = super().softmax_(x)
            Lr = x.shape[-1]
            m = -(-Lr // 128)
            ref = torch.softmax(X, -1)
            bound = 2 * ref * U * ((X - X.amax(-1, keepdim=True)).abs() + m + 12) + TINY
            self._rec("softmax", "-", y, ref, bound)
            return y

        # ---------------------------------------------------------------- products
        def _gemm_check(self, method, A, Bm, bias, mask, alpha, act, y):
            """A [nb, M, K], Bm [nb, K, N] float64; y the kernel's [nb, M, N]"""
            name, args, _ = self.calls[-1]
            assert name == "vfi_gm_gemm"
            variant = gemm_variant(args[0], args[1] or 0, args[2] or 0, args[6], args[7], args[8], args[9], args[10], args[11],
                                   args[13], args[14])
            al = f32(alpha)
            ref = al * torch.matmul(A, Bm)
            S = abs(al) * torch.matmul(A.abs(), Bm.abs())
            if bias is not None:
                ref, S = ref + bias, S + bias.abs()
            if mask is not None:
                mk = mask[torch.arange(A.shape[0], device=mask.device) % mask.shape[0]]
                ref, S = ref + mk, S + mk.abs()
            K = A.shape[-1]
            bound = 2 * (K + 3) * U * S
            if act == 1:
                v = ref
                ref = F.gelu(v)
                bound = 1.2 * bound + U * (v.abs() * (4 + v.abs()) + 2 * ref.abs())
            self._rec(method, variant, y, ref, bound)

        def linear(self, x, w, b=None, act=0):
            X, W_, B_ = _d(x), _d(w), _d(b)
            y = super().linear(x, w, b, act)
            k = x.shape[-1]
            self._gemm_check("linear", X.reshape(1, -1, k), W_.t()[None], B_, None, 1.0, act, y.reshape(1, -1, w.shape[0]))
            return y

        def bmm(self, a, b, bt, alpha=1.0, mask=None):
            A, B_, M_ = _d(a), _d(b), _d(mask)
            y = super().bmm(a, b, bt, alpha, mask)
            self._gemm_check("bmm", A, B_.transpose(1, 2) if bt else B_, None, M_, alpha, 0, y)
            return y

        # ---------------------------------------------------------------- data movement (bit-exact)
        def transpose(self, x):
            X = _d(x)
            y = super().transpose(x)
            self._rec("transpose", "-", y, X.transpose(1, 2), torch.zeros_like(y, dtype=torch.float64))
            return y

        def window(self, x, k, sh, sw, to_windows, b, h, w, c):
            X = _d(x)
            y = super().window(x, k, sh, sw, to_windows, b, h, w, c)
            ref = _window_split(X, b, h, w, c, k, sh, sw) if to_windows else _window_merge(X, b, h, w, c, k, sh, sw)
            self._rec("window", "shift" if (sh or sw) else "plain", y, ref, torch.zeros_like(ref))
            return y

        def to_tokens(self, x):
            X = _d(x)
            y = super().to_tokens(x)
            self._rec("nchw_tokens", "to_tokens", y, X.flatten(2).transpose(1, 2), torch.zeros_like(y, dtype=torch.float64))
            return y

        def to_nchw(self, t, h, w):
            T = _d(t)
            y = super().to_nchw(t, h, w)
            ref = T.transpose(1, 2).reshape(t.shape[0], t.shape[2], h, w)
            self._rec("nchw_tokens", "to_nchw", y, ref, torch.zeros_like(ref))
            return y

        def pixel_shuffle2(self, x):
            X = _d(x)
            y = super().pixel_shuffle2(x)
            self._rec("pixel_shuffle2", "-", y, F.pixel_shuffle(X, 2), torch.zeros_like(y, dtype=torch.float64))
            return y

        def copy_slice(self, src, dst, c, s_coff=0, d_coff=0, src_nhwc=False, dst_nhwc=False, mean=None, std=None):
            S_, before, Mn, Sd = _d(src), dst.detach().clone(), _d(mean), _d(std)
            y = super().copy_slice(src, dst, c, s_coff, d_coff, src_nhwc, dst_nhwc, mean, std)
            s = S_.permute(0, 3, 1, 2) if src_nhwc else S_
            s = s[:, s_coff:s_coff + c]
            g = y.permute(0, 3, 1, 2) if dst_nhwc else y
            hd, wd = g.shape[2], g.shape[3]
            ref = torch.zeros(s.shape[0], c, hd, wd, dtype=torch.float64, device=s.device)
            hh, ww = min(hd, s.shape[2]), min(wd, s.shape[3])
            ref[:, :, :hh, :ww] = s[:, :, :hh, :ww]
            bound = torch.zeros_like(ref)
            if Mn is not None:
                mv, sv = Mn.view(1, -1, 1, 1), Sd.view(1, -1, 1, 1)
                bound[:, :, :hh, :ww] = (4 * U * (s[:, :, :hh, :ww].abs() + mv.abs()) / sv.abs())
                ref[:, :, :hh, :ww] = (ref[:, :, :hh, :ww] - mv) / sv
            variant = ("nhwc" if src_nhwc else "nchw") + ">" + ("nhwc" if dst_nhwc else "nchw") + ("+norm" if Mn is not None else "")
            self._rec("copy_slice", variant, g[:, d_coff:d_coff + c], ref, bound)
            keep = torch.ones_like(before, dtype=torch.bool)
            if dst_nhwc:
                keep[..., d_coff:d_coff + c] = False
            else:
                keep[:, d_coff:d_coff + c] = False
            self._untouched("copy_slice", variant, before, y, keep)
            return y

        def axpby(self, a, b=None, alpha=1.0, beta=1.0, gamma=0.0, post=0, out=None):
            A, B_ = _d(a), _d(b)
            y = super().axpby(a, b, alpha, beta, gamma, post, out)
            al, be, ga = f32(alpha), f32(beta), f32(gamma)
            ref, S = al * A + ga, (al * A).abs() + abs(ga)
            if B_ is not None:
                ref, S = ref + be * B_, S + (be * B_).abs()
            if post == 1:
                ref = ref.clamp(min=0)
            elif post == 2:
                ref = ref.clamp(0, 1)
            self._rec("axpby", "inplace" if out is not None and out.data_ptr() == a.data_ptr() else "-", y, ref, 6 * U * S)
            return y

        # ---------------------------------------------------------------- position, matching, propagation
        def add_position_(self, x, k):
            X = _d(x)
            y = super().add_position_(x, k)
            pos, arg = ref_position(x.shape, k, x.device)
            ref = X + pos
            self._rec("add_position", "-", y, ref, 2 * U * (32 * arg.abs() + 4 + ref.abs()))
            return y

        def local_match(self, f0, f1, r):
            A, B_ = _d(f0), _d(f1)
            y = super().local_match(f0, f1, r)
            for comp, (ref, bound) in enumerate(ref_local_match(A, B_, r)):
                self._rec("local_match", f"R{r}", y[:, comp], ref, bound)
            return y

        def local_prop(self, q, k, flow):
            Q, K_, Fl = _d(q), _d(k), _d(flow)
            y = super().local_prop(q, k, flow)
            for comp, (ref, bound) in enumerate(ref_local_prop(Q, K_, Fl)):
                self._rec("local_prop", "-", y[:, comp], ref, bound)
            return y

        def convex_up(self, mask, flow, f):
            Mk, Fl = _d(mask), _d(flow)
            y = super().convex_up(mask, flow, f)
            for comp, (ref, bound) in enumerate(ref_convex_up(Mk, Fl, f)):
                self._rec("convex_up", "-", y[:, comp], ref, bound)
            return y

        # ---------------------------------------------------------------- resampling
        def warp(self, x, flow):
            X, Fl = _d(x), _d(flow)
            y = super().warp(x, flow)
            ref, e = ref_warp(X, Fl)
            self._rec("warp_zeros", "-", y, ref, 2 * e)
            return y

        def resize(self, x, ho, wo, align=False, mul=1.0):
            X = _d(x)
            y = super().resize(x, ho, wo, align, mul)
            b, c, h, w = x.shape
            mu = f32(mul)
            ref = F.interpolate(X, size=(ho, wo), mode="bilinear", align_corners=bool(align)) * mu
            dev = x.device
            yy = torch.arange(ho, device=dev, dtype=torch.float64)
            xx = torch.arange(wo, device=dev, dtype=torch.float64)
            if align:
                cy = yy * ((h - 1) / (ho - 1) if ho > 1 else 0.0)
                cx = xx * ((w - 1) / (wo - 1) if wo > 1 else 0.0)
            else:
                cy = ((yy + 0.5) * h / ho - 0.5).clamp(min=0)
                cx = ((xx + 0.5) * w / wo - 0.5).clamp(min=0)
            cy, cx = cy.view(1, ho, 1).expand(b * c, ho, wo), cx.view(1, 1, wo).expand(b * c, ho, wo)
            lip, amax = _cells(X.reshape(b * c, h, w), cx, cy, 4 * U * (cx + 1), 4 * U * (cy + 1), False)
            bound = 2 * ((lip + 8 * U * amax).view_as(ref) * abs(mu) + U * ref.abs())
            self._rec("resize", "align" if align else "half-pixel", y, ref, bound)
            return y

        def metric_input(self, i0, i1, f01, f10):
            I0, I1, A, Cf = _d(i0), _d(i1), _d(f01), _d(f10)
            y = super().metric_input(i0, i1, f01, f10)
            b, _, h, w = i0.shape
            dev = i0.device
            s1, e1 = ref_warp(I1, A)
            s0, e0 = ref_warp(I0, Cf)
            zero = torch.zeros_like(I0)
            self._rec("metric_input", "images", y[:, 0:6], torch.cat([I0, I1], 1), torch.cat([zero, zero], 1))
            ph = torch.cat([-(I0 - s1).abs().mean(1, keepdim=True), -(I1 - s0).abs().mean(1, keepdim=True)], 1)
            pb = torch.cat([e1.sum(1, keepdim=True) / 3 + U * (I0.abs() + s1.abs()).sum(1, keepdim=True),
                            e0.sum(1, keepdim=True) / 3 + U * (I1.abs() + s0.abs()).sum(1, keepdim=True)], 1)
            self._rec("metric_input", "photometric", y[:, 6:8], ph, 2 * (pb + U * ph.abs()))
            nrm = torch.tensor([(w - 1) / 2.0, (h - 1) / 2.0], dtype=torch.float64, device=dev).view(1, 2, 1, 1)
            fl = torch.cat([A / nrm, Cf / nrm], 1)
            self._rec("metric_input", "flows", y[:, 8:12], fl, 2 * U * fl.abs())
            # forward-backward consistency flags
            for ch, (margin, allow) in zip((12, 13), ref_fb_margins(A, Cf)):
                ref = (margin > 0).double()
                got = y[:, ch].double()
                flip = got != ref
                r = torch.where(flip, margin.abs() / allow, torch.zeros_like(margin))
                r = torch.where(torch.isfinite(got) & ((got == 0) | (got == 1)), r, torch.full_like(r, math.inf))
                wv, at = _argmax(r)
                self.stats.add("metric_input", "occlusion", got.shape, wv, at)
                self.stats.occ_near += int((margin.abs() <= allow).sum())
                self.stats.occ_flips += int(flip.sum())
                self.stats.occ_pixels += int(margin.numel())
            return y

    Shadow.__name__ = "ShadowOps"
    return Shadow


def shadow_class():
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.gmfss import Ops
    return make_shadow_class(Ops)


def shadow(ops):
    """turn the product's Ops instance (its registered weight layouts kept) into a ShadowOps in place"""
    ops.__class__ = shadow_class()
    ops._shadow_init()
    return ops


# ----------------------------------------------------------------------------------------------- the soft splat
def splat_reference(x, flow, metric):
    """float64 soft splat with addeps: index_add_ of x e^m w and e^m w over the four corners at the exact coordinate;
    returns (out, bound) with the bound of the module docstring"""
    X, Fl, Mt = x.double(), flow.double(), metric.double()
    b, c, h, w = X.shape
    dev = X.device
    gx = torch.arange(w, device=dev, dtype=torch.float64).view(1, w).expand(h, w)
    gy = torch.arange(h, device=dev, dtype=torch.float64).view(h, 1).expand(h, w)
    out = torch.zeros(b, c, h, w, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(out)
    for n in range(b):
        cx, cy = gx + Fl[n, 0], gy + Fl[n, 1]
        dcx, dcy = U * cx.abs(), U * cy.abs()
        e = torch.exp(Mt[n, 0])
        xe = X[n] * e                                   # [c, h, w]
        num = torch.zeros(c, h * w, dtype=torch.float64, device=dev)
        absn = torch.zeros_like(num)
        crd = torch.zeros_like(num)
        den = torch.zeros(1, h * w, dtype=torch.float64, device=dev)
        absd, crdd, cnt = torch.zeros_like(den), torch.zeros_like(den), torch.zeros_like(den)

        def corners(px, py):
            x0, y0 = torch.floor(px), torch.floor(py)
            for ox, oy in ((0, 0), (1, 0), (0, 1), (1, 1)):
                tx, ty = x0 + ox, y0 + oy
                inside = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
                idx = (ty.clamp(0, h - 1) * w + tx.clamp(0, w - 1)).long().reshape(-1)
                yield tx, ty, inside.reshape(-1).double(), idx

        for tx, ty, inside, idx in corners(cx, cy):
            wt = ((1 - (cx - tx).abs()) * (1 - (cy - ty).abs())).reshape(-1) * inside
            num.index_add_(1, idx, xe.reshape(c, -1) * wt)
            absn.index_add_(1, idx, xe.reshape(c, -1).abs() * wt)
            den.index_add_(1, idx, (e.reshape(-1) * wt)[None])
            absd.index_add_(1, idx, (e.reshape(-1) * wt)[None])
        for sx in (-1.0, 1.0):
            for sy in (-1.0, 1.0):
                for _, _, inside, idx in corners(cx + sx * dcx, cy + sy * dcy):
                    dc = (dcx + dcy).reshape(-1) * inside
                    crd.index_add_(1, idx, xe.reshape(c, -1).abs() * dc)
                    crdd.index_add_(1, idx, (e.reshape(-1) * dc)[None])
                    cnt.index_add_(1, idx, inside[None])
        D = den + 1e-7
        o = num / D
        EN = crd + 8 * U * absn + (cnt + 1) * U * absn
        ED = crdd + 8 * U * absd + (cnt + 1) * U * absd
        out[n] = o.view(c, h, w)
        bound[n] = (2 * ((EN + o.abs() * (ED + U * D)) / D + U * o.abs())).view(c, h, w)
    return out, bound


def shadow_splat(splat, stats: ShadowStats):
    """wrap a splat callable (x, flow, metric) -> soft splat: each call checked against splat_reference"""
    def call(x, flow, metric):
        X, Fl, Mt = _d(x), _d(flow), _d(metric)
        y = splat(x, flow, metric)
        ref, bound = splat_reference(X, Fl, Mt)
        r = ratio_of(y, ref, bound)
        w, at = _argmax(r)
        stats.add("splat", "soft", y.shape, w, at)
        return y
    return call


# ----------------------------------------------------------------------------------------------- standalone case matrix
def case_matrix(o, seed=0):
    """every kernel at the shapes and edges where such kernels go wrong, on a ShadowOps `o` (any device); the results land
    in o.stats.  Returns the variants each gemm case was expected to take."""
    from cfi_b200.gmfss import _shift_mask
    dev = o.dev
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev)            # noqa: E731
    ru = lambda *s: torch.rand(*s, generator=g).to(dev)                                   # noqa: E731
    expect = {}
    # conv: every packed (k, s), the generic kernel at k = 7 s1 and k = 5; Cout 1 / 17 / 19, Wo 1 / 7 / 9 / 17; channel
    # slices in and out, res1 + res2, post 0..3
    for k, s in ((3, 1), (3, 2), (1, 1), (1, 2), (7, 2), (7, 1), (5, 1), (5, 2)):
        for cout, wo in ((1, 1), (17, 7), (19, 9), (16, 17)):
            pd = k // 2
            wi = (wo - 1) * s + 1 + (k - 1) - 2 * pd
            wi = max(wi, 1)
            hi = 5
            x = rn(2, 9, hi, wi)
            w = rn(cout, 5, k, k, scale=0.3)
            if (k, s) not in ((7, 1), (5, 1), (5, 2)):
                o.register_conv(w)
            b = rn(cout)
            ho = (hi + 2 * pd - k) // s + 1
            wo_ = (wi + 2 * pd - k) // s + 1
            for post in (0, 1, 2, 3):
                r1, r2 = rn(2, cout, ho, wo_), rn(2, cout, ho, wo_)
                out = o.new(2, cout + 6, ho, wo_)
                o.conv(x, w, b, stride=s, pad=pd, pre=0.3 if post != 2 else None, post=post, post_slope=0.2, res1=r1,
                       res2=r2 if post in (1, 3) else None, out=out, out_coff=4, in_coff=2, cin=5)
            o.conv(x[:, :5].contiguous(), w, None, stride=s, pad=pd)
    # convt4: Cout not a multiple of 16, 1 x 1 inputs
    for cout, h, w in ((19, 1, 1), (17, 3, 5), (32, 4, 4)):
        o.convt4(rn(2, 6, h, w), rn(6, cout, 4, 4, scale=0.3), rn(cout), pre=0.2)
        o.convt4(rn(1, 3, h, w), rn(3, cout, 4, 4, scale=0.3), rn(cout))
    # gemm: nn8<8> / <4> / <2> with a partial last row tile; bt; unaligned lda; N % 8 != 0; masks with nmask 1 and > 1;
    # GELU; bias
    for rows, want in ((60001, "nn8<8>"), (40003, "nn8<4>"), (37, "nn8<2>")):
        o.bmm(rn(1, rows, 8), rn(1, 8, 64), False, 0.25)
        expect[("bmm", rows)] = want
    wl = rn(24, 16, scale=0.3)
    o.register_linear(wl)
    o.linear(rn(3, 7, 16), wl, rn(24), act=1)                       # nn8<2>, 21 rows, GELU, bias
    o.linear(rn(3, 7, 16), rn(12, 16), rn(12), act=1)               # N % 8 != 0: the generic bt form
    o.linear(rn(2, 5, 6), rn(8, 6), None)                           # K = 6: unaligned lda, generic bt
    o.bmm(rn(2, 9, 6), rn(2, 6, 16), False, 0.5)                    # lda = 6: the generic nn kernel
    o.bmm(rn(2, 9, 8), rn(2, 8, 12), False, 0.5)                    # N = 12: the generic nn kernel
    mask = _shift_mask(8, 12, 2).to(dev)                             # [4, 24, 24] of 0 / -100
    q, kk = rn(8, 24, 16), rn(8, 24, 16)
    o.scores(q, kk, 0.25, mask)                                      # nmask 4, transposed keys, nn8
    o.bmm(q, kk, True, 0.25, mask)                                   # nmask 4, the bt kernel
    o.bmm(q, kk, True, 0.25, mask[:1].contiguous())                  # nmask 1
    o.scores(rn(2, 10, 16), rn(2, 17, 16), 0.5)                      # 17 keys: bt
    # softmax: rows of 1, 127, 129, 8160, with logits >= 100
    for l in (1, 127, 129, 8160):
        x = rn(3, l, scale=4.0)
        x[1] += 120.0
        x[2, : (l + 1) // 2] += 100.0
        o.softmax_(x)
    # norms: a large mean offset (|mean| >> std), planes up to 130560 elements
    for hw_, off in ((7, 0.0), (130, 300.0), (16 * 300, 300.0), (130560, 300.0)):
        o.inorm((rn(2, 3, 1, hw_) + off).contiguous(), relu=False)
        o.inorm((rn(1, 2, 1, hw_) - off).contiguous(), relu=True)
    for c, off in ((128, 1000.0), (127, 0.0), (129, -1000.0), (7, 50.0)):
        t = rn(3, 40, c) + off
        o.layer_norm(t, 1 + rn(c, scale=0.1), rn(c), src=rn(3, 40, c))
        o.layer_norm(t, 1 + rn(c, scale=0.1), rn(c))
    # windows with and without the shift at k = 2, 3, 8; position embedding
    for k, h, w in ((2, 8, 12), (3, 9, 12), (8, 16, 24)):
        tok = rn(2, h * w, 5)
        for sh, sw in ((0, 0), ((h // k) // 2, (w // k) // 2), (0, 1), (1, 0)):
            win = o.window(tok, k, sh, sw, True, 2, h, w, 5)
            o.window(win, k, sh, sw, False, 2, h, w, 5)
        o.add_position_(rn(2, 16, h, w), k)
    # local_match at R = 1..4, also on planes smaller than the window; local_prop and convex_up at the borders
    for r in (1, 2, 3, 4):
        for h, w in ((5, 7), (2, 3), (1, 1)):
            o.local_match(rn(1, 16, h, w), rn(1, 16, h, w), r)
    for h, w in ((5, 7), (1, 1), (2, 9)):
        o.local_prop(rn(2, h * w, 16, scale=2.0), rn(2, h * w, 16, scale=2.0), rn(2, 2, h, w, scale=3.0))
        o.convex_up(rn(1, 9 * 16, h, w, scale=3.0), rn(1, 2, h, w, scale=3.0), 4)
    # warps with flows leaving all four sides, and integer flows; resize with odd sizes, both align settings and mul
    x = ru(2, 3, 9, 13)
    fl = rn(2, 2, 9, 13, scale=6.0)
    fl[:, 0, :, :3] = -20.0
    fl[:, 0, :, -3:] = 20.0
    fl[:, 1, :2] = -15.0
    fl[:, 1, -2:] = 15.0
    o.warp(x, fl)
    o.warp(x, torch.round(fl))
    o.warp(x, torch.round(fl / 8))
    for (h, w, ho, wo) in ((9, 13, 4, 6), (9, 13, 5, 7), (9, 13, 18, 26), (7, 11, 15, 21), (1, 5, 1, 9)):
        for align in (False, True):
            for mul in (1.0, 0.3, 2.0):
                o.resize(rn(2, 3, h, w), ho, wo, align=align, mul=mul)
    i0, i1 = ru(2, 3, 9, 13), ru(2, 3, 9, 13)
    o.metric_input(i0, i1, fl, rn(2, 2, 9, 13, scale=6.0))
    o.metric_input(i0, i1, torch.round(fl), torch.round(-fl))
    o.metric_input(i0, i1, rn(2, 2, 9, 13, scale=0.3), rn(2, 2, 9, 13, scale=0.3))
    # copies: NHWC <-> NCHW with mean / std, crops and zero padding; axpby with out aliasing a; pixel shuffle; transpose
    mean, std = torch.tensor([0.485, 0.456, 0.406], device=dev), torch.tensor([0.229, 0.224, 0.225], device=dev)
    src = ru(2, 7, 9, 5)
    for hd, wd in ((7, 9), (5, 6), (8, 12)):
        o.copy_slice(src, o.new(2, hd, wd, 8), 3, 1, 2, src_nhwc=True, dst_nhwc=True, mean=mean, std=std)
        o.copy_slice(src, o.new(2, 6, hd, wd), 3, 2, 1, src_nhwc=True, dst_nhwc=False, mean=mean, std=std)
        o.copy_slice(ru(2, 5, 7, 9), o.new(2, hd, wd, 4), 3, 2, 0, src_nhwc=False, dst_nhwc=True)
        o.copy_slice(ru(2, 5, 7, 9), o.new(2, 7, hd, wd), 3, 0, 3)
    a = rn(3, 5, 7)
    o.axpby(a, rn(3, 5, 7), 0.3, -1.7, 0.25, post=0, out=a)
    o.axpby(rn(4, 9), rn(4, 9), 1.0, 1.0, post=1)
    o.axpby(rn(4, 9), None, 0.7, post=2)
    o.pixel_shuffle2(rn(2, 12, 5, 3))
    o.transpose(rn(3, 7, 5))
    o.to_nchw(o.to_tokens(rn(2, 5, 3, 7)), 3, 7)
    return expect


# ----------------------------------------------------------------------------------------------- refusals
def refusals(o):
    """each refused call: (what, rc, message, output untouched)"""
    L = o.L._lib if isinstance(o.L, _Recorder) else o.L
    dev = o.dev
    st = o._st()
    res = []

    def guard(*shape):
        return torch.full(shape, NAN, device=dev)

    def check(what, rc, out):
        msg = L.vfi_last_error().decode()
        res.append((what, rc, msg, bool(torch.isnan(out).all())))

    x, out = torch.rand(1, 4, 8, 8, device=dev), guard(1, 16, 8, 8)
    wt = torch.zeros(4 * 25, 16, device=dev)
    check("conv2d_packed k=5", L.vfi_gm_conv2d_packed(x.data_ptr(), wt.data_ptr(), None, None, None, out.data_ptr(), 1, 4, 8, 8, 16, 16,
                                                      5, 1, 2, 4, 0, 16, 0, 0, 0.0, 0, 0.0, st), out)
    t, out = torch.rand(1, 10 * 8, 4, device=dev), guard(1, 10 * 8, 4)
    check("window H % k", L.vfi_gm_window(t.data_ptr(), out.data_ptr(), 1, 10, 8, 4, 4, 0, 0, 1, st), out)
    f0, out = torch.rand(1, 4, 6, 6, device=dev), guard(1, 2, 6, 6)
    check("local_match R=5", L.vfi_gm_local_match(f0.data_ptr(), f0.data_ptr(), out.data_ptr(), 1, 4, 6, 6, 5, st), out)
    a, m, out = torch.rand(1, 8, 8, device=dev), torch.zeros(1, 8, 8, device=dev), guard(1, 8, 8)
    check("gemm mask nmask=0", L.vfi_gm_gemm(0, a.data_ptr(), a.data_ptr(), None, m.data_ptr(), out.data_ptr(), 1, 8, 8, 8, 8, 8, 8,
                                             64, 64, 64, 1.0, 0, 0, st), out)
    s, mean, out = torch.rand(1, 3, 4, 4, device=dev), torch.rand(3, device=dev), guard(1, 3, 4, 4)
    check("copy_slice mean only", L.vfi_gm_copy_slice(s.data_ptr(), out.data_ptr(), 1, 3, 4, 4, 4, 4, 3, 0, 3, 0, 0, 0, mean.data_ptr(),
                                                       None, st), out)
    check("copy_slice std only", L.vfi_gm_copy_slice(s.data_ptr(), out.data_ptr(), 1, 3, 4, 4, 4, 4, 3, 0, 3, 0, 0, 0, None,
                                                     mean.data_ptr(), st), out)
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)
    return res


GEMM_VARIANTS = {"nn8<8>", "nn8<4>", "nn8<2>", "bt", "nn"}
CONV_VARIANTS = {"packed(3,1)", "packed(3,2)", "packed(1,1)", "packed(1,2)", "packed(7,2)", "generic(7,1)", "generic(5,1)",
                 "generic(5,2)"}


def check_matrix(o):
    """case_matrix on `o`: every element within its bound, every kernel variant reached"""
    case_matrix(o)
    st = o.stats
    print("\n" + "\n".join(st.lines()))
    assert not st.failures(), st.failures()
    assert st.variants("bmm") | st.variants("linear") >= GEMM_VARIANTS
    assert st.variants("conv") >= CONV_VARIANTS
    assert {"R1", "R2", "R3", "R4"} <= st.variants("local_match")
    assert {"shift", "plain"} <= st.variants("window")
    assert st.variants("axpby") >= {"inplace", "-"}


def check_refusals(o):
    """each refused launch returns VFI_E_INVALID (-1) with a message and leaves its output alone"""
    res = refusals(o)
    assert len(res) == 6
    for what, rc, msg, untouched in res:
        assert rc == -1 and msg.startswith("vfi_gm: ") and untouched, (what, rc, msg, untouched)
