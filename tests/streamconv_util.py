"""Shared by test_streamconv_host.py (CUDA-core checker, host emulation) and test_gpu_zstreamconv.py (wgmma kernel and
checker on the GPU): the case table of streamconv layers, a float64 reference of the operation that does not share the
checker's packed weights or plan, and the runner that drives the C hook vfi_streamconv_debug_conv with guarded output
tensors.

Reference: the 16-bit inputs and the weights rounded to the operand type (round to nearest, like torch.Tensor.to), both
widened to float64, plus the fp32 shift; F.pad with the requested rows / columns before and after, then a valid conv2d;
temporal tap dt of output plane t reads input plane t + dt - pad_t of the same sample (zero outside [0, T_in)); then the
epilogue (ext 0: LeakyReLU(0.2) or identity; ext 1: PReLU(slope) then + residual; ext 2: + residual then per-channel
PReLU, columns [0, n_f32) in fp32).  With K = kt * ksize^2 * (c0 + c1) products per output and
S = conv(|x|, |w|) + |shift| (+ |residual|), times max(1, |slope|) where a PReLU follows (a sign flip near 0 moves the
result by at most that factor), every element satisfies
    16-bit columns:  |y - y^| <= ulp_T(y^) + 2 K 2^-24 S
    fp32 columns:    |y - y^| <= 2 K 2^-24 S
(the bound of tests/test_gpu_layers.py).

Guards: the output is a channel slice at a 32-byte offset of a tensor with a wider pixel pitch, between a guard image
before and one after, all filled with a sentinel bit pattern (a NaN); the fp32 tensor likewise.  Every cell outside the
slice must keep its bits and no cell inside it may keep the sentinel.  The source tensors carry NaN in every channel
outside the slice the layer reads.
"""
import ctypes as C

import torch
import torch.nn.functional as F

from test_gpu_layers import U32, _ulp

SPEC_KEYS = ("ksize", "c0", "c1", "n_total", "act", "ext", "n_f32", "pad_before", "pad_before_x", "kt", "pad_t", "T_in",
             "T_out")
SENT16 = {torch.float16: 0x7E5A, torch.bfloat16: 0x7FDA}   # quiet NaNs of each type
SENT32 = 0x7FBADBAD
DTYPES = {"float16": (0, torch.float16), "bfloat16": (1, torch.bfloat16)}

DEFAULT = dict(ksize=3, c0=64, c1=0, n_total=64, act=1, ext=0, n_f32=0, pad_before=-1, pad_before_x=-1, kt=1, pad_t=0,
               T_in=1, T_out=1, slope=1.0, B=2, H=17, W=9, pitch0=None, off0=0, pitch1=None, off1=0, out_off=16,
               out_pitch=None, res=None, f32_off=2, f32_pitch=12, num_sms=0)


def case(name, **kw):
    c = dict(DEFAULT, name=name)
    c.update(kw)
    if c["pitch0"] is None:
        c["pitch0"] = c["off0"] + c["c0"]
    if c["pitch1"] is None:
        c["pitch1"] = c["off1"] + c["c1"]
    if c["out_pitch"] is None:
        c["out_pitch"] = c["out_off"] + c["n_total"] + 16
    return c


def spec_of(c):
    return [int(c[k]) for k in SPEC_KEYS]


def _cases():
    out = []
    # every wgmma N (nsplit 1) and the split widths 144 / 192 / 256 / 512 (n_cta 48 / 96 / 128 / 128, nsplit 3 / 2 / 2 / 4),
    # crossed with the three epilogues: all 48 kernel instantiations of the two operand types
    for n in (16, 32, 48, 64, 80, 96, 112, 128, 144, 192, 256, 512):
        out.append(case(f"n{n}_ext0", n_total=n, act=n % 32 == 0))
        out.append(case(f"n{n}_ext1", n_total=n, ext=1, act=0, slope=0.25, res="sep"))
        out.append(case(f"n{n}_ext2", n_total=n, ext=2, act=0, n_f32=2, res="sep"))
    # padding: 'same' for k = 1, 2, 3; the stride-2 form (k 2, one row / column before); the four transposed-conv phases
    for k in (1, 2, 3):
        out.append(case(f"same_k{k}", ksize=k, H=19, W=11))
    out.append(case("s2d_stride2", ksize=2, pad_before=1, ext=1, act=0, slope=-0.7, c0=256, n_total=128))
    for py in (0, 1):
        for px in (0, 1):
            out.append(case(f"convt_phase{py}{px}", ksize=2, pad_before=1 - py, pad_before_x=1 - px, ext=2, act=0, n_f32=4,
                            n_total=64, c0=192))
    # sources: two of different pitches, both at channel offsets; a slice at element 8 of a 136-wide tensor; FILM's
    # widest fusion input (2 x 960 + 64 aligned channels + 512 decoder channels: 39 k-blocks)
    out.append(case("two_sources", c0=64, off0=8, pitch0=136, c1=128, off1=64, pitch1=256, n_total=96))
    out.append(case("slice_at_8", c0=128, off0=8, pitch0=136, n_total=48))
    out.append(case("two_sources_ext2", c0=128, c1=64, pitch1=72, off1=8, ext=2, act=0, n_f32=8, res="sep", n_total=144))
    out.append(case("film_widest_fusion", c0=1984, c1=512, n_total=32, B=1, H=5, W=7))
    # temporal taps: kt 1..4, pad_t in {0, 1, kt - 1}, T_in != T_out, 2 samples
    tt = [(4, 4), (3, 5), (4, 1), (5, 3)]
    i = 0
    for kt in (1, 2, 3, 4):
        for pt in sorted({0, 1, kt - 1}):
            if pt >= kt and kt > 1:
                continue
            ti, to = tt[i % len(tt)]
            i += 1
            out.append(case(f"kt{kt}_pt{pt}_T{ti}to{to}", kt=kt, pad_t=pt, T_in=ti, T_out=to, H=9, W=10, n_total=32,
                            ext=i % 2, act=0, slope=0.0))
    # image sizes: FILM's coarsest levels (halo larger than the image), one exact tile, one tile + 1 row / column, odd
    # tile counts (the second MMA warpgroup idles in the last pass)
    for (b, h, w) in ((1, 1, 1), (2, 1, 1), (1, 2, 3), (3, 2, 3), (2, 16, 8), (1, 17, 9), (1, 48, 8), (3, 16, 8)):
        out.append(case(f"img{b}x{h}x{w}", B=b, H=h, W=w))
        out.append(case(f"img{b}x{h}x{w}_ext2", B=b, H=h, W=w, ext=2, act=0, n_f32=2, n_total=32, res="sep"))
    # ring wrap: one CTA per split walks every pass, and 2 nsplit + 1 CTAs
    for n in (64, 256):
        for grid in ("nsplit", "2nsplit+1"):
            out.append(case(f"ring_n{n}_{grid}", n_total=n, num_sms=grid, B=2, H=40, W=24, c0=128, kt=2, pad_t=1, T_in=2,
                            T_out=2, ext=1, act=0, slope=0.25, res="sep"))
    # ext 1 slopes x residual (absent, separate, in place: Sepconv's hor[r][1] / ver[r][1])
    for s in (1.0, 0.0, 0.25, -0.7, 3.0):
        for r in (None, "sep", "inplace"):
            out.append(case(f"ext1_slope{s}_res{r}", ext=1, act=0, slope=s, res=r, n_total=64))
    # ext 2: per-channel slopes (negative ones and 1.0), n_f32 in {0, 2, 8} x residual, and with nsplit > 1
    for nf in (0, 2, 8):
        for r in (None, "sep", "inplace"):
            out.append(case(f"ext2_nf{nf}_res{r}", ext=2, act=0, n_f32=nf, res=r, n_total=48))
        out.append(case(f"ext2_nf{nf}_nsplit2", ext=2, act=0, n_f32=nf, res="sep", n_total=256))
    # an output slice at offset 0 of a tensor exactly n_total wide
    out.append(case("out_packed", out_off=0, out_pitch=64))
    # the plans the models ship (test_gpu_zstreamconv.py fails on a shipped plan no case here has): 1x1 layers (FILM's
    # flow heads, FLAVR's downsample and feature_fuse); the four transposed-conv phases at IFRNet's ConvT widths (ext 2)
    # and at FLAVR's, with three temporal taps on two sources (ext 0); 2x2 'same' (FILM's fusion) and stride-2 forms;
    # 3x3x3 layers; IFRNet-L's wide 3x3 layers (nsplit 3 and 4 at n_cta 128, 112, 80)
    for n in (16, 32, 128, 256, 512):
        out.append(case(f"k1_n{n}", ksize=1, c0=128, n_total=n))
    out.append(case("k1_kt4_fuse", ksize=1, kt=4, T_in=4, T_out=1, n_total=64))
    for py in (0, 1):
        for px in (0, 1):
            pads = dict(ksize=2, pad_before=1 - py, pad_before_x=1 - px)
            for n in (16, 32, 48, 80, 112, 160):
                out.append(case(f"convt{py}{px}_n{n}", **pads, c0=128, n_total=n, ext=2, act=0, n_f32=4, res="sep"))
            for n in (64, 128):
                out.append(case(f"convt{py}{px}_kt3_n{n}", **pads, c0=64, c1=64, n_total=n, kt=3, pad_t=1, T_in=4,
                                T_out=4, B=1, act=0))
    for n in (128, 256, 512):
        out.append(case(f"k2_same_n{n}", ksize=2, c0=128, n_total=n))
    for n, ext, kt in ((64, 1, 1), (256, 1, 1), (512, 1, 1), (128, 2, 1), (192, 2, 1), (128, 1, 3), (256, 1, 3)):
        out.append(case(f"s2d_n{n}_ext{ext}_kt{kt}", ksize=2, pad_before=1, c0=128, n_total=n, ext=ext, act=0, slope=0.25,
                        kt=kt, pad_t=kt // 2, T_in=4 if kt > 1 else 1, T_out=4 if kt > 1 else 1, B=1 if kt > 1 else 2))
    for n in (64, 128, 256, 512):
        for ext in (0, 1):
            out.append(case(f"k3_kt3_n{n}_ext{ext}", c0=64, n_total=n, kt=3, pad_t=1, T_in=4, T_out=4, B=1, ext=ext, act=0,
                            slope=0.0))
    for n in (320, 384, 448):
        out.append(case(f"k3_n{n}_ext2", c0=128, n_total=n, ext=2, act=0, res="sep"))
    return out


CASES = _cases()

# (what the launcher refuses, the spec / argument change, the text of its refusal)
ALIGN = "tensor slices must be 16-byte (inputs) / 32-byte (output) aligned"
F32 = "an IFRNet epilogue needs its slopes, and an 8-byte aligned fp32 slice"
SHAPE = "unsupported layer shape"
REFUSALS = [
    ("odd_pitch0", dict(pitch0=65), ALIGN),
    ("out_pitch_not_16", dict(out_pitch=88), ALIGN),
    ("out_not_32B_aligned", dict(out_off=8, out_pitch=96), ALIGN),
    ("res_with_ext0", dict(res="sep"), "a residual needs an ext layer"),
    ("n_f32_odd", dict(ext=2, act=0, n_f32=3), F32),
    ("n_f32_over_8", dict(ext=2, act=0, n_f32=10, f32_pitch=12), F32),
    ("f32_pitch_below_n_f32", dict(ext=2, act=0, n_f32=8, f32_pitch=4, f32_off=0), F32),
    ("ksize4", dict(ksize=4), SHAPE),
    ("c0_32", dict(c0=32), SHAPE),
    ("n_total_24", dict(n_total=24, out_pitch=64), SHAPE),
    ("kt5", dict(kt=5, T_in=5, T_out=5), SHAPE),
]


def bind(L):
    """argtypes of the two hooks on a ctypes library (the product .so or the host emulation)."""
    vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
    L.vfi_streamconv_debug_conv.argtypes = [vp, i32, f32, i32, vp, vp, vp, vp, i32, vp, i32, vp, i32, vp, vp, i32, i32, i32,
                                            i32, i32, i32, vp]
    L.vfi_streamconv_debug_conv.restype = i32
    L.vfi_streamconv_plan.argtypes = [vp, i32, vp, i32]
    L.vfi_streamconv_plan.restype = i32
    L.vfi_last_error.restype = C.c_char_p
    return L


def plan(L, c):
    """{n_cta, nsplit, a_slots, b_slots, smem_bytes, halo_y0, halo_x0} of a case, or None when refused."""
    spec = (C.c_int32 * 13)(*spec_of(c))
    info = (C.c_int32 * 7)()
    if L.vfi_streamconv_plan(spec, 13, info, 7) != 0:
        return None
    return dict(zip(("n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes", "halo_y0", "halo_x0"), list(info)))


def plan_key(c, p):
    """What distinguishes one launch plan of the kernel from another."""
    py = -p["halo_y0"]
    px = -p["halo_x0"]
    return (p["n_cta"], p["nsplit"], c["ksize"], (py, px), c["kt"], c["ext"], p["a_slots"], p["b_slots"])


class Inputs:
    """Seeded tensors of one case on `dev`: guarded sources, weights, shift, slopes, residual, guarded outputs."""

    def __init__(self, c, tdt, dev, seed):
        g = torch.Generator().manual_seed(seed)
        B, H, W, n = c["B"], c["H"], c["W"], c["n_total"]
        bi, bo = B * c["T_in"], B * c["T_out"]
        cin = c["c0"] + c["c1"]
        K = c["kt"] * c["ksize"] ** 2 * cin
        nan = float("nan")

        def src(ch, off, pitch):
            t = torch.full((bi, H, W, max(pitch, off + ch)), nan, dtype=tdt)
            t[..., off:off + ch] = (torch.rand(bi, H, W, ch, generator=g) * 2 - 1).to(tdt)
            return t.to(dev)

        self.s0 = src(c["c0"], c["off0"], c["pitch0"])
        self.s1 = src(c["c1"], c["off1"], c["pitch1"]) if c["c1"] else None
        self.w = (torch.randn(n, c["kt"], c["ksize"] ** 2, cin, generator=g) * (2.0 / K) ** 0.5).float()
        self.shift = (torch.rand(n, generator=g) * 2 - 1).float()
        sl = (torch.rand(n, generator=g) * 3 - 1.5).float()
        sl[0::4] = 1.0
        sl[1::4] = -sl[1::4].abs() - 0.1
        self.slopes = sl
        op = c["out_pitch"]
        self.out = torch.full((bo + 2, H, W, op), SENT16[tdt], dtype=torch.int16, device=dev)
        self.f32 = torch.full((bo + 2, H, W, c["f32_pitch"]), SENT32, dtype=torch.int32, device=dev)
        self.res = None
        r = (torch.rand(bo, H, W, n, generator=g) * 2 - 1).to(tdt).to(dev)
        oo = c["out_off"]
        if c["res"] == "sep":
            self.resbuf = torch.full((bo, H, W, op), nan, dtype=tdt, device=dev)
            self.resbuf[..., oo:oo + n] = r
            self.res = r
        elif c["res"] == "inplace":
            self.out[1:-1, ..., oo:oo + n] = r.view(torch.int16)
            self.res = r
        self.before = self.out.clone()
        self.sent = SENT16[tdt]

    def ptr16(self, t, off):
        return t.data_ptr() + 2 * off

    def call(self, L, c, tdt, impl, num_sms=None, stream=None):
        op_type = 1 if tdt == torch.bfloat16 else 0
        spec = (C.c_int32 * 13)(*spec_of(c))
        oo = c["out_off"]
        optr = self.ptr16(self.out[1], oo)
        rptr = None
        if c["res"] == "sep":
            rptr = self.ptr16(self.resbuf, oo)
        elif c["res"] == "inplace":
            rptr = optr
        fptr = self.f32[1].data_ptr() + 4 * c["f32_off"] if c["ext"] == 2 else None
        w = self.w.contiguous()
        rc = L.vfi_streamconv_debug_conv(
            spec, 13, float(c["slope"]), op_type, w.data_ptr(), self.shift.data_ptr(),
            self.slopes.data_ptr() if c["ext"] == 2 else None,
            self.ptr16(self.s0, c["off0"]), c["pitch0"],
            None if self.s1 is None else self.ptr16(self.s1, c["off1"]), c["pitch1"],
            optr, c["out_pitch"], rptr, fptr, c["f32_pitch"], c["B"], c["H"], c["W"],
            int(num_sms if num_sms is not None else c["num_sms"]), impl, stream)
        return rc

    def result(self, c, tdt):
        """(16-bit slice as float64 [B*T_out, H, W, n], fp32 columns as float64 [.., n_f32]) of the last call."""
        oo, n = c["out_off"], c["n_total"]
        y = self.out[1:-1, ..., oo:oo + n].view(tdt).double()
        f = self.f32[1:-1, ..., c["f32_off"]:c["f32_off"] + c["n_f32"]].view(torch.float32).double()
        return y, f

    def check_guards(self, c):
        """Bits outside the slice unchanged; no sentinel left inside it (the 16-bit cells of the fp32 columns are not
        written: they keep what they held)."""
        oo, n, nf = c["out_off"], c["n_total"], c["n_f32"] if c["ext"] == 2 else 0
        now, was = self.out, self.before
        assert torch.equal(now[0], was[0]) and torch.equal(now[-1], was[-1]), "store into a guard image"
        assert torch.equal(now[1:-1, ..., :oo], was[1:-1, ..., :oo]), "store before the output slice"
        assert torch.equal(now[1:-1, ..., oo + n:], was[1:-1, ..., oo + n:]), "store after the output slice"
        assert torch.equal(now[1:-1, ..., oo:oo + nf], was[1:-1, ..., oo:oo + nf]), "16-bit store of an fp32 column"
        body = now[1:-1, ..., oo + nf:oo + n]
        if c["res"] != "inplace":
            left = int((body == self.sent).sum())
            assert left == 0, f"{left} output cells never written"
        fo, fp = c["f32_off"], c["f32_pitch"]
        f, fw = self.f32, torch.full_like(self.f32, SENT32)
        assert torch.equal(f[0], fw[0]) and torch.equal(f[-1], fw[-1]), "fp32 store into a guard image"
        assert torch.equal(f[1:-1, ..., :fo], fw[1:-1, ..., :fo]), "fp32 store before the fp32 slice"
        assert torch.equal(f[1:-1, ..., fo + nf:], fw[1:-1, ..., fo + nf:]), "fp32 store outside the fp32 columns"
        if nf:
            left = int((f[1:-1, ..., fo:fo + nf] == SENT32).sum())
            assert left == 0, f"{left} fp32 cells never written"


def reference(c, inp, tdt):
    """(y^, S) float64 NHWC [B*T_out, H, W, n_total] on the inputs' device."""
    dev = inp.s0.device
    k, kt, n = c["ksize"], c["kt"], c["n_total"]
    x = inp.s0[..., c["off0"]:c["off0"] + c["c0"]]
    if inp.s1 is not None:
        x = torch.cat([x, inp.s1[..., c["off1"]:c["off1"] + c["c1"]]], -1)
    x = x.double().permute(0, 3, 1, 2)
    py = c["pad_before"] if c["pad_before"] >= 0 else (k - 1) // 2
    px = c["pad_before_x"] if c["pad_before_x"] >= 0 else py
    x = F.pad(x, (px, k - 1 - px, py, k - 1 - py))
    w = inp.w.to(tdt).double().to(dev).view(n, kt, k, k, -1).permute(0, 1, 4, 2, 3)
    B, T_in, T_out = c["B"], c["T_in"], c["T_out"]
    acc = torch.zeros(B * T_out, n, c["H"], c["W"], dtype=torch.float64, device=dev)
    S = torch.zeros_like(acc)
    for dt in range(kt):
        o_idx, i_idx = [], []
        for b in range(B * T_out):
            s, t = divmod(b, T_out)
            pl = t + dt - c["pad_t"]
            if 0 <= pl < T_in:
                o_idx.append(b)
                i_idx.append(s * T_in + pl)
        if not o_idx:
            continue
        xi = x[torch.tensor(i_idx, device=dev)]
        o = torch.tensor(o_idx, device=dev)
        acc[o] += F.conv2d(xi, w[:, dt])
        S[o] += F.conv2d(xi.abs(), w[:, dt].abs())
    sh = inp.shift.double().to(dev).view(1, n, 1, 1)
    v = (acc + sh).permute(0, 2, 3, 1)
    S = (S + sh.abs()).permute(0, 2, 3, 1)
    res = inp.res.double() if inp.res is not None else None
    if c["ext"] == 0:
        y = F.leaky_relu(v, 0.2) if c["act"] else v
    elif c["ext"] == 1:
        a = float(torch.tensor(c["slope"], dtype=torch.float32))
        y = torch.where(v > 0, v, a * v)
        S = S * max(1.0, abs(a))
        if res is not None:
            y = y + res
            S = S + res.abs()
    else:
        if res is not None:
            v = v + res
            S = S + res.abs()
        a = inp.slopes.double().to(dev)
        y = torch.where(v > 0, v, a * v)
        S = S * a.abs().clamp(min=1.0)
    return y, S


def worst_ratio(got, ref, S, K, tdt):
    """max over elements of |got - ref| / bound, and where (b, y, x, c); NaN anywhere gives inf."""
    err = (got - ref).abs()
    bound = 2.0 * K * U32 * S
    if tdt is not None:
        bound = bound + _ulp(ref, tdt)
    ratio = err / bound
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    if ratio.numel() == 0:
        return 0.0, ()
    i = int(torch.argmax(ratio))
    at = []
    for d in reversed(ratio.shape):
        at.append(i % d)
        i //= d
    return float(ratio.max()), tuple(reversed(at))


def check_case(L, c, tdt, dev, impl, seed=0, num_sms=None, stream=None, determinism=False):
    """Run one case, check guards and the per-element bound; returns {ratio16, ratio32}."""
    inp = Inputs(c, tdt, dev, seed)
    if num_sms is None and isinstance(c["num_sms"], str):   # "nsplit" / "2nsplit+1": CTAs walk many passes
        ns = plan(L, c)["nsplit"]
        num_sms = ns if c["num_sms"] == "nsplit" else 2 * ns + 1
    rc = inp.call(L, c, tdt, impl, num_sms, stream)
    assert rc == 0, (c["name"], rc, L.vfi_last_error())
    inp.check_guards(c)
    y, f = inp.result(c, tdt)
    ref, S = reference(c, inp, tdt)
    K = c["kt"] * c["ksize"] ** 2 * (c["c0"] + c["c1"])
    nf = c["n_f32"] if c["ext"] == 2 else 0
    r16, at16 = worst_ratio(y[..., nf:], ref[..., nf:], S[..., nf:], K, tdt)
    assert r16 <= 1.0, f"{c['name']}: 16-bit columns: error / bound {r16:.3f} at (b,y,x,c-{nf}) {at16}"
    r32 = 0.0
    if nf:
        r32, at32 = worst_ratio(f, ref[..., :nf], S[..., :nf], K, None)
        assert r32 <= 1.0, f"{c['name']}: fp32 columns: error / bound {r32:.3f} at (b,y,x,c) {at32}"
    if determinism and c["res"] != "inplace":
        first, first32 = inp.out.clone(), inp.f32.clone()
        assert inp.call(L, c, tdt, impl, num_sms, stream) == 0, L.vfi_last_error()
        assert torch.equal(first, inp.out) and torch.equal(first32, inp.f32), f"{c['name']}: two runs differ (a race)"
    return dict(ratio16=r16, ratio32=r32)


def check_refusal(L, c, tdt, dev, impl, why):
    """The launch is refused with the text `why` and nothing is written (the same checks stand before either kernel)."""
    inp = Inputs(c, tdt, dev, 0)
    rc = inp.call(L, c, tdt, impl)
    msg = L.vfi_last_error().decode()
    assert rc != 0, c["name"]
    assert why in msg, (c["name"], msg)
    assert torch.equal(inp.out, inp.before), f"{c['name']}: refused, yet the output changed"
    assert bool((inp.f32 == SENT32).all()), f"{c['name']}: refused, yet the fp32 output changed"
