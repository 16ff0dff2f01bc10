"""-m gpu: every kernel of the path, through the C ABI, against the CPU oracle's operator on the same inputs.

Bounds: the tensor-core kernels take 16-bit operands (fp16 or bf16) and accumulate in fp32.  The reference y^ is the same
operator in float64 on the SAME 16-bit inputs and the SAME packed weights as the library (round_T(w); ResConv:
round_T(w*beta) with the shift b*beta, csrc/rife46.cu conv2d with beta), so only accumulation order and the output store
differ.  With K products per output and S = conv(|x|, |w|) + |shift| + |residual|, every element satisfies
    16-bit outputs:  |y - y^| <= ulp_T(y^) + 2 K 2^-24 S
    fp32 outputs:    |y - y^| <= 2 K 2^-24 S
(K u S is the classical bound of a K-term fp32 sum with unit roundoff u = 2^-24; the factor 2 leaves room for a
tensor-core adder that does not round to nearest).  A failure names the worst element (b, y, x, c) and its error / bound.
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import s2d, un_s2d, nhwc, nchw
from oracle import rife46 as O

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64)
U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(7)
    e = {"float16": Rife46Engine(sd, 0, "float16"), "bfloat16": Rife46Engine(sd, 0, "bfloat16")}
    yield sd, e
    for v in e.values():
        v.close()


def _tdt(dtype):
    return torch.float16 if dtype == "float16" else torch.bfloat16


def _rw(sd, name, dtype):
    """A weight as the library packs it: rounded to the operand type, here widened to float64."""
    return O.q16(sd[name], _tdt(dtype)).double()


def _ulp(y, tdt):
    """ulp of the 16-bit type tdt at |y| (subnormal spacing below its smallest normal)."""
    mant, emin = (10, -14) if tdt == torch.float16 else (7, -126)
    _, e = torch.frexp(y.abs())
    e = torch.where(y == 0, torch.full_like(e, emin), e - 1).clamp(min=emin)
    return torch.ldexp(torch.ones_like(y), e - mant)


def _assert_bound(label, got, ref, S, K, tdt=None):
    """|got - ref| <= [ulp_tdt(ref)] + 2 K 2^-24 S element-wise over NHWC tensors (tdt None: fp32 output)."""
    err = (got.double().cpu() - ref).abs()
    bound = 2.0 * K * U32 * S
    if tdt is not None:
        bound = bound + _ulp(ref, tdt)
    ratio = err / bound
    i = int(torch.argmax(ratio))
    at = []
    for d in reversed(ratio.shape):
        at.append(i % d)
        i //= d
    at = tuple(reversed(at))
    worst = float(ratio.max())
    print(f"{label}: max |err| {float(err.max()):.3e}, worst error / bound {worst:.3f} at (b,y,x,c) {at}")
    assert worst <= 1.0, (f"{label}: |err| {float(err[at]):.3e} > bound {float(bound[at]):.3e} at (b,y,x,c) {at} "
                          f"(error / bound {worst:.3f})")


def _lrelu(v):
    return F.leaky_relu(v, O.LRELU_SLOPE)


def _resconv_ref(sd, q, x, dtype):
    """(y^, S) of ResConv q on the 16-bit input x (NHWC), as the library computes it."""
    w, shift = O.resconv_packed(sd, q, _tdt(dtype))
    xd = nchw(x.double())
    y = _lrelu(F.conv2d(xd, w, shift, padding=1) + xd)
    S = F.conv2d(xd.abs(), w.abs(), shift.abs(), padding=1) + xd.abs()
    return nhwc(y), nhwc(S)


def _conv_s2_ref(sd, p, x, dtype):
    """(y^, S) of conv0.x ``p`` (stride 2, + LeakyReLU) on the 16-bit NHWC input x (its real channels only)."""
    w, b = _rw(sd, p + "weight", dtype), sd[p + "bias"].double()
    xd = nchw(x.double())
    y = _lrelu(F.conv2d(xd, w, b, stride=2, padding=1))
    S = F.conv2d(xd.abs(), w.abs(), b.abs(), stride=2, padding=1)
    return nhwc(y), nhwc(S)


def _lastconv_ref(sd, p, x, dtype):
    """(tmp^, S) of ConvTranspose2d(c, n, 4, 2, 1) + PixelShuffle(2), NCHW, on the 16-bit NHWC input x."""
    w, b = _rw(sd, p + "weight", dtype), sd[p + "bias"].double()
    xd = nchw(x.double())
    y = F.pixel_shuffle(F.conv_transpose2d(xd, w, b, stride=2, padding=1), 2)
    S = F.pixel_shuffle(F.conv_transpose2d(xd.abs(), w.abs(), b.abs(), stride=2, padding=1), 2)
    return y, S


def test_warp_primitive(engines):
    sd, e = engines
    eng = e["float16"]
    g = torch.Generator().manual_seed(0)
    for c in (3, 4, 8):
        img = torch.rand(2, 37, 53, c, generator=g)
        flow = 9 * torch.randn(2, 37, 53, 2, generator=g)
        out = eng.warp(img.cuda(), flow.cuda()).cpu()
        ref = nhwc(O.warp(nchw(img), nchw(flow)))
        assert (out - ref).abs().max().item() < 3e-5  # the reference's normalise/denormalise rounding


IMPLS = [pytest.param(1, id="ref"), pytest.param(0, id="tc")]  # CUDA-core checker / wgmma kernel
# (impl, dtype) pairs: the wgmma kernel in both operand types, the CUDA-core checker in one (no skipped combinations)
IMPL_DTYPE = [pytest.param(1, "float16", id="ref-float16"), pytest.param(0, "float16", id="tc-float16"),
              pytest.param(0, "bfloat16", id="tc-bfloat16")]


@pytest.mark.parametrize("block", [3, 2, 1, 0])
@pytest.mark.parametrize("impl,dtype", IMPL_DTYPE)
def test_resconv(engines, block, dtype, impl):
    sd, e = engines
    eng, c, tdt = e[dtype], BLOCK_C[block], _tdt(dtype)
    g = torch.Generator().manual_seed(block)
    x = (0.5 * torch.randn(2, 21, 29, c, generator=g)).to(tdt)  # partial tiles in both directions
    for j in (0, 5):
        q = f"block{block}.convblock.{j}."
        out = torch.empty_like(x, device="cuda")
        eng.debug_layer(block, 2 + j, x.cuda(), out, impl=impl)
        ref, S = _resconv_ref(sd, q, x, dtype)
        _assert_bound(f"block {block} ResConv {j}", out, ref, S, 9 * c, tdt)


@pytest.mark.parametrize("block", [3, 1, 0])
def test_resconv_many_tiles(engines, block):
    """More tiles than persistent CTAs: every CTA walks several tiles, so the window stages, both MMA warpgroups' tiles
    and all mbarrier phases wrap several times (blocks 0 and 1 stream their weights: the weight slots wrap too)."""
    sd, e = engines
    eng, c = e["float16"], BLOCK_C[block]
    g = torch.Generator().manual_seed(40 + block)
    x = (0.5 * torch.randn(3, 203, 181, c, generator=g)).half()
    q = f"block{block}.convblock.3."
    out = torch.empty_like(x, device="cuda")
    eng.debug_layer(block, 2 + 3, x.cuda(), out, impl=0)
    ref, S = _resconv_ref(sd, q, x, "float16")
    _assert_bound(f"block {block} ResConv 3, 3 x 203 x 181", out, ref, S, 9 * c, torch.float16)


@pytest.mark.parametrize("block", [3, 1, 0])
@pytest.mark.parametrize("impl,dtype", IMPL_DTYPE)
def test_conv0(engines, block, dtype, impl):
    """conv0.0 then conv0.1 (both stride 2) on space-to-depth inputs."""
    sd, e = engines
    eng, c, tdt = e[dtype], BLOCK_C[block], _tdt(dtype)
    cin = 7 if block == 0 else 12
    g = torch.Generator().manual_seed(10 + block)
    hs, ws = 40, 56  # block-input grid; conv0.0 grid 20x28, conv0.1 grid 10x14
    x = torch.zeros(2, hs, ws, 16)
    x[..., :cin] = torch.randn(2, hs, ws, cin, generator=g)
    x = x.to(tdt)
    p = f"block{block}."
    # conv0.0: reads s2d(x) [2,20,28,64], writes s2d form of its [2,20,28,c/2] output = [2,10,14,2c]
    y0 = torch.empty(2, hs // 4, ws // 4, 2 * c, dtype=tdt, device="cuda")
    eng.debug_layer(block, 0, s2d(x).cuda(), y0, impl=impl)
    ref0, S0 = _conv_s2_ref(sd, p + "conv0.0.0.", x[..., :cin], dtype)
    got0 = un_s2d(y0.cpu(), c // 2)
    _assert_bound(f"block {block} conv0.0", got0, ref0, S0, 9 * cin, tdt)
    # conv0.1 on the oracle's (rounded) conv0.0 output
    x1 = ref0.to(tdt)
    y1 = torch.empty(2, hs // 4, ws // 4, c, dtype=tdt, device="cuda")
    eng.debug_layer(block, 1, s2d(x1).cuda(), y1, impl=impl)
    ref1, S1 = _conv_s2_ref(sd, p + "conv0.1.0.", x1, dtype)
    _assert_bound(f"block {block} conv0.1", y1, ref1, S1, 9 * (c // 2), tdt)


@pytest.mark.parametrize("block", [3, 2, 1, 0])
@pytest.mark.parametrize("impl,dtype", IMPL_DTYPE)
def test_lastconv(engines, block, dtype, impl):
    """ConvTranspose2d(c,24,4,2,1)+PixelShuffle(2) as one 3x3 tap conv producing 4x4 sub-pixel patches."""
    sd, e = engines
    eng, c, tdt = e[dtype], BLOCK_C[block], _tdt(dtype)
    g = torch.Generator().manual_seed(20 + block)
    x = (0.5 * torch.randn(2, 19, 13, c, generator=g)).to(tdt)
    p = f"block{block}."
    flow = torch.full((2, 76, 52, 4), float("nan"), device="cuda")
    mask = torch.full((2, 76, 52), float("nan"), device="cuda")
    eng.debug_layer(block, 10, x.cuda(), flow, out_mask=mask, impl=impl)
    tmp, S = _lastconv_ref(sd, p + "lastconv.0.", x, dtype)
    # fp32 outputs; K = the 9 taps x c products the kernel's 3x3 form of the transposed conv accumulates
    _assert_bound(f"block {block} lastconv flow", flow, nhwc(tmp[:, :4]), nhwc(S[:, :4]), 9 * c)
    _assert_bound(f"block {block} lastconv mask", mask.unsqueeze(-1), nhwc(tmp[:, 4:5]), nhwc(S[:, 4:5]), 9 * c)


def test_layer_plans(engines):
    sd, e = engines
    eng = e["float16"]
    for b in range(4):
        for l in range(11):
            pl = eng.layer_plan(b, l)
            assert pl["stages"] >= 1 and pl["smem_bytes"] <= 232448, (b, l, pl)


# ---- arch 4.26 (rife426.pth): the fifth block (c = 32: a single 32-channel k-block), the 52-channel lastconv split in
# ---- its flow + mask part (layer 10) and its 8 feature channels (layer 11, [B, 4H, 4W, 8] 16-bit), every block width
BLOCK_C426 = (192, 128, 96, 64, 32)


@pytest.fixture(scope="module")
def engines426(pkg):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(17, arch="4.26")
    e = {"float16": Rife46Engine(sd, 0, "float16"), "bfloat16": Rife46Engine(sd, 0, "bfloat16")}
    yield sd, e
    for v in e.values():
        v.close()


@pytest.mark.parametrize("impl,dtype", IMPL_DTYPE)
def test_block4_resconv_and_conv0(engines426, dtype, impl):
    sd, e = engines426
    eng, c, tdt = e[dtype], 32, _tdt(dtype)
    g = torch.Generator().manual_seed(77)
    x = (0.5 * torch.randn(2, 37, 29, c, generator=g)).to(tdt)
    q = "block4.convblock.2."
    out = torch.empty_like(x, device="cuda")
    eng.debug_layer(4, 2 + 2, x.cuda(), out, impl=impl)
    ref, S = _resconv_ref(sd, q, x, dtype)
    _assert_bound("block 4 ResConv 2", out, ref, S, 9 * c, tdt)
    # conv0.0 (28 real of 32 channels -> 16) and conv0.1 (16 -> 32), both stride 2 on space-to-depth inputs
    hs, ws = 40, 56
    xi = torch.zeros(2, hs, ws, 32)
    xi[..., :28] = torch.randn(2, hs, ws, 28, generator=g)
    xi = xi.to(tdt)
    y0 = torch.empty(2, hs // 4, ws // 4, 4 * 16, dtype=tdt, device="cuda")
    eng.debug_layer(4, 0, s2d(xi).cuda(), y0, impl=impl)
    ref0, S0 = _conv_s2_ref(sd, "block4.conv0.0.0.", xi[..., :28], dtype)
    _assert_bound("block 4 conv0.0", un_s2d(y0.cpu(), 16), ref0, S0, 9 * 28, tdt)
    x1 = ref0.to(tdt)
    y1 = torch.empty(2, hs // 4, ws // 4, 32, dtype=tdt, device="cuda")
    eng.debug_layer(4, 1, s2d(x1).cuda(), y1, impl=impl)
    ref1, S1 = _conv_s2_ref(sd, "block4.conv0.1.0.", x1, dtype)
    _assert_bound("block 4 conv0.1", y1, ref1, S1, 9 * 16, tdt)


@pytest.mark.parametrize("block", [4, 3, 2, 1, 0])
@pytest.mark.parametrize("impl,dtype", IMPL_DTYPE)
def test_lastconv426(engines426, block, dtype, impl):
    """ConvTranspose2d(c,52,4,2,1)+PixelShuffle(2): channels 0-4 (flow, mask) as fp32 planes, 5-12 (features) as a
    16-bit [B,4H,4W,8] tensor from a second tap conv over the same input."""
    sd, e = engines426
    eng, c, tdt = e[dtype], BLOCK_C426[block], _tdt(dtype)
    g = torch.Generator().manual_seed(120 + block)
    x = (0.5 * torch.randn(2, 19, 13, c, generator=g)).to(tdt)
    p = f"block{block}."
    tmp, S = _lastconv_ref(sd, p + "lastconv.0.", x, dtype)
    assert tmp.shape[1] == 13
    flow = torch.full((2, 76, 52, 4), float("nan"), device="cuda")
    mask = torch.full((2, 76, 52), float("nan"), device="cuda")
    eng.debug_layer(block, 10, x.cuda(), flow, out_mask=mask, impl=impl)
    _assert_bound(f"block {block} lastconv flow", flow, nhwc(tmp[:, :4]), nhwc(S[:, :4]), 9 * c)
    _assert_bound(f"block {block} lastconv mask", mask.unsqueeze(-1), nhwc(tmp[:, 4:5]), nhwc(S[:, 4:5]), 9 * c)
    if block < 4:  # the last block's features are never used (rife_arch.py:563-587): no such layer
        feat = torch.full((2, 76, 52, 8), float("nan"), dtype=tdt, device="cuda")
        eng.debug_layer(block, 11, x.cuda(), feat, impl=impl)
        _assert_bound(f"block {block} lastconv features", feat, nhwc(tmp[:, 5:]), nhwc(S[:, 5:]), 9 * c, tdt)
    else:
        from cfi_b200._lib import VfiError
        with pytest.raises(VfiError):
            eng.debug_layer(block, 11, x.cuda(), torch.empty(2, 76, 52, 8, dtype=tdt, device="cuda"), impl=impl)


def test_layer_plans426(engines426):
    sd, e = engines426
    eng = e["float16"]
    for b in range(5):
        for l in range(12 if b < 4 else 11):
            pl = eng.layer_plan(b, l)
            assert pl["stages"] >= 1 and pl["smem_bytes"] <= 232448, (b, l, pl)
