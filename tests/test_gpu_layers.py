"""-m gpu: every kernel of the path, through the C ABI, against the CPU oracle's operator on the same inputs.

Tolerances: the tensor-core kernels take 16-bit operands (fp16 or bf16) and accumulate in fp32; the oracle side
is evaluated in fp32 on the SAME 16-bit-rounded inputs and weights, so what is compared is the algorithm
(taps, padding, packing, epilogue), not the operand rounding.  Remaining differences: fp32 accumulation order
and the 16-bit rounding of the stored output -> max relative error <= 4e-3 (fp16) / 2e-2 (bf16).
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import s2d, un_s2d, nhwc, nchw, rel_err
from oracle import rife46 as O

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64)


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


def _tol(dtype):
    return 4e-3 if dtype == "float16" else 2e-2


def _rw(sd, name, dtype):
    return sd[name].to(_tdt(dtype)).float()


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
        ref = nhwc(O.resconv(nchw(x.float()), _rw(sd, q + "conv.weight", dtype), sd[q + "conv.bias"], sd[q + "beta"]))
        assert rel_err(out.cpu().float(), ref) < _tol(dtype)


@pytest.mark.parametrize("block", [3, 1, 0])
def test_resconv_many_tiles(engines, block):
    """More tiles than persistent CTAs: every CTA walks several tiles, so the window stages / ring slots, both MMA warpgroups'
    tiles and all mbarrier phases wrap several times (blocks 0 and 1 run the k-block ring pipeline)."""
    sd, e = engines
    eng, c = e["float16"], BLOCK_C[block]
    g = torch.Generator().manual_seed(40 + block)
    x = (0.5 * torch.randn(3, 203, 181, c, generator=g)).half()
    q = f"block{block}.convblock.3."
    out = torch.empty_like(x, device="cuda")
    eng.debug_layer(block, 2 + 3, x.cuda(), out, impl=0)
    ref = nhwc(O.resconv(nchw(x.float()), _rw(sd, q + "conv.weight", "float16"), sd[q + "conv.bias"], sd[q + "beta"]))
    assert rel_err(out.cpu().float(), ref) < _tol("float16")


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
    ref0 = nhwc(O.conv_lrelu(nchw(x[..., :cin].float()), _rw(sd, p + "conv0.0.0.weight", dtype),
                             sd[p + "conv0.0.0.bias"], 2))
    got0 = un_s2d(y0.cpu(), c // 2)
    assert rel_err(got0.float(), ref0) < _tol(dtype)
    # conv0.1 on the oracle's (rounded) conv0.0 output
    x1 = ref0.to(tdt)
    y1 = torch.empty(2, hs // 4, ws // 4, c, dtype=tdt, device="cuda")
    eng.debug_layer(block, 1, s2d(x1).cuda(), y1, impl=impl)
    ref1 = nhwc(O.conv_lrelu(nchw(x1.float()), _rw(sd, p + "conv0.1.0.weight", dtype), sd[p + "conv0.1.0.bias"], 2))
    assert rel_err(y1.cpu().float(), ref1) < _tol(dtype)


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
    tmp = F.pixel_shuffle(F.conv_transpose2d(nchw(x.float()), _rw(sd, p + "lastconv.0.weight", dtype),
                                             sd[p + "lastconv.0.bias"], stride=2, padding=1), 2)
    assert rel_err(flow.cpu(), nhwc(tmp[:, :4])) < 1e-4   # fp32 outputs: only accumulation order differs
    assert rel_err(mask.cpu(), tmp[:, 4]) < 1e-4


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
    ref = nhwc(O.resconv(nchw(x.float()), _rw(sd, q + "conv.weight", dtype), sd[q + "conv.bias"], sd[q + "beta"]))
    assert rel_err(out.cpu().float(), ref) < _tol(dtype)
    # conv0.0 (28 real of 32 channels -> 16) and conv0.1 (16 -> 32), both stride 2 on space-to-depth inputs
    hs, ws = 40, 56
    xi = torch.zeros(2, hs, ws, 32)
    xi[..., :28] = torch.randn(2, hs, ws, 28, generator=g)
    xi = xi.to(tdt)
    y0 = torch.empty(2, hs // 4, ws // 4, 4 * 16, dtype=tdt, device="cuda")
    eng.debug_layer(4, 0, s2d(xi).cuda(), y0, impl=impl)
    ref0 = nhwc(O.conv_lrelu(nchw(xi[..., :28].float()), _rw(sd, "block4.conv0.0.0.weight", dtype),
                             sd["block4.conv0.0.0.bias"], 2))
    assert rel_err(un_s2d(y0.cpu(), 16).float(), ref0) < _tol(dtype)
    x1 = ref0.to(tdt)
    y1 = torch.empty(2, hs // 4, ws // 4, 32, dtype=tdt, device="cuda")
    eng.debug_layer(4, 1, s2d(x1).cuda(), y1, impl=impl)
    ref1 = nhwc(O.conv_lrelu(nchw(x1.float()), _rw(sd, "block4.conv0.1.0.weight", dtype), sd["block4.conv0.1.0.bias"], 2))
    assert rel_err(y1.cpu().float(), ref1) < _tol(dtype)


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
    tmp = F.pixel_shuffle(F.conv_transpose2d(nchw(x.float()), _rw(sd, p + "lastconv.0.weight", dtype),
                                             sd[p + "lastconv.0.bias"], stride=2, padding=1), 2)
    assert tmp.shape[1] == 13
    flow = torch.full((2, 76, 52, 4), float("nan"), device="cuda")
    mask = torch.full((2, 76, 52), float("nan"), device="cuda")
    eng.debug_layer(block, 10, x.cuda(), flow, out_mask=mask, impl=impl)
    assert rel_err(flow.cpu(), nhwc(tmp[:, :4])) < 1e-4
    assert rel_err(mask.cpu(), tmp[:, 4]) < 1e-4
    if block < 4:  # the last block's features are never used (rife_arch.py:563-587): no such layer
        feat = torch.full((2, 76, 52, 8), float("nan"), dtype=tdt, device="cuda")
        eng.debug_layer(block, 11, x.cuda(), feat, impl=impl)
        assert rel_err(feat.cpu().float(), nhwc(tmp[:, 5:])) < _tol(dtype)
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
